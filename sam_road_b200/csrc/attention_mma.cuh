// sam_road_b200 :: tensor-core encoder attention (head_dim 64 or 80), windowed or global, with the
// decomposed relative-position bias.  Same semantics as the SIMT kernel in attention.cu.
//
// Unit = (image, window, head).  Its real queries (the window's tokens inside the s x s grid, ry x rx
// of them) are numbered j = qh * rx + qw and cut into 16-row m-tiles, one per warp at a time, so edge
// windows run only the rows they have.  Three kernels run the same tile math and differ in who owns
// what:
//   attention_unit_kernel : window blocks (win < s) whose whole window fits in shared memory twice
//              per SM.  One CTA per unit: K, V and the tables are staged once, and the CTA's warps
//              walk the unit's m-tiles (tile = warp, warp + NW, ...).  After the one barrier that
//              publishes K/V, a warp touches only its own scratch rows, so tiles need __syncwarp only.
//   attention_wide_kernel : one window per image (global blocks, a window larger than the grid).  A
//              unit is cut into CTAs of 2 * kAmWarps m-tiles, two per warp, so that every K and V
//              fragment read from shared memory feeds two MMAs; each CTA streams the unit's K/V in
//              double-buffered chunks.
//   attention_mma_kernel  : windows too large to be resident.  As the wide kernel with one m-tile per
//              warp; a CTA past the unit's last tile exits at once.  It keeps its own copy of the
//              tile math (it predates the shared helpers and is left as measured).
// Keys sit in slots k = kh * winP + kw, winP = win rounded up to a power of two
// (>= 8): a 64-key chunk then holds whole key rows, kh = k >> lg and kw = k & (winP - 1) need no
// division, and each n8 tile of scores lies in one key row.
//   prologue : Q tile (fp16) and the rel-pos tables, each fp32 row R split into fp16 hi = fp16(R)
//              and lo = fp16(R - hi) -> smem.  M = Q [hi | lo]^T on mma.sync (both into one fp32
//              accumulator; q is exactly fp16, so this is the fp32 dot product to ~1e-6 relative),
//              and M[q][r] goes to relh[q][kh] with kh = qh - r + win - 1 (relw with qw alike)
//              -> smem, in the exp2 domain.  Entries for kh >= win or kw >= win (slots that are no
//              key of the window) hold -inf, which masks those slots in the bias add.
//   main loop: 64-key chunks of K and V (fp16), loaded with cp.async (streamed: double-buffered, one
//              barrier per chunk); window padding keys (beyond the s x s grid) are copies of the
//              fp16 qkv bias, non-key slots are zeros.  S = Q K^T on mma.sync m16n8k16 (fp32
//              accumulate), S * scale + relh[kh] + relw[kw], online softmax in the exp2 domain, P
//              rounded to fp16 and fed from registers into O += P V (V fragments by ldmatrix.trans).
//              A last chunk with no key in its upper half skips that half's MMAs.
//   epilogue : O / l -> fp16, real query tokens only
// Padded tokens of a window (beyond the s x s grid) have x = 0, so their q = k = v = qkv bias: they
// are real softmax keys, and their query rows are never computed.
#pragma once

#include "common.cuh"
#include "ops.h"

namespace srb {

constexpr int kAmWarps = 4;       // warps per CTA, one 16-row m-tile each
constexpr int kAmKC = 64;         // key slots per chunk

template <int HD>
struct AmLayout {
  static constexpr int kRows = 16 * kAmWarps;                      // query rows per CTA
  static constexpr int kPitch = HD + 8;                         // halves; ldmatrix rows conflict-free
  static constexpr int kQBytes = kRows * kPitch * 2;
  static constexpr int kStageBytes = 2 * kAmKC * kPitch * 2;    // K and V of one chunk
  int winP, lg;                   // key-row pitch (power of two >= 8) and its log2
  int nslots, nchunks;
  int relH, relPitch;             // relh columns (whole chunks, padded), row pitch of sRel in floats
  int tabRows;                    // 2 * win - 1 table rows, padded to n8 tiles
  int relOffset, padOffset, bytes;                // streamed kernel
  int kvSlots, uTabOffset, uWarpOffset, uWarpBytes;   // one-CTA-per-unit kernel: [K | V | tables | warp scratch]
  int kvBytes;                                    // the streamed kernels' 2 stages of K, V (or the tables)
  // streamed kernel with two m-tiles per warp: [Q 2 kRows | stages | rel 2 kRows | pad]
  __host__ __device__ int wide_rel_offset() const { return 2 * kQBytes + kvBytes; }
  __host__ __device__ int wide_pad_offset() const { return wide_rel_offset() + 2 * kRows * relPitch * 4; }
  __host__ __device__ int wide_bytes() const { return wide_pad_offset() + 2 * HD * 2; }
  __host__ __device__ int unit_bytes(int nwarps) const { return uWarpOffset + nwarps * uWarpBytes; }
  __host__ __device__ explicit AmLayout(int win) {
    winP = 8; lg = 3;
    while (winP < win) { winP <<= 1; ++lg; }
    nslots = win * winP;
    nchunks = (nslots + kAmKC - 1) / kAmKC;
    relH = ((nchunks * kAmKC / winP + 7) / 8) * 8;
    relPitch = ((relH + winP - 8 + 31) / 32) * 32 + 8;          // = 8 mod 32: float2 row reads in 2 wavefronts
    tabRows = ((2 * win - 1 + 7) / 8) * 8;
    const int tab = 4 * tabRows * kPitch * 2;                   // [h hi | h lo | w hi | w lo]
    const int kv = tab > 2 * kStageBytes ? tab : 2 * kStageBytes;
    kvBytes = kv;
    relOffset = kQBytes + kv;
    padOffset = relOffset + kRows * relPitch * 4;
    bytes = padOffset + 2 * HD * 2;
    kvSlots = ((nslots + kAmKC / 2 - 1) / (kAmKC / 2)) * (kAmKC / 2);   // a keyless upper half chunk is never read
    uTabOffset = 2 * kvSlots * kPitch * 2;
    uWarpOffset = uTabOffset + tab;
    const int q = 16 * kPitch * 2, rel = 16 * relPitch * 4;     // a warp's Q tile, then its relh | relw rows
    uWarpBytes = q > rel ? q : rel;
  }
};

__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x2(uint32_t addr, uint32_t& r0, uint32_t& r1) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x2.shared.b16 {%0, %1}, [%2];" : "=r"(r0), "=r"(r1) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x2_trans(uint32_t addr, uint32_t& r0, uint32_t& r1) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x2.trans.shared.b16 {%0, %1}, [%2];"
               : "=r"(r0), "=r"(r1) : "r"(addr));
}
// D[16x8] += A[16x16] * B[16x8], fp16 operands, fp32 accumulate
__device__ __forceinline__ void mma_16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
      "{%0, %1, %2, %3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }

__device__ __forceinline__ uint4 am_bias8(const float* __restrict__ bp) {
  uint4 u;
  u.x = pack_half2(__ldg(bp + 0), __ldg(bp + 1));
  u.y = pack_half2(__ldg(bp + 2), __ldg(bp + 3));
  u.z = pack_half2(__ldg(bp + 4), __ldg(bp + 5));
  u.w = pack_half2(__ldg(bp + 6), __ldg(bp + 7));
  return u;
}

// Both rel-pos tables as fp16 [h hi | h lo | w hi | w lo], each padded with zero rows to TR.
template <int HD, int NTH>
__device__ __forceinline__ void am_stage_tables(__half* sTab, const float* __restrict__ rel_h,
                                                const float* __restrict__ rel_w, int win, int TR, int tid) {
  constexpr int P = AmLayout<HD>::kPitch;
  const int L = 2 * win - 1;
  for (int idx = tid; idx < 2 * TR * (HD / 2); idx += NTH) {
    const int t = idx / (TR * (HD / 2)), rem = idx - t * TR * (HD / 2);
    const int r = rem / (HD / 2), c = 2 * (rem - r * (HD / 2));
    float2 v = make_float2(0.f, 0.f);
    if (r < L) v = __ldg(reinterpret_cast<const float2*>((t ? rel_w : rel_h) + r * HD + c));
    const __half2 hi = __float22half2_rn(v);
    const float2 hf = __half22float2(hi);
    const __half2 lo = __float22half2_rn(make_float2(v.x - hf.x, v.y - hf.y));
    __half* dst = sTab + (2 * t * TR + r) * P + c;
    *reinterpret_cast<__half2*>(dst) = hi;
    *reinterpret_cast<__half2*>(dst + TR * P) = lo;
  }
}

// Rel-pos of one m-tile on the tensor cores: relh[q][kh] = q . Rh[qh - kh + win - 1], relw alike, into
// the thread's two rows dA and dA + 8 * RP (queries jA, jB of the unit), in the exp2 domain.
template <int HD>
__device__ __forceinline__ void am_relpos(const uint32_t (&qa)[HD / 16][4], const __half* sTab, int TR, int win,
                                          int rx, int jA, int jB, float* dA0, int RP, int relH, int lane) {
  constexpr int P = AmLayout<HD>::kPitch;
  constexpr int KS = HD / 16;
  const int cq = 2 * (lane & 3);
  const int qhA = jA / rx, qhB = jB / rx;
  const int qwA = jA - qhA * rx, qwB = jB - qhB * rx;
#pragma unroll
  for (int t = 0; t < 2; ++t) {
    const __half* hi = sTab + 2 * t * TR * P;
    const __half* lo = hi + TR * P;
    const int cA = (t ? qwA : qhA) + win - 1, cB = (t ? qwB : qhB) + win - 1;
    float* dA = dA0 + (t ? relH : 0);
    float* dB = dA + 8 * RP;
    for (int nt = 0; nt < TR / 8; ++nt) {
      float acc[4] = {0.f, 0.f, 0.f, 0.f};
      const int boff = (nt * 8 + (lane & 7)) * P + ((lane >> 3) & 1) * 8;
#pragma unroll
      for (int k = 0; k < KS; ++k) {
        uint32_t b0, b1;
        ldsm_x2(smem_u32(hi + boff + k * 16), b0, b1);
        mma_16816(acc, qa[k], b0, b1);
        ldsm_x2(smem_u32(lo + boff + k * 16), b0, b1);
        mma_16816(acc, qa[k], b0, b1);
      }
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int r = nt * 8 + cq + e;
        const int khA = cA - r, khB = cB - r;
        if (static_cast<unsigned>(khA) < static_cast<unsigned>(win)) dA[khA] = acc[e] * 1.4426950408889634f;
        if (static_cast<unsigned>(khB) < static_cast<unsigned>(win)) dB[khB] = acc[2 + e] * 1.4426950408889634f;
      }
    }
  }
}

// Running softmax state of one m-tile in a warp: the thread's rows A (lane / 4) and B (A + 8).
template <int HD>
struct AmTile {
  float o[HD / 8][4];
  float mA, mB, lA, lB;
  __device__ __forceinline__ void reset() {
#pragma unroll
    for (int j = 0; j < HD / 8; ++j) o[j][0] = o[j][1] = o[j][2] = o[j][3] = 0.f;
    mA = mB = -INFINITY;
    lA = lB = 0.f;
  }
};

// One 64-slot chunk (slots k0 ..) of K (sK) and V (sV) against the warp's MT m-tiles: every K and V fragment
// read from shared memory feeds MT MMAs.  `full` is false when the chunk's upper 32 slots hold no key.
// rel[m]: the thread's [relh | relw] row A of tile m, row B at + 8 * RP.
template <int HD, int MT>
__device__ __forceinline__ void am_chunk(AmTile<HD> (&t)[MT], const uint32_t (&qa)[MT][HD / 16][4], const __half* sK,
                                         const __half* sV, int k0, bool full, const float* const (&rel)[MT], int RP,
                                         int relH, int lg, int winP, float scale_log2e, int lane) {
  constexpr int P = AmLayout<HD>::kPitch;
  constexpr int NT = HD / 8;
  constexpr int KS = HD / 16;
  const int cq = 2 * (lane & 3);
  // S = Q K^T : 16 rows x 64 keys per tile
  float sc[MT][kAmKC / 8][4];
#pragma unroll
  for (int n = 0; n < kAmKC / 8; ++n) {
#pragma unroll
    for (int m = 0; m < MT; ++m) sc[m][n][0] = sc[m][n][1] = sc[m][n][2] = sc[m][n][3] = 0.f;
    if (n < kAmKC / 16 || full) {
#pragma unroll
      for (int k = 0; k < KS; ++k) {
        uint32_t b0, b1;
        ldsm_x2(smem_u32(sK + (n * 8 + (lane & 7)) * P + k * 16 + ((lane >> 3) & 1) * 8), b0, b1);
#pragma unroll
        for (int m = 0; m < MT; ++m) mma_16816(sc[m][n], qa[m][k], b0, b1);
      }
    }
  }
  // scale + bias (-inf on non-key slots), row maxima, rescale of the running state
#pragma unroll
  for (int m = 0; m < MT; ++m) {
    const float* relA = rel[m];
    const float* relB = relA + 8 * RP;
    float cmA = -INFINITY, cmB = -INFINITY;
#pragma unroll
    for (int n = 0; n < kAmKC / 8; ++n) {
      const int kh = (k0 + n * 8) >> lg;           // one key row per n8 tile
      const int kw = (n * 8 + cq) & (winP - 1);
      const float hA = relA[kh], hB = relB[kh];
      const float2 wA = *reinterpret_cast<const float2*>(relA + relH + kw);
      const float2 wB = *reinterpret_cast<const float2*>(relB + relH + kw);
      sc[m][n][0] = fmaf(sc[m][n][0], scale_log2e, hA + wA.x);
      sc[m][n][1] = fmaf(sc[m][n][1], scale_log2e, hA + wA.y);
      sc[m][n][2] = fmaf(sc[m][n][2], scale_log2e, hB + wB.x);
      sc[m][n][3] = fmaf(sc[m][n][3], scale_log2e, hB + wB.y);
      cmA = fmaxf(cmA, fmaxf(sc[m][n][0], sc[m][n][1]));
      cmB = fmaxf(cmB, fmaxf(sc[m][n][2], sc[m][n][3]));
    }
#pragma unroll
    for (int off = 1; off <= 2; off <<= 1) {
      cmA = fmaxf(cmA, __shfl_xor_sync(0xffffffffu, cmA, off));
      cmB = fmaxf(cmB, __shfl_xor_sync(0xffffffffu, cmB, off));
    }
    const float nmA = fmaxf(t[m].mA, cmA), nmB = fmaxf(t[m].mB, cmB);
    const float alA = ex2_approx(t[m].mA - nmA), alB = ex2_approx(t[m].mB - nmB);   // first chunk: 2^-inf = 0
    t[m].mA = nmA; t[m].mB = nmB;
    t[m].lA *= alA; t[m].lB *= alB;
#pragma unroll
    for (int j = 0; j < NT; ++j) {
      t[m].o[j][0] *= alA; t[m].o[j][1] *= alA; t[m].o[j][2] *= alB; t[m].o[j][3] *= alB;
    }
  }
  // P (fp16) and O += P V, 16 keys per MMA
#pragma unroll
  for (int kc = 0; kc < kAmKC / 16; ++kc) {
    if (kc >= kAmKC / 32 && !full) continue;
    uint32_t pa[MT][4];
#pragma unroll
    for (int m = 0; m < MT; ++m) {
      float p[2][4];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int n = 2 * kc + h;
        p[h][0] = ex2_approx(sc[m][n][0] - t[m].mA);
        p[h][1] = ex2_approx(sc[m][n][1] - t[m].mA);
        p[h][2] = ex2_approx(sc[m][n][2] - t[m].mB);
        p[h][3] = ex2_approx(sc[m][n][3] - t[m].mB);
      }
      pa[m][0] = pack_half2(p[0][0], p[0][1]);
      pa[m][1] = pack_half2(p[0][2], p[0][3]);
      pa[m][2] = pack_half2(p[1][0], p[1][1]);
      pa[m][3] = pack_half2(p[1][2], p[1][3]);
      // the softmax denominator sums the same fp16-rounded P the MMA consumes
      const float2 f0 = __half22float2(*reinterpret_cast<const __half2*>(&pa[m][0]));
      const float2 f1 = __half22float2(*reinterpret_cast<const __half2*>(&pa[m][1]));
      const float2 f2 = __half22float2(*reinterpret_cast<const __half2*>(&pa[m][2]));
      const float2 f3 = __half22float2(*reinterpret_cast<const __half2*>(&pa[m][3]));
      t[m].lA += f0.x + f0.y + f2.x + f2.y;
      t[m].lB += f1.x + f1.y + f3.x + f3.y;
    }
#pragma unroll
    for (int j = 0; j < NT; ++j) {
      uint32_t b0, b1;
      ldsm_x2_trans(smem_u32(sV + (kc * 16 + (lane & 15)) * P + j * 8), b0, b1);
#pragma unroll
      for (int m = 0; m < MT; ++m) mma_16816(t[m].o[j], pa[m], b0, b1);
    }
  }
}

// O / l -> fp16 for the thread's rows j0 and j0 + 8 of the unit, real query tokens only; `op0` points at
// the unit's first token, this head.
template <int HD>
__device__ __forceinline__ void am_store(AmTile<HD>& t, int j0, int nreal, int rx, int s, int D, __half* op0,
                                         int lane) {
#pragma unroll
  for (int off = 1; off <= 2; off <<= 1) {
    t.lA += __shfl_xor_sync(0xffffffffu, t.lA, off);
    t.lB += __shfl_xor_sync(0xffffffffu, t.lB, off);
  }
  const float invA = 1.0f / t.lA, invB = 1.0f / t.lB;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int j = j0 + 8 * h;
    if (j >= nreal) continue;
    const int qh = j / rx, qw = j - qh * rx;
    __half* op = op0 + static_cast<size_t>(qh * s + qw) * D + 2 * (lane & 3);
    const float inv = h ? invB : invA;
#pragma unroll
    for (int j8 = 0; j8 < HD / 8; ++j8)
      *reinterpret_cast<uint32_t*>(op + j8 * 8) = pack_half2(t.o[j8][2 * h] * inv, t.o[j8][2 * h + 1] * inv);
  }
}

template <int HD>
__global__ void __launch_bounds__(kAmWarps * 32)
attention_mma_kernel(const __half* __restrict__ qkv, const float* __restrict__ qkv_bias,
                     const float* __restrict__ rel_h, const float* __restrict__ rel_w, int s, int win,
                     int nwin, int heads, int qblocks, float scale_log2e, __half* __restrict__ out) {
  using LY = AmLayout<HD>;
  constexpr int NTH = kAmWarps * 32;
  constexpr int P = LY::kPitch;
  constexpr int NT = HD / 8;          // n8 tiles of the output
  constexpr int KS = HD / 16;         // k16 steps of Q K^T
  constexpr int RG = NTH / NT;        // key rows per pass of the chunk loader
  const LY ly(win);
  const int winP = ly.winP, lg = ly.lg, RP = ly.relPitch;
  extern __shared__ __align__(16) uint8_t smem_am[];
  __half* sQ = reinterpret_cast<__half*>(smem_am);
  uint8_t* sKV = smem_am + LY::kQBytes;                                     // 2 stages of K, V
  __half* sTab = reinterpret_cast<__half*>(sKV);                            // prologue only
  float* sRel = reinterpret_cast<float*>(smem_am + ly.relOffset);          // [kRows][relh | relw]
  __half* sPad = reinterpret_cast<__half*>(smem_am + ly.padOffset);        // k, v of a window padding token

  const int D = heads * HD, ld = 3 * D;
  const int unit = blockIdx.x / qblocks;           // (image, window, head), head fastest
  const int head = unit % heads;
  const int widx = (unit / heads) % (nwin * nwin);
  const int b = unit / (heads * nwin * nwin);
  const int wy = widx / nwin, wx = widx % nwin;
  const int gy0 = wy * win, gx0 = wx * win;
  const int ry = min(win, s - gy0), rx = min(win, s - gx0);
  const int nreal = ry * rx;
  const int row0 = (blockIdx.x - unit * qblocks) * LY::kRows;
  if (row0 >= nreal) return;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const bool active = row0 + warp * 16 < nreal;    // warp-uniform; idle warps still load and sync
  const __half* img = qkv + static_cast<size_t>(b) * s * s * ld + head * HD;

  // ---- Q tile (rows past the real queries repeat the last one), tables as fp16 hi / lo ----
  for (int idx = tid; idx < LY::kRows * NT; idx += NTH) {
    const int r = idx / NT, c8 = idx % NT;
    const int j = min(row0 + r, nreal - 1), qh = j / rx, qw = j - qh * rx;
    *reinterpret_cast<uint4*>(sQ + r * P + c8 * 8) =
        *reinterpret_cast<const uint4*>(img + ((gy0 + qh) * s + gx0 + qw) * ld + c8 * 8);
  }
  const int L = 2 * win - 1, TR = ly.tabRows;
  for (int idx = tid; idx < 2 * TR * (HD / 2); idx += NTH) {
    const int t = idx / (TR * (HD / 2)), rem = idx - t * TR * (HD / 2);
    const int r = rem / (HD / 2), c = 2 * (rem - r * (HD / 2));
    float2 v = make_float2(0.f, 0.f);
    if (r < L) v = __ldg(reinterpret_cast<const float2*>((t ? rel_w : rel_h) + r * HD + c));
    const __half2 hi = __float22half2_rn(v);
    const float2 hf = __half22float2(hi);
    const __half2 lo = __float22half2_rn(make_float2(v.x - hf.x, v.y - hf.y));
    __half* dst = sTab + (2 * t * TR + r) * P + c;
    *reinterpret_cast<__half2*>(dst) = hi;
    *reinterpret_cast<__half2*>(dst + TR * P) = lo;
  }
  if (tid < 2 * NT)
    *reinterpret_cast<uint4*>(sPad + tid * 8) = am_bias8(qkv_bias + (1 + tid / NT) * D + head * HD + (tid % NT) * 8);
  for (int r = tid; r < LY::kRows; r += NTH) {     // slots that are no key: -inf
    for (int c = win; c < ly.relH; ++c) sRel[r * RP + c] = -INFINITY;
    for (int c = win; c < winP; ++c) sRel[r * RP + ly.relH + c] = -INFINITY;
  }
  __syncthreads();

  // ---- Q fragments (A operand) ----
  uint32_t qa[KS][4];
  {
    const int r = warp * 16 + (lane & 15);
    const int cofs = (lane >> 4) * 8;
#pragma unroll
    for (int k = 0; k < KS; ++k)
      ldsm_x4(smem_u32(sQ + r * P + k * 16 + cofs), qa[k][0], qa[k][1], qa[k][2], qa[k][3]);
  }
  const int rA = warp * 16 + (lane >> 2);          // this thread's two query rows: rA, rA + 8
  const int cq = 2 * (lane & 3);                   // and its column pair in every n8 tile

  // ---- rel-pos on the tensor cores: relh[q][kh] = q . Rh[qh - kh + win - 1], relw alike ----
  if (active) {
    const int jA = min(row0 + rA, nreal - 1), jB = min(row0 + rA + 8, nreal - 1);
    const int qhA = jA / rx, qhB = jB / rx;
    const int qwA = jA - qhA * rx, qwB = jB - qhB * rx;
#pragma unroll
    for (int t = 0; t < 2; ++t) {
      const __half* hi = sTab + 2 * t * TR * P;
      const __half* lo = hi + TR * P;
      const int cA = (t ? qwA : qhA) + win - 1, cB = (t ? qwB : qhB) + win - 1;
      float* dA = sRel + rA * RP + (t ? ly.relH : 0);
      float* dB = dA + 8 * RP;
      for (int nt = 0; nt < TR / 8; ++nt) {
        float acc[4] = {0.f, 0.f, 0.f, 0.f};
        const int boff = (nt * 8 + (lane & 7)) * P + ((lane >> 3) & 1) * 8;
#pragma unroll
        for (int k = 0; k < KS; ++k) {
          uint32_t b0, b1;
          ldsm_x2(smem_u32(hi + boff + k * 16), b0, b1);
          mma_16816(acc, qa[k], b0, b1);
          ldsm_x2(smem_u32(lo + boff + k * 16), b0, b1);
          mma_16816(acc, qa[k], b0, b1);
        }
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int r = nt * 8 + cq + e;
          const int khA = cA - r, khB = cB - r;
          if (static_cast<unsigned>(khA) < static_cast<unsigned>(win)) dA[khA] = acc[e] * 1.4426950408889634f;
          if (static_cast<unsigned>(khB) < static_cast<unsigned>(win)) dB[khB] = acc[2 + e] * 1.4426950408889634f;
        }
      }
    }
  }

  // ---- K/V chunk loader: thread owns column group c8 of key rows lr0, lr0 + RG, ... ----
  const bool loader = tid < RG * NT;
  const int c8 = tid % NT, lr0 = tid / NT;
  const __half* ksrc = img + D + c8 * 8;
  __half* kdst = reinterpret_cast<__half*>(sKV) + lr0 * P + c8 * 8;
  const uint4* kpad = reinterpret_cast<const uint4*>(sPad) + c8;   // fp16 bias of k; of v at + NT
  auto load_chunk = [&](int c) {
    if (loader) {
      __half* dk = kdst + (c & 1) * (LY::kStageBytes / 2);
      for (int r = lr0; r < kAmKC; r += RG, dk += RG * P) {
        const int k = c * kAmKC + r, kh = k >> lg, kw = k & (winP - 1);
        __half* dv = dk + kAmKC * P;
        if (kh < win && kw < win) {
          const int gy = gy0 + kh, gx = gx0 + kw;
          if (gy < s && gx < s) {
            const __half* src = ksrc + (gy * s + gx) * ld;
            cp_async16(smem_u32(dk), src);
            cp_async16(smem_u32(dv), src + D);
          } else {
            *reinterpret_cast<uint4*>(dk) = kpad[0];
            *reinterpret_cast<uint4*>(dv) = kpad[NT];
          }
        } else {
          *reinterpret_cast<uint4*>(dk) = make_uint4(0u, 0u, 0u, 0u);
          *reinterpret_cast<uint4*>(dv) = make_uint4(0u, 0u, 0u, 0u);
        }
      }
    }
    cp_async_commit();
  };
  __syncthreads();                                 // tables consumed, sRel written
  load_chunk(0);

  const float* relA = sRel + rA * RP;
  const float* relB = relA + 8 * RP;
  float o[NT][4];
#pragma unroll
  for (int j = 0; j < NT; ++j) o[j][0] = o[j][1] = o[j][2] = o[j][3] = 0.f;
  float mA = -INFINITY, mB = -INFINITY, lA = 0.f, lB = 0.f;

  for (int c = 0; c < ly.nchunks; ++c) {
    cp_async_wait_all();
    __syncthreads();                               // chunk c landed; chunk c - 1 consumed
    if (c + 1 < ly.nchunks) load_chunk(c + 1);
    if (!active) continue;
    const __half* sK = reinterpret_cast<const __half*>(sKV + (c & 1) * LY::kStageBytes);
    const __half* sV = sK + kAmKC * P;
    const int k0 = c * kAmKC;
    const bool full = k0 + kAmKC / 2 < ly.nslots;  // else the upper 32 slots hold no key

    // S = Q K^T : 16 rows x 64 keys per warp
    float sc[kAmKC / 8][4];
#pragma unroll
    for (int n = 0; n < kAmKC / 8; ++n) {
      sc[n][0] = sc[n][1] = sc[n][2] = sc[n][3] = 0.f;
      if (n < kAmKC / 16 || full) {
#pragma unroll
        for (int k = 0; k < KS; ++k) {
          uint32_t b0, b1;
          ldsm_x2(smem_u32(sK + (n * 8 + (lane & 7)) * P + k * 16 + ((lane >> 3) & 1) * 8), b0, b1);
          mma_16816(sc[n], qa[k], b0, b1);
        }
      }
    }
    // scale + bias (-inf on non-key slots), row maxima
    float cmA = -INFINITY, cmB = -INFINITY;
#pragma unroll
    for (int n = 0; n < kAmKC / 8; ++n) {
      const int kh = (k0 + n * 8) >> lg;           // one key row per n8 tile
      const int kw = (n * 8 + cq) & (winP - 1);
      const float hA = relA[kh], hB = relB[kh];
      const float2 wA = *reinterpret_cast<const float2*>(relA + ly.relH + kw);
      const float2 wB = *reinterpret_cast<const float2*>(relB + ly.relH + kw);
      sc[n][0] = fmaf(sc[n][0], scale_log2e, hA + wA.x);
      sc[n][1] = fmaf(sc[n][1], scale_log2e, hA + wA.y);
      sc[n][2] = fmaf(sc[n][2], scale_log2e, hB + wB.x);
      sc[n][3] = fmaf(sc[n][3], scale_log2e, hB + wB.y);
      cmA = fmaxf(cmA, fmaxf(sc[n][0], sc[n][1]));
      cmB = fmaxf(cmB, fmaxf(sc[n][2], sc[n][3]));
    }
#pragma unroll
    for (int off = 1; off <= 2; off <<= 1) {
      cmA = fmaxf(cmA, __shfl_xor_sync(0xffffffffu, cmA, off));
      cmB = fmaxf(cmB, __shfl_xor_sync(0xffffffffu, cmB, off));
    }
    const float nmA = fmaxf(mA, cmA), nmB = fmaxf(mB, cmB);
    const float alA = ex2_approx(mA - nmA), alB = ex2_approx(mB - nmB);   // first chunk: 2^-inf = 0
    mA = nmA; mB = nmB;
    lA *= alA; lB *= alB;
#pragma unroll
    for (int j = 0; j < NT; ++j) {
      o[j][0] *= alA; o[j][1] *= alA; o[j][2] *= alB; o[j][3] *= alB;
    }
    // P (fp16) and O += P V, 16 keys per MMA
#pragma unroll
    for (int kc = 0; kc < kAmKC / 16; ++kc) {
      if (kc >= kAmKC / 32 && !full) continue;
      uint32_t pa[4];
      float p[2][4];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int n = 2 * kc + h;
        p[h][0] = ex2_approx(sc[n][0] - mA);
        p[h][1] = ex2_approx(sc[n][1] - mA);
        p[h][2] = ex2_approx(sc[n][2] - mB);
        p[h][3] = ex2_approx(sc[n][3] - mB);
      }
      pa[0] = pack_half2(p[0][0], p[0][1]);
      pa[1] = pack_half2(p[0][2], p[0][3]);
      pa[2] = pack_half2(p[1][0], p[1][1]);
      pa[3] = pack_half2(p[1][2], p[1][3]);
      // the softmax denominator sums the same fp16-rounded P the MMA consumes
      const float2 f0 = __half22float2(*reinterpret_cast<const __half2*>(&pa[0]));
      const float2 f1 = __half22float2(*reinterpret_cast<const __half2*>(&pa[1]));
      const float2 f2 = __half22float2(*reinterpret_cast<const __half2*>(&pa[2]));
      const float2 f3 = __half22float2(*reinterpret_cast<const __half2*>(&pa[3]));
      lA += f0.x + f0.y + f2.x + f2.y;
      lB += f1.x + f1.y + f3.x + f3.y;
#pragma unroll
      for (int j = 0; j < NT; ++j) {
        uint32_t b0, b1;
        ldsm_x2_trans(smem_u32(sV + (kc * 16 + (lane & 15)) * P + j * 8), b0, b1);
        mma_16816(o[j], pa, b0, b1);
      }
    }
  }
  if (!active) return;

  // ---- epilogue ----
#pragma unroll
  for (int off = 1; off <= 2; off <<= 1) {
    lA += __shfl_xor_sync(0xffffffffu, lA, off);
    lB += __shfl_xor_sync(0xffffffffu, lB, off);
  }
  const float invA = 1.0f / lA, invB = 1.0f / lB;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int j = row0 + rA + 8 * h;
    if (j >= nreal) continue;
    const int qh = j / rx, qw = j - qh * rx;
    __half* op = out + (static_cast<size_t>(b) * s * s + (gy0 + qh) * s + gx0 + qw) * D + head * HD + cq;
    const float inv = h ? invB : invA;
#pragma unroll
    for (int j8 = 0; j8 < NT; ++j8)
      *reinterpret_cast<uint32_t*>(op + j8 * 8) = pack_half2(o[j8][2 * h] * inv, o[j8][2 * h + 1] * inv);
  }
}

// Window blocks: one CTA of NW warps per unit, the whole window resident in shared memory.
template <int HD, int NW>
__global__ void __launch_bounds__(NW * 32, 2)
attention_unit_kernel(const __half* __restrict__ qkv, const float* __restrict__ qkv_bias,
                      const float* __restrict__ rel_h, const float* __restrict__ rel_w, int s, int win,
                      int nwin, int heads, float scale_log2e, __half* __restrict__ out) {
  using LY = AmLayout<HD>;
  constexpr int NTH = NW * 32;
  constexpr int P = LY::kPitch;
  constexpr int NT = HD / 8;
  constexpr int KS = HD / 16;
  constexpr int RG = NTH / NT;        // key slots per pass of the loader
  const LY ly(win);
  const int winP = ly.winP, lg = ly.lg, RP = ly.relPitch;
  extern __shared__ __align__(16) uint8_t smem_am[];
  __half* sK = reinterpret_cast<__half*>(smem_am);
  __half* sV = sK + ly.kvSlots * P;
  __half* sTab = reinterpret_cast<__half*>(smem_am + ly.uTabOffset);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  uint8_t* scratch = smem_am + ly.uWarpOffset + warp * ly.uWarpBytes;
  __half* sQ = reinterpret_cast<__half*>(scratch);     // the warp's Q tile, until its fragments are in registers,
  float* sRel = reinterpret_cast<float*>(scratch);     // then its 16 [relh | relw] rows

  const int D = heads * HD, ld = 3 * D;
  const int unit = blockIdx.x;                     // (image, window, head), head fastest
  const int head = unit % heads;
  const int widx = (unit / heads) % (nwin * nwin);
  const int b = unit / (heads * nwin * nwin);
  const int wy = widx / nwin, wx = widx % nwin;
  const int gy0 = wy * win, gx0 = wx * win;
  const int ry = min(win, s - gy0), rx = min(win, s - gx0);
  const int nreal = ry * rx, ntiles = (nreal + 15) / 16;
  const __half* img = qkv + static_cast<size_t>(b) * s * s * ld + head * HD;

  // ---- the unit's K and V, requested at once: thread owns column group c8 of slots lr0, lr0 + RG, ... ----
  if (tid < RG * NT) {
    const int c8 = tid % NT;
    const __half* ksrc = img + D + c8 * 8;
    uint4 kpad = make_uint4(0u, 0u, 0u, 0u), vpad = kpad;
    if (nreal < win * win) {                       // an edge window: padding keys carry the fp16 qkv bias
      kpad = am_bias8(qkv_bias + D + head * HD + c8 * 8);
      vpad = am_bias8(qkv_bias + 2 * D + head * HD + c8 * 8);
    }
    for (int k = tid / NT; k < ly.kvSlots; k += RG) {
      const int kh = k >> lg, kw = k & (winP - 1);
      __half* dk = sK + k * P + c8 * 8;
      __half* dv = sV + k * P + c8 * 8;
      if (kh < win && kw < win) {
        if (kh < ry && kw < rx) {
          const __half* src = ksrc + ((gy0 + kh) * s + gx0 + kw) * ld;
          cp_async16(smem_u32(dk), src);
          cp_async16(smem_u32(dv), src + D);
        } else {
          *reinterpret_cast<uint4*>(dk) = kpad;
          *reinterpret_cast<uint4*>(dv) = vpad;
        }
      } else {
        *reinterpret_cast<uint4*>(dk) = make_uint4(0u, 0u, 0u, 0u);
        *reinterpret_cast<uint4*>(dv) = make_uint4(0u, 0u, 0u, 0u);
      }
    }
  }
  cp_async_commit();
  am_stage_tables<HD, NTH>(sTab, rel_h, rel_w, win, ly.tabRows, tid);
  __syncthreads();                                 // tables staged

  const int rA = lane >> 2;                        // this thread's rows of the warp's tile: rA, rA + 8
  const float* relA = sRel + rA * RP;
  __half* out0 = out + (static_cast<size_t>(b) * s * s + gy0 * s + gx0) * D + head * HD;
  for (int tile = warp; tile < ntiles || tile == warp; tile += NW) {
    const bool active = tile < ntiles;             // false only for a warp with no tile at all
    uint32_t qa[1][KS][4];
    if (active) {
      // Q tile (rows past the real queries repeat the last one) -> fragments
      for (int idx = lane; idx < 16 * NT; idx += 32) {
        const int r = idx / NT, c8 = idx % NT;
        const int j = min(tile * 16 + r, nreal - 1), qh = j / rx, qw = j - qh * rx;
        *reinterpret_cast<uint4*>(sQ + r * P + c8 * 8) =
            *reinterpret_cast<const uint4*>(img + ((gy0 + qh) * s + gx0 + qw) * ld + c8 * 8);
      }
      __syncwarp();
#pragma unroll
      for (int k = 0; k < KS; ++k)
        ldsm_x4(smem_u32(sQ + (lane & 15) * P + k * 16 + (lane >> 4) * 8), qa[0][k][0], qa[0][k][1], qa[0][k][2],
                qa[0][k][3]);
      __syncwarp();
      for (int r = lane; r < 16; r += 32) {        // slots that are no key: -inf
        for (int c = win; c < ly.relH; ++c) sRel[r * RP + c] = -INFINITY;
        for (int c = win; c < winP; ++c) sRel[r * RP + ly.relH + c] = -INFINITY;
      }
      am_relpos<HD>(qa[0], sTab, ly.tabRows, win, rx, min(tile * 16 + rA, nreal - 1),
                    min(tile * 16 + rA + 8, nreal - 1), sRel + rA * RP, RP, ly.relH, lane);
      __syncwarp();
    }
    if (tile == warp) {                            // every warp's first round: K and V have landed
      cp_async_wait_all();
      __syncthreads();
    }
    if (!active) break;
    AmTile<HD> t[1];
    t[0].reset();
    const float* const rel[1] = {relA};
    for (int c = 0; c < ly.nchunks; ++c) {
      const int k0 = c * kAmKC;
      am_chunk<HD, 1>(t, qa, sK + k0 * P, sV + k0 * P, k0, k0 + kAmKC / 2 < ly.nslots, rel, RP, ly.relH, lg, winP,
                      scale_log2e, lane);
    }
    am_store<HD>(t[0], tile * 16 + rA, nreal, rx, s, D, out0, lane);
    __syncwarp();                                  // the tile's rel rows are read; the next Q tile may land
  }
}

// Global blocks: the streamed kernel with two m-tiles per warp (128 query rows per CTA), so that every K and V
// fragment read from shared memory feeds two MMAs and a unit's K/V is streamed by half as many CTAs.
template <int HD>
__global__ void __launch_bounds__(kAmWarps * 32, 2)
attention_wide_kernel(const __half* __restrict__ qkv, const float* __restrict__ qkv_bias,
                      const float* __restrict__ rel_h, const float* __restrict__ rel_w, int s, int win,
                      int heads, int qblocks, float scale_log2e, __half* __restrict__ out) {
  using LY = AmLayout<HD>;
  constexpr int NTH = kAmWarps * 32;
  constexpr int P = LY::kPitch;
  constexpr int NT = HD / 8;
  constexpr int KS = HD / 16;
  constexpr int RG = NTH / NT;        // key rows per pass of the chunk loader
  constexpr int ROWS = 2 * LY::kRows;
  const LY ly(win);
  const int winP = ly.winP, lg = ly.lg, RP = ly.relPitch;
  extern __shared__ __align__(16) uint8_t smem_am[];
  __half* sQ = reinterpret_cast<__half*>(smem_am);
  uint8_t* sKV = smem_am + 2 * LY::kQBytes;                                 // 2 stages of K, V
  __half* sTab = reinterpret_cast<__half*>(sKV);                            // prologue only
  float* sRel = reinterpret_cast<float*>(smem_am + ly.wide_rel_offset());  // [ROWS][relh | relw]
  __half* sPad = reinterpret_cast<__half*>(smem_am + ly.wide_pad_offset());

  const int D = heads * HD, ld = 3 * D;
  const int unit = blockIdx.x / qblocks;           // (image, head), head fastest: one window per image
  const int head = unit % heads, b = unit / heads;
  const int ry = min(win, s), rx = ry, nreal = ry * rx;
  const int row0 = (blockIdx.x - unit * qblocks) * ROWS;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const bool active = row0 + warp * 32 < nreal;    // warp-uniform; idle warps still load and sync
  const __half* img = qkv + static_cast<size_t>(b) * s * s * ld + head * HD;

  for (int idx = tid; idx < ROWS * NT; idx += NTH) {   // rows past the real queries repeat the last one
    const int r = idx / NT, c8 = idx % NT;
    const int j = min(row0 + r, nreal - 1), qh = j / rx, qw = j - qh * rx;
    *reinterpret_cast<uint4*>(sQ + r * P + c8 * 8) =
        *reinterpret_cast<const uint4*>(img + (qh * s + qw) * ld + c8 * 8);
  }
  am_stage_tables<HD, NTH>(sTab, rel_h, rel_w, win, ly.tabRows, tid);
  if (tid < 2 * NT)
    *reinterpret_cast<uint4*>(sPad + tid * 8) = am_bias8(qkv_bias + (1 + tid / NT) * D + head * HD + (tid % NT) * 8);
  for (int r = tid; r < ROWS; r += NTH) {          // slots that are no key: -inf
    for (int c = win; c < ly.relH; ++c) sRel[r * RP + c] = -INFINITY;
    for (int c = win; c < winP; ++c) sRel[r * RP + ly.relH + c] = -INFINITY;
  }
  __syncthreads();

  uint32_t qa[2][KS][4];
  const int rA = warp * 32 + (lane >> 2);          // this thread's query rows: rA, rA + 8 and those + 16
#pragma unroll
  for (int m = 0; m < 2; ++m) {
#pragma unroll
    for (int k = 0; k < KS; ++k)
      ldsm_x4(smem_u32(sQ + (warp * 32 + m * 16 + (lane & 15)) * P + k * 16 + (lane >> 4) * 8), qa[m][k][0],
              qa[m][k][1], qa[m][k][2], qa[m][k][3]);
    if (active)
      am_relpos<HD>(qa[m], sTab, ly.tabRows, win, rx, min(row0 + rA + m * 16, nreal - 1),
                    min(row0 + rA + m * 16 + 8, nreal - 1), sRel + (rA + m * 16) * RP, RP, ly.relH, lane);
  }

  // ---- K/V chunk loader: thread owns column group c8 of key rows lr0, lr0 + RG, ... ----
  const bool loader = tid < RG * NT;
  const int c8 = tid % NT, lr0 = tid / NT;
  const __half* ksrc = img + D + c8 * 8;
  __half* kdst = reinterpret_cast<__half*>(sKV) + lr0 * P + c8 * 8;
  const uint4* kpad = reinterpret_cast<const uint4*>(sPad) + c8;   // fp16 bias of k; of v at + NT
  auto load_chunk = [&](int c) {
    if (loader) {
      __half* dk = kdst + (c & 1) * (LY::kStageBytes / 2);
      for (int r = lr0; r < kAmKC; r += RG, dk += RG * P) {
        const int k = c * kAmKC + r, kh = k >> lg, kw = k & (winP - 1);
        __half* dv = dk + kAmKC * P;
        if (kh < win && kw < win) {
          if (kh < s && kw < s) {
            const __half* src = ksrc + (kh * s + kw) * ld;
            cp_async16(smem_u32(dk), src);
            cp_async16(smem_u32(dv), src + D);
          } else {
            *reinterpret_cast<uint4*>(dk) = kpad[0];
            *reinterpret_cast<uint4*>(dv) = kpad[NT];
          }
        } else {
          *reinterpret_cast<uint4*>(dk) = make_uint4(0u, 0u, 0u, 0u);
          *reinterpret_cast<uint4*>(dv) = make_uint4(0u, 0u, 0u, 0u);
        }
      }
    }
    cp_async_commit();
  };
  __syncthreads();                                 // tables consumed, sRel written
  load_chunk(0);

  const float* const rel[2] = {sRel + rA * RP, sRel + (rA + 16) * RP};
  AmTile<HD> t[2];
  t[0].reset();
  t[1].reset();
  for (int c = 0; c < ly.nchunks; ++c) {
    cp_async_wait_all();
    __syncthreads();                               // chunk c landed; chunk c - 1 consumed
    if (c + 1 < ly.nchunks) load_chunk(c + 1);
    if (!active) continue;
    const __half* sK = reinterpret_cast<const __half*>(sKV + (c & 1) * LY::kStageBytes);
    const int k0 = c * kAmKC;
    am_chunk<HD, 2>(t, qa, sK, sK + kAmKC * P, k0, k0 + kAmKC / 2 < ly.nslots, rel, RP, ly.relH, lg, winP,
                    scale_log2e, lane);
  }
  if (!active) return;
  __half* out0 = out + static_cast<size_t>(b) * s * s * D + head * HD;
#pragma unroll
  for (int m = 0; m < 2; ++m) am_store<HD>(t[m], row0 + rA + m * 16, nreal, rx, s, D, out0, lane);
}

// Warps of a one-CTA-per-unit block, and the shared memory that still lets two such CTAs share an SM
// (228 KB per SM, 1 KB reserved per CTA).  A full 14 x 14 window is 13 m-tiles: 5 warps walk them in three
// rounds (13 of 15 slots used, 4 warps 13 of 16) at 10 warps per SM; 6 warps need a fourth of the time for one
// tile, and 7 warps (two rounds) would have to fit 146 registers and spill.  At head dim 80 only 4 warps'
// scratch fits (8 warps per SM).
template <int HD> constexpr int kAuWarps = HD == 64 ? 5 : 4;
constexpr int kAuMaxBytes = (228 * 1024) / 2 - 1024;

template <int HD>
int launch_attention_mma(const __half* qkv, const float* qkv_bias, const float* rel_h, const float* rel_w,
                         int B, int s, int win, int heads, __half* out, cudaStream_t st) {
  using LY = AmLayout<HD>;
  constexpr int NW = kAuWarps<HD>;
  const LY ly(win);
  const int nwin = (s + win - 1) / win;
  const float scale_log2e = 1.4426950408889634f / sqrtf(static_cast<float>(HD));
  const bool resident = win < s && ly.unit_bytes(NW) <= kAuMaxBytes;
  const int w0 = win < s ? win : s;       // real queries of the fullest window: w0 x w0
  const bool wide = win >= s;              // one window per image: two m-tiles per warp
  const int qblocks = resident ? 1 : ((w0 * w0 + 15) / 16 + (wide ? 2 : 1) * kAmWarps - 1) / ((wide ? 2 : 1) * kAmWarps);
  const long blocks = static_cast<long>(qblocks) * B * nwin * nwin * heads;
  SRB_REQUIRE(blocks <= 2147483647L, "attention: %ld CTAs exceed the grid limit (B=%d s=%d win=%d heads=%d)",
              blocks, B, s, win, heads);
  const unsigned grid = static_cast<unsigned>(blocks);
  if (resident) {
    auto kern = attention_unit_kernel<HD, NW>;
    SRB_TRY(allow_dynamic_smem(kern, ly.unit_bytes(NW)));
    SRB_LAUNCH(kern, grid, NW * 32, ly.unit_bytes(NW), st, qkv, qkv_bias, rel_h, rel_w, s, win, nwin, heads,
               scale_log2e, out);
  } else if (wide) {
    auto kern = attention_wide_kernel<HD>;
    SRB_TRY(allow_dynamic_smem(kern, ly.wide_bytes()));
    SRB_LAUNCH(kern, grid, kAmWarps * 32, ly.wide_bytes(), st, qkv, qkv_bias, rel_h, rel_w, s, win, heads, qblocks,
               scale_log2e, out);
  } else {
    auto kern = attention_mma_kernel<HD>;
    SRB_TRY(allow_dynamic_smem(kern, ly.bytes));
    SRB_LAUNCH(kern, grid, kAmWarps * 32, ly.bytes, st, qkv, qkv_bias, rel_h, rel_w, s, win, nwin, heads, qblocks,
               scale_log2e, out);
  }
  return 0;
}

}  // namespace srb
