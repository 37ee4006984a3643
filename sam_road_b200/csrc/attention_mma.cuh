// sam_road_b200 :: tensor-core encoder attention (head_dim 64 or 80), windowed or global, with the
// decomposed relative-position bias.  Same semantics as the SIMT kernel in attention.cu.
//
// Unit = (image, window, head).  Its real queries (the window's tokens inside the s x s grid, ry x rx
// of them) are numbered j = qh * rx + qw and cut into 16-row m-tiles, one per warp at a time, so edge
// windows run only the rows they have.  Three kernels:
//   attention_unit_kernel : window blocks (win < s) whose whole window fits in shared memory twice
//              per SM.  One CTA per unit: K, V and the tables are staged once, and the CTA's warps
//              walk the unit's m-tiles (tile = warp, warp + NW, ...).  After the one barrier that
//              publishes K/V, a warp touches only its own scratch rows, so tiles need __syncwarp only.
//   attention_global_kernel : global blocks (win == s), on TMA and wgmma; described at the kernel.
//   attention_mma_kernel  : windows too large to be resident, the one padded window of a grid smaller
//              than its window, and global blocks whose rings do not fit.  Each CTA streams the unit's
//              K/V in double-buffered chunks for one m-tile per warp; a CTA past the unit's last tile
//              exits at once.  It keeps its own copy of the tile math (it predates the shared helpers
//              and is left as measured).
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

// Global blocks (win == s): one persistent CTA per SM, three warpgroups.  A work item is (image, head, block of
// 128 query rows), the query block fastest, so that the CTAs reading one unit's K/V run together and share it in
// L2.  Warpgroup 0 issues TMA loads: the item's Q (a [128 rows x HD] box of qkv viewed as [B s s, 3 D]) into a
// ring of Q stages, and K and V of each 128-slot key block (a box {HD, winP, 128 / winP} of qkv viewed as
// [B][s][s][3 D]; kw >= s and kh >= s arrive as zeros and are masked by the -inf of relw / relh) into a ring of
// K/V stages.  Warpgroups 1 and 2 own the item's query rows 0..63 and 64..127: S = Q K^T on wgmma from shared
// memory, the bias and online softmax of am_chunk on the accumulator (its per-warp row and column layout is that
// of mma.sync), P rounded to fp16 and O += P V on wgmma with P from registers and V MN-major.  Within a
// consumer the next block's Q K^T is issued with this block's P V, and both run under the softmax of the next
// block; the two consumers take turns to issue (named barriers 2 and 3), so one's softmax runs under the
// other's MMAs.  At head dim 80 each row is a 128B-swizzled 64-column box and a 32B-swizzled 16-column box.
constexpr int kAgRows = 128;        // query rows per work item
constexpr int kAgSlots = 128;       // key slots per K/V block
constexpr int kAgThreads = 384;
constexpr int kAgMaxBytes = 227 * 1024 - 1024;   // the dynamic limit, less the 1 KB alignment of the base

template <int HD>
struct AgLayout {
  static_assert(HD == 64 || HD == 80, "head dim 64 or 80");
  static constexpr int kTailOffset = kAgRows * 128;            // the 16-column box of a Q, K or V buffer
  static constexpr int kBoxBytes = kAgRows * HD * 2;           // one Q, K or V buffer
  int winP, lg, nblocks, relH, relPitch, tabRows;
  int qStages, kvStages;              // 0: shared memory does not hold even the smallest rings
  int tabOffset, relOffset, barOffset, bytes;
  __host__ __device__ explicit AgLayout(int s) {
    winP = 8; lg = 3;
    while (winP < s) { winP <<= 1; ++lg; }
    nblocks = (s * winP + kAgSlots - 1) / kAgSlots;
    relH = ((nblocks * kAgSlots / winP + 7) / 8) * 8;
    relPitch = ((relH + winP - 8 + 31) / 32) * 32 + 8;
    tabRows = ((2 * s - 1 + 7) / 8) * 8;
    const int fixed = 4 * tabRows * AmLayout<HD>::kPitch * 2 + 2 * 64 * relPitch * 4 + 16 * 8;
    // the deepest rings that fit: three K/V stages keep the next block's loads ahead of both consumers
    const int cand[3][2] = {{2, 3}, {2, 2}, {1, 2}};
    qStages = kvStages = 0;
    for (int i = 0; i < 3 && qStages == 0; ++i)
      if ((cand[i][0] + 2 * cand[i][1]) * kBoxBytes + fixed <= kAgMaxBytes) {
        qStages = cand[i][0];
        kvStages = cand[i][1];
      }
    tabOffset = (qStages + 2 * kvStages) * kBoxBytes;          // [Q stages | K, V stages | tables | rel | bars]
    relOffset = tabOffset + 4 * tabRows * AmLayout<HD>::kPitch * 2;
    barOffset = relOffset + 2 * 64 * relPitch * 4;
    bytes = barOffset + 16 * 8 + 1024;
  }
};

template <int HD>
__global__ void __launch_bounds__(kAgThreads, 1)
attention_global_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmQt,
                        const __grid_constant__ CUtensorMap tmKV, const __grid_constant__ CUtensorMap tmKVt,
                        const float* __restrict__ rel_h, const float* __restrict__ rel_w, int s, int heads,
                        int nitems, float scale_log2e, __half* __restrict__ out) {
  using LY = AgLayout<HD>;
  constexpr bool kTail = HD == 80;
  constexpr int KS = HD / 16;
  const LY ly(s);
  const int winP = ly.winP, lg = ly.lg, RP = ly.relPitch, nb = ly.nblocks;
  const int QS = ly.qStages, KVS = ly.kvStages;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* sQ = smem;
  uint8_t* sKV = smem + QS * LY::kBoxBytes;                      // stage i: K at 2 i, V at 2 i + 1 boxes
  __half* sTab = reinterpret_cast<__half*>(smem + ly.tabOffset);
  float* sRel = reinterpret_cast<float*>(smem + ly.relOffset);  // [2 consumers x 64 rows][relh | relw]
  uint64_t* qfull = reinterpret_cast<uint64_t*>(smem + ly.barOffset);
  uint64_t* qempty = qfull + 2;
  uint64_t* kfull = qempty + 2;
  uint64_t* kempty = kfull + 3;
  uint64_t* vfull = kempty + 3;
  uint64_t* vempty = vfull + 3;

  const int D = heads * HD, nreal = s * s;
  const int qblocks = (nreal + kAgRows - 1) / kAgRows;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = warp >> 2;
  if (threadIdx.x == 0) {
    for (int i = 0; i < QS; ++i) {
      mbar_init(&qfull[i], 1);
      mbar_init(&qempty[i], 8);                                 // every consumer warp
    }
    for (int i = 0; i < KVS; ++i) {
      mbar_init(&kfull[i], 1);
      mbar_init(&kempty[i], 8);
      mbar_init(&vfull[i], 1);
      mbar_init(&vempty[i], 8);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    // ===================== TMA producer =====================
    setmaxnreg_dec<40>();
    if (warp == 0 && lane == 0) {
      tma_prefetch_desc(&tmQ);
      tma_prefetch_desc(&tmKV);
      int qs = 0, ks = 0;
      uint32_t qph = 0, kph = 0;
      for (int item = blockIdx.x; item < nitems; item += gridDim.x) {
        const int qb = item % qblocks, unit = item / qblocks;
        const int head = unit % heads, b = unit / heads;
        uint8_t* q = sQ + qs * LY::kBoxBytes;
        mbar_wait(&qempty[qs], qph ^ 1u);
        mbar_arrive_expect_tx(&qfull[qs], LY::kBoxBytes);
        tma_load_2d(q, &tmQ, &qfull[qs], head * HD, b * nreal + qb * kAgRows);
        if (kTail) tma_load_2d(q + LY::kTailOffset, &tmQt, &qfull[qs], head * HD + 64, b * nreal + qb * kAgRows);
        if (++qs == QS) { qs = 0; qph ^= 1u; }
        for (int kb = 0; kb < nb; ++kb) {
          const int kh0 = kb * (kAgSlots / winP);
          uint8_t* k = sKV + 2 * ks * LY::kBoxBytes;
          uint8_t* v = k + LY::kBoxBytes;
          mbar_wait(&kempty[ks], kph ^ 1u);
          mbar_arrive_expect_tx(&kfull[ks], LY::kBoxBytes);
          tma_load_4d(k, &tmKV, &kfull[ks], D + head * HD, 0, kh0, b);
          if (kTail) tma_load_4d(k + LY::kTailOffset, &tmKVt, &kfull[ks], D + head * HD + 64, 0, kh0, b);
          mbar_wait(&vempty[ks], kph ^ 1u);
          mbar_arrive_expect_tx(&vfull[ks], LY::kBoxBytes);
          tma_load_4d(v, &tmKV, &vfull[ks], 2 * D + head * HD, 0, kh0, b);
          if (kTail) tma_load_4d(v + LY::kTailOffset, &tmKVt, &vfull[ks], 2 * D + head * HD + 64, 0, kh0, b);
          if (++ks == KVS) { ks = 0; kph ^= 1u; }
        }
      }
    }
    return;
  }

  // ===================== consumers =====================
  setmaxnreg_inc<232>();
  const int g = wg - 1, w = warp & 3;
  const int ctid = threadIdx.x - 128;
  am_stage_tables<HD, 256>(sTab, rel_h, rel_w, s, ly.tabRows, ctid);
  for (int r = ctid; r < 128; r += 256) {                       // slots that are no key: -inf
    for (int c = s; c < ly.relH; ++c) sRel[r * RP + c] = -INFINITY;
    for (int c = s; c < winP; ++c) sRel[r * RP + ly.relH + c] = -INFINITY;
  }
  named_bar_sync(1, 256);

  const int rW = 64 * g + 16 * w;                               // the warp's first row of the item
  const int cq = 2 * (lane & 3);
  float* relA = sRel + (rW + (lane >> 2)) * RP;                 // the thread's rows A and B = A + 8
  const float* relB = relA + 8 * RP;
  if (g == 1) named_bar_arrive(2, 256);                         // consumer 0 issues first
  int qs = 0, ks = 0;
  uint32_t qph = 0, kph = 0;
  for (int item = blockIdx.x; item < nitems; item += gridDim.x) {
    const int qb = item % qblocks, unit = item / qblocks;
    const int head = unit % heads, b = unit / heads;
    const uint32_t q = smem_u32(sQ + qs * LY::kBoxBytes);
    mbar_wait(&qfull[qs], qph);

    // ---- rel-pos of the warp's 16 rows on mma.sync, from the swizzled Q box ----
    {
      uint32_t qa[KS][4];
      const int r = rW + (lane & 15);
#pragma unroll
      for (int k = 0; k < KS; ++k) {
        const uint32_t a = k < 4 ? q + r * 128 + (((2 * k + (lane >> 4)) ^ (r & 7)) << 4)
                                 : q + LY::kTailOffset + r * 32 + (((lane >> 4) ^ ((r >> 2) & 1)) << 4);
        ldsm_x4(a, qa[k][0], qa[k][1], qa[k][2], qa[k][3]);
      }
      const int j = qb * kAgRows + rW + (lane >> 2);
      am_relpos<HD>(qa, sTab, ly.tabRows, s, s, min(j, nreal - 1), min(j + 8, nreal - 1), relA, RP, ly.relH, lane);
      __syncwarp();
    }

    const uint64_t qd = wgmma_desc_k128(q + g * 64 * 128);
    const uint64_t qdt = wgmma_desc_k32(q + LY::kTailOffset + g * 64 * 32);
    float sc[64];                     // S of one block: n8 tile n at sc[4 n ..], rows A (0, 1) and B (2, 3)
    float o[32], ot[kTail ? 8 : 1];   // O columns 0..63 and, at head dim 80, 64..79
    uint32_t pa[kAgSlots / 16][4];    // P (fp16) as the A operand of P V, one k16 step per row
    float mA = -INFINITY, mB = -INFINITY, lA = 0.f, lB = 0.f;
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] = 0.f;
#pragma unroll
    for (int i = 0; i < (kTail ? 8 : 1); ++i) ot[i] = 0.f;

    auto issue_s = [&](int stage) {
      const uint32_t k = smem_u32(sKV + 2 * stage * LY::kBoxBytes);
      const uint64_t kd = wgmma_desc_k128(k);
#pragma unroll
      for (int kk = 0; kk < 4; ++kk)
        wgmma_m64n128k16(sc, qd + static_cast<uint64_t>(2 * kk), kd + static_cast<uint64_t>(2 * kk), kk != 0);
      if constexpr (kTail) wgmma_m64n128k16(sc, qdt, wgmma_desc_k32(k + LY::kTailOffset), 1u);
      wgmma_commit();
    };
    // scale + bias, then P = 2^(S - m) in place; returns the rescale factors of the running state
    auto softmax = [&](int kb, float& alA, float& alB) {
      const int k0 = kb * kAgSlots;
      float cmA = -INFINITY, cmB = -INFINITY;
#pragma unroll
      for (int n = 0; n < kAgSlots / 8; ++n) {
        const int kh = (k0 + n * 8) >> lg;                      // one key row per n8 tile
        const int kw = (n * 8 + cq) & (winP - 1);
        const float hA = relA[kh], hB = relB[kh];
        const float2 wA = *reinterpret_cast<const float2*>(relA + ly.relH + kw);
        const float2 wB = *reinterpret_cast<const float2*>(relB + ly.relH + kw);
        sc[4 * n + 0] = fmaf(sc[4 * n + 0], scale_log2e, hA + wA.x);
        sc[4 * n + 1] = fmaf(sc[4 * n + 1], scale_log2e, hA + wA.y);
        sc[4 * n + 2] = fmaf(sc[4 * n + 2], scale_log2e, hB + wB.x);
        sc[4 * n + 3] = fmaf(sc[4 * n + 3], scale_log2e, hB + wB.y);
        cmA = fmaxf(cmA, fmaxf(sc[4 * n + 0], sc[4 * n + 1]));
        cmB = fmaxf(cmB, fmaxf(sc[4 * n + 2], sc[4 * n + 3]));
      }
#pragma unroll
      for (int off = 1; off <= 2; off <<= 1) {
        cmA = fmaxf(cmA, __shfl_xor_sync(0xffffffffu, cmA, off));
        cmB = fmaxf(cmB, __shfl_xor_sync(0xffffffffu, cmB, off));
      }
      const float nmA = fmaxf(mA, cmA), nmB = fmaxf(mB, cmB);
      alA = ex2_approx(mA - nmA);                               // first block: 2^-inf = 0
      alB = ex2_approx(mB - nmB);
      mA = nmA; mB = nmB;
#pragma unroll
      for (int n = 0; n < kAgSlots / 8; ++n) {
        sc[4 * n + 0] = ex2_approx(sc[4 * n + 0] - mA);
        sc[4 * n + 1] = ex2_approx(sc[4 * n + 1] - mA);
        sc[4 * n + 2] = ex2_approx(sc[4 * n + 2] - mB);
        sc[4 * n + 3] = ex2_approx(sc[4 * n + 3] - mB);
      }
    };
    // once the previous P V has finished: rescale O and l, round P to fp16; l sums the rounded P
    auto take_p = [&](float alA, float alB) {
#pragma unroll
      for (int i = 0; i < 32; i += 4) { o[i] *= alA; o[i + 1] *= alA; o[i + 2] *= alB; o[i + 3] *= alB; }
#pragma unroll
      for (int i = 0; i < (kTail ? 8 : 0); i += 4) { ot[i] *= alA; ot[i + 1] *= alA; ot[i + 2] *= alB; ot[i + 3] *= alB; }
      lA *= alA; lB *= alB;
#pragma unroll
      for (int kc = 0; kc < kAgSlots / 16; ++kc) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          pa[kc][e] = pack_half2(sc[8 * kc + 2 * e], sc[8 * kc + 2 * e + 1]);
          const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&pa[kc][e]));
          if (e & 1) lB += f.x + f.y; else lA += f.x + f.y;
        }
      }
    };

    // ---- block 0 ----
    mbar_wait(&kfull[ks], kph);
    wgmma_fence();
    issue_s(ks);
    wgmma_wait<0>();
    wgmma_fence_operand(sc);
    if (lane == 0) mbar_arrive(&kempty[ks]);
    {
      float alA, alB;
      softmax(0, alA, alB);
      take_p(alA, alB);
    }
    // P V of the block in stage ks; issued in this consumer's turn, after the next block's Q K^T if any
    auto issue_pv = [&]() {
      mbar_wait(&vfull[ks], kph);
      const uint32_t v = smem_u32(sKV + (2 * ks + 1) * LY::kBoxBytes);
#pragma unroll
      for (int kc = 0; kc < kAgSlots / 16; ++kc) {
        wgmma_m64n64k16_rs_t(o, pa[kc], wgmma_desc_k128(v + kc * 16 * 128), 1u);
        if constexpr (kTail)
          wgmma_m64n16k16_rs_t(*reinterpret_cast<float(*)[8]>(ot), pa[kc],
                               wgmma_desc_k32(v + LY::kTailOffset + kc * 16 * 32), 1u);
      }
      wgmma_commit();
      named_bar_arrive(2 + (g ^ 1), 256);                       // the other consumer's turn
    };
    auto begin_turn = [&]() {
      named_bar_sync(2 + g, 256);                               // this consumer's turn to issue
      wgmma_fence_operand(o);
      wgmma_fence_operand(ot);
      wgmma_fence_operand(pa);
      wgmma_fence();
    };
    auto end_pv = [&]() {
      wgmma_fence_operand(o);
      wgmma_fence_operand(ot);
      wgmma_fence_operand(pa);
      if (lane == 0) mbar_arrive(&vempty[ks]);
    };
    // every block but the last: the next block's S = Q K^T runs with this block's P V, its softmax under P V.
    // The last block is peeled so that the number of MMA groups in flight never depends on a branch.
    for (int kb = 0; kb + 1 < nb; ++kb) {
      const int ks1 = ks + 1 == KVS ? 0 : ks + 1;
      const uint32_t kph1 = ks1 == 0 ? kph ^ 1u : kph;
      begin_turn();
      mbar_wait(&kfull[ks1], kph1);
      issue_s(ks1);
      issue_pv();
      wgmma_wait<1>();                                          // S of block kb + 1
      wgmma_fence_operand(sc);
      if (lane == 0) mbar_arrive(&kempty[ks1]);
      float alA, alB;
      softmax(kb + 1, alA, alB);
      wgmma_wait<0>();                                          // P V of block kb
      end_pv();
      take_p(alA, alB);
      ks = ks1;
      kph = kph1;
    }
    begin_turn();
    issue_pv();
    wgmma_wait<0>();
    end_pv();
    if (++ks == KVS) { ks = 0; kph ^= 1u; }
    if (lane == 0) mbar_arrive(&qempty[qs]);
    if (++qs == QS) { qs = 0; qph ^= 1u; }

    // ---- O / l -> fp16, real query rows only ----
#pragma unroll
    for (int off = 1; off <= 2; off <<= 1) {
      lA += __shfl_xor_sync(0xffffffffu, lA, off);
      lB += __shfl_xor_sync(0xffffffffu, lB, off);
    }
    const float invA = 1.0f / lA, invB = 1.0f / lB;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int j = qb * kAgRows + rW + (lane >> 2) + 8 * h;
      if (j >= nreal) continue;
      __half* op = out + (static_cast<size_t>(b) * nreal + j) * D + head * HD + cq;
      const float inv = h ? invB : invA;
#pragma unroll
      for (int j8 = 0; j8 < 8; ++j8)
        *reinterpret_cast<uint32_t*>(op + j8 * 8) = pack_half2(o[4 * j8 + 2 * h] * inv, o[4 * j8 + 2 * h + 1] * inv);
#pragma unroll
      for (int j8 = 0; j8 < (kTail ? 2 : 0); ++j8)
        *reinterpret_cast<uint32_t*>(op + 64 + j8 * 8) =
            pack_half2(ot[4 * j8 + 2 * h] * inv, ot[4 * j8 + 2 * h + 1] * inv);
    }
  }
  if (g == 0) named_bar_sync(2, 256);                           // consumer 1's last turn handed back
}

template <int HD>
int launch_attention_global(const __half* qkv, const float* rel_h, const float* rel_w, int B, int s, int heads,
                            __half* out, cudaStream_t st) {
  const AgLayout<HD> ly(s);
  const uint64_t D = static_cast<uint64_t>(heads) * HD, tokens = static_cast<uint64_t>(B) * s * s;
  CUtensorMap tmQ, tmQt, tmKV, tmKVt;
  SRB_TRY(make_tmap_f16_2d(&tmQ, qkv, tokens, 3 * D, 3 * D, kAgRows, 64));
  const uint64_t dims[4] = {3 * D, static_cast<uint64_t>(s), static_cast<uint64_t>(s), static_cast<uint64_t>(B)};
  const uint64_t strides[3] = {3 * D, 3 * D * s, 3 * D * s * s};
  const uint32_t box[4] = {64, static_cast<uint32_t>(ly.winP), static_cast<uint32_t>(kAgSlots / ly.winP), 1};
  SRB_TRY(make_tmap_f16_4d(&tmKV, qkv, dims, strides, box));
  tmQt = tmQ;
  tmKVt = tmKV;
  if (HD == 80) {
    const uint32_t tbox[4] = {16, box[1], box[2], 1};
    SRB_TRY(make_tmap_f16_2d(&tmQt, qkv, tokens, 3 * D, 3 * D, kAgRows, 16));
    SRB_TRY(make_tmap_f16_4d(&tmKVt, qkv, dims, strides, tbox));
  }
  const long items = static_cast<long>(B) * heads * ((s * s + kAgRows - 1) / kAgRows);
  SRB_REQUIRE(items <= 2147483647L, "attention: %ld work items exceed the int range (B=%d s=%d heads=%d)", items,
              B, s, heads);
  const int grid = items < device_sm_count() ? static_cast<int>(items) : device_sm_count();
  const float scale_log2e = 1.4426950408889634f / sqrtf(static_cast<float>(HD));
  auto kern = attention_global_kernel<HD>;
  SRB_TRY(allow_dynamic_smem(kern, ly.bytes));
  SRB_LAUNCH(kern, grid, kAgThreads, ly.bytes, st, tmQ, tmQt, tmKV, tmKVt, rel_h, rel_w, s, heads,
             static_cast<int>(items), scale_log2e, out);
  return 0;
}

// Warps of a one-CTA-per-unit block, and the shared memory that still lets two such CTAs share an SM
// (228 KB per SM, 1 KB reserved per CTA).  A full 14 x 14 window is 13 m-tiles: 5 warps walk them in three
// rounds (13 of 15 slots used, 4 warps 13 of 16) at 10 warps per SM; 6 warps need a fourth of the time for one
// tile, and 7 warps (two rounds) would have to fit 146 registers and spill.  At head dim 80 only 4 warps'
// scratch fits (8 warps per SM).
template <int HD> constexpr int kAuWarps = HD == 64 ? 5 : 4;
constexpr int kAuMaxBytes = (228 * 1024) / 2 - 1024;

// The kernel launch_attention_mma runs for (s, win): global blocks whose rings fit take the wgmma kernel, window
// blocks whose window is resident the unit kernel, everything else the streamed kernel.  Ring depths are those of
// the global kernel (0 on the other paths).
enum class AmPath { kUnit = 0, kStreamed = 1, kGlobal = 2 };
struct AmChoice {
  AmPath path;
  int qStages, kvStages;
};
template <int HD>
AmChoice attention_mma_choice(int s, int win) {
  if (win == s) {
    const AgLayout<HD> ag(s);
    if (ag.qStages > 0) return {AmPath::kGlobal, ag.qStages, ag.kvStages};
  }
  const bool resident = win < s && AmLayout<HD>(win).unit_bytes(kAuWarps<HD>) <= kAuMaxBytes;
  return {resident ? AmPath::kUnit : AmPath::kStreamed, 0, 0};
}

template <int HD>
int launch_attention_mma(const __half* qkv, const float* qkv_bias, const float* rel_h, const float* rel_w,
                         int B, int s, int win, int heads, __half* out, cudaStream_t st) {
  using LY = AmLayout<HD>;
  constexpr int NW = kAuWarps<HD>;
  const AmPath path = attention_mma_choice<HD>(s, win).path;
  if (path == AmPath::kGlobal) return launch_attention_global<HD>(qkv, rel_h, rel_w, B, s, heads, out, st);
  const LY ly(win);
  const int nwin = (s + win - 1) / win;
  const float scale_log2e = 1.4426950408889634f / sqrtf(static_cast<float>(HD));
  const bool resident = path == AmPath::kUnit;
  const int w0 = win < s ? win : s;       // real queries of the fullest window: w0 x w0
  const int qblocks = resident ? 1 : ((w0 * w0 + 15) / 16 + kAmWarps - 1) / kAmWarps;
  const long blocks = static_cast<long>(qblocks) * B * nwin * nwin * heads;
  SRB_REQUIRE(blocks <= 2147483647L, "attention: %ld CTAs exceed the grid limit (B=%d s=%d win=%d heads=%d)",
              blocks, B, s, win, heads);
  const unsigned grid = static_cast<unsigned>(blocks);
  if (resident) {
    auto kern = attention_unit_kernel<HD, NW>;
    SRB_TRY(allow_dynamic_smem(kern, ly.unit_bytes(NW)));
    SRB_LAUNCH(kern, grid, NW * 32, ly.unit_bytes(NW), st, qkv, qkv_bias, rel_h, rel_w, s, win, nwin, heads,
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
