// sam_road_b200 :: tensor-core encoder attention (head_dim 64 or 80), windowed or global, with the
// decomposed relative-position bias.  Same semantics as the SIMT kernel in attention.cu.
//
// Unit = (image, window, head).  Its real queries (the window's tokens inside the s x s grid, ry x rx
// of them) are numbered j = qh * rx + qw and cut into 16-row m-tiles, one per warp, kAmWarps per CTA;
// a CTA whose m-tiles all lie past the unit's real queries exits at once, so edge windows run only
// the rows they have.  Keys sit in slots k = kh * winP + kw, winP = win rounded up to a power of two
// (>= 8): a 64-key chunk then holds whole key rows, kh = k >> lg and kw = k & (winP - 1) need no
// division, and each n8 tile of scores lies in one key row.
//   prologue : Q tile (fp16) and the rel-pos tables, each fp32 row R split into fp16 hi = fp16(R)
//              and lo = fp16(R - hi) -> smem.  M = Q [hi | lo]^T on mma.sync (both into one fp32
//              accumulator; q is exactly fp16, so this is the fp32 dot product to ~1e-6 relative),
//              and M[q][r] goes to relh[q][kh] with kh = qh - r + win - 1 (relw with qw alike)
//              -> smem, in the exp2 domain.  Entries for kh >= win or kw >= win (slots that are no
//              key of the window) hold -inf, which masks those slots in the bias add.
//   main loop: 64-key chunks of K and V (fp16), double-buffered with cp.async (one barrier per
//              chunk); window padding keys (beyond the s x s grid) are copied from the fp16 qkv bias
//              staged once in smem, non-key slots are zeros.  S = Q K^T on mma.sync m16n8k16 (fp32
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
  int relOffset, padOffset, bytes;
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

// One bit per CUDA device (function attributes are per device) for each head dim.  Internal linkage,
// unlike a static local of the launcher template: two builds of the library loaded into one process
// (tools/attention_bench.py --lib-b) each keep their own flags.
static uint64_t g_am_attr_devs[2] = {0, 0};

template <int HD>
int launch_attention_mma(const __half* qkv, const float* qkv_bias, const float* rel_h, const float* rel_w,
                         int B, int s, int win, int heads, __half* out, cudaStream_t st) {
  using LY = AmLayout<HD>;
  const int nwin = (s + win - 1) / win;
  const int smem = LY(win).bytes;
  auto kern = attention_mma_kernel<HD>;
  if (first_use_on_device(&g_am_attr_devs[HD == 80])) {   // the largest window the encoder supports (s <= 64)
    SRB_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, LY(64).bytes));
  }
  const int w0 = win < s ? win : s;       // real queries of the fullest window: w0 x w0
  const int qblocks = ((w0 * w0 + 15) / 16 + kAmWarps - 1) / kAmWarps;
  const long blocks = static_cast<long>(qblocks) * B * nwin * nwin * heads;
  SRB_REQUIRE(blocks <= 2147483647L, "attention: %ld CTAs exceed the grid limit (B=%d s=%d win=%d heads=%d)",
              blocks, B, s, win, heads);
  const unsigned grid = static_cast<unsigned>(blocks);
  const float scale_log2e = 1.4426950408889634f / sqrtf(static_cast<float>(HD));
  kern<<<grid, kAmWarps * 32, smem, st>>>(qkv, qkv_bias, rel_h, rel_w, s, win, nwin, heads, qblocks, scale_log2e,
                                       out);
  SRB_CUDA_OK(cudaGetLastError());
  note_launch();
  return 0;
}

}  // namespace srb
