// sam_road_b200 :: tensor-core encoder attention (head_dim 64 or 80), windowed or global, with the
// decomposed relative-position bias.  Same semantics as the SIMT kernel in attention.cu.
//
// One CTA = 64 query tokens of one (image, window, head) unit, all on grid.x; 4 warps, 16 query rows each.
//   prologue : Q tile (fp16) and the rel-pos tables (fp32, row pitch HD + 1: lanes reading
//              consecutive rows hit distinct banks) -> smem; per query the rel-pos dot products
//              relh[q][kh] = q . rel_pos_h[qh - kh + win - 1], relw[q][kw] = q . rel_pos_w[qw - kw + win - 1]
//              in fp32 (unscaled q, image_encoder.py:325-361) -> smem
//   main loop: 64-key chunks of K and V (fp16) -> smem; S = Q K^T on mma.sync m16n8k16 (fp32
//              accumulate), bias added, online softmax in the exp2 domain, P rounded to fp16 and fed
//              from registers into O += P V (V fragments by ldmatrix.trans)
//   epilogue : O / l -> fp16, real query tokens only
// Padded tokens of a window (beyond the s x s grid) have x = 0, so their q = k = v = qkv bias: they
// are real softmax keys, and their query rows are never written.
#pragma once

#include "common.cuh"
#include "ops.h"

namespace srb {

constexpr int kAmThreads = 128;
constexpr int kAmQ = 64;          // query rows per CTA
constexpr int kAmKC = 64;         // keys per chunk

template <int HD>
struct AmSmem {
  static constexpr int kPitch = HD + 8;                         // halves; ldmatrix rows conflict-free
  static constexpr int kQBytes = kAmQ * kPitch * 2;
  static constexpr int kKBytes = kAmKC * kPitch * 2;
  static constexpr int kKVOffset = kQBytes;                     // K, V chunks; the rel-pos tables before
  static __host__ __device__ int tab_bytes(int win) { return 2 * (2 * win - 1) * (HD + 1) * 4; }
  static __host__ __device__ int kv_bytes(int win) {
    return tab_bytes(win) > 2 * kKBytes ? tab_bytes(win) : 2 * kKBytes;
  }
  static __host__ __device__ int rel_offset(int win) { return kKVOffset + kv_bytes(win); }   // fp32 [kAmQ][2 * win]
  static int bytes(int win) { return rel_offset(win) + kAmQ * 2 * win * 4; }
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

// One token's q/k/v head slice (HD fp16) of window (wy, wx), index t inside the window, or the bias
// when the token is padding.  Writes 8 halves per call (c8 = column / 8).
__device__ __forceinline__ uint4 am_token8(const __half* __restrict__ qkv, const float* __restrict__ qkv_bias,
                                           int b, int s, int win, int wy, int wx, int t, int ld, int col, int c8) {
  const int gy = wy * win + t / win, gx = wx * win + t % win;
  if (gy < s && gx < s)
    return *reinterpret_cast<const uint4*>(qkv + (static_cast<size_t>(b) * s * s + gy * s + gx) * ld + col + c8 * 8);
  uint4 u;
  const float* bp = qkv_bias + col + c8 * 8;
  u.x = pack_half2(__ldg(bp + 0), __ldg(bp + 1));
  u.y = pack_half2(__ldg(bp + 2), __ldg(bp + 3));
  u.z = pack_half2(__ldg(bp + 4), __ldg(bp + 5));
  u.w = pack_half2(__ldg(bp + 6), __ldg(bp + 7));
  return u;
}

template <int HD>
__global__ void __launch_bounds__(kAmThreads)
attention_mma_kernel(const __half* __restrict__ qkv, const float* __restrict__ qkv_bias,
                     const float* __restrict__ rel_h, const float* __restrict__ rel_w, int s, int win,
                     int nwin, int heads, float scale_log2e, __half* __restrict__ out) {
  using SM = AmSmem<HD>;
  constexpr int P = SM::kPitch;
  constexpr int NT = HD / 8;          // n8 tiles of the output
  constexpr int KS = HD / 16;         // k16 steps of Q K^T
  extern __shared__ __align__(16) uint8_t smem_am[];
  __half* sQ = reinterpret_cast<__half*>(smem_am);
  __half* sK = reinterpret_cast<__half*>(smem_am + SM::kKVOffset);
  __half* sV = reinterpret_cast<__half*>(smem_am + SM::kKVOffset + SM::kKBytes);
  float* sTab = reinterpret_cast<float*>(smem_am + SM::kKVOffset);     // [rel_h rows ; rel_w rows][HD + 1]
  float* sRel = reinterpret_cast<float*>(smem_am + SM::rel_offset(win));   // [kAmQ][relh win | relw win]

  const int D = heads * HD, ld = 3 * D;
  const int nkeys = win * win;
  const int qblocks = (nkeys + kAmQ - 1) / kAmQ;
  const int unit = blockIdx.x / qblocks;           // (image, window, head), head fastest
  const int head = unit % heads;
  const int widx = (unit / heads) % (nwin * nwin);
  const int b = unit / (heads * nwin * nwin);
  const int wy = widx / nwin, wx = widx % nwin;
  const int q0 = (blockIdx.x - unit * qblocks) * kAmQ;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

  // ---- Q tile ----
  for (int idx = tid; idx < kAmQ * NT; idx += kAmThreads) {
    const int r = idx / NT, c8 = idx % NT;
    uint4 u = make_uint4(0u, 0u, 0u, 0u);
    if (q0 + r < nkeys) u = am_token8(qkv, qkv_bias, b, s, win, wy, wx, q0 + r, ld, head * HD, c8);
    *reinterpret_cast<uint4*>(sQ + r * P + c8 * 8) = u;
  }
  const int L = 2 * win - 1;
  for (int idx = tid; idx < 2 * L * HD; idx += kAmThreads) {
    const int r = idx / HD, c = idx % HD;
    sTab[r * (HD + 1) + c] = r < L ? __ldg(rel_h + idx) : __ldg(rel_w + idx - L * HD);
  }
  __syncthreads();
  // ---- rel-pos dot products (fp32) ----
  for (int idx = tid; idx < kAmQ * 2 * win; idx += kAmThreads) {
    const int r = idx / (2 * win), j = idx % (2 * win);
    const int qi = q0 + r;
    float acc = 0.f;
    if (qi < nkeys) {
      const int kh = j < win ? j : j - win;
      const int d = (j < win ? qi / win : qi % win) - kh + win - 1;
      const float* tab = sTab + ((j < win ? 0 : L) + d) * (HD + 1);
      const __half2* qr = reinterpret_cast<const __half2*>(sQ + r * P);
#pragma unroll 8
      for (int c = 0; c < HD / 2; ++c) {
        const float2 qf = __half22float2(qr[c]);
        acc = fmaf(qf.x, tab[2 * c], acc);
        acc = fmaf(qf.y, tab[2 * c + 1], acc);
      }
    }
    sRel[idx] = acc * 1.4426950408889634f;        // exp2 domain
  }

  // ---- Q fragments (A operand) ----
  uint32_t qa[KS][4];
  {
    const int r = warp * 16 + (lane & 15);
    const int cofs = (lane >> 4) * 8;
#pragma unroll
    for (int k = 0; k < KS; ++k)
      ldsm_x4(smem_u32(sQ + r * P + k * 16 + cofs), qa[k][0], qa[k][1], qa[k][2], qa[k][3]);
  }
  const int rA = warp * 16 + (lane >> 2);        // this thread's two query rows: rA, rA + 8
  const float* relA = sRel + rA * 2 * win;
  const float* relB = relA + 8 * 2 * win;

  float o[NT][4];
#pragma unroll
  for (int j = 0; j < NT; ++j) o[j][0] = o[j][1] = o[j][2] = o[j][3] = 0.f;
  float mA = -INFINITY, mB = -INFINITY, lA = 0.f, lB = 0.f;

  for (int k0 = 0; k0 < nkeys; k0 += kAmKC) {
    __syncthreads();                               // previous chunk consumed (and sRel written)
    for (int idx = tid; idx < kAmKC * NT; idx += kAmThreads) {
      const int r = idx / NT, c8 = idx % NT;
      uint4 uk = make_uint4(0u, 0u, 0u, 0u), uv = uk;
      if (k0 + r < nkeys) {
        uk = am_token8(qkv, qkv_bias, b, s, win, wy, wx, k0 + r, ld, D + head * HD, c8);
        uv = am_token8(qkv, qkv_bias, b, s, win, wy, wx, k0 + r, ld, 2 * D + head * HD, c8);
      }
      *reinterpret_cast<uint4*>(sK + r * P + c8 * 8) = uk;
      *reinterpret_cast<uint4*>(sV + r * P + c8 * 8) = uv;
    }
    __syncthreads();

    // S = Q K^T : 16 rows x 64 keys per warp
    float sc[kAmKC / 8][4];
#pragma unroll
    for (int n = 0; n < kAmKC / 8; ++n) {
      sc[n][0] = sc[n][1] = sc[n][2] = sc[n][3] = 0.f;
#pragma unroll
      for (int k = 0; k < KS; ++k) {
        uint32_t b0, b1;
        ldsm_x2(smem_u32(sK + (n * 8 + (lane & 7)) * P + k * 16 + ((lane >> 3) & 1) * 8), b0, b1);
        mma_16816(sc[n], qa[k], b0, b1);
      }
    }
    // scale + bias, masking, row maxima
    float cmA = -INFINITY, cmB = -INFINITY;
#pragma unroll
    for (int n = 0; n < kAmKC / 8; ++n) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int kk = k0 + n * 8 + 2 * (lane & 3) + e;
        if (kk < nkeys) {
          const int kh = kk / win, kw = kk - kh * win;
          sc[n][e] = fmaf(sc[n][e], scale_log2e, relA[kh] + relA[win + kw]);
          sc[n][2 + e] = fmaf(sc[n][2 + e], scale_log2e, relB[kh] + relB[win + kw]);
        } else {
          sc[n][e] = -INFINITY;
          sc[n][2 + e] = -INFINITY;
        }
        cmA = fmaxf(cmA, sc[n][e]);
        cmB = fmaxf(cmB, sc[n][2 + e]);
      }
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

  // ---- epilogue ----
#pragma unroll
  for (int off = 1; off <= 2; off <<= 1) {
    lA += __shfl_xor_sync(0xffffffffu, lA, off);
    lB += __shfl_xor_sync(0xffffffffu, lB, off);
  }
  const float invA = 1.0f / lA, invB = 1.0f / lB;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int qi = q0 + rA + 8 * h;
    if (qi >= nkeys) continue;
    const int gy = wy * win + qi / win, gx = wx * win + qi % win;
    if (gy >= s || gx >= s) continue;
    __half* op = out + (static_cast<size_t>(b) * s * s + gy * s + gx) * D + head * HD + 2 * (lane & 3);
    const float inv = h ? invB : invA;
#pragma unroll
    for (int j = 0; j < NT; ++j)
      *reinterpret_cast<uint32_t*>(op + j * 8) = pack_half2(o[j][2 * h] * inv, o[j][2 * h + 1] * inv);
  }
}

template <int HD>
int launch_attention_mma(const __half* qkv, const float* qkv_bias, const float* rel_h, const float* rel_w,
                         int B, int s, int win, int heads, __half* out, cudaStream_t st) {
  const int nwin = (s + win - 1) / win;
  const int smem = AmSmem<HD>::bytes(win);
  auto kern = attention_mma_kernel<HD>;
  static uint64_t attr_devs = 0;          // one bit per CUDA device: function attributes are per device
  if (first_use_on_device(&attr_devs)) {  // the largest window the encoder supports (s <= 64)
    SRB_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, AmSmem<HD>::bytes(64)));
  }
  const long blocks = static_cast<long>((win * win + kAmQ - 1) / kAmQ) * B * nwin * nwin * heads;
  SRB_REQUIRE(blocks <= 2147483647L, "attention: %ld CTAs exceed the grid limit (B=%d s=%d win=%d heads=%d)",
              blocks, B, s, win, heads);
  const unsigned grid = static_cast<unsigned>(blocks);
  const float scale_log2e = 1.4426950408889634f / sqrtf(static_cast<float>(HD));
  kern<<<grid, kAmThreads, smem, st>>>(qkv, qkv_bias, rel_h, rel_w, s, win, nwin, heads, scale_log2e, out);
  SRB_CUDA_OK(cudaGetLastError());
  note_launch();
  return 0;
}

}  // namespace srb
