// sam_road_b200 :: SAM mask-decoder path (USE_SAM_DECODER: True; reference model.py:260-282,471-488,
// sam/segment_anything/modeling/{mask_decoder.py:112-149, transformer.py:62-240,
// prompt_encoder.py:128-205}).
//   * image side ([B*T,256] tokens): k/v/q projections, the image->token out_proj + norm4 and the
//     ConvTranspose upscaler run on the wgmma GEMM (gemm_ops.cu) with fused LN / GELU epilogues;
//   * token side (4 output tokens per image): the tokens of ALL images form one [4B, 256] fp32 matrix; every
//     linear layer is one small fp32 GEMM over it (weights read once for the whole batch instead of once
//     per image), self-attention / token->image attention (online softmax over T keys) / LayerNorm are
//     small batched kernels.  (The first version ran one thread block per image through the whole layer:
//     2.2 of the decoder's 3.3 ms per 64-tile batch were those latency-bound blocks re-reading the
//     weights.)  Layer 0's self-attention acts on the constant output tokens and is computed once per
//     weight load (sam_decoder_prepare);
//   * the token batch of 1 broadcasts against the B images from the first cross-attention on, and
//     layer 0 REPLACES the queries by its self-attention output (transformer.py:155-161; P6).
#include "common.cuh"
#include "ops.h"

namespace srb {

namespace {

constexpr int kTok = 4;      // iou token + 3 mask tokens
constexpr int kC = 256;
constexpr int kThreads = 256;

// y[tok][n] = sum_k x[tok][k] W[n][k] + b[n]; W row-major [N,K]; x, y in shared memory
__device__ void block_linear(const float* __restrict__ W, const float* __restrict__ b,
                             const float* x, int ldx, float* y, int ldy, int N, int K, bool relu) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  for (int n = warp; n < N; n += nw) {
    float acc[kTok] = {0.f, 0.f, 0.f, 0.f};
    const float* w = W + static_cast<size_t>(n) * K;
    for (int k = lane; k < K; k += 32) {
      const float wv = __ldg(w + k);
#pragma unroll
      for (int t = 0; t < kTok; ++t) acc[t] = fmaf(x[t * ldx + k], wv, acc[t]);
    }
#pragma unroll
    for (int t = 0; t < kTok; ++t) acc[t] = warp_sum(acc[t]);
    if (lane == 0) {
      const float bb = b ? __ldg(b + n) : 0.f;
#pragma unroll
      for (int t = 0; t < kTok; ++t) {
        const float v = acc[t] + bb;
        y[t * ldy + n] = relu ? fmaxf(v, 0.f) : v;
      }
    }
  }
  __syncthreads();
}

// x[tok][:] = LayerNorm(x[tok][:] (+ add[tok][:])) over 256 channels, eps 1e-5 (nn.LayerNorm default)
__device__ void block_add_layernorm(float* x, const float* add, const float* __restrict__ g,
                                    const float* __restrict__ b) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp < kTok) {
    float v[8];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int c = lane + 32 * i;
      v[i] = x[warp * kC + c] + (add ? add[warp * kC + c] : 0.f);
      s += v[i];
    }
    const float mean = warp_sum(s) * (1.0f / kC);
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) q += (v[i] - mean) * (v[i] - mean);
    const float rstd = rsqrtf(warp_sum(q) * (1.0f / kC) + 1e-5f);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int c = lane + 32 * i;
      x[warp * kC + c] = (v[i] - mean) * rstd * __ldg(g + c) + __ldg(b + c);
    }
  }
  __syncthreads();
}

// attention among the 4 tokens themselves (self_attn, internal dim 256 = 8 heads x 32)
__device__ void block_self_attention(const float* q, const float* k, const float* v, float* out) {
  // thread = (token i, channel c) over 4 x 256 = 1024 work items
  for (int idx = threadIdx.x; idx < kTok * kC; idx += blockDim.x) {
    const int i = idx / kC, c = idx % kC, h = c / 32;
    float sc[kTok], mx = -INFINITY;
#pragma unroll
    for (int j = 0; j < kTok; ++j) {
      float a = 0.f;
      for (int d = 0; d < 32; ++d) a = fmaf(q[i * kC + h * 32 + d], k[j * kC + h * 32 + d], a);
      sc[j] = a * 0.17677669529663687f;      // / sqrt(32), applied after QK^T (transformer.py:231-232)
      mx = fmaxf(mx, sc[j]);
    }
    float l = 0.f, o = 0.f;
#pragma unroll
    for (int j = 0; j < kTok; ++j) {
      const float p = expf(sc[j] - mx);
      l += p;
      o = fmaf(p, v[j * kC + c], o);
    }
    out[idx] = o / l;
  }
  __syncthreads();
}

struct AttnW {       // one transformer.py Attention module (fp32, token side)
  const float *qw, *qb, *kw, *kb, *vw, *vb, *ow, *ob;
};
struct SamLayerW {
  AttnW self_attn, t2i, i2t;
  const float *n1g, *n1b, *n2g, *n2b, *n3g, *n3b;
  const float *l1w, *l1b, *l2w, *l2b;
};

// ------------------------------------------------------------------------------------------------
// layer-0 self-attention on the (batch independent) output tokens: queries0 = norm1(self_attn(tok))
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads)
sam_tokens_init_kernel(const float* __restrict__ tokens, AttnW w, const float* n1g, const float* n1b,
                       float* __restrict__ q0) {
  __shared__ float x[kTok * kC], q[kTok * kC], k[kTok * kC], v[kTok * kC], a[kTok * kC];
  for (int i = threadIdx.x; i < kTok * kC; i += blockDim.x) x[i] = tokens[i];
  __syncthreads();
  block_linear(w.qw, w.qb, x, kC, q, kC, kC, kC, false);
  block_linear(w.kw, w.kb, x, kC, k, kC, kC, kC, false);
  block_linear(w.vw, w.vb, x, kC, v, kC, kC, kC, false);
  block_self_attention(q, k, v, a);
  block_linear(w.ow, w.ob, a, kC, x, kC, kC, kC, false);        // queries = attn_out (no residual)
  block_add_layernorm(x, nullptr, n1g, n1b);
  for (int i = threadIdx.x; i < kTok * kC; i += blockDim.x) q0[i] = x[i];
}

struct SamFinalW {
  AttnW attn;
  const float *ng, *nb;
  const float* hw[2][3];   // hypernetwork MLP i+1: layers 0..2 weights
  const float* hb[2][3];
};

// ------------------------------------------------------------------------------------------------
// batched token side: every kernel below works on the [Bt = 4B, C] fp32 token matrix of all images
// ------------------------------------------------------------------------------------------------
// out[m][n] = act(sum_k (A[m][k] + pe[m % 4][k]) * W[n][k] + b[n]); fp32 SIMT.  A CTA owns a 32 x 64 output
// tile (2 x 4 outputs per thread); the k dimension is walked in slabs of 16 through shared memory, each
// thread fetching one float4 of W (and half the threads one of A) for the NEXT slab before it computes the
// current one, so the global-load latency hides under the FMAs.  K % 4 == 0; pe may be null.
__global__ void __launch_bounds__(256)
tok_gemm_kernel(const float* __restrict__ A, int lda, const float* __restrict__ pe, int ldpe,
                const float* __restrict__ W, const float* __restrict__ bias, int M, int N, int K, int relu,
                float* __restrict__ out, int ldo) {
  __shared__ float As[2][16][32 + 1], Ws[2][16][64 + 1];
  const int m0 = blockIdx.y * 32, n0 = blockIdx.x * 64;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;      // 16 x 16 threads: rows ty*2.., cols tx*4..
  const int lr = threadIdx.x >> 2, lk = (threadIdx.x & 3) * 4;  // loader: row lr (0..63), k offset lk
  float acc[2][4];
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  auto fetch = [&](int k0, float4& a, float4& w) {
    a = make_float4(0.f, 0.f, 0.f, 0.f);
    w = a;
    const int k = k0 + lk;
    if (k < K) {
      if (lr < 32 && m0 + lr < M) {
        a = *reinterpret_cast<const float4*>(A + static_cast<size_t>(m0 + lr) * lda + k);
        if (pe) {
          const float4 p4 = __ldg(reinterpret_cast<const float4*>(pe + ((m0 + lr) & 3) * ldpe + k));
          a.x += p4.x; a.y += p4.y; a.z += p4.z; a.w += p4.w;
        }
      }
      if (n0 + lr < N) w = __ldg(reinterpret_cast<const float4*>(W + static_cast<size_t>(n0 + lr) * K + k));
    }
  };
  auto stash = [&](int buf, const float4& a, const float4& w) {
    if (lr < 32) { As[buf][lk][lr] = a.x; As[buf][lk + 1][lr] = a.y; As[buf][lk + 2][lr] = a.z; As[buf][lk + 3][lr] = a.w; }
    Ws[buf][lk][lr] = w.x; Ws[buf][lk + 1][lr] = w.y; Ws[buf][lk + 2][lr] = w.z; Ws[buf][lk + 3][lr] = w.w;
  };
  float4 a4, w4;
  fetch(0, a4, w4);
  stash(0, a4, w4);
  __syncthreads();
  const int nslab = (K + 15) / 16;
  for (int sI = 0; sI < nslab; ++sI) {
    const int buf = sI & 1;
    if (sI + 1 < nslab) fetch((sI + 1) * 16, a4, w4);          // in flight while this slab is multiplied
#pragma unroll
    for (int kk = 0; kk < 16; ++kk) {
      const float a0 = As[buf][kk][ty * 2], a1 = As[buf][kk][ty * 2 + 1];
      float w[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) w[j] = Ws[buf][kk][tx * 4 + j];
#pragma unroll
      for (int j = 0; j < 4; ++j) { acc[0][j] = fmaf(a0, w[j], acc[0][j]); acc[1][j] = fmaf(a1, w[j], acc[1][j]); }
    }
    if (sI + 1 < nslab) stash(buf ^ 1, a4, w4);
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int m = m0 + ty * 2 + i;
    if (m >= M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx * 4 + j;
      if (n >= N) continue;
      const float v = acc[i][j] + (bias ? __ldg(bias + n) : 0.f);
      out[static_cast<size_t>(m) * ldo + n] = relu ? fmaxf(v, 0.f) : v;
    }
  }
}

int tok_gemm(const float* A, int lda, const float* pe, const float* W, const float* bias, int M, int N, int K,
             bool relu, float* out, int ldo, cudaStream_t st) {
  if (M <= 0) return 0;
  SRB_REQUIRE(K % 4 == 0 && lda % 4 == 0 && (reinterpret_cast<uintptr_t>(A) & 15u) == 0,
              "tok_gemm: K=%d lda=%d must be multiples of 4 and A 16-byte aligned", K, lda);
  dim3 grid((N + 63) / 64, (M + 31) / 32);
  SRB_LAUNCH(tok_gemm_kernel, grid, 256, 0, st, A, lda, pe, kC, W, bias, M, N, K, relu ? 1 : 0, out, ldo);
  return 0;
}

// x[m][:] = LayerNorm(x[m][:] + add[m][:]) over 256 channels, eps 1e-5; one warp per row.  When
// x_bcast != null the input row is x_bcast[m % 4] (layer 0: the same queries for every image).
__global__ void __launch_bounds__(256)
tok_add_layernorm_kernel(float* __restrict__ x, const float* __restrict__ x_bcast, const float* __restrict__ add,
                         const float* __restrict__ g, const float* __restrict__ b, int M) {
  const int m = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (m >= M) return;
  const float* xin = x_bcast ? x_bcast + (m & 3) * kC : x + static_cast<size_t>(m) * kC;
  float v[8], s = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int c = lane + 32 * i;
    v[i] = xin[c] + (add ? add[static_cast<size_t>(m) * kC + c] : 0.f);
    s += v[i];
  }
  const float mean = warp_sum(s) * (1.0f / kC);
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) q += (v[i] - mean) * (v[i] - mean);
  const float rstd = rsqrtf(warp_sum(q) * (1.0f / kC) + 1e-5f);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int c = lane + 32 * i;
    x[static_cast<size_t>(m) * kC + c] = (v[i] - mean) * rstd * __ldg(g + c) + __ldg(b + c);
  }
}

// x[m][:] = src[m % 4][:]  (layer 0 starts from the same queries for every image)
__global__ void tok_broadcast_kernel(const float* __restrict__ src, long total, float* __restrict__ x) {
  const long idx = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx < total) x[idx] = src[idx % (kTok * kC)];
}

// self-attention among the 4 tokens of every image: q, k, v [Bt][256] -> out [Bt][256] (8 heads x 32)
__global__ void __launch_bounds__(256)
tok_self_attention_kernel(const float* __restrict__ q, const float* __restrict__ k, const float* __restrict__ v,
                          long total, float* __restrict__ out) {
  const long idx = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;    // (row m, channel c)
  if (idx >= total) return;
  const long m = idx / kC;
  const int c = static_cast<int>(idx % kC), h = c / 32;
  const long base = (m & ~3L) * kC;                         // first token row of this image
  float sc[kTok], mx = -INFINITY;
#pragma unroll
  for (int j = 0; j < kTok; ++j) {
    float a = 0.f;
    for (int d = 0; d < 32; ++d) a = fmaf(q[m * kC + h * 32 + d], k[base + j * kC + h * 32 + d], a);
    sc[j] = a * 0.17677669529663687f;      // / sqrt(32), applied after QK^T (transformer.py:231-232)
    mx = fmaxf(mx, sc[j]);
  }
  float l = 0.f, o = 0.f;
#pragma unroll
  for (int j = 0; j < kTok; ++j) {
    const float p = expf(sc[j] - mx);
    l += p;
    o = fmaf(p, v[base + j * kC + c], o);
  }
  out[idx] = o / l;
}

// token -> image attention, one CTA per (image, head): 4 tokens x 64 key partitions = 256 threads, online
// softmax per partition, then a shared-memory merge of the 64 partitions of each token.  q [Bt][128]
// (projected queries), K32 / V32 [B*T][128] fp32, 8 heads x 16; out [Bt][128].
__global__ void __launch_bounds__(kThreads)
tok_t2i_attention_kernel(const float* __restrict__ qg, const float* __restrict__ K32,
                         const float* __restrict__ V32, int T, float* __restrict__ out) {
  __shared__ float red[kTok][64][18];
  const int b = blockIdx.x, h = blockIdx.y;
  const int i = threadIdx.x >> 6, part = threadIdx.x & 63;
  const float* K = K32 + static_cast<size_t>(b) * T * 128 + h * 16;
  const float* V = V32 + static_cast<size_t>(b) * T * 128 + h * 16;
  float q[16];
#pragma unroll
  for (int d = 0; d < 16; ++d) q[d] = qg[(static_cast<size_t>(b) * kTok + i) * 128 + h * 16 + d] * 0.25f;   // / sqrt(16)
  float m = -INFINITY, l = 0.f, o[16];
#pragma unroll
  for (int d = 0; d < 16; ++d) o[d] = 0.f;
  for (int t = part; t < T; t += 64) {
    const float4* kp = reinterpret_cast<const float4*>(K + static_cast<size_t>(t) * 128);
    float sc = 0.f;
#pragma unroll
    for (int d4 = 0; d4 < 4; ++d4) {
      const float4 kv = __ldg(kp + d4);
      sc = fmaf(q[4 * d4], kv.x, sc); sc = fmaf(q[4 * d4 + 1], kv.y, sc);
      sc = fmaf(q[4 * d4 + 2], kv.z, sc); sc = fmaf(q[4 * d4 + 3], kv.w, sc);
    }
    const float mn = fmaxf(m, sc);
    const float a = expf(m - mn), p = expf(sc - mn);
    l = l * a + p;
    const float4* vp = reinterpret_cast<const float4*>(V + static_cast<size_t>(t) * 128);
#pragma unroll
    for (int d4 = 0; d4 < 4; ++d4) {
      const float4 vv = __ldg(vp + d4);
      o[4 * d4] = fmaf(p, vv.x, o[4 * d4] * a); o[4 * d4 + 1] = fmaf(p, vv.y, o[4 * d4 + 1] * a);
      o[4 * d4 + 2] = fmaf(p, vv.z, o[4 * d4 + 2] * a); o[4 * d4 + 3] = fmaf(p, vv.w, o[4 * d4 + 3] * a);
    }
    m = mn;
  }
  float* r = red[i][part];
  r[0] = m; r[1] = l;
#pragma unroll
  for (int d = 0; d < 16; ++d) r[2 + d] = o[d];
  __syncthreads();
  if (part < 16) {          // thread (token i, channel part) merges the 64 partitions for its channel
    float Mx = -INFINITY;
    for (int pp = 0; pp < 64; ++pp) Mx = fmaxf(Mx, red[i][pp][0]);
    float L = 0.f, O = 0.f;
    for (int pp = 0; pp < 64; ++pp) {
      const float a = red[i][pp][0] == -INFINITY ? 0.f : expf(red[i][pp][0] - Mx);
      L = fmaf(red[i][pp][1], a, L);
      O = fmaf(red[i][pp][2 + part], a, O);
    }
    out[(static_cast<size_t>(b) * kTok + i) * 128 + h * 16 + part] = O / L;
  }
}

// ------------------------------------------------------------------------------------------------
// image side elementwise kernels
// ------------------------------------------------------------------------------------------------
// keys32[m][c] = emb_nchw[b][c][t] + no_mask_embed[c]  (mask_decoder.py:126-127 with the dense prompt
// of prompt_encoder.py:164-166)
__global__ void sam_keys_init_kernel(const float* __restrict__ emb, const float* __restrict__ nme, int T,
                                     long total, float* __restrict__ keys) {
  const long idx = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int c = static_cast<int>(idx % kC);
  const long m = idx / kC;
  const int t = static_cast<int>(m % T);
  const long b = m / T;
  keys[idx] = emb[(b * kC + c) * T + t] + __ldg(nme + c);
}
// ka16 = fp16(keys + pe[t]), va16 = fp16(keys)
__global__ void sam_keys_prep_kernel(const float* __restrict__ keys, const float* __restrict__ pe, int T,
                                     long total, __half* __restrict__ ka16, __half* __restrict__ va16) {
  const long idx = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int c = static_cast<int>(idx % kC);
  const int t = static_cast<int>((idx / kC) % T);
  const float v = keys[idx];
  ka16[idx] = __float2half_rn(v + __ldg(pe + static_cast<size_t>(t) * kC + c));
  va16[idx] = __float2half_rn(v);
}
// image -> token attention per image token: softmax over the 4 tokens (8 heads x 16), out fp16 [M,128]
__global__ void sam_i2t_attention_kernel(const float* __restrict__ q32 /* [M][128] */,
                                         const float* __restrict__ k4, const float* __restrict__ v4,
                                         int T, long M, __half* __restrict__ out) {
  const long idx = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;   // (m, head)
  if (idx >= M * 8) return;
  const int h = static_cast<int>(idx & 7);
  const long m = idx >> 3;
  const long b = m / T;
  const float4* qp = reinterpret_cast<const float4*>(q32 + m * 128 + h * 16);
  float q[16];
#pragma unroll
  for (int d4 = 0; d4 < 4; ++d4) {
    const float4 f = qp[d4];
    q[4 * d4] = f.x; q[4 * d4 + 1] = f.y; q[4 * d4 + 2] = f.z; q[4 * d4 + 3] = f.w;
  }
  float sc[kTok], mx = -INFINITY;
#pragma unroll
  for (int j = 0; j < kTok; ++j) {
    const float* kp = k4 + (b * kTok + j) * 128 + h * 16;
    float a = 0.f;
#pragma unroll
    for (int d = 0; d < 16; ++d) a = fmaf(q[d], __ldg(kp + d), a);
    sc[j] = a * 0.25f;
    mx = fmaxf(mx, sc[j]);
  }
  float l = 0.f, o[16];
#pragma unroll
  for (int d = 0; d < 16; ++d) o[d] = 0.f;
#pragma unroll
  for (int j = 0; j < kTok; ++j) {
    const float p = expf(sc[j] - mx);
    l += p;
    const float* vp = v4 + (b * kTok + j) * 128 + h * 16;
#pragma unroll
    for (int d = 0; d < 16; ++d) o[d] = fmaf(p, __ldg(vp + d), o[d]);
  }
  const float inv = 1.0f / l;
  __half* op = out + m * 128 + h * 16;
#pragma unroll
  for (int d = 0; d < 16; d += 2) *reinterpret_cast<uint32_t*>(op + d) = pack_half2(o[d] * inv, o[d + 1] * inv);
}
// low-res masks: rows of U2 [16M, 32] (pixel hierarchy r = ((b*s*s + i*s + j)*4 + d1)*4 + d2) dotted with
// hyper[b][k][32] -> lr[b][y][x][k] at 4s x 4s resolution
__global__ void sam_lowres_masks_kernel(const __half* __restrict__ u2, const float* __restrict__ hyper,
                                        int s, long rows, float* __restrict__ lr) {
  const long r = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (r >= rows) return;
  const int d2 = static_cast<int>(r & 3), d1 = static_cast<int>((r >> 2) & 3);
  const long pix = r >> 4;
  const long b = pix / (s * s);
  const int ij = static_cast<int>(pix % (s * s));
  const int i = ij / s, j = ij % s;
  const int y = (i * 2 + (d1 >> 1)) * 2 + (d2 >> 1), x = (j * 2 + (d1 & 1)) * 2 + (d2 & 1);
  float a0 = 0.f, a1 = 0.f;
  const __half* up = u2 + r * 32;
  const float* h0 = hyper + b * 64;
#pragma unroll
  for (int c = 0; c < 32; ++c) {
    const float u = __half2float(up[c]);
    a0 = fmaf(u, __ldg(h0 + c), a0);
    a1 = fmaf(u, __ldg(h0 + 32 + c), a1);
  }
  const int S4 = 4 * s;
  float* o = lr + ((b * S4 + y) * S4 + x) * 2;
  o[0] = a0; o[1] = a1;
}
// F.interpolate(..., (P,P), bilinear, align_corners=False) of [B,4s,4s,2] by 4 + sigmoid -> NHWC [B,P,P,2]
__global__ void sam_upsample4_kernel(const float* __restrict__ lr, int S4, long total, float* __restrict__ logits,
                                     float* __restrict__ scores) {
  const long idx = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;   // (b, y, x)
  if (idx >= total) return;
  const int P = S4 * 4;
  const int x = static_cast<int>(idx % P), y = static_cast<int>((idx / P) % P);
  const long b = idx / (static_cast<long>(P) * P);
  // source coordinate: (dst + 0.5) * (in/out) - 0.5, clamped at 0 (torch upsample_bilinear2d)
  const float sy = fmaxf((y + 0.5f) * 0.25f - 0.5f, 0.f), sx = fmaxf((x + 0.5f) * 0.25f - 0.5f, 0.f);
  const int y0 = static_cast<int>(sy), x0 = static_cast<int>(sx);
  const int y1 = min(y0 + 1, S4 - 1), x1 = min(x0 + 1, S4 - 1);
  const float ly = sy - y0, lx = sx - x0;
  const float* base = lr + b * S4 * S4 * 2;
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    const float v00 = base[(y0 * S4 + x0) * 2 + k], v01 = base[(y0 * S4 + x1) * 2 + k];
    const float v10 = base[(y1 * S4 + x0) * 2 + k], v11 = base[(y1 * S4 + x1) * 2 + k];
    const float v = (1.f - ly) * ((1.f - lx) * v00 + lx * v01) + ly * ((1.f - lx) * v10 + lx * v11);
    if (logits) logits[idx * 2 + k] = v;
    if (scores) scores[idx * 2 + k] = 1.0f / (1.0f + expf(-v));
  }
}

}  // namespace

struct SamDecoderWs {
  float* keys32; __half* ka16; __half* va16; float* K32; float* V32; float* Q32; __half* att16;
  float* X; float* T0; float* T1; float* T2; float* T3; float* Hd; float* Qc; float* A2;
  float* k4; float* v4; float* hyper; __half* u1; __half* u2; float* lr;
  size_t total;
};

SamDecoderWs layout_sam_decoder(int B, int T, void* base) {
  const size_t M = static_cast<size_t>(B) * T;
  const size_t Bts = static_cast<size_t>(B) * 4;
  Layout L(base, 1024);
  SamDecoderWs b;
  b.keys32 = L.take<float>(M * 256);
  b.ka16 = L.take<__half>(M * 256);
  b.va16 = L.take<__half>(M * 256);
  b.K32 = L.take<float>(M * 128);
  b.V32 = L.take<float>(M * 128);
  b.Q32 = L.take<float>(M * 128);
  b.att16 = L.take<__half>(M * 128);
  b.X = L.take<float>(Bts * 256);
  b.T0 = L.take<float>(Bts * 256);
  b.T1 = L.take<float>(Bts * 256);
  b.T2 = L.take<float>(Bts * 256);
  b.T3 = L.take<float>(Bts * 256);
  b.Hd = L.take<float>(Bts * 2048);
  b.Qc = L.take<float>(Bts * 128);
  b.A2 = L.take<float>(Bts * 128);
  b.k4 = L.take<float>(Bts * 128);
  b.v4 = L.take<float>(Bts * 128);
  b.hyper = L.take<float>(static_cast<size_t>(B) * 64);
  b.u1 = L.take<__half>(M * 256);
  b.u2 = L.take<__half>(M * 4 * 128);
  b.lr = L.take<float>(M * 16 * 2);
  b.total = L.bytes();
  return b;
}

size_t sam_decoder_ws_bytes(int B, int T) { return layout_sam_decoder(B, T, nullptr).total; }

int sam_decoder_checkpoints(int B, int T, void* ws, float* queries, float* keys, float* hyper, float* lowres,
                            cudaStream_t st) {
  const SamDecoderWs b = layout_sam_decoder(B, T, ws);
  const size_t M = static_cast<size_t>(B) * T;
  const struct { float* dst; const float* src; size_t n; } cp[] = {
      {queries, b.X, static_cast<size_t>(B) * kTok * kC}, {keys, b.keys32, M * kC},
      {hyper, b.hyper, static_cast<size_t>(B) * 64}, {lowres, b.lr, M * 16 * 2}};
  for (const auto& c : cp)
    if (c.dst) SRB_CUDA_OK(cudaMemcpyAsync(c.dst, c.src, c.n * sizeof(float), cudaMemcpyDeviceToDevice, st));
  return 0;
}

int sam_decoder_forward(const SamDecoderWeights& W, const float* emb_nchw, int B, int s, int P, void* ws,
                        float* mask_scores, float* mask_logits, cudaStream_t st) {
  const int T = s * s;
  const long M = static_cast<long>(B) * T;
  auto cv = [](const SamAttnW& a) { return AttnW{a.qw, a.qb, a.kw, a.kb, a.vw, a.vb, a.ow, a.ob}; };
  struct {
    const float *tokens, *no_mask_embed, *dense_pe;
    SamLayerW layer[2];
    SamFinalW fin;
    const __half *t2i_kw[3], *t2i_vw[3], *i2t_qw[2], *i2t_ow[2], *up1_w, *up2_w;
    const float *t2i_kb[3], *t2i_vb[3], *i2t_qb[2], *i2t_ob[2], *n4g[2], *n4b[2];
    const float *up1_b, *up1_g, *up1_beta, *up2_b;
  } w;
  w.tokens = W.tokens; w.no_mask_embed = W.no_mask_embed; w.dense_pe = W.dense_pe;
  for (int l = 0; l < 2; ++l) {
    w.layer[l] = SamLayerW{cv(W.self_attn[l]), cv(W.t2i[l]), cv(W.i2t[l]), W.n1g[l], W.n1b[l], W.n2g[l],
                           W.n2b[l], W.n3g[l], W.n3b[l], W.l1w[l], W.l1b[l], W.l2w[l], W.l2b[l]};
    w.t2i_kw[l] = W.t2i_kw16[l]; w.t2i_vw[l] = W.t2i_vw16[l];
    w.t2i_kb[l] = W.t2i[l].kb; w.t2i_vb[l] = W.t2i[l].vb;
    w.i2t_qw[l] = W.i2t_qw16[l]; w.i2t_ow[l] = W.i2t_ow16[l];
    w.i2t_qb[l] = W.i2t[l].qb; w.i2t_ob[l] = W.i2t[l].ob;
    w.n4g[l] = W.n4g[l]; w.n4b[l] = W.n4b[l];
  }
  w.t2i_kw[2] = W.t2i_kw16[2]; w.t2i_vw[2] = W.t2i_vw16[2];
  w.t2i_kb[2] = W.final_attn.kb; w.t2i_vb[2] = W.final_attn.vb;
  w.fin.attn = cv(W.final_attn); w.fin.ng = W.nfg; w.fin.nb = W.nfb;
  for (int mi = 0; mi < 2; ++mi)
    for (int j = 0; j < 3; ++j) { w.fin.hw[mi][j] = W.hw[mi][j]; w.fin.hb[mi][j] = W.hb[mi][j]; }
  w.up1_w = W.up1_w; w.up2_w = W.up2_w; w.up1_b = W.up1_b; w.up1_g = W.up1_g; w.up1_beta = W.up1_beta;
  w.up2_b = W.up2_b;
  const SamDecoderWs b = layout_sam_decoder(B, T, ws);

  SRB_REQUIRE(W.q0 != nullptr, "SAM decoder: weights not prepared (sam_decoder_prepare)");
  const int Mi = static_cast<int>(M);
  const int Bt = 4 * B;
  const float* pe = w.tokens;            // query_pe = the output tokens themselves (transformer.py:95,101)
  auto LN = [&](float* x, const float* add, const float* g, const float* bb) -> int {
    SRB_LAUNCH(tok_add_layernorm_kernel, (Bt + 7) / 8, 256, 0, st, x, nullptr, add, g, bb, Bt);
    return 0;
  };
  auto t2i = [&](const AttnW& a, const float* g, const float* bb) -> int {
    // queries = norm(queries + out_proj(softmax(q_proj(queries + pe) K^T / 4) V))   (transformer.py:168-172,99-104)
    if (int rc = tok_gemm(b.X, kC, pe, a.qw, a.qb, Bt, 128, kC, false, b.Qc, 128, st)) return rc;
    SRB_LAUNCH(tok_t2i_attention_kernel, dim3(B, 8), kThreads, 0, st, b.Qc, b.K32, b.V32, T, b.A2);
    if (int rc = tok_gemm(b.A2, 128, nullptr, a.ow, a.ob, Bt, kC, 128, false, b.T1, kC, st)) return rc;
    SRB_TRY(LN(b.X, b.T1, g, bb));
    return 0;
  };

  SRB_LAUNCH(sam_keys_init_kernel, blocks_for(M * 256, 256), 256, 0, st, emb_nchw, w.no_mask_embed, T, M * 256,
             b.keys32);
  SRB_LAUNCH(tok_broadcast_kernel, blocks_for(static_cast<long>(Bt) * kC, 256), 256, 0, st, W.q0,
             static_cast<long>(Bt) * kC, b.X);
  for (int l = 0; l < 2; ++l) {
    const SamLayerW& L = w.layer[l];
    SRB_LAUNCH(sam_keys_prep_kernel, blocks_for(M * 256, 256), 256, 0, st, b.keys32, w.dense_pe, T, M * 256, b.ka16,
               b.va16);
    if (int rc = gemm_f32out(b.ka16, 256, w.t2i_kw[l], 256, Mi, 128, 256, w.t2i_kb[l], nullptr, nullptr, 0, b.K32, 128, st)) return rc;
    if (int rc = gemm_f32out(b.va16, 256, w.t2i_vw[l], 256, Mi, 128, 256, w.t2i_vb[l], nullptr, nullptr, 0, b.V32, 128, st)) return rc;
    if (int rc = gemm_f32out(b.ka16, 256, w.i2t_qw[l], 256, Mi, 128, 256, w.i2t_qb[l], nullptr, nullptr, 0, b.Q32, 128, st)) return rc;
    if (l > 0) {   // q = k = queries + pe, v = queries; queries = norm1(queries + attn)  (transformer.py:162-166)
      if (int rc = tok_gemm(b.X, kC, pe, L.self_attn.qw, L.self_attn.qb, Bt, kC, kC, false, b.T1, kC, st)) return rc;
      if (int rc = tok_gemm(b.X, kC, pe, L.self_attn.kw, L.self_attn.kb, Bt, kC, kC, false, b.T2, kC, st)) return rc;
      if (int rc = tok_gemm(b.X, kC, nullptr, L.self_attn.vw, L.self_attn.vb, Bt, kC, kC, false, b.T3, kC, st)) return rc;
      SRB_LAUNCH(tok_self_attention_kernel, blocks_for(static_cast<long>(Bt) * kC, 256), 256, 0, st, b.T1, b.T2, b.T3,
                 static_cast<long>(Bt) * kC, b.T0);
      if (int rc = tok_gemm(b.T0, kC, nullptr, L.self_attn.ow, L.self_attn.ob, Bt, kC, kC, false, b.T1, kC, st)) return rc;
      SRB_TRY(LN(b.X, b.T1, L.n1g, L.n1b));
    }
    if (int rc = t2i(L.t2i, L.n2g, L.n2b)) return rc;
    // MLP (transformer.py:174-177): queries = norm3(queries + lin2(relu(lin1(queries))))
    if (int rc = tok_gemm(b.X, kC, nullptr, L.l1w, L.l1b, Bt, 2048, kC, true, b.Hd, 2048, st)) return rc;
    if (int rc = tok_gemm(b.Hd, 2048, nullptr, L.l2w, L.l2b, Bt, kC, 2048, false, b.T1, kC, st)) return rc;
    SRB_TRY(LN(b.X, b.T1, L.n3g, L.n3b));
    // image -> token attention (transformer.py:179-182): k = k_proj(queries + pe), v = v_proj(queries)
    if (int rc = tok_gemm(b.X, kC, pe, L.i2t.kw, L.i2t.kb, Bt, 128, kC, false, b.k4, 128, st)) return rc;
    if (int rc = tok_gemm(b.X, kC, nullptr, L.i2t.vw, L.i2t.vb, Bt, 128, kC, false, b.v4, 128, st)) return rc;
    SRB_LAUNCH(sam_i2t_attention_kernel, blocks_for(M * 8, 256), 256, 0, st, b.Q32, b.k4, b.v4, T, M, b.att16);
    // keys = norm4(keys + out_proj(attn))
    if (int rc = gemm_ln(b.att16, 128, w.i2t_ow[l], 128, Mi, 256, 128, w.i2t_ob[l], b.keys32, w.n4g[l], w.n4b[l],
                         1e-5f, 256, ACT_NONE, nullptr, b.keys32, nullptr, 1, 256, st)) return rc;
  }
  // final token -> image attention + norm_final_attn (transformer.py:99-106), then the hypernetwork MLPs
  SRB_LAUNCH(sam_keys_prep_kernel, blocks_for(M * 256, 256), 256, 0, st, b.keys32, w.dense_pe, T, M * 256, b.ka16,
             b.va16);
  if (int rc = gemm_f32out(b.ka16, 256, w.t2i_kw[2], 256, Mi, 128, 256, w.t2i_kb[2], nullptr, nullptr, 0, b.K32, 128, st)) return rc;
  if (int rc = gemm_f32out(b.va16, 256, w.t2i_vw[2], 256, Mi, 128, 256, w.t2i_vb[2], nullptr, nullptr, 0, b.V32, 128, st)) return rc;
  if (int rc = t2i(w.fin.attn, w.fin.ng, w.fin.nb)) return rc;
  // hypernetworks of mask tokens 1 and 2 (rows 2 and 3 of every image; multimask_output keeps masks [1:],
  // mask_decoder.py:102-106,137-141): three small GEMMs each over the B rows of that token
  for (int mi = 0; mi < 2; ++mi) {
    const float* rows = b.X + (2 + mi) * kC;
    if (int rc = tok_gemm(rows, kTok * kC, nullptr, w.fin.hw[mi][0], w.fin.hb[mi][0], B, kC, kC, true, b.T0, kC, st)) return rc;
    if (int rc = tok_gemm(b.T0, kC, nullptr, w.fin.hw[mi][1], w.fin.hb[mi][1], B, kC, kC, true, b.T2, kC, st)) return rc;
    if (int rc = tok_gemm(b.T2, kC, nullptr, w.fin.hw[mi][2], w.fin.hb[mi][2], B, 32, kC, false, b.hyper + mi * 32, 64, st)) return rc;
  }
  // upscaler: ConvT(256->64)+LN2d+GELU, ConvT(64->32)+GELU as GEMMs (va16 = fp16(keys))
  if (int rc = gemm_ln(b.va16, 256, w.up1_w, 256, Mi, 256, 256, w.up1_b, nullptr, w.up1_g, w.up1_beta, 1e-6f, 64,
                       ACT_GELU, b.u1, nullptr, nullptr, 1, 256, st)) return rc;
  if (int rc = gemm_f16out(b.u1, 64, w.up2_w, 64, 4 * Mi, 128, 64, w.up2_b, ACT_GELU, b.u2, 128, st)) return rc;
  SRB_LAUNCH(sam_lowres_masks_kernel, blocks_for(16 * M, 256), 256, 0, st, b.u2, b.hyper, s, 16 * M, b.lr);
  SRB_LAUNCH(sam_upsample4_kernel, blocks_for(static_cast<long>(B) * P * P, 256), 256, 0, st, b.lr, 4 * s,
             static_cast<long>(B) * P * P, mask_logits, mask_scores);
  return 0;
}

// Layer 0's self-attention block acts on the constant output tokens (the token batch is 1 and has no
// positional term in layer 0, transformer.py:155-161): queries0 = norm1(self_attn(tokens)), computed once
// per weight load into q0 [4][256].
int sam_decoder_prepare(const SamDecoderWeights& W, float* q0, cudaStream_t st) {
  AttnW a{W.self_attn[0].qw, W.self_attn[0].qb, W.self_attn[0].kw, W.self_attn[0].kb,
          W.self_attn[0].vw, W.self_attn[0].vb, W.self_attn[0].ow, W.self_attn[0].ob};
  SRB_LAUNCH(sam_tokens_init_kernel, 1, kThreads, 0, st, W.tokens, a, W.n1g[0], W.n1b[0], q0);
  return 0;
}

}  // namespace srb
