// sam_road_b200 :: TopoNet pieces that are not GEMMs (reference: model.py:29-148).
//
//   BilinearSampler.forward   model.py:34-58    grid_sample(bilinear, align_corners=False, zeros)
//   TopoNet.forward           model.py:88-148   gather pairs, pair_proj, 3 post-norm encoder layers
//                                               over sequences of n_pairs with key-padding mask,
//                                               output_proj, sigmoid
//
// pair_proj(concat[src, tgt, offset]) is evaluated as  Ws*f[src] + Wt*f[tgt] + Wo*offset + b  with
// Ws*f and Wt*f computed once per keypoint by a GEMM (16x fewer rows than per pair).
// Eval-mode semantics of torch's nested-tensor fast path are reproduced (SURVEY.md §8a P4): masked
// keys are excluded from the softmax, and masked slots report output_proj(0) = bias.
#include "common.cuh"
#include "ops.h"
#include "toponet_tc.cuh"

namespace srb {

// ------------------------------------------------------------------------------------------------
// Bilinear sampling of image_embeddings [B,C,s,s] fp32 at pixel-space points (x,y):
//   g = pt / P * 2 - 1 (model.py:47) ; grid_sample unnormalise: u = ((g + 1) * s - 1) / 2 ;
//   4 taps, out-of-range taps contribute zero (SURVEY.md §8a P8).  One block per point, one thread
//   per channel.  Output [B*N, C] = A operand of feature_proj: fp16 for inference, fp32 for training.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void store_feature(__half* p, float v) { *p = __float2half_rn(v); }
__device__ __forceinline__ void store_feature(float* p, float v) { *p = v; }

template <typename T>
__global__ void __launch_bounds__(256)
topo_sample_kernel(const float* __restrict__ feat, int C, int s, float P, const void* points,
                   int pts_dtype, int N, T* __restrict__ out) {
  const int pt = blockIdx.x;           // b*N + n
  const int b = pt / N;
  const float px = load_coord(points, pts_dtype, static_cast<size_t>(pt) * 2 + 0);
  const float py = load_coord(points, pts_dtype, static_cast<size_t>(pt) * 2 + 1);
  const float gx = (px / P) * 2.0f - 1.0f;
  const float gy = (py / P) * 2.0f - 1.0f;
  const float ux = ((gx + 1.0f) * static_cast<float>(s) - 1.0f) * 0.5f;
  const float uy = ((gy + 1.0f) * static_cast<float>(s) - 1.0f) * 0.5f;
  const float fx0 = floorf(ux), fy0 = floorf(uy);
  const int x0 = static_cast<int>(fx0), y0 = static_cast<int>(fy0);
  const float tx = ux - fx0, ty = uy - fy0;
  const float w00 = (1.f - tx) * (1.f - ty), w01 = tx * (1.f - ty);
  const float w10 = (1.f - tx) * ty, w11 = tx * ty;
  const bool vx0 = x0 >= 0 && x0 < s, vx1 = x0 + 1 >= 0 && x0 + 1 < s;
  const bool vy0 = y0 >= 0 && y0 < s, vy1 = y0 + 1 >= 0 && y0 + 1 < s;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const float* f = feat + (static_cast<size_t>(b) * C + c) * s * s;
    float acc = 0.f;
    if (vy0 && vx0) acc += f[y0 * s + x0] * w00;
    if (vy0 && vx1) acc += f[y0 * s + x0 + 1] * w01;
    if (vy1 && vx0) acc += f[(y0 + 1) * s + x0] * w10;
    if (vy1 && vx1) acc += f[(y0 + 1) * s + x0 + 1] * w11;
    store_feature(out + static_cast<size_t>(pt) * C + c, acc);
  }
}

template <typename T>
int topo_sample_launch(const float* feat_nchw, int B, int C, int s, int P, const void* points,
                       int pts_dtype, int N, T* out, cudaStream_t st) {
  SRB_REQUIRE(pts_dtype >= 0 && pts_dtype <= 2, "topo_sample: points dtype %d", pts_dtype);
  if (B * N <= 0) return 0;
  topo_sample_kernel<T><<<B * N, 256, 0, st>>>(feat_nchw, C, s, static_cast<float>(P), points,
                                               pts_dtype, N, out);
  SRB_CUDA_OK(cudaGetLastError());
  note_launch();
  return 0;
}

int topo_sample_features(const float* feat_nchw, int B, int C, int s, int P, const void* points,
                         int pts_dtype, int N, __half* out, cudaStream_t st) {
  return topo_sample_launch(feat_nchw, B, C, s, P, points, pts_dtype, N, out, st);
}

int topo_sample_features_f32(const float* feat_nchw, int B, int C, int s, int P, const void* points,
                             int pts_dtype, int N, float* out, cudaStream_t st) {
  return topo_sample_launch(feat_nchw, B, C, s, P, points, pts_dtype, N, out, st);
}

// ------------------------------------------------------------------------------------------------
// Pair features (model.py:96-120):  x = relu(PS[b,src] + PT[b,tgt] + Wo (pt[tgt]-pt[src]) + bias)
//   pst: [B*N, 256] fp32, columns 0..127 = Ws f, 128..255 = Wt f.   One block (128 thr) per token.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128)
topo_pair_kernel(const TopoPairInputs in, float* __restrict__ x32, __half* __restrict__ x16) {
  const size_t tok = blockIdx.x;
  const PairToken pr = resolve_pair(in, tok);
  const int c = threadIdx.x;
  float v = __ldg(in.pst + pr.ps * 256 + c) + __ldg(in.pst + pr.pt * 256 + 128 + c);
  v += __ldg(in.w_off + c * 2 + 0) * pr.ox + __ldg(in.w_off + c * 2 + 1) * pr.oy + __ldg(in.bias + c);
  v = fmaxf(v, 0.f);
  x32[tok * 128 + c] = v;
  x16[tok * 128 + c] = __float2half_rn(v);
}

int topo_pair_features(const TopoPairInputs& in, int tokens, float* x32, __half* x16, cudaStream_t st) {
  SRB_REQUIRE(in.pairs_dtype == 1 || in.pairs_dtype == 2, "topo_pair: pairs dtype %d", in.pairs_dtype);
  if (tokens <= 0) return 0;
  topo_pair_kernel<<<static_cast<unsigned>(tokens), 128, 0, st>>>(in, x32, x16);
  SRB_CUDA_OK(cudaGetLastError());
  note_launch();
  return 0;
}

// rows whose pairs are all invalid are flipped to all-valid (model.py:128-130)
__global__ void topo_fix_valid_kernel(const uint8_t* __restrict__ valid, int rows, int Np,
                                      uint8_t* __restrict__ out) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= rows) return;
  int any = 0;
  for (int p = 0; p < Np; ++p) any |= valid[static_cast<size_t>(r) * Np + p] != 0;
  for (int p = 0; p < Np; ++p)
    out[static_cast<size_t>(r) * Np + p] = any ? (valid[static_cast<size_t>(r) * Np + p] != 0) : 1;
}
int topo_fix_valid(const uint8_t* valid, int rows, int Np, uint8_t* out, cudaStream_t st) {
  if (rows <= 0) return 0;
  topo_fix_valid_kernel<<<(rows + 255) / 256, 256, 0, st>>>(valid, rows, Np, out);
  SRB_CUDA_OK(cudaGetLastError());
  note_launch();
  return 0;
}

// ------------------------------------------------------------------------------------------------
// Self-attention inside each sample (sequence of Np <= KMAX pairs, 4 heads x 32), key-padding mask.
//   qkv: [rows*Np, 384] fp16 (q | k | v), torch MHA scales q by 1/sqrt(32).
//   One thread per (sample, head, query); a 128-thread block covers 128/(4*Np) samples.
//   KMAX = 16 for Np <= 16, 32 above.
// ------------------------------------------------------------------------------------------------
template <int KMAX>
__global__ void __launch_bounds__(128)
topo_attention_kernel(const __half* __restrict__ qkv, const uint8_t* __restrict__ valid, int rows,
                      int Np, __half* __restrict__ out) {
  const int per_block = 128 / (4 * Np);
  const int local = threadIdx.x / (4 * Np);
  const int r = blockIdx.x * per_block + local;
  const int hq = threadIdx.x % (4 * Np);
  const int head = hq / Np, qi = hq % Np;
  if (local >= per_block || r >= rows) return;
  const size_t tok0 = static_cast<size_t>(r) * Np;
  const __half* qp = qkv + (tok0 + qi) * 384 + head * 32;
  float q[32];
#pragma unroll
  for (int c = 0; c < 32; c += 2) {
    const float2 f = __half22float2(*reinterpret_cast<const __half2*>(qp + c));
    q[c] = f.x; q[c + 1] = f.y;
  }
  const float scale = 0.17677669529663687f;   // 1/sqrt(32)
  float sc[KMAX];
  float mx = -INFINITY;
#pragma unroll
  for (int j = 0; j < KMAX; ++j) {
    sc[j] = -INFINITY;
    if (j < Np && valid[tok0 + j]) {
      const __half* kp = qkv + (tok0 + j) * 384 + 128 + head * 32;
      float acc = 0.f;
#pragma unroll
      for (int c = 0; c < 32; c += 2) {
        const float2 f = __half22float2(*reinterpret_cast<const __half2*>(kp + c));
        acc = fmaf(q[c], f.x, acc);
        acc = fmaf(q[c + 1], f.y, acc);
      }
      sc[j] = acc * scale;
      mx = fmaxf(mx, sc[j]);
    }
  }
  float o[32];
#pragma unroll
  for (int c = 0; c < 32; ++c) o[c] = 0.f;
  float l = 0.f;
#pragma unroll
  for (int j = 0; j < KMAX; ++j) {
    if (j < Np && sc[j] > -INFINITY) {
      const float p = __expf(sc[j] - mx);
      l += p;
      const __half* vp = qkv + (tok0 + j) * 384 + 256 + head * 32;
#pragma unroll
      for (int c = 0; c < 32; c += 2) {
        const float2 f = __half22float2(*reinterpret_cast<const __half2*>(vp + c));
        o[c] = fmaf(p, f.x, o[c]);
        o[c + 1] = fmaf(p, f.y, o[c + 1]);
      }
    }
  }
  const float inv = 1.0f / l;
  __half* op = out + (tok0 + qi) * 128 + head * 32;
#pragma unroll
  for (int c = 0; c < 32; c += 2)
    *reinterpret_cast<uint32_t*>(op + c) = pack_half2(o[c] * inv, o[c + 1] * inv);
}

int topo_attention(const __half* qkv, const uint8_t* valid, int rows, int Np, __half* out,
                   cudaStream_t st) {
  SRB_REQUIRE(Np >= 1 && Np <= 32, "topo_attention: n_pairs=%d must be in 1..32", Np);
  if (rows <= 0) return 0;
  const int per_block = 128 / (4 * Np);
  auto* kernel = Np <= 16 ? topo_attention_kernel<16> : topo_attention_kernel<32>;
  kernel<<<(rows + per_block - 1) / per_block, 128, 0, st>>>(qkv, valid, rows, Np, out);
  SRB_CUDA_OK(cudaGetLastError());
  note_launch();
  return 0;
}

// ------------------------------------------------------------------------------------------------
// output_proj (128 -> 1) + sigmoid (model.py:144-146); masked slots report the bias (fast path).
// One warp per token.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
topo_output_kernel(const float* __restrict__ x32, const uint8_t* __restrict__ valid,
                   const float* __restrict__ w, const float* __restrict__ b, long tokens,
                   float* __restrict__ logits, float* __restrict__ scores) {
  const long tok = static_cast<long>(blockIdx.x) * 8 + (threadIdx.x >> 5);
  if (tok >= tokens) return;
  const int lane = threadIdx.x & 31;
  const float4 xv = *reinterpret_cast<const float4*>(x32 + tok * 128 + lane * 4);
  const float4 wv = __ldg(reinterpret_cast<const float4*>(w) + lane);
  float acc = xv.x * wv.x + xv.y * wv.y + xv.z * wv.z + xv.w * wv.w;
  acc = warp_sum(acc);
  if (lane == 0) {
    float lg = acc + __ldg(b);
    if (valid && !valid[tok]) lg = __ldg(b);
    if (logits) logits[tok] = lg;
    if (scores) scores[tok] = 1.0f / (1.0f + expf(-lg));
  }
}

int topo_output(const float* x32, const uint8_t* valid_fixed, const float* w, const float* b,
                int tokens, float* logits, float* scores, cudaStream_t st) {
  if (tokens <= 0) return 0;
  topo_output_kernel<<<(tokens + 7) / 8, 256, 0, st>>>(x32, valid_fixed, w, b, tokens, logits,
                                                       scores);
  SRB_CUDA_OK(cudaGetLastError());
  note_launch();
  return 0;
}

// ------------------------------------------------------------------------------------------------
// fused transformer launcher (n_pairs == 16 or 32): pair features are formed in the kernel from the
// per-point projections pst; weights = 18 chunks [128x128] fp16 in consumption order (per layer:
// Wq, Wk, Wv, Wo, W1, W2)
// ------------------------------------------------------------------------------------------------
int topo_transformer_fused(const TopoPairInputs& in, const __half* w_chunks, const TopoLayerParams* layers,
                           const float* out_w, const float* out_b, const uint8_t* valid_fixed, int tokens,
                           int Np, float* logits, float* scores, cudaStream_t st) {
  SRB_REQUIRE(Np == 16 || Np == 32, "topo fused: n_pairs=%d must be 16 or 32", Np);
  if (tokens <= 0) return 0;
  SRB_REQUIRE(in.pairs_dtype == 1 || in.pairs_dtype == 2, "topo fused: pairs dtype %d", in.pairs_dtype);
  CUtensorMap tmW;
  if (int rc = make_tmap_f16_2d(&tmW, w_chunks, 18 * 128, 128, 128, 128)) return rc;
  // one bit per CUDA device and instantiation: function attributes are per device and function
  static uint64_t attr_devs[2] = {0, 0};
  auto* kernel = Np == 16 ? toponet_tc_kernel<16> : toponet_tc_kernel<32>;
  if (first_use_on_device(&attr_devs[Np == 32])) {
    SRB_CUDA_OK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kTtcSmemBytes));
  }
  TtcParams p;
  for (int l = 0; l < 3; ++l) p.layer[l] = layers[l];
  p.in = in;
  p.valid = valid_fixed; p.out_w = out_w; p.out_b = out_b;
  p.logits = logits; p.scores = scores; p.tokens = tokens;
  p.num_tiles = (tokens + 127) / 128;
  const int grid = p.num_tiles < device_sm_count() ? p.num_tiles : device_sm_count();
  kernel<<<grid, kTtcThreads, kTtcSmemBytes, st>>>(tmW, p);
  SRB_CUDA_OK(cudaGetLastError());
  note_launch();
  return 0;
}

}  // namespace srb
