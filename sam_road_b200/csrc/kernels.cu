// sam_road_b200 :: HBM-bound data-movement kernels around the GEMMs: LayerNorm, patch im2col (with
// the pixel normalisation of model.py:465-467 fused in), 3x3 im2col for the neck, mask fusion.
// All are one-pass streaming kernels with 128-bit accesses; the arithmetic is fp32.
#include "common.cuh"
#include "ops.h"

namespace srb {

// ------------------------------------------------------------------------------------------------
// LayerNorm over the last dim (nn.LayerNorm, biased variance, eps inside sqrt):
//   image_encoder.py:151,161,168,180 (eps 1e-6 via model.py:250).  One warp per row; fp32 in,
//   fp16 out (the A operand of the next GEMM).  D % 128 == 0, D <= 1280.
// ------------------------------------------------------------------------------------------------
constexpr int kLNMaxVec = 10;

__global__ void __launch_bounds__(256)
layernorm_f16_kernel(const float* __restrict__ x, const float* __restrict__ gamma,
                     const float* __restrict__ beta, float eps, int M, int D,
                     __half* __restrict__ out, int reverse) {
  const int blk = reverse ? static_cast<int>(gridDim.x) - 1 - static_cast<int>(blockIdx.x) : static_cast<int>(blockIdx.x);
  const int row = blk * 8 + (threadIdx.x >> 5);
  if (row >= M) return;
  const int lane = threadIdx.x & 31;
  const int nvec = D >> 7;   // float4 per lane
  const float4* xr = reinterpret_cast<const float4*>(x + static_cast<size_t>(row) * D);
  float4 v[kLNMaxVec];
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < kLNMaxVec; ++i) {
    if (i < nvec) {
      v[i] = xr[lane + 32 * i];
      sum += (v[i].x + v[i].y) + (v[i].z + v[i].w);
    }
  }
  const float mean = warp_sum(sum) / static_cast<float>(D);
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < kLNMaxVec; ++i) {
    if (i < nvec) {
      const float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
      sq += (a * a + b * b) + (c * c + d * d);
    }
  }
  const float rstd = rsqrtf(warp_sum(sq) / static_cast<float>(D) + eps);
  const float4* g4 = reinterpret_cast<const float4*>(gamma);
  const float4* b4 = reinterpret_cast<const float4*>(beta);
  uint2* orow = reinterpret_cast<uint2*>(out + static_cast<size_t>(row) * D);
#pragma unroll
  for (int i = 0; i < kLNMaxVec; ++i) {
    if (i < nvec) {
      const float4 g = __ldg(g4 + lane + 32 * i);
      const float4 b = __ldg(b4 + lane + 32 * i);
      uint2 o;
      o.x = pack_half2((v[i].x - mean) * rstd * g.x + b.x, (v[i].y - mean) * rstd * g.y + b.y);
      o.y = pack_half2((v[i].z - mean) * rstd * g.z + b.z, (v[i].w - mean) * rstd * g.w + b.w);
      orow[lane + 32 * i] = o;
    }
  }
}

int layernorm_f16(const float* x, const float* gamma, const float* beta, float eps, int M, int D,
                  __half* out, bool reverse, cudaStream_t st) {
  SRB_REQUIRE(D % 128 == 0 && D <= 128 * kLNMaxVec, "layernorm: D=%d unsupported", D);
  if (M <= 0) return 0;
  SRB_LAUNCH(layernorm_f16_kernel, (M + 7) / 8, 256, 0, st, x, gamma, beta, eps, M, D, out, reverse ? 1 : 0);
  return 0;
}

// ------------------------------------------------------------------------------------------------
// Patch im2col: rgb[B,P,P,3] (fp32 0..255 or uint8) -> A[B*s*s, 768] fp16 with
//   A[token, ky*48 + kx*3 + c] = (rgb[b, ty*16+ky, tx*16+kx, c] - mean[c]) / std[c]
// i.e. the normalisation of model.py:465-467 and the unfold of the 16x16/s16 conv
// (image_encoder.py:387-395).  In this K order each (token, ky) is 48 contiguous input values;
// the patch-embed weight is permuted to the same order at pack time.  One thread = 8 values.
// ------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256)
im2col_patch16_kernel(const T* __restrict__ rgb, int B, int P, float m0, float m1, float m2,
                      float i0, float i1, float i2, __half* __restrict__ out) {
  const int s = P >> 4;
  const long total = static_cast<long>(B) * s * s * 16 * 6;
  const long idx = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int g = static_cast<int>(idx % 6);
  const int ky = static_cast<int>((idx / 6) % 16);
  const long token = idx / 96;
  const int tx = static_cast<int>(token % s);
  const int ty = static_cast<int>((token / s) % s);
  const int b = static_cast<int>(token / (static_cast<long>(s) * s));
  const size_t src = ((static_cast<size_t>(b) * P + (ty * 16 + ky)) * P + tx * 16) * 3 + g * 8;
  float v[8];
  if constexpr (sizeof(T) == 4) {
    const float4 a = *reinterpret_cast<const float4*>(rgb + src);
    const float4 c = *reinterpret_cast<const float4*>(rgb + src + 4);
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = c.x; v[5] = c.y; v[6] = c.z; v[7] = c.w;
  } else {
    const uint2 u = *reinterpret_cast<const uint2*>(rgb + src);
    v[0] = static_cast<float>(u.x & 0xff); v[1] = static_cast<float>((u.x >> 8) & 0xff);
    v[2] = static_cast<float>((u.x >> 16) & 0xff); v[3] = static_cast<float>(u.x >> 24);
    v[4] = static_cast<float>(u.y & 0xff); v[5] = static_cast<float>((u.y >> 8) & 0xff);
    v[6] = static_cast<float>((u.y >> 16) & 0xff); v[7] = static_cast<float>(u.y >> 24);
  }
  const int c0 = (g * 8) % 3;   // channel of element 0 (8 mod 3 = 2 -> 0,2,1,0,2,1)
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const int c = (c0 + e) % 3;
    const float mean = c == 0 ? m0 : (c == 1 ? m1 : m2);
    const float inv = c == 0 ? i0 : (c == 1 ? i1 : i2);
    // the reference divides by std; (x-mean)/std and (x-mean)*(1/std) differ by <=1 ulp fp32,
    // far below the fp16 rounding applied next.
    v[e] = (v[e] - mean) * inv;
  }
  uint4 o;
  o.x = pack_half2(v[0], v[1]); o.y = pack_half2(v[2], v[3]);
  o.z = pack_half2(v[4], v[5]); o.w = pack_half2(v[6], v[7]);
  *reinterpret_cast<uint4*>(out + static_cast<size_t>(token) * 768 + ky * 48 + g * 8) = o;
}

int im2col_patch16(const void* rgb, int dtype, int B, int P, const float* mean,
                   const float* inv_std, __half* out, cudaStream_t st) {
  SRB_REQUIRE(P % 16 == 0 && P > 0, "im2col_patch16: P=%d must be a positive multiple of 16", P);
  SRB_REQUIRE(dtype == 0 || dtype == 1, "im2col_patch16: rgb dtype %d (want 0=f32, 1=u8)", dtype);
  if (B <= 0) return 0;
  const int s = P / 16;
  const long total = static_cast<long>(B) * s * s * 96;
  const int blocks = static_cast<int>((total + 255) / 256);
  if (dtype == 0)
    SRB_LAUNCH(im2col_patch16_kernel<float>, blocks, 256, 0, st, static_cast<const float*>(rgb), B, P, mean[0], mean[1],
               mean[2], inv_std[0], inv_std[1], inv_std[2], out);
  else
    SRB_LAUNCH(im2col_patch16_kernel<uint8_t>, blocks, 256, 0, st, static_cast<const uint8_t*>(rgb), B, P, mean[0],
               mean[1], mean[2], inv_std[0], inv_std[1], inv_std[2], out);
  return 0;
}

// ------------------------------------------------------------------------------------------------
// Tile crop (inferencer.py:43-58 crop_img_patch / get_batch_img_patches): uint8 scene [H,W,3] ->
// uint8 tiles [B,P,P,3] at the given origins.  One thread = 4 destination bytes (one aligned store);
// the source row starts at an arbitrary byte, so it is read bytewise (L1-resident, 3 B per pixel).
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
crop_tiles_kernel(const uint8_t* __restrict__ scene, int W, const int* __restrict__ txy, int B, int P,
                  uint8_t* __restrict__ out) {
  const int row_words = P * 3 / 4;
  const long total = static_cast<long>(B) * P * row_words;
  const long idx = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int wq = static_cast<int>(idx % row_words);
  const int y = static_cast<int>((idx / row_words) % P);
  const int b = static_cast<int>(idx / (static_cast<long>(row_words) * P));
  const int x0 = __ldg(txy + 2 * b), y0 = __ldg(txy + 2 * b + 1);
  const uint8_t* src = scene + (static_cast<size_t>(y0 + y) * W + x0) * 3 + wq * 4;
  const uint32_t v = static_cast<uint32_t>(src[0]) | (static_cast<uint32_t>(src[1]) << 8) |
                     (static_cast<uint32_t>(src[2]) << 16) | (static_cast<uint32_t>(src[3]) << 24);
  reinterpret_cast<uint32_t*>(out)[idx] = v;
}

int crop_tiles(const uint8_t* scene, int H, int W, const int* tile_xy, int B, int P, uint8_t* out,
               cudaStream_t st) {
  SRB_REQUIRE(P % 4 == 0 && P > 0 && P <= H && P <= W, "crop_tiles: P=%d vs scene %dx%d", P, H, W);
  if (B <= 0) return 0;
  const long total = static_cast<long>(B) * P * (P * 3 / 4);
  SRB_LAUNCH(crop_tiles_kernel, static_cast<int>((total + 255) / 256), 256, 0, st, scene, W, tile_xy, B, P, out);
  return 0;
}

// ------------------------------------------------------------------------------------------------
// 3x3 / pad 1 im2col on NHWC fp16 (neck conv, image_encoder.py:96-102): one thread = 8 channels.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
im2col_3x3_kernel(const __half* __restrict__ x, int B, int s, int C, __half* __restrict__ out) {
  const int cg = C >> 3;
  const long total = static_cast<long>(B) * s * s * 9 * cg;
  const long idx = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int g = static_cast<int>(idx % cg);
  const int tap = static_cast<int>((idx / cg) % 9);
  const long m = idx / (9L * cg);
  const int xx = static_cast<int>(m % s);
  const int yy = static_cast<int>((m / s) % s);
  const long b = m / (static_cast<long>(s) * s);
  const int sy = yy + tap / 3 - 1, sx = xx + tap % 3 - 1;
  uint4 v = make_uint4(0, 0, 0, 0);
  if (sy >= 0 && sy < s && sx >= 0 && sx < s)
    v = *reinterpret_cast<const uint4*>(x + ((b * s + sy) * s + sx) * C + g * 8);
  *reinterpret_cast<uint4*>(out + m * (9L * C) + tap * C + g * 8) = v;
}

int im2col_3x3(const __half* x, int B, int s, int C, __half* out, cudaStream_t st) {
  SRB_REQUIRE(C % 8 == 0, "im2col_3x3: C=%d must be a multiple of 8", C);
  if (B <= 0) return 0;
  const long total = static_cast<long>(B) * s * s * 9 * (C / 8);
  SRB_LAUNCH(im2col_3x3_kernel, static_cast<int>((total + 255) / 256), 256, 0, st, x, B, s, C, out);
  return 0;
}

// fp32 -> fp16 copy (A operand of the neck 1x1 conv, image_encoder.py:114: no norm before the neck)
__global__ void __launch_bounds__(256)
convert_f32_f16_kernel(const float* __restrict__ x, long n8, __half* __restrict__ out) {
  const long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n8) return;
  const float4 a = reinterpret_cast<const float4*>(x)[2 * i];
  const float4 b = reinterpret_cast<const float4*>(x)[2 * i + 1];
  uint4 o;
  o.x = pack_half2(a.x, a.y); o.y = pack_half2(a.z, a.w);
  o.z = pack_half2(b.x, b.y); o.w = pack_half2(b.z, b.w);
  reinterpret_cast<uint4*>(out)[i] = o;
}
int convert_f32_f16(const float* x, long n, __half* out, cudaStream_t st) {
  SRB_REQUIRE(n % 8 == 0, "convert_f32_f16: n=%ld must be a multiple of 8", n);
  if (n <= 0) return 0;
  SRB_LAUNCH(convert_f32_f16_kernel, static_cast<int>((n / 8 + 255) / 256), 256, 0, st, x, n / 8, out);
  return 0;
}

// ------------------------------------------------------------------------------------------------
// Mask fusion (inferencer.py:79-110).  The reference adds every tile's scores into scene-sized
// fp32 accumulators in tile-list order (x outer, y inner: dataset.py:56-67), divides by the
// coverage counter, multiplies by 255 and truncates to uint8.  Here one thread owns one scene pixel
// and performs the same additions in the same order, so the result is bit-identical for
// identical scores.  Tiles are given by their origins; tile t covers [x0,x0+P) x [y0,y0+P).
// Pixels no tile covers are 0/0 = NaN in the reference, whose uint8 cast yields 0.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
fuse_masks_kernel(const float* __restrict__ scores, int n_tiles, int P,
                  const int* __restrict__ tx0, const int* __restrict__ ty0, int H, int W,
                  uint8_t* __restrict__ kp, uint8_t* __restrict__ road) {
  // the CTA owns 256 consecutive pixels of one scene row; it first lists (in tile-list order) the tiles that
  // touch that segment at all, so that a pixel walks a few dozen candidates instead of every tile of the scene
  __shared__ int s_list[1024];
  __shared__ int s_n;
  __shared__ int sw[33];
  const int xb = blockIdx.x * blockDim.x;
  const int x = xb + threadIdx.x;
  const int y = blockIdx.y;
  float a0 = 0.f, a1 = 0.f, cnt = 0.f;
  for (int t0 = 0; t0 < n_tiles; t0 += 1024) {       // chunks of 1024 tiles keep the list in shared memory
    if (threadIdx.x == 0) s_n = 0;
    __syncthreads();
    for (int b = 0; b < 1024; b += 256) {
      const int t = t0 + b + threadIdx.x;
      bool hit = false;
      if (t < n_tiles) {
        const int ox = __ldg(tx0 + t), oy = __ldg(ty0 + t);
        hit = y >= oy && y < oy + P && ox < xb + 256 && ox + P > xb;
      }
      // ordered append: exclusive scan of the hit flags over the block
      const unsigned bal = __ballot_sync(0xffffffffu, hit);
      const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
      if (lane == 0) sw[wid] = __popc(bal);
      __syncthreads();
      int base = s_n;
      for (int w = 0; w < wid; ++w) base += sw[w];
      if (hit) s_list[base + __popc(bal & ((1u << lane) - 1u))] = t;
      __syncthreads();
      if (threadIdx.x == 0) { int tot = 0; for (int w = 0; w < 8; ++w) tot += sw[w]; s_n += tot; }
      __syncthreads();
    }
    const int n = s_n;
    if (x < W) {
      for (int i = 0; i < n; ++i) {
        const int t = s_list[i];
        const int lx = x - __ldg(tx0 + t), ly = y - __ldg(ty0 + t);
        if (lx >= 0 && lx < P) {
          const float2 sc = *reinterpret_cast<const float2*>(
              scores + ((static_cast<size_t>(t) * P + ly) * P + lx) * 2);
          a0 = __fadd_rn(a0, sc.x);
          a1 = __fadd_rn(a1, sc.y);
          cnt = __fadd_rn(cnt, 1.0f);
        }
      }
    }
    __syncthreads();
  }
  if (x >= W) return;
  uint8_t o0 = 0, o1 = 0;
  if (cnt > 0.f) {
    const float f0 = __fmul_rn(__fdiv_rn(a0, cnt), 255.0f);
    const float f1 = __fmul_rn(__fdiv_rn(a1, cnt), 255.0f);
    o0 = static_cast<uint8_t>(static_cast<int>(f0));   // truncation toward zero, as .to(uint8)
    o1 = static_cast<uint8_t>(static_cast<int>(f1));
  }
  kp[static_cast<size_t>(y) * W + x] = o0;
  road[static_cast<size_t>(y) * W + x] = o1;
}

int fuse_masks(const float* scores, int n_tiles, int P, const int* tile_x0, const int* tile_y0,
               int H, int W, uint8_t* keypoint_u8, uint8_t* road_u8, cudaStream_t st) {
  SRB_REQUIRE(H > 0 && W > 0 && P > 0 && n_tiles >= 0, "fuse_masks: bad sizes H=%d W=%d P=%d n=%d",
              H, W, P, n_tiles);
  dim3 grid((W + 255) / 256, H);
  SRB_LAUNCH(fuse_masks_kernel, grid, 256, 0, st, scores, n_tiles, P, tile_x0, tile_y0, H, W, keypoint_u8, road_u8);
  return 0;
}

}  // namespace srb
