// sam_road_b200 :: GEMM instantiations and tile-shape dispatch.
#include <cstring>

#include "gemm_tc.cuh"
#include "ops.h"

namespace srb {

// 128x256 tiles (3-stage ring) when N allows and the grid still fills the GPU, otherwise 128x128
// tiles (5-stage ring).

static inline bool use_bn256(int M, int N) {
  if (N % 256 != 0) return false;
  const long tiles256 = static_cast<long>((M + kGemmBM - 1) / kGemmBM) * (N / 256);
  return tiles256 >= device_sm_count();
}

int gemm_f16out(const __half* A, int lda, const __half* W, int ldw, int M, int N, int K,
                const float* bias, int act, __half* out, int ldo, cudaStream_t st) {
  EpiF16::Params p{out, bias, ldo, act};
  SRB_REQUIRE(ldo % 8 == 0, "gemm_f16out: ldo=%d must be a multiple of 8", ldo);
  if (use_bn256(M, N)) return launch_gemm_tc<256, 3, EpiF16>(A, lda, W, ldw, M, N, K, p, st);
  return launch_gemm_tc<128, 5, EpiF16>(A, lda, W, ldw, M, N, K, p, st);
}

int gemm_f32out(const __half* A, int lda, const __half* W, int ldw, int M, int N, int K,
                const float* bias, const float* resid, const float* pos, int pos_rows, float* out,
                int ldo, cudaStream_t st) {
  EpiF32::Params p{out, bias, resid, pos, ldo, pos_rows > 0 ? pos_rows : 1, N};
  SRB_REQUIRE(ldo % 4 == 0, "gemm_f32out: ldo=%d must be a multiple of 4", ldo);
  if (use_bn256(M, N)) return launch_gemm_tc<256, 3, EpiF32>(A, lda, W, ldw, M, N, K, p, st);
  return launch_gemm_tc<128, 5, EpiF32>(A, lda, W, ldw, M, N, K, p, st);
}

int gemm_ln(const __half* A, int lda, const __half* W, int ldw, int M, int N, int K,
            const float* bias, const float* resid, const float* gamma, const float* beta, float eps,
            int group, int act, __half* out16, float* out32, float* out_nchw, int tokens, int ldo,
            cudaStream_t st, int conv_s) {
  SRB_REQUIRE(group == 64 || group == 128 || group == 256, "gemm_ln: group=%d must be 64, 128 or 256", group);
  SRB_REQUIRE(N % group == 0, "gemm_ln: N=%d not a multiple of group=%d", N, group);
  EpiLN::Params p{out16, out32, out_nchw, bias, resid, gamma, beta, eps, ldo, group, act,
                  tokens > 0 ? tokens : 1, N};
  if (group == 256 || use_bn256(M, N))
    return launch_gemm_tc<256, 3, EpiLN>(A, lda, W, ldw, M, N, K, p, st, conv_s);
  return launch_gemm_tc<128, 5, EpiLN>(A, lda, W, ldw, M, N, K, p, st, conv_s);
}

template <bool kPerToken>
static int launch_dec_final(const __half* A, int lda, const __half* W, int ldw, int M, int K,
                            const float* bias3, const float* w4, const float* bias4, int s, int P,
                            float* scores, float* logits, cudaStream_t st) {
  typename EpiDecFinal<kPerToken>::Params p;
  memset(&p, 0, sizeof(p));
  const int B = M / (16 * s * s);
  const uint64_t rowb = static_cast<uint64_t>(P) * 2 * sizeof(float);
  const uint64_t dims[4] = {static_cast<uint64_t>(P) * 2, 2, 2, static_cast<uint64_t>(B) * P / 4};
  const uint64_t strides[3] = {rowb, 2 * rowb, 4 * rowb};
  const uint32_t box[4] = {kPerToken ? 32u : 64u, 2, 1, 4};
  if (scores) { if (int rc = make_tmap_f32_4d_dense(&p.tm_scores, scores, dims, strides, box)) return rc; }
  if (logits) { if (int rc = make_tmap_f32_4d_dense(&p.tm_logits, logits, dims, strides, box)) return rc; }
  p.has_scores = scores != nullptr;
  p.has_logits = logits != nullptr;
  p.bias3 = bias3; p.w4 = w4; p.bias4 = bias4; p.s = s; p.P = P;
  return launch_gemm_tc<128, 5, EpiDecFinal<kPerToken>>(A, lda, W, ldw, M, 128, K, p, st);
}

int gemm_dec_final(const __half* A, int lda, const __half* W, int ldw, int M, int K,
                   const float* bias3, const float* w4, const float* bias4, int s, int P,
                   float* scores, float* logits, cudaStream_t st) {
  SRB_REQUIRE(P == 16 * s && M % (16 * s * s) == 0, "gemm_dec_final: M=%d s=%d P=%d inconsistent", M, s, P);
  // a warp stores two consecutive tokens: one 32-pixel box when they are always row neighbours (s
  // even), one 16-pixel box per token otherwise (a pair can wrap to the next row or image)
  if (s % 2 == 0) return launch_dec_final<false>(A, lda, W, ldw, M, K, bias3, w4, bias4, s, P, scores, logits, st);
  return launch_dec_final<true>(A, lda, W, ldw, M, K, bias3, w4, bias4, s, P, scores, logits, st);
}

// ------------------------------------------------------------------------------------------------
// test-only checker: one thread per output element, fp32 FMA chain over K
// ------------------------------------------------------------------------------------------------
__global__ void gemm_ref_simt_kernel(const __half* __restrict__ A, int lda,
                                     const __half* __restrict__ W, int ldw, int M, int N, int K,
                                     float* __restrict__ out, int ldo) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  const int m = blockIdx.y;
  if (n >= N || m >= M) return;
  const __half* a = A + static_cast<size_t>(m) * lda;
  const __half* w = W + static_cast<size_t>(n) * ldw;
  float acc = 0.f;
  for (int k = 0; k < K; ++k) acc = fmaf(__half2float(a[k]), __half2float(w[k]), acc);
  out[static_cast<size_t>(m) * ldo + n] = acc;
}

int gemm_ref_simt(const __half* A, int lda, const __half* W, int ldw, int M, int N, int K,
                  float* out, int ldo, cudaStream_t st) {
  dim3 grid((N + 127) / 128, M);
  gemm_ref_simt_kernel<<<grid, 128, 0, st>>>(A, lda, W, ldw, M, N, K, out, ldo);
  SRB_CUDA_OK(cudaGetLastError());
  note_launch();
  return 0;
}

}  // namespace srb
