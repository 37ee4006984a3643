// sam_road_b200 :: ViT encoder attention with decomposed relative-position bias.
//
// Reference: sam/segment_anything/modeling/image_encoder.py
//   Attention.forward            :224-240   attn = (q*scale) k^T ; + rel-pos ; softmax ; attn v
//   add_decomposed_rel_pos       :325-361   bias[q,(kh,kw)] = q . Rh[qh,kh] + q . Rw[qw,kw]  (UNscaled q)
//   get_rel_pos                  :292-322   Rh[qh,kh] = rel_pos_h[qh - kh + (K-1)]
//   window_partition/unpartition :243-289   zero pad to a multiple of 14 AFTER norm1 (:168-172)
//
// The window partition is never materialised: the kernel addresses tokens of window (wy,wx) by index
// math, and a padded token (y >= s or x >= s) has x = 0 so q = k = v = qkv bias (SURVEY.md §8a P1):
// such tokens are real softmax keys but their query rows are never written.
//
// Two kernels: the tensor-core kernel (attention_mma.cuh) on the hot path, and an fp32 SIMT
// flash-style kernel (one thread = one query row, keys streamed through shared memory in chunks of 32
// with an online softmax) -- the straightforward, easily-audited statement of the math and the
// on-device checker for the tensor-core version.
#include "attention_mma.cuh"
#include "common.cuh"
#include "ops.h"

#define SRB_TRY_RC(expr) do { int _rc = (expr); if (_rc != 0) return _rc; } while (0)

namespace srb {

constexpr int kAttThreads = 128;
constexpr int kAttChunk = 32;

template <int HD>
__global__ void __launch_bounds__(kAttThreads)
encoder_attention_simt_kernel(const __half* __restrict__ qkv, const float* __restrict__ qkv_bias,
                              const float* __restrict__ rel_h, const float* __restrict__ rel_w,
                              int B, int s, int win, int nwin, int heads, float scale,
                              __half* __restrict__ out) {
  extern __shared__ float smem_att[];
  float* sK = smem_att;                         // [kAttChunk][HD]
  float* sV = sK + kAttChunk * HD;              // [kAttChunk][HD]
  float* sRel = sV + kAttChunk * HD;            // [kAttThreads][2*win]

  const int D = heads * HD;
  const int ld = 3 * D;
  const int head = blockIdx.y % heads;
  const int widx = (blockIdx.y / heads) % (nwin * nwin);
  const int b = blockIdx.y / (heads * nwin * nwin);
  const int wy = widx / nwin, wx = widx % nwin;
  const int nkeys = win * win;

  const int tid = threadIdx.x;
  const int qi = blockIdx.x * kAttThreads + tid;
  const int qy = qi / win, qx = qi % win;
  const int gy = wy * win + qy, gx = wx * win + qx;
  const bool q_in_win = qi < nkeys;
  const bool q_real = q_in_win && gy < s && gx < s;

  // ---- q row (fp32) ----
  float q[HD];
  if (q_real) {
    const __half* qp = qkv + (static_cast<size_t>(b) * s * s + gy * s + gx) * ld + head * HD;
#pragma unroll
    for (int c = 0; c < HD; c += 8) {
      const uint4 u = *reinterpret_cast<const uint4*>(qp + c);
      const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 f = __half22float2(h[e]);
        q[c + 2 * e] = f.x;
        q[c + 2 * e + 1] = f.y;
      }
    }
  } else {
#pragma unroll
    for (int c = 0; c < HD; ++c) q[c] = q_in_win ? __ldg(qkv_bias + head * HD + c) : 0.f;
  }

  // ---- decomposed rel-pos rows for this query: relh[kh], relw[kw] ----
  float* myrel = sRel + tid * (2 * win);
  if (q_in_win) {
    for (int k = 0; k < win; ++k) {
      const float* th = rel_h + static_cast<size_t>(qy - k + win - 1) * HD;
      const float* tw = rel_w + static_cast<size_t>(qx - k + win - 1) * HD;
      float ah = 0.f, aw = 0.f;
#pragma unroll
      for (int c = 0; c < HD; ++c) {
        ah = fmaf(q[c], __ldg(th + c), ah);
        aw = fmaf(q[c], __ldg(tw + c), aw);
      }
      myrel[k] = ah;
      myrel[win + k] = aw;
    }
  }

  float o[HD];
#pragma unroll
  for (int c = 0; c < HD; ++c) o[c] = 0.f;
  float m_run = -INFINITY, l_run = 0.f;

  for (int k0 = 0; k0 < nkeys; k0 += kAttChunk) {
    __syncthreads();
    // cooperative load of K and V chunk (fp32 in smem); pad tokens take the bias
    for (int idx = tid; idx < kAttChunk * (HD / 8); idx += kAttThreads) {
      const int r = idx / (HD / 8), c8 = (idx % (HD / 8)) * 8;
      const int kk = k0 + r;
      float kv[8], vv[8];
      bool loaded = false;
      if (kk < nkeys) {
        const int ky = wy * win + kk / win, kx = wx * win + kk % win;
        if (ky < s && kx < s) {
          const __half* base =
              qkv + (static_cast<size_t>(b) * s * s + ky * s + kx) * ld + head * HD + c8;
          const uint4 uk = *reinterpret_cast<const uint4*>(base + D);
          const uint4 uv = *reinterpret_cast<const uint4*>(base + 2 * D);
          const __half2* hk = reinterpret_cast<const __half2*>(&uk);
          const __half2* hv = reinterpret_cast<const __half2*>(&uv);
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const float2 fk = __half22float2(hk[e]);
            const float2 fv = __half22float2(hv[e]);
            kv[2 * e] = fk.x; kv[2 * e + 1] = fk.y;
            vv[2 * e] = fv.x; vv[2 * e + 1] = fv.y;
          }
          loaded = true;
        }
      }
      if (!loaded) {
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          kv[e] = __ldg(qkv_bias + D + head * HD + c8 + e);
          vv[e] = __ldg(qkv_bias + 2 * D + head * HD + c8 + e);
        }
      }
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        sK[r * HD + c8 + e] = kv[e];
        sV[r * HD + c8 + e] = vv[e];
      }
    }
    __syncthreads();

    if (q_in_win) {
      float sc[kAttChunk];
      float m_new = m_run;
#pragma unroll
      for (int r = 0; r < kAttChunk; ++r) {
        const int kk = k0 + r;
        float acc = 0.f;
#pragma unroll
        for (int c = 0; c < HD; ++c) acc = fmaf(q[c], sK[r * HD + c], acc);
        if (kk < nkeys) {
          acc = acc * scale + myrel[kk / win] + myrel[win + kk % win];
        } else {
          acc = -INFINITY;
        }
        sc[r] = acc;
        m_new = fmaxf(m_new, acc);
      }
      const float alpha = __expf(m_run - m_new);   // m_run = -inf on first chunk -> 0
      l_run *= alpha;
#pragma unroll
      for (int c = 0; c < HD; ++c) o[c] *= alpha;
#pragma unroll
      for (int r = 0; r < kAttChunk; ++r) {
        const float p = __expf(sc[r] - m_new);
        l_run += p;
#pragma unroll
        for (int c = 0; c < HD; ++c) o[c] = fmaf(p, sV[r * HD + c], o[c]);
      }
      m_run = m_new;
    }
  }

  if (q_real) {
    const float inv = 1.0f / l_run;
    __half* op = out + (static_cast<size_t>(b) * s * s + gy * s + gx) * D + head * HD;
#pragma unroll
    for (int c = 0; c < HD; c += 8) {
      uint4 u;
      u.x = pack_half2(o[c + 0] * inv, o[c + 1] * inv);
      u.y = pack_half2(o[c + 2] * inv, o[c + 3] * inv);
      u.z = pack_half2(o[c + 4] * inv, o[c + 5] * inv);
      u.w = pack_half2(o[c + 6] * inv, o[c + 7] * inv);
      *reinterpret_cast<uint4*>(op + c) = u;
    }
  }
}

template <int HD>
static int launch_attention_simt(const __half* qkv, const float* qkv_bias, const float* rel_h,
                                 const float* rel_w, int B, int s, int win, int heads, __half* out,
                                 cudaStream_t st) {
  const int nwin = (s + win - 1) / win;
  const size_t smem = (2 * kAttChunk * HD + kAttThreads * 2 * win) * sizeof(float);
  auto kern = encoder_attention_simt_kernel<HD>;
  SRB_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   static_cast<int>(smem)));
  dim3 grid((win * win + kAttThreads - 1) / kAttThreads, B * nwin * nwin * heads);
  const float scale = 1.0f / sqrtf(static_cast<float>(HD));
  kern<<<grid, kAttThreads, smem, st>>>(qkv, qkv_bias, rel_h, rel_w, B, s, win, nwin, heads, scale,
                                        out);
  SRB_CUDA_OK(cudaGetLastError());
  note_launch();
  return 0;
}

static bool g_force_simt = false;
void attention_force_simt(int mode) { g_force_simt = (mode & 1) != 0; }

int encoder_attention(const __half* qkv, const float* qkv_bias, const float* rel_h,
                      const float* rel_w, int B, int s, int win, int heads, int hd, __half* out,
                      cudaStream_t st) {
  // win > s is one padded window (a window block on a grid smaller than its window)
  SRB_REQUIRE(win > 0 && win <= 64 && s > 0 && s <= 64, "attention: win=%d s=%d unsupported", win, s);
  if (B <= 0) return 0;
  if (!g_force_simt) {
    if (hd == 64) return launch_attention_mma<64>(qkv, qkv_bias, rel_h, rel_w, B, s, win, heads, out, st);
    if (hd == 80) return launch_attention_mma<80>(qkv, qkv_bias, rel_h, rel_w, B, s, win, heads, out, st);
  }
  if (hd == 64) return launch_attention_simt<64>(qkv, qkv_bias, rel_h, rel_w, B, s, win, heads, out, st);
  if (hd == 80) return launch_attention_simt<80>(qkv, qkv_bias, rel_h, rel_w, B, s, win, heads, out, st);
  set_last_error("attention: head_dim=%d unsupported (64 or 80)", hd);
  return 2;
}

}  // namespace srb
