// sam_road_b200 :: training step of the heads with a frozen encoder (FREEZE_ENCODER), DESIGN.md §12.
//
// Reference: SAMRoad.training_step (model.py:511-544) with the encoder in no param group
// (configure_optimizers, model.py:637-685): the naive map decoder (model.py:286-295) and TopoNet
// (model.py:61-148, torch's slow path of TransformerEncoderLayer with dropout 0.1) are trained.
//
//   forward   the encoder exactly as samroad_encode_masks (embeddings only), then the heads: tensor-core
//             GEMMs (mma.sync, fp16 operands, fp32 accumulation) and fp32 elementwise / LayerNorm kernels,
//             saving what backward needs; the loss values use the validation element terms
//             (loss_terms.cuh) summed in fp64 in a fixed order.
//   backward  the same GEMM for the input gradients and for the weight gradients, which are split over the
//             rows in fixed chunks whose partials are summed in chunk order, then scaled in fp32; LayerNorm,
//             GELU / ReLU, dropout and attention backward, and a segmented (CSR) reduction of the pair
//             tokens onto their src / tgt points.  No float atomics: a step is bitwise reproducible.
//
// Layouts.  A ConvTranspose2d(k=2, s=2) is a per-pixel linear map Cin -> 4*Cout.  Decoder activations are
// stored in "quad-tree" row order: the 4 children of row r are rows 4r+d, d = di*2+dj, so every stage is
// a plain [rows, C] matrix and the pixel (y, x) of a final row is decoded from its base-4 digits.
// Dropout masks are counter-based Philox4x32-10 of (seed, layer, site, element), regenerated in backward.
#include "../../include/samroad_b200.h"

#include <cuda_runtime.h>

#include <cmath>
#include <cstring>
#include <string>

#include "common.cuh"
#include "loss_terms.cuh"
#include "ops.h"
#include "scan.cuh"
#include "toponet_tc.cuh"   // load_coord, resolve_pair

using namespace srb;

// model.cu: the parts of the handle's configuration the heads need
int samroad_handle_head_config(samroad_handle_t h, int* patch_size, int* toponet_version, int* use_sam_decoder);

namespace {

// ---- head parameters in the reference layout ------------------------------------------------------------
enum HeadParam {
  HP_DEC0_W, HP_DEC0_B, HP_DEC1_W, HP_DEC1_B, HP_DEC3_W, HP_DEC3_B, HP_DEC5_W, HP_DEC5_B, HP_DEC7_W, HP_DEC7_B,
  HP_FP_W, HP_FP_B, HP_PP_W, HP_PP_B, HP_OUT_W, HP_OUT_B,
  HP_LAYER0,   // + 12 * l + LP_*
  HP_COUNT = HP_LAYER0 + 36
};
enum LayerParam { LP_IN_W, LP_IN_B, LP_OUT_W, LP_OUT_B, LP_L1_W, LP_L1_B, LP_L2_W, LP_L2_B, LP_N1_G, LP_N1_B, LP_N2_G, LP_N2_B };

const char* const kHeadNames[16] = {
  "map_decoder.0.weight", "map_decoder.0.bias", "map_decoder.1.weight", "map_decoder.1.bias",
  "map_decoder.3.weight", "map_decoder.3.bias", "map_decoder.5.weight", "map_decoder.5.bias",
  "map_decoder.7.weight", "map_decoder.7.bias", "topo_net.feature_proj.weight", "topo_net.feature_proj.bias",
  "topo_net.pair_proj.weight", "topo_net.pair_proj.bias", "topo_net.output_proj.weight", "topo_net.output_proj.bias"};
const char* const kLayerNames[12] = {
  "self_attn.in_proj_weight", "self_attn.in_proj_bias", "self_attn.out_proj.weight", "self_attn.out_proj.bias",
  "linear1.weight", "linear1.bias", "linear2.weight", "linear2.bias",
  "norm1.weight", "norm1.bias", "norm2.weight", "norm2.bias"};

int head_param_index(const char* key) {
  for (int i = 0; i < 16; ++i)
    if (std::strcmp(key, kHeadNames[i]) == 0) return i;
  for (int l = 0; l < 3; ++l)
    for (int i = 0; i < 12; ++i) {
      const std::string k = "topo_net.transformer_encoder.layers." + std::to_string(l) + "." + kLayerNames[i];
      if (k == key) return HP_LAYER0 + 12 * l + i;
    }
  return -1;
}

struct HeadPtrs { const float* p[HP_COUNT]; };

int resolve_params(const char* const* keys, const float* const* params, int n, bool with_layers,
                   HeadPtrs* out, int* slot_of /*[n] or null*/) {
  SRB_REQUIRE(n >= 0 && (n == 0 || (keys && params)), "train: null parameter table");
  for (int i = 0; i < HP_COUNT; ++i) out->p[i] = nullptr;
  for (int i = 0; i < n; ++i) {
    SRB_REQUIRE(keys[i] && params[i], "train: null key or pointer at %d", i);
    const int k = head_param_index(keys[i]);
    SRB_REQUIRE(k >= 0 && (with_layers || k < HP_LAYER0),
                "train: '%s' is not a trainable head parameter of this configuration", keys[i]);
    SRB_REQUIRE(out->p[k] == nullptr, "train: '%s' given twice", keys[i]);
    out->p[k] = params[i];
    if (slot_of) slot_of[i] = k;
  }
  const int need = with_layers ? HP_COUNT : HP_LAYER0;
  for (int k = 0; k < need; ++k) {
    if (out->p[k]) continue;
    if (k < 16) SRB_REQUIRE(false, "train: missing head parameter '%s'", kHeadNames[k]);
    SRB_REQUIRE(false, "train: missing head parameter 'topo_net.transformer_encoder.layers.%d.%s'",
                (k - HP_LAYER0) / 12, kLayerNames[(k - HP_LAYER0) % 12]);
  }
  return 0;
}

// ---- dropout: Philox4x32-10 keyed by the seed, counter (element, layer * 4 + site) -----------------------------
struct Dropout {
  unsigned long long seed;
  uint32_t thr;      // keep when the 32-bit draw >= thr (thr = p * 2^32)
  float scale;       // 1 / (1 - p)
  bool on;
};

__host__ __device__ inline uint32_t mulhilo(uint32_t a, uint32_t b, uint32_t* hi) {
  const unsigned long long p = static_cast<unsigned long long>(a) * b;
  *hi = static_cast<uint32_t>(p >> 32);
  return static_cast<uint32_t>(p);
}

__host__ __device__ inline uint32_t philox_draw(unsigned long long seed, unsigned long long elem, uint32_t stream) {
  uint32_t c0 = static_cast<uint32_t>(elem), c1 = static_cast<uint32_t>(elem >> 32), c2 = stream, c3 = 0;
  uint32_t k0 = static_cast<uint32_t>(seed), k1 = static_cast<uint32_t>(seed >> 32);
  for (int r = 0; r < 10; ++r) {
    uint32_t hi0, hi1;
    const uint32_t lo0 = mulhilo(0xD2511F53u, c0, &hi0);
    const uint32_t lo1 = mulhilo(0xCD9E8D57u, c2, &hi1);
    const uint32_t n0 = hi1 ^ c1 ^ k0, n2 = hi0 ^ c3 ^ k1;
    c0 = n0; c1 = lo1; c2 = n2; c3 = lo0;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  return c0;
}

// multiplier of element `elem` of dropout site `site` (0 attention probabilities, 1 dropout1 after out_proj,
// 2 dropout between ReLU and linear2, 3 dropout2 after linear2) of layer `layer`: 0 or 1 / (1 - p)
__device__ __forceinline__ float drop_mul(const Dropout& d, int layer, int site, unsigned long long elem) {
  if (!d.on) return 1.0f;
  return philox_draw(d.seed, elem, static_cast<uint32_t>(layer * 4 + site)) >= d.thr ? d.scale : 0.0f;
}

Dropout make_dropout(float p, unsigned long long seed) {
  Dropout d;
  d.seed = seed;
  d.on = p > 0.0f;
  const double t = static_cast<double>(p) * 4294967296.0;
  d.thr = d.on ? static_cast<uint32_t>(t >= 4294967295.0 ? 4294967295.0 : t) : 0u;
  d.scale = d.on ? 1.0f / (1.0f - p) : 1.0f;
  return d;
}

// ---- tensor-core GEMM: C[m, n] = sum_k A(m, k) B(k, n) over k in chunk z --------------------------------------
// mma.sync m16n8k16, split fp16 operands (hi + lo), fp32 accumulation.  Operands are read from fp32 activations
// through loaders and split on their way to shared memory, so transposes, the ConvTranspose weight layout,
// dropout masks and a row of ones (the bias gradient as one more output row) need no copies.  The order of the
// k steps is fixed, so every output is deterministic.  Gradients enter unscaled (the loss derivative per logit
// is O(1)); the loss scales, ~1e-7 for the mean over B*P*P*2 pixels, are applied in fp32 when the parameter
// gradients are written (wgrad_finish_kernel, colsum_finish_kernel).
struct Mat {   // value = p[m * sm + k * sk] (* dropout multiplier of that element); m == ones -> 1
  const float* p;
  long long sm, sk;
  long long ones = -1;
  Dropout drop{};
  int layer = 0, site = 0;
  __device__ __forceinline__ float operator()(long long m, long long k) const {
    if (m == ones) return 1.0f;
    const long long e = m * sm + k * sk;
    float v = p[e];
    if (drop.on) v *= drop_mul(drop, layer, site, static_cast<unsigned long long>(e));
    return v;
  }
  // which index walks contiguous memory (the tile loads let consecutive threads follow it)
  __device__ __forceinline__ bool first_unit() const { return sm == 1; }
  __device__ __forceinline__ bool second_unit() const { return sk == 1; }
};
// ConvTranspose weight [Cin, Cout, 2, 2] as the B operand: forward (k = ci, n = d*Cout + co) or, with
// `t`, its transpose for the input gradient (k = d*Cout + co, n = ci)
struct ConvTW {
  const float* p;
  int cout;
  bool t;
  __device__ __forceinline__ float operator()(long long k, long long n) const {
    const long long ci = t ? n : k, j = t ? k : n;
    return p[(ci * cout + j % cout) * 4 + j / cout];
  }
  __device__ __forceinline__ bool first_unit() const { return true; }   // small weights: L1 / L2 resident
  __device__ __forceinline__ bool second_unit() const { return true; }
};
struct Store {   // out[m, n] = v (+ add[m, n])
  float* p;
  long long ld;
  const float* add = nullptr;
  __device__ __forceinline__ void operator()(int, long long m, long long n, float v) const {
    const long long i = m * ld + n;
    p[i] = add ? v + add[i] : v;
  }
};
struct Partial {   // out[z][m][n] = v
  float* p;
  long long M, N;
  __device__ __forceinline__ void operator()(int z, long long m, long long n, float v) const {
    p[(z * M + m) * N + n] = v;
  }
};

constexpr int kTile = 64, kTk = 32, kLdh = kTk + 8;   // 64x64 tile, 32-deep k stage, padded fp16 rows

__device__ __forceinline__ uint32_t ld_h2(const __half* p) { return *reinterpret_cast<const uint32_t*>(p); }

__device__ __forceinline__ void mma16816(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3,
                                         uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

// Each fp32 operand v is split into fp16 hi = fp16(v) and lo = fp16(v - hi); a product is hi*hi + hi*lo + lo*hi
// (three mma.sync), which keeps about 21 bits of the operands: the forward tracks the fp32 reference closely
// enough that ReLU / GELU decisions near zero agree with it, where plain fp16 operands flip them.
// 8 warps in a 4 x 2 grid; each warp owns 16 x 32 of the tile = four m16n8 accumulators
template <class LA, class LB, class OUT>
__global__ void __launch_bounds__(256) gemm_mma_kernel(LA A, LB Bm, OUT out, long long M, long long N, long long K,
                                                       long long kchunk) {
  __shared__ __align__(16) __half As[2][kTile][kLdh];   // hi / lo, [m][k]
  __shared__ __align__(16) __half Bs[2][kTile][kLdh];   // hi / lo, [n][k]
  const long long n0 = static_cast<long long>(blockIdx.x) * kTile;
  const int z = blockIdx.z;
  const long long kb = z * kchunk, ke = kb + kchunk < K ? kb + kchunk : K;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int wm = (warp >> 1) * 16, wn = (warp & 1) * 32;
  const bool a_kfast = A.second_unit(), b_kfast = Bm.first_unit();
  // one row tile per block unless M has more row tiles than grid.y holds
  for (long long m0 = static_cast<long long>(blockIdx.y) * kTile; m0 < M; m0 += static_cast<long long>(gridDim.y) * kTile) {
    float acc[4][4];
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int r = 0; r < 4; ++r) acc[j][r] = 0.f;
    for (long long k0 = kb; k0 < ke; k0 += kTk) {
      for (int i = threadIdx.x; i < kTk * kTile; i += 256) {
        int mm = a_kfast ? i / kTk : i % kTile, kk = a_kfast ? i % kTk : i / kTile;
        long long r = m0 + mm, k = k0 + kk;
        float v = (r < M && k < ke) ? A(r, k) : 0.f;
        __half h = __float2half_rn(v);
        As[0][mm][kk] = h;
        As[1][mm][kk] = __float2half_rn(v - __half2float(h));
        mm = b_kfast ? i / kTk : i % kTile;
        kk = b_kfast ? i % kTk : i / kTile;
        r = n0 + mm;
        k = k0 + kk;
        v = (r < N && k < ke) ? Bm(k, r) : 0.f;
        h = __float2half_rn(v);
        Bs[0][mm][kk] = h;
        Bs[1][mm][kk] = __float2half_rn(v - __half2float(h));
      }
      __syncthreads();
#pragma unroll
      for (int ks = 0; ks < kTk; ks += 16) {
        uint32_t a[2][4];
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          a[u][0] = ld_h2(&As[u][wm + g][ks + 2 * t]);
          a[u][1] = ld_h2(&As[u][wm + g + 8][ks + 2 * t]);
          a[u][2] = ld_h2(&As[u][wm + g][ks + 2 * t + 8]);
          a[u][3] = ld_h2(&As[u][wm + g + 8][ks + 2 * t + 8]);
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const uint32_t bh0 = ld_h2(&Bs[0][wn + 8 * j + g][ks + 2 * t]), bh1 = ld_h2(&Bs[0][wn + 8 * j + g][ks + 2 * t + 8]);
          const uint32_t bl0 = ld_h2(&Bs[1][wn + 8 * j + g][ks + 2 * t]), bl1 = ld_h2(&Bs[1][wn + 8 * j + g][ks + 2 * t + 8]);
          mma16816(acc[j], a[1][0], a[1][1], a[1][2], a[1][3], bh0, bh1);   // small terms first
          mma16816(acc[j], a[0][0], a[0][1], a[0][2], a[0][3], bl0, bl1);
          mma16816(acc[j], a[0][0], a[0][1], a[0][2], a[0][3], bh0, bh1);
        }
      }
      __syncthreads();
    }
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const long long m = m0 + wm + g + (r >> 1) * 8, n = n0 + wn + 8 * j + 2 * t + (r & 1);
        if (m < M && n < N) out(z, m, n, acc[j][r]);
      }
  }
}

// Column tiles on grid.x, row tiles on grid.y, k chunks on grid.z.  A GEMM with more than 65535 row tiles (the
// decoder's stage-3 GEMMs have 64 B (P/16)^2 rows: from B = 16 @1024) launches 65535 of them and each block walks
// its row tiles with that stride; smaller GEMMs run one tile per block.
template <class LA, class LB, class OUT>
int tc_gemm(LA A, LB Bm, OUT out, long long M, long long N, long long K, int chunks, cudaStream_t st) {
  if (M <= 0 || N <= 0) return 0;
  const long long kchunk = chunks > 1 ? ((K + chunks - 1) / chunks + kTk - 1) / kTk * kTk : (K > 0 ? K : 1);
  const long long z = K > 0 ? (K + kchunk - 1) / kchunk : 1;
  const long long mt = (M + kTile - 1) / kTile, nt = (N + kTile - 1) / kTile;
  // make_dims bounds every GEMM of a step far below these limits
  SRB_REQUIRE(nt < 65536 && z < 65536, "train: GEMM of %lld x %lld (%lld chunks) is too large", M, N, z);
  const dim3 grid(static_cast<unsigned>(nt), static_cast<unsigned>(mt < 65535 ? mt : 65535), static_cast<unsigned>(z));
  SRB_LAUNCH(gemm_mma_kernel<LA, LB, OUT>, grid, 256, 0, st, A, Bm, out, M, N, K, kchunk);
  return 0;
}

// Number of row chunks a weight gradient over R rows is split into, and the resulting chunk count.
constexpr int kWgradChunks = 128;
long long wgrad_chunks(long long R) {
  const long long kchunk = ((R + kWgradChunks - 1) / kWgradChunks + kTk - 1) / kTk * kTk;
  return kchunk > 0 ? (R + kchunk - 1) / kchunk : 1;
}

// sum the z partials [z][M][N] in chunk order, then scatter to the reference layout:
//   mode 0 (nn.Linear): dW[n * ld + col0 + m] for m < K0, bias row m == K0 -> db[n]
//   mode 1 (ConvTranspose, N = 4*cout): dW[(m * cout + co) * 4 + d] for n = d*cout + co, db[co] = sum_d
__global__ void wgrad_finish_kernel(const float* __restrict__ part, int Z, int K0, int M, int N, int mode, int cout,
                                    long long ld, int col0, float* __restrict__ dW, float* __restrict__ db,
                                    const float* __restrict__ scale) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long MN = static_cast<long long>(M) * N;
  if (i >= MN) return;
  const int m = static_cast<int>(i / N), n = static_cast<int>(i % N);
  if (mode == 1 && m == K0) {   // bias: the four sub-pixel columns of co, each summed over the chunks
    if (n >= cout) return;
    float b = 0.f;
    for (int d = 0; d < 4; ++d) {
      float s = 0.f;
      for (int z = 0; z < Z; ++z) s += part[static_cast<long long>(z) * MN + static_cast<long long>(m) * N + d * cout + n];
      b += s;
    }
    db[n] = b * scale[0];
    return;
  }
  float s = 0.f;
  for (int z = 0; z < Z; ++z) s += part[static_cast<long long>(z) * MN + i];
  s *= scale[0];
  if (m == K0) {
    if (db) db[n] = s;
  } else if (mode == 0) {
    dW[static_cast<long long>(n) * ld + col0 + m] = s;
  } else {
    const int co = n % cout, d = n / cout;
    dW[(static_cast<long long>(m) * cout + co) * 4 + d] = s;
  }
}

// dW (and db) = sum_r A[r, :]^T G[r, :] over R rows: A is the layer input [R, K0] read through `a`
// (a.ones = K0 appends the bias row when db != null), G the output gradient [R, N]
template <class LG>
int wgrad(Mat a, int K0, LG g, int N, long long R, int mode, int cout, long long ld, int col0, float* dW,
          float* db, float* part, const float* scale, cudaStream_t st) {
  a.ones = db ? K0 : -1;
  const int M = K0 + (db ? 1 : 0);
  // A(m, r) with m the input channel: swap the strides of the row-major activation
  Mat at = a;
  at.sm = a.sk; at.sk = a.sm;
  const long long Z = wgrad_chunks(R);
  SRB_TRY(tc_gemm(at, g, Partial{part, M, N}, M, N, R, kWgradChunks, st));
  const long long MN = static_cast<long long>(M) * N;
  SRB_LAUNCH(wgrad_finish_kernel, static_cast<unsigned>((MN + 255) / 256), 256, 0, st, part, static_cast<int>(Z), K0, M,
             N, mode, cout, ld, col0, dW, db, scale);
  return 0;
}

// ---- elementwise kernels -------------------------------------------------------------------------------
__device__ __forceinline__ float gelu_f(float u) { return 0.5f * u * (1.0f + erff(u * 0.70710678118654752f)); }
__device__ __forceinline__ float gelu_grad(float u) {
  return 0.5f * (1.0f + erff(u * 0.70710678118654752f)) + u * 0.39894228040143268f * expf(-0.5f * u * u);
}

#define GRID_STRIDE(i, n) \
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < (n); \
       i += static_cast<long long>(gridDim.x) * blockDim.x)

inline unsigned ew_grid(long long n) {
  const long long g = (n + 255) / 256;
  return static_cast<unsigned>(g < 8192 ? (g > 0 ? g : 1) : 8192);
}

// z[i] += bias[i % C]; then act (1 GELU, 2 ReLU) into a (or in place when a == null)
__global__ void bias_act_kernel(float* __restrict__ z, const float* __restrict__ bias, int C, long long n, int act,
                                float* __restrict__ a) {
  GRID_STRIDE(i, n) {
    const float v = z[i] + bias[i % C];
    const float y = act == 1 ? gelu_f(v) : (act == 2 ? fmaxf(v, 0.f) : v);
    if (a) { z[i] = v; a[i] = y; } else { z[i] = y; }
  }
}
// g[i] *= act'(at x[i]): kind 1 GELU' of the pre-activation, 2 ReLU' from the post-activation, 3 ReLU' and
// the dropout multiplier of element i (site `site` of `layer`)
__global__ void act_grad_kernel(float* __restrict__ g, const float* __restrict__ x, long long n, int kind,
                                Dropout d, int layer, int site) {
  GRID_STRIDE(i, n) {
    float v = g[i];
    if (kind == 1) v *= gelu_grad(x[i]);
    else v = x[i] > 0.f ? v : 0.f;
    if (kind == 3) v *= drop_mul(d, layer, site, static_cast<unsigned long long>(i));
    g[i] = v;
  }
}
// emb [B, C, T] (NCHW) -> rows [B*T, C]
__global__ void nchw_rows_kernel(const float* __restrict__ x, int C, int T, long long n, float* __restrict__ out) {
  GRID_STRIDE(i, n) {
    const long long m = i / C;
    const int c = static_cast<int>(i % C);
    const long long b = m / T, t = m % T;
    out[i] = x[(b * C + c) * T + t];
  }
}

// LayerNorm over 128 channels, one warp per row: in = z (+ bias) [+ residual + dropout(...)]
//   decoder (LayerNorm2d, eps 1e-6):   r = z + bias;            out = GELU(g xhat + b)
//   TopoNet (post-norm, eps 1e-5):     r = x + drop(z + bias);  out = g xhat + b
__global__ void ln_fwd_kernel(const float* __restrict__ z, const float* __restrict__ bias,
                              const float* __restrict__ resid, Dropout d, int layer, int site,
                              const float* __restrict__ gam, const float* __restrict__ bet, float eps, int gelu,
                              long long rows, float* __restrict__ xh, float* __restrict__ rs, float* __restrict__ out) {
  const long long r = static_cast<long long>(blockIdx.x) * 8 + (threadIdx.x >> 5);
  if (r >= rows) return;
  const int lane = threadIdx.x & 31;
  float v[4];
  float sum = 0.f;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int c = lane + 32 * j;
    const long long e = r * 128 + c;
    float t = z[e] + bias[c];
    if (resid) t = resid[e] + t * drop_mul(d, layer, site, static_cast<unsigned long long>(e));
    v[j] = t;
    sum += t;
  }
  const float mean = warp_sum(sum) * (1.0f / 128.0f);
  float sq = 0.f;
#pragma unroll
  for (int j = 0; j < 4; ++j) { v[j] -= mean; sq += v[j] * v[j]; }
  const float rstd = rsqrtf(warp_sum(sq) * (1.0f / 128.0f) + eps);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int c = lane + 32 * j;
    const long long e = r * 128 + c;
    const float xhat = v[j] * rstd;
    xh[e] = xhat;
    const float u = gam[c] * xhat + bet[c];
    out[e] = gelu ? gelu_f(u) : u;
  }
  if (lane == 0) rs[r] = rstd;
}

// LayerNorm backward over 128 channels, one warp per row.  g: gradient of the LayerNorm output (of the GELU
// output when `gelu`, which is first turned into the gradient of g xhat + b in place, for the gamma / beta
// sums).  dx = rstd (gg - mean(gg) - xhat mean(gg xhat)), gg = g * gamma.  dx may alias g.
__global__ void ln_bwd_kernel(float* __restrict__ g, const float* __restrict__ xh, const float* __restrict__ rs,
                              const float* __restrict__ gam, const float* __restrict__ bet, int gelu, long long rows,
                              float* dx) {
  const long long r = static_cast<long long>(blockIdx.x) * 8 + (threadIdx.x >> 5);
  if (r >= rows) return;
  const int lane = threadIdx.x & 31;
  float gg[4], xv[4];
  float s1 = 0.f, s2 = 0.f;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int c = lane + 32 * j;
    const long long e = r * 128 + c;
    xv[j] = xh[e];
    float gv = g[e];
    if (gelu) {
      gv *= gelu_grad(gam[c] * xv[j] + bet[c]);
      g[e] = gv;
    }
    gg[j] = gv * gam[c];
    s1 += gg[j];
    s2 += gg[j] * xv[j];
  }
  const float m1 = warp_sum(s1) * (1.0f / 128.0f), m2 = warp_sum(s2) * (1.0f / 128.0f);
  const float rstd = rs[r];
#pragma unroll
  for (int j = 0; j < 4; ++j) dx[r * 128 + lane + 32 * j] = rstd * (gg[j] - m1 - xv[j] * m2);
}

// gamma / beta gradients of a 128-channel LayerNorm: per chunk of rows sum g*xhat and g per channel, then
// the chunks in order
constexpr int kColChunks = 256;
__global__ void __launch_bounds__(128) colsum_kernel(const float* __restrict__ g, const float* __restrict__ xh,
                                                     long long rows, long long chunk, float* __restrict__ part) {
  const int c = threadIdx.x;
  const long long r0 = blockIdx.x * chunk, r1 = r0 + chunk < rows ? r0 + chunk : rows;
  float a = 0.f, b = 0.f;
  for (long long r = r0; r < r1; ++r) {
    const float gv = g[r * 128 + c];
    a = fmaf(gv, xh[r * 128 + c], a);
    b += gv;
  }
  part[(blockIdx.x * 2 + 0) * 128 + c] = a;
  part[(blockIdx.x * 2 + 1) * 128 + c] = b;
}
__global__ void colsum_finish_kernel(const float* __restrict__ part, int Z, float* __restrict__ dg, float* __restrict__ db,
                                     const float* __restrict__ scale) {
  const int c = threadIdx.x;
  float a = 0.f, b = 0.f;
  for (int z = 0; z < Z; ++z) {
    a += part[(z * 2 + 0) * 128 + c];
    b += part[(z * 2 + 1) * 128 + c];
  }
  dg[c] = a * scale[0];
  db[c] = b * scale[0];
}
int ln_param_grads(const float* g, const float* xh, long long rows, float* part, float* dg, float* db,
                   const float* scale, cudaStream_t st) {
  const long long chunk = rows > 0 ? (rows + kColChunks - 1) / kColChunks : 1;
  const int Z = static_cast<int>(rows > 0 ? (rows + chunk - 1) / chunk : 1);
  SRB_LAUNCH(colsum_kernel, Z, 128, 0, st, g, xh, rows, chunk, part);
  SRB_LAUNCH(colsum_finish_kernel, 1, 128, 0, st, part, Z, dg, db, scale);
  return 0;
}

// ---- losses ---------------------------------------------------------------------------------------------
constexpr int kLossBlocks = 1024;

__device__ __forceinline__ double block_sum_f64(double v, double* sh /*[8]*/) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  if (lane == 0) sh[wid] = v;
  __syncthreads();
  double s = 0.0;
  if (threadIdx.x == 0)
    for (int w = 0; w < static_cast<int>(blockDim.x >> 5); ++w) s += sh[w];
  return s;
}

// Decoder logits in quad-tree order [R4, 2] (+ bias) -> the mask loss terms against the [B, P, P] targets, and
// the unscaled derivative of each term, in place.  Row r4 = (((m*4 + d1)*4 + d2)*4 + d3)*4 + d4 with m = b*T +
// ty*s + tx is pixel (ty*16 + 8 di1 + 4 di2 + 2 di3 + di4, tx*16 + ...), d = di*2 + dj.
__global__ void __launch_bounds__(256) mask_loss_kernel(float* __restrict__ lg, const float* __restrict__ bias,
                                                        const float* __restrict__ kp, const float* __restrict__ road,
                                                        long long R4, int T, int s, int P, int focal,
                                                        double* __restrict__ part) {
  __shared__ double sh[8];
  double sum = 0.0;
  GRID_STRIDE(r, R4) {
    long long q = r;
    int y = 0, x = 0;
#pragma unroll
    for (int lev = 0; lev < 4; ++lev) {
      const int d = static_cast<int>(q & 3);
      q >>= 2;
      y |= (d >> 1) << lev;
      x |= (d & 1) << lev;
    }
    const long long b = q / T, t = q % T;
    y += static_cast<int>(t / s) * 16;
    x += static_cast<int>(t % s) * 16;
    const long long pix = (b * P + y) * P + x;
    const float tgt[2] = {kp[pix], road[pix]};
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      const float xv = lg[r * 2 + c] + bias[c];
      sum += static_cast<double>(focal ? focal_term(xv, tgt[c]) : bce_term(xv, tgt[c]));
      lg[r * 2 + c] = focal ? focal_grad(xv, tgt[c]) : bce_grad(xv, tgt[c]);
    }
  }
  const double s2 = block_sum_f64(sum, sh);
  if (threadIdx.x == 0) part[blockIdx.x] = s2;
}

// output_proj: logit[t] = x[t] . w + b, one warp per token
__global__ void topo_logit_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ b,
                                  long long tok, float* __restrict__ out) {
  const long long t = static_cast<long long>(blockIdx.x) * 8 + (threadIdx.x >> 5);
  if (t >= tok) return;
  const int lane = threadIdx.x & 31;
  float acc = 0.f;
#pragma unroll
  for (int j = 0; j < 4; ++j) acc = fmaf(x[t * 128 + lane + 32 * j], w[lane + 32 * j], acc);
  acc = warp_sum(acc);
  if (lane == 0) out[t] = acc + b[0];
}

// topology BCE over the valid slots; the logit buffer becomes (sigmoid(x) - y) * valid
__global__ void __launch_bounds__(256) topo_loss_kernel(float* __restrict__ lg, const uint8_t* __restrict__ conn,
                                                        const uint8_t* __restrict__ valid, long long tok,
                                                        double* __restrict__ part) {
  __shared__ double sh[8];
  double sum = 0.0, cnt = 0.0;
  GRID_STRIDE(t, tok) {
    const float y = conn[t] ? 1.0f : 0.0f;
    const bool v = valid[t] != 0;
    const float xv = lg[t];
    if (v) {
      sum += static_cast<double>(bce_term(xv, y));
      cnt += 1.0;
    }
    lg[t] = v ? bce_grad(xv, y) : 0.0f;
  }
  const double s = block_sum_f64(sum, sh);
  __syncthreads();
  const double c = block_sum_f64(cnt, sh);
  if (threadIdx.x == 0) {
    part[2 * blockIdx.x] = s;
    part[2 * blockIdx.x + 1] = c;
  }
}

// losses[0] = mask mean, losses[1] = topology mean (NaN without a valid slot); stats = {count_valid}
__global__ void loss_finish_kernel(const double* __restrict__ mpart, const double* __restrict__ tpart, int g,
                                   double n_mask, float* __restrict__ losses, float* __restrict__ stats) {
  if (threadIdx.x != 0) return;
  double m = 0.0, t = 0.0, c = 0.0;
  for (int i = 0; i < g; ++i) {
    m += mpart[i];
    t += tpart[2 * i];
    c += tpart[2 * i + 1];
  }
  losses[0] = __double2float_rn(m / n_mask);
  losses[1] = __double2float_rn(t) / static_cast<float>(c);   // 0 / 0 = NaN, as the reference
  stats[0] = static_cast<float>(c);
}

// scale[0] = g_mask / (2 B P^2), scale[1] = g_topo / sum(valid) (NaN or inf without a valid slot, as in the
// reference): the fp32 factors of the decoder's and TopoNet's parameter gradients
__global__ void loss_scale_kernel(const float* __restrict__ g, double n_mask, const float* __restrict__ stats,
                                  float* __restrict__ scale) {
  scale[0] = static_cast<float>(static_cast<double>(g[0]) / n_mask);
  scale[1] = g[1] / stats[0];
}

// ---- TopoNet pieces --------------------------------------------------------------------------------------
// x0 = relu(PST[src] + PST[tgt, 128:] + Wo . offset + b) with Wo the last two columns of pair_proj.weight
// [128, 258]; saves the offsets and the clamped global point indices
__global__ void __launch_bounds__(128) tr_pair_kernel(const TopoPairInputs in, const float* __restrict__ w,
                                                      float* __restrict__ x0, float* __restrict__ off,
                                                      int* __restrict__ src, int* __restrict__ tgt) {
  const long long t = blockIdx.x;
  const PairToken pr = resolve_pair(in, static_cast<size_t>(t));
  const int c = threadIdx.x;
  float v = in.pst[pr.ps * 256 + c] + in.pst[pr.pt * 256 + 128 + c];
  v += w[c * 258 + 256] * pr.ox + w[c * 258 + 257] * pr.oy + in.bias[c];
  x0[t * 128 + c] = fmaxf(v, 0.f);
  if (c == 0) {
    off[t * 2] = pr.ox;
    off[t * 2 + 1] = pr.oy;
    src[t] = static_cast<int>(pr.ps);
    tgt[t] = static_cast<int>(pr.pt);
  }
}

// Self-attention of one (sample, head): Np <= 32 queries / keys of 32 dims, key-padding mask, dropout on the
// probabilities (site 0).  One 32-thread block per (sample, head), thread i = query i.
__global__ void __launch_bounds__(32) tr_attn_fwd_kernel(const float* __restrict__ qkv, const uint8_t* __restrict__ vf,
                                                         int Np, Dropout d, int layer, float* __restrict__ out) {
  __shared__ float ks[32][33], vs[32][33];
  const long long row = blockIdx.x / 4;
  const int hd = blockIdx.x % 4, i = threadIdx.x;
  const long long tok0 = row * Np;
  for (int e = threadIdx.x; e < Np * 32; e += 32) {
    const int j = e / 32, c = e % 32;
    ks[j][c] = qkv[(tok0 + j) * 384 + 128 + hd * 32 + c];
    vs[j][c] = qkv[(tok0 + j) * 384 + 256 + hd * 32 + c];
  }
  __syncthreads();
  if (i >= Np) return;
  float q[32];
#pragma unroll
  for (int c = 0; c < 32; ++c) q[c] = qkv[(tok0 + i) * 384 + hd * 32 + c];
  const float scale = 0.17677669529663687f;
  float sc[32];
  float mx = -INFINITY;
  for (int j = 0; j < Np; ++j) {
    float a = 0.f;
#pragma unroll
    for (int c = 0; c < 32; ++c) a = fmaf(q[c], ks[j][c], a);
    sc[j] = vf[tok0 + j] ? a * scale : -INFINITY;
    mx = fmaxf(mx, sc[j]);
  }
  float l = 0.f;
  for (int j = 0; j < Np; ++j) {
    sc[j] = sc[j] > -INFINITY ? expf(sc[j] - mx) : 0.f;
    l += sc[j];
  }
  float o[32];
#pragma unroll
  for (int c = 0; c < 32; ++c) o[c] = 0.f;
  const unsigned long long pbase = ((static_cast<unsigned long long>(row) * 4 + hd) * Np + i) * Np;
  for (int j = 0; j < Np; ++j) {
    const float p = sc[j] / l * drop_mul(d, layer, 0, pbase + j);
#pragma unroll
    for (int c = 0; c < 32; ++c) o[c] = fmaf(p, vs[j][c], o[c]);
  }
#pragma unroll
  for (int c = 0; c < 32; ++c) out[(tok0 + i) * 128 + hd * 32 + c] = o[c];
}

// Backward of tr_attn_fwd_kernel: dO [tok, 128] -> dQKV [tok, 384].  Phase 1 (thread = query i): the
// probabilities again, dP, dS and dq.  Phase 2 (thread = key j): dk, dv summed over the queries in order.
__global__ void __launch_bounds__(32) tr_attn_bwd_kernel(const float* __restrict__ qkv, const uint8_t* __restrict__ vf,
                                                         const float* __restrict__ dout, int Np, Dropout d, int layer,
                                                         float* __restrict__ dqkv) {
  __shared__ float qs[32][33], ks[32][33], vs[32][33], dos[32][33], pd[32][33], ds[32][33];
  const long long row = blockIdx.x / 4;
  const int hd = blockIdx.x % 4, i = threadIdx.x;
  const long long tok0 = row * Np;
  for (int e = threadIdx.x; e < 32 * 32; e += 32) {
    const int j = e / 32, c = e % 32;
    const bool in = j < Np;
    qs[j][c] = in ? qkv[(tok0 + j) * 384 + hd * 32 + c] : 0.f;
    ks[j][c] = in ? qkv[(tok0 + j) * 384 + 128 + hd * 32 + c] : 0.f;
    vs[j][c] = in ? qkv[(tok0 + j) * 384 + 256 + hd * 32 + c] : 0.f;
    dos[j][c] = in ? dout[(tok0 + j) * 128 + hd * 32 + c] : 0.f;
    pd[j][c] = ds[j][c] = 0.f;
  }
  __syncthreads();
  const float scale = 0.17677669529663687f;
  if (i < Np) {
    float p[32];
    float mx = -INFINITY;
    for (int j = 0; j < Np; ++j) {
      float a = 0.f;
#pragma unroll
      for (int c = 0; c < 32; ++c) a = fmaf(qs[i][c], ks[j][c], a);
      p[j] = vf[tok0 + j] ? a * scale : -INFINITY;
      mx = fmaxf(mx, p[j]);
    }
    float l = 0.f;
    for (int j = 0; j < Np; ++j) {
      p[j] = p[j] > -INFINITY ? expf(p[j] - mx) : 0.f;
      l += p[j];
    }
    const unsigned long long pbase = ((static_cast<unsigned long long>(row) * 4 + hd) * Np + i) * Np;
    float dot = 0.f;
    float dp[32];
    for (int j = 0; j < Np; ++j) {
      p[j] = p[j] / l;
      const float m = drop_mul(d, layer, 0, pbase + j);
      pd[i][j] = p[j] * m;
      float a = 0.f;
#pragma unroll
      for (int c = 0; c < 32; ++c) a = fmaf(dos[i][c], vs[j][c], a);
      dp[j] = a * m;
      dot = fmaf(p[j], dp[j], dot);
    }
    float dq[32];
#pragma unroll
    for (int c = 0; c < 32; ++c) dq[c] = 0.f;
    for (int j = 0; j < Np; ++j) {
      const float sj = p[j] * (dp[j] - dot);
      ds[i][j] = sj;
#pragma unroll
      for (int c = 0; c < 32; ++c) dq[c] = fmaf(sj, ks[j][c], dq[c]);
    }
#pragma unroll
    for (int c = 0; c < 32; ++c) dqkv[(tok0 + i) * 384 + hd * 32 + c] = dq[c] * scale;
  }
  __syncthreads();
  const int j = threadIdx.x;
  if (j >= Np) return;
  float dk[32], dv[32];
#pragma unroll
  for (int c = 0; c < 32; ++c) dk[c] = dv[c] = 0.f;
  for (int q = 0; q < Np; ++q) {
    const float sq = ds[q][j], pq = pd[q][j];
#pragma unroll
    for (int c = 0; c < 32; ++c) {
      dk[c] = fmaf(sq, qs[q][c], dk[c]);
      dv[c] = fmaf(pq, dos[q][c], dv[c]);
    }
  }
#pragma unroll
  for (int c = 0; c < 32; ++c) {
    dqkv[(tok0 + j) * 384 + 128 + hd * 32 + c] = dk[c] * scale;
    dqkv[(tok0 + j) * 384 + 256 + hd * 32 + c] = dv[c];
  }
}

// dX[t, c] = g[t] * w[c]
__global__ void outer_kernel(const float* __restrict__ g, const float* __restrict__ w, long long n, float* __restrict__ out) {
  GRID_STRIDE(i, n) out[i] = g[i / 128] * w[i % 128];
}

// ---- CSR of the pair tokens by point (deterministic segmented sums) --------------------------------------
__global__ void csr_count_kernel(const int* __restrict__ idx, long long n, int* __restrict__ cnt) {
  GRID_STRIDE(i, n) atomicAdd(cnt + idx[i], 1);
}
__global__ void csr_fill_kernel(const int* __restrict__ idx, long long n, const int* __restrict__ start,
                                int* __restrict__ cursor, int* __restrict__ list) {
  GRID_STRIDE(i, n) {
    const int p = idx[i];
    list[start[p] + atomicAdd(cursor + p, 1)] = static_cast<int>(i);
  }
}
// the fill order is not deterministic: sort every segment ascending.  One block per point; the token ids of a
// segment are distinct, so each one's rank is the number of smaller ids (padded samples can send thousands of
// tokens to one point, which a one-thread sort would serialise)
__global__ void __launch_bounds__(256) csr_sort_kernel(const int* __restrict__ start, int* __restrict__ list,
                                                       int* __restrict__ tmp) {
  const int b = start[blockIdx.x], e = start[blockIdx.x + 1];
  if (e - b <= 1) return;
  for (int i = b + threadIdx.x; i < e; i += blockDim.x) {
    const int v = list[i];
    int r = 0;
    for (int j = b; j < e; ++j) r += list[j] < v;
    tmp[b + r] = v;
  }
  __syncthreads();
  for (int i = b + threadIdx.x; i < e; i += blockDim.x) list[i] = tmp[i];
}
// out[p, c] = sum over the tokens of p's segment, in token order, of g[t, c]
__global__ void __launch_bounds__(128) segsum_kernel(const int* __restrict__ start, const int* __restrict__ list,
                                                     const float* __restrict__ g, float* __restrict__ out) {
  const int p = blockIdx.x, c = threadIdx.x;
  float a = 0.f;
  for (int i = start[p]; i < start[p + 1]; ++i) a += g[static_cast<long long>(list[i]) * 128 + c];
  out[static_cast<long long>(p) * 128 + c] = a;
}

__global__ void keep_kernel(Dropout d, int layer, int site, long long n, uint8_t* __restrict__ out) {
  GRID_STRIDE(i, n) out[i] = drop_mul(d, layer, site, static_cast<unsigned long long>(i)) != 0.0f;
}

#define EW(kernel, n, ...) SRB_LAUNCH(kernel, ew_grid(n), 256, 0, st, __VA_ARGS__)
#define ROWS8(kernel, rows, ...)                                                                     \
  do {                                                                                              \
    if ((rows) > 0) SRB_LAUNCH(kernel, static_cast<unsigned>(((rows) + 7) / 8), 256, 0, st, __VA_ARGS__); \
  } while (0)

// ---- workspace --------------------------------------------------------------------------------------------
struct Dims {
  int B, N, Ns, Np, P, s, T, topo_version;
  long long M, R1, R2, R3, R4, pts, tok, rows;
  bool tf;
};

int make_dims(samroad_handle_t h, const SamRoadTrainArgs* a, Dims* d) {
  SRB_REQUIRE(h && a, "train: null handle or arguments");
  int P = 0, tv = 0, sam = 0;
  SRB_TRY(samroad_handle_head_config(h, &P, &tv, &sam));
  SRB_REQUIRE(!sam, "train: USE_SAM_DECODER needs the TwoWayTransformer backward, which is not implemented");
  SRB_REQUIRE(a->B >= 1 && a->N >= 1 && a->Ns >= 1, "train: B=%d, N=%d, Ns=%d must be positive", a->B, a->N, a->Ns);
  SRB_REQUIRE(a->Np >= 1 && a->Np <= 32, "train: n_pairs=%d must be in 1..32", a->Np);
  SRB_REQUIRE(a->loss_kind == SAMROAD_LOSS_BCE || a->loss_kind == SAMROAD_LOSS_FOCAL, "train: loss kind %d",
              a->loss_kind);
  SRB_REQUIRE(a->dropout_p >= 0.0f && a->dropout_p < 1.0f, "train: dropout p=%g must be in [0, 1)",
              static_cast<double>(a->dropout_p));
  d->B = a->B; d->N = a->N; d->Ns = a->Ns; d->Np = a->Np; d->P = P; d->s = P / 16; d->T = d->s * d->s;
  d->topo_version = tv;
  d->tf = tv != SAMROAD_TOPO_NO_TRANSFORMER;
  d->M = static_cast<long long>(a->B) * d->T;
  d->R1 = 4 * d->M; d->R2 = 16 * d->M; d->R3 = 64 * d->M; d->R4 = 256 * d->M;
  d->pts = static_cast<long long>(a->B) * a->N;
  d->rows = static_cast<long long>(a->B) * a->Ns;
  d->tok = d->rows * a->Np;
  SRB_REQUIRE(d->R4 < (1LL << 31) && d->tok < (1LL << 31) / 4 && d->pts < (1LL << 31) / 256,
              "train: batch too large for one step");
  return 0;
}

struct LayerWs { float *qkv, *att, *xh1, *rs1, *x1, *h, *xh2, *rs2; };
struct TrainWs {
  // forward, kept for backward
  float* emb;                           // [B, 256, T] image embeddings
  float *f0, *xh1, *rs1, *a1, *z2, *a2, *z3, *a3, *dl;   // decoder (dl: unscaled dlogits [R4, 2])
  float *fs, *pf, *pst, *off;           // TopoNet: sampled features, relu(feature_proj), Ws f | Wt f, offsets
  int *src, *tgt, *src_start, *tgt_start, *src_list, *tgt_list, *cursor, *sort_tmp, *scan_tmp;
  uint8_t* vf;                          // fixed key-padding mask
  float* x[4];                          // layer inputs / outputs [tok, 128]
  LayerWs L[3];
  float* dlt;                           // unscaled topology dlogits [tok]
  double* part;                         // loss partials
  float* stats;                         // [1] valid count
  // backward scratch
  float* scale;                         // [2] loss scales of the decoder / TopoNet gradients
  float *g3, *g2, *g1, *gx, *gr, *gy, *gh, *gq, *gp, *gps, *gpt, *wpart;
  size_t total;
};

TrainWs layout_train(const Dims& d, void* base) {
  Layout L(base);
  TrainWs w{};
  const long long tok = d.tok, pts = d.pts;
  w.emb = L.take<float>(d.M * 256);
  w.f0 = L.take<float>(d.M * 256);
  w.xh1 = L.take<float>(d.R1 * 128); w.rs1 = L.take<float>(d.R1); w.a1 = L.take<float>(d.R1 * 128);
  w.z2 = L.take<float>(d.R2 * 64); w.a2 = L.take<float>(d.R2 * 64);
  w.z3 = L.take<float>(d.R3 * 32); w.a3 = L.take<float>(d.R3 * 32);
  w.dl = L.take<float>(d.R4 * 2);
  w.fs = L.take<float>(pts * 256); w.pf = L.take<float>(pts * 128); w.pst = L.take<float>(pts * 256);
  w.off = L.take<float>(tok * 2);
  w.src = L.take<int>(tok); w.tgt = L.take<int>(tok);
  w.src_start = L.take<int>(pts + 1); w.tgt_start = L.take<int>(pts + 1);
  w.src_list = L.take<int>(tok); w.tgt_list = L.take<int>(tok); w.cursor = L.take<int>(pts);
  w.sort_tmp = L.take<int>(tok); w.scan_tmp = L.take<int>(scan_scratch_elems(pts));
  w.vf = L.take<uint8_t>(tok);
  const int nx = d.tf ? 4 : 1;
  for (int l = 0; l < 4; ++l) w.x[l] = l < nx ? L.take<float>(tok * 128) : nullptr;
  for (int l = 0; l < (d.tf ? 3 : 0); ++l) {
    LayerWs& y = w.L[l];
    y.qkv = L.take<float>(tok * 384); y.att = L.take<float>(tok * 128);
    y.xh1 = L.take<float>(tok * 128); y.rs1 = L.take<float>(tok); y.x1 = L.take<float>(tok * 128);
    y.h = L.take<float>(tok * 128);
    y.xh2 = L.take<float>(tok * 128); y.rs2 = L.take<float>(tok);
  }
  w.dlt = L.take<float>(tok);
  w.part = L.take<double>(3 * kLossBlocks);
  w.stats = L.take<float>(1);
  w.scale = L.take<float>(2); w.g3 = L.take<float>(d.R3 * 32); w.g2 = L.take<float>(d.R2 * 64);
  w.g1 = L.take<float>(d.R1 * 128);
  w.gx = L.take<float>(tok * 128); w.gr = L.take<float>(tok * 128); w.gy = L.take<float>(tok * 128);
  w.gh = L.take<float>(tok * 128);
  w.gq = L.take<float>(tok * 384); w.gp = L.take<float>(pts * 128); w.gps = L.take<float>(pts * 128);
  w.gpt = L.take<float>(pts * 128);
  w.wpart = L.take<float>(static_cast<long long>(kWgradChunks) * 257 * 512 > kColChunks * 256LL
                  ? static_cast<long long>(kWgradChunks) * 257 * 512 : kColChunks * 256LL);
  w.total = L.bytes();
  return w;
}

const float* LP(const HeadPtrs& hp, int l, int k) { return hp.p[HP_LAYER0 + 12 * l + k]; }

// CSR of tokens by their point index
int build_csr(const int* idx, long long tok, long long pts, int* start, int* list, int* cursor, int* tmp,
              int* scan_tmp, cudaStream_t st) {
  SRB_CUDA_OK(cudaMemsetAsync(cursor, 0, pts * 4, st));
  EW(csr_count_kernel, tok, idx, tok, cursor);
  SRB_TRY(exclusive_scan(cursor, start, pts, start + pts, scan_tmp, st));
  SRB_CUDA_OK(cudaMemsetAsync(cursor, 0, pts * 4, st));
  EW(csr_fill_kernel, tok, idx, tok, start, cursor, list);
  SRB_LAUNCH(csr_sort_kernel, static_cast<unsigned>(pts), 256, 0, st, start, list, tmp);
  return 0;
}

Mat rowmajor(const float* p, long long ld) { Mat m; m.p = p; m.sm = ld; m.sk = 1; return m; }
Mat colmajor(const float* p, long long ld) { Mat m; m.p = p; m.sm = 1; m.sk = ld; return m; }
Mat dropped(Mat m, Dropout d, int layer, int site) { m.drop = d; m.layer = layer; m.site = site; return m; }

}  // namespace

// =================================================================================================
// C ABI
// =================================================================================================
extern "C" int samroad_train_workspace_bytes(samroad_handle_t h, const SamRoadTrainArgs* args, size_t* bytes) {
  SRB_REQUIRE(bytes, "samroad_train_workspace_bytes: null output");
  Dims d;
  SRB_TRY(make_dims(h, args, &d));
  *bytes = layout_train(d, nullptr).total;
  return 0;
}

extern "C" int samroad_train_forward(samroad_handle_t h, const SamRoadTrainArgs* args, const char* const* keys,
                                     const float* const* params, int n_params, const void* rgb, int rgb_dtype,
                                     const void* points, int pts_dtype, const void* pairs, int pairs_dtype,
                                     const uint8_t* valid, const uint8_t* connected, const float* keypoint_mask,
                                     const float* road_mask, void* ws, size_t ws_bytes, float* losses,
                                     float* image_embeddings, void* stream) {
  Dims d;
  SRB_TRY(make_dims(h, args, &d));
  HeadPtrs hp;
  SRB_TRY(resolve_params(keys, params, n_params, d.tf, &hp, nullptr));
  SRB_REQUIRE(rgb && points && pairs && valid && connected && keypoint_mask && road_mask && ws && losses,
              "samroad_train_forward: null input");
  SRB_REQUIRE(pts_dtype == SAMROAD_F32 || pts_dtype == SAMROAD_I64 || pts_dtype == SAMROAD_I32,
              "samroad_train_forward: points dtype %d", pts_dtype);
  SRB_REQUIRE(pairs_dtype == SAMROAD_I64 || pairs_dtype == SAMROAD_I32, "samroad_train_forward: pairs dtype %d",
              pairs_dtype);
  const TrainWs w = layout_train(d, ws);
  SRB_REQUIRE(ws_bytes >= w.total, "samroad_train_forward: workspace of %zu bytes, %zu needed", ws_bytes, w.total);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const Dropout drop = make_dropout(args->dropout_p, args->seed);
  const Dropout none = make_dropout(0.0f, 0);

  // encoder, exactly as the inference path (embeddings only)
  SRB_TRY(samroad_encode_masks(h, rgb, rgb_dtype, d.B, nullptr, nullptr, w.emb, stream));
  if (image_embeddings)
    SRB_CUDA_OK(cudaMemcpyAsync(image_embeddings, w.emb, d.M * 256 * 4, cudaMemcpyDeviceToDevice, st));

  // ---- map decoder (model.py:286-295) in quad-tree rows ----
  const float* const* P_ = hp.p;
  EW(nchw_rows_kernel, d.M * 256, w.emb, 256, d.T, d.M * 256, w.f0);
  float* z1 = w.g1;   // pre-LN scratch (backward scratch is free during the forward)
  SRB_TRY(tc_gemm(rowmajor(w.f0, 256), ConvTW{P_[HP_DEC0_W], 128, false}, Store{z1, 512}, d.M, 512, 256, 1, st));
  ROWS8(ln_fwd_kernel, d.R1, z1, P_[HP_DEC0_B], nullptr, none, 0, 0, P_[HP_DEC1_W], P_[HP_DEC1_B], 1e-6f, 1, d.R1,
        w.xh1, w.rs1, w.a1);
  SRB_TRY(tc_gemm(rowmajor(w.a1, 128), ConvTW{P_[HP_DEC3_W], 64, false}, Store{w.z2, 256}, d.R1, 256, 128, 1, st));
  EW(bias_act_kernel, d.R2 * 64, w.z2, P_[HP_DEC3_B], 64, d.R2 * 64, 1, w.a2);
  SRB_TRY(tc_gemm(rowmajor(w.a2, 64), ConvTW{P_[HP_DEC5_W], 32, false}, Store{w.z3, 128}, d.R2, 128, 64, 1, st));
  EW(bias_act_kernel, d.R3 * 32, w.z3, P_[HP_DEC5_B], 32, d.R3 * 32, 1, w.a3);
  SRB_TRY(tc_gemm(rowmajor(w.a3, 32), ConvTW{P_[HP_DEC7_W], 2, false}, Store{w.dl, 8}, d.R3, 8, 32, 1, st));
  SRB_LAUNCH(mask_loss_kernel, kLossBlocks, 256, 0, st, w.dl, P_[HP_DEC7_B], keypoint_mask, road_mask, d.R4, d.T, d.s,
             d.P, args->loss_kind == SAMROAD_LOSS_FOCAL, w.part);

  // ---- TopoNet (model.py:88-148), slow-path semantics ----
  SRB_TRY(topo_sample_features_f32(w.emb, d.B, 256, d.s, d.P, points, pts_dtype, d.N, w.fs, st));
  SRB_TRY(tc_gemm(rowmajor(w.fs, 256), colmajor(P_[HP_FP_W], 256), Store{w.pf, 128}, d.pts, 128, 256, 1, st));
  EW(bias_act_kernel, d.pts * 128, w.pf, P_[HP_FP_B], 128, d.pts * 128, 2, nullptr);
  SRB_TRY(tc_gemm(rowmajor(w.pf, 128), colmajor(P_[HP_PP_W], 258), Store{w.pst, 256}, d.pts, 128, 128, 1, st));
  SRB_TRY(tc_gemm(rowmajor(w.pf, 128), colmajor(P_[HP_PP_W] + 128, 258), Store{w.pst + 128, 256}, d.pts, 128, 128, 1,
                st));
  const TopoPairInputs pin{w.pst, nullptr, P_[HP_PP_B], points, pairs, pts_dtype, pairs_dtype, d.N, d.Ns * d.Np,
                           d.topo_version == SAMROAD_TOPO_NO_OFFSET};
  SRB_LAUNCH(tr_pair_kernel, static_cast<unsigned>(d.tok), 128, 0, st, pin, P_[HP_PP_W], w.x[0], w.off, w.src, w.tgt);
  SRB_TRY(build_csr(w.src, d.tok, d.pts, w.src_start, w.src_list, w.cursor, w.sort_tmp, w.scan_tmp, st));
  SRB_TRY(build_csr(w.tgt, d.tok, d.pts, w.tgt_start, w.tgt_list, w.cursor, w.sort_tmp, w.scan_tmp, st));
  SRB_TRY(topo_fix_valid(valid, static_cast<int>(d.rows), d.Np, w.vf, st));
  const float* xl = w.x[0];
  if (d.tf) {
    for (int l = 0; l < 3; ++l) {
      const LayerWs& L = w.L[l];
      SRB_TRY(tc_gemm(rowmajor(xl, 128), colmajor(LP(hp, l, LP_IN_W), 128), Store{L.qkv, 384}, d.tok, 384, 128, 1, st));
      EW(bias_act_kernel, d.tok * 384, L.qkv, LP(hp, l, LP_IN_B), 384, d.tok * 384, 0, nullptr);
      SRB_LAUNCH(tr_attn_fwd_kernel, static_cast<unsigned>(d.rows * 4), 32, 0, st, L.qkv, w.vf, d.Np, drop, l, L.att);
      SRB_TRY(tc_gemm(rowmajor(L.att, 128), colmajor(LP(hp, l, LP_OUT_W), 128), Store{w.gy, 128}, d.tok, 128, 128, 1, st));
      ROWS8(ln_fwd_kernel, d.tok, w.gy, LP(hp, l, LP_OUT_B), xl, drop, l, 1, LP(hp, l, LP_N1_G), LP(hp, l, LP_N1_B),
            1e-5f, 0, d.tok, L.xh1, L.rs1, L.x1);
      SRB_TRY(tc_gemm(rowmajor(L.x1, 128), colmajor(LP(hp, l, LP_L1_W), 128), Store{L.h, 128}, d.tok, 128, 128, 1, st));
      EW(bias_act_kernel, d.tok * 128, L.h, LP(hp, l, LP_L1_B), 128, d.tok * 128, 2, nullptr);
      SRB_TRY(tc_gemm(dropped(rowmajor(L.h, 128), drop, l, 2), colmajor(LP(hp, l, LP_L2_W), 128), Store{w.gy, 128},
                    d.tok, 128, 128, 1, st));
      ROWS8(ln_fwd_kernel, d.tok, w.gy, LP(hp, l, LP_L2_B), L.x1, drop, l, 3, LP(hp, l, LP_N2_G), LP(hp, l, LP_N2_B),
            1e-5f, 0, d.tok, L.xh2, L.rs2, w.x[l + 1]);
      xl = w.x[l + 1];
    }
  }
  ROWS8(topo_logit_kernel, d.tok, xl, P_[HP_OUT_W], P_[HP_OUT_B], d.tok, w.dlt);
  SRB_LAUNCH(topo_loss_kernel, kLossBlocks, 256, 0, st, w.dlt, connected, valid, d.tok, w.part + kLossBlocks);
  SRB_LAUNCH(loss_finish_kernel, 1, 32, 0, st, w.part, w.part + kLossBlocks, kLossBlocks,
             2.0 * static_cast<double>(d.R4), losses, w.stats);
  return 0;
}

extern "C" int samroad_train_backward(samroad_handle_t h, const SamRoadTrainArgs* args, const char* const* keys,
                                      const float* const* params, float* const* grads, int n_params, void* ws,
                                      size_t ws_bytes, const float* g, void* stream) {
  Dims d;
  SRB_TRY(make_dims(h, args, &d));
  HeadPtrs hp;
  int slot_of[HP_COUNT];
  SRB_REQUIRE(n_params <= HP_COUNT, "samroad_train_backward: %d parameters", n_params);
  SRB_TRY(resolve_params(keys, params, n_params, d.tf, &hp, slot_of));
  SRB_REQUIRE(ws && g && (n_params == 0 || grads), "samroad_train_backward: null argument");
  float* G[HP_COUNT] = {};
  for (int i = 0; i < n_params; ++i) {
    SRB_REQUIRE(grads[i], "samroad_train_backward: null gradient for '%s'", keys[i]);
    G[slot_of[i]] = grads[i];
  }
  const TrainWs w = layout_train(d, ws);
  SRB_REQUIRE(ws_bytes >= w.total, "samroad_train_backward: workspace of %zu bytes, %zu needed", ws_bytes, w.total);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const Dropout drop = make_dropout(args->dropout_p, args->seed);
  const float* const* P_ = hp.p;

  // ---- map decoder ----
  SRB_LAUNCH(loss_scale_kernel, 1, 1, 0, st, g, 2.0 * static_cast<double>(d.R4), w.stats, w.scale);
  SRB_TRY(wgrad(rowmajor(w.a3, 32), 32, rowmajor(w.dl, 8), 8, d.R3, 1, 2, 0, 0, G[HP_DEC7_W], G[HP_DEC7_B], w.wpart, w.scale, st));
  SRB_TRY(tc_gemm(rowmajor(w.dl, 8), ConvTW{P_[HP_DEC7_W], 2, true}, Store{w.g3, 32}, d.R3, 32, 8, 1, st));
  EW(act_grad_kernel, d.R3 * 32, w.g3, w.z3, d.R3 * 32, 1, drop, 0, 0);
  SRB_TRY(wgrad(rowmajor(w.a2, 64), 64, rowmajor(w.g3, 128), 128, d.R2, 1, 32, 0, 0, G[HP_DEC5_W], G[HP_DEC5_B],
                w.wpart, w.scale, st));
  SRB_TRY(tc_gemm(rowmajor(w.g3, 128), ConvTW{P_[HP_DEC5_W], 32, true}, Store{w.g2, 64}, d.R2, 64, 128, 1, st));
  EW(act_grad_kernel, d.R2 * 64, w.g2, w.z2, d.R2 * 64, 1, drop, 0, 0);
  SRB_TRY(wgrad(rowmajor(w.a1, 128), 128, rowmajor(w.g2, 256), 256, d.R1, 1, 64, 0, 0, G[HP_DEC3_W], G[HP_DEC3_B],
                w.wpart, w.scale, st));
  SRB_TRY(tc_gemm(rowmajor(w.g2, 256), ConvTW{P_[HP_DEC3_W], 64, true}, Store{w.g1, 128}, d.R1, 128, 256, 1, st));
  // GELU' into g1 (gradient of g xhat + b), then the LayerNorm2d backward in place
  ROWS8(ln_bwd_kernel, d.R1, w.g1, w.xh1, w.rs1, P_[HP_DEC1_W], P_[HP_DEC1_B], 1, d.R1, w.g2);
  SRB_TRY(ln_param_grads(w.g1, w.xh1, d.R1, w.wpart, G[HP_DEC1_W], G[HP_DEC1_B], w.scale, st));
  SRB_TRY(wgrad(rowmajor(w.f0, 256), 256, rowmajor(w.g2, 512), 512, d.M, 1, 128, 0, 0, G[HP_DEC0_W], G[HP_DEC0_B],
                w.wpart, w.scale, st));

  // ---- TopoNet ----
  const float* xl = d.tf ? w.x[3] : w.x[0];
  SRB_TRY(wgrad(rowmajor(xl, 128), 128, rowmajor(w.dlt, 1), 1, d.tok, 0, 0, 128, 0, G[HP_OUT_W], G[HP_OUT_B], w.wpart, w.scale + 1, st));
  EW(outer_kernel, d.tok * 128, w.dlt, P_[HP_OUT_W], d.tok * 128, w.gx);   // gx: gradient of the layer output
  if (d.tf) {
    for (int l = 2; l >= 0; --l) {
      const LayerWs& L = w.L[l];
      // norm2: gr = d(x1 + drop2(y2)), then gamma / beta
      ROWS8(ln_bwd_kernel, d.tok, w.gx, L.xh2, L.rs2, LP(hp, l, LP_N2_G), LP(hp, l, LP_N2_B), 0, d.tok, w.gr);
      SRB_TRY(ln_param_grads(w.gx, L.xh2, d.tok, w.wpart, G[HP_LAYER0 + 12 * l + LP_N2_G],
                             G[HP_LAYER0 + 12 * l + LP_N2_B], w.scale + 1, st));
      // linear2 on drop(h): dW2 = drop3(gr)^T drop2(h), db2; gh = drop3(gr) W2 * drop2' * relu'
      const Mat gy2 = dropped(rowmajor(w.gr, 128), drop, l, 3);
      SRB_TRY(wgrad(dropped(rowmajor(L.h, 128), drop, l, 2), 128, gy2, 128, d.tok, 0, 0, 128, 0,
                    G[HP_LAYER0 + 12 * l + LP_L2_W], G[HP_LAYER0 + 12 * l + LP_L2_B], w.wpart, w.scale + 1, st));
      SRB_TRY(tc_gemm(gy2, rowmajor(LP(hp, l, LP_L2_W), 128), Store{w.gh, 128}, d.tok, 128, 128, 1, st));
      EW(act_grad_kernel, d.tok * 128, w.gh, L.h, d.tok * 128, 3, drop, l, 2);
      // linear1: dW1 = gh^T x1; gx = gr + gh W1 (gradient of x1)
      SRB_TRY(wgrad(rowmajor(L.x1, 128), 128, rowmajor(w.gh, 128), 128, d.tok, 0, 0, 128, 0,
                    G[HP_LAYER0 + 12 * l + LP_L1_W], G[HP_LAYER0 + 12 * l + LP_L1_B], w.wpart, w.scale + 1, st));
      SRB_TRY(tc_gemm(rowmajor(w.gh, 128), rowmajor(LP(hp, l, LP_L1_W), 128), Store{w.gx, 128, w.gr}, d.tok, 128, 128,
                    1, st));
      // norm1: gr = d(x + drop1(y1))
      ROWS8(ln_bwd_kernel, d.tok, w.gx, L.xh1, L.rs1, LP(hp, l, LP_N1_G), LP(hp, l, LP_N1_B), 0, d.tok, w.gr);
      SRB_TRY(ln_param_grads(w.gx, L.xh1, d.tok, w.wpart, G[HP_LAYER0 + 12 * l + LP_N1_G],
                             G[HP_LAYER0 + 12 * l + LP_N1_B], w.scale + 1, st));
      // out_proj: dWo = drop1(gr)^T att; gy = drop1(gr) Wo (gradient of the attention output)
      const Mat gy1 = dropped(rowmajor(w.gr, 128), drop, l, 1);
      SRB_TRY(wgrad(rowmajor(L.att, 128), 128, gy1, 128, d.tok, 0, 0, 128, 0, G[HP_LAYER0 + 12 * l + LP_OUT_W],
                    G[HP_LAYER0 + 12 * l + LP_OUT_B], w.wpart, w.scale + 1, st));
      SRB_TRY(tc_gemm(gy1, rowmajor(LP(hp, l, LP_OUT_W), 128), Store{w.gy, 128}, d.tok, 128, 128, 1, st));
      SRB_LAUNCH(tr_attn_bwd_kernel, static_cast<unsigned>(d.rows * 4), 32, 0, st, L.qkv, w.vf, w.gy, d.Np, drop, l,
                 w.gq);
      // in_proj: dWin = gq^T x; gx = gr + gq Win (gradient of the layer input)
      const float* xin = w.x[l];
      SRB_TRY(wgrad(rowmajor(xin, 128), 128, rowmajor(w.gq, 384), 384, d.tok, 0, 0, 128, 0,
                    G[HP_LAYER0 + 12 * l + LP_IN_W], G[HP_LAYER0 + 12 * l + LP_IN_B], w.wpart, w.scale + 1, st));
      SRB_TRY(tc_gemm(rowmajor(w.gq, 384), rowmajor(LP(hp, l, LP_IN_W), 128), Store{w.gx, 128, w.gr}, d.tok, 128, 384,
                    1, st));
    }
  }
  // pair features: relu', then the offset columns and bias of pair_proj over the tokens
  EW(act_grad_kernel, d.tok * 128, w.gx, w.x[0], d.tok * 128, 2, drop, 0, 0);
  SRB_TRY(wgrad(rowmajor(w.off, 2), 2, rowmajor(w.gx, 128), 128, d.tok, 0, 0, 258, 256, G[HP_PP_W], G[HP_PP_B],
                w.wpart, w.scale + 1, st));
  // per-point sums of the token gradients by src and by tgt, then Ws / Wt over the points
  SRB_LAUNCH(segsum_kernel, static_cast<unsigned>(d.pts), 128, 0, st, w.src_start, w.src_list, w.gx, w.gps);
  SRB_LAUNCH(segsum_kernel, static_cast<unsigned>(d.pts), 128, 0, st, w.tgt_start, w.tgt_list, w.gx, w.gpt);
  SRB_TRY(wgrad(rowmajor(w.pf, 128), 128, rowmajor(w.gps, 128), 128, d.pts, 0, 0, 258, 0, G[HP_PP_W], nullptr,
                w.wpart, w.scale + 1, st));
  SRB_TRY(wgrad(rowmajor(w.pf, 128), 128, rowmajor(w.gpt, 128), 128, d.pts, 0, 0, 258, 128, G[HP_PP_W], nullptr,
                w.wpart, w.scale + 1, st));
  SRB_TRY(tc_gemm(rowmajor(w.gps, 128), rowmajor(P_[HP_PP_W], 258), Store{w.gp, 128}, d.pts, 128, 128, 1, st));
  SRB_TRY(tc_gemm(rowmajor(w.gpt, 128), rowmajor(P_[HP_PP_W] + 128, 258), Store{w.gp, 128, w.gp}, d.pts, 128, 128, 1,
                st));
  EW(act_grad_kernel, d.pts * 128, w.gp, w.pf, d.pts * 128, 2, drop, 0, 0);
  SRB_TRY(wgrad(rowmajor(w.fs, 256), 256, rowmajor(w.gp, 128), 128, d.pts, 0, 0, 256, 0, G[HP_FP_W], G[HP_FP_B],
                w.wpart, w.scale + 1, st));
  return 0;
}

extern "C" int samroad_debug_train_dropout_keep(float p, uint64_t seed, int layer, int site, int64_t n,
                                                uint8_t* keep, void* stream) {
  SRB_REQUIRE(keep && n >= 0, "samroad_debug_train_dropout_keep: bad arguments");
  SRB_REQUIRE(p >= 0.0f && p < 1.0f && layer >= 0 && layer < 3 && site >= 0 && site < 4,
              "samroad_debug_train_dropout_keep: p=%g layer=%d site=%d", static_cast<double>(p), layer, site);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (n == 0) return 0;
  EW(keep_kernel, n, make_dropout(p, seed), layer, site, n, keep);
  return 0;
}
