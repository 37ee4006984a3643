// sam_road_b200 :: wgmma GEMM  C[M,N] = A[M,K] * W[N,K]^T  (+ fused epilogue)
//
// One kernel template covers every dense contraction of the hot path (SURVEY.md §2.4 K2, K5, K9,
// K10, K11, K12, K16): fp16 operands (both K-major), fp32 accumulation in registers.
//
//   warpgroup 0     : TMA producer (one thread; cp.async.bulk.tensor, 128B-swizzled 128x64 / BNx64
//                     boxes), registers handed to the consumers with setmaxnreg
//   warpgroups 1, 2 : consumers.  Each issues wgmma m64 x BN x 16 for its 64 rows of the 128-row
//                     tile, then stages its fp32 accumulators in shared memory and runs the fused
//                     epilogue over them: warp w of consumer g reads rows 32*(2g + (w&1)) .. +31 (one
//                     row per lane) and columns half (w>>1) of the tile.  Streaming epilogues (EpiF16)
//                     transpose each 32x32 fp32 block through a per-warp smem scratch so that global
//                     stores are row-contiguous (8 lanes x 16 B per row); row-statistics epilogues
//                     (EpiLN, EpiDecFinal) keep one row per thread.
//
// Persistent CTAs (grid = min(#tiles, #SMs)) and a STAGES-deep smem ring between TMA and the MMAs.
// The accumulator staging area reuses the ring (an m128 x n256 fp32 tile needs 130 KB, and a second
// buffer of that size does not fit next to the ring in 227 KB), so the producer starts the next
// tile's loads once the epilogue has read the accumulators.  Tile order is n-fastest so the CTAs
// running concurrently share the same A rows (L2 reuse); the weights (<= 4.7 MB per layer) stay
// L2-resident.
//
// Reference semantics implemented by the epilogues:
//   nn.Linear (+bias)                       image_encoder.py:212-213,227,238; common.py:21-26
//   GELU(erf)                               common.py:18-26, model.py:285
//   x + pos_embed, shortcut + x             image_encoder.py:108-109,179-180
//   LayerNorm2d (biased var, eps in sqrt)   common.py:31-43
//   nn.LayerNorm post-norm (TopoNet)        model.py:74-85 (torch TransformerEncoderLayer)
//   ConvTranspose2d(k=2,s=2) as GEMM        model.py:286-295 (SURVEY.md §8a P7)
#pragma once

#include <type_traits>

#include "common.cuh"
#include "ops.h"

namespace srb {

constexpr int kGemmBM = 128;
constexpr int kGemmBK = 64;
constexpr int kGemmThreads = 384;
constexpr int kGemmEpiWarps = 8;
constexpr int kGemmScratchFloats = 32 * 36;   // per epilogue warp: 32x32 fp32 block, rows padded to 36


__device__ __forceinline__ float apply_act(float x, int act) {
  if (act == ACT_GELU || act == ACT_GELU_SCALAR) return gelu_erf_fast(x);
  if (act == ACT_RELU) return fmaxf(x, 0.0f);
  if (act == ACT_SIGMOID) return sigmoidf_(x);
  return x;
}

// One accumulator row (this lane's row of the tile, starting at the warp's first column) in the
// shared-memory staging area.
struct AccRow {
  const float* p;
  __device__ __forceinline__ void load(int chunk, float (&v)[32]) const {
    const float4* s = reinterpret_cast<const float4*>(p + chunk * 32);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float4 x = s[i];
      v[4 * i] = x.x; v[4 * i + 1] = x.y; v[4 * i + 2] = x.z; v[4 * i + 3] = x.w;
    }
  }
};

// ------------------------------------------------------------------------------------------------
// Streaming epilogues.  A warp owns 32 tile rows (a row quarter of the tile) x n_cols columns.  Per
// 32-column chunk: lane r holds row r's 32 accumulators -> scratch[r][0..31] (row pitch 36 floats,
// float4 accesses, conflict-free) -> re-read as "lane l holds columns 4*(l&7).. of row 4*j + (l>>3)", j = 0..7 ->
// bias / activation / residual in that layout -> 8 lanes cover 128 (fp32) or 64 (fp16) contiguous
// bytes of a row per store instruction.
// ------------------------------------------------------------------------------------------------
template <class F>
__device__ __forceinline__ void epi_stream_chunks(int n_cols, const AccRow& row, float* scratch,
                                                  int lane, F&& body) {
  const int nchunks = n_cols >> 5;
  const int cc = (lane & 7) * 4, rsub = lane >> 3;
  for (int c = 0; c < nchunks; ++c) {
    float v[32];
    row.load(c, v);
    // 16-byte accesses with a 36-float row pitch are bank-conflict free in both directions
    float4* wp = reinterpret_cast<float4*>(scratch + lane * 36);
#pragma unroll
    for (int i = 0; i < 8; ++i) wp[i] = make_float4(v[4 * i], v[4 * i + 1], v[4 * i + 2], v[4 * i + 3]);
    __syncwarp();
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int rr = 4 * j + rsub;
      body(c, rr, cc, *reinterpret_cast<const float4*>(scratch + rr * 36 + cc));
    }
    __syncwarp();
  }
}

// Epilogue 1: out16[m,n] = act(acc + bias[n])                       (qkv, MLP lin1, TopoNet lin)
struct EpiF16 {
  static constexpr bool kSplitCols = true;
  struct Params {
    __half* out;          // [M, ldo]
    const float* bias;    // [N] or null
    int ldo;
    int act;
  };
  static __device__ __forceinline__ void run(const Params& p, int m0, int M, int n_base, int n_cols,
                                             const AccRow& row, float* scratch, int lane) {
    if (p.act >= ACT_PROBE_SKIP) {          // timing ablations (tools/gemm_probe.py), never a result
      if (p.act == ACT_PROBE_SKIP) return;
      if (p.act == ACT_PROBE_ACC) {
        float acc = 0.f;
        for (int c = 0; c < (n_cols >> 5); ++c) {
          float v[32];
          row.load(c, v);
#pragma unroll
          for (int i = 0; i < 32; ++i) acc += v[i];
        }
        if (acc == 1234.5678f) p.out[0] = __float2half(acc);
        return;
      }
    }
    const bool probe_nostore = p.act == ACT_PROBE_NOSTORE;
    const int act = probe_nostore ? ACT_GELU : p.act;
    epi_stream_chunks(n_cols, row, scratch, lane, [&](int c, int rr, int cc, float4 x) {
      const int n = n_base + c * 32 + cc;
      if (p.bias) {
        const float4 b = __ldg(reinterpret_cast<const float4*>(p.bias + n));
        x.x += b.x; x.y += b.y; x.z += b.z; x.w += b.w;
      }
      if (act == ACT_GELU) {
        const float2 g0 = gelu_erf_fast2(make_float2(x.x, x.y));
        const float2 g1 = gelu_erf_fast2(make_float2(x.z, x.w));
        x = make_float4(g0.x, g0.y, g1.x, g1.y);
      } else if (act != ACT_NONE) {
        x.x = apply_act(x.x, act); x.y = apply_act(x.y, act);
        x.z = apply_act(x.z, act); x.w = apply_act(x.w, act);
      }
      const int m = m0 + rr;
      if (m < M && !(probe_nostore && x.x != 1234.5678f)) {
        uint2 u;
        u.x = pack_half2(x.x, x.y);
        u.y = pack_half2(x.z, x.w);
        *reinterpret_cast<uint2*>(p.out + static_cast<size_t>(m) * p.ldo + n) = u;
      }
    });
  }
};

// Epilogue 2: out32[m,n] = acc + bias[n] + resid[m,n] + pos[m % pos_rows, n]
//             (patch-embed + pos_embed, attention proj + shortcut, MLP lin2 + shortcut; plain f32)
struct EpiF32 {
  static constexpr bool kSplitCols = true;
  struct Params {
    float* out;           // [M, ldo]
    const float* bias;    // [N] or null
    const float* resid;   // [M, ldo] or null (may alias out)
    const float* pos;     // [pos_rows, N] or null
    int ldo;
    int pos_rows;
    int n_total;
  };
  // fp32 in/out makes this epilogue HBM-bound for short K (attention proj): one row per lane with
  // 128 B contiguous per lane and chunk, and the residual of chunk c+1 prefetched into registers
  // while chunk c is processed, keeps more bytes in flight than the transposed scheme.
  static __device__ __forceinline__ void run(const Params& p, int m0, int M, int n_base, int n_cols,
                                             const AccRow& row, float* /*scratch*/, int lane) {
    const int nchunks = n_cols >> 5;
    const int m = m0 + lane;
    const bool valid = m < M;
    const float* rrow = (p.resid && valid) ? p.resid + static_cast<size_t>(m) * p.ldo + n_base : nullptr;
    const float* prow = (p.pos && valid)
                            ? p.pos + static_cast<size_t>(m % p.pos_rows) * p.n_total + n_base
                            : nullptr;
    float* orow = p.out + static_cast<size_t>(valid ? m : 0) * p.ldo + n_base;
    float4 nxt[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) nxt[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (rrow && nchunks > 0) {
#pragma unroll
      for (int i = 0; i < 8; ++i) nxt[i] = reinterpret_cast<const float4*>(rrow)[i];
    }
    for (int c = 0; c < nchunks; ++c) {
      float4 cur[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) cur[i] = nxt[i];
      if (rrow && c + 1 < nchunks) {
#pragma unroll
        for (int i = 0; i < 8; ++i) nxt[i] = reinterpret_cast<const float4*>(rrow + (c + 1) * 32)[i];
      }
      float v[32];
      row.load(c, v);
      const int n0 = c * 32;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        float4 x = make_float4(v[4 * i] + cur[i].x, v[4 * i + 1] + cur[i].y, v[4 * i + 2] + cur[i].z,
                               v[4 * i + 3] + cur[i].w);
        if (p.bias) {
          const float4 b = __ldg(reinterpret_cast<const float4*>(p.bias + n_base + n0) + i);
          x.x += b.x; x.y += b.y; x.z += b.z; x.w += b.w;
        }
        if (prow) {
          const float4 b = __ldg(reinterpret_cast<const float4*>(prow + n0) + i);
          x.x += b.x; x.y += b.y; x.z += b.z; x.w += b.w;
        }
        if (valid) reinterpret_cast<float4*>(orow + n0)[i] = x;
      }
    }
  }
};

// ------------------------------------------------------------------------------------------------
// Epilogue 3: grouped row LayerNorm.  x = acc + bias + resid; per group of `group` consecutive
// columns: y = (x - mean) / sqrt(var + eps) * gamma[n % group] + beta[n % group]; y = act(y).
// The tile must hold whole groups (BN % group == 0).  Three accumulator passes (mean, var, write) keep the
// exact two-pass variance of torch.  All eight epilogue warps work: the two warps of a row
// quarter split the tile's columns; when a group fits into one half they are independent, when it
// spans the tile (neck: group = BN = 256) they combine their partial sums through their smem scratch
// and a 64-thread named barrier.  Outputs (each optional): fp16 row-major, fp32 row-major, fp32 NCHW
// ([b, n, tok] with tok = m % tokens, b = m / tokens) for the API-visible embeddings.
// ------------------------------------------------------------------------------------------------
struct EpiLN {
  static constexpr bool kSplitCols = true;
  struct Params {
    __half* out16;        // [M, ldo] or null
    float* out32;         // [M, ldo] or null
    float* out_nchw;      // [M/tokens, N, tokens] or null
    const float* bias;    // [N] or null
    const float* resid;   // [M, ldo] fp32 or null
    const float* gamma;   // [group]
    const float* beta;    // [group]
    float eps;
    int ldo;
    int group;
    int act;
    int tokens;
    int n_total;
  };
  static __device__ __forceinline__ void load_x(const Params& p, int m, bool valid, int n0,
                                                int chunk, const AccRow& row, float (&v)[32]) {
    row.load(chunk, v);
    if (p.bias) {
      const float4* b4 = reinterpret_cast<const float4*>(p.bias + n0);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float4 b = __ldg(b4 + i);
        v[4 * i + 0] += b.x; v[4 * i + 1] += b.y; v[4 * i + 2] += b.z; v[4 * i + 3] += b.w;
      }
    }
    if (p.resid && valid) {
      const float4* r4 =
          reinterpret_cast<const float4*>(p.resid + static_cast<size_t>(m) * p.ldo + n0);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float4 b = r4[i];
        v[4 * i + 0] += b.x; v[4 * i + 1] += b.y; v[4 * i + 2] += b.z; v[4 * i + 3] += b.w;
      }
    }
  }
  static __device__ __forceinline__ void run(const Params& p, int m0, int M, int n_base, int n_cols,
                                             const AccRow& row, float* scratch, int lane) {
    const int m = m0 + lane;
    const bool valid = m < M;
    if (n_cols <= 0) return;
    const bool shared = p.group > n_cols;              // one group spans both column halves
    const int span = shared ? n_cols : p.group;        // columns of a group this warp owns
    const int cpg = span >> 5;                         // chunks per group (mine)
    const int ngroups = n_cols / span;
    const float inv_g = 1.0f / static_cast<float>(p.group);
    // partner warp of the same row quarter: its scratch is 4 slots away
    const int half = (n_base / n_cols) & 1;
    const float* partner = scratch + (half ? -4 : 4) * kGemmScratchFloats;
    const int pair_bar = 1 + ((m0 >> 5) & 3);
    for (int g = 0; g < ngroups; ++g) {
      float mean = 0.f;
      for (int c = 0; c < cpg; ++c) {
        float v[32];
        load_x(p, m, valid, n_base + (g * cpg + c) * 32, g * cpg + c, row, v);
#pragma unroll
        for (int i = 0; i < 32; ++i) mean += v[i];
      }
      if (shared) {
        scratch[lane] = mean;
        asm volatile("bar.sync %0, 64;" ::"r"(pair_bar) : "memory");
        mean += partner[lane];
      }
      mean *= inv_g;
      float var = 0.f;
      for (int c = 0; c < cpg; ++c) {
        float v[32];
        load_x(p, m, valid, n_base + (g * cpg + c) * 32, g * cpg + c, row, v);
#pragma unroll
        for (int i = 0; i < 32; ++i) {
          const float d = v[i] - mean;
          var = fmaf(d, d, var);
        }
      }
      if (shared) {
        scratch[32 + lane] = var;
        asm volatile("bar.sync %0, 64;" ::"r"(pair_bar) : "memory");
        var += partner[32 + lane];
      }
      const float rstd = rsqrtf(var * inv_g + p.eps);
      for (int c = 0; c < cpg; ++c) {
        float v[32];
        const int n0 = n_base + (g * cpg + c) * 32;
        load_x(p, m, valid, n0, g * cpg + c, row, v);
        const int gi = n0 % p.group;                   // column inside its LayerNorm group
#pragma unroll
        for (int i = 0; i < 32; i += 2) {
          const float2 gm = __ldg(reinterpret_cast<const float2*>(p.gamma + gi + i));
          const float2 bt = __ldg(reinterpret_cast<const float2*>(p.beta + gi + i));
          float2 y = make_float2((v[i] - mean) * rstd * gm.x + bt.x, (v[i + 1] - mean) * rstd * gm.y + bt.y);
          if (p.act == ACT_GELU) y = gelu_erf_fast2(y);
          else if (p.act != ACT_NONE) y = make_float2(apply_act(y.x, p.act), apply_act(y.y, p.act));
          v[i] = y.x; v[i + 1] = y.y;
        }
        if (valid) {
          if (p.out16) {
            uint4* o = reinterpret_cast<uint4*>(p.out16 + static_cast<size_t>(m) * p.ldo + n0);
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              uint4 u;
              u.x = pack_half2(v[8 * i + 0], v[8 * i + 1]);
              u.y = pack_half2(v[8 * i + 2], v[8 * i + 3]);
              u.z = pack_half2(v[8 * i + 4], v[8 * i + 5]);
              u.w = pack_half2(v[8 * i + 6], v[8 * i + 7]);
              o[i] = u;
            }
          }
          if (p.out32) {
            float4* o = reinterpret_cast<float4*>(p.out32 + static_cast<size_t>(m) * p.ldo + n0);
#pragma unroll
            for (int i = 0; i < 8; ++i)
              o[i] = make_float4(v[4 * i + 0], v[4 * i + 1], v[4 * i + 2], v[4 * i + 3]);
          }
          if (p.out_nchw) {
            const int b = m / p.tokens, t = m % p.tokens;
            float* o = p.out_nchw + (static_cast<size_t>(b) * p.n_total + n0) * p.tokens + t;
#pragma unroll
            for (int i = 0; i < 32; ++i) o[static_cast<size_t>(i) * p.tokens] = v[i];
          }
        }
      }
    }
  }
};

// ------------------------------------------------------------------------------------------------
// Epilogue 4: last two stages of the naive map decoder (model.py:292-294,490-491).
// The GEMM is ConvT(64->32,k2,s2) with columns ordered (sub3, co): a tile row is one 128x128-res
// ... one stage-3 input pixel; each 32-column chunk is one 2x upsampled sub-pixel with 32 channels.
// Per chunk: h = GELU(acc + b3) ; ConvT(32->2,k2,s2): out[co, di, dj] = sum_ci h[ci] W4[ci,co,di,dj]
// + b4[co]; writes logits and sigmoid scores straight into NHWC [B, P, P, 2].
// Row index r of the GEMM encodes the pixel hierarchy: r = ((b*s*s + i*s + j)*4 + d1)*4 + d2,
// d = di*2 + dj (see decoder weight packing in pack.cu).
//
// kPerToken = false (even s): a warp's two tokens (i, j), (i, j+1) are horizontally adjacent and leave
// in one 32-pixel-wide box.  kPerToken = true (odd s): the warp's first token has an even index, so a
// pair can straddle a row end ((i, s-1) with (i+1, 0)) or an image boundary; each token is staged
// separately and stored with a 16-pixel-wide box at its own (b, i, j).
// ------------------------------------------------------------------------------------------------
template <bool kPerToken>
struct EpiDecFinal {
  static constexpr bool kSplitCols = true;     // column half 0: sub-pixels d3 = 0,1; half 1: d3 = 2,3
  struct Params {
    // [B, P, P, 2] fp32 seen as 4-D (x: 2P floats | di: 2 | h: 2 | k: B*P/4), image row = 4k + 2h + di;
    // box {64 floats, 2, 1, 4}: the 2 x 16 output pixels x 8 rows one warp produces per tile and half
    // (kPerToken: box {32 floats, 2, 1, 4}, one token's 16 pixels)
    CUtensorMap tm_scores, tm_logits;
    int has_scores, has_logits;
    const float* bias3;   // [32]
    const float* w4;      // [32 ci][8 = (di,dj,co)] fp32
    const float* bias4;   // [2]
    int s;                // feature map side (P/16)
    int P;
  };
  // One lane = one stage-3 pixel (tile row), this warp's column half = two of its four 2x-upsampled
  // sub-pixels d3; per sub-pixel: h = GELU(acc + b3) (32 channels, packed fp32x2 math), the final
  // ConvT(32->2,k2,s2) as 8 dot products, sigmoid.  The warp's 32 rows are 2 adjacent tokens, i.e. a
  // 16-row x 32-pixel patch of the mask of which this half owns rows 4k + 2*half + di: staged in smem
  // as the dense TMA box and written with one 4-D TMA store per output (whole 128 B lines, where the
  // old direct epilogue scattered 16 B pieces).
  static __device__ __forceinline__ void run(const Params& p, int m0, int M, int n_base, int n_cols,
                                             const AccRow& row, float* scratch, int lane) {
    const int half = n_base >> 6;
    const int m = m0 + lane;
    const int d2 = m & 3, d1 = (m >> 2) & 3;
    const int tl = lane >> 4;                                   // which of the warp's two tokens
    const int k = (d1 >> 1) * 2 + (d2 >> 1);                    // image row group inside the token
    const int xq = (d1 & 1) * 2 + (d2 & 1);                     // 4-pixel column group inside the token
    float* sS = scratch;                                        // [k 4][di 2][64 floats]
    float* sL = scratch + 512;
    const float2 b4 = make_float2(__ldg(p.bias4 + 0), __ldg(p.bias4 + 1));
    if (lane == 0) bulk_wait_group_read<0>();                   // previous tile's stores have left smem
    __syncwarp();
#pragma unroll
    for (int cc = 0; cc < 2; ++cc) {
      float v[32];
      row.load(cc, v);
      float2 o[4];                                              // (di,dj) x co
#pragma unroll
      for (int q = 0; q < 4; ++q) o[q] = b4;
#pragma unroll
      for (int ci = 0; ci < 32; ci += 2) {
        const float2 bb = __ldg(reinterpret_cast<const float2*>(p.bias3 + ci));
        const float2 hh = gelu_erf_fast2(fadd2(make_float2(v[ci], v[ci + 1]), bb));
        const float4* wp = reinterpret_cast<const float4*>(p.w4 + ci * 8);
        const float4 w0 = __ldg(wp), w1 = __ldg(wp + 1), w2 = __ldg(wp + 2), w3 = __ldg(wp + 3);
        const float2 h0 = make_float2(hh.x, hh.x), h1 = make_float2(hh.y, hh.y);
        o[0] = ffma2(h0, make_float2(w0.x, w0.y), o[0]);
        o[1] = ffma2(h0, make_float2(w0.z, w0.w), o[1]);
        o[2] = ffma2(h0, make_float2(w1.x, w1.y), o[2]);
        o[3] = ffma2(h0, make_float2(w1.z, w1.w), o[3]);
        o[0] = ffma2(h1, make_float2(w2.x, w2.y), o[0]);
        o[1] = ffma2(h1, make_float2(w2.z, w2.w), o[1]);
        o[2] = ffma2(h1, make_float2(w3.x, w3.y), o[2]);
        o[3] = ffma2(h1, make_float2(w3.z, w3.w), o[3]);
      }
#pragma unroll
      for (int di = 0; di < 2; ++di) {
        // even s: [k 4][di 2][64 floats = 2 tokens x 16 px x 2]; odd s: [token 2][k 4][di 2][32 floats]
        const int off = kPerToken ? tl * 256 + (k * 2 + di) * 32 + ((xq * 2 + cc) * 2) * 2
                                  : (k * 2 + di) * 64 + (tl * 16 + (xq * 2 + cc) * 2) * 2;
        const float4 lg = make_float4(o[di * 2].x, o[di * 2].y, o[di * 2 + 1].x, o[di * 2 + 1].y);
        if (p.has_logits) *reinterpret_cast<float4*>(sL + off) = lg;
        if (p.has_scores)
          *reinterpret_cast<float4*>(sS + off) =
              make_float4(sigmoidf_(lg.x), sigmoidf_(lg.y), sigmoidf_(lg.z), sigmoidf_(lg.w));
      }
    }
    fence_proxy_async_smem();
    __syncwarp();
    if (lane == 0 && m0 < M) {
      const int pix0 = m0 >> 4;                                 // first of the warp's two tokens
      const int ss = p.s * p.s;
#pragma unroll
      for (int t = 0; t < (kPerToken ? 2 : 1); ++t) {
        const int pix = pix0 + t;
        if (kPerToken && pix >= (M >> 4)) break;                // B*s*s odd: the last warp has one token
        const int b = pix / ss;
        const int ij = pix - b * ss;
        const int i = ij / p.s, j = ij - i * p.s;
        const int c0 = j * 32, c3 = (b * p.P + i * 16) >> 2;
        if (p.has_scores) tma_store_4d(&p.tm_scores, sS + t * 256, c0, 0, half, c3);
        if (p.has_logits) tma_store_4d(&p.tm_logits, sL + t * 256, c0, 0, half, c3);
      }
      bulk_commit_group();
    }
    (void)n_cols;
  }
  static __device__ __forceinline__ void drain(int lane) {
    if (lane == 0) bulk_wait_group<0>();
  }
};

// ------------------------------------------------------------------------------------------------
// The kernel
// ------------------------------------------------------------------------------------------------
template <int BN, int STAGES>
struct GemmSmem {
  static constexpr int kABytes = kGemmBM * kGemmBK * 2;
  static constexpr int kBBytes = BN * kGemmBK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kAccPitch = BN + 4;                       // floats; conflict-free row reads
  static_assert(kGemmBM * kAccPitch * 4 <= STAGES * kStageBytes, "accumulators must fit the ring");
  static constexpr int kBarOffset = STAGES * kStageBytes;
  static constexpr int kScratchOffset = kBarOffset + 256;
  static constexpr int kTotal = kScratchOffset + kGemmEpiWarps * kGemmScratchFloats * 4 + 1024;
};

template <int BN>
struct WgmmaTile;
template <>
struct WgmmaTile<128> {
  static __device__ __forceinline__ void mma(float (&d)[64], uint64_t a, uint64_t b, uint32_t acc) {
    wgmma_m64n128k16(d, a, b, acc);
  }
};
template <>
struct WgmmaTile<256> {
  static __device__ __forceinline__ void mma(float (&d)[128], uint64_t a, uint64_t b, uint32_t acc) {
    wgmma_m64n256k16(d, a, b, acc);
  }
};

template <int BN, int STAGES, class Epi>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
               int M, int N, int K, const __grid_constant__ typename Epi::Params ep, int conv_s) {
  // conv_s > 0: implicit 3x3 / pad 1 convolution over an NHWC fp16 image [B, conv_s, conv_s, C] (tmA
  // is then its 4-D map with box {64 ch, conv_s, 128/conv_s, 1}): row m is a pixel, K = 9*C is
  // ordered (tap, channel) and k-block kb reads the channel block of the tap-shifted 128-pixel slab;
  // out-of-image taps arrive as TMA zero fill.  (neck conv, image_encoder.py:96-103)
  using SM = GemmSmem<BN, STAGES>;
  static_assert(Epi::kSplitCols, "the consumer warps split every tile into two column halves");
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + ((1024u - (raw_addr & 1023u)) & 1023u);

  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + SM::kBarOffset);
  uint64_t* empty_bar = full_bar + STAGES;
  uint64_t* accfree_bar = empty_bar + STAGES;     // the epilogue has read the staged accumulators

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = warp >> 2;

  const int num_m = (M + kGemmBM - 1) / kGemmBM;
  const int num_n = (N + BN - 1) / BN;
  const int num_tiles = num_m * num_n;
  const int num_k = (K + kGemmBK - 1) / kGemmBK;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], kGemmEpiWarps);
    }
    mbar_init(accfree_bar, kGemmEpiWarps);
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    // ===================== TMA producer =====================
    setmaxnreg_dec<40>();
    if (warp == 0 && lane == 0) {
      int stage = 0;
      uint32_t phase = 0, accphase = 0;
      bool first = true;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int m_blk = tile / num_n, n_blk = tile % num_n;
        if (!first) {                      // the ring holds the previous tile's accumulators
          mbar_wait(accfree_bar, accphase);
          accphase ^= 1u;
        }
        first = false;
        for (int kb = 0; kb < num_k; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1u);
          uint8_t* sa = smem + stage * SM::kStageBytes;
          uint8_t* sb = sa + SM::kABytes;
          mbar_arrive_expect_tx(&full_bar[stage], SM::kStageBytes);
          if (conv_s > 0) {
            const int cbs = K / (9 * kGemmBK);           // channel blocks per tap
            const int tap = kb / cbs, cb = kb - tap * cbs;
            const int tok0 = m_blk * kGemmBM, ss = conv_s * conv_s;
            const int b = tok0 / ss, y0 = (tok0 - b * ss) / conv_s;
            tma_load_4d(sa, &tmA, &full_bar[stage], cb * kGemmBK, tap % 3 - 1, y0 + tap / 3 - 1, b);
          } else {
            tma_load_2d(sa, &tmA, &full_bar[stage], kb * kGemmBK, m_blk * kGemmBM);
          }
          tma_load_2d(sb, &tmB, &full_bar[stage], kb * kGemmBK, n_blk * BN);
          if (++stage == STAGES) { stage = 0; phase ^= 1u; }
        }
      }
    }
  } else {
    // ===================== consumers: MMA + epilogue =====================
    setmaxnreg_inc<232>();
    const int g = wg - 1;                      // consumer index: tile rows 64g .. 64g+63
    const int w = warp & 3;                    // warp inside the warpgroup
    const int q = 2 * g + (w & 1);             // epilogue row quarter
    const int half = w >> 1;                   // epilogue column half
    float* scratch = reinterpret_cast<float*>(smem + SM::kScratchOffset) + (half * 4 + q) * kGemmScratchFloats;
    float* accs = reinterpret_cast<float*>(smem);
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int m_blk = tile / num_n, n_blk = tile % num_n;
      float d[BN / 2];
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) d[i] = 0.f;
      int prev = -1;
      for (int kb = 0; kb < num_k; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t a_addr = smem_u32(smem + stage * SM::kStageBytes);
        const uint64_t adesc = wgmma_desc_k128(a_addr + g * (64 * kGemmBK * 2));
        const uint64_t bdesc = wgmma_desc_k128(a_addr + SM::kABytes);
        wgmma_fence_operand(d);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kGemmBK / 16; ++k)
          WgmmaTile<BN>::mma(d, adesc + static_cast<uint64_t>(2 * k), bdesc + static_cast<uint64_t>(2 * k),
                             (kb | k) != 0 ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<1>();                       // the previous k-block's MMAs have read their stage
        wgmma_fence_operand(d);
        if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
        prev = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1u; }
      }
      wgmma_wait<0>();
      wgmma_fence_operand(d);
      if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
      // both consumers are done with the ring: stage the accumulators there
      named_bar_sync(5, 256);
      {
        const int r0 = 64 * g + 16 * w + (lane >> 2);
        const int c0 = 2 * (lane & 3);
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          *reinterpret_cast<float2*>(accs + r0 * SM::kAccPitch + 8 * j + c0) = make_float2(d[4 * j], d[4 * j + 1]);
          *reinterpret_cast<float2*>(accs + (r0 + 8) * SM::kAccPitch + 8 * j + c0) =
              make_float2(d[4 * j + 2], d[4 * j + 3]);
        }
      }
      named_bar_sync(6 + g, 128);             // this consumer's 64 rows are staged
      const int m0 = m_blk * kGemmBM + q * 32;
      const int n_tile = min(BN, N - n_blk * BN);          // valid columns of this tile
      const int col0 = half * (BN / 2);
      const int n_cols = max(0, min(BN / 2, n_tile - col0));
      AccRow row{accs + (q * 32 + lane) * SM::kAccPitch + col0};
      Epi::run(ep, m0, M, n_blk * BN + col0, n_cols, row, scratch, lane);
      fence_proxy_async_smem();               // generic accesses before the next TMA writes
      __syncwarp();
      if (lane == 0) mbar_arrive(accfree_bar);
    }
    if constexpr (std::is_same<Epi, EpiDecFinal<false>>::value || std::is_same<Epi, EpiDecFinal<true>>::value)
      Epi::drain(lane);
  }
}

// ------------------------------------------------------------------------------------------------
// host launcher
// ------------------------------------------------------------------------------------------------
int device_sm_count();

template <int BN, int STAGES, class Epi>
int launch_gemm_tc(const __half* A, int lda, const __half* W, int ldw, int M, int N, int K,
                   const typename Epi::Params& ep, cudaStream_t stream, int conv_s = 0) {
  using SM = GemmSmem<BN, STAGES>;
  SRB_REQUIRE(M > 0 && N > 0 && K > 0, "gemm: empty problem M=%d N=%d K=%d", M, N, K);
  SRB_REQUIRE(N % 32 == 0, "gemm: N=%d must be a multiple of 32", N);
  SRB_REQUIRE(K % 8 == 0 && lda % 8 == 0 && ldw % 8 == 0,
              "gemm: K/lda/ldw (%d/%d/%d) must be multiples of 8", K, lda, ldw);
  CUtensorMap tmA, tmB;
  if (conv_s > 0) {
    // A = NHWC image [M / conv_s^2, conv_s, conv_s, C = lda]
    const int C = lda;
    SRB_REQUIRE(K == 9 * C && C % kGemmBK == 0 && kGemmBM % conv_s == 0 && (conv_s * conv_s) % kGemmBM == 0 &&
                    M % (conv_s * conv_s) == 0,
                "gemm conv3x3: unsupported shape M=%d K=%d C=%d s=%d", M, K, C, conv_s);
    const uint64_t dims[4] = {static_cast<uint64_t>(C), static_cast<uint64_t>(conv_s),
                              static_cast<uint64_t>(conv_s), static_cast<uint64_t>(M / (conv_s * conv_s))};
    const uint64_t strides[3] = {static_cast<uint64_t>(C), static_cast<uint64_t>(conv_s) * C,
                                 static_cast<uint64_t>(conv_s) * conv_s * C};
    const uint32_t box[4] = {kGemmBK, static_cast<uint32_t>(conv_s), static_cast<uint32_t>(kGemmBM / conv_s), 1};
    if (int rc = make_tmap_f16_4d(&tmA, A, dims, strides, box)) return rc;
  } else {
    if (int rc = make_tmap_f16_2d(&tmA, A, M, K, lda, kGemmBM)) return rc;
  }
  if (int rc = make_tmap_f16_2d(&tmB, W, N, K, ldw, BN)) return rc;
  auto kern = gemm_tc_kernel<BN, STAGES, Epi>;
  static uint64_t attr_devs = 0;          // one bit per CUDA device: function attributes are per device   // per template instantiation
  if (first_use_on_device(&attr_devs)) {
    SRB_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SM::kTotal));
  }
  const int num_tiles = ((M + kGemmBM - 1) / kGemmBM) * ((N + BN - 1) / BN);
  const int grid = num_tiles < device_sm_count() ? num_tiles : device_sm_count();
  kern<<<grid, kGemmThreads, SM::kTotal, stream>>>(tmA, tmB, M, N, K, ep, conv_s);
  SRB_CUDA_OK(cudaGetLastError());
  note_launch(1);
  return 0;
}

}  // namespace srb
