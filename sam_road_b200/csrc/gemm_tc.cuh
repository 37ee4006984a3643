// sam_road_b200 :: wgmma GEMM  C[M,N] = A[M,K] * W[N,K]^T  (+ fused epilogue)
//
// Two kernel templates cover every dense contraction of the hot path (SURVEY.md §2.4 K2, K5, K9,
// K10, K11, K12, K16): fp16 operands (both K-major), fp32 accumulation in registers.  The streaming
// epilogues (EpiF16, EpiF32) run on gemm_pp_kernel (below, at the end of the file); the
// row-statistics epilogues (EpiLN, EpiDecFinal) on gemm_tc_kernel:
//
//   warpgroup 0     : TMA producer (one thread; cp.async.bulk.tensor, 128B-swizzled 128x64 / BNx64
//                     boxes), registers handed to the consumers with setmaxnreg
//   warpgroups 1, 2 : consumers.  Each issues wgmma m64 x BN x 16 for its 64 rows of the 128-row
//                     tile, then stages its fp32 accumulators in shared memory and runs the fused
//                     epilogue over them: warp w of consumer g reads rows 32*(2g + (w&1)) .. +31 (one
//                     row per lane) and columns half (w>>1) of the tile.
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

#include "common.cuh"
#include "ops.h"

namespace srb {

constexpr int kGemmBM = 128;
constexpr int kGemmBK = 64;
constexpr int kGemmThreads = 384;
constexpr int kGemmEpiWarps = 8;
constexpr int kGemmScratchFloats = 32 * 36;   // per epilogue warp: 32x32 fp32 block, rows padded to 36


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
// Streaming epilogues of the ping-pong kernel, straight from the wgmma accumulator fragments of one
// consumer warpgroup's 128x128 tile: d[h] is the m64n128 fragment of tile rows 64h .. 64h+63, so a
// thread (warp w of the warpgroup, lane l) holds, per n8 block j, the two adjacent columns
// 8j + 2(l&3) .. +1 of rows 16w + l/4 and 16w + l/4 + 8 of each half.  The four lanes of a quad
// cover 32 contiguous bytes of an fp32 row (one sector) and 16 of an fp16 row.  In EpiF32 every output
// element is read (residual) and written by the one thread that holds its accumulator, which keeps
// `out` aliasing `resid` legal.
// ------------------------------------------------------------------------------------------------
struct FragPos {
  int r0;       // first of this thread's four rows r0, r0 + 8, r0 + 64, r0 + 72
  int n_tile;   // first column of the tile
  int c0;       // this thread's column pair in n8 block j: c0 + 8j, c0 + 8j + 1
  __device__ __forceinline__ FragPos(int m_tile, int n_tile_, int w, int lane)
      : r0(m_tile + 16 * w + (lane >> 2)), n_tile(n_tile_), c0(n_tile_ + 2 * (lane & 3)) {}
  // row of fragment element pair q = 2h + hr (half h, lower/upper 8-row group hr)
  __device__ __forceinline__ int row(int q) const { return r0 + 64 * (q >> 1) + 8 * (q & 1); }
  // N is a multiple of 32, so a 16- or 32-column chunk is wholly inside or wholly outside the matrix
  __device__ __forceinline__ bool cols_in(int col, int N) const { return n_tile + col < N; }
};

// Phase trace (built only with -DSRB_GEMM_TRACE, by tools/gemm_trace.py): clock64 stamps per CTA and local tile i
// into buf[(cta * tiles + i) * kGemmTraceEvents + event], CTAs < ctas and tiles < tiles only.  The consumer that
// owns tile i stamps, from lane 0 of its first warp, TR_* events 0..5 and the epilogue's sub-phases (TR_EPI_LOADED:
// its first operands are in registers; TR_EPI_STAGED: the tile is packed into the staging buffer); the producer adds
// up the clocks it spent waiting on empty_bar for the tile's k-blocks (TR_EMPTY_WAIT).  With -DSRB_GEMM_TRACE_NOSTORE
// as well, the epilogues issue no global stores, which leaves the length of their loads and math (the values that
// are not stored still feed TR_EPI_STAGED, so the compiler keeps their computation).
enum { TR_ORDER_WAIT, TR_ORDER_DONE, TR_FIRST_FULL, TR_LAST_ISSUE, TR_DRAINED, TR_EPI_DONE, TR_EMPTY_WAIT,
       TR_EPI_LOADED, TR_EPI_STAGED, kGemmTraceEvents = 10 };
#ifdef SRB_GEMM_TRACE
struct GemmTrace {
  long long* buf;
  int ctas, tiles;
};
static __device__ GemmTrace g_gemm_trace;
__device__ __forceinline__ long long* gemm_trace_slot(int i) {
  const GemmTrace t = g_gemm_trace;
  if (t.buf == nullptr || static_cast<int>(blockIdx.x) >= t.ctas || i >= t.tiles) return nullptr;
  return t.buf + (static_cast<size_t>(blockIdx.x) * t.tiles + i) * kGemmTraceEvents;
}
// Stamps `event` once `dep` (a value the phase produced) is in a register: the store of dep has to wait for it,
// and the clock read is not moved above that store.
__device__ __forceinline__ void gemm_trace_stamp(long long* tr, int event, float dep) {
  if (tr == nullptr) return;
  tr[kGemmTraceEvents - 1] = __float_as_int(dep);
  long long t;
  asm volatile("mov.u64 %0, %%clock64;" : "=l"(t)::"memory");
  tr[event] = t;
}
#define GEMM_TRACE(...) __VA_ARGS__
#else
#define GEMM_TRACE(...)
#endif
#if defined(SRB_GEMM_TRACE) && defined(SRB_GEMM_TRACE_NOSTORE)
#define GEMM_STORE(...)
#else
#define GEMM_STORE(...) __VA_ARGS__
#endif

// Each epilogue gets its warp's part of the consumer's staging buffer (Epi::kStageBytes per consumer, a quarter
// per warp; EpiF16 has none) and two mbarriers of the warp for loads into it.  Epi::prefetch runs on lane 0 of
// each warp once the tile's first k-block is issued, Epi::run after the tile's last MMAs, Epi::drain at the end.
// Operands read from global memory are loaded before the stores that the compiler must assume alias them: a load
// issued after those stores costs one L2 round trip each, and at K = 768 the epilogue then outlasts the other
// consumer's mainloop.

// Epilogue 1: out16[m,n] = act(acc + bias[n])                       (qkv, MLP lin1, TopoNet lin)
// Per 32-column chunk and row, the quad's four lanes transpose their packed half2 pairs with two shuffles so that
// lane t holds all eight columns of n8 block 4c + t: one 16-byte store per lane, 64 contiguous bytes per quad.
// Stored straight from the fragment as 4-byte half2s (half-sector writes), the same output nearly doubled the
// other consumer's TMA-fed mainloop at K = 768 (tools/gemm_trace.py, DESIGN.md).  Needs `out` 16-byte aligned.
// Bias and activation are template arguments of the tile loop: tested per column pair, each pair's add, activation,
// pack and shuffles ran as a block of their own, back to back, and the epilogue outlasted the other consumer's
// mainloop; as one branch-free block the compiler interleaves the independent pairs.
struct EpiF16 {
  static constexpr int kStageBytes = 0;
  struct Params {
    __half* out;          // [M, ldo]
    const float* bias;    // [N] or null
    int ldo;
    int act;
  };
  static __device__ __forceinline__ void prefetch(const Params&, int, int, int, int, uint8_t*, uint64_t*) {}
  static __device__ __forceinline__ void run(const Params& p, int M, int N, const FragPos& f, float (&d)[2][64],
                                             uint8_t* /*stage*/, uint64_t* /*bar*/, uint32_t (&)[2], long long* tr) {
    float2 b[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      b[j] = make_float2(0.f, 0.f);
      if (p.bias && f.cols_in(32 * (j >> 2), N)) b[j] = __ldg(reinterpret_cast<const float2*>(p.bias + f.c0 + 8 * j));
    }
    GEMM_TRACE(float dep = 0.f; for (int j = 0; j < 16; ++j) dep += b[j].x + b[j].y;
               gemm_trace_stamp(tr, TR_EPI_LOADED, dep));
    if (p.bias) {
      if (p.act == ACT_GELU) tile<true, ACT_GELU>(p, M, N, f, d, b, tr);
      else if (p.act == ACT_RELU) tile<true, ACT_RELU>(p, M, N, f, d, b, tr);
      else tile<true, ACT_NONE>(p, M, N, f, d, b, tr);
    } else {
      if (p.act == ACT_GELU) tile<false, ACT_GELU>(p, M, N, f, d, b, tr);
      else if (p.act == ACT_RELU) tile<false, ACT_RELU>(p, M, N, f, d, b, tr);
      else tile<false, ACT_NONE>(p, M, N, f, d, b, tr);
    }
  }
  template <bool kBias, int kAct>
  static __device__ __forceinline__ void tile(const Params& p, int M, int N, const FragPos& f, float (&d)[2][64],
                                              const float2 (&b)[16], long long* tr) {
    GEMM_TRACE(uint32_t sink = 0);             // every value the tile computes feeds the last stamp
    const int t = threadIdx.x & 3;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      if (!f.cols_in(32 * c, N)) continue;
      const int n = f.n_tile + 8 * (4 * c + t);
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        uint32_t x[4];                         // x[u]: this lane's column pair of n8 block 4c + u
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int j = 4 * c + u;
          float2 v = make_float2(d[q >> 1][4 * j + 2 * (q & 1)], d[q >> 1][4 * j + 2 * (q & 1) + 1]);
          if (kBias) { v.x += b[j].x; v.y += b[j].y; }
          if (kAct == ACT_GELU) v = gelu_erf_fast2(v);
          else if (kAct == ACT_RELU) v = make_float2(fmaxf(v.x, 0.0f), fmaxf(v.y, 0.0f));
          x[u] = pack_half2(v.x, v.y);
        }
        // 4x4 transpose across the quad: afterwards x[s] is lane s's column pair of n8 block 4c + t
#pragma unroll
        for (int k = 0; k < 4; k += 2) {
          const uint32_t r = __shfl_xor_sync(0xffffffffu, (t & 1) ? x[k] : x[k + 1], 1);
          if (t & 1) x[k] = r; else x[k + 1] = r;
        }
#pragma unroll
        for (int k = 0; k < 2; ++k) {
          const uint32_t r = __shfl_xor_sync(0xffffffffu, (t & 2) ? x[k] : x[k + 2], 2);
          if (t & 2) x[k] = r; else x[k + 2] = r;
        }
        const int m = f.row(q);
        GEMM_STORE(if (m < M) *reinterpret_cast<uint4*>(p.out + static_cast<size_t>(m) * p.ldo + n) = make_uint4(x[0], x[1], x[2], x[3]));
        GEMM_TRACE(sink ^= x[0] ^ x[1] ^ x[2] ^ x[3];
                   if (c == 3 && q == 3) gemm_trace_stamp(tr, TR_EPI_STAGED, __uint_as_float(sink)));
      }
    }
  }
  static __device__ __forceinline__ void drain(int /*lane*/) {}
};

// Epilogue 2: out32[m,n] = acc + resid[m,n] + bias[n] + pos[m % pos_rows, n]
//             (patch-embed + pos_embed, attention proj + shortcut, MLP lin2 + shortcut; plain f32)
// fp32 in/out makes this epilogue HBM-bound for short K (attention proj).  Each warp works in slabs of 32
// columns of its 32 rows (16 of each 64-row half), through its 8 KB of the staging buffer: two 4 KB slab buffers
// used in turn, each two 16-row x 32-column boxes (half h at 2 KB * h), 128B-swizzled (16-byte chunk k of row r
// at k ^ (r & 7)).  The residual of a slab arrives in its buffer by TMA: slabs 0 and 1 are requested while the
// tile's mainloop runs (prefetch), slab s + 2 as soon as the stores of slab s have read the buffer.  Each thread
// reads the residual of its accumulator's element from the buffer and writes the sum back to the same place;
// lane 0 then stores the slab with TMA through the output map (N x M, row pitch ldo), which clips the M tail and
// the columns >= N.  A slab's residual has been read before the slab is stored, and the tiles of a launch do not
// overlap, so `out` may alias `resid`.  Bias and pos-embed (L1- / L2-resident) are loaded per 16-column chunk.
struct EpiF32 {
  static constexpr int kStageBytes = 4 * 8192;
  struct Params {
    CUtensorMap tm_out;   // [M, N] fp32, row pitch ldo; box 32 columns x 16 rows, 128B swizzle
    CUtensorMap tm_resid; // the same for resid, when there is one
    const float* bias;    // [N] or null
    const float* resid;   // [M, ldo] or null (may alias the output)
    const float* pos;     // [pos_rows, N] or null
    int pos_rows;
    int n_total;
  };
  // residual of slab s of the warp's rows (row0 .. +15 and row0 + 64 .. +15) into slab buffer s & 1, completing on
  // bar[s & 1]; a box wholly below M is not loaded (its rows are not stored), and with neither box the arrive
  // alone completes the barrier's phase.  One thread.
  static __device__ __forceinline__ void load_slab(const Params& p, int M, int N, int n_tile, int row0, int s,
                                                   uint8_t* stage, uint64_t* bar) {
    if (n_tile + 32 * s >= N) return;
    const int boxes = (row0 < M) + (row0 + 64 < M);
    mbar_arrive_expect_tx(&bar[s & 1], 2048 * boxes);
    for (int h = 0; h < boxes; ++h)
      tma_load_2d(stage + 4096 * (s & 1) + 2048 * h, &p.tm_resid, &bar[s & 1], n_tile + 32 * s, row0 + 64 * h);
  }
  // Called by lane 0 of each warp once the tile's first k-block is issued: the buffers are free when the stores of
  // the warp's previous tile have read them.
  static __device__ __forceinline__ void prefetch(const Params& p, int M, int N, int n_tile, int row0, uint8_t* stage,
                                                  uint64_t* bar) {
    if (p.resid == nullptr) return;
    bulk_wait_group_read<0>();
    load_slab(p, M, N, n_tile, row0, 0, stage, bar);
    load_slab(p, M, N, n_tile, row0, 1, stage, bar);
  }
  static __device__ __forceinline__ void run(const Params& p, int M, int N, const FragPos& f, float (&d)[2][64],
                                             uint8_t* stage, uint64_t* bar, uint32_t (&bar_phase)[2], long long* tr) {
    const int lane = threadIdx.x & 31;
    const int row0 = f.r0 - (lane >> 2);         // the first of the warp's 16 rows in half 0
    int pos_row[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) pos_row[q] = p.pos ? f.row(q) % p.pos_rows : 0;
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      if (!f.cols_in(16 * c, N)) continue;
      float* slab = reinterpret_cast<float*>(stage + 4096 * ((c >> 1) & 1));
      if ((c & 1) == 0) {
        if (p.resid) {                           // the slab's residual has arrived
          mbar_wait(&bar[(c >> 1) & 1], bar_phase[(c >> 1) & 1]);
          bar_phase[(c >> 1) & 1] ^= 1u;
        } else {                                 // the stores of the slab before last (at c = 0: of the previous
          if (lane == 0) {                       // tile) have read the buffer
            if (c == 0) bulk_wait_group_read<0>();
            else bulk_wait_group_read<1>();
          }
          __syncwarp();
        }
        GEMM_TRACE(if (c == 0) gemm_trace_stamp(tr, TR_EPI_LOADED, slab[0]));
      }
      float2 b[2], e[8];
#pragma unroll
      for (int jj = 0; jj < 2; ++jj) {
        const int n = f.c0 + 8 * (2 * c + jj);
        b[jj] = p.bias ? __ldg(reinterpret_cast<const float2*>(p.bias + n)) : make_float2(0.f, 0.f);
#pragma unroll
        for (int q = 0; q < 4; ++q)
          e[4 * jj + q] = p.pos && f.row(q) < M
                              ? __ldg(reinterpret_cast<const float2*>(p.pos + static_cast<size_t>(pos_row[q]) * p.n_total + n))
                              : make_float2(0.f, 0.f);
      }
#pragma unroll
      for (int jj = 0; jj < 2; ++jj) {
        const int j = 2 * c + jj;
        // 16-byte chunk of this lane's column pair inside the slab row, and the pair's half of it
        const int k = 4 * (c & 1) + 2 * jj + ((lane & 3) >> 1);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int row = (lane >> 2) + 8 * (q & 1);
          float2* at = reinterpret_cast<float2*>(slab + 512 * (q >> 1) + 32 * row + 4 * (k ^ (row & 7)) + 2 * (lane & 1));
          const float2 r = p.resid ? *at : make_float2(0.f, 0.f);
          float2 x = make_float2(d[q >> 1][4 * j + 2 * (q & 1)] + r.x, d[q >> 1][4 * j + 2 * (q & 1) + 1] + r.y);
          if (p.bias) { x.x += b[jj].x; x.y += b[jj].y; }
          if (p.pos) { x.x += e[4 * jj + q].x; x.y += e[4 * jj + q].y; }
          *at = x;
        }
      }
      if (c & 1) {                               // the slab is complete (N is a multiple of 32)
        fence_proxy_async_smem();                // the slab's writes are visible to the TMA unit
        __syncwarp();
        GEMM_TRACE(if (c == 7) gemm_trace_stamp(tr, TR_EPI_STAGED, 0.f));
        if (lane == 0) {
#pragma unroll
          for (int h = 0; h < 2; ++h)
            if (row0 + 64 * h < M)
              GEMM_STORE(tma_store_2d(&p.tm_out, slab + 512 * h, f.n_tile + 32 * (c >> 1), row0 + 64 * h));
          bulk_commit_group();
          if (c < 4 && p.resid) {                // slab c/2 + 2 reuses this buffer once the stores have read it
            bulk_wait_group_read<0>();
            load_slab(p, M, N, f.n_tile, row0, (c >> 1) + 2, stage, bar);
          }
        }
      }
    }
  }
  static __device__ __forceinline__ void drain(int lane) {
    if (lane == 0) bulk_wait_group<0>();
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
          else if (p.act == ACT_RELU) y = make_float2(fmaxf(y.x, 0.0f), fmaxf(y.y, 0.0f));
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
  static __device__ __forceinline__ void drain(int /*lane*/) {}
};

// ------------------------------------------------------------------------------------------------
// Epilogue 4: last two stages of the naive map decoder (model.py:292-294,490-491).
// The GEMM is ConvT(64->32,k2,s2) with columns ordered (sub3, co): a tile row is one 128x128-res
// ... one stage-3 input pixel; each 32-column chunk is one 2x upsampled sub-pixel with 32 channels.
// Per chunk: h = GELU(acc + b3) ; ConvT(32->2,k2,s2): out[co, di, dj] = sum_ci h[ci] W4[ci,co,di,dj]
// + b4[co]; writes logits and sigmoid scores straight into NHWC [B, P, P, 2].
// Row index r of the GEMM encodes the pixel hierarchy: r = ((b*s*s + i*s + j)*4 + d1)*4 + d2,
// d = di*2 + dj.
//
// kPerToken = false (even s): a warp's two tokens (i, j), (i, j+1) are horizontally adjacent and leave
// in one 32-pixel-wide box.  kPerToken = true (odd s): the warp's first token has an even index, so a
// pair can straddle a row end ((i, s-1) with (i+1, 0)) or an image boundary; each token is staged
// separately and stored with a 16-pixel-wide box at its own (b, i, j).
// ------------------------------------------------------------------------------------------------
template <bool kPerToken>
struct EpiDecFinal {
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
    Epi::drain(lane);
  }
}

// ------------------------------------------------------------------------------------------------
// host launcher
// ------------------------------------------------------------------------------------------------
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
  SRB_TRY(allow_dynamic_smem(kern, SM::kTotal));
  const int num_tiles = ((M + kGemmBM - 1) / kGemmBM) * ((N + BN - 1) / BN);
  const int grid = num_tiles < device_sm_count() ? num_tiles : device_sm_count();
  SRB_LAUNCH(kern, grid, kGemmThreads, SM::kTotal, stream, tmA, tmB, M, N, K, ep, conv_s);
  return 0;
}

// ------------------------------------------------------------------------------------------------
// Ping-pong kernel for the streaming epilogues (EpiF16, EpiF32).  Same block as gemm_tc_kernel
// (warpgroup 0 = TMA producer, warpgroups 1 and 2 = consumers), but each consumer owns whole 128x128
// tiles: two wgmma m64n128k16 per k16 step, 2 x 64 fp32 accumulators per thread.  The CTA's tiles
// t0, t1, t2, ... alternate between the consumers (t0, t2, ... and t1, t3, ...), and an ordering
// mbarrier pair starts a consumer's mainloop when the other's has issued its last MMAs, so one
// warpgroup is on the tensor cores while the other runs its epilogue (EpiF32 through its own staging buffer).  The ring
// holds operands only; the producer never waits for an epilogue.
//
// Ring bookkeeping.  The producer fills ring positions p = 0, 1, 2, ... in CTA tile order: local
// tile i (the CTA's i-th tile) owns positions i*num_k .. i*num_k + num_k - 1, slot p % STAGES,
// fill number n = p / STAGES of that slot.  The consumer of tile i waits on full_bar[slot] with
// parity n & 1 and, once its MMAs have read the slot, releases it with one arrive per warp
// (empty_bar count 4); the other consumer never touches the slot for that fill.  Invariant: when a
// consumer waits on position p, every position before p has already been seen full by its own
// consumer (its own earlier k-blocks, and through the ordering barrier every k-block of the tiles
// before), so fill n - 1 of the slot is complete and fill n + 1 cannot start before this consumer
// releases fill n: the slot's full barrier is exactly one phase from the waited parity, never two.
// ------------------------------------------------------------------------------------------------
// Shared memory: the operand ring, then each consumer's epilogue staging buffer (kEpiBytes, 1024-aligned for the
// 128B swizzle), then the barriers.
template <int STAGES, int kEpiBytes>
struct GemmPPSmem {
  static constexpr int kABytes = kGemmBM * kGemmBK * 2;
  static constexpr int kBBytes = 128 * kGemmBK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kEpiOffset = STAGES * kStageBytes;
  static constexpr int kBarOffset = kEpiOffset + 2 * kEpiBytes;
  static constexpr int kTotal = kBarOffset + 256 + 1024;
  static_assert(kTotal <= 227 * 1024, "gemm_pp_kernel: shared memory over the 227 KB an H100 block may use");
  static_assert((2 * STAGES + 2 + 16) * 8 <= 256, "gemm_pp_kernel: barriers (full, empty, order, staging) over 256 B");
};

template <int STAGES, class Epi>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_pp_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
               int M, int N, int K, const __grid_constant__ typename Epi::Params ep) {
  using SM = GemmPPSmem<STAGES, Epi::kStageBytes>;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + ((1024u - (raw_addr & 1023u)) & 1023u);

  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + SM::kBarOffset);
  uint64_t* empty_bar = full_bar + STAGES;
  uint64_t* order_bar = empty_bar + STAGES;       // [g]: the other consumer has issued its mainloop
  uint64_t* stage_bar = order_bar + 2;            // [4g + w][2]: loads into warp w's staging buffers (EpiF32)

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = warp >> 2;

  const int num_n = (N + 127) / 128;
  const int num_tiles = ((M + kGemmBM - 1) / kGemmBM) * num_n;
  const int num_k = (K + kGemmBK - 1) / kGemmBK;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 4);
    }
    mbar_init(&order_bar[0], 4);
    mbar_init(&order_bar[1], 4);
    if (Epi::kStageBytes > 0)
      for (int i = 0; i < 16; ++i) mbar_init(&stage_bar[i], 1);
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    // ===================== TMA producer =====================
    setmaxnreg_dec<40>();
    if (warp == 0 && lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      GEMM_TRACE(int ti = 0);
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int m_blk = tile / num_n, n_blk = tile % num_n;
        GEMM_TRACE(long long stall = 0);
        for (int kb = 0; kb < num_k; ++kb) {
          GEMM_TRACE(const long long t0 = clock64());
          mbar_wait(&empty_bar[stage], phase ^ 1u);
          GEMM_TRACE(stall += clock64() - t0);
          uint8_t* sa = smem + stage * SM::kStageBytes;
          mbar_arrive_expect_tx(&full_bar[stage], SM::kStageBytes);
          tma_load_2d(sa, &tmA, &full_bar[stage], kb * kGemmBK, m_blk * kGemmBM);
          tma_load_2d(sa + SM::kABytes, &tmB, &full_bar[stage], kb * kGemmBK, n_blk * 128);
          if (++stage == STAGES) { stage = 0; phase ^= 1u; }
        }
        GEMM_TRACE(if (long long* t = gemm_trace_slot(ti++)) t[TR_EMPTY_WAIT] = stall);
      }
    }
  } else {
    // ===================== consumers: MMA + epilogue, alternating tiles =====================
    setmaxnreg_inc<232>();
    const int g = wg - 1;
    const int w = warp & 3;
    uint8_t* staging = smem + SM::kEpiOffset + g * Epi::kStageBytes + w * (Epi::kStageBytes / 4);
    uint64_t* bar = stage_bar + 2 * (4 * g + w);
    uint32_t order_phase = 0, bar_phase[2] = {0u, 0u};
    int i = g;                                 // local tile index
    for (int tile = blockIdx.x + g * gridDim.x; tile < num_tiles; tile += 2 * gridDim.x, i += 2) {
      const int m_blk = tile / num_n, n_blk = tile % num_n;
      long long* tr = nullptr;
      GEMM_TRACE(if (w == 0 && lane == 0) tr = gemm_trace_slot(i);
                 if (tr) tr[TR_ORDER_WAIT] = clock64());
      if (i > 0) {                             // the other consumer has issued tile i - 1
        mbar_wait(&order_bar[g], order_phase);
        order_phase ^= 1u;
      }
      GEMM_TRACE(if (tr) tr[TR_ORDER_DONE] = clock64());
      const int pos = i * num_k;
      int stage = pos % STAGES;
      uint32_t phase = static_cast<uint32_t>(pos / STAGES) & 1u;
      float d[2][64];
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int r = 0; r < 64; ++r) d[h][r] = 0.f;
      int prev = -1;
      for (int kb = 0; kb < num_k; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        GEMM_TRACE(if (tr && kb == 0) tr[TR_FIRST_FULL] = clock64());
        const uint32_t a_addr = smem_u32(smem + stage * SM::kStageBytes);
        const uint64_t adesc0 = wgmma_desc_k128(a_addr);
        const uint64_t adesc1 = wgmma_desc_k128(a_addr + 64 * kGemmBK * 2);
        const uint64_t bdesc = wgmma_desc_k128(a_addr + SM::kABytes);
        wgmma_fence_operand(d[0]);
        wgmma_fence_operand(d[1]);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kGemmBK / 16; ++k) {
          const uint32_t acc = (kb | k) != 0 ? 1u : 0u;
          wgmma_m64n128k16(d[0], adesc0 + static_cast<uint64_t>(2 * k), bdesc + static_cast<uint64_t>(2 * k), acc);
          wgmma_m64n128k16(d[1], adesc1 + static_cast<uint64_t>(2 * k), bdesc + static_cast<uint64_t>(2 * k), acc);
        }
        wgmma_commit();
        GEMM_TRACE(if (tr && kb == num_k - 1) tr[TR_LAST_ISSUE] = clock64());
        if (kb == 0 && lane == 0) Epi::prefetch(ep, M, N, n_blk * 128, m_blk * kGemmBM + 16 * w, staging, bar);
        wgmma_wait<1>();                       // the previous k-block's MMAs have read their stage
        wgmma_fence_operand(d[0]);
        wgmma_fence_operand(d[1]);
        if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
        prev = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1u; }
      }
      if (lane == 0) mbar_arrive(&order_bar[g ^ 1]);   // the other consumer may start its mainloop
      wgmma_wait<0>();
      wgmma_fence_operand(d[0]);
      wgmma_fence_operand(d[1]);
      GEMM_TRACE(if (tr) tr[TR_DRAINED] = clock64());
      if (lane == 0) mbar_arrive(&empty_bar[prev]);
      Epi::run(ep, M, N, FragPos(m_blk * kGemmBM, n_blk * 128, w, lane), d, staging, bar, bar_phase, tr);
      GEMM_TRACE(if (tr) tr[TR_EPI_DONE] = clock64());
    }
    Epi::drain(lane);
  }
}

template <class Epi>
int launch_gemm_pp(const __half* A, int lda, const __half* W, int ldw, int M, int N, int K,
                   const typename Epi::Params& ep, cudaStream_t stream) {
  constexpr int kStages = 5;
  using SM = GemmPPSmem<kStages, Epi::kStageBytes>;
  SRB_REQUIRE(M > 0 && N > 0 && K > 0, "gemm: empty problem M=%d N=%d K=%d", M, N, K);
  SRB_REQUIRE(N % 32 == 0, "gemm: N=%d must be a multiple of 32", N);
  SRB_REQUIRE(K % 8 == 0 && lda % 8 == 0 && ldw % 8 == 0,
              "gemm: K/lda/ldw (%d/%d/%d) must be multiples of 8", K, lda, ldw);
  CUtensorMap tmA, tmB;
  if (int rc = make_tmap_f16_2d(&tmA, A, M, K, lda, kGemmBM)) return rc;
  if (int rc = make_tmap_f16_2d(&tmB, W, N, K, ldw, 128)) return rc;
  auto kern = gemm_pp_kernel<kStages, Epi>;
  SRB_TRY(allow_dynamic_smem(kern, SM::kTotal));
  const int num_tiles = ((M + kGemmBM - 1) / kGemmBM) * ((N + 127) / 128);
  const int grid = num_tiles < device_sm_count() ? num_tiles : device_sm_count();
  SRB_LAUNCH(kern, grid, kGemmThreads, SM::kTotal, stream, tmA, tmB, M, N, K, ep);
  return 0;
}

}  // namespace srb
