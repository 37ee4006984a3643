// sam_road_b200 :: fused TopoNet transformer (model.py:74-86,135-146): all three post-norm encoder
// layers + output_proj for a tile of 128 pair tokens (8 samples x 16 pairs) in ONE persistent kernel.
//
// Per layer (torch TransformerEncoderLayer, d=128, 4 heads, ff=128, relu, LN eps 1e-5, eval mode):
//   qkv = x W_in^T + b_in -> per-sample 16x16 masked attention per head -> x = LN1(x + att W_o^T + b_o)
//   -> x = LN2(x + relu(x W_1^T + b_1) W_2^T + b_2)
// Everything between the GEMMs stays on chip:
//   registers  the fp32 residual stream x (a token thread keeps its 32 columns of the row)
//   smem  A buffer 32 KB  current fp16 GEMM A operand (x -> attention output -> x' -> hidden -> x'')
//         KV buffer 66 KB k and v of the tile as fp16 rows; after the attention, the fp32 [128][132]
//                         staging area of the out_proj / linear2 results
//         weight ring 3 x 32 KB  the 18 [128x128] weight chunks streamed by TMA in consumption order
// Warps 0..15 = 512 token threads in four warpgroups, warp 16 = TMA producer.  Warpgroup g owns
// columns 32g..32g+31 = head g: it computes them for every GEMM on wgmma (two m64 x n32 x k16 per
// k-step, A and the weight chunk read from 128B-swizzled smem), and as token threads its warp q holds
// rows 32q..32q+31 (one per lane) of the same columns.  So the accumulators reach the token threads
// through a warpgroup-local smem exchange, and only the A operand, which every warpgroup reads whole,
// needs the 512-thread barrier.  LayerNorm statistics and the output dot product are combined across
// the four warpgroups through a small smem exchange per row quarter, always summed in part order.
// The 16 x 16 x 32 attention of a (sample, head) runs on warp-level mma.sync: a warp owns two
// samples of its head; q (bias, 1/sqrt(32), fp16) is staged in the warp's own rows of the A buffer,
// k / v fragments come from the k|v rows by ldmatrix / ldmatrix.trans, softmax in fp32 on the S
// fragments, P (fp16) feeds the PV mma from registers.  Key-padding semantics (SURVEY.md §8a P4):
// masked keys are excluded from the softmax; masked slots report output_proj.bias.
#pragma once

#include "common.cuh"
#include "ops.h"

namespace srb {

constexpr int kTtcThreads = 544;          // 16 token warps + 1 producer warp
constexpr int kTtcTokenThreads = 512;
constexpr int kTtcWStages = 3;
constexpr int kTtcOffA = 0;                       // 2 k-blocks x 16 KB
constexpr int kTtcOffKV = 32768;                  // 128 rows x 528 B (k|v fp16, padded: ldmatrix rows hit 32 banks)
constexpr int kTtcKVStride = 528;
constexpr int kTtcStgPitch = 132;                 // fp32 staging rows (overlays the KV buffer)
static_assert(128 * kTtcStgPitch * 4 <= 68608, "staging must fit the KV buffer");
constexpr int kTtcOffW = kTtcOffKV + 68608;       // 3 x 32 KB
constexpr int kTtcOffBar = kTtcOffW + kTtcWStages * 32768;
constexpr int kTtcOffXch = kTtcOffBar + 256;      // 3 slots x 4 parts x 128 floats: partial sums of the parts
constexpr int kTtcSmemBytes = kTtcOffXch + 3 * 2048 + 1024;
constexpr int kTtcChunksPerLayer = 6;             // Wq, Wk, Wv, Wo, W1, W2 as packed
// consumption order of a layer's chunks: k and v first, q last (q is written into the A buffer,
// which may only happen once every warpgroup has finished the in_proj GEMMs)
__host__ __device__ constexpr int ttc_chunk(int i) { return i == 0 ? 1 : (i == 1 ? 2 : (i == 2 ? 0 : i)); }

struct TtcParams {
  TopoLayerParams layer[3];
  TopoPairInputs in;      // the kernel forms the pair features itself
  const uint8_t* valid;   // [tokens] fixed validity (all-invalid rows already flipped), or null
  const float* out_w;     // [128]
  const float* out_b;     // [1]
  float* logits;          // [tokens] or null
  float* scores;          // [tokens] or null
  int tokens;
  int num_tiles;
};

// ------------------------------------------------------------------------------------------------
// Pair-token gather, shared with topo_pair_kernel (toponet.cu)
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float load_coord(const void* p, int dtype, size_t idx) {
  if (dtype == 0) return static_cast<const float*>(p)[idx];
  if (dtype == 1) return static_cast<float>(static_cast<const long long*>(p)[idx]);
  return static_cast<float>(static_cast<const int*>(p)[idx]);
}
__device__ __forceinline__ long long load_index(const void* p, int dtype, size_t idx) {
  if (dtype == 1) return static_cast<const long long*>(p)[idx];
  return static_cast<long long>(static_cast<const int*>(p)[idx]);
}

// Rows of a pair token's source and target point in pst / points (b * N + index) and its offset
// pt[tgt] - pt[src] (zero for TOPONET_VERSION 'no_offset').
struct PairToken {
  size_t ps, pt;
  float ox, oy;
};
__device__ __forceinline__ PairToken resolve_pair(const TopoPairInputs& in, size_t tok) {
  const size_t b = tok / in.tokens_per_b;
  // indices are clamped into [0, N): an out-of-range pair (an IndexError in the reference) must not
  // become an out-of-bounds read here
  const long long nm1 = static_cast<long long>(in.N) - 1;
  PairToken r;
  r.ps = b * in.N + min(max(load_index(in.pairs, in.pairs_dtype, tok * 2 + 0), 0LL), nm1);
  r.pt = b * in.N + min(max(load_index(in.pairs, in.pairs_dtype, tok * 2 + 1), 0LL), nm1);
  r.ox = r.oy = 0.f;
  if (!in.zero_offset) {
    r.ox = load_coord(in.points, in.pts_dtype, r.pt * 2 + 0) - load_coord(in.points, in.pts_dtype, r.ps * 2 + 0);
    r.oy = load_coord(in.points, in.pts_dtype, r.pt * 2 + 1) - load_coord(in.points, in.pts_dtype, r.ps * 2 + 1);
  }
  return r;
}

// warp-level MMA for the 16 x 16 attention of one sample and head (far too small for a UMMA tile)
__device__ __forceinline__ void ttc_ldmatrix_x4(uint32_t (&r)[4], uint32_t saddr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(saddr) : "memory");
}
__device__ __forceinline__ void ttc_ldmatrix_x4_trans(uint32_t (&r)[4], uint32_t saddr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(saddr) : "memory");
}
// d (16x8, fp32) += a (16x16, fp16, row) * b (16x8, fp16, col)
__device__ __forceinline__ void ttc_mma_16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
               "{%0, %1, %2, %3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}


// named barriers: 1 = all 512 token threads, 2..5 = row quarter q (its warps in the four warpgroups),
// 6..9 = warpgroup g
__device__ __forceinline__ void ttc_bar_all() { asm volatile("bar.sync 1, 512;" ::: "memory"); }
__device__ __forceinline__ void named_bar_sync_quarter(int quarter) {
  asm volatile("bar.sync %0, 128;" ::"r"(quarter + 2) : "memory");
}
__device__ __forceinline__ void ttc_bar_group(int g) {
  asm volatile("bar.sync %0, 128;" ::"r"(g + 6) : "memory");
}

// D[64 x 32] (+)= A[64 x 16] * B[32 x 16]^T, both operands K-major in shared memory
__device__ __forceinline__ void wgmma_m64n32k16(float (&d)[16], uint64_t desc_a, uint64_t desc_b,
                                             uint32_t accumulate) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "setp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 "
      "{"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15"
      "}, %16, %17, p, 1, 1, 0, 0;\n\t"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(desc_a), "l"(desc_b), "r"(accumulate));
}


__global__ void __launch_bounds__(kTtcThreads, 1)
toponet_tc_kernel(const __grid_constant__ CUtensorMap tmW, TtcParams p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + ((1024u - (raw_addr & 1023u)) & 1023u);
  uint8_t* sA = smem + kTtcOffA;
  uint8_t* sKV = smem + kTtcOffKV;
  uint8_t* sW = smem + kTtcOffW;
  float* stg = reinterpret_cast<float*>(sKV);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kTtcOffBar);
  uint64_t* w_full = bars;          // [3]
  uint64_t* w_empty = bars + 3;     // [3]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (warp == 16 && lane == 0) {
    tma_prefetch_desc(&tmW);
    for (int i = 0; i < kTtcWStages; ++i) { mbar_init(&w_full[i], 1); mbar_init(&w_empty[i], 4); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 16) {
    // =========================== TMA producer ===========================
    if (lane == 0) {
      int wc = 0;
      for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
        for (int i = 0; i < 3 * kTtcChunksPerLayer; ++i, ++wc) {
          const int ch = (i / kTtcChunksPerLayer) * kTtcChunksPerLayer + ttc_chunk(i % kTtcChunksPerLayer);
          const int st = wc % kTtcWStages;
          mbar_wait(&w_empty[st], ((wc / kTtcWStages) & 1) ^ 1u);
          mbar_arrive_expect_tx(&w_full[st], 32768);
          tma_load_2d(sW + st * 32768, &tmW, &w_full[st], 0, ch * 128);
          tma_load_2d(sW + st * 32768 + 16384, &tmW, &w_full[st], 64, ch * 128);
        }
      }
    }
    return;
  }

  // =========================== token threads / MMA warpgroups ===========================
  const int quarter = warp & 3;
  const int part = warp >> 2;                       // warpgroup; columns 32*part .. +31, head `part`
  const int row = quarter * 32 + lane;
  const int sw = row & 7;
  uint8_t* myA = sA + row * 128;
  float* xch = reinterpret_cast<float*>(smem + kTtcOffXch);   // [3][4 parts][128 rows]
  // accumulator fragment coordinates (wgmma m64nN): rows fr0 (+8) (+64 for the second product),
  // columns 8j + fc (+1) of this warpgroup's 32
  const int fr0 = quarter * 16 + (lane >> 2), fc = 2 * (lane & 3);
  int ti = 0, wc = 0;

  auto write_a_chunk = [&](int c, const float (&v)[32]) {   // 32 fp32 -> fp16 into the swizzled A buffer
    uint8_t* dst = myA + (c >> 1) * 16384;
#pragma unroll
    for (int q4 = 0; q4 < 4; ++q4) {
      uint4 u;
      u.x = pack_half2(v[q4 * 8 + 0], v[q4 * 8 + 1]);
      u.y = pack_half2(v[q4 * 8 + 2], v[q4 * 8 + 3]);
      u.z = pack_half2(v[q4 * 8 + 4], v[q4 * 8 + 5]);
      u.w = pack_half2(v[q4 * 8 + 6], v[q4 * 8 + 7]);
      *reinterpret_cast<uint4*>(dst + ((((c & 1) * 4 + q4) ^ sw) << 4)) = u;
    }
  };
  // fp16 pair (columns 32h + 8j + fc, +1) of tile row r into the swizzled A buffer
  auto a_pair = [&](int r, int h, int j) -> uint32_t* {
    return reinterpret_cast<uint32_t*>(sA + (h >> 1) * 16384 + r * 128 + ((((h & 1) * 4 + j) ^ (r & 7)) << 4) + fc * 2);
  };
  // the four parts' partials of the same row, summed in part order (slot: 0 sum, 1 var, 2 dot): every
  // thread of a row gets the same value
  auto combine = [&](int slot, float mine) -> float {
    float* x = xch + slot * 512 + row;
    x[part * 128] = mine;
    named_bar_sync_quarter(quarter);
    return ((x[0] + x[128]) + x[256]) + x[384];
  };
  auto ldg32 = [&](const float* src, float (&v)[32]) {     // 32 consecutive floats (128 B aligned)
    const float4* s4 = reinterpret_cast<const float4*>(src);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float4 t = __ldg(s4 + i);
      v[4 * i + 0] = t.x; v[4 * i + 1] = t.y; v[4 * i + 2] = t.z; v[4 * i + 3] = t.w;
    }
  };
  // this warpgroup's 32 output columns of the next weight chunk for all 128 rows: acc[h] = rows 64h..
  auto gemm = [&](float (&acc)[2][16]) {
    const int st = wc % kTtcWStages;
    mbar_wait(&w_full[st], (wc / kTtcWStages) & 1);
    const uint32_t abase = smem_u32(sA), wbase = smem_u32(sW + st * 32768) + part * 32 * 128;
    wgmma_fence_operand(acc[0]);
    wgmma_fence_operand(acc[1]);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const uint64_t bdesc = wgmma_desc_k128(wbase + (k >> 2) * 16384) + 2 * (k & 3);
#pragma unroll
      for (int h = 0; h < 2; ++h)
        wgmma_m64n32k16(acc[h], wgmma_desc_k128(abase + (k >> 2) * 16384 + h * 8192) + 2 * (k & 3), bdesc,
                        k != 0 ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_operand(acc[0]);
    wgmma_fence_operand(acc[1]);
    if ((threadIdx.x & 127) == 0) mbar_arrive(&w_empty[st]);
    ++wc;
  };
  // accumulators -> fp32 staging rows (this warpgroup's columns), then visible to its token threads
  auto stage = [&](const float (&acc)[2][16]) {
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int r = h * 64 + fr0, c = part * 32 + 8 * j + fc;
        *reinterpret_cast<float2*>(stg + r * kTtcStgPitch + c) = make_float2(acc[h][4 * j], acc[h][4 * j + 1]);
        *reinterpret_cast<float2*>(stg + (r + 8) * kTtcStgPitch + c) =
            make_float2(acc[h][4 * j + 2], acc[h][4 * j + 3]);
      }
    ttc_bar_group(part);
  };
  float res[32];                                    // residual stream: row `row`, columns 32*part ..
  // x = LayerNorm(res + acc + bias) ; res <- x ; optionally A buffer <- fp16(x); returns x.w_out
  // (this part's 32 columns; exact two-pass statistics over the whole row).  acc is in the staging rows.
  auto residual_layernorm = [&](const float* bias, const float* gamma, const float* beta,
                                bool write_a, const float* wdot) -> float {
    const int c = part;
    float r[32];
    float sum = 0.f;
    {
      float bv[32];
      ldg32(bias + c * 32, bv);
      const float4* s4 = reinterpret_cast<const float4*>(stg + row * kTtcStgPitch + c * 32);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float4 a = s4[i];
        r[4 * i + 0] = res[4 * i + 0] + (a.x + bv[4 * i + 0]);
        r[4 * i + 1] = res[4 * i + 1] + (a.y + bv[4 * i + 1]);
        r[4 * i + 2] = res[4 * i + 2] + (a.z + bv[4 * i + 2]);
        r[4 * i + 3] = res[4 * i + 3] + (a.w + bv[4 * i + 3]);
      }
#pragma unroll
      for (int i = 0; i < 32; ++i) sum += r[i];
    }
    const float mean = combine(0, sum) * (1.0f / 128.0f);
    float var = 0.f;
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const float d = r[i] - mean;
      var = fmaf(d, d, var);
    }
    const float rstd = rsqrtf(combine(1, var) * (1.0f / 128.0f) + 1e-5f);
    float dot = 0.f;
    {
      float gv[32], bt[32];
      ldg32(gamma + c * 32, gv);
      ldg32(beta + c * 32, bt);
#pragma unroll
      for (int i = 0; i < 32; ++i) r[i] = (r[i] - mean) * rstd * gv[i] + bt[i];
      if (wdot) {
        ldg32(wdot + c * 32, gv);
#pragma unroll
        for (int i = 0; i < 32; ++i) dot = fmaf(r[i], gv[i], dot);
      }
    }
#pragma unroll
    for (int i = 0; i < 32; ++i) res[i] = r[i];
    if (write_a) write_a_chunk(c, r);
    return dot;
  };

  // source / target rows and offset of this thread's pair token in tile `t` (index -> address chain
  // of the gather; issued one tile ahead so that only the pst loads themselves are exposed)
  PairToken nx{0, 0, 0.f, 0.f};
  auto pair_lookup = [&](int t) {
    const long tk = static_cast<long>(t) * 128 + row;
    nx = PairToken{0, 0, 0.f, 0.f};
    if (t < p.num_tiles && tk < p.tokens) nx = resolve_pair(p.in, static_cast<size_t>(tk));
  };
  for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x, ++ti) {
      const long tok = static_cast<long>(tile) * 128 + row;
      const bool tok_ok = tok < p.tokens;
      // key-validity bits of this token's sample (16 consecutive tokens)
      uint32_t kmask = 0xffffu;
      bool my_valid = true;
      if (p.valid) {
        kmask = 0;
        const long s0 = static_cast<long>(tile) * 128 + (row & ~15);
#pragma unroll
        for (int j = 0; j < 16; ++j)
          if (s0 + j < p.tokens && p.valid[s0 + j]) kmask |= 1u << j;
        if (kmask == 0) kmask = 0xffffu;            // tail rows beyond `tokens`
        my_valid = tok_ok && p.valid[tok];
      }

    // ---- pair features of this token -> residual (fp32 registers) and A buffer (fp16) ----
    {
      if (ti == 0) pair_lookup(tile);              // later tiles: looked up during the previous tile
      const float ox = nx.ox, oy = nx.oy;
      const size_t ps = nx.ps, pt = nx.pt;
        {
          const int c = part;
          float v[32];
          const float4* a4 = reinterpret_cast<const float4*>(p.in.pst + ps * 256 + c * 32);
          const float4* b4 = reinterpret_cast<const float4*>(p.in.pst + pt * 256 + 128 + c * 32);
          const float4* w4 = reinterpret_cast<const float4*>(p.in.w_off + c * 64);
          const float4* c4 = reinterpret_cast<const float4*>(p.in.bias + c * 32);
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const float4 a = a4[i], bb = b4[i], w0 = __ldg(w4 + 2 * i), w1 = __ldg(w4 + 2 * i + 1),
                         cb = __ldg(c4 + i);
            float x0 = a.x + bb.x, x1 = a.y + bb.y, x2 = a.z + bb.z, x3 = a.w + bb.w;
            x0 += w0.x * ox + w0.y * oy + cb.x;
            x1 += w0.z * ox + w0.w * oy + cb.y;
            x2 += w1.x * ox + w1.y * oy + cb.z;
            x3 += w1.z * ox + w1.w * oy + cb.w;
            v[4 * i + 0] = tok_ok ? fmaxf(x0, 0.f) : 0.f;
            v[4 * i + 1] = tok_ok ? fmaxf(x1, 0.f) : 0.f;
            v[4 * i + 2] = tok_ok ? fmaxf(x2, 0.f) : 0.f;
            v[4 * i + 3] = tok_ok ? fmaxf(x3, 0.f) : 0.f;
          }
#pragma unroll
          for (int i = 0; i < 32; ++i) res[i] = v[i];
          write_a_chunk(c, v);
        }
    }
    fence_proxy_async_smem();
    ttc_bar_all();

    float dot = 0.f;
#pragma unroll 1
    for (int l = 0; l < 3; ++l) {
      const TopoLayerParams& L = p.layer[l];
      float acc[2][16];
      // ================= in_proj: k, v of head `part` -> smem (fp16 rows, bias added) =================
#pragma unroll 1
      for (int kv = 0; kv < 2; ++kv) {
        gemm(acc);
        const int c = kv * 4 + part;               // 32-column chunk of the k|v rows
        const float* bias = L.in_b + 128 + c * 32;
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const float2 bb = __ldg(reinterpret_cast<const float2*>(bias + 8 * j + fc));
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int r = h * 64 + fr0 + 8 * e;
              const int sxs = ((r >> 4) & 1) << 6;
              *reinterpret_cast<uint32_t*>(sKV + r * kTtcKVStride + ((c * 64) ^ sxs) + (8 * j + fc) * 2) =
                  pack_half2(acc[h][4 * j + 2 * e] + bb.x, acc[h][4 * j + 2 * e + 1] + bb.y);
            }
          }
      }
      // ================= in_proj: q of head `part` -> A buffer (bias, 1/sqrt(32), fp16) =================
      gemm(acc);
      ttc_bar_all();                               // every warpgroup has read the A operand
      {
        const float* bias = L.in_b + part * 32;
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const float2 bb = __ldg(reinterpret_cast<const float2*>(bias + 8 * j + fc));
#pragma unroll
            for (int e = 0; e < 2; ++e) {            // torch MHA scales q by 1/sqrt(head_dim)
              const int r = h * 64 + fr0 + 8 * e;
              *a_pair(r, part, j) = pack_half2((acc[h][4 * j + 2 * e] + bb.x) * 0.17677669529663687f,
                                               (acc[h][4 * j + 2 * e + 1] + bb.y) * 0.17677669529663687f);
            }
          }
      }
      ttc_bar_group(part);                         // q, k, v of head `part` are in smem
      {
        // ---- attention of head `part` for the warp's two samples on mma.sync (16 queries x 16 keys x
        // 32 dims per sample): k and v come straight from their smem rows through ldmatrix, P stays in
        // registers (S fragments -> A fragments), O is normalised and stored as the out_proj A operand.
        const int h = part;
          __syncwarp();
          const int g8 = lane >> 2, t4 = lane & 3;   // fragment coordinates: row g8 (+8), column pair t4
          const int mi = lane >> 3, rr = lane & 7;   // ldmatrix: this lane addresses row rr of matrix mi
          const uint32_t sA_h = smem_u32(sA) + (h >> 1) * 16384;
#pragma unroll
          for (int sh = 0; sh < 2; ++sh) {
            const int r0 = quarter * 32 + sh * 16;                 // first tile row of the sample
            const int sxs = ((r0 >> 4) & 1) << 6;                  // odd samples: k|v columns XOR 64 B
            const uint32_t km = __shfl_sync(0xffffffffu, kmask, sh * 16);
            // S = Q K^T : two 8-key column tiles, two 16-dim k-steps
            float sacc[2][4];
#pragma unroll
            for (int nt = 0; nt < 2; ++nt)
#pragma unroll
              for (int i = 0; i < 4; ++i) sacc[nt][i] = 0.f;
#pragma unroll
            for (int ks = 0; ks < 2; ++ks) {
              uint32_t qa[4], kb[4];
              {   // matrices: (rows 0-7 | 8-15) x (dims ks*16 + 0-7 | 8-15)
                const int qr = r0 + (mi & 1) * 8 + rr;
                const int piece = (h & 1) * 4 + ks * 2 + (mi >> 1);
                ttc_ldmatrix_x4(qa, sA_h + qr * 128 + ((piece ^ (qr & 7)) << 4));
              }
              {   // matrices: (keys 0-7 | 8-15) x (dims ks*16 + 0-7 | 8-15) -> b0, b1 of tile 0; of tile 1
                const int kr = r0 + (mi >> 1) * 8 + rr;
                ttc_ldmatrix_x4(kb, smem_u32(sKV) + kr * kTtcKVStride + ((h * 64) ^ sxs) +
                                        (ks * 16 + (mi & 1) * 8) * 2);
              }
              ttc_mma_16816(sacc[0], qa, kb[0], kb[1]);
              ttc_mma_16816(sacc[1], qa, kb[2], kb[3]);
            }
            // masked softmax of rows g8 (values [nt][0..1]) and g8 + 8 ([nt][2..3]); keys nt*8 + 2*t4 (+1)
            float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
            for (int nt = 0; nt < 2; ++nt)
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                const bool on = (km >> (nt * 8 + 2 * t4 + e)) & 1u;
                sacc[nt][e] = on ? sacc[nt][e] : -INFINITY;
                sacc[nt][2 + e] = on ? sacc[nt][2 + e] : -INFINITY;
                mx0 = fmaxf(mx0, sacc[nt][e]);
                mx1 = fmaxf(mx1, sacc[nt][2 + e]);
              }
            mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
            mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
            mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
            mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
            float l0 = 0.f, l1 = 0.f;
#pragma unroll
            for (int nt = 0; nt < 2; ++nt)
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                sacc[nt][e] = __expf(sacc[nt][e] - mx0);           // exp(-inf) = 0 for masked keys
                sacc[nt][2 + e] = __expf(sacc[nt][2 + e] - mx1);
                l0 += sacc[nt][e];
                l1 += sacc[nt][2 + e];
              }
            l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
            l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
            l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
            l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
            uint32_t pa[4];
            pa[0] = pack_half2(sacc[0][0], sacc[0][1]);
            pa[1] = pack_half2(sacc[0][2], sacc[0][3]);
            pa[2] = pack_half2(sacc[1][0], sacc[1][1]);
            pa[3] = pack_half2(sacc[1][2], sacc[1][3]);
            // O = P V : four 8-dim column tiles, one 16-key k-step
            float oacc[4][4];
#pragma unroll
            for (int j = 0; j < 4; ++j)
#pragma unroll
              for (int i = 0; i < 4; ++i) oacc[j][i] = 0.f;
#pragma unroll
            for (int dh = 0; dh < 2; ++dh) {
              uint32_t vb[4];   // transposed matrices: (keys 0-7 | 8-15) x (dims dh*16 + 0-7 | 8-15)
              const int vr = r0 + (mi & 1) * 8 + rr;
              ttc_ldmatrix_x4_trans(vb, smem_u32(sKV) + vr * kTtcKVStride + ((256 + h * 64) ^ sxs) +
                                            (dh * 16 + (mi >> 1) * 8) * 2);
              ttc_mma_16816(oacc[dh * 2 + 0], pa, vb[0], vb[1]);
              ttc_mma_16816(oacc[dh * 2 + 1], pa, vb[2], vb[3]);
            }
            const float inv0 = 1.0f / l0, inv1 = 1.0f / l1;
            __syncwarp();                            // every lane's Q fragments of this sample are loaded
            const int ra = r0 + g8, rb = r0 + g8 + 8;
#pragma unroll
            for (int j = 0; j < 4; ++j) {            // attention output columns h*32 + j*8 + 2*t4 (+1)
              const int piece = (h & 1) * 4 + j;
              *reinterpret_cast<uint32_t*>(sA + (h >> 1) * 16384 + ra * 128 + ((piece ^ (ra & 7)) << 4) + t4 * 4) =
                  pack_half2(oacc[j][0] * inv0, oacc[j][1] * inv0);
              *reinterpret_cast<uint32_t*>(sA + (h >> 1) * 16384 + rb * 128 + ((piece ^ (rb & 7)) << 4) + t4 * 4) =
                  pack_half2(oacc[j][2] * inv1, oacc[j][3] * inv1);
            }
          }
        }
      fence_proxy_async_smem();
      ttc_bar_all();
      // ================= out_proj + residual + LayerNorm1 =================
      gemm(acc);
      ttc_bar_all();                               // A operand read by every warpgroup
      stage(acc);
      residual_layernorm(L.out_b, L.n1_g, L.n1_b, true, nullptr);
      fence_proxy_async_smem();
      ttc_bar_all();
      // ================= linear1 + relu =================
      gemm(acc);
      ttc_bar_all();
      {
        const float* bias = L.l1_b + part * 32;
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const float2 bb = __ldg(reinterpret_cast<const float2*>(bias + 8 * j + fc));
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int r = h * 64 + fr0 + 8 * e;
              *a_pair(r, part, j) = pack_half2(fmaxf(acc[h][4 * j + 2 * e] + bb.x, 0.f),
                                               fmaxf(acc[h][4 * j + 2 * e + 1] + bb.y, 0.f));
            }
          }
      }
      fence_proxy_async_smem();
      ttc_bar_all();
      if (l == 2) pair_lookup(tile + static_cast<int>(gridDim.x));   // next tile's indices, off the critical path
      // ================= linear2 + residual + LayerNorm2 =================
      gemm(acc);
      ttc_bar_all();
      stage(acc);
      dot = residual_layernorm(L.l2_b, L.n2_g, L.n2_b, l < 2, l == 2 ? p.out_w : nullptr);
      if (l < 2) {
        fence_proxy_async_smem();
        ttc_bar_all();
      }
    }
    // ================= output_proj + sigmoid =================
    dot = combine(2, dot);
    if (tok_ok && part == 0) {
      const float b = __ldg(p.out_b);
      const float lg = my_valid ? dot + b : b;
      if (p.logits) p.logits[tok] = lg;
      if (p.scores) p.scores[tok] = 1.0f / (1.0f + expf(-lg));
    }
  }
}

}  // namespace srb
