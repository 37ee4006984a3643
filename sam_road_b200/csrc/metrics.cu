// sam_road_b200 :: metrics.cu -- exact binary precision-recall curves for threshold search.
//
// Replaces the three torchmetrics BinaryPrecisionRecallCurve(ignore_index=-1) of SAMRoad (reference
// model.py:361-363) that test_step feeds (model.py:602-617) and on_test_end reads (model.py:619-634).
//
//   update   every kept (score, label) pair becomes one 32-bit key  float_bits(score) << 1 | label
//            (< 2^31 because scores are in [0, 1]) appended to a device buffer: 4 B per entry.
//   compute  LSD radix sort of the keys (4 passes of 8 bits), then per distinct score the number of
//            positives / negatives at or above it as exact int64 counts, then precision, recall and F1 in
//            float32 with the reference's operations in its order, and torch.argmax of F1.
//
// torchmetrics keeps float32 scores and int64 labels, sorts descending and takes a float32 cumsum of the
// labels; that cumsum is exact only while partial sums stay <= 2^24.  Here the counts are integers, so
// the curve is the exact one rounded once to float32 (DESIGN.md §10).
#include "../../include/samroad_b200.h"

#include <cuda_runtime.h>

#include <cmath>
#include <cstdio>
#include <cstring>

#include "common.cuh"
#include "ops.h"

using namespace srb;

namespace {

// Device-side state of one accumulator.  `staged` runs ahead of `committed` while an update appends;
// the commit kernel keeps or drops the update's entries as a whole.
struct PrcState {
  unsigned long long committed;   // entries accepted so far
  unsigned long long staged;      // committed + entries of the update in flight
  unsigned int flags;             // kBad* bits of the update in flight
  unsigned long long first_bad;   // smallest offending element index of the update in flight
  unsigned int sticky_count;      // refused updates not yet reported
  unsigned int sticky_flags;      // union of their kBad* bits
  unsigned long long sticky_bad;  // offending element of the first of them
  long long sticky_update;        // serial number of the first of them (counted from the last reset)
  unsigned long long best;        // compute: argmax key, see best_key()
};

constexpr unsigned kBadPred = 1u, kBadTarget = 2u;

// Tile sizes.  The radix sort gives one warp a chunk of kSortChunk keys (stable within the warp by
// __match_any_sync ranks); scans and the curve kernel give a 256-thread block kTile elements.
constexpr int kSortChunk = 4096;
constexpr int kSortWarps = 8;
constexpr int kTile = 4096;
constexpr int kTileItems = kTile / 256;

}  // namespace

struct samroad_prc_ctx {
  int device = 0;
  PrcState* state = nullptr;       // device
  uint32_t* keys = nullptr;        // device, cap entries
  uint32_t* alt = nullptr;         // compute: radix ping-pong buffer
  size_t cap = 0, alt_cap = 0;
  size_t reserved = 0;             // host upper bound of state->committed
  long long n_updates = 0;         // updates since the last reset
  // scratch of compute
  uint32_t* hist = nullptr;        // per (digit, chunk) counts, scanned in place
  uint32_t* tile_sums = nullptr;
  unsigned long long* tile_cnt = nullptr;   // curve: (starts << 32 | positives) per tile, then scanned
  size_t hist_cap = 0, tile_sums_cap = 0, tile_cnt_cap = 0;
  // the curve of the last successful compute
  float* thr = nullptr;            // [T]
  float* prec = nullptr;           // [T+1]
  float* rec = nullptr;            // [T+1]
  long long* tps = nullptr;        // [T]
  long long* fps = nullptr;        // [T]
  size_t curve_cap = 0;
  long long T = -1;                // -1: no curve
  PrcState* h_state = nullptr;     // pinned read-back

  ~samroad_prc_ctx() {
    if (keys) {   // allocated stream-ordered by samroad_prc_update
      cudaFreeAsync(keys, 0);
      cudaStreamSynchronize(0);
    }
    for (void* p : {static_cast<void*>(state), static_cast<void*>(alt),
                    static_cast<void*>(hist), static_cast<void*>(tile_sums), static_cast<void*>(tile_cnt),
                    static_cast<void*>(thr), static_cast<void*>(prec), static_cast<void*>(rec),
                    static_cast<void*>(tps), static_cast<void*>(fps)})
      if (p) cudaFree(p);
    if (h_state) cudaFreeHost(h_state);
  }
};

namespace {

inline int grid_for(long long n, int per) { return static_cast<int>((n + per - 1) / per); }

// Grows a synchronously owned scratch buffer (compute synchronises anyway).
template <typename T>
int ensure(T*& p, size_t& cap, size_t n) {
  if (n <= cap) return 0;
  if (p) SRB_CUDA_OK(cudaFree(p));
  p = nullptr;
  cap = 0;
  const size_t want = n + n / 4 + 64;
  SRB_CUDA_OK(cudaMalloc(&p, sizeof(T) * want));
  cap = want;
  return 0;
}

// ---------------------------------------------------------------------------------------------------
// update
// ---------------------------------------------------------------------------------------------------
// The label is int32(target) (torch's .to(torch.int32) truncates), valid only when it is 0 or 1.  A
// score must lie in [0, 1]: torchmetrics would sigmoid the whole batch instead, which a probability
// output never asks for, so such a batch is refused.  -0.0 is stored as +0.0 (the same threshold).
// Warp-aggregated append of the kept keys at st->staged; the order inside the buffer is irrelevant,
// compute sorts the keys.
__device__ __forceinline__ void append_key(bool keep, uint32_t key, uint32_t* keys, PrcState* st) {
  const unsigned lane = threadIdx.x & 31;
  const unsigned m = __ballot_sync(0xffffffffu, keep);
  if (m == 0) return;
  const int leader = __ffs(m) - 1;
  unsigned long long base = 0;
  if (static_cast<int>(lane) == leader) base = atomicAdd(&st->staged, static_cast<unsigned long long>(__popc(m)));
  base = __shfl_sync(0xffffffffu, base, leader);
  if (keep) keys[base + __popc(m & ((1u << lane) - 1u))] = key;
}

template <bool kU8Target>
__global__ void __launch_bounds__(256) prc_append_kernel(const float* __restrict__ preds, long long pstride,
                                                         const void* __restrict__ target,
                                                         const uint8_t* __restrict__ valid, long long n,
                                                         uint32_t* __restrict__ keys, PrcState* __restrict__ st) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  bool keep = false;
  uint32_t key = 0;
  if (i < n && (valid == nullptr || valid[i] != 0)) {
    const float s = preds[i * pstride];
    int label;
    bool tgt_ok;
    if (kU8Target) {
      const unsigned t = static_cast<const uint8_t*>(target)[i];
      label = static_cast<int>(t);
      tgt_ok = t <= 1u;
    } else {
      const float t = static_cast<const float*>(target)[i];
      tgt_ok = t > -1.0f && t < 2.0f;          // false for NaN; truncates to 0 or 1 otherwise
      label = tgt_ok ? static_cast<int>(t) : 0;
    }
    const bool pred_ok = s >= 0.0f && s <= 1.0f;   // false for NaN
    if (!pred_ok || !tgt_ok) {
      atomicOr(&st->flags, (pred_ok ? 0u : kBadPred) | (tgt_ok ? 0u : kBadTarget));
      atomicMin(&st->first_bad, static_cast<unsigned long long>(i));
    } else {
      keep = true;
      key = (__float_as_uint(s == 0.0f ? 0.0f : s) << 1) | static_cast<uint32_t>(label);
    }
  }
  append_key(keep, key, keys, st);
}

// Keys made by another accumulator (samroad_prc_export_keys), e.g. on another rank.  A key whose score
// part is not in [0, 1] refuses the update like a bad prediction.
__global__ void __launch_bounds__(256) prc_append_keys_kernel(const uint32_t* __restrict__ in, long long n,
                                                              uint32_t* __restrict__ keys,
                                                              PrcState* __restrict__ st) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  bool keep = false;
  uint32_t key = 0;
  if (i < n) {
    key = in[i];
    keep = (key >> 1) <= 0x3F800000u;          // float bits of a score in [0, 1]
    if (!keep) {
      atomicOr(&st->flags, kBadPred);
      atomicMin(&st->first_bad, static_cast<unsigned long long>(i));
    }
  }
  append_key(keep, key, keys, st);
}

__global__ void prc_begin_kernel(PrcState* st) {
  st->staged = st->committed;
  st->flags = 0;
  st->first_bad = ~0ull;
}

// Keeps the update's entries, or drops all of them and counts the refusal (the first one in detail) until a
// synchronising call reports it.
__global__ void prc_commit_kernel(PrcState* st, long long serial) {
  if (st->flags == 0) {
    st->committed = st->staged;
  } else {
    if (st->sticky_count == 0) {
      st->sticky_bad = st->first_bad;
      st->sticky_update = serial;
    }
    ++st->sticky_count;
    st->sticky_flags |= st->flags;
  }
  st->staged = st->committed;
}

// ---------------------------------------------------------------------------------------------------
// LSD radix sort of 32-bit keys, 8 bits per pass: per (digit, warp chunk) histogram, one exclusive scan
// of the digit-major histogram (global offsets of every digit in every chunk), ordered scatter.  A warp
// walks its chunk in 32-key steps; __match_any_sync ranks equal digits within a step in lane order, so
// each pass is stable and the result does not depend on scheduling.
// ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(32 * kSortWarps) radix_hist_kernel(const uint32_t* __restrict__ keys, long long n,
                                                                    int nchunks, int shift,
                                                                    uint32_t* __restrict__ hist) {
  __shared__ uint32_t h[kSortWarps][256];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int chunk = blockIdx.x * kSortWarps + w;
  for (int d = lane; d < 256; d += 32) h[w][d] = 0;
  __syncwarp();
  if (chunk < nchunks) {
    const long long base = static_cast<long long>(chunk) * kSortChunk;
    for (int it = 0; it < kSortChunk / 32; ++it) {
      const long long i = base + it * 32 + lane;
      if (i < n) atomicAdd(&h[w][(keys[i] >> shift) & 255u], 1u);
    }
    __syncwarp();
    for (int d = lane; d < 256; d += 32) hist[static_cast<size_t>(d) * nchunks + chunk] = h[w][d];
  }
}

__global__ void __launch_bounds__(32 * kSortWarps) radix_scatter_kernel(const uint32_t* __restrict__ in, long long n,
                                                                       int nchunks, int shift,
                                                                       const uint32_t* __restrict__ off,
                                                                       uint32_t* __restrict__ out) {
  __shared__ uint32_t o[kSortWarps][256];
  const int w = threadIdx.x >> 5;
  const unsigned lane = threadIdx.x & 31;
  const int chunk = blockIdx.x * kSortWarps + w;
  if (chunk >= nchunks) return;
  for (int d = lane; d < 256; d += 32) o[w][d] = off[static_cast<size_t>(d) * nchunks + chunk];
  __syncwarp();
  const long long base = static_cast<long long>(chunk) * kSortChunk;
  for (int it = 0; it < kSortChunk / 32; ++it) {
    const long long i = base + it * 32 + lane;
    const bool ok = i < n;
    const uint32_t key = ok ? in[i] : 0u;
    const unsigned d = ok ? ((key >> shift) & 255u) : (256u + lane);   // idle lanes match only themselves
    const unsigned peers = __match_any_sync(0xffffffffu, d);
    const unsigned r = __popc(peers & ((1u << lane) - 1u));
    uint32_t pos = 0;
    if (ok) pos = o[w][d] + r;
    __syncwarp();
    if (ok && r == 0) o[w][d] += __popc(peers);
    __syncwarp();
    if (ok) out[pos] = key;
  }
}

// ---------------------------------------------------------------------------------------------------
// exclusive scans: 256-thread block scan, tile sums -> one-block scan of the sums -> tile scan
// ---------------------------------------------------------------------------------------------------
template <typename T>
__device__ __forceinline__ T block_excl_scan256(T v, T* sw /*[9]*/, T& total) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  T inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const T t = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += t;
  }
  if (lane == 31) sw[wid] = inc;
  __syncthreads();
  if (threadIdx.x == 0) {
    T acc = 0;
    for (int k = 0; k < 8; ++k) {
      const T t = sw[k];
      sw[k] = acc;
      acc += t;
    }
    sw[8] = acc;
  }
  __syncthreads();
  const T res = inc - v + sw[wid];
  total = sw[8];
  __syncthreads();
  return res;
}

__global__ void __launch_bounds__(256) tile_sum_kernel(const uint32_t* __restrict__ a, long long m,
                                                       uint32_t* __restrict__ sums) {
  __shared__ uint32_t sw[9];
  const long long base = static_cast<long long>(blockIdx.x) * kTile;
  uint32_t s = 0;
  for (int it = 0; it < kTileItems; ++it) {
    const long long i = base + it * 256 + threadIdx.x;
    if (i < m) s += a[i];
  }
  uint32_t total;
  block_excl_scan256(s, sw, total);
  if (threadIdx.x == 0) sums[blockIdx.x] = total;
}

// in-place exclusive scan of m values by one block
template <typename T>
__global__ void __launch_bounds__(256) scan_one_block_kernel(T* __restrict__ a, int m) {
  __shared__ T sw[9];
  T carry = 0;
  for (int base = 0; base < m; base += 256) {
    const int i = base + threadIdx.x;
    const T v = i < m ? a[i] : T(0);
    T total;
    const T ex = block_excl_scan256(v, sw, total);
    if (i < m) a[i] = carry + ex;
    carry += total;
  }
}

__global__ void __launch_bounds__(256) tile_scan_kernel(uint32_t* __restrict__ a, long long m,
                                                        const uint32_t* __restrict__ tile_off) {
  __shared__ uint32_t sw[9];
  const long long base = static_cast<long long>(blockIdx.x) * kTile;
  uint32_t carry = tile_off[blockIdx.x];
  for (int it = 0; it < kTileItems; ++it) {
    const long long i = base + it * 256 + threadIdx.x;
    const uint32_t v = i < m ? a[i] : 0u;
    uint32_t total;
    const uint32_t ex = block_excl_scan256(v, sw, total);
    if (i < m) a[i] = carry + ex;
    carry += total;
  }
}

// ---------------------------------------------------------------------------------------------------
// curve over the sorted keys.  Element i starts a run when its score differs from element i-1's; run j
// (ascending score) is threshold j.  Runs and positives are counted per tile, the tile counts are scanned
// (packed as starts << 32 | positives: both stay below 2^31), then each run start knows how many
// positives lie below it.
// ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ bool run_start(const uint32_t* keys, long long i) {
  return i == 0 || (keys[i] >> 1) != (keys[i - 1] >> 1);
}

__global__ void __launch_bounds__(256) curve_count_kernel(const uint32_t* __restrict__ keys, long long n,
                                                          unsigned long long* __restrict__ tile_cnt) {
  __shared__ unsigned long long sw[9];
  const long long base = static_cast<long long>(blockIdx.x) * kTile;
  unsigned long long c = 0;
  for (int it = 0; it < kTileItems; ++it) {
    const long long i = base + it * 256 + threadIdx.x;
    if (i < n) c += (run_start(keys, i) ? (1ull << 32) : 0ull) + (keys[i] & 1u);
  }
  unsigned long long total;
  block_excl_scan256(c, sw, total);
  if (threadIdx.x == 0) tile_cnt[blockIdx.x] = total;
}

// torch.argmax order of F1 values: NaN above every number, then larger value, then smaller index.
// F1 is NaN or in [0, 1], so the float bits of a number order it.
__device__ __forceinline__ unsigned long long best_key(float f1, long long j) {
  const unsigned long long v = isnan(f1) ? 0xFFFFFFFFull : static_cast<unsigned long long>(__float_as_uint(f1));
  return (v << 32) | (0xFFFFFFFFull - static_cast<unsigned long long>(j));
}

// tps / fps of threshold j count the entries with score >= threshold j: all positives minus those below
// the run, and the entries from the run start on minus tps (the scan from the highest score down).
// precision = tps / (tps + fps), recall = tps / tps_total, f1 = 2 * (p * r) / (p + r) in float32, each
// operation rounded to nearest as torch performs it (the intrinsics keep that under any build flags).
__global__ void __launch_bounds__(256) curve_fill_kernel(const uint32_t* __restrict__ keys, long long n,
                                                         const unsigned long long* __restrict__ tile_off,
                                                         long long n_pos, long long T, float* __restrict__ thr,
                                                         float* __restrict__ prec, float* __restrict__ rec,
                                                         long long* __restrict__ tps_out,
                                                         long long* __restrict__ fps_out,
                                                         PrcState* __restrict__ st) {
  __shared__ unsigned long long sw[9];
  __shared__ unsigned long long best_sh;
  if (threadIdx.x == 0) best_sh = 0;
  const long long base = static_cast<long long>(blockIdx.x) * kTile;
  unsigned long long carry = tile_off[blockIdx.x];
  unsigned long long best = 0;
  const float total_f = __ll2float_rn(n_pos);
  for (int it = 0; it < kTileItems; ++it) {
    const long long i = base + it * 256 + threadIdx.x;
    const bool in = i < n;
    const uint32_t key = in ? keys[i] : 0u;
    const bool start = in && run_start(keys, i);
    const unsigned long long c = (start ? (1ull << 32) : 0ull) + (in ? (key & 1u) : 0u);
    unsigned long long total;
    const unsigned long long ex = carry + block_excl_scan256(c, sw, total);
    carry += total;
    if (start) {
      const long long j = static_cast<long long>(ex >> 32);
      const long long pos_below = static_cast<long long>(ex & 0xFFFFFFFFull);
      const long long tp = n_pos - pos_below;
      const long long fp = (n - i) - tp;
      const float tf = __ll2float_rn(tp), ff = __ll2float_rn(fp);
      const float p = __fdiv_rn(tf, __fadd_rn(tf, ff));
      const float r = __fdiv_rn(tf, total_f);
      const float f1 = __fdiv_rn(__fmul_rn(2.0f, __fmul_rn(p, r)), __fadd_rn(p, r));
      thr[j] = __uint_as_float(key >> 1);
      prec[j] = p;
      rec[j] = r;
      tps_out[j] = tp;
      fps_out[j] = fp;
      const unsigned long long b = best_key(f1, j);
      best = b > best ? b : best;
    }
  }
  // the final point (precision 1, recall 0, f1 0) never wins: f1 at threshold 0 is > 0 or NaN
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    prec[T] = 1.0f;
    rec[T] = 0.0f;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long t = __shfl_xor_sync(0xffffffffu, best, o);
    best = t > best ? t : best;
  }
  __syncthreads();
  if ((threadIdx.x & 31) == 0 && best) atomicMax(&best_sh, best);
  __syncthreads();
  if (threadIdx.x == 0 && best_sh) atomicMax(&st->best, best_sh);
}

int read_state(samroad_prc_ctx* p, cudaStream_t st) {
  SRB_CUDA_OK(cudaMemcpyAsync(p->h_state, p->state, sizeof(PrcState), cudaMemcpyDeviceToHost, st));
  SRB_CUDA_OK(cudaStreamSynchronize(st));
  return 0;
}

// Synchronises, and fails with code 3 while refused updates are unreported: it reports them all (their
// number, the first in detail) and clears the count, so no later call can succeed past an unreported
// refusal.  On success *committed holds the number of accepted entries.
int take_refusals(samroad_prc_ctx* p, const char* what, long long* committed, cudaStream_t st) {
  if (int rc = read_state(p, st)) return rc;
  const PrcState s = *p->h_state;
  p->reserved = s.committed;
  *committed = static_cast<long long>(s.committed);
  if (s.sticky_count == 0) return 0;
  SRB_CUDA_OK(cudaMemsetAsync(&p->state->sticky_count, 0, sizeof(unsigned int), st));
  SRB_CUDA_OK(cudaMemsetAsync(&p->state->sticky_flags, 0, sizeof(unsigned int), st));
  SRB_CUDA_OK(cudaStreamSynchronize(st));
  set_last_error("%s: %u update(s) since the last report were refused and added nothing; the first, "
                 "update #%lld since the last reset, at element %llu:%s%s",
                 what, s.sticky_count, s.sticky_update, s.sticky_bad,
                 (s.sticky_flags & kBadPred) ? " a prediction is NaN or outside [0, 1]" : "",
                 (s.sticky_flags & kBadTarget) ? " a target is not 0 or 1 after truncation to int32" : "");
  return 3;
}

void free_curve(samroad_prc_ctx* p) {
  for (void** a : {reinterpret_cast<void**>(&p->thr), reinterpret_cast<void**>(&p->prec),
                   reinterpret_cast<void**>(&p->rec), reinterpret_cast<void**>(&p->tps),
                   reinterpret_cast<void**>(&p->fps)}) {
    if (*a) cudaFree(*a);
    *a = nullptr;
  }
  p->curve_cap = 0;
}

// The five curve arrays for T thresholds; all of them or none (curve_cap 0) after a failure.
int ensure_curve(samroad_prc_ctx* p, size_t T) {
  const size_t need = T + 1;
  if (need <= p->curve_cap) return 0;
  free_curve(p);
  const size_t c = need + need / 4 + 64;
  if (cudaMalloc(&p->thr, sizeof(float) * c) != cudaSuccess || cudaMalloc(&p->prec, sizeof(float) * c) != cudaSuccess ||
      cudaMalloc(&p->rec, sizeof(float) * c) != cudaSuccess ||
      cudaMalloc(&p->tps, sizeof(long long) * c) != cudaSuccess ||
      cudaMalloc(&p->fps, sizeof(long long) * c) != cudaSuccess) {
    cudaGetLastError();
    free_curve(p);
    set_last_error("samroad_prc_compute: out of device memory for a curve of %zu thresholds", T);
    return 1;
  }
  p->curve_cap = c;
  return 0;
}

// Room for n more keys after the `reserved` ones, grown stream-ordered (no host synchronisation).
int grow_keys(samroad_prc_ctx* p, long long n, const char* what, cudaStream_t st) {
  // keys are indexed and counted in 32 bits by compute
  SRB_REQUIRE(p->reserved + static_cast<size_t>(n) < (1ull << 31), "%s: more than 2^31-1 entries in one accumulator",
              what);
  const size_t need = p->reserved + static_cast<size_t>(n);
  if (need <= p->cap) return 0;
  const size_t want = need > 2 * p->cap ? need : 2 * p->cap;
  uint32_t* nk = nullptr;
  SRB_CUDA_OK(cudaMallocAsync(reinterpret_cast<void**>(&nk), sizeof(uint32_t) * want, st));
  if (p->keys) {
    if (p->reserved)
      SRB_CUDA_OK(cudaMemcpyAsync(nk, p->keys, sizeof(uint32_t) * p->reserved, cudaMemcpyDeviceToDevice, st));
    SRB_CUDA_OK(cudaFreeAsync(p->keys, st));
  }
  p->keys = nk;
  p->cap = want;
  return 0;
}

// exclusive scan of m uint32 in place (values and their total < 2^32)
int scan_u32(samroad_prc_ctx* p, uint32_t* a, long long m, cudaStream_t st) {
  const int tiles = grid_for(m, kTile);
  if (int rc = ensure(p->tile_sums, p->tile_sums_cap, static_cast<size_t>(tiles))) return rc;
  tile_sum_kernel<<<tiles, 256, 0, st>>>(a, m, p->tile_sums);
  scan_one_block_kernel<uint32_t><<<1, 256, 0, st>>>(p->tile_sums, tiles);
  tile_scan_kernel<<<tiles, 256, 0, st>>>(a, m, p->tile_sums);
  SRB_CUDA_OK(cudaGetLastError());
  note_launch(3);
  return 0;
}

int radix_sort(samroad_prc_ctx* p, long long n, cudaStream_t st) {
  if (int rc = ensure(p->alt, p->alt_cap, static_cast<size_t>(n))) return rc;
  const int nchunks = grid_for(n, kSortChunk);
  const long long m = 256LL * nchunks;
  if (int rc = ensure(p->hist, p->hist_cap, static_cast<size_t>(m))) return rc;
  const int blocks = grid_for(nchunks, kSortWarps);
  uint32_t* src = p->keys;
  uint32_t* dst = p->alt;
  for (int shift = 0; shift < 32; shift += 8) {    // 4 passes: the sorted keys end up back in p->keys
    radix_hist_kernel<<<blocks, 32 * kSortWarps, 0, st>>>(src, n, nchunks, shift, p->hist);
    SRB_CUDA_OK(cudaGetLastError());
    note_launch(1);
    if (int rc = scan_u32(p, p->hist, m, st)) return rc;
    radix_scatter_kernel<<<blocks, 32 * kSortWarps, 0, st>>>(src, n, nchunks, shift, p->hist, dst);
    SRB_CUDA_OK(cudaGetLastError());
    note_launch(1);
    uint32_t* t = src;
    src = dst;
    dst = t;
  }
  return 0;
}

}  // namespace

// =================================================================================================
// C ABI
// =================================================================================================
extern "C" int samroad_prc_create(int device, samroad_prc_t* out) {
  SRB_REQUIRE(out != nullptr, "samroad_prc_create: null argument");
  int ndev = 0;
  SRB_CUDA_OK(cudaGetDeviceCount(&ndev));
  SRB_REQUIRE(ndev > 0, "no CUDA device: libsamroad_b200 has no CPU fallback");
  SRB_REQUIRE(device >= 0 && device < ndev, "device %d out of range (0..%d)", device, ndev - 1);
  SRB_CUDA_OK(cudaSetDevice(device));
  samroad_prc_ctx* p = new samroad_prc_ctx();
  p->device = device;
  if (cudaMalloc(&p->state, sizeof(PrcState)) != cudaSuccess ||
      cudaMemset(p->state, 0, sizeof(PrcState)) != cudaSuccess ||
      cudaMallocHost(&p->h_state, sizeof(PrcState)) != cudaSuccess) {
    delete p;
    set_last_error("samroad_prc_create: device or pinned allocation failed");
    return 1;
  }
  *out = p;
  return 0;
}

extern "C" int samroad_prc_destroy(samroad_prc_t p) {
  if (!p) return 0;
  cudaSetDevice(p->device);
  cudaDeviceSynchronize();
  delete p;
  return 0;
}

extern "C" int samroad_prc_reset(samroad_prc_t p, void* stream) {
  SRB_REQUIRE(p != nullptr, "samroad_prc_reset: null handle");
  SRB_CUDA_OK(cudaSetDevice(p->device));
  SRB_CUDA_OK(cudaMemsetAsync(p->state, 0, sizeof(PrcState), static_cast<cudaStream_t>(stream)));
  p->reserved = 0;
  p->n_updates = 0;
  p->T = -1;
  return 0;
}

extern "C" int samroad_prc_update(samroad_prc_t p, const float* preds, int64_t pred_stride, const void* target,
                                  int target_dtype, const uint8_t* valid, int64_t n, void* stream) {
  SRB_REQUIRE(p != nullptr, "samroad_prc_update: null handle");
  SRB_REQUIRE(n >= 0 && pred_stride >= 1, "samroad_prc_update: n=%lld, pred_stride=%lld",
              static_cast<long long>(n), static_cast<long long>(pred_stride));
  SRB_REQUIRE(target_dtype == SAMROAD_F32 || target_dtype == SAMROAD_U8,
              "samroad_prc_update: target dtype %d (SAMROAD_F32 or SAMROAD_U8)", target_dtype);
  if (n == 0) return 0;
  SRB_REQUIRE(preds && target, "samroad_prc_update: null argument");
  SRB_CUDA_OK(cudaSetDevice(p->device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (int rc = grow_keys(p, n, "samroad_prc_update", st)) return rc;
  prc_begin_kernel<<<1, 1, 0, st>>>(p->state);
  if (target_dtype == SAMROAD_U8)
    prc_append_kernel<true><<<grid_for(n, 256), 256, 0, st>>>(preds, pred_stride, target, valid, n, p->keys, p->state);
  else
    prc_append_kernel<false><<<grid_for(n, 256), 256, 0, st>>>(preds, pred_stride, target, valid, n, p->keys, p->state);
  prc_commit_kernel<<<1, 1, 0, st>>>(p->state, p->n_updates);
  SRB_CUDA_OK(cudaGetLastError());
  note_launch(3);
  p->reserved += static_cast<size_t>(n);
  ++p->n_updates;
  return 0;
}

extern "C" int samroad_prc_append_keys(samroad_prc_t p, const uint32_t* keys, int64_t n, void* stream) {
  SRB_REQUIRE(p != nullptr && n >= 0, "samroad_prc_append_keys: null handle or n < 0");
  if (n == 0) return 0;
  SRB_REQUIRE(keys != nullptr, "samroad_prc_append_keys: null argument");
  SRB_CUDA_OK(cudaSetDevice(p->device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (int rc = grow_keys(p, n, "samroad_prc_append_keys", st)) return rc;
  prc_begin_kernel<<<1, 1, 0, st>>>(p->state);
  prc_append_keys_kernel<<<grid_for(n, 256), 256, 0, st>>>(keys, n, p->keys, p->state);
  prc_commit_kernel<<<1, 1, 0, st>>>(p->state, p->n_updates);
  SRB_CUDA_OK(cudaGetLastError());
  note_launch(3);
  p->reserved += static_cast<size_t>(n);
  ++p->n_updates;
  return 0;
}

extern "C" int samroad_prc_export_keys(samroad_prc_t p, uint32_t* keys, int64_t cap, int64_t* n_keys, void* stream) {
  SRB_REQUIRE(p != nullptr && n_keys != nullptr, "samroad_prc_export_keys: null argument");
  SRB_CUDA_OK(cudaSetDevice(p->device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  long long n = 0;
  if (int rc = take_refusals(p, "samroad_prc_export_keys", &n, st)) return rc;
  *n_keys = n;
  if (keys == nullptr || n == 0) return 0;
  SRB_REQUIRE(cap >= n, "samroad_prc_export_keys: room for %lld keys, %lld needed", static_cast<long long>(cap), n);
  SRB_CUDA_OK(cudaMemcpyAsync(keys, p->keys, sizeof(uint32_t) * static_cast<size_t>(n), cudaMemcpyDefault, st));
  return 0;
}

extern "C" int samroad_prc_compute(samroad_prc_t p, int64_t* counts, float* best, void* stream) {
  SRB_REQUIRE(p != nullptr && counts && best, "samroad_prc_compute: null argument");
  SRB_CUDA_OK(cudaSetDevice(p->device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  p->T = -1;
  long long n = 0;
  if (int rc = take_refusals(p, "samroad_prc_compute", &n, st)) return rc;
  SRB_REQUIRE(n > 0, "samroad_prc_compute: no entries (nothing was updated since the last reset)");
  if (int rc = radix_sort(p, n, st)) return rc;
  const int tiles = grid_for(n, kTile);
  if (int rc = ensure(p->tile_cnt, p->tile_cnt_cap, static_cast<size_t>(tiles) + 1)) return rc;
  curve_count_kernel<<<tiles, 256, 0, st>>>(p->keys, n, p->tile_cnt);
  SRB_CUDA_OK(cudaMemsetAsync(p->tile_cnt + tiles, 0, sizeof(unsigned long long), st));
  scan_one_block_kernel<unsigned long long><<<1, 256, 0, st>>>(p->tile_cnt, tiles + 1);
  SRB_CUDA_OK(cudaGetLastError());
  note_launch(2);
  unsigned long long tot = 0;
  SRB_CUDA_OK(cudaMemcpyAsync(&tot, p->tile_cnt + tiles, sizeof(tot), cudaMemcpyDeviceToHost, st));
  SRB_CUDA_OK(cudaStreamSynchronize(st));
  const long long T = static_cast<long long>(tot >> 32), n_pos = static_cast<long long>(tot & 0xFFFFFFFFull);
  if (int rc = ensure_curve(p, static_cast<size_t>(T))) return rc;
  SRB_CUDA_OK(cudaMemsetAsync(&p->state->best, 0, sizeof(unsigned long long), st));
  curve_fill_kernel<<<tiles, 256, 0, st>>>(p->keys, n, p->tile_cnt, n_pos, T, p->thr, p->prec, p->rec, p->tps,
                                           p->fps, p->state);
  SRB_CUDA_OK(cudaGetLastError());
  note_launch(1);
  if (int rc = read_state(p, st)) return rc;
  const unsigned long long bk = p->h_state->best;
  const long long bi = static_cast<long long>(0xFFFFFFFFull - (bk & 0xFFFFFFFFull));
  SRB_REQUIRE(bk != 0 && bi >= 0 && bi < T, "samroad_prc_compute: internal error (no best point)");
  float v[3];
  SRB_CUDA_OK(cudaMemcpyAsync(&v[0], p->thr + bi, sizeof(float), cudaMemcpyDeviceToHost, st));
  SRB_CUDA_OK(cudaMemcpyAsync(&v[1], p->prec + bi, sizeof(float), cudaMemcpyDeviceToHost, st));
  SRB_CUDA_OK(cudaMemcpyAsync(&v[2], p->rec + bi, sizeof(float), cudaMemcpyDeviceToHost, st));
  SRB_CUDA_OK(cudaStreamSynchronize(st));
  const uint32_t fbits = static_cast<uint32_t>(bk >> 32);
  float f1;
  memcpy(&f1, &fbits, sizeof(f1));
  best[0] = v[0];
  best[1] = v[1];
  best[2] = v[2];
  best[3] = fbits == 0xFFFFFFFFu ? NAN : f1;
  counts[0] = n;
  counts[1] = n_pos;
  counts[2] = T;
  counts[3] = bi;
  p->T = T;
  return 0;
}

extern "C" int samroad_prc_read_curve(samroad_prc_t p, float* thresholds, float* precision, float* recall,
                                      int64_t* tps, int64_t* fps, void* stream) {
  SRB_REQUIRE(p != nullptr, "samroad_prc_read_curve: null handle");
  SRB_REQUIRE(p->T >= 0, "samroad_prc_read_curve: no curve (call samroad_prc_compute successfully first)");
  SRB_CUDA_OK(cudaSetDevice(p->device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const size_t T = static_cast<size_t>(p->T);
  const cudaMemcpyKind k = cudaMemcpyDefault;
  if (thresholds) SRB_CUDA_OK(cudaMemcpyAsync(thresholds, p->thr, sizeof(float) * T, k, st));
  if (precision) SRB_CUDA_OK(cudaMemcpyAsync(precision, p->prec, sizeof(float) * (T + 1), k, st));
  if (recall) SRB_CUDA_OK(cudaMemcpyAsync(recall, p->rec, sizeof(float) * (T + 1), k, st));
  if (tps) SRB_CUDA_OK(cudaMemcpyAsync(tps, p->tps, sizeof(int64_t) * T, k, st));
  if (fps) SRB_CUDA_OK(cudaMemcpyAsync(fps, p->fps, sizeof(int64_t) * T, k, st));
  return 0;
}
