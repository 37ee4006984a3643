// sam_road_b200 :: metrics.cu -- exact binary precision-recall curves for threshold search, and the
// losses and metrics of the validation loop (second half of the file, DESIGN.md §11).
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

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>

#include "common.cuh"
#include "loss_terms.cuh"
#include "ops.h"

using namespace srb;

namespace {

// Refusal bookkeeping shared by the accumulators: an update in flight raises flag bits; its commit either
// accepts it or counts it as refused (the first one in detail) until a synchronising call reports it.
struct Refusals {
  unsigned int flags;             // kBad* bits of the update in flight
  unsigned long long first_bad;   // smallest offending element index of the update in flight
  unsigned int sticky_count;      // refused updates not yet reported
  unsigned int sticky_flags;      // union of their kBad* bits
  unsigned long long sticky_bad;  // offending element of the first of them
  long long sticky_update;        // serial number of the first of them (counted from the last reset)
};

// Device-side state of one precision-recall accumulator.  `staged` runs ahead of `committed` while an
// update appends; the commit kernel keeps or drops the update's entries as a whole.
struct PrcState {
  unsigned long long committed;   // entries accepted so far
  unsigned long long staged;      // committed + entries of the update in flight
  Refusals ref;
  unsigned long long best;        // compute: argmax key, see best_key()
};

constexpr unsigned kBadPred = 1u, kBadTarget = 2u;
const char* const kPrcBadText[] = {" a prediction is NaN or outside [0, 1]",
                                   " a target is not 0 or 1 after truncation to int32"};

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

__device__ __forceinline__ void refusal_note(Refusals* r, unsigned flag, unsigned long long i) {
  atomicOr(&r->flags, flag);
  atomicMin(&r->first_bad, i);
}

__device__ __forceinline__ void refusal_begin(Refusals* r) {
  r->flags = 0;
  r->first_bad = ~0ull;
}

// true: the update in flight is accepted.  Otherwise it is counted as refused.  Single thread.
__device__ __forceinline__ bool refusal_commit(Refusals* r, long long serial) {
  if (r->flags == 0) return true;
  if (r->sticky_count == 0) {
    r->sticky_bad = r->first_bad;
    r->sticky_update = serial;
  }
  ++r->sticky_count;
  r->sticky_flags |= r->flags;
  return false;
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
      refusal_note(&st->ref, (pred_ok ? 0u : kBadPred) | (tgt_ok ? 0u : kBadTarget),
                   static_cast<unsigned long long>(i));
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
    if (!keep) refusal_note(&st->ref, kBadPred, static_cast<unsigned long long>(i));
  }
  append_key(keep, key, keys, st);
}

__global__ void prc_begin_kernel(PrcState* st) {
  st->staged = st->committed;
  refusal_begin(&st->ref);
}

// Keeps the update's entries, or drops all of them and counts the refusal (the first one in detail) until a
// synchronising call reports it.
__global__ void prc_commit_kernel(PrcState* st, long long serial) {
  if (refusal_commit(&st->ref, serial)) st->committed = st->staged;
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

// `s` is a synchronised host copy of the device bookkeeping `dev`.  Fails with code 3 while refused
// updates are unreported: it reports them all (their number, the first in detail, the text of every
// flag bit raised) and clears the count, so no later call can succeed past an unreported refusal.
int report_refusals(const Refusals& s, Refusals* dev, const char* what, const char* const* bad_text, int n_bad,
                    cudaStream_t st) {
  if (s.sticky_count == 0) return 0;
  SRB_CUDA_OK(cudaMemsetAsync(&dev->sticky_count, 0, sizeof(unsigned int), st));
  SRB_CUDA_OK(cudaMemsetAsync(&dev->sticky_flags, 0, sizeof(unsigned int), st));
  SRB_CUDA_OK(cudaStreamSynchronize(st));
  char why[512] = "";
  for (int b = 0; b < n_bad; ++b)
    if (s.sticky_flags & (1u << b)) strncat(why, bad_text[b], sizeof(why) - strlen(why) - 1);
  set_last_error("%s: %u update(s) since the last report were refused and added nothing; the first, "
                 "update #%lld since the last reset, at element %llu:%s",
                 what, s.sticky_count, s.sticky_update, s.sticky_bad, why);
  return 3;
}

// Synchronises and reports refused updates (report_refusals).  On success *committed holds the number of
// accepted entries.
int take_refusals(samroad_prc_ctx* p, const char* what, long long* committed, cudaStream_t st) {
  if (int rc = read_state(p, st)) return rc;
  const PrcState s = *p->h_state;
  p->reserved = s.committed;
  *committed = static_cast<long long>(s.committed);
  return report_refusals(s.ref, &p->state->ref, what, kPrcBadText, 2, st);
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

// =================================================================================================
// Validation: the losses, IoUs and F1 of SAMRoad.validation_step / on_validation_epoch_end (reference
// model.py:349-359, 547-600).  One update is one validation step: a grid-stride pass over the pixels (both
// mask channels), a pass over the pair slots, then one block that reduces the per-block partials in a fixed
// order, writes the step's (mask_loss, topo_loss, loss) and commits the step to the epoch state.  Sums of
// the float32 loss terms are fp64, counts are integers, so the result does not depend on scheduling.
// =================================================================================================
namespace {

constexpr unsigned kBadMaskTarget = 1u, kBadScore = 2u, kBadPairByte = 4u;
const char* const kValBadText[] = {" a mask target is not exactly 0.0 or 1.0",
                                   " a counted score is NaN or outside [0, 1]",
                                   " a connected or valid byte is not 0 or 1"};
constexpr int kValCounts = 11;      // keypoint tp fp fn tn, road tp fp fn tn, topology tp fp fn
constexpr int kValBlocksPerSm = 4;  // blocks per SM of each pass (grid-stride beyond that)

struct ValState {
  double loss_wsum[3];              // Σ f64(step value) · B over the accepted steps
  long long steps, samples;         // accepted steps, Σ B
  long long counts[kValCounts];
  Refusals ref;
};

// One block's share of a step.  Mask pass: Σ terms of both channels; tp, fp, fn of keypoint then road.
// Pair pass: Σ terms over valid slots; n_valid, tp, fp, fn.
struct ValPartial {
  double sum;
  unsigned long long c[6];
};

// Block-wide sum of a partial in a fixed order; the result is valid in thread 0.
template <int kN>
__device__ __forceinline__ void block_sum_partial(double& sum, unsigned long long (&c)[kN], ValPartial* sh /*[8]*/) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    sum += __shfl_down_sync(0xffffffffu, sum, o);
#pragma unroll
    for (int k = 0; k < kN; ++k) c[k] += __shfl_down_sync(0xffffffffu, c[k], o);
  }
  if (lane == 0) {
    sh[wid].sum = sum;
#pragma unroll
    for (int k = 0; k < kN; ++k) sh[wid].c[k] = c[k];
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < static_cast<int>(blockDim.x >> 5); ++w) {
      sum += sh[w].sum;
#pragma unroll
      for (int k = 0; k < kN; ++k) c[k] += sh[w].c[k];
    }
  }
}

__device__ __forceinline__ void note_bad(unsigned& bad, unsigned long long& first, unsigned flag,
                                         unsigned long long i) {
  bad |= flag;
  first = i < first ? i : first;
}

// Pixels: logits / scores are [npix] float2 (the two channels of [B,P,P,2]), kp / road [npix] float.
// Element index of a refusal: pixel * 2 + channel.
template <bool kFocal>
__global__ void __launch_bounds__(256) val_mask_kernel(const float2* __restrict__ logits,
                                                       const float2* __restrict__ scores,
                                                       const float* __restrict__ kp, const float* __restrict__ road,
                                                       long long npix, ValPartial* __restrict__ part,
                                                       Refusals* __restrict__ ref) {
  __shared__ ValPartial sh[8];
  double sum = 0.0;
  unsigned c[6] = {0, 0, 0, 0, 0, 0};
  unsigned bad = 0;
  unsigned long long first = ~0ull;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < npix; i += stride) {
    const float2 x = logits[i], s = scores[i];
    const float y[2] = {kp[i], road[i]};
    const float xs[2] = {x.x, x.y}, ss[2] = {s.x, s.y};
#pragma unroll
    for (int ch = 0; ch < 2; ++ch) {
      const unsigned long long e = static_cast<unsigned long long>(i) * 2 + ch;
      if (!(y[ch] == 0.0f || y[ch] == 1.0f)) note_bad(bad, first, kBadMaskTarget, e);
      if (!(ss[ch] >= 0.0f && ss[ch] <= 1.0f)) note_bad(bad, first, kBadScore, e);
      sum += static_cast<double>(kFocal ? focal_term(xs[ch], y[ch]) : bce_term(xs[ch], y[ch]));
      const bool pred = ss[ch] > 0.5f, lab = y[ch] == 1.0f;
      c[3 * ch + 0] += pred && lab;
      c[3 * ch + 1] += pred && !lab;
      c[3 * ch + 2] += !pred && lab;
    }
  }
  if (bad) refusal_note(ref, bad, first);
  unsigned long long cc[6];
#pragma unroll
  for (int k = 0; k < 6; ++k) cc[k] = c[k];
  block_sum_partial<6>(sum, cc, sh);
  if (threadIdx.x == 0) {
    part[blockIdx.x].sum = sum;
#pragma unroll
    for (int k = 0; k < 6; ++k) part[blockIdx.x].c[k] = cc[k];
  }
}

// Pair slots [n]: topology BCE over the valid ones (label = connected), counts of the valid ones.  An
// invalid slot is skipped, which equals the reference's `* valid` because its logit is finite.  Element
// index of a refusal: elem_base + slot.
__global__ void __launch_bounds__(256) val_pair_kernel(const float* __restrict__ logits,
                                                       const float* __restrict__ scores,
                                                       const uint8_t* __restrict__ connected,
                                                       const uint8_t* __restrict__ valid, long long n,
                                                       unsigned long long elem_base, ValPartial* __restrict__ part,
                                                       Refusals* __restrict__ ref) {
  __shared__ ValPartial sh[8];
  double sum = 0.0;
  unsigned c[4] = {0, 0, 0, 0};   // n_valid, tp, fp, fn
  unsigned bad = 0;
  unsigned long long first = ~0ull;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
    const unsigned v = valid[i], lab = connected[i];
    const unsigned long long e = elem_base + static_cast<unsigned long long>(i);
    if (v > 1u || lab > 1u) note_bad(bad, first, kBadPairByte, e);
    if (v == 1u) {
      const float s = scores[i];
      if (!(s >= 0.0f && s <= 1.0f)) note_bad(bad, first, kBadScore, e);
      sum += static_cast<double>(bce_term(logits[i], lab == 1u ? 1.0f : 0.0f));
      const bool pred = s > 0.5f, pos = lab == 1u;
      c[0] += 1;
      c[1] += pred && pos;
      c[2] += pred && !pos;
      c[3] += !pred && pos;
    }
  }
  if (bad) refusal_note(ref, bad, first);
  unsigned long long cc[4] = {c[0], c[1], c[2], c[3]};
  block_sum_partial<4>(sum, cc, sh);
  if (threadIdx.x == 0) {
    part[blockIdx.x].sum = sum;
    part[blockIdx.x].c[0] = cc[0];
    part[blockIdx.x].c[1] = cc[1];
    part[blockIdx.x].c[2] = cc[2];
    part[blockIdx.x].c[3] = cc[3];
    part[blockIdx.x].c[4] = part[blockIdx.x].c[5] = 0;
  }
}

// Fixed-order sum of g partials by the whole block (result in thread 0).
__device__ void reduce_partials(const ValPartial* __restrict__ part, int g, ValPartial* sh, double& sum,
                                unsigned long long (&c)[6]) {
  sum = 0.0;
#pragma unroll
  for (int k = 0; k < 6; ++k) c[k] = 0;
  for (int b = threadIdx.x; b < g; b += blockDim.x) {
    sum += part[b].sum;
#pragma unroll
    for (int k = 0; k < 6; ++k) c[k] += part[b].c[k];
  }
  block_sum_partial<6>(sum, c, sh);
  __syncthreads();   // sh is reused by the next call
}

// One 256-thread block: the step's three values into out, then the step is committed to the epoch state or
// refused as a whole.  Leaves the refusal flags cleared for the next step.
__global__ void __launch_bounds__(256) val_finish_kernel(const ValPartial* __restrict__ mask_part, int g_mask,
                                                         const ValPartial* __restrict__ pair_part, int g_pair,
                                                         long long npix, int B, float* __restrict__ out,
                                                         ValState* __restrict__ st, long long serial) {
  __shared__ ValPartial sh[8];
  double msum, psum;
  unsigned long long mc[6], pc[6];
  reduce_partials(mask_part, g_mask, sh, msum, mc);
  reduce_partials(pair_part, g_pair, sh, psum, pc);
  if (threadIdx.x != 0) return;
  if (!refusal_commit(&st->ref, serial)) {
    out[0] = out[1] = out[2] = __int_as_float(0x7fc00000);
  } else {
    const float mask_loss = __double2float_rn(msum / static_cast<double>(2 * npix));
    const float topo_loss = pc[0] ? __double2float_rn(psum / static_cast<double>(pc[0])) : __int_as_float(0x7fc00000);
    const float loss = __fadd_rn(mask_loss, topo_loss);
    const float v[3] = {mask_loss, topo_loss, loss};
    for (int k = 0; k < 3; ++k) {
      out[k] = v[k];
      st->loss_wsum[k] = __dadd_rn(st->loss_wsum[k], __dmul_rn(static_cast<double>(v[k]), static_cast<double>(B)));
    }
    st->steps += 1;
    st->samples += B;
    for (int ch = 0; ch < 2; ++ch) {
      const long long tp = mc[3 * ch], fp = mc[3 * ch + 1], fn = mc[3 * ch + 2];
      st->counts[4 * ch + 0] += tp;
      st->counts[4 * ch + 1] += fp;
      st->counts[4 * ch + 2] += fn;
      st->counts[4 * ch + 3] += npix - tp - fp - fn;
    }
    st->counts[8] += pc[1];
    st->counts[9] += pc[2];
    st->counts[10] += pc[3];
  }
  refusal_begin(&st->ref);
}

__global__ void val_reset_kernel(ValState* st) {
  ValState z = {};
  z.ref.first_bad = ~0ull;
  *st = z;
}

}  // namespace

struct samroad_val_ctx {
  int device = 0;
  int max_blocks = 0;              // per pass
  ValState* state = nullptr;       // device
  ValPartial* part = nullptr;      // device, 2 * max_blocks: mask pass, then pair pass
  ValState* h_state = nullptr;     // pinned read-back
  long long n_updates = 0;         // updates since the last reset

  ~samroad_val_ctx() {
    if (state) cudaFree(state);
    if (part) cudaFree(part);
    if (h_state) cudaFreeHost(h_state);
  }
};

extern "C" int samroad_val_create(int device, samroad_val_t* out) {
  SRB_REQUIRE(out != nullptr, "samroad_val_create: null argument");
  int ndev = 0;
  SRB_CUDA_OK(cudaGetDeviceCount(&ndev));
  SRB_REQUIRE(ndev > 0, "no CUDA device: libsamroad_b200 has no CPU fallback");
  SRB_REQUIRE(device >= 0 && device < ndev, "device %d out of range (0..%d)", device, ndev - 1);
  SRB_CUDA_OK(cudaSetDevice(device));
  samroad_val_ctx* v = new samroad_val_ctx();
  v->device = device;
  v->max_blocks = kValBlocksPerSm * device_sm_count();
  if (cudaMalloc(&v->state, sizeof(ValState)) != cudaSuccess ||
      cudaMalloc(&v->part, sizeof(ValPartial) * 2 * v->max_blocks) != cudaSuccess ||
      cudaMallocHost(&v->h_state, sizeof(ValState)) != cudaSuccess) {
    cudaGetLastError();
    delete v;
    set_last_error("samroad_val_create: device or pinned allocation failed");
    return 1;
  }
  val_reset_kernel<<<1, 1>>>(v->state);
  if (cudaGetLastError() != cudaSuccess || cudaDeviceSynchronize() != cudaSuccess) {
    delete v;
    set_last_error("samroad_val_create: initialising the state failed");
    return 1;
  }
  note_launch(1);
  *out = v;
  return 0;
}

extern "C" int samroad_val_destroy(samroad_val_t v) {
  if (!v) return 0;
  cudaSetDevice(v->device);
  cudaDeviceSynchronize();
  delete v;
  return 0;
}

extern "C" int samroad_val_reset(samroad_val_t v, void* stream) {
  SRB_REQUIRE(v != nullptr, "samroad_val_reset: null handle");
  SRB_CUDA_OK(cudaSetDevice(v->device));
  val_reset_kernel<<<1, 1, 0, static_cast<cudaStream_t>(stream)>>>(v->state);
  SRB_CUDA_OK(cudaGetLastError());
  note_launch(1);
  v->n_updates = 0;
  return 0;
}

extern "C" int samroad_val_update(samroad_val_t v, const float* mask_logits, const float* mask_scores,
                                  const float* keypoint_mask, const float* road_mask, const float* topo_logits,
                                  const float* topo_scores, const uint8_t* connected, const uint8_t* valid, int B,
                                  int P, int Ns, int Np, int loss_kind, float* out, void* stream) {
  SRB_REQUIRE(v != nullptr, "samroad_val_update: null handle");
  SRB_REQUIRE(B >= 1 && P >= 1 && Ns >= 0 && Np >= 0, "samroad_val_update: B=%d, P=%d, Ns=%d, Np=%d", B, P, Ns,
              Np);
  SRB_REQUIRE(loss_kind == SAMROAD_LOSS_BCE || loss_kind == SAMROAD_LOSS_FOCAL,
              "samroad_val_update: loss kind %d (SAMROAD_LOSS_BCE or SAMROAD_LOSS_FOCAL)", loss_kind);
  const long long n_pairs = static_cast<long long>(B) * Ns * Np;
  SRB_REQUIRE(mask_logits && mask_scores && keypoint_mask && road_mask && out, "samroad_val_update: null argument");
  SRB_REQUIRE(n_pairs == 0 || (topo_logits && topo_scores && connected && valid),
              "samroad_val_update: null topology argument");
  SRB_REQUIRE(reinterpret_cast<uintptr_t>(mask_logits) % 8 == 0 && reinterpret_cast<uintptr_t>(mask_scores) % 8 == 0,
              "samroad_val_update: mask logits and scores must be 8-byte aligned ([B,P,P,2] float32)");
  SRB_CUDA_OK(cudaSetDevice(v->device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long long npix = static_cast<long long>(B) * P * P;
  const int g_mask = static_cast<int>(std::min<long long>(grid_for(npix, 256), v->max_blocks));
  const int g_pair = static_cast<int>(std::min<long long>(grid_for(n_pairs, 256), v->max_blocks));
  ValPartial* pair_part = v->part + v->max_blocks;
  if (loss_kind == SAMROAD_LOSS_FOCAL)
    val_mask_kernel<true><<<g_mask, 256, 0, st>>>(reinterpret_cast<const float2*>(mask_logits),
                                                  reinterpret_cast<const float2*>(mask_scores), keypoint_mask,
                                                  road_mask, npix, v->part, &v->state->ref);
  else
    val_mask_kernel<false><<<g_mask, 256, 0, st>>>(reinterpret_cast<const float2*>(mask_logits),
                                                   reinterpret_cast<const float2*>(mask_scores), keypoint_mask,
                                                   road_mask, npix, v->part, &v->state->ref);
  if (g_pair > 0)
    val_pair_kernel<<<g_pair, 256, 0, st>>>(topo_logits, topo_scores, connected, valid, n_pairs,
                                            static_cast<unsigned long long>(2 * npix), pair_part, &v->state->ref);
  val_finish_kernel<<<1, 256, 0, st>>>(v->part, g_mask, pair_part, g_pair, npix, B, out, v->state, v->n_updates);
  SRB_CUDA_OK(cudaGetLastError());
  note_launch(g_pair > 0 ? 3 : 2);
  ++v->n_updates;
  return 0;
}

extern "C" int samroad_val_read(samroad_val_t v, int64_t* counts, float* means, int64_t* totals, void* stream) {
  SRB_REQUIRE(v != nullptr && counts && means && totals, "samroad_val_read: null argument");
  SRB_CUDA_OK(cudaSetDevice(v->device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  SRB_CUDA_OK(cudaMemcpyAsync(v->h_state, v->state, sizeof(ValState), cudaMemcpyDeviceToHost, st));
  SRB_CUDA_OK(cudaStreamSynchronize(st));
  const ValState s = *v->h_state;
  if (int rc = report_refusals(s.ref, &v->state->ref, "samroad_val_read", kValBadText, 3, st)) return rc;
  for (int k = 0; k < kValCounts; ++k) counts[k] = s.counts[k];
  for (int k = 0; k < 3; ++k)
    means[k] = s.samples ? static_cast<float>(s.loss_wsum[k] / static_cast<double>(s.samples)) : NAN;
  totals[0] = s.steps;
  totals[1] = s.samples;
  return 0;
}
