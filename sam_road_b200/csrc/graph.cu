// sam_road_b200 :: graph.cu -- the middle and the tail of inferencer.infer_one_img on the device.
//
// The reference runs three pieces of host code between / after its two model passes (SURVEY.md §8f
// rows 1-2); at GPU tile rates they are the critical path of a scene, so they live here:
//   * keypoint extraction   graph_extraction.extract_graph_points  graph_extraction.py:24-28,130-139
//                           graph_utils.nms_points                 graph_utils.py:572-591
//   * pair-query build      inferencer.py:126-197 (rtree box query + KDTree kNN per tile)
//   * edge aggregation      inferencer.py:206-230 (dict of float32 sums in (tile, sample, pair) order)
// All of it is integer / index work plus one ordered fp32 sum, so the results are bit-exact
// restatements, not approximations.  Two third-party orderings the reference inherits are
// implementation-defined and are made explicit here (DESIGN.md §9):
//   - np.argsort (unstable introsort / AVX-512 sort) decides the visiting order of equal-score
//     candidates in the greedy NMS.  `samroad_extract_graph_points` takes an optional host callback
//     that supplies NumPy's permutation (bit-exact with the reference on that host); without it the
//     device sorts with the order np.argsort(kind='stable')[::-1] would give.
//   - scipy's cKDTree returns equidistant neighbours in traversal order; here ties are ordered by
//     point index.
//
// Everything is HBM/L2-latency-bound integer work on arrays of at most a few MB (the scene masks are
// 4 MB each at 2048^2); the kernels are sized for parallelism and ordered compaction, not for the
// tensor cores.
#include "../../include/samroad_b200.h"

#include <cuda_runtime.h>

#include <chrono>
#include <climits>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <memory>
#include <thread>
#include <vector>

#include "common.cuh"
#include "ops.h"
#include "scan.cuh"

using namespace srb;

namespace {

// Grows a scratch buffer to at least `bytes`, with 25 % + 256 B of slack.  Work queued on the caller's
// stream may still read the old block, so the device is synchronised before it is replaced.
int grow(DeviceBuffer& b, size_t bytes) {
  if (bytes <= b.capacity()) return 0;
  if (b.get()) SRB_CUDA_OK(cudaDeviceSynchronize());
  return b.reserve(bytes + bytes / 4 + 256, "samroad_graph");
}

// Every count written on the device and read back by the host, one field each.  The entry points that
// use them clear them all on entry.
struct Counters {
  int cand[2];       // candidates per mask
  int order_err;     // visiting order: 1 = host index out of range, 2 = not non-increasing
  int n_mortal;      // entries of an NMS pass that can be suppressed
  int survivors;     // entries an NMS pass keeps
  int bad_score;     // aggregation: a score outside [0, 1]
  int n_edges;
  int max_deg;       // most points within the neighbour radius of one point
  int nnz;           // (src, tgt) slots of the aggregation
};

constexpr size_t kPinBytes = 256;

}  // namespace

struct samroad_graph_ctx {
  int device = 0;
  DeviceBuffer counters;                  // one Counters
  // keypoint extraction
  DeviceBuffer blk;                       // compaction: counts of the chunks, scanned in place, + scan scratch
  DeviceBuffer cand_pix[2], cand_score[2]; // candidates of the two masks, np.where order
  DeviceBuffer order, sorted_pix, immune; // visiting order of one NMS pass
  DeviceBuffer list[3];                   // kept pixels of passes 1 / 2 / 3, visiting order
  DeviceBuffer cand3, cls3;               // pass 3 input: concatenation + class (1 = keypoint mask)
  DeviceBuffer cell;                      // scene-sized rank/state image
  DeviceBuffer tile_und, round_cnt;       // NMS rounds
  DeviceBuffer ghist;                     // counting sort: histogram + scan scratch (host order: its permutation)
  PinnedBuffer h_pin;                     // kPinBytes of pinned host memory for small read-backs
  // pair queries
  DeviceBuffer pts32, t_cnt, t_off, members, nbr, tile_xy;
  std::vector<int> h_cnt, h_off;
  int N = 0, n_tiles = 0, P = 0;
  long total = 0;
  int d2lt = 0;                           // neighbours satisfy d^2 < d2lt
  int max_nbr = 0;                        // K the plan was made for (fill / aggregate take K <= max_nbr)
  int nbr_stride = 16;                    // row length of nbr: 16 for max_nbr <= 16, else 32
  // aggregation
  DeviceBuffer adj_off, adj_src, adj_tgt, adj_sum, adj_cnt, adj_first, eflags, tile_soff;
};

namespace {

constexpr uint32_t kNone = 0xFFFFFFFFu;
constexpr uint32_t kUndecided = 0u, kKept = 1u, kSuppressed = 2u;

// ---------------------------------------------------------------------------------------------------
// ordered stream compaction: count per 1024-element chunk -> exclusive scan of the counts -> fill.
// F provides   __device__ bool pred(int i) const;   __device__ void emit(int i, int pos) const;
// Output positions follow the input order (what np.where / boolean indexing produce).
// ---------------------------------------------------------------------------------------------------
constexpr int kChunk = 1024;

template <class F>
__global__ void __launch_bounds__(256) compact_count_kernel(F f, int n, int* __restrict__ blk_cnt) {
  __shared__ int sw[33];
  const int base = blockIdx.x * kChunk + threadIdx.x * 4;
  int c = 0;
#pragma unroll
  for (int e = 0; e < 4; ++e)
    if (base + e < n && f.pred(base + e)) ++c;
  int total;
  block_exclusive_scan(c, sw, total);
  if (threadIdx.x == 0) blk_cnt[blockIdx.x] = total;
}

template <class F>
__global__ void __launch_bounds__(256) compact_fill_kernel(F f, int n, const int* __restrict__ blk_off) {
  __shared__ int sw[33];
  const int base = blockIdx.x * kChunk + threadIdx.x * 4;
  bool p[4];
  int c = 0;
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    p[e] = base + e < n && f.pred(base + e);
    c += p[e] ? 1 : 0;
  }
  int total;
  int pos = blk_off[blockIdx.x] + block_exclusive_scan(c, sw, total);
#pragma unroll
  for (int e = 0; e < 4; ++e)
    if (p[e]) f.emit(base + e, pos++);
}

// host driver: returns the number of emitted elements in *n_out_dev (device int) -- no sync
template <class F>
int compact(samroad_graph_ctx* g, const F& f, int n, int* n_out_dev, cudaStream_t st) {
  const int nblk = blocks_for(n, kChunk);
  if (nblk == 0) {
    SRB_CUDA_OK(cudaMemsetAsync(n_out_dev, 0, sizeof(int), st));
    return 0;
  }
  if (int rc = grow(g->blk, sizeof(int) * (nblk + scan_scratch_elems(nblk)))) return rc;
  int* blk = g->blk.as<int>();
  SRB_LAUNCH(compact_count_kernel<F>, nblk, 256, 0, st, f, n, blk);
  if (int rc = exclusive_scan(blk, blk, nblk, n_out_dev, blk + nblk, st)) return rc;
  SRB_LAUNCH(compact_fill_kernel<F>, nblk, 256, 0, st, f, n, blk);
  return 0;
}

// ---- predicates ---------------------------------------------------------------------------------------
struct MaskCand {   // graph_extraction.py:24-28: np.where(mask > thr) in row-major order + mask[mask > thr]
  const uint8_t* mask;
  int t_int;        // mask > thr  <=>  mask >= t_int
  int32_t* pix;
  uint8_t* score;
  __device__ bool pred(int i) const { return static_cast<int>(mask[i]) >= t_int; }
  __device__ void emit(int i, int pos) const { pix[pos] = i; score[pos] = mask[i]; }
};

struct KeptByRank {  // sorted_points[kept] (graph_utils.py:588-591): survivors in visiting order
  const uint32_t* cell;
  const int32_t* pix;   // visiting order
  int32_t* out;
  __device__ bool pred(int i) const { return cell[pix[i]] == ((static_cast<uint32_t>(i) << 2) | kKept); }
  __device__ void emit(int i, int pos) const { out[pos] = pix[i]; }
};

struct EdgeFlag {    // edges in dict-insertion (first occurrence) order, inferencer.py:223-229
  const int32_t* flags;
  const int32_t* adj_src;
  const int32_t* adj_tgt;
  int64_t* out;
  int cap;
  __device__ bool pred(int i) const { return flags[i] >= 0; }
  __device__ void emit(int i, int pos) const {
    if (pos < cap) {
      const int s = flags[i];
      out[2 * static_cast<size_t>(pos)] = adj_src[s];
      out[2 * static_cast<size_t>(pos) + 1] = adj_tgt[s];
    }
  }
};

// device visiting order:  np.argsort(scores, kind='stable')[::-1]  for uint8 scores (descending score,
// equal scores in descending candidate index): one stable counting-sort pass on the score, ranks reversed.
struct ReversedOrder {
  const uint8_t* score;
  int n;
  int32_t* order;
  __device__ uint32_t key(long long i) const { return __ldg(score + i); }
  __device__ unsigned digit(uint32_t k) const { return k; }
  __device__ void emit(long long i, uint32_t, uint32_t pos) const { order[n - 1 - pos] = static_cast<int32_t>(i); }
};

// host permutation (ascending argsort, int64) -> visiting order (its reverse, int32)
__global__ void order_from_host_kernel(const int64_t* __restrict__ asc, int n, int32_t* __restrict__ order,
                                       int* __restrict__ err) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int64_t v = asc[n - 1 - i];
  if (v < 0 || v >= n) { atomicOr(err, 1); order[i] = 0; return; }
  order[i] = static_cast<int32_t>(v);
}

// sorted_points = points[order]; immune = score > 1.0 (never suppressed, graph_utils.py:573,585).
// Also checks that the order really is non-increasing in score (a bad callback would silently change
// the greedy result) and counts the entries that can be suppressed at all.  In pass 3 `score` is the
// class (1 or 0), so nothing is immune there.
__global__ void gather_sorted_kernel(const int32_t* __restrict__ pix, const uint8_t* __restrict__ score,
                                     const int32_t* __restrict__ order, int n,
                                     int32_t* __restrict__ sorted_pix, uint8_t* __restrict__ immune,
                                     int* __restrict__ n_mortal, int* __restrict__ err) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int o = order[i];
  const uint8_t s = score[o];
  sorted_pix[i] = pix[o];
  immune[i] = s >= 2 ? 1 : 0;              // uint8 score > 1.0
  if (s < 2) atomicAdd(n_mortal, 1);
  if (i > 0 && score[order[i - 1]] < s) atomicOr(err, 2);
}

// ---------------------------------------------------------------------------------------------------
// Greedy radius NMS (graph_utils.py:572-591) as a fixed point on a scene-sized image.
//
// In descending-score visiting order a point is kept iff it is immune (score > 1) or no kept point
// visited earlier lies within the radius (inclusive, KDTree.query_ball_point).  Every candidate is a
// pixel, so the state lives in an image: cell = rank << 2 | state.  A pixel holding the same
// coordinates twice (pass 3: present in both masks) keeps the lower rank; the later copy is always
// suppressed by the earlier one or by whatever suppressed it.
//
// One round: every undecided pixel looks at its disc; a kept pixel of lower rank suppresses it, an
// undecided one of lower rank makes it wait, otherwise it is kept.  Decisions only ever use final
// states of lower ranks, so the fixed point is the sequential greedy result whatever the schedule.
// A CTA owns a 32x32 pixel tile, stages tile + halo in shared memory (odd row stride: the 32 lanes of
// a warp scan 32 different rows of one disc, conflict-free) and iterates locally until nothing in the
// tile changes; rounds repeat until no undecided pixel is left in the scene.
// ---------------------------------------------------------------------------------------------------
constexpr int kNmsTile = 32;       // pixels per CTA tile side (64 was measured: NMS 1.4 -> 2.4 ms, rounds 10 -> 6)
constexpr int kNmsMaxHalo = 32;

__global__ void cell_build_kernel(const int32_t* __restrict__ sorted_pix, const uint8_t* __restrict__ immune,
                                  int n, uint32_t* __restrict__ cell) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t st = (immune && immune[i]) ? kKept : kUndecided;
  atomicMin(&cell[sorted_pix[i]], (static_cast<uint32_t>(i) << 2) | st);
}

__global__ void __launch_bounds__(256)
nms_round_kernel(uint32_t* __restrict__ cell, int H, int W, int halo, int d2max,
                 int* __restrict__ tile_und, int* __restrict__ round_total) {
  extern __shared__ uint32_t smem_u32_[];
  const int tile_id = blockIdx.y * gridDim.x + blockIdx.x;
  if (tile_und[tile_id] == 0) return;
  const int S = kNmsTile + 2 * halo + 1;          // odd stride
  const int SH = kNmsTile + 2 * halo;
  volatile uint32_t* s = smem_u32_;               // [SH][S]
  int* wtab = reinterpret_cast<int*>(smem_u32_ + SH * S);         // [2*halo+1] half-widths
  unsigned short* list = reinterpret_cast<unsigned short*>(wtab + 2 * halo + 1);   // [kNmsTile^2]
  __shared__ int list_n, changed_any;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int gx0 = blockIdx.x * kNmsTile - halo, gy0 = blockIdx.y * kNmsTile - halo;
  for (int i = tid; i < SH * SH; i += 256) {
    const int ly = i / SH, lx = i - ly * SH;
    const int gx = gx0 + lx, gy = gy0 + ly;
    uint32_t v = kNone;
    if (gx >= 0 && gx < W && gy >= 0 && gy < H) v = cell[static_cast<size_t>(gy) * W + gx];
    s[ly * S + lx] = v;
  }
  for (int r = tid; r < 2 * halo + 1; r += 256) {
    const int dy = r - halo;
    const int rem = d2max - dy * dy;
    int w = -1;
    if (rem >= 0) {
      w = static_cast<int>(sqrtf(static_cast<float>(rem)));
      while ((w + 1) * (w + 1) <= rem) ++w;
      while (w * w > rem) --w;
    }
    wtab[r] = w;
  }
  __syncthreads();

  for (int iter = 0; iter < 64; ++iter) {
    if (tid == 0) { list_n = 0; changed_any = 0; }
    __syncthreads();
    for (int ly = warp; ly < kNmsTile; ly += 8) {
#pragma unroll
      for (int lx = lane; lx < kNmsTile; lx += 32) {
        const uint32_t v = s[(ly + halo) * S + lx + halo];
        if (v != kNone && (v & 3u) == kUndecided) {
          const int p = atomicAdd(&list_n, 1);
          list[p] = static_cast<unsigned short>(ly * kNmsTile + lx);
        }
      }
    }
    __syncthreads();
    const int cnt = list_n;
    if (cnt == 0) break;
    for (int c = warp; c < cnt; c += 8) {
      const int ly = list[c] / kNmsTile, lx = list[c] % kNmsTile;
      const uint32_t word = s[(ly + halo) * S + lx + halo];
      const uint32_t rp = word >> 2;
      bool sup = false, blk = false;
      for (int r = lane; r < 2 * halo + 1; r += 32) {
        const int w = wtab[r];
        if (w < 0) continue;
        const volatile uint32_t* row = s + (ly + r) * S + lx + halo;
        for (int dx = -w; dx <= w; ++dx) {
          const uint32_t qv = row[dx];
          if (qv != kNone && (qv >> 2) < rp) {
            const uint32_t qs = qv & 3u;
            sup |= qs == kKept;
            blk |= qs == kUndecided;
          }
        }
      }
      sup = __any_sync(0xffffffffu, sup);
      blk = __any_sync(0xffffffffu, blk);
      if (lane == 0) {
        if (sup) { s[(ly + halo) * S + lx + halo] = word | kSuppressed; changed_any = 1; }
        else if (!blk) { s[(ly + halo) * S + lx + halo] = word | kKept; changed_any = 1; }
      }
    }
    __syncthreads();
    if (!changed_any) break;
    __syncthreads();
  }
  // write back the decisions of this tile, count what is still open
  int open = 0;
  for (int ly = warp; ly < kNmsTile; ly += 8) {
#pragma unroll
    for (int lx = lane; lx < kNmsTile; lx += 32) {
      const int gx = blockIdx.x * kNmsTile + lx, gy = blockIdx.y * kNmsTile + ly;
      const uint32_t v = s[(ly + halo) * S + lx + halo];
      if (v != kNone && gx < W && gy < H) {
        if ((v & 3u) == kUndecided) ++open;
        else cell[static_cast<size_t>(gy) * W + gx] = v;
      }
    }
  }
  for (int o = 16; o > 0; o >>= 1) open += __shfl_xor_sync(0xffffffffu, open, o);
  __shared__ int open_tot;
  if (tid == 0) open_tot = 0;
  __syncthreads();
  if (lane == 0 && open) atomicAdd(&open_tot, open);
  __syncthreads();
  if (tid == 0) {
    tile_und[tile_id] = open_tot;
    if (open_tot) atomicAdd(round_total, open_tot);
  }
}

// radius too large for the shared-memory tile: same rule straight from global memory (slow, correct)
__global__ void __launch_bounds__(256)
nms_round_generic_kernel(uint32_t* __restrict__ cell, const int32_t* __restrict__ sorted_pix, int n, int H,
                         int W, int halo, int d2max, int* __restrict__ round_total) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int pix = sorted_pix[i];
  const uint32_t word = cell[pix];
  if (word != ((static_cast<uint32_t>(i) << 2) | kUndecided)) return;
  const int px = pix % W, py = pix / W;
  bool sup = false, blk = false;
  for (int dy = -halo; dy <= halo && !sup; ++dy) {
    const int y = py + dy;
    if (y < 0 || y >= H) continue;
    for (int dx = -halo; dx <= halo; ++dx) {
      const int x = px + dx;
      if (x < 0 || x >= W || dx * dx + dy * dy > d2max) continue;
      const uint32_t qv = *reinterpret_cast<volatile uint32_t*>(&cell[static_cast<size_t>(y) * W + x]);
      if (qv != kNone && (qv >> 2) < static_cast<uint32_t>(i)) {
        sup |= (qv & 3u) == kKept;
        blk |= (qv & 3u) == kUndecided;
      }
    }
  }
  if (sup) cell[pix] = word | kSuppressed;
  else if (!blk) cell[pix] = word | kKept;
  else atomicAdd(round_total, 1);
}

// pass 3 input = concat(kept0, kept1) and its class: the keypoint-mask entries score 1.0, the rest 0.0
// (graph_extraction.py:136-137)
__global__ void concat_kernel(const int32_t* __restrict__ a, int na, const int32_t* __restrict__ b, int nb,
                              int32_t* __restrict__ out, uint8_t* __restrict__ cls) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < na) { out[i] = a[i]; cls[i] = 1; }
  else if (i < na + nb) { out[i] = b[i - na]; cls[i] = 0; }
}

__global__ void pix_to_xy_kernel(const int32_t* __restrict__ pix, int n, int W, int64_t* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int p = pix[i];
  out[2 * static_cast<size_t>(i)] = p % W;        // x
  out[2 * static_cast<size_t>(i) + 1] = p / W;    // y
}

// read a small device object back (synchronises the stream)
template <typename T>
int read_back(samroad_graph_ctx* g, const T* dev, T* host, cudaStream_t st) {
  static_assert(sizeof(T) <= kPinBytes, "read-back larger than the pinned staging buffer");
  SRB_CUDA_OK(cudaMemcpyAsync(g->h_pin.get(), dev, sizeof(T), cudaMemcpyDeviceToHost, st));
  SRB_CUDA_OK(cudaStreamSynchronize(st));
  std::memcpy(host, g->h_pin.get(), sizeof(T));
  return 0;
}

// mask > thr for a uint8 mask and a real threshold  <=>  mask >= t
int thr_to_int(double thr) {
  if (!(thr >= 0.0)) return 0;         // negative (or NaN-safe default): every pixel qualifies
  if (thr >= 255.0) return 256;        // nothing qualifies
  return static_cast<int>(std::floor(thr)) + 1;
}

using clk = std::chrono::steady_clock;
int32_t us_since(clk::time_point t) {
  return static_cast<int32_t>(std::chrono::duration_cast<std::chrono::microseconds>(clk::now() - t).count());
}

// Visiting order from the host: the reverse of the callback's ascending argsort of the `n` device keys,
// which it sees as `key_dtype` (SAMROAD_U8, or SAMROAD_F64 holding the same values).  `pre_asc`, when
// given, is that argsort already made.  An index out of range sets bit 1 of *err.  Synchronises.
int host_order(samroad_graph_ctx* g, const uint8_t* key, int n, int key_dtype, samroad_argsort_fn cb, void* user,
               const std::vector<int64_t>* pre_asc, int32_t* order, int* err, cudaStream_t st) {
  std::vector<int64_t> own;
  if (!pre_asc) {
    std::vector<uint8_t> keys(n);
    SRB_CUDA_OK(cudaMemcpyAsync(keys.data(), key, n, cudaMemcpyDeviceToHost, st));
    SRB_CUDA_OK(cudaStreamSynchronize(st));
    own.resize(n);
    if (key_dtype == SAMROAD_F64) {
      const std::vector<double> keys64(keys.begin(), keys.end());
      SRB_REQUIRE(cb(keys64.data(), SAMROAD_F64, n, own.data(), user) == 0,
                  "argsort callback failed (float64 priorities)");
    } else {
      SRB_REQUIRE(cb(keys.data(), SAMROAD_U8, n, own.data(), user) == 0, "argsort callback failed (uint8 scores)");
    }
  }
  const std::vector<int64_t>& asc = pre_asc ? *pre_asc : own;
  if (int rc = grow(g->ghist, sizeof(int64_t) * n)) return rc;
  SRB_CUDA_OK(cudaMemcpyAsync(g->ghist.get(), asc.data(), sizeof(int64_t) * n, cudaMemcpyHostToDevice, st));
  SRB_LAUNCH(order_from_host_kernel, blocks_for(n, 256), 256, 0, st, g->ghist.as<int64_t>(), n, order, err);
  SRB_CUDA_OK(cudaStreamSynchronize(st));   // `asc` is pageable host memory: keep it alive until copied
  return 0;
}

// Visiting order on the device: np.argsort(key, kind='stable')[::-1] by the counting sort
int stable_order(samroad_graph_ctx* g, const uint8_t* key, int n, int32_t* order, cudaStream_t st) {
  const long long m = digit_hist_elems<1024>(n);
  if (int rc = grow(g->ghist, sizeof(uint32_t) * (m + scan_scratch_elems(m)))) return rc;
  uint32_t* hist = g->ghist.as<uint32_t>();
  return stable_digit_pass<1024>(ReversedOrder{key, n, order}, n, hist, hist + m, st);
}

struct PassStats {
  int kept = 0, rounds = 0;
  int32_t us_order = 0, us_nms = 0;    // host wall clock of the two halves, each ending on a synchronisation
};

// One greedy NMS pass (graph_utils.py:572-591) from candidates to survivors: visiting order -> gather
// and check -> fixed point -> compaction.  `key` holds one uint8 per candidate: the mask score in passes
// 1 and 2, the class in pass 3.  With a callback the host decides the order of equal keys (see
// host_order), without one the device sorts stably.  `what` names the pass in errors.  Returns the
// survivors (visiting order) in `out`.  Synchronises.
int nms_pass(samroad_graph_ctx* g, const int32_t* pix, const uint8_t* key, int n, int key_dtype,
             samroad_argsort_fn cb, void* user, const std::vector<int64_t>* pre_asc, const char* what, int H,
             int W, double radius, int32_t* out, PassStats* ps, cudaStream_t st) {
  *ps = PassStats{};
  if (n == 0) return 0;
  if (int rc = grow(g->order, sizeof(int32_t) * static_cast<size_t>(n))) return rc;
  if (int rc = grow(g->sorted_pix, sizeof(int32_t) * static_cast<size_t>(n))) return rc;
  if (int rc = grow(g->immune, static_cast<size_t>(n))) return rc;
  int32_t* order = g->order.as<int32_t>();
  int32_t* sorted_pix = g->sorted_pix.as<int32_t>();
  uint8_t* immune = g->immune.as<uint8_t>();
  Counters* ctr = g->counters.as<Counters>();
  clk::time_point t0 = clk::now();
  if (int rc = cb ? host_order(g, key, n, key_dtype, cb, user, pre_asc, order, &ctr->order_err, st)
                  : stable_order(g, key, n, order, st))
    return rc;
  SRB_CUDA_OK(cudaMemsetAsync(&ctr->n_mortal, 0, sizeof(int), st));
  SRB_LAUNCH(gather_sorted_kernel, blocks_for(n, 256), 256, 0, st, pix, key, order, n, sorted_pix, immune,
             &ctr->n_mortal, &ctr->order_err);
  Counters c;
  if (int rc = read_back(g, ctr, &c, st)) return rc;
  SRB_REQUIRE(c.order_err == 0, "argsort callback returned an invalid permutation (code %d) for %s", c.order_err,
              what);
  ps->us_order = us_since(t0);
  t0 = clk::now();
  if (c.n_mortal == 0) {        // every score > 1: nothing can be suppressed, the pass only reorders
    SRB_CUDA_OK(cudaMemcpyAsync(out, sorted_pix, sizeof(int32_t) * n, cudaMemcpyDeviceToDevice, st));
    ps->kept = n;
    ps->us_nms = us_since(t0);
    return 0;
  }
  SRB_REQUIRE(radius >= 0.0 && radius < 4096.0, "nms radius %.3f unsupported", radius);
  const double r2 = radius * radius;                    // KDTree compares squared distances
  const int d2max = static_cast<int>(std::floor(r2));   // d^2 <= r^2 on integer d^2
  const int halo = static_cast<int>(std::floor(radius));
  const size_t npx = static_cast<size_t>(H) * W;
  if (int rc = grow(g->cell, npx * 4)) return rc;
  uint32_t* cell = g->cell.as<uint32_t>();
  SRB_CUDA_OK(cudaMemsetAsync(cell, 0xFF, npx * 4, st));
  SRB_LAUNCH(cell_build_kernel, blocks_for(n, 256), 256, 0, st, sorted_pix, immune, n, cell);
  const int tx = (W + kNmsTile - 1) / kNmsTile, ty = (H + kNmsTile - 1) / kNmsTile;
  constexpr int kMaxRounds = 4096;
  if (int rc = grow(g->round_cnt, sizeof(int) * kMaxRounds)) return rc;
  if (int rc = grow(g->tile_und, sizeof(int) * tx * ty)) return rc;
  int* round_cnt = g->round_cnt.as<int>();
  SRB_CUDA_OK(cudaMemsetAsync(round_cnt, 0, sizeof(int) * kMaxRounds, st));
  SRB_CUDA_OK(cudaMemsetAsync(g->tile_und.get(), 0x01, sizeof(int) * tx * ty, st));
  const bool tiled = halo <= kNmsMaxHalo;
  const int SH = kNmsTile + 2 * halo;
  const size_t smem = tiled ? (static_cast<size_t>(SH) * (SH + 1) + 2 * halo + 1) * 4 + kNmsTile * kNmsTile * 2 : 0;
  if (tiled && smem > 48 * 1024) SRB_TRY(allow_dynamic_smem(nms_round_kernel, smem));
  int round = 0;
  while (true) {
    const int burst = round == 0 ? 2 : 4;
    for (int b = 0; b < burst && round < kMaxRounds; ++b, ++round) {
      if (tiled)
        SRB_LAUNCH(nms_round_kernel, dim3(tx, ty), 256, smem, st, cell, H, W, halo, d2max, g->tile_und.as<int>(),
                   round_cnt + round);
      else
        SRB_LAUNCH(nms_round_generic_kernel, blocks_for(n, 256), 256, 0, st, cell, sorted_pix, n, H, W, halo, d2max,
                   round_cnt + round);
    }
    int open = 0;
    if (int rc = read_back(g, round_cnt + round - 1, &open, st)) return rc;
    if (open == 0) break;
    SRB_REQUIRE(round < kMaxRounds, "greedy NMS did not converge in %d rounds (%d pixels open)", round, open);
  }
  ps->rounds = round;
  KeptByRank kb{cell, sorted_pix, out};
  if (int rc = compact(g, kb, n, &ctr->survivors, st)) return rc;
  if (int rc = read_back(g, &ctr->survivors, &ps->kept, st)) return rc;
  ps->us_nms = us_since(t0);
  return 0;
}

}  // namespace

// =================================================================================================
// lifetime
// =================================================================================================
extern "C" int samroad_graph_create(int device, samroad_graph_t* out) {
  SRB_REQUIRE(out != nullptr, "samroad_graph_create: null argument");
  if (int rc = open_device(device)) return rc;
  std::unique_ptr<samroad_graph_ctx> g(new samroad_graph_ctx());
  g->device = device;
  if (g->h_pin.reserve(kPinBytes, "samroad_graph_create")) return 1;
  if (int rc = grow(g->counters, sizeof(Counters))) return rc;
  *out = g.release();
  return 0;
}

extern "C" int samroad_graph_destroy(samroad_graph_t g) {
  if (!g) return 0;
  cudaSetDevice(g->device);
  cudaDeviceSynchronize();
  delete g;
  return 0;
}

// =================================================================================================
// keypoint extraction  (graph_extraction.py:130-139)
// =================================================================================================
extern "C" int samroad_extract_graph_points(samroad_graph_t g, const uint8_t* keypoint_mask,
                                            const uint8_t* road_mask, int H, int W, double itsc_thr255,
                                            double road_thr255, double itsc_radius, double road_radius,
                                            samroad_argsort_fn argsort, void* user, int64_t* points_xy,
                                            int cap, int* n_points, int32_t* stats, void* stream) {
  SRB_REQUIRE(g && keypoint_mask && road_mask && n_points, "samroad_extract_graph_points: null argument");
  SRB_REQUIRE(H > 0 && W > 0 && static_cast<long>(H) * W < (1L << 30),
              "samroad_extract_graph_points: scene %dx%d unsupported (needs H*W < 2^30)", H, W);
  SRB_CUDA_OK(cudaSetDevice(g->device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int npx = H * W;
  Counters* ctr = g->counters.as<Counters>();
  SRB_CUDA_OK(cudaMemsetAsync(ctr, 0, sizeof(Counters), st));
  const uint8_t* masks[2] = {keypoint_mask, road_mask};
  const double thr[2] = {itsc_thr255, road_thr255};
  const double radius[2] = {itsc_radius, road_radius};
  const clk::time_point t_begin = clk::now();

  // candidates of both masks (np.where order).  Worst case every pixel qualifies.
  for (int m = 0; m < 2; ++m) {
    if (int rc = grow(g->cand_pix[m], sizeof(int32_t) * static_cast<size_t>(npx))) return rc;
    if (int rc = grow(g->cand_score[m], static_cast<size_t>(npx))) return rc;
    MaskCand mc{masks[m], thr_to_int(thr[m]), g->cand_pix[m].as<int32_t>(), g->cand_score[m].as<uint8_t>()};
    if (int rc = compact(g, mc, npx, &ctr->cand[m], st)) return rc;
  }
  Counters c;
  if (int rc = read_back(g, ctr, &c, st)) return rc;
  const int n_cand[2] = {c.cand[0], c.cand[1]};
  const int32_t us_cand = us_since(t_begin);

  // Host permutations (NumPy tie order): when every candidate score is > 1 the first two passes only reorder,
  // so the sizes of the third pass are known now and the three argsorts can run side by side (np.argsort
  // releases the GIL): uint8 scores of the two masks, float64 priorities [1]*n0 + [0]*n1.
  std::vector<int64_t> pre_asc[3];
  bool have_pre = false;
  int32_t us_presort = 0;
  if (argsort && thr_to_int(thr[0]) >= 2 && thr_to_int(thr[1]) >= 2 && n_cand[0] + n_cand[1] > 0) {
    const clk::time_point t0 = clk::now();
    std::vector<uint8_t> keys[2];
    for (int m = 0; m < 2; ++m) {
      keys[m].resize(n_cand[m]);
      if (n_cand[m])
        SRB_CUDA_OK(cudaMemcpyAsync(keys[m].data(), g->cand_score[m].get(), n_cand[m], cudaMemcpyDeviceToHost, st));
    }
    SRB_CUDA_OK(cudaStreamSynchronize(st));
    const int n3p = n_cand[0] + n_cand[1];
    std::vector<double> pri(n3p);
    for (int i = 0; i < n3p; ++i) pri[i] = i < n_cand[0] ? 1.0 : 0.0;
    for (int m = 0; m < 2; ++m) pre_asc[m].resize(n_cand[m]);
    pre_asc[2].resize(n3p);
    int rcs[3] = {0, 0, 0};
    std::thread th[3];
    const void* kptr[3] = {keys[0].data(), keys[1].data(), pri.data()};
    const int kdt[3] = {SAMROAD_U8, SAMROAD_U8, SAMROAD_F64};
    const int64_t kn[3] = {n_cand[0], n_cand[1], n3p};
    for (int i = 0; i < 3; ++i)
      th[i] = std::thread([&, i] { rcs[i] = kn[i] ? argsort(kptr[i], kdt[i], kn[i], pre_asc[i].data(), user) : 0; });
    for (int i = 0; i < 3; ++i) th[i].join();
    SRB_REQUIRE(rcs[0] == 0 && rcs[1] == 0 && rcs[2] == 0, "argsort callback failed (%d %d %d)", rcs[0], rcs[1], rcs[2]);
    have_pre = true;
    us_presort = us_since(t0);
  }

  // passes 1 and 2: per-mask NMS (graph_extraction.py:131-134)
  PassStats ps[3];
  for (int m = 0; m < 2; ++m) {
    const int n = n_cand[m];
    if (int rc = grow(g->list[m], sizeof(int32_t) * static_cast<size_t>(n > 0 ? n : 1))) return rc;
    if (int rc = nms_pass(g, g->cand_pix[m].as<int32_t>(), g->cand_score[m].as<uint8_t>(), n, SAMROAD_U8, argsort,
                          user, have_pre ? &pre_asc[m] : nullptr, m == 0 ? "mask 0" : "mask 1", H, W, radius[m],
                          g->list[m].as<int32_t>(), &ps[m], st))
      return rc;
  }

  // pass 3: intersections first (graph_extraction.py:135-138), radius = ROAD_NMS_RADIUS.  The reference
  // sorts float64 priorities here, whose ties NumPy orders differently from uint8 ones (DESIGN.md §9).
  const int m0 = ps[0].kept, m1 = ps[1].kept, n3 = m0 + m1;
  if (n3 > 0) {
    if (int rc = grow(g->cand3, sizeof(int32_t) * static_cast<size_t>(n3))) return rc;
    if (int rc = grow(g->cls3, static_cast<size_t>(n3))) return rc;
    if (int rc = grow(g->list[2], sizeof(int32_t) * static_cast<size_t>(n3))) return rc;
    SRB_LAUNCH(concat_kernel, blocks_for(n3, 256), 256, 0, st, g->list[0].as<int32_t>(), m0, g->list[1].as<int32_t>(),
               m1, g->cand3.as<int32_t>(), g->cls3.as<uint8_t>());
    const bool pre3 = have_pre && m0 == n_cand[0] && m1 == n_cand[1];
    if (int rc = nms_pass(g, g->cand3.as<int32_t>(), g->cls3.as<uint8_t>(), n3, SAMROAD_F64, argsort, user,
                          pre3 ? &pre_asc[2] : nullptr, "the merged pass", H, W, road_radius, g->list[2].as<int32_t>(),
                          &ps[2], st))
      return rc;
  }
  const int n_out = ps[2].kept;
  SRB_REQUIRE(points_xy != nullptr || n_out == 0, "samroad_extract_graph_points: null output");
  SRB_REQUIRE(n_out <= cap, "samroad_extract_graph_points: %d keypoints exceed the output capacity %d", n_out, cap);
  if (n_out > 0) {
    SRB_LAUNCH(pix_to_xy_kernel, blocks_for(n_out, 256), 256, 0, st, g->list[2].as<int32_t>(), n_out, W, points_xy);
  }
  *n_points = n_out;
  if (stats) {
    stats[0] = n_cand[0]; stats[1] = n_cand[1]; stats[2] = m0; stats[3] = m1;
    stats[4] = ps[0].rounds; stats[5] = ps[1].rounds; stats[6] = ps[2].rounds; stats[7] = n_out;
    // host wall-clock split in microseconds (each stage ends on a stream synchronisation)
    stats[8] = us_cand; stats[9] = ps[0].us_order + us_presort; stats[10] = ps[1].us_order;
    stats[11] = ps[2].us_order; stats[12] = ps[0].us_nms; stats[13] = ps[1].us_nms; stats[14] = ps[2].us_nms;
    stats[15] = us_since(t_begin);
  }
  return 0;
}

// =================================================================================================
// pair queries  (inferencer.py:126-197)
// =================================================================================================
namespace {

__global__ void points_to_i32_kernel(const int64_t* __restrict__ in, int n2, int32_t* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n2) out[i] = static_cast<int32_t>(in[i]);
}

// rtree.intersection((x0, y0, x1, y1)) on point boxes: inclusive on all four sides (inferencer.py:150)
__device__ __forceinline__ bool in_tile(int x, int y, int x0, int y0, int P) {
  return x >= x0 && x <= x0 + P && y >= y0 && y <= y0 + P;
}

__global__ void __launch_bounds__(256)
tile_count_kernel(const int32_t* __restrict__ pts, int N, const int32_t* __restrict__ txy, int P,
                  int* __restrict__ cnt) {
  __shared__ int sw[33];
  const int t = blockIdx.x;
  const int x0 = txy[2 * t], y0 = txy[2 * t + 1];
  int c = 0;
  for (int i = threadIdx.x; i < N; i += 256) c += in_tile(pts[2 * i], pts[2 * i + 1], x0, y0, P) ? 1 : 0;
  int total;
  block_exclusive_scan(c, sw, total);
  if (threadIdx.x == 0) cnt[t] = total;
}

// members[off[t] + j] = global index of the tile's j-th point, ascending (the idx_patch2all map)
__global__ void __launch_bounds__(256)
tile_fill_kernel(const int32_t* __restrict__ pts, int N, const int32_t* __restrict__ txy, int P,
                 const int* __restrict__ off, int32_t* __restrict__ members) {
  __shared__ int sw[33];
  const int t = blockIdx.x;
  const int x0 = txy[2 * t], y0 = txy[2 * t + 1];
  int base = off[t];
  for (int b = 0; b < N; b += 256) {
    const int i = b + threadIdx.x;
    const bool in = i < N && in_tile(pts[2 * i], pts[2 * i + 1], x0, y0, P);
    int total;
    const int pos = block_exclusive_scan(in ? 1 : 0, sw, total);
    if (in) members[base + pos] = i;
    base += total;
  }
}

// KDTree.query(k = K+1, distance_upper_bound = R) minus self (inferencer.py:159-163): the (up to) KN
// nearest other points of the same tile with d < R, ascending distance; equal distances in ascending
// index; nbr rows are KN long.  Brute force per tile (a tile holds a few hundred points).
template <int KN>
__global__ void __launch_bounds__(128)
knn_kernel(const int32_t* __restrict__ pts, const int* __restrict__ cnt, const int* __restrict__ off,
           const int32_t* __restrict__ members, int d2lt, int32_t* __restrict__ nbr) {
  __shared__ int sx[128], sy[128];
  const int t = blockIdx.x;
  const int n = cnt[t];
  if (static_cast<int>(blockIdx.y) * 128 >= n) return;
  const int base = off[t];
  const int j = blockIdx.y * 128 + threadIdx.x;
  int px = 0, py = 0;
  if (j < n) { const int gi = members[base + j]; px = pts[2 * gi]; py = pts[2 * gi + 1]; }
  int bd[KN], bi[KN];
#pragma unroll
  for (int k = 0; k < KN; ++k) { bd[k] = INT_MAX; bi[k] = -1; }
  for (int c0 = 0; c0 < n; c0 += 128) {
    const int c = c0 + threadIdx.x;
    if (c < n) { const int gi = members[base + c]; sx[threadIdx.x] = pts[2 * gi]; sy[threadIdx.x] = pts[2 * gi + 1]; }
    __syncthreads();
    const int lim = n - c0 < 128 ? n - c0 : 128;
    if (j < n) {
      for (int q = 0; q < lim; ++q) {
        const int lc = c0 + q;
        const int dx = sx[q] - px, dy = sy[q] - py;
        const int d2 = dx * dx + dy * dy;
        if (lc == j || d2 >= d2lt || d2 >= bd[KN - 1]) continue;
        int cd = d2, ci = lc;
        bool ins = false;
#pragma unroll
        for (int k = 0; k < KN; ++k) {
          if (ins || cd < bd[k]) {
            const int td = bd[k], ti = bi[k];
            bd[k] = cd; bi[k] = ci; cd = td; ci = ti;
            ins = true;
          }
        }
      }
    }
    __syncthreads();
  }
  if (j < n) {
#pragma unroll
    for (int k = 0; k < KN; ++k) nbr[(static_cast<size_t>(base) + j) * KN + k] = bi[k];
  }
}

// padded batch tensors (inferencer.py:164-185): points relative to the tile origin, pairs (src, tgt or src),
// prefix-valid mask; rows beyond the tile's point count are zero (np.pad).  nbr rows are NS long.
template <int NS>
__global__ void fill_batch_kernel(const int32_t* __restrict__ pts, const int32_t* __restrict__ txy,
                                  const int* __restrict__ cnt, const int* __restrict__ off,
                                  const int32_t* __restrict__ members, const int32_t* __restrict__ nbr,
                                  int tile_begin, int B, int nmax, int K, int32_t* __restrict__ out_pts,
                                  int32_t* __restrict__ out_pairs, uint8_t* __restrict__ out_valid) {
  const long idx = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long total = static_cast<long>(B) * nmax * K;
  if (idx >= total) return;
  const int k = static_cast<int>(idx % K);
  const int j = static_cast<int>((idx / K) % nmax);
  const int b = static_cast<int>(idx / (static_cast<long>(K) * nmax));
  const int t = tile_begin + b;
  const int n = cnt[t];
  int src = 0, tgt = 0;
  uint8_t v = 0;
  if (j < n) {
    const int nb = nbr[(static_cast<size_t>(off[t]) + j) * NS + k];
    v = nb >= 0 ? 1 : 0;
    src = j;
    tgt = nb >= 0 ? nb : j;
  }
  out_pairs[2 * idx] = src;
  out_pairs[2 * idx + 1] = tgt;
  out_valid[idx] = v;
  if (k == 0) {
    int x = 0, y = 0;
    if (j < n) {
      const int gi = members[off[t] + j];
      x = pts[2 * gi] - txy[2 * t];
      y = pts[2 * gi + 1] - txy[2 * t + 1];
    }
    const size_t o = (static_cast<size_t>(b) * nmax + j) * 2;
    out_pts[o] = x;
    out_pts[o + 1] = y;
  }
}

}  // namespace

extern "C" int samroad_pair_queries_plan_k(samroad_graph_t g, const int64_t* points_xy, int N,
                                           const int32_t* tile_xy_host, int n_tiles, int P, double radius,
                                           int max_nbr, int32_t* tile_counts_host, void* stream) {
  SRB_REQUIRE(g && tile_xy_host && tile_counts_host, "samroad_pair_queries_plan: null argument");
  SRB_REQUIRE(max_nbr >= 1 && max_nbr <= 32, "samroad_pair_queries_plan: MAX_NEIGHBOR_QUERIES=%d must be in 1..32",
              max_nbr);
  SRB_REQUIRE(N >= 0 && n_tiles > 0 && P > 0, "samroad_pair_queries_plan: bad sizes N=%d tiles=%d P=%d", N, n_tiles, P);
  SRB_REQUIRE(N == 0 || points_xy != nullptr, "samroad_pair_queries_plan: null points");
  SRB_REQUIRE(radius >= 0.0 && radius < 30000.0, "samroad_pair_queries_plan: radius %.3f", radius);
  SRB_CUDA_OK(cudaSetDevice(g->device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  g->N = N; g->n_tiles = n_tiles; g->P = P;
  g->max_nbr = max_nbr;
  g->nbr_stride = max_nbr <= 16 ? 16 : 32;
  g->d2lt = static_cast<int>(std::ceil(radius * radius));        // d < R  <=>  d^2 < R^2  on integer d^2
  g->h_cnt.assign(n_tiles, 0);
  g->h_off.assign(n_tiles + 1, 0);
  g->total = 0;
  if (int rc = grow(g->tile_xy, sizeof(int32_t) * 2 * n_tiles)) return rc;
  if (int rc = grow(g->t_cnt, sizeof(int) * n_tiles)) return rc;
  if (int rc = grow(g->t_off, sizeof(int) * (n_tiles + 1))) return rc;
  SRB_CUDA_OK(cudaMemcpyAsync(g->tile_xy.get(), tile_xy_host, sizeof(int32_t) * 2 * n_tiles, cudaMemcpyHostToDevice, st));
  if (N == 0) {
    SRB_CUDA_OK(cudaMemsetAsync(g->t_cnt.get(), 0, sizeof(int) * n_tiles, st));
    SRB_CUDA_OK(cudaMemsetAsync(g->t_off.get(), 0, sizeof(int) * (n_tiles + 1), st));
    SRB_CUDA_OK(cudaStreamSynchronize(st));
    for (int t = 0; t < n_tiles; ++t) tile_counts_host[t] = 0;
    return 0;
  }
  if (int rc = grow(g->pts32, sizeof(int32_t) * 2 * static_cast<size_t>(N))) return rc;
  SRB_LAUNCH(points_to_i32_kernel, blocks_for(2L * N, 256), 256, 0, st, points_xy, 2 * N, g->pts32.as<int32_t>());
  SRB_LAUNCH(tile_count_kernel, n_tiles, 256, 0, st, g->pts32.as<int32_t>(), N, g->tile_xy.as<int32_t>(), P,
             g->t_cnt.as<int>());
  SRB_CUDA_OK(cudaMemcpyAsync(g->h_cnt.data(), g->t_cnt.get(), sizeof(int) * n_tiles, cudaMemcpyDeviceToHost, st));
  SRB_CUDA_OK(cudaStreamSynchronize(st));
  int max_cnt = 0;
  for (int t = 0; t < n_tiles; ++t) {
    g->h_off[t + 1] = g->h_off[t] + g->h_cnt[t];
    tile_counts_host[t] = g->h_cnt[t];
    if (g->h_cnt[t] > max_cnt) max_cnt = g->h_cnt[t];
  }
  g->total = g->h_off[n_tiles];
  SRB_REQUIRE(g->total * g->max_nbr < 2147483647L, "samroad_pair_queries_plan: %ld (tile, point) instances is too many", g->total);
  SRB_CUDA_OK(cudaMemcpyAsync(g->t_off.get(), g->h_off.data(), sizeof(int) * (n_tiles + 1), cudaMemcpyHostToDevice, st));
  if (g->total == 0) { SRB_CUDA_OK(cudaStreamSynchronize(st)); return 0; }
  if (int rc = grow(g->members, sizeof(int32_t) * static_cast<size_t>(g->total))) return rc;
  if (int rc = grow(g->nbr, sizeof(int32_t) * g->nbr_stride * static_cast<size_t>(g->total))) return rc;
  SRB_LAUNCH(tile_fill_kernel, n_tiles, 256, 0, st, g->pts32.as<int32_t>(), N, g->tile_xy.as<int32_t>(), P,
             g->t_off.as<int>(), g->members.as<int32_t>());
  const dim3 knn_grid(n_tiles, (max_cnt + 127) / 128);
  if (g->nbr_stride == 16)
    SRB_LAUNCH(knn_kernel<16>, knn_grid, 128, 0, st, g->pts32.as<int32_t>(), g->t_cnt.as<int>(), g->t_off.as<int>(),
               g->members.as<int32_t>(), g->d2lt, g->nbr.as<int32_t>());
  else
    SRB_LAUNCH(knn_kernel<32>, knn_grid, 128, 0, st, g->pts32.as<int32_t>(), g->t_cnt.as<int>(), g->t_off.as<int>(),
               g->members.as<int32_t>(), g->d2lt, g->nbr.as<int32_t>());
  SRB_CUDA_OK(cudaStreamSynchronize(st));    // h_off was copied from pageable memory
  return 0;
}

extern "C" int samroad_pair_queries_plan(samroad_graph_t g, const int64_t* points_xy, int N,
                                         const int32_t* tile_xy_host, int n_tiles, int P, double radius,
                                         int32_t* tile_counts_host, void* stream) {
  return samroad_pair_queries_plan_k(g, points_xy, N, tile_xy_host, n_tiles, P, radius, 16, tile_counts_host,
                                     stream);
}

extern "C" int samroad_pair_queries_fill(samroad_graph_t g, int tile_begin, int B, int nmax, int K,
                                         int32_t* points, int32_t* pairs, uint8_t* valid, void* stream) {
  SRB_REQUIRE(g && points && pairs && valid, "samroad_pair_queries_fill: null argument");
  SRB_REQUIRE(K >= 1 && K <= 32, "samroad_pair_queries_fill: MAX_NEIGHBOR_QUERIES=%d must be in 1..32", K);
  SRB_REQUIRE(tile_begin >= 0 && B >= 0 && tile_begin + B <= g->n_tiles,
              "samroad_pair_queries_fill: tiles [%d,%d) outside the planned %d", tile_begin, tile_begin + B, g->n_tiles);
  if (B == 0 || nmax <= 0) return 0;
  SRB_REQUIRE(K <= g->max_nbr, "samroad_pair_queries_fill: MAX_NEIGHBOR_QUERIES=%d but the pair queries were "
              "planned for %d", K, g->max_nbr);
  for (int b = 0; b < B; ++b)
    SRB_REQUIRE(g->h_cnt[tile_begin + b] <= nmax, "samroad_pair_queries_fill: tile %d has %d points > nmax=%d",
                tile_begin + b, g->h_cnt[tile_begin + b], nmax);
  SRB_CUDA_OK(cudaSetDevice(g->device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long total = static_cast<long>(B) * nmax * K;
  auto* fill = g->nbr_stride == 16 ? fill_batch_kernel<16> : fill_batch_kernel<32>;
  SRB_LAUNCH(fill, blocks_for(total, 256), 256, 0, st, g->pts32.as<int32_t>(), g->tile_xy.as<int32_t>(),
             g->t_cnt.as<int>(), g->t_off.as<int>(), g->members.as<int32_t>(), g->nbr.as<int32_t>(), tile_begin, B,
             nmax, K, points, pairs, valid);
  return 0;
}

// =================================================================================================
// edge aggregation  (inferencer.py:206-230)
// =================================================================================================
namespace {

// number of points within the neighbour radius of each point = upper bound of its distinct targets
__global__ void __launch_bounds__(128)
adj_kernel(const int32_t* __restrict__ pts, int N, int d2lt, const int* __restrict__ adj_off,
           int* __restrict__ deg, int32_t* __restrict__ adj_src, int32_t* __restrict__ adj_tgt,
           int* __restrict__ max_deg) {
  __shared__ int sx[128], sy[128];
  const int i = blockIdx.x * 128 + threadIdx.x;
  int px = 0, py = 0;
  if (i < N) { px = pts[2 * i]; py = pts[2 * i + 1]; }
  int c = 0;
  const int base = (adj_off && i < N) ? adj_off[i] : 0;
  for (int c0 = 0; c0 < N; c0 += 128) {
    const int q = c0 + threadIdx.x;
    if (q < N) { sx[threadIdx.x] = pts[2 * q]; sy[threadIdx.x] = pts[2 * q + 1]; }
    __syncthreads();
    const int lim = N - c0 < 128 ? N - c0 : 128;
    if (i < N) {
      for (int k = 0; k < lim; ++k) {
        const int dx = sx[k] - px, dy = sy[k] - py;
        if (c0 + k != i && dx * dx + dy * dy < d2lt) {
          if (adj_off) { adj_src[base + c] = i; adj_tgt[base + c] = c0 + k; }
          ++c;
        }
      }
    }
    __syncthreads();
  }
  if (!adj_off && i < N) {
    deg[i] = c;
    if (max_deg) atomicMax(max_deg, c);
  }
}

__device__ __forceinline__ int lower_bound_i32(const int32_t* a, int n, int v) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (a[mid] < v) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// arguments of the two aggregation kernels
struct AggArgs {
  const int32_t* pts;              // [N,2] keypoints
  int N;
  const int32_t* txy;              // [n_tiles,2] tile origins
  int n_tiles, P;
  const int *cnt, *off;            // the pair-query plan: per-tile count, offset, members, neighbour rows
  const int32_t *members, *nbr;
  const float* scores;             // tile t's block starts at tile_soff[t] (< 0: batch skipped)
  const int64_t* tile_soff;
  int K;
  const int* adj_off;              // adjacency slots of each source, targets ascending
  const int32_t* adj_tgt;
  float *sum, *num;                // per slot: score sum, count and first occurrence
  int32_t* first;
  int* bad;                        // set when a score lies outside [0, 1]
};

// One WARP per source point walks its tiles in tile-list order and its pair slots in order: for a fixed
// (src, tgt) that is exactly the order in which the reference's triple loop adds the scores, so the
// float32 sum is bit-identical.  The lanes own the source's adjacency slots (slot = lane + 32 d) and keep
// sum / count / first occurrence in registers; a tile's K (target, score) pairs are loaded by K lanes at
// once and broadcast one by one.  first[] records the key's first occurrence in the loop (dict order).
// nbr rows are NS long.
template <int DPL, int NS>
__global__ void __launch_bounds__(256) aggregate_warp_kernel(const AggArgs a) {
  const int S = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (S >= a.N) return;
  const int px = a.pts[2 * S], py = a.pts[2 * S + 1];
  const int a0 = a.adj_off[S], deg = a.adj_off[S + 1] - a0;
  int tg[DPL], fi[DPL];
  float sm[DPL], nm[DPL];
#pragma unroll
  for (int d = 0; d < DPL; ++d) {
    const int sl = lane + 32 * d;
    tg[d] = sl < deg ? a.adj_tgt[a0 + sl] : -2;
    fi[d] = -1; sm[d] = 0.f; nm[d] = 0.f;
  }
  const int K = a.K;
  bool badv = false;
  for (int t = 0; t < a.n_tiles; ++t) {
    if (!in_tile(px, py, a.txy[2 * t], a.txy[2 * t + 1], a.P)) continue;
    const int64_t so = a.tile_soff[t];
    if (so < 0) continue;                                   // batch skipped: no points (inferencer.py:188-189)
    const int base = a.off[t];
    const int j = lower_bound_i32(a.members + base, a.cnt[t], S);
    int Tk = -1;
    float vk = 0.f;
    if (lane < K) {
      const int nb = a.nbr[(static_cast<size_t>(base) + j) * NS + lane];
      if (nb >= 0) {
        Tk = a.members[base + nb];
        vk = a.scores[so + static_cast<int64_t>(j) * K + lane];
      }
    }
    for (int k = 0; k < K; ++k) {
      const int T = __shfl_sync(0xffffffffu, Tk, k);
      if (T < 0) break;                                      // prefix-valid
      float v = __shfl_sync(0xffffffffu, vk, k);
      if (v != v) v = -100.0f;                               // inferencer.py:206
      if (!(v >= 0.0f && v <= 1.0f)) badv = true;            // the reference asserts (inferencer.py:219)
#pragma unroll
      for (int d = 0; d < DPL; ++d) {
        if (tg[d] == T) {
          sm[d] = __fadd_rn(sm[d], v);
          nm[d] = __fadd_rn(nm[d], 1.0f);
          if (fi[d] < 0) fi[d] = (base + j) * K + k;
        }
      }
    }
  }
#pragma unroll
  for (int d = 0; d < DPL; ++d) {
    const int sl = lane + 32 * d;
    if (sl < deg) { a.sum[a0 + sl] = sm[d]; a.num[a0 + sl] = nm[d]; a.first[a0 + sl] = fi[d]; }
  }
  if (badv && lane == 0) atomicOr(a.bad, 1);
}

// Fallback for sources with more than 128 points within the neighbour radius (tiny NMS radii): one thread per
// source, slots in global memory.  Same order of additions.
template <int NS>
__global__ void __launch_bounds__(128) aggregate_kernel(const AggArgs a) {
  const int S = blockIdx.x * blockDim.x + threadIdx.x;
  if (S >= a.N) return;
  const int px = a.pts[2 * S], py = a.pts[2 * S + 1];
  const int a0 = a.adj_off[S], deg = a.adj_off[S + 1] - a0;
  const int K = a.K;
  for (int t = 0; t < a.n_tiles; ++t) {
    if (!in_tile(px, py, a.txy[2 * t], a.txy[2 * t + 1], a.P)) continue;
    const int64_t so = a.tile_soff[t];
    if (so < 0) continue;                                   // batch skipped: no points (inferencer.py:188-189)
    const int base = a.off[t];
    const int j = lower_bound_i32(a.members + base, a.cnt[t], S);
    const float* sc = a.scores + so + static_cast<int64_t>(j) * K;
    for (int k = 0; k < K; ++k) {
      const int nb = a.nbr[(static_cast<size_t>(base) + j) * NS + k];
      if (nb < 0) break;                                     // prefix-valid
      const int T = a.members[base + nb];
      float v = sc[k];
      if (v != v) v = -100.0f;                               // inferencer.py:206
      if (!(v >= 0.0f && v <= 1.0f)) atomicOr(a.bad, 1);     // the reference asserts (inferencer.py:219)
      const int slot = a0 + lower_bound_i32(a.adj_tgt + a0, deg, T);
      a.sum[slot] = __fadd_rn(a.sum[slot], v);
      a.num[slot] = __fadd_rn(a.num[slot], 1.0f);
      if (a.first[slot] < 0) a.first[slot] = (base + j) * K + k;
    }
  }
}

template <int NS>
int launch_aggregate(int max_deg, const AggArgs& a, cudaStream_t st) {
  if (max_deg <= 32)
    SRB_LAUNCH(aggregate_warp_kernel<1, NS>, blocks_for(32L * a.N, 256), 256, 0, st, a);
  else if (max_deg <= 64)
    SRB_LAUNCH(aggregate_warp_kernel<2, NS>, blocks_for(32L * a.N, 256), 256, 0, st, a);
  else if (max_deg <= 128)
    SRB_LAUNCH(aggregate_warp_kernel<4, NS>, blocks_for(32L * a.N, 256), 256, 0, st, a);
  else
    SRB_LAUNCH(aggregate_kernel<NS>, blocks_for(a.N, 128), 128, 0, st, a);
  return 0;
}

__global__ void edge_select_kernel(const float* __restrict__ sum, const float* __restrict__ num,
                                   const int32_t* __restrict__ first, int nnz, float thr,
                                   int32_t* __restrict__ eflags) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= nnz) return;
  if (num[s] > 0.0f && __fdiv_rn(sum[s], num[s]) > thr) eflags[first[s]] = s;
}

}  // namespace

extern "C" int samroad_aggregate_edges(samroad_graph_t g, const float* topo_scores, const int64_t* tile_score_offset_host,
                                       int K, float threshold, int64_t* edges, int cap, int* n_edges,
                                       int* bad_score, void* stream) {
  SRB_REQUIRE(g && n_edges && tile_score_offset_host, "samroad_aggregate_edges: null argument");
  SRB_REQUIRE(K >= 1 && K <= 32, "samroad_aggregate_edges: MAX_NEIGHBOR_QUERIES=%d must be in 1..32", K);
  SRB_CUDA_OK(cudaSetDevice(g->device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  *n_edges = 0;
  if (bad_score) *bad_score = 0;
  const int N = g->N;
  if (N == 0 || g->total == 0) return 0;
  SRB_REQUIRE(K <= g->max_nbr, "samroad_aggregate_edges: MAX_NEIGHBOR_QUERIES=%d but the pair queries were "
              "planned for %d", K, g->max_nbr);
  SRB_REQUIRE(topo_scores != nullptr, "samroad_aggregate_edges: null scores");
  const int32_t* pts = g->pts32.as<int32_t>();
  // adj_off: the degrees, scanned in place into N + 1 offsets, then the scan's scratch
  if (int rc = grow(g->adj_off, sizeof(int) * (N + 1 + scan_scratch_elems(N)))) return rc;
  if (int rc = grow(g->tile_soff, sizeof(int64_t) * g->n_tiles)) return rc;
  SRB_CUDA_OK(cudaMemcpyAsync(g->tile_soff.get(), tile_score_offset_host, sizeof(int64_t) * g->n_tiles,
                              cudaMemcpyHostToDevice, st));
  Counters* ctr = g->counters.as<Counters>();
  SRB_CUDA_OK(cudaMemsetAsync(ctr, 0, sizeof(Counters), st));
  int* adj_off = g->adj_off.as<int>();
  SRB_LAUNCH(adj_kernel, blocks_for(N, 128), 128, 0, st, pts, N, g->d2lt, nullptr, adj_off, nullptr, nullptr,
             &ctr->max_deg);
  if (int rc = exclusive_scan(adj_off, adj_off, N, &ctr->nnz, adj_off + N + 1, st)) return rc;
  Counters c;
  if (int rc = read_back(g, ctr, &c, st)) return rc;
  const int max_deg = c.max_deg, nnz = c.nnz;
  SRB_CUDA_OK(cudaMemcpyAsync(adj_off + N, &ctr->nnz, sizeof(int), cudaMemcpyDeviceToDevice, st));
  if (nnz == 0) return 0;
  const size_t nz = static_cast<size_t>(nnz);
  if (int rc = grow(g->adj_src, 4 * nz)) return rc;
  if (int rc = grow(g->adj_tgt, 4 * nz)) return rc;
  if (int rc = grow(g->adj_sum, 4 * nz)) return rc;
  if (int rc = grow(g->adj_cnt, 4 * nz)) return rc;
  if (int rc = grow(g->adj_first, 4 * nz)) return rc;
  const long n_entries = g->total * K;
  if (int rc = grow(g->eflags, 4 * static_cast<size_t>(n_entries))) return rc;
  SRB_CUDA_OK(cudaMemsetAsync(g->adj_sum.get(), 0, 4 * nz, st));
  SRB_CUDA_OK(cudaMemsetAsync(g->adj_cnt.get(), 0, 4 * nz, st));
  SRB_CUDA_OK(cudaMemsetAsync(g->adj_first.get(), 0xFF, 4 * nz, st));
  SRB_CUDA_OK(cudaMemsetAsync(g->eflags.get(), 0xFF, 4 * static_cast<size_t>(n_entries), st));
  SRB_LAUNCH(adj_kernel, blocks_for(N, 128), 128, 0, st, pts, N, g->d2lt, adj_off, nullptr, g->adj_src.as<int32_t>(),
             g->adj_tgt.as<int32_t>(), nullptr);
  const AggArgs args{pts, N, g->tile_xy.as<int32_t>(), g->n_tiles, g->P, g->t_cnt.as<int>(), g->t_off.as<int>(),
                     g->members.as<int32_t>(), g->nbr.as<int32_t>(), topo_scores, g->tile_soff.as<int64_t>(), K,
                     adj_off, g->adj_tgt.as<int32_t>(), g->adj_sum.as<float>(), g->adj_cnt.as<float>(),
                     g->adj_first.as<int32_t>(), &ctr->bad_score};
  if (g->nbr_stride == 16)
    SRB_TRY(launch_aggregate<16>(max_deg, args, st));
  else
    SRB_TRY(launch_aggregate<32>(max_deg, args, st));
  SRB_LAUNCH(edge_select_kernel, blocks_for(nnz, 256), 256, 0, st, g->adj_sum.as<float>(), g->adj_cnt.as<float>(),
             g->adj_first.as<int32_t>(), nnz, threshold, g->eflags.as<int32_t>());
  EdgeFlag ef{g->eflags.as<int32_t>(), g->adj_src.as<int32_t>(), g->adj_tgt.as<int32_t>(), edges, edges ? cap : 0};
  if (int rc = compact(g, ef, static_cast<int>(n_entries), &ctr->n_edges, st)) return rc;
  if (int rc = read_back(g, ctr, &c, st)) return rc;
  if (bad_score) *bad_score = c.bad_score;
  *n_edges = c.n_edges;
  SRB_REQUIRE(c.n_edges <= cap || edges == nullptr, "samroad_aggregate_edges: %d edges exceed the output capacity %d",
              c.n_edges, cap);
  return 0;
}
