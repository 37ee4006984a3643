// sam_road_b200 :: scan.cuh -- the integer building blocks of the graph stage, the precision-recall curve,
// training and labels: a block-wide exclusive scan, the exclusive scan of a device array, and one pass of a
// stable 8-bit digit sort.
//
// None of them allocates or synchronises: each caller sizes the scratch with the *_elems helpers and grows it
// under its own policy.  Every launch goes through SRB_LAUNCH.  The sums are integer sums, so a scan's
// result does not depend on how it is split over threads and blocks.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "common.cuh"

namespace srb {

constexpr int kScanTile = 4096;    // elements per 256-thread block of the tiled array scan
constexpr int kScanBlock = 1024;   // threads of the one-block array scan
constexpr int kDigitWarps = 8;     // warps per block of a digit pass; each warp owns one chunk

// Exclusive scan of one value per thread over the block (blockDim.x a multiple of 32, at most 1024), by two
// levels of warp shuffles.  `total` gets the block's sum in every thread.  Every thread of the block must
// call it; `smem` may be reused as soon as it returns.
template <typename T>
__device__ __forceinline__ T block_exclusive_scan(T v, T* smem /*[33]*/, T& total) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
  T inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const T t = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += t;
  }
  if (lane == 31) smem[wid] = inc;
  __syncthreads();
  if (wid == 0) {
    const T w = lane < nw ? smem[lane] : T(0);
    T wi = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const T t = __shfl_up_sync(0xffffffffu, wi, o);
      if (lane >= o) wi += t;
    }
    if (lane < nw) smem[lane] = wi - w;
    if (lane == 31) smem[32] = wi;
  }
  __syncthreads();
  const T res = inc - v + smem[wid];
  total = smem[32];
  __syncthreads();
  return res;
}

// Elements of scratch that exclusive_scan needs for n values.
inline long long scan_scratch_elems(long long n) { return blocks_for(n, kScanTile); }

// Elements of the histogram of a stable_digit_pass<kChunk> over n keys: 256 digits x chunks.
template <int kChunk>
long long digit_hist_elems(long long n) {
  return 256LL * blocks_for(n, kChunk);
}

// out[i] = in[0] + ... + in[i-1] for i < n, walked 1024 at a time by one block; *total (when not null) = the sum
template <typename T>
__global__ void __launch_bounds__(kScanBlock) scan_block_kernel(const T* in, T* out, long long n, T* total) {
  __shared__ T sm[33];
  T carry = 0;
  for (long long base = 0; base < n; base += kScanBlock) {
    const long long i = base + threadIdx.x;
    const T v = i < n ? in[i] : T(0);
    T t;
    const T ex = block_exclusive_scan(v, sm, t);
    if (i < n) out[i] = carry + ex;
    carry += t;
  }
  if (total && threadIdx.x == 0) *total = carry;
}

template <typename T>
__global__ void __launch_bounds__(256) scan_sums_kernel(const T* __restrict__ in, long long n,
                                                            T* __restrict__ sums) {
  __shared__ T sm[33];
  const long long base = static_cast<long long>(blockIdx.x) * kScanTile;
  T s = 0;
  for (int it = 0; it < kScanTile / 256; ++it) {
    const long long i = base + it * 256 + threadIdx.x;
    if (i < n) s += in[i];
  }
  T total;
  block_exclusive_scan(s, sm, total);
  if (threadIdx.x == 0) sums[blockIdx.x] = total;
}

// the scan of one tile, starting from the tile's offset
template <typename T>
__global__ void __launch_bounds__(256) scan_tile_kernel(const T* in, T* out, long long n,
                                                        const T* __restrict__ tile_off) {
  __shared__ T sm[33];
  const long long base = static_cast<long long>(blockIdx.x) * kScanTile;
  T carry = tile_off[blockIdx.x];
  for (int it = 0; it < kScanTile / 256; ++it) {
    const long long i = base + it * 256 + threadIdx.x;
    const T v = i < n ? in[i] : T(0);
    T total;
    const T ex = block_exclusive_scan(v, sm, total);
    if (i < n) out[i] = carry + ex;
    carry += total;
  }
}

// A digit pass gives one warp a chunk of kChunk consecutive elements.  The histogram is digit-major:
// hist[d * nchunks + c] counts digit d in chunk c, so its exclusive scan is every (digit, chunk)'s first
// output position.
template <int kChunk, class F>
__global__ void __launch_bounds__(32 * kDigitWarps) digit_hist_kernel(const F f, long long n, int nchunks,
                                                                     uint32_t* __restrict__ hist) {
  __shared__ uint32_t h[kDigitWarps][256];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int chunk = blockIdx.x * kDigitWarps + w;
  if (chunk >= nchunks) return;
  for (int d = lane; d < 256; d += 32) h[w][d] = 0;
  __syncwarp();
  const long long base = static_cast<long long>(chunk) * kChunk;
  for (int it = 0; it < kChunk / 32; ++it) {
    const long long i = base + it * 32 + lane;
    if (i < n) atomicAdd(&h[w][f.digit(f.key(i))], 1u);
  }
  __syncwarp();
  for (int d = lane; d < 256; d += 32) hist[static_cast<size_t>(d) * nchunks + chunk] = h[w][d];
}

// A warp walks its chunk 32 elements at a time; __match_any_sync ranks equal digits of a step in lane order,
// so the pass is stable and does not depend on scheduling.
template <int kChunk, class F>
__global__ void __launch_bounds__(32 * kDigitWarps) digit_scatter_kernel(const F f, long long n, int nchunks,
                                                                        const uint32_t* __restrict__ off) {
  __shared__ uint32_t o[kDigitWarps][256];
  const int w = threadIdx.x >> 5;
  const unsigned lane = threadIdx.x & 31;
  const int chunk = blockIdx.x * kDigitWarps + w;
  if (chunk >= nchunks) return;
  for (int d = lane; d < 256; d += 32) o[w][d] = off[static_cast<size_t>(d) * nchunks + chunk];
  __syncwarp();
  const long long base = static_cast<long long>(chunk) * kChunk;
  for (int it = 0; it < kChunk / 32; ++it) {
    const long long i = base + it * 32 + lane;
    const bool ok = i < n;
    const uint32_t key = ok ? f.key(i) : 0u;
    const unsigned d = ok ? f.digit(key) : (256u + lane);   // idle lanes match only themselves
    const unsigned peers = __match_any_sync(0xffffffffu, d);
    const unsigned r = __popc(peers & ((1u << lane) - 1u));
    uint32_t pos = 0;
    if (ok) pos = o[w][d] + r;
    __syncwarp();
    if (ok && r == 0) o[w][d] += __popc(peers);
    __syncwarp();
    if (ok) f.emit(i, key, pos);
  }
}

// Exclusive scan of n values of T (int, uint32_t or unsigned long long) from `in` to `out`, which may be the
// same array; *total_dev (when not null) gets the sum.  Up to one tile it is one launch of the one-block scan;
// beyond, tile sums -> the one-block scan of the sums in `scratch` (scan_scratch_elems(n)) -> tile scan.
template <typename T>
int exclusive_scan(const T* in, T* out, long long n, T* total_dev, T* scratch, cudaStream_t st) {
  if (n <= kScanTile) {
    SRB_LAUNCH(scan_block_kernel<T>, 1, kScanBlock, 0, st, in, out, n, total_dev);
  } else {
    const int tiles = blocks_for(n, kScanTile);
    SRB_LAUNCH(scan_sums_kernel<T>, tiles, 256, 0, st, in, n, scratch);
    SRB_LAUNCH(scan_block_kernel<T>, 1, kScanBlock, 0, st, scratch, scratch, tiles, total_dev);
    SRB_LAUNCH(scan_tile_kernel<T>, tiles, 256, 0, st, in, out, n, scratch);
  }
  return 0;
}

// One stable pass of a counting sort on an 8-bit digit over n > 0 elements: histogram per (digit, chunk of
// kChunk elements), exclusive scan of the histogram in place, ordered scatter.  Elements of equal digit keep
// their index order.  F supplies
//   __device__ uint32_t key(long long i) const;                         element i's key (read once per pass
//                                                                       and element by the scatter)
//   __device__ unsigned digit(uint32_t key) const;                      its digit, 0..255
//   __device__ void emit(long long i, uint32_t key, uint32_t pos) const;  element i has rank pos
// hist holds digit_hist_elems<kChunk>(n) values, scratch scan_scratch_elems of that.
template <int kChunk, class F>
int stable_digit_pass(const F& f, long long n, uint32_t* hist, uint32_t* scratch, cudaStream_t st) {
  static_assert(kChunk % 32 == 0, "a warp walks its chunk 32 elements at a time");
  const int nchunks = blocks_for(n, kChunk);
  const int blocks = blocks_for(nchunks, kDigitWarps);
  SRB_LAUNCH(digit_hist_kernel<kChunk, F>, blocks, 32 * kDigitWarps, 0, st, f, n, nchunks, hist);
  if (int rc = exclusive_scan<uint32_t>(hist, hist, 256LL * nchunks, nullptr, scratch, st)) return rc;
  SRB_LAUNCH(digit_scatter_kernel<kChunk, F>, blocks, 32 * kDigitWarps, 0, st, f, n, nchunks, hist);
  return 0;
}

}  // namespace srb
