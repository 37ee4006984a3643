// sam_road_b200 :: training / evaluation batches on the device (DESIGN.md §13).
//
// Reference: SatMapDataset.__getitem__ (dataset.py:402-445), GraphLabelGenerator.sample_patch
// (dataset.py:127-231) and graph_collate_fn (dataset.py:287-302).  What GraphLabelGenerator.__init__ builds
// once per scene (subdivided graph, excluded points, NMS immunity, sample weights, CSR adjacency) is computed
// on the host by sam_road_b200/dataset.py and uploaded here; a batch of B patches is then five kernels:
//
//   draw_kernel     Philox draws into device arrays: patch (scene, x0, y0, rot), one U[0,1) per candidate
//                   (NMS score), one U[0,1) per source, one N(0,1) pair per point.  The test hook skips it and
//                   takes caller-filled arrays; every later stage is a deterministic function of the arrays.
//   crop_kernel     RGB / keypoint / road crop with np.rot90(., rot, (0, 1)); float32 0..255 and /255.
//   patch_kernel    one block per patch: inclusive box query minus the excluded points (ascending id),
//                   scores, bitonic sort by (score desc, id asc), cell-bucketed greedy NMS in shared memory,
//                   the weighted choice of the sources.
//   pairs_kernel    one warp per source: the k+1 nearest survivors strictly inside NEIGHBOR_RADIUS (ties by
//                   survivor index), the first one dropped; then the depth-limited BFS over the subdivided
//                   graph that stops at the targets, with a shared-memory hash set of reached nodes.
//   points_kernel   survivors minus the origin, rotated about the patch centre in float64, plus the noise,
//                   rounded once to float32, zero-padded to the batch's largest point count.
//
// The host reads back once per batch (the survivor counts, to size the points, and a status word).
#include "../../include/samroad_b200.h"

#include <cuda_runtime.h>

#include <algorithm>
#include <climits>
#include <cmath>
#include <cstring>
#include <vector>

#include "common.cuh"

using namespace srb;

namespace {

constexpr int kPatchThreads = 1024;
constexpr int kPairWarps = 4;
constexpr int kBfsList = 1024;            // nodes one BFS may reach
constexpr int kBfsHash = 2 * kBfsList;    // open-addressing slots: load factor stays below 1/2
constexpr int kMaxCells = 33;             // NMS cells per patch side (cell side >= max(radius, P / 32))
enum : uint8_t { kExcluded = 1, kImmune = 2 };
enum : uint32_t { kStreamPatch = 0, kStreamScore = 1, kStreamSource = 2, kStreamNoise = 3 };
enum : int { kBadPatch = 1, kBfsOverflow = 2, kOverCap = 4 };

struct SceneDev {
  const double* pts;         // [n, 2] (x, y)
  const uint8_t* flags;      // [n] kExcluded | kImmune
  const float* weight;       // [n] sample weights
  const int32_t* adj_start;  // [n + 1] CSR of the subdivided graph
  const int32_t* adj;
  const uint8_t* rgb;        // [size, size, 3]
  const uint8_t* kp;         // [size, size]
  const uint8_t* road;       // [size, size]
  int32_t n;
};

struct Params {
  const SceneDev* scenes;
  int n_scenes, P, size, lo, hi;     // origins in [lo, hi]
  int S, Np, depth, cap, ncell;
  double r_nms2, r_nbr2, cell;
};

struct Work {          // per-batch device arrays, [B, ...]
  int32_t* patch;      // [B, 4] scene, x0, y0, rot
  double* score_u;     // [B, cap]
  double* src_u;       // [B, S]
  double* noise;       // [B, cap, 2]
  int32_t* cand;       // [B, cap] candidate ids (ascending), then sorted ids
  int32_t* surv;       // [B, cap] survivor ids in visiting order
  double* sxy;         // [B, cap, 2] survivor coordinates
  double* cdf;         // [B, cap] running sum of the survivors' weights
  int32_t* src;        // [B, S] source, index into the survivors
  int32_t* status;     // [1] kBadPatch | kBfsOverflow | kOverCap
  int32_t* nsurv;      // [B] survivors (0: empty patch), right after the status word
};

// ---- Philox4x32-10 keyed by the 64-bit seed, counter (ctr, element, stream, 0) ---------------------------------
__device__ __forceinline__ uint32_t mulhilo(uint32_t a, uint32_t b, uint32_t* hi) {
  const unsigned long long p = static_cast<unsigned long long>(a) * b;
  *hi = static_cast<uint32_t>(p >> 32);
  return static_cast<uint32_t>(p);
}

__device__ __forceinline__ uint4 philox4(unsigned long long seed, uint32_t elem, uint32_t stream, uint32_t ctr) {
  uint32_t c0 = ctr, c1 = elem, c2 = stream, c3 = 0;
  uint32_t k0 = static_cast<uint32_t>(seed), k1 = static_cast<uint32_t>(seed >> 32);
  for (int r = 0; r < 10; ++r) {
    uint32_t hi0, hi1;
    const uint32_t lo0 = mulhilo(0xD2511F53u, c0, &hi0);
    const uint32_t lo1 = mulhilo(0xCD9E8D57u, c2, &hi1);
    const uint32_t n0 = hi1 ^ c1 ^ k0, n2 = hi0 ^ c3 ^ k1;
    c0 = n0; c1 = lo1; c2 = n2; c3 = lo0;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  return make_uint4(c0, c1, c2, c3);
}

__device__ __forceinline__ unsigned long long join64(uint32_t hi, uint32_t lo) {
  return (static_cast<unsigned long long>(hi) << 32) | lo;
}
// U[0, 1) with 53 random bits
__device__ __forceinline__ double u53(uint32_t hi, uint32_t lo) {
  return static_cast<double>(join64(hi, lo) >> 11) * 0x1.0p-53;
}
// uniform integer in [0, n)
__device__ __forceinline__ int uniform_int(uint32_t hi, uint32_t lo, int n) {
  return static_cast<int>(__umul64hi(join64(hi, lo), static_cast<unsigned long long>(n)));
}

__global__ void draw_kernel(Work w, Params p, int draw_patch, unsigned long long seed) {
  const int b = blockIdx.y;
  const int len = max(p.cap, p.S);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < len; i += gridDim.x * blockDim.x) {
    if (i < p.cap) {
      const uint4 r = philox4(seed, b, kStreamScore, i);
      w.score_u[static_cast<size_t>(b) * p.cap + i] = u53(r.x, r.y);
      // Box-Muller: one pair of normals per point, x then y
      const uint4 q = philox4(seed, b, kStreamNoise, i);
      const double u1 = 1.0 - u53(q.x, q.y), u2 = u53(q.z, q.w);
      const double rad = sqrt(-2.0 * log(u1));
      double s, c;
      sincospi(2.0 * u2, &s, &c);
      w.noise[(static_cast<size_t>(b) * p.cap + i) * 2] = rad * c;
      w.noise[(static_cast<size_t>(b) * p.cap + i) * 2 + 1] = rad * s;
    }
    if (i < p.S) {
      const uint4 r = philox4(seed, b, kStreamSource, i);
      w.src_u[static_cast<size_t>(b) * p.S + i] = u53(r.x, r.y);
    }
  }
  if (draw_patch && blockIdx.x == 0 && threadIdx.x == 0) {
    const uint4 r0 = philox4(seed, b, kStreamPatch, 0), r1 = philox4(seed, b, kStreamPatch, 1);
    const int span = p.hi - p.lo + 1;
    w.patch[4 * b + 0] = uniform_int(r0.x, r0.y, p.n_scenes);
    w.patch[4 * b + 1] = p.lo + uniform_int(r0.z, r0.w, span);
    w.patch[4 * b + 2] = p.lo + uniform_int(r1.x, r1.y, span);
    w.patch[4 * b + 3] = uniform_int(r1.z, r1.w, 4);
  }
}

__device__ __forceinline__ bool patch_ok(const Params& p, const int32_t* pa) {
  return pa[0] >= 0 && pa[0] < p.n_scenes && pa[1] >= p.lo && pa[1] <= p.hi && pa[2] >= p.lo &&
         pa[2] <= p.hi && pa[3] >= 0 && pa[3] < 4;
}

// out[i][j] = A[y0 + si][x0 + sj] with (si, sj) the source of np.rot90(A, rot, (0, 1)) at (i, j)
__global__ void crop_kernel(Params p, const int32_t* patch, float* rgb, float* kp, float* road) {
  const int b = blockIdx.y;
  const int64_t pp = static_cast<int64_t>(p.P) * p.P;
  const int64_t idx = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= pp) return;
  const int32_t* pa = patch + 4 * b;
  const int64_t o = static_cast<int64_t>(b) * pp + idx;
  if (!patch_ok(p, pa)) {
    rgb[3 * o] = rgb[3 * o + 1] = rgb[3 * o + 2] = 0.0f;
    kp[o] = road[o] = 0.0f;
    return;
  }
  const int i = static_cast<int>(idx / p.P), j = static_cast<int>(idx % p.P), e = p.P - 1;
  int si = i, sj = j;
  switch (pa[3]) {
    case 1: si = j; sj = e - i; break;
    case 2: si = e - i; sj = e - j; break;
    case 3: si = e - j; sj = i; break;
    default: break;
  }
  const SceneDev& sc = p.scenes[pa[0]];
  const int64_t s = static_cast<int64_t>(pa[2] + si) * p.size + (pa[1] + sj);
  rgb[3 * o] = sc.rgb[3 * s];
  rgb[3 * o + 1] = sc.rgb[3 * s + 1];
  rgb[3 * o + 2] = sc.rgb[3 * s + 2];
  kp[o] = __fdiv_rn(static_cast<float>(sc.kp[s]), 255.0f);
  road[o] = __fdiv_rn(static_cast<float>(sc.road[s]), 255.0f);
}

// exclusive prefix sum of v over the block; *total gets the block sum.  All threads must call it.
__device__ int block_scan_excl(int v, int* warp_tot, int* total) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
  int x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) warp_tot[wid] = x;
  __syncthreads();
  if (wid == 0) {
    const int t = lane < nw ? warp_tot[lane] : 0;
    int s = t;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, s, o);
      if (lane >= o) s += y;
    }
    if (lane < nw) warp_tot[lane] = s - t;
    if (lane == 31) *total = s;
  }
  __syncthreads();
  const int r = warp_tot[wid] + x - v;
  __syncthreads();
  return r;
}

// sort order of the NMS visit: score descending, then id ascending
__device__ __forceinline__ bool precedes(unsigned long long ka, int ia, unsigned long long kb, int ib) {
  return ka > kb || (ka == kb && ia < ib);
}

__device__ __forceinline__ double dist2(double ax, double ay, double bx, double by) {
  const double dx = __dsub_rn(ax, bx), dy = __dsub_rn(ay, by);
  return __dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy));
}

// Dynamic shared memory of patch_kernel: the sort keys (8 + 4 bytes per slot of the power-of-two sort),
// later reused for the rank-ordered coordinates (16 bytes per candidate); then the 4-byte arrays (cell of each
// candidate, candidates by cell, the cell table) and last the immunity and suppression bytes.
size_t patch_smem_bytes(int cap) {
  size_t pow2 = 1;
  while (pow2 < static_cast<size_t>(cap)) pow2 <<= 1;
  size_t a = pow2 * 12 > static_cast<size_t>(cap) * 16 ? pow2 * 12 : static_cast<size_t>(cap) * 16;
  a = (a + 15) & ~static_cast<size_t>(15);
  return a + static_cast<size_t>(cap) * (1 + 1 + 4 + 4) + 2 * 4 * (kMaxCells * kMaxCells + 1);
}

__global__ void __launch_bounds__(kPatchThreads) patch_kernel(Params p, Work w) {
  extern __shared__ __align__(16) unsigned char smem[];
  __shared__ int warp_tot[32];
  __shared__ int s_total;
  const int b = blockIdx.x, tid = threadIdx.x;
  const int32_t* pa = w.patch + 4 * b;
  if (!patch_ok(p, pa)) {
    if (tid == 0) {
      atomicOr(w.status, kBadPatch);
      w.nsurv[b] = 0;
    }
    return;
  }
  const SceneDev sc = p.scenes[pa[0]];
  const double bx0 = pa[1], by0 = pa[2], bx1 = pa[1] + p.P, by1 = pa[2] + p.P;
  const size_t off = static_cast<size_t>(b) * p.cap;
  int32_t* cand = w.cand + off;

  // 1. inclusive box query minus the excluded points, in ascending id (ordered compaction)
  int M = 0;
  for (int base = 0; base < sc.n; base += blockDim.x) {
    const int i = base + tid;
    int keep = 0;
    if (i < sc.n) {
      const double x = sc.pts[2 * i], y = sc.pts[2 * i + 1];
      keep = x >= bx0 && x <= bx1 && y >= by0 && y <= by1 && !(sc.flags[i] & kExcluded);
    }
    const int pos = block_scan_excl(keep, warp_tot, &s_total);
    const int tot = s_total;
    if (keep && M + pos < p.cap) cand[M + pos] = i;
    M += tot;
  }
  if (M > p.cap) {   // the host sized cap from every admissible window: not reached
    if (tid == 0) atomicOr(w.status, kOverCap);
    M = p.cap;
  }
  if (M == 0) {
    if (tid == 0) w.nsurv[b] = 0;
    return;
  }

  // 2. scores max(U(0.9, 1), override) as order-preserving bit patterns (all scores are positive)
  int pow2 = 1;
  while (pow2 < M) pow2 <<= 1;
  unsigned long long* key = reinterpret_cast<unsigned long long*>(smem);
  int* kid = reinterpret_cast<int*>(key + pow2);
  size_t a_bytes = static_cast<size_t>(p.cap);
  {
    size_t q = 1;
    while (q < a_bytes) q <<= 1;
    a_bytes = q * 12 > a_bytes * 16 ? q * 12 : a_bytes * 16;
    a_bytes = (a_bytes + 15) & ~static_cast<size_t>(15);
  }
  double* xy = reinterpret_cast<double*>(smem);                   // [M, 2], after the sort
  int* cell_of = reinterpret_cast<int*>(smem + a_bytes);          // [cap]
  int* citem = cell_of + p.cap;                                   // [cap]
  int* cstart = citem + p.cap;                                    // [ncell^2 + 1]
  int* ccur = cstart + kMaxCells * kMaxCells + 1;                 // [ncell^2]
  uint8_t* imm = reinterpret_cast<uint8_t*>(ccur + kMaxCells * kMaxCells);   // [cap]
  uint8_t* supp = imm + p.cap;                                    // [cap]
  const unsigned long long two = static_cast<unsigned long long>(__double_as_longlong(2.0));
  for (int j = tid; j < pow2; j += blockDim.x) {
    if (j < M) {
      const int id = cand[j];
      double s = __dadd_rn(0.9, __dmul_rn(1.0 - 0.9, w.score_u[off + j]));
      if (sc.flags[id] & kImmune) s = fmax(s, 2.0);
      key[j] = static_cast<unsigned long long>(__double_as_longlong(s));
      kid[j] = id;
    } else {
      key[j] = 0;
      kid[j] = INT_MAX;
    }
  }
  __syncthreads();

  // 3. bitonic sort into visiting order
  for (int k = 2; k <= pow2; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = tid; i < pow2; i += blockDim.x) {
        const int l = i ^ j;
        if (l > i) {
          const bool up = (i & k) == 0;
          const unsigned long long ki = key[i], kl = key[l];
          const int ii = kid[i], il = kid[l];
          if (up ? precedes(kl, il, ki, ii) : precedes(ki, ii, kl, il)) {
            key[i] = kl; key[l] = ki;
            kid[i] = il; kid[l] = ii;
          }
        }
      }
      __syncthreads();
    }
  }

  // 4. rank-ordered ids, immunity and cells; then the coordinates over the sort buffer
  const int nc = p.ncell;
  for (int c = tid; c < nc * nc + 1; c += blockDim.x) cstart[c] = 0;
  for (int k = tid; k < M; k += blockDim.x) {
    cand[k] = kid[k];
    imm[k] = key[k] == two;
    supp[k] = 0;
  }
  __syncthreads();
  for (int k = tid; k < M; k += blockDim.x) {
    const int id = cand[k];
    const double x = sc.pts[2 * id], y = sc.pts[2 * id + 1];
    xy[2 * k] = x;
    xy[2 * k + 1] = y;
    const int cx = min(max(static_cast<int>(floor((x - bx0) / p.cell)), 0), nc - 1);
    const int cy = min(max(static_cast<int>(floor((y - by0) / p.cell)), 0), nc - 1);
    cell_of[k] = cy * nc + cx;
    atomicAdd(&cstart[cy * nc + cx + 1], 1);
  }
  __syncthreads();
  {
    int carry = 0;
    for (int base = 0; base < nc * nc + 1; base += blockDim.x) {
      const int c = base + tid;
      const int v = c < nc * nc + 1 ? cstart[c] : 0;
      const int ex = block_scan_excl(v, warp_tot, &s_total);
      if (c < nc * nc + 1) cstart[c] = carry + ex + v;
      carry += s_total;
    }
  }
  for (int c = tid; c < nc * nc; c += blockDim.x) ccur[c] = cstart[c];
  __syncthreads();
  for (int k = tid; k < M; k += blockDim.x) citem[atomicAdd(&ccur[cell_of[k]], 1)] = k;
  __syncthreads();

  // 5. greedy NMS in visiting order (one warp): a kept point suppresses every later non-immune point within
  //    ROAD_NMS_RADIUS, inclusive; cells are at least one radius wide, so the 3 x 3 block around it suffices
  if (tid < 32) {
    const int lane = tid;
    int n = 0;
    for (int k = 0; k < M; ++k) {
      if (supp[k]) continue;
      const double xk = xy[2 * k], yk = xy[2 * k + 1];
      if (lane == 0) {
        w.surv[off + n] = cand[k];
        w.sxy[2 * (off + n)] = xk;
        w.sxy[2 * (off + n) + 1] = yk;
      }
      ++n;
      const int ci = cell_of[k] % nc, cj = cell_of[k] / nc;
      for (int y = max(cj - 1, 0); y <= min(cj + 1, nc - 1); ++y)
        for (int x = max(ci - 1, 0); x <= min(ci + 1, nc - 1); ++x) {
          const int c = y * nc + x;
          for (int t = cstart[c] + lane; t < cstart[c + 1]; t += 32) {
            const int kk = citem[t];
            if (kk > k && !imm[kk] && dist2(xy[2 * kk], xy[2 * kk + 1], xk, yk) <= p.r_nms2) supp[kk] = 1;
          }
        }
      __syncwarp();
    }
    if (lane == 0) w.nsurv[b] = n;
  }
  __syncthreads();

  // 6. sources: TOPO_SAMPLE_NUM draws with replacement, P(i) = weight_i / sum (inverse of the running sum)
  const int n = w.nsurv[b];
  double* cdf = w.cdf + off;
  if (tid == 0) {
    double acc = 0.0;
    for (int i = 0; i < n; ++i) {
      acc = __dadd_rn(acc, static_cast<double>(sc.weight[w.surv[off + i]]));
      cdf[i] = acc;
    }
  }
  __syncthreads();
  const double total = cdf[n - 1];
  for (int s = tid; s < p.S; s += blockDim.x) {
    const double v = __dmul_rn(w.src_u[static_cast<size_t>(b) * p.S + s], total);
    int lo = 0, hi = n;   // first i with cdf[i] > v
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (cdf[mid] > v) hi = mid; else lo = mid + 1;
    }
    w.src[static_cast<size_t>(b) * p.S + s] = min(lo, n - 1);
  }
}

struct BfsSmem {
  int hash[kBfsHash];
  int list[kBfsList];
  int stop[32];
  int count;
  int overflow;
};

__device__ __forceinline__ bool hash_insert(int* hash, int v) {
  unsigned h = (static_cast<unsigned>(v) * 2654435761u) & (kBfsHash - 1);
  while (true) {
    const int old = atomicCAS(&hash[h], -1, v);
    if (old == -1) return true;
    if (old == v) return false;
    h = (h + 1) & (kBfsHash - 1);
  }
}

__device__ __forceinline__ bool hash_find(const int* hash, int v) {
  unsigned h = (static_cast<unsigned>(v) * 2654435761u) & (kBfsHash - 1);
  while (true) {
    const int cur = hash[h];
    if (cur == v) return true;
    if (cur == -1) return false;
    h = (h + 1) & (kBfsHash - 1);
  }
}

// One warp per (patch, source): kNN among the survivors, then BFS from the source to depth NEIGHBOR_RADIUS // 4
// that reaches but does not expand the targets.  Writes pairs / valid / connected.
__global__ void __launch_bounds__(32 * kPairWarps, 4) pairs_kernel(Params p, Work w, int32_t* pairs, uint8_t* connected,
                                                               uint8_t* valid) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  BfsSmem& sm = reinterpret_cast<BfsSmem*>(smem_raw)[threadIdx.x >> 5];
  const int lane = threadIdx.x & 31;
  const int b = blockIdx.y, s = blockIdx.x * kPairWarps + (threadIdx.x >> 5);
  if (s >= p.S) return;
  const size_t slot = (static_cast<size_t>(b) * p.S + s) * p.Np;
  const int n = w.nsurv[b];
  if (n == 0) {   // empty patch (dataset.py:135-142): one point at (0, 0), all-false samples
    for (int k = lane; k < p.Np; k += 32) {
      pairs[2 * (slot + k)] = 0;
      pairs[2 * (slot + k) + 1] = 0;
      valid[slot + k] = 0;
      connected[slot + k] = 0;
    }
    return;
  }
  const size_t off = static_cast<size_t>(b) * p.cap;
  const double* sxy = w.sxy + 2 * off;
  const int si = w.src[static_cast<size_t>(b) * p.S + s];
  const double xs = sxy[2 * si], ys = sxy[2 * si + 1];

  // k+1 nearest in (distance, index) order, strictly inside the radius; the first is dropped
  double pd = -1.0;
  int pi = -1, hits = 0, my_tgt = -1;
  for (int r = 0; r <= p.Np; ++r) {
    double bd = INFINITY;
    int bi = INT_MAX;
    for (int i = lane; i < n; i += 32) {
      const double d = dist2(sxy[2 * i], sxy[2 * i + 1], xs, ys);
      if (d < p.r_nbr2 && (d > pd || (d == pd && i > pi)) && (d < bd || (d == bd && i < bi))) {
        bd = d;
        bi = i;
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const double od = __shfl_xor_sync(0xffffffffu, bd, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (od < bd || (od == bd && oi < bi)) {
        bd = od;
        bi = oi;
      }
    }
    if (bi == INT_MAX) break;
    if (r > 0 && lane == r - 1) my_tgt = bi;
    pd = bd;
    pi = bi;
    ++hits;
  }
  const int nt = hits > 0 ? hits - 1 : 0;   // targets held by lanes 0 .. nt-1
  if (nt == 0) {   // no target in range: every slot is padding and the walk decides nothing
    for (int k = lane; k < p.Np; k += 32) {
      pairs[2 * (slot + k)] = si;
      pairs[2 * (slot + k) + 1] = si;
      valid[slot + k] = 0;
      connected[slot + k] = 0;
    }
    return;
  }

  // BFS (graph_utils.py:594-630): reached = visited set
  for (int h = lane; h < kBfsHash; h += 32) sm.hash[h] = -1;
  sm.stop[lane] = lane < nt ? w.surv[off + my_tgt] : -1;
  const int source = w.surv[off + si];
  if (lane == 0) {
    sm.count = 1;
    sm.overflow = 0;
    sm.list[0] = source;
  }
  __syncwarp();
  if (lane == 0) hash_insert(sm.hash, source);
  __syncwarp();
  const SceneDev& sc = p.scenes[w.patch[4 * b]];
  int lo = 0, hi = 1;
  for (int d = 0; d < p.depth && lo < hi; ++d) {
    for (int i = lo + lane; i < hi; i += 32) {
      const int u = sm.list[i];
      bool stop = false;
      for (int t = 0; t < nt; ++t) stop |= sm.stop[t] == u;
      if (stop) continue;
      for (int e = sc.adj_start[u]; e < sc.adj_start[u + 1]; ++e) {
        if (*static_cast<volatile int*>(&sm.overflow)) break;
        const int v = sc.adj[e];
        if (hash_insert(sm.hash, v)) {
          const int pos = atomicAdd(&sm.count, 1);
          if (pos < kBfsList) sm.list[pos] = v; else sm.overflow = 1;
        }
      }
    }
    __syncwarp();
    lo = hi;
    hi = min(sm.count, kBfsList);
    __syncwarp();
  }
  if (lane == 0 && sm.overflow) atomicOr(w.status, kBfsOverflow);
  for (int k = lane; k < p.Np; k += 32) {
    const bool ok = k < nt;
    pairs[2 * (slot + k)] = si;
    pairs[2 * (slot + k) + 1] = ok ? my_tgt : si;
    valid[slot + k] = ok;
    connected[slot + k] = ok && hash_find(sm.hash, sm.stop[k]);
  }
}

// points[b, i] = rot^k(survivor - origin - c) + c + noise, float64, rounded once to float32; zero padding
__global__ void points_kernel(Params p, Work w, int N, float* points) {
  const int b = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  const int n = w.nsurv[b];
  float* o = points + 2 * (static_cast<size_t>(b) * N + i);
  if (i >= n) {
    o[0] = o[1] = 0.0f;
    return;
  }
  const size_t at = static_cast<size_t>(b) * p.cap + i;
  const int32_t* pa = w.patch + 4 * b;
  const double c = 0.5 * p.P;
  double x = __dsub_rn(__dsub_rn(w.sxy[2 * at], static_cast<double>(pa[1])), c);
  double y = __dsub_rn(__dsub_rn(w.sxy[2 * at + 1], static_cast<double>(pa[2])), c);
  for (int r = 0; r < pa[3]; ++r) {   // (x, y) -> (y, -x): dataset.py:219-224 in image (x, y)
    const double t = x;
    x = y;
    y = -t;
  }
  x = __dadd_rn(x, c);
  y = __dadd_rn(y, c);
  o[0] = __double2float_rn(__dadd_rn(x, w.noise[2 * at]));
  o[1] = __double2float_rn(__dadd_rn(y, w.noise[2 * at + 1]));
}

unsigned grid_of(long long n, int block) { return static_cast<unsigned>((n + block - 1) / block); }

}  // namespace

struct samroad_labels_ctx {
  SamRoadLabelCfg cfg;
  int device = 0;
  std::vector<SceneDev> scenes;
  std::vector<void*> allocs;
  SceneDev* d_scenes = nullptr;
  int d_scenes_n = -1;
  int B_alloc = 0;
  void* work_mem = nullptr;
  Work work{};
  int32_t* h_read = nullptr;   // pinned [1 + B]: status word, then the survivor counts
  size_t smem_patch = 0;
};

namespace {

int cfg_check(const SamRoadLabelCfg* c) {
  SRB_REQUIRE(c != nullptr, "labels: null configuration");
  SRB_REQUIRE(c->patch_size >= 1 && c->image_size >= 1 && c->sample_margin >= 0 &&
                  c->patch_size + 2 * static_cast<long long>(c->sample_margin) <= c->image_size,
              "labels: PATCH_SIZE %d with margin %d does not fit a %d-pixel scene", c->patch_size,
              c->sample_margin, c->image_size);
  SRB_REQUIRE(c->topo_sample_num >= 1, "labels: TOPO_SAMPLE_NUM must be >= 1 (got %d)", c->topo_sample_num);
  SRB_REQUIRE(c->max_neighbor_queries >= 1 && c->max_neighbor_queries <= 32,
              "labels: MAX_NEIGHBOR_QUERIES must be in 1..32 (got %d)", c->max_neighbor_queries);
  SRB_REQUIRE(std::isfinite(c->road_nms_radius) && c->road_nms_radius > 0.0,
              "labels: ROAD_NMS_RADIUS must be a positive number (got %g)", c->road_nms_radius);
  SRB_REQUIRE(std::isfinite(c->neighbor_radius) && c->neighbor_radius > 0.0,
              "labels: NEIGHBOR_RADIUS must be a positive number (got %g)", c->neighbor_radius);
  SRB_REQUIRE(std::floor(c->neighbor_radius / 4.0) <= static_cast<double>(INT_MAX),
              "labels: NEIGHBOR_RADIUS %g gives a BFS depth NEIGHBOR_RADIUS // 4 beyond %d", c->neighbor_radius,
              INT_MAX);
  SRB_REQUIRE(c->max_patch_points >= 1, "labels: max_patch_points must be >= 1 (got %d)", c->max_patch_points);
  return 0;
}

Params make_params(const samroad_labels_ctx* L) {
  const SamRoadLabelCfg& c = L->cfg;
  Params p;
  p.scenes = L->d_scenes;
  p.n_scenes = static_cast<int>(L->scenes.size());
  p.P = c.patch_size;
  p.size = c.image_size;
  p.lo = c.sample_margin;
  p.hi = c.image_size - c.patch_size - c.sample_margin;
  p.S = c.topo_sample_num;
  p.Np = c.max_neighbor_queries;
  p.depth = static_cast<int>(std::floor(c.neighbor_radius / 4.0));
  p.cap = c.max_patch_points;
  p.cell = std::max(c.road_nms_radius, c.patch_size / static_cast<double>(kMaxCells - 1));
  p.ncell = std::min(static_cast<int>(std::floor(c.patch_size / p.cell)) + 1, kMaxCells);
  p.r_nms2 = c.road_nms_radius * c.road_nms_radius;
  p.r_nbr2 = c.neighbor_radius * c.neighbor_radius;
  return p;
}

int ensure_work(samroad_labels_ctx* L, int B) {
  if (L->d_scenes_n != static_cast<int>(L->scenes.size())) {
    if (L->d_scenes) cudaFree(L->d_scenes);
    L->d_scenes = nullptr;
    SRB_CUDA_OK(cudaMalloc(&L->d_scenes, sizeof(SceneDev) * L->scenes.size()));
    SRB_CUDA_OK(cudaMemcpy(L->d_scenes, L->scenes.data(), sizeof(SceneDev) * L->scenes.size(),
                           cudaMemcpyHostToDevice));
    L->d_scenes_n = static_cast<int>(L->scenes.size());
  }
  if (B <= L->B_alloc) return 0;
  if (L->work_mem) cudaFree(L->work_mem);
  if (L->h_read) cudaFreeHost(L->h_read);
  L->work_mem = nullptr;
  L->h_read = nullptr;
  L->B_alloc = 0;
  const size_t cap = L->cfg.max_patch_points, S = L->cfg.topo_sample_num, nb = B;
  // the last region is the status word followed by nsurv [B], so that one copy of 1 + B words reads both for
  // any batch up to B_alloc (a status word after nsurv [B_alloc] would be missed by smaller batches)
  const size_t bytes[] = {16 * nb, 8 * cap * nb, 8 * S * nb, 16 * cap * nb, 4 * cap * nb, 4 * cap * nb,
                          16 * cap * nb, 8 * cap * nb, 4 * S * nb, 4 * (nb + 1)};
  size_t total = 0;
  for (size_t x : bytes) total += (x + 255) & ~static_cast<size_t>(255);
  SRB_CUDA_OK(cudaMalloc(&L->work_mem, total));
  SRB_CUDA_OK(cudaMallocHost(&L->h_read, sizeof(int32_t) * (B + 1)));
  char* q = static_cast<char*>(L->work_mem);
  void* ptrs[10];
  for (int i = 0; i < 10; ++i) {
    ptrs[i] = q;
    q += (bytes[i] + 255) & ~static_cast<size_t>(255);
  }
  Work& w = L->work;
  w.patch = static_cast<int32_t*>(ptrs[0]);
  w.score_u = static_cast<double*>(ptrs[1]);
  w.src_u = static_cast<double*>(ptrs[2]);
  w.noise = static_cast<double*>(ptrs[3]);
  w.cand = static_cast<int32_t*>(ptrs[4]);
  w.surv = static_cast<int32_t*>(ptrs[5]);
  w.sxy = static_cast<double*>(ptrs[6]);
  w.cdf = static_cast<double*>(ptrs[7]);
  w.src = static_cast<int32_t*>(ptrs[8]);
  w.status = static_cast<int32_t*>(ptrs[9]);
  w.nsurv = w.status + 1;
  L->B_alloc = B;
  return 0;
}

int run_batch(samroad_labels_ctx* L, int B, unsigned long long seed, const int32_t* patches, const double* score_u,
              const double* src_u, const double* noise, bool injected, void* const* export_to, float* rgb, float* kp, float* road,
              float* points, int32_t* pairs, uint8_t* connected, uint8_t* valid, int32_t* n_points, void* stream,
              const char* what) {
  SRB_REQUIRE(L != nullptr, "%s: null labels object", what);
  SRB_REQUIRE(B >= 1, "%s: batch size must be >= 1 (got %d)", what, B);
  SRB_REQUIRE(!L->scenes.empty(), "%s: no scene uploaded", what);
  SRB_REQUIRE(rgb && kp && road && points && pairs && connected && valid && n_points, "%s: null output", what);
  SRB_CUDA_OK(cudaSetDevice(L->device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (int rc = ensure_work(L, B)) return rc;
  Work w = L->work;
  const Params p = make_params(L);
  const size_t cap = p.cap, S = p.S;
  if (injected) {   // caller-filled draws: copied into the batch arrays, the stages below are unchanged
    SRB_CUDA_OK(cudaMemcpyAsync(w.patch, patches, 16 * B, cudaMemcpyDefault, st));
    SRB_CUDA_OK(cudaMemcpyAsync(w.score_u, score_u, 8 * cap * B, cudaMemcpyDefault, st));
    SRB_CUDA_OK(cudaMemcpyAsync(w.src_u, src_u, 8 * S * B, cudaMemcpyDefault, st));
    SRB_CUDA_OK(cudaMemcpyAsync(w.noise, noise, 16 * cap * B, cudaMemcpyDefault, st));
  } else {
    if (patches) SRB_CUDA_OK(cudaMemcpyAsync(w.patch, patches, 16 * B, cudaMemcpyDefault, st));
    const unsigned gx = std::min<unsigned>(grid_of(std::max(p.cap, p.S), 256), 64u);
    draw_kernel<<<dim3(gx, B), 256, 0, st>>>(w, p, patches == nullptr, seed);
    note_launch(1);
  }
  SRB_CUDA_OK(cudaMemsetAsync(w.status, 0, sizeof(int32_t), st));
  crop_kernel<<<dim3(grid_of(static_cast<long long>(p.P) * p.P, 256), B), 256, 0, st>>>(p, w.patch, rgb, kp, road);
  patch_kernel<<<B, kPatchThreads, L->smem_patch, st>>>(p, w);
  pairs_kernel<<<dim3(grid_of(p.S, kPairWarps), B), 32 * kPairWarps, sizeof(BfsSmem) * kPairWarps, st>>>(
      p, w, pairs, connected, valid);
  SRB_CUDA_OK(cudaGetLastError());
  note_launch(3);
  SRB_CUDA_OK(cudaMemcpyAsync(L->h_read, w.status, sizeof(int32_t) * (B + 1), cudaMemcpyDeviceToHost, st));
  SRB_CUDA_OK(cudaStreamSynchronize(st));
  const int status = L->h_read[0];
  SRB_REQUIRE(!(status & kBadPatch), "%s: a patch names a missing scene, an origin outside [%d, %d] or a "
              "rotation outside 0..3", what, p.lo, p.hi);
  SRB_REQUIRE(!(status & kOverCap), "%s: a patch holds more than max_patch_points=%d candidates", what, p.cap);
  SRB_REQUIRE(!(status & kBfsOverflow), "%s: a BFS reached more than %d nodes within NEIGHBOR_RADIUS // 4 = %d "
              "steps", what, kBfsList, p.depth);
  int N = 1;
  for (int b = 0; b < B; ++b) N = std::max(N, L->h_read[1 + b]);
  points_kernel<<<dim3(grid_of(N, 128), B), 128, 0, st>>>(p, w, N, points);
  SRB_CUDA_OK(cudaGetLastError());
  note_launch(1);
  if (export_to) {
    SRB_CUDA_OK(cudaMemcpyAsync(export_to[0], w.patch, 16 * B, cudaMemcpyDefault, st));
    SRB_CUDA_OK(cudaMemcpyAsync(export_to[1], w.score_u, 8 * cap * B, cudaMemcpyDefault, st));
    SRB_CUDA_OK(cudaMemcpyAsync(export_to[2], w.src_u, 8 * S * B, cudaMemcpyDefault, st));
    SRB_CUDA_OK(cudaMemcpyAsync(export_to[3], w.noise, 16 * cap * B, cudaMemcpyDefault, st));
  }
  *n_points = N;
  return 0;
}

}  // namespace

extern "C" int samroad_labels_create(int device, const SamRoadLabelCfg* cfg, samroad_labels_t* out) {
  SRB_REQUIRE(out != nullptr, "samroad_labels_create: null argument");
  if (int rc = cfg_check(cfg)) return rc;
  const size_t smem = patch_smem_bytes(cfg->max_patch_points);
  int ndev = 0;
  SRB_CUDA_OK(cudaGetDeviceCount(&ndev));
  SRB_REQUIRE(ndev > 0, "no CUDA device: libsamroad_b200 has no CPU fallback");
  SRB_REQUIRE(device >= 0 && device < ndev, "device %d out of range (0..%d)", device, ndev - 1);
  SRB_CUDA_OK(cudaSetDevice(device));
  int optin = 0;
  SRB_CUDA_OK(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device));
  SRB_REQUIRE(smem + 32 * 4 + 64 <= static_cast<size_t>(optin),
              "samroad_labels_create: a patch window holds up to %d labelled points; the on-chip NMS of one patch "
              "takes %zu bytes of shared memory and this device allows %d", cfg->max_patch_points, smem, optin);
  SRB_CUDA_OK(cudaFuncSetAttribute(patch_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
  SRB_CUDA_OK(cudaFuncSetAttribute(pairs_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   static_cast<int>(sizeof(BfsSmem) * kPairWarps)));
  samroad_labels_ctx* L = new samroad_labels_ctx();
  L->cfg = *cfg;
  L->device = device;
  L->smem_patch = smem;
  *out = L;
  return 0;
}

extern "C" int samroad_labels_destroy(samroad_labels_t L) {
  if (!L) return 0;
  cudaSetDevice(L->device);
  cudaDeviceSynchronize();
  for (void* a : L->allocs) cudaFree(a);
  if (L->d_scenes) cudaFree(L->d_scenes);
  if (L->work_mem) cudaFree(L->work_mem);
  if (L->h_read) cudaFreeHost(L->h_read);
  delete L;
  return 0;
}

extern "C" int samroad_labels_upload(samroad_labels_t L, const uint8_t* rgb, const uint8_t* keypoint_mask,
                                     const uint8_t* road_mask, int32_t n_points, const double* points,
                                     const uint8_t* flags, const float* weights, const int32_t* adj_start,
                                     const int32_t* adj, int32_t* scene_index) {
  SRB_REQUIRE(L != nullptr, "samroad_labels_upload: null labels object");
  SRB_REQUIRE(rgb && keypoint_mask && road_mask && points && flags && weights && adj_start && scene_index,
              "samroad_labels_upload: null argument");
  SRB_REQUIRE(n_points >= 1, "samroad_labels_upload: a scene needs at least one graph point (got %d)", n_points);
  SRB_REQUIRE(adj_start[0] == 0, "samroad_labels_upload: adjacency offsets must start at 0");
  for (int32_t i = 0; i < n_points; ++i) {
    SRB_REQUIRE(adj_start[i + 1] >= adj_start[i], "samroad_labels_upload: adjacency offsets decrease at %d", i);
    SRB_REQUIRE(std::isfinite(points[2 * i]) && std::isfinite(points[2 * i + 1]),
                "samroad_labels_upload: point %d is not finite", i);
    // np.random.choice(p=w / w.sum()) refuses a window whose weights are all zero; the running sum would
    // silently pick its last survivor, so every weight must be positive
    SRB_REQUIRE(std::isfinite(weights[i]) && weights[i] > 0.0f,
                "samroad_labels_upload: weight %d is not a positive finite number (got %g)", i,
                static_cast<double>(weights[i]));
  }
  const int32_t m = adj_start[n_points];
  SRB_REQUIRE(m == 0 || adj != nullptr, "samroad_labels_upload: null adjacency");
  for (int32_t e = 0; e < m; ++e)
    SRB_REQUIRE(adj[e] >= 0 && adj[e] < n_points, "samroad_labels_upload: neighbour %d out of range", adj[e]);
  SRB_CUDA_OK(cudaSetDevice(L->device));
  const size_t px = static_cast<size_t>(L->cfg.image_size) * L->cfg.image_size;
  const size_t sizes[] = {16 * static_cast<size_t>(n_points), static_cast<size_t>(n_points),
                          4 * static_cast<size_t>(n_points), 4 * (static_cast<size_t>(n_points) + 1),
                          4 * static_cast<size_t>(m > 0 ? m : 1), 3 * px, px, px};
  const void* src[] = {points, flags, weights, adj_start, adj, rgb, keypoint_mask, road_mask};
  void* dst[8];
  for (int i = 0; i < 8; ++i) {
    SRB_CUDA_OK(cudaMalloc(&dst[i], sizes[i]));
    L->allocs.push_back(dst[i]);
    if (src[i] && !(i == 4 && m == 0)) SRB_CUDA_OK(cudaMemcpy(dst[i], src[i], sizes[i], cudaMemcpyHostToDevice));
  }
  SceneDev s;
  s.pts = static_cast<const double*>(dst[0]);
  s.flags = static_cast<const uint8_t*>(dst[1]);
  s.weight = static_cast<const float*>(dst[2]);
  s.adj_start = static_cast<const int32_t*>(dst[3]);
  s.adj = static_cast<const int32_t*>(dst[4]);
  s.rgb = static_cast<const uint8_t*>(dst[5]);
  s.kp = static_cast<const uint8_t*>(dst[6]);
  s.road = static_cast<const uint8_t*>(dst[7]);
  s.n = n_points;
  L->scenes.push_back(s);
  *scene_index = static_cast<int32_t>(L->scenes.size()) - 1;
  return 0;
}

extern "C" int samroad_labels_batch(samroad_labels_t L, int B, uint64_t seed, const int32_t* patches, float* rgb,
                                    float* keypoint_mask, float* road_mask, float* points, int32_t* pairs,
                                    uint8_t* connected, uint8_t* valid, int32_t* n_points, void* stream) {
  return run_batch(L, B, seed, patches, nullptr, nullptr, nullptr, false, nullptr, rgb, keypoint_mask, road_mask,
                   points, pairs, connected, valid, n_points, stream, "samroad_labels_batch");
}

extern "C" int samroad_debug_labels_batch_draws(samroad_labels_t L, int B, int mode, uint64_t seed, int32_t* patches,
                                                double* score_u, double* source_u, double* noise, float* rgb,
                                                float* keypoint_mask, float* road_mask, float* points, int32_t* pairs,
                                                uint8_t* connected, uint8_t* valid, int32_t* n_points, void* stream) {
  SRB_REQUIRE(mode == 0 || mode == 1, "samroad_debug_labels_batch_draws: mode must be 0 (inject) or 1 (export)");
  SRB_REQUIRE(patches && score_u && source_u && noise, "samroad_debug_labels_batch_draws: null draw array");
  if (mode == 0)
    return run_batch(L, B, 0, patches, score_u, source_u, noise, true, nullptr, rgb, keypoint_mask, road_mask, points,
                     pairs, connected, valid, n_points, stream, "samroad_debug_labels_batch_draws");
  void* const to[4] = {patches, score_u, source_u, noise};
  return run_batch(L, B, seed, nullptr, nullptr, nullptr, nullptr, false, to, rgb, keypoint_mask, road_mask, points,
                   pairs, connected, valid, n_points, stream, "samroad_debug_labels_batch_draws");
}
