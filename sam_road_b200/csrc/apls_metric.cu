// sam_road_b200 :: the APLS graph metric on the device (DESIGN.md §15).
//
// Reference: cityscale_metrics/apls/main.go (spacenet_metrics/apls/main.go differs only in its small-tile
// parameters).  The host (sam_road_b200/apls_metric.py) converts and densifies both graphs, computes every directed
// arc weight int(GPSDistance(u, v) * 100.0) once, selects the control points and runs the greedy one-to-one
// snapping.  This file takes the three stages that are quadratic or worse:
//
//   knn_kernel     snapping candidates: one warp per control point over all nodes of the other graph, the 10
//                  nearest under squared distance to the node's +-1e-6 degree box, ties by ascending node id
//                  (each lane keeps a sorted top 10 of its strided nodes, then 10 warp-wide arg-min rounds).
//   sssp_kernel    exact integer shortest paths from every source on both graphs of a direction.  Chains of
//                  degree-2 nodes are contracted into one arc per direction on the library's host side (the
//                  distances are integer sums, so they are unchanged); one CTA per source relaxes the contracted
//                  graph round by round from a frontier, with its distances in shared memory when they fit.  The
//                  shortest distance is unique, so the order of the relaxations does not matter.
//   pair_kernel    the pair score over every unordered pair of control points: the counts per rule and the sum of
//                  the terms as a 192-bit fixed-point integer (LSB 2^-128), added exactly; the host rounds it once.
//
// Compiled with -fmad=false: the candidate distance and the pair term are the host's and the oracle's float64
// expressions operation by operation.  No float atomics: two runs are bitwise equal.
#include "../../include/samroad_b200.h"

#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

#include "common.cuh"

using namespace srb;

namespace {

constexpr int kK = SAMROAD_APLS_CANDIDATES;
constexpr double kBoxTol = 0.000001;     // main.go `tol`: each proposal node is indexed as a +-1e-6 box
constexpr int32_t kInf = 0x7fffffff;
constexpr int kSsspThreads = 512;
constexpr int kPairThreads = 256;
constexpr int kKnnWarps = 8;
enum : uint32_t { kBadTerm = 1 };

// Squared distance from q to the box [x - tol, x + tol] in raw degree space (longitude not scaled)
__device__ __forceinline__ double box_d2(double q0, double q1, double x0, double x1) {
  const double lo0 = x0 - kBoxTol, hi0 = x0 + kBoxTol, lo1 = x1 - kBoxTol, hi1 = x1 + kBoxTol;
  const double d0 = q0 < lo0 ? lo0 - q0 : (q0 > hi0 ? q0 - hi0 : 0.0);
  const double d1 = q1 < lo1 ? lo1 - q1 : (q1 > hi1 ? q1 - hi1 : 0.0);
  return d0 * d0 + d1 * d1;
}

__device__ __forceinline__ bool key_less(double da, int32_t ia, double db, int32_t ib) {
  return da < db || (da == db && ia < ib);
}

__global__ void __launch_bounds__(32 * kKnnWarps) knn_kernel(const double* __restrict__ ll, int32_t n,
                                                             const double* __restrict__ q, int32_t nq,
                                                             int32_t* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int query = blockIdx.x * kKnnWarps + (threadIdx.x >> 5);
  if (query >= nq) return;
  const double q0 = q[2 * query], q1 = q[2 * query + 1];
  double bd[kK];
  int32_t bi[kK];
#pragma unroll
  for (int k = 0; k < kK; ++k) {
    bd[k] = INFINITY;
    bi[k] = INT32_MAX;
  }
  for (int32_t v = lane; v < n; v += 32) {
    const double d = box_d2(q0, q1, ll[2 * v], ll[2 * v + 1]);
    if (!key_less(d, v, bd[kK - 1], bi[kK - 1])) continue;
    // insertion into the sorted list; fully unrolled so the list stays in registers
    double cd = d;
    int32_t ci = v;
#pragma unroll
    for (int k = 0; k < kK; ++k) {
      if (key_less(cd, ci, bd[k], bi[k])) {
        const double td = bd[k];
        const int32_t ti = bi[k];
        bd[k] = cd;
        bi[k] = ci;
        cd = td;
        ci = ti;
      }
    }
  }
  // merge: each round the lane holding the smallest head hands it out and shifts its list
#pragma unroll 1
  for (int r = 0; r < kK; ++r) {
    double md = bd[0];
    int32_t mi = bi[0];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const double od = __shfl_xor_sync(0xffffffffu, md, o);
      const int32_t oi = __shfl_xor_sync(0xffffffffu, mi, o);
      if (key_less(od, oi, md, mi)) {
        md = od;
        mi = oi;
      }
    }
    if (lane == 0) out[kK * query + r] = mi == INT32_MAX ? -1 : mi;
    if (mi != INT32_MAX && bi[0] == mi) {   // node ids are unique, so exactly one lane matches
#pragma unroll
      for (int k = 0; k < kK - 1; ++k) {
        bd[k] = bd[k + 1];
        bi[k] = bi[k + 1];
      }
      bd[kK - 1] = INFINITY;
      bi[kK - 1] = INT32_MAX;
    }
  }
}

struct SsspGraph {
  const int32_t* off;     // [nt + 1] contracted CSR over terminal indices
  const int32_t* dst;
  const int32_t* w;
  const int32_t* src;     // [nsrc] terminal index of each source (sources are also the targets)
  int32_t* mat;           // [nsrc, nsrc] out: cm, -1 when unreachable
  int32_t nt, nsrc;
};

// A CTA's shortest-path scratch for nt terminals: distances and two frontier flag arrays
struct SsspScratch {
  int32_t* dist;
  uint8_t* fa;
  uint8_t* fb;
};
__host__ __device__ inline SsspScratch sssp_scratch(Layout& L, int32_t nt) {
  SsspScratch s;
  s.dist = L.take<int32_t>(nt);
  s.fa = L.take<uint8_t>(nt);
  s.fb = L.take<uint8_t>(nt);
  return s;
}

// One CTA per (graph, source), grid-stride.  dist / two frontier flag arrays live in dynamic shared memory when
// `scratch` is null, else in the CTA's slice of it.
__global__ void __launch_bounds__(kSsspThreads) sssp_kernel(SsspGraph g0, SsspGraph g1, char* scratch,
                                                            size_t scratch_per_cta) {
  extern __shared__ __align__(16) char smem[];
  char* base = scratch ? scratch + scratch_per_cta * blockIdx.x : smem;
  const int njobs = g0.nsrc + g1.nsrc;
  for (int job = blockIdx.x; job < njobs; job += gridDim.x) {
    const SsspGraph& g = job < g0.nsrc ? g0 : g1;
    const int s = job < g0.nsrc ? job : job - g0.nsrc;
    Layout L(base);
    const SsspScratch sc = sssp_scratch(L, g.nt);
    int32_t* dist = sc.dist;
    uint8_t* fa = sc.fa;
    uint8_t* fb = sc.fb;
    for (int i = threadIdx.x; i < g.nt; i += blockDim.x) {
      dist[i] = kInf;
      fa[i] = 0;
      fb[i] = 0;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      dist[g.src[s]] = 0;
      fa[g.src[s]] = 1;
    }
    __syncthreads();
    volatile int32_t* vdist = dist;
    bool more = true;
    while (more) {
      int any = 0;
      for (int i = threadIdx.x; i < g.nt; i += blockDim.x) {
        if (!fa[i]) continue;
        fa[i] = 0;
        const int32_t d = vdist[i];
        for (int32_t e = g.off[i]; e < g.off[i + 1]; ++e) {
          const int32_t v = g.dst[e];
          const int32_t nd = d + g.w[e];    // below 2^31: the upload refuses a graph whose weights could exceed it
          if (nd < vdist[v] && nd < atomicMin(dist + v, nd)) {
            fb[v] = 1;
            any = 1;
          }
        }
      }
      more = __syncthreads_or(any);
      uint8_t* t = fa;
      fa = fb;
      fb = t;
    }
    for (int j = threadIdx.x; j < g.nsrc; j += blockDim.x) {
      const int32_t d = dist[g.src[j]];
      g.mat[static_cast<size_t>(s) * g.nsrc + j] = d == kInf ? -1 : d;
    }
    __syncthreads();
  }
}

struct PairPartial {
  unsigned long long fx[3];       // sum of the terms, LSB 2^-128
  long long penalty, skipped, scored;
  unsigned int status;
  unsigned int pad;
};

__device__ __forceinline__ void add192(unsigned long long* w, int word, unsigned long long lo, unsigned long long hi) {
  unsigned long long c = 0;
  const unsigned long long a = w[word] + lo;
  c = a < lo;
  w[word] = a;
  if (word + 1 < 3) {
    const unsigned long long b = w[word + 1] + hi;
    const unsigned long long c1 = b < hi;
    w[word + 1] = b + c;
    c = c1 | (w[word + 1] < c);
    if (word + 2 < 3) w[word + 2] += c;
  }
}

// Adds a double s in [0, 1] exactly; false when s has a bit below 2^-128
__device__ __forceinline__ bool add_fixed(unsigned long long* w, double s) {
  const unsigned long long bits = static_cast<unsigned long long>(__double_as_longlong(s));
  const int ex = static_cast<int>((bits >> 52) & 0x7ff);
  unsigned long long mant = bits & ((1ull << 52) - 1);
  if (ex == 0) return mant == 0;
  mant |= 1ull << 52;
  int shift = ex - 1075 + 128;   // s = mant * 2^(ex - 1075)
  while (shift < 0 && !(mant & 1)) {
    mant >>= 1;
    ++shift;
  }
  if (shift < 0) return false;
  const int word = shift >> 6, off = shift & 63;
  const unsigned long long lo = mant << off, hi = off ? mant >> (64 - off) : 0ull;
  add192(w, word, lo, hi);
  return true;
}

__global__ void __launch_bounds__(kPairThreads) pair_kernel(int32_t n_cp, const int32_t* __restrict__ gi,
                                                            const int32_t* __restrict__ pi,
                                                            const int32_t* __restrict__ dg, int32_t ng,
                                                            const int32_t* __restrict__ dp, int32_t np_,
                                                            double filter, PairPartial* part) {
  unsigned long long fx[3] = {0, 0, 0};
  long long pen = 0, skip = 0, sc = 0;
  unsigned int status = 0;
  for (int i = blockIdx.x; i < n_cp; i += gridDim.x) {
    const int32_t a = gi[i];
    for (int j = i + 1 + threadIdx.x; j < n_cp; j += blockDim.x) {
      const int32_t b = gi[j];
      if (a < 0 || b < 0) {
        ++pen;
        continue;
      }
      const double d1 = static_cast<double>(dg[static_cast<size_t>(a) * ng + b]) / 100.0;
      if (!(d1 > filter)) {
        ++skip;
        continue;
      }
      double d2 = static_cast<double>(dp[static_cast<size_t>(pi[i]) * np_ + pi[j]]) / 100.0;
      if (d2 < 0) d2 = 0;
      double s = fabs(d1 - d2) / d1;
      if (s > 1.0) s = 1.0;
      if (!add_fixed(fx, s)) status |= kBadTerm;
      ++sc;
    }
  }
  __shared__ PairPartial sp[kPairThreads];
  PairPartial& me = sp[threadIdx.x];
  me.fx[0] = fx[0];
  me.fx[1] = fx[1];
  me.fx[2] = fx[2];
  me.penalty = pen;
  me.skipped = skip;
  me.scored = sc;
  me.status = status;
  __syncthreads();
  if (threadIdx.x == 0) {
    PairPartial t = sp[0];
    for (int k = 1; k < kPairThreads; ++k) {
      add192(t.fx, 0, sp[k].fx[0], 0);
      add192(t.fx, 1, sp[k].fx[1], 0);
      t.fx[2] += sp[k].fx[2];
      t.penalty += sp[k].penalty;
      t.skipped += sp[k].skipped;
      t.scored += sp[k].scored;
      t.status |= sp[k].status;
    }
    part[blockIdx.x] = t;
  }
}

// The 192-bit value w * 2^-128, rounded once to the nearest double, ties to even
double round192(const unsigned long long* w) {
  int top = -1;
  for (int b = 191; b >= 0; --b)
    if ((w[b >> 6] >> (b & 63)) & 1ull) {
      top = b;
      break;
    }
  if (top < 0) return 0.0;
  auto bit = [&](int b) -> unsigned long long { return b < 0 ? 0ull : (w[b >> 6] >> (b & 63)) & 1ull; };
  unsigned long long m = 0;
  const int low = top - 52;   // lowest kept bit
  for (int b = top; b >= std::max(low, 0); --b) m = (m << 1) | bit(b);
  if (low <= 0) return std::ldexp(static_cast<double>(m), -128);   // exact: at most 53 bits
  const bool half = bit(low - 1);
  bool sticky = false;
  for (int b = low - 2; b >= 0 && !sticky; --b) sticky = bit(b);
  if (half && (sticky || (m & 1))) ++m;   // m may become 2^53: still exact in a double
  return std::ldexp(static_cast<double>(m), low - 128);
}

struct HostGraph {
  int32_t n = 0;
  std::vector<int32_t> off, col, w;
  std::vector<uint8_t> chain;            // 1: self-loops aside, out- and in-neighbours are the same two nodes
  std::vector<int32_t> nb0, nb1;         // those two neighbours
  std::vector<int32_t> w0, w1;           // the lightest arc to each
};

// The graph shortest paths run on: `src` nodes and every node that is not a chain node are terminals; each chain
// of chain nodes between two terminals becomes one arc per direction carrying the summed weight.
struct Contracted {
  std::vector<int32_t> off, dst, w, src;   // src: terminal index per source
};

bool contract(const HostGraph& g, const std::vector<int32_t>& sources, Contracted& c, std::vector<int32_t>& tid) {
  tid.assign(g.n, -1);
  int32_t nt = 0;
  for (int32_t v : sources)
    if (tid[v] < 0) tid[v] = -2;
  for (int32_t v = 0; v < g.n; ++v)
    if (tid[v] == -2 || !g.chain[v]) tid[v] = nt++;
  c.off.assign(nt + 1, 0);
  c.dst.clear();
  c.w.clear();
  int32_t t = 0;
  for (int32_t v = 0; v < g.n; ++v) {
    if (tid[v] < 0) continue;
    c.off[t++] = static_cast<int32_t>(c.dst.size());
    for (int32_t e = g.off[v]; e < g.off[v + 1]; ++e) {
      int32_t prev = v, cur = g.col[e];
      if (cur == v) continue;              // a self-loop never shortens a path
      int64_t sum = g.w[e];
      int64_t steps = 0;
      while (tid[cur] < 0) {               // a chain node: leave by the neighbour it was not entered from
        const bool first = g.nb0[cur] != prev;
        const int32_t nx = first ? g.nb0[cur] : g.nb1[cur];
        sum += first ? g.w0[cur] : g.w1[cur];
        prev = cur;
        cur = nx;
        if (++steps > g.n) return false;
      }
      c.dst.push_back(tid[cur]);
      c.w.push_back(static_cast<int32_t>(sum));
    }
  }
  c.off[nt] = static_cast<int32_t>(c.dst.size());
  c.src.resize(sources.size());
  for (size_t i = 0; i < sources.size(); ++i) c.src[i] = tid[sources[i]];
  return true;
}

}  // namespace

struct samroad_apls_ctx {
  int device = 0;
  SamRoadAplsCaps caps{};
  cudaStream_t stream = nullptr;   // the handle's own non-blocking stream: a call waits for its own work only
  HostGraph host[2];
  DeviceBuffer ll[2];                   // node lat/lon on the device, for the candidate search
  DeviceBuffer work;                    // per call: contracted graphs, matrices, partials; grown on demand
  std::vector<char> staging;            // host copy of the per-call inputs, sent in one transfer
  int smem_optin = 0;
};

extern "C" int samroad_apls_create(int device, const SamRoadAplsCaps* caps, samroad_apls_t* out) {
  SRB_REQUIRE(out != nullptr && caps != nullptr, "samroad_apls_create: null argument");
  SRB_REQUIRE(caps->max_nodes >= 1 && caps->max_arcs >= 1 && caps->max_control_points >= 1,
              "samroad_apls_create: capacities must be positive");
  SRB_REQUIRE(caps->max_nodes <= (1 << 26) && caps->max_arcs <= (1 << 28) && caps->max_control_points <= (1 << 16),
              "samroad_apls_create: a capacity is larger than this build supports");
  if (int rc = open_device(device)) return rc;
  int optin = 0;
  SRB_CUDA_OK(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device));
  SRB_TRY(allow_dynamic_smem(sssp_kernel, optin));
  cudaStream_t st = nullptr;
  SRB_CUDA_OK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
  samroad_apls_ctx* A = new samroad_apls_ctx();
  A->device = device;
  A->caps = *caps;
  A->stream = st;
  A->smem_optin = optin;
  *out = A;
  return 0;
}

extern "C" int samroad_apls_destroy(samroad_apls_t A) {
  if (!A) return 0;
  cudaSetDevice(A->device);
  cudaStreamSynchronize(A->stream);
  cudaStreamDestroy(A->stream);
  delete A;
  return 0;
}

extern "C" int samroad_apls_upload_graph(samroad_apls_t A, int which, int32_t n_nodes, const double* latlon,
                                         const int32_t* row_start, const int32_t* col, const int32_t* weight) {
  const char* what = "samroad_apls_upload_graph";
  SRB_REQUIRE(A != nullptr, "%s: null handle", what);
  SRB_REQUIRE(which == 0 || which == 1, "%s: which must be 0 (ground truth) or 1 (proposal)", what);
  SRB_REQUIRE(n_nodes >= 0, "%s: negative node count", what);
  SRB_REQUIRE(n_nodes <= A->caps.max_nodes, "%s: a graph of %d nodes exceeds max_nodes = %d", what, n_nodes,
              A->caps.max_nodes);
  SRB_REQUIRE(n_nodes == 0 || (latlon && row_start), "%s: null argument", what);
  const int32_t m = n_nodes ? row_start[n_nodes] : 0;
  if (n_nodes)
    if (int rc = check_csr(what, n_nodes, row_start, col)) return rc;
  SRB_REQUIRE(m <= A->caps.max_arcs, "%s: a graph of %d arcs exceeds max_arcs = %d", what, m, A->caps.max_arcs);
  SRB_REQUIRE(m == 0 || weight, "%s: null adjacency", what);
  int64_t total = 0;
  for (int32_t e = 0; e < m; ++e) {
    SRB_REQUIRE(weight[e] >= 0, "%s: arc %d has a negative weight", what, e);
    total += weight[e];
  }
  SRB_REQUIRE(total < INT32_MAX, "%s: the arc weights sum to %lld cm, so a distance could exceed int32", what,
              static_cast<long long>(total));
  for (int32_t i = 0; i < 2 * n_nodes; ++i)
    SRB_REQUIRE(std::isfinite(latlon[i]), "%s: node %d has a coordinate that is not finite", what, i / 2);
  SRB_CUDA_OK(cudaSetDevice(A->device));
  HostGraph& g = A->host[which];
  g.n = 0;
  if (n_nodes > 0) {   // calls are synchronous: nothing of this handle still reads the old buffer
    if (A->ll[which].reserve(16ull * n_nodes, what)) return 1;
    SRB_CUDA_OK(cudaMemcpyAsync(A->ll[which].get(), latlon, 16ull * n_nodes, cudaMemcpyHostToDevice, A->stream));
    SRB_CUDA_OK(cudaStreamSynchronize(A->stream));
  }
  g.off.assign(row_start, row_start + (n_nodes ? n_nodes + 1 : 0));
  g.col.assign(col, col + m);
  g.w.assign(weight, weight + m);
  g.chain.assign(n_nodes, 0);
  g.nb0.assign(n_nodes, -1);
  g.nb1.assign(n_nodes, -1);
  g.w0.assign(n_nodes, 0);
  g.w1.assign(n_nodes, 0);
  // a chain node v has, self-loops aside, exactly two distinct out-neighbours {a, b} and exactly the in-neighbours
  // {a, b}: a walk can then only enter v from a or b and leave by the other, so contracting it keeps every path.
  // The in-neighbours are collected first (up to two distinct ones; `in_more` marks a third).
  std::vector<int32_t> in0(n_nodes, -1), in1(n_nodes, -1);
  std::vector<uint8_t> in_more(n_nodes, 0);
  for (int32_t u = 0; u < n_nodes; ++u)
    for (int32_t e = g.off[u]; e < g.off[u + 1]; ++e) {
      const int32_t v = g.col[e];
      if (v == u || in_more[v]) continue;
      if (in0[v] < 0 || in0[v] == u) in0[v] = u;
      else if (in1[v] < 0 || in1[v] == u) in1[v] = u;
      else in_more[v] = 1;
    }
  for (int32_t v = 0; v < n_nodes; ++v) {
    int32_t a = -1, b = -1, wa = 0, wb = 0;
    bool ok = !in_more[v];
    for (int32_t e = g.off[v]; e < g.off[v + 1] && ok; ++e) {
      const int32_t u = g.col[e];
      if (u == v) continue;
      if (a < 0 || u == a) {
        wa = a < 0 ? g.w[e] : std::min(wa, g.w[e]);
        a = u;
      } else if (b < 0 || u == b) {
        wb = b < 0 ? g.w[e] : std::min(wb, g.w[e]);
        b = u;
      } else {
        ok = false;
      }
    }
    if (!ok || b < 0) continue;
    // at most two distinct in-neighbours: they are {a, b} exactly when both are among them
    const bool back_a = in0[v] == a || in1[v] == a, back_b = in0[v] == b || in1[v] == b;
    if (!back_a || !back_b) continue;
    g.chain[v] = 1;
    g.nb0[v] = a;
    g.nb1[v] = b;
    g.w0[v] = wa;
    g.w1[v] = wb;
  }
  g.n = n_nodes;
  return 0;
}

extern "C" int samroad_apls_candidates(samroad_apls_t A, int which, int32_t n_queries, const double* query_latlon,
                                       int32_t* out) {
  const char* what = "samroad_apls_candidates";
  SRB_REQUIRE(A != nullptr, "%s: null handle", what);
  SRB_REQUIRE(which == 0 || which == 1, "%s: which must be 0 or 1", what);
  SRB_REQUIRE(n_queries >= 0, "%s: negative query count", what);
  SRB_REQUIRE(n_queries <= A->caps.max_control_points, "%s: %d queries exceed max_control_points = %d", what,
              n_queries, A->caps.max_control_points);
  if (n_queries == 0) return 0;
  SRB_REQUIRE(query_latlon && out, "%s: null argument", what);
  for (int32_t i = 0; i < 2 * n_queries; ++i)
    SRB_REQUIRE(std::isfinite(query_latlon[i]), "%s: query %d is not finite", what, i / 2);
  const int32_t n = A->host[which].n;
  if (n == 0) {
    std::fill(out, out + static_cast<size_t>(kK) * n_queries, -1);
    return 0;
  }
  SRB_CUDA_OK(cudaSetDevice(A->device));
  double* dq = nullptr;
  int32_t* dout = nullptr;
  auto carve = [&](void* base) {
    Layout L(base);
    dq = L.take<double>(2ull * n_queries);
    dout = L.take<int32_t>(1ull * kK * n_queries);
    return L.bytes();
  };
  if (A->work.reserve(carve(nullptr), what)) return 1;
  carve(A->work.get());
  cudaStream_t st = A->stream;
  SRB_CUDA_OK(cudaMemcpyAsync(dq, query_latlon, 16ull * n_queries, cudaMemcpyHostToDevice, st));
  SRB_LAUNCH(knn_kernel, (n_queries + kKnnWarps - 1) / kKnnWarps, 32 * kKnnWarps, 0, st, A->ll[which].as<double>(), n,
             dq, n_queries, dout);
  SRB_CUDA_OK(cudaMemcpyAsync(out, dout, 4ull * kK * n_queries, cudaMemcpyDeviceToHost, st));
  SRB_CUDA_OK(cudaStreamSynchronize(st));
  return 0;
}

extern "C" int samroad_apls_one_way(samroad_apls_t A, int gt_role, int32_t n_cp, const int32_t* cp_gt,
                                    const int32_t* cp_match, double min_distance_filter, SamRoadAplsResult* out,
                                    int32_t* dist_gt, int32_t* dist_prop) {
  const char* what = "samroad_apls_one_way";
  SRB_REQUIRE(A != nullptr, "%s: null handle", what);
  SRB_REQUIRE(gt_role == 0 || gt_role == 1, "%s: gt_role must be 0 or 1", what);
  SRB_REQUIRE(out != nullptr, "%s: null result", what);
  SRB_REQUIRE(n_cp >= 0, "%s: negative control point count", what);
  SRB_REQUIRE(n_cp <= A->caps.max_control_points, "%s: %d control points exceed max_control_points = %d", what,
              n_cp, A->caps.max_control_points);
  SRB_REQUIRE(n_cp == 0 || (cp_gt && cp_match), "%s: null argument", what);
  SRB_REQUIRE(std::isfinite(min_distance_filter) && min_distance_filter >= 0.0,
              "%s: min_distance_filter must be finite and non-negative", what);
  const HostGraph& G = A->host[gt_role];
  const HostGraph& P = A->host[1 - gt_role];
  // sources: matched control points on the GT-role graph, their distinct matches on the other graph
  std::vector<int32_t> gi(n_cp, -1), pi(n_cp, -1), src_g, src_p;
  std::vector<int32_t> pslot(P.n, -1);
  for (int32_t i = 0; i < n_cp; ++i) {
    SRB_REQUIRE(cp_gt[i] >= 0 && cp_gt[i] < G.n, "%s: control point %d names node %d, outside its graph", what, i,
                cp_gt[i]);
    SRB_REQUIRE(i == 0 || cp_gt[i] > cp_gt[i - 1], "%s: control points must be in ascending node id (at %d)", what,
                i);
    const int32_t mt = cp_match[i];
    if (mt < 0) continue;
    SRB_REQUIRE(mt < P.n, "%s: control point %d is matched to node %d, outside the other graph", what, i, mt);
    gi[i] = static_cast<int32_t>(src_g.size());
    src_g.push_back(cp_gt[i]);
    if (pslot[mt] < 0) {
      pslot[mt] = static_cast<int32_t>(src_p.size());
      src_p.push_back(mt);
    }
    pi[i] = pslot[mt];
  }
  Contracted cg, cpr;
  std::vector<int32_t> tid;
  SRB_REQUIRE(contract(G, src_g, cg, tid) && contract(P, src_p, cpr, tid), "%s: a chain does not end", what);
  const int32_t ng = static_cast<int32_t>(src_g.size()), np_ = static_cast<int32_t>(src_p.size());
  const int32_t ntg = static_cast<int32_t>(cg.off.size()) - 1, ntp = static_cast<int32_t>(cpr.off.size()) - 1;

  SRB_CUDA_OK(cudaSetDevice(A->device));
  int sms = 0;
  SRB_CUDA_OK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, A->device));
  const int32_t ntmax = std::max(ntg, ntp);
  Layout cta(nullptr);
  sssp_scratch(cta, ntmax);
  const size_t per_cta = cta.bytes();
  const bool in_smem = per_cta <= static_cast<size_t>(A->smem_optin);
  const int njobs = ng + np_;
  int sssp_grid = std::max(1, std::min(njobs, 4 * sms));
  const int pair_grid = std::max(1, std::min(n_cp, 4 * sms));
  // device layout: contracted graphs, sources, per-cp indices, matrices, partials, and (global path) scratch
  const std::vector<int32_t>* arrs[] = {&cg.off, &cg.dst, &cg.w, &cg.src, &cpr.off, &cpr.dst, &cpr.w, &cpr.src, &gi,
                                        &pi};
  // device layout: contracted graphs, sources and per-cp indices (each at least one element, sent in one copy),
  // then the matrices, the partials and (global path) the scratch
  int32_t* dptr[10];
  int32_t *dmg = nullptr, *dmp = nullptr;
  PairPartial* dpart = nullptr;
  char* dscratch = nullptr;
  size_t staged = 0;
  auto carve = [&](void* base) {
    Layout L(base);
    for (int k = 0; k < 10; ++k) dptr[k] = L.take<int32_t>(std::max<size_t>(arrs[k]->size(), 1));
    staged = L.bytes();
    dmg = L.take<int32_t>(std::max<size_t>(1ull * ng * ng, 1));
    dmp = L.take<int32_t>(std::max<size_t>(1ull * np_ * np_, 1));
    dpart = L.take<PairPartial>(pair_grid);
    dscratch = L.take<char>(in_smem ? 0 : per_cta * sssp_grid);
    return L.bytes();
  };
  if (A->work.reserve(carve(nullptr), what)) return 1;
  char* base = A->work.as<char>();
  carve(base);
  if (in_smem) dscratch = nullptr;
  cudaStream_t st = A->stream;
  // one staging buffer, one copy
  A->staging.assign(staged, 0);
  for (int k = 0; k < 10; ++k)
    if (!arrs[k]->empty())
      std::memcpy(A->staging.data() + (reinterpret_cast<char*>(dptr[k]) - base), arrs[k]->data(), 4 * arrs[k]->size());
  SRB_CUDA_OK(cudaMemcpyAsync(base, A->staging.data(), staged, cudaMemcpyHostToDevice, st));
  SsspGraph s0{dptr[0], dptr[1], dptr[2], dptr[3], dmg, ntg, ng};
  SsspGraph s1{dptr[4], dptr[5], dptr[6], dptr[7], dmp, ntp, np_};
  if (njobs > 0) {
    SRB_LAUNCH(sssp_kernel, sssp_grid, kSsspThreads, in_smem ? per_cta : 0, st, s0, s1, dscratch, per_cta);
  }
  SRB_LAUNCH(pair_kernel, pair_grid, kPairThreads, 0, st, n_cp, dptr[8], dptr[9], dmg, ng, dmp, np_,
             min_distance_filter, dpart);
  std::vector<PairPartial> part(pair_grid);
  SRB_CUDA_OK(cudaMemcpyAsync(part.data(), dpart, sizeof(PairPartial) * pair_grid, cudaMemcpyDeviceToHost, st));
  if (dist_gt && ng) SRB_CUDA_OK(cudaMemcpyAsync(dist_gt, dmg, 4ull * ng * ng, cudaMemcpyDeviceToHost, st));
  if (dist_prop && np_) SRB_CUDA_OK(cudaMemcpyAsync(dist_prop, dmp, 4ull * np_ * np_, cudaMemcpyDeviceToHost, st));
  SRB_CUDA_OK(cudaStreamSynchronize(st));
  SamRoadAplsResult r{};
  unsigned long long w[3] = {0, 0, 0};
  unsigned int status = 0;
  for (const PairPartial& p : part) {
    const unsigned long long a = w[0] + p.fx[0];
    const unsigned long long c0 = a < p.fx[0];
    w[0] = a;
    const unsigned long long b = w[1] + p.fx[1];
    const unsigned long long c1 = b < p.fx[1];
    w[1] = b + c0;
    const unsigned long long c2 = c1 | (w[1] < c0);
    w[2] += p.fx[2] + c2;
    r.penalty += p.penalty;
    r.skipped += p.skipped;
    r.scored += p.scored;
    status |= p.status;
  }
  SRB_REQUIRE(!(status & kBadTerm), "%s: a pair term has a bit below 2^-128, which the exact sum cannot hold", what);
  w[2] += static_cast<unsigned long long>(r.penalty);   // each penalty pair adds exactly 1
  r.pairs = static_cast<int64_t>(n_cp) * (n_cp - 1) / 2;
  r.cc = r.penalty + r.scored;
  std::copy(w, w + 3, r.sum_fixed);
  r.sum = round192(w);
  r.n_sources_gt = ng;
  r.n_sources_prop = np_;
  r.terminals_gt = ntg;
  r.terminals_prop = ntp;
  *out = r;
  return 0;
}
