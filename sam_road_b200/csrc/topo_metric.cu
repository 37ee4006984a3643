// sam_road_b200 :: the TOPO graph metric on the device (DESIGN.md §14).
//
// Reference: cityscale_metrics/topo/topo.py TOPOWithPairs and graph.py RoadGraph.TOPOWalk.  The host
// (sam_road_b200/topo_metric.py) builds both graphs, the starting points and the (GT, proposal) pairs and uploads
// them; this file runs, for every pair, what TOPOWithPairs does between picking the pair and writing its line:
//
//   walk_kernel    one warp per walk, grid (pair slot, walk): walk 0 places the marbles on the proposal graph,
//                  walk 1 the holes on the GT graph, walk 2 the bidirectional holes on the GT graph.  Each walk is
//                  the reference's FIFO label-correcting traversal, run by all 32 lanes in lockstep (every lane
//                  computes the same scalars, lane 0 stores); the lanes split the exact-tuple de-duplication scan
//                  of the marble list.  The queue, the covered-edge map and the marbles live in global memory;
//                  the node distances are a dense map per slot, stamped with the chunk's serial.
//   match_kernel   one block per pair: candidate edges (the rtree box test, distance < threshold, the
//                  latlonNorm angle test) built as two CSR adjacencies by a block-wide two-pass count / scan /
//                  fill, then a maximum matching on each (augmenting paths from a greedy start; the size of a
//                  maximum matching is unique, so it equals what Hopcroft-Karp returns).
//
// Every float64 operation is the reference's, in its order; this file is compiled with -fmad=false so nothing
// is contracted into an FMA.  sqrt and division are IEEE.  cos of a node's latitude comes from the host; cos of
// an interpolated latitude (a marble's, for the candidate distance) is CUDA's cos.  No atomics: each pair's
// counts are a deterministic function of its inputs.  A walk or a pair past a capacity sets a status bit and
// the run is refused, never truncated.
#include "../../include/samroad_b200.h"

#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

#include "common.cuh"

using namespace srb;

namespace {

constexpr double kDegToRad = 0.017453292519943295;   // CPython's degToRad = pi / 180.0
constexpr double kTwin = 0.00001;                     // the bidirectional twin's offset and the index box half-side
constexpr int kMatchThreads = 256;
enum : int32_t { kOverMarbles = 1, kOverQueue = 2, kOverCovered = 4, kOverCand = 8 };

struct GraphDev {
  const double* ll = nullptr;      // [n, 2] (lat, lon)
  const double* cosl = nullptr;    // [n] math.cos(math.radians(lat)) from the host
  const int32_t* ls = nullptr;     // [n + 1] / li: nodeLink CSR, in the reference's list order
  const int32_t* li = nullptr;
  const int32_t* rs = nullptr;     // [n + 1] / ri: nodeLinkReverse CSR
  const int32_t* ri = nullptr;
  int32_t n = 0;
};

struct QEntry {
  int32_t node, prev;
  double dist;
};

struct WalkWs {          // one walk of one slot
  double4* marbles;      // [cap_marbles] (lat, lon, dlat, dlon)
  QEntry* queue;         // [cap_queue] ring
  uint64_t* ckey;        // [hash] covered-edge keys (cur << 32 | next)
  double* cval;          // [hash]
  uint32_t* cstamp;      // [hash]
  double* dist;          // [n of the walked graph]
  uint32_t* dstamp;      // [n]
};

struct Params {
  GraphDev prop, gt;
  const int32_t* pn;     // [npairs, 4] gpsn1, gpsn2, osmn1, osmn2
  const double* pd;      // [npairs, 4] gpsd1, gpsd2, osmd1, osmd2
  int32_t* out;          // [npairs, 6] marbles, holes, holes_bidirection, matched (precision), matched (recall), status
  int32_t* wcount;       // [slots, 3] marbles per walk
  int32_t* wstatus;      // [slots, 3]
  double r, step, threshold, cos40;
  int cap_marbles, cap_queue, cap_covered, hash_size, cap_cand;
  int first_pair, npairs;
  uint32_t serial;
};

struct Ws {              // slot workspaces
  char* walk;            // per slot, per walk
  size_t walk_bytes_prop, walk_bytes_gt, slot_walk_bytes;
  char* match;           // per slot
  size_t slot_match_bytes;
};

// The workspace of one walk over a graph of n nodes (host: sized with a null base; device: carved)
__host__ __device__ inline WalkWs walk_ws(Layout& L, const Params& p, int32_t n) {
  WalkWs w;
  w.marbles = L.take<double4>(p.cap_marbles);
  w.queue = L.take<QEntry>(p.cap_queue);
  w.ckey = L.take<uint64_t>(p.hash_size);
  w.cval = L.take<double>(p.hash_size);
  w.cstamp = L.take<uint32_t>(p.hash_size);
  w.dist = L.take<double>(n);
  w.dstamp = L.take<uint32_t>(n);
  return w;
}

// graph.py distance(p1, p2): a = p1[0] - p2[0]; b = (p1[1] - p2[1]) * cos(radians(p1[0])); sqrt(a*a + b*b)
__device__ __forceinline__ double dist_ll(double a0, double a1, double b0, double b1, double cos_a0) {
  const double a = a0 - b0;
  const double b = (a1 - b1) * cos_a0;
  return sqrt(a * a + b * b);
}

__device__ __forceinline__ bool in_list(const int32_t* s, const int32_t* idx, int32_t u, int32_t v) {
  for (int32_t k = s[u]; k < s[u + 1]; ++k)
    if (idx[k] == v) return true;
  return false;
}

// The k-th entry of nodeLink[u] + nodeLinkReverse[u]
__device__ __forceinline__ int32_t nbr(const GraphDev& g, int32_t u, int32_t k, int32_t nl) {
  return k < nl ? g.li[g.ls[u] + k] : g.ri[g.rs[u] + (k - nl)];
}

struct Walker {
  const GraphDev& g;
  const Params& p;
  WalkWs w;
  int lane;
  int cnt = 0, status = 0;

  __device__ Walker(const GraphDev& g_, const Params& p_, WalkWs w_, int lane_) : g(g_), p(p_), w(w_), lane(lane_) {}

  // `if (latI, lonI, dlat, dlon) not in mables: append (and the twin)`; false when the list is full
  __device__ bool add(double la, double lo, double d0, double d1, bool twin_rule) {
    bool dup = false;
    for (int i = lane; i < cnt; i += 32) {
      const double4 q = w.marbles[i];
      dup |= (q.x == la) & (q.y == lo) & (q.z == d0) & (q.w == d1);
    }
    if (__any_sync(0xffffffffu, dup)) return true;
    const int need = twin_rule ? 2 : 1;
    if (cnt + need > p.cap_marbles) {
      status |= kOverMarbles;
      return false;
    }
    if (lane == 0) {
      w.marbles[cnt] = make_double4(la, lo, d0, d1);
      if (twin_rule) w.marbles[cnt + 1] = make_double4(la + kTwin, lo + kTwin, d0, d1);
    }
    cnt += need;
    __syncwarp();
    return true;
  }

  __device__ int find_covered(uint64_t key) const {
    uint32_t h = static_cast<uint32_t>((key * 0x9E3779B97F4A7C15ull) >> 32) & (p.hash_size - 1);
    while (w.cstamp[h] == p.serial) {
      if (w.ckey[h] == key) return static_cast<int>(h);
      h = (h + 1) & (p.hash_size - 1);
    }
    return -1 - static_cast<int>(h);   // the empty slot where the key would go
  }

  // TOPOWalk(newstyle=True, direction=False, metaData=None, CheckGPS=None)
  __device__ void run(int32_t nid1, int32_t nid2, double dist1, double dist2, bool bidirection) {
    const double r = p.r, step = p.step;
    int head = 0, tail = 0, covered = 0;
    auto push = [&](int32_t node, int32_t prev, double d) -> bool {
      if (tail - head >= p.cap_queue) {
        status |= kOverQueue;
        return false;
      }
      if (lane == 0) w.queue[tail % p.cap_queue] = QEntry{node, prev, d};
      ++tail;
      __syncwarp();
      return true;
    };
    if (!push(nid1, -1, dist1) || !push(nid2, -1, dist2)) return;

    {  // holes between nid1 and nid2
      const double lat1 = g.ll[2 * nid1], lon1 = g.ll[2 * nid1 + 1];
      const double lat2 = g.ll[2 * nid2], lon2 = g.ll[2 * nid2 + 1];
      const double l = dist_ll(lat2, lon2, lat1, lon1, g.cosl[nid2]);
      const bool twin = bidirection && in_list(g.ls, g.li, nid2, nid1) && in_list(g.ls, g.li, nid1, nid2);
      const double d0 = lat2 - lat1, d1 = lon2 - lon1;
      double alpha = 0.0;
      while (true) {
        const double latI = lat1 * alpha + lat2 * (1.0 - alpha);
        const double lonI = lon1 * alpha + lon2 * (1.0 - alpha);
        const double cI = cos(latI * kDegToRad);
        const double e1 = dist_ll(latI, lonI, lat1, lon1, cI);
        const double e2 = dist_ll(latI, lonI, lat2, lon2, cI);
        if (dist1 - e1 < r || dist2 - e2 < r)
          if (!add(latI, lonI, d0, d1, twin)) return;
        alpha += step / l;
        if (alpha > 1.0) break;
      }
    }

    while (head < tail) {
      const QEntry e = w.queue[head % p.cap_queue];
      ++head;
      const int32_t cur = e.node, prev = e.prev;
      const double dist = e.dist;
      double old_node_dist = 1.0;
      if (w.dstamp[cur] == p.serial) {
        old_node_dist = w.dist[cur];
        if (old_node_dist <= dist) continue;
      }
      if (dist > r) continue;
      if (lane == 0) {
        w.dstamp[cur] = p.serial;
        w.dist[cur] = dist;
      }
      __syncwarp();
      const double lat1 = g.ll[2 * cur], lon1 = g.ll[2 * cur + 1];
      const int32_t nl = g.ls[cur + 1] - g.ls[cur];
      const int32_t nt = nl + g.rs[cur + 1] - g.rs[cur];
      for (int32_t k = 0; k < nt; ++k) {
        const int32_t nx = nbr(g, cur, k, nl);
        if (nx == prev || nx == cur || nx == nid1 || nx == nid2) continue;
        bool seen = false;                       // visited_next_node
        for (int32_t j = 0; j < k && !seen; ++j) seen = nbr(g, cur, j, nl) == nx;
        if (seen) continue;
        const double lat2 = g.ll[2 * nx], lon2 = g.ll[2 * nx + 1];
        const double l = dist_ll(lat2, lon2, lat1, lon1, g.cosl[nx]);
        const double bias = step * ceil(dist / step) - dist;
        double cs = bias;
        if (old_node_dist + l < r) {
          if (!push(nx, cur, dist + l)) return;
          continue;
        }
        const uint64_t kf = (static_cast<uint64_t>(static_cast<uint32_t>(cur)) << 32) | static_cast<uint32_t>(nx);
        const uint64_t kb = (static_cast<uint64_t>(static_cast<uint32_t>(nx)) << 32) | static_cast<uint32_t>(cur);
        const int hf = find_covered(kf), hb = find_covered(kb);
        const double start_lim = hf >= 0 ? w.cval[hf] : 0.0;
        const double end_lim = hb >= 0 ? l - w.cval[hb] : l;
        const bool twin = bidirection && in_list(g.ls, g.li, cur, nx) && in_list(g.ls, g.li, nx, cur);
        const double d0 = lat2 - lat1, d1 = lon2 - lon1;
        while (cs < l) {
          const double alpha = cs / l;
          if (dist + l * alpha > r) break;
          if (l * alpha < start_lim) {
            cs += step;
            continue;
          }
          if (l * alpha > end_lim) break;
          const double latI = lat2 * alpha + lat1 * (1.0 - alpha);
          const double lonI = lon2 * alpha + lon1 * (1.0 - alpha);
          if (!add(latI, lonI, d0, d1, twin)) return;
          cs += step;
        }
        int slot = hf;
        if (slot < 0) {
          if (covered >= p.cap_covered) {
            status |= kOverCovered;
            return;
          }
          ++covered;
          slot = -1 - hf;
          if (lane == 0) {
            w.cstamp[slot] = p.serial;
            w.ckey[slot] = kf;
          }
        }
        if (lane == 0) w.cval[slot] = cs - step;
        __syncwarp();
        if (!push(nx, cur, dist + l)) return;
      }
    }
  }
};

__global__ void __launch_bounds__(32) walk_kernel(Params p, Ws ws) {
  const int slot = blockIdx.x, which = blockIdx.y, lane = threadIdx.x;
  const int pair = p.first_pair + slot;
  if (pair >= p.npairs) return;
  const GraphDev& g = which == 0 ? p.prop : p.gt;
  char* base = ws.walk + ws.slot_walk_bytes * slot;
  if (which > 0) base += ws.walk_bytes_prop + (which - 1) * ws.walk_bytes_gt;
  Layout L(base);
  Walker wk(g, p, walk_ws(L, p, g.n), lane);
  const int32_t* n = p.pn + 4 * pair;
  const double* d = p.pd + 4 * pair;
  if (which == 0) wk.run(n[0], n[1], d[0], d[1], false);
  else wk.run(n[2], n[3], d[2], d[3], which == 2);
  if (lane == 0) {
    p.wcount[3 * slot + which] = wk.cnt;
    p.wstatus[3 * slot + which] = wk.status;
  }
}

// latlonNorm(p) with lat = 40: (p0 / l, p1 cos40 / l), l = sqrt((p1 cos40)^2 + p0^2)
__device__ __forceinline__ void latlon_norm(double p0, double p1, double cos40, double& o0, double& o1) {
  const double p11 = p1 * cos40;
  const double l = sqrt(p11 * p11 + p0 * p0);
  o0 = p0 / l;
  o1 = p11 / l;
}

// The candidate test of TOPOWithPairs for (marble, hole).  The indexed side's box is +-0.00001 around its point,
// the query box +-1.8 * threshold around the other one (q_is_marble: the marble is the query, as in the
// precision loop; else the hole is, as in the recall loop); the boxes meet with inclusive bounds.
__device__ __forceinline__ bool candidate(const double4& m, const double4& h, bool q_is_marble, const Params& p) {
  const double rr = p.threshold * 1.8;
  const double4& q = q_is_marble ? m : h;
  const double4& x = q_is_marble ? h : m;
  const double bx0 = x.x - kTwin, by0 = x.y - kTwin, bx1 = x.x + kTwin, by1 = x.y + kTwin;
  const double qx0 = q.x - rr, qy0 = q.y - rr, qx1 = q.x + rr, qy1 = q.y + rr;
  if (!(bx0 <= qx1 && bx1 >= qx0 && by0 <= qy1 && by1 >= qy0)) return false;
  const double ddd = dist_ll(m.x, m.y, h.x, h.y, cos(m.x * kDegToRad));
  double angle_d = 0.0;
  if (m.z != m.w && h.z != h.w) {
    double a0, a1, b0, b1;
    latlon_norm(m.z, m.w, p.cos40, a0, a1);
    latlon_norm(h.z, h.w, p.cos40, b0, b1);
    angle_d = 1.0 - fabs(a0 * b0 + a1 * b1);
  }
  return ddd < p.threshold && angle_d < 0.29;
}

struct MatchWs {
  int32_t* off;      // [cap_marbles + 1]
  int32_t* adj;      // [cap_cand]
  int32_t* match_r;  // [cap_marbles]
  int32_t* match_l;  // [cap_marbles]
  int32_t* visit;    // [cap_marbles]
  int32_t* stack;    // [2 * cap_marbles]
};

// The workspace of one matching (a slot has two: precision, then recall)
__host__ __device__ inline MatchWs match_ws(Layout& L, const Params& p) {
  MatchWs m;
  m.off = L.take<int32_t>(p.cap_marbles + 1);
  m.adj = L.take<int32_t>(p.cap_cand);
  m.match_r = L.take<int32_t>(p.cap_marbles);
  m.match_l = L.take<int32_t>(p.cap_marbles);
  m.visit = L.take<int32_t>(p.cap_marbles);
  m.stack = L.take<int32_t>(2ull * p.cap_marbles);
  return m;
}

// Candidate edges of the left list against the right list as CSR (right ids ascending per left vertex).
// Each thread owns a contiguous range of left vertices: count, block scan of the per-thread totals, fill.
// Returns false (uniformly) when the edges exceed cap_cand.
__device__ bool build_csr(const double4* left, int nl, const double4* right, int nr, bool left_is_marble,
                          const Params& p, MatchWs m, int32_t* s_tot) {
  const int t = threadIdx.x, T = blockDim.x;
  const int lo = static_cast<int>((static_cast<long long>(nl) * t) / T);
  const int hi = static_cast<int>((static_cast<long long>(nl) * (t + 1)) / T);
  int count = 0;
  for (int i = lo; i < hi; ++i)
    for (int j = 0; j < nr; ++j)
      count += left_is_marble ? candidate(left[i], right[j], true, p) : candidate(right[j], left[i], false, p);
  s_tot[t] = count;
  __syncthreads();
  if (t == 0) {
    long long run = 0;
    for (int k = 0; k < T; ++k) {
      const long long c = s_tot[k];
      s_tot[k] = static_cast<int32_t>(std::min<long long>(run, INT32_MAX));
      run += c;
    }
    s_tot[T] = static_cast<int32_t>(std::min<long long>(run, static_cast<long long>(INT32_MAX)));
  }
  __syncthreads();
  const bool ok = s_tot[T] <= p.cap_cand;
  if (ok) {
    int e = s_tot[t];
    for (int i = lo; i < hi; ++i) {
      m.off[i] = e;
      for (int j = 0; j < nr; ++j) {
        const bool c = left_is_marble ? candidate(left[i], right[j], true, p) : candidate(right[j], left[i], false, p);
        if (c) m.adj[e++] = j;
      }
    }
    if (t == T - 1) m.off[nl] = e;
  }
  __syncthreads();
  return ok;
}

// Size of a maximum matching: greedy start, then one augmenting-path search (iterative DFS) per free left vertex.
__device__ int max_matching(int nl, int nr, MatchWs m) {
  for (int j = 0; j < nr; ++j) {
    m.match_r[j] = -1;
    m.visit[j] = 0;
  }
  int size = 0;
  for (int i = 0; i < nl; ++i) {
    m.match_l[i] = -1;
    for (int e = m.off[i]; e < m.off[i + 1]; ++e)
      if (m.match_r[m.adj[e]] < 0) {
        m.match_r[m.adj[e]] = i;
        m.match_l[i] = m.adj[e];
        ++size;
        break;
      }
  }
  for (int u = 0; u < nl; ++u) {
    if (m.match_l[u] >= 0) continue;
    const int stamp = u + 1;
    int top = 0;
    m.stack[0] = u;
    m.stack[1] = m.off[u];
    bool found = false;
    while (top >= 0 && !found) {
      const int x = m.stack[2 * top];
      const int e = m.stack[2 * top + 1];
      if (e == m.off[x + 1]) {
        --top;
        continue;
      }
      m.stack[2 * top + 1] = e + 1;
      const int v = m.adj[e];
      if (m.visit[v] == stamp) continue;
      m.visit[v] = stamp;
      if (m.match_r[v] < 0) {
        // augment: frame k took the edge at stack[2k+1] - 1
        for (int k = top; k >= 0; --k) {
          const int xk = m.stack[2 * k];
          const int vk = m.adj[m.stack[2 * k + 1] - 1];
          m.match_r[vk] = xk;
          m.match_l[xk] = vk;
        }
        found = true;
      } else {
        ++top;
        m.stack[2 * top] = m.match_r[v];
        m.stack[2 * top + 1] = m.off[m.match_r[v]];
      }
    }
    size += found;
  }
  return size;
}

__global__ void __launch_bounds__(kMatchThreads) match_kernel(Params p, Ws ws) {
  __shared__ int32_t s_tot[kMatchThreads + 1];
  const int slot = blockIdx.x;
  const int pair = p.first_pair + slot;
  if (pair >= p.npairs) return;
  int32_t* out = p.out + 6 * pair;
  const int nm = p.wcount[3 * slot], nh = p.wcount[3 * slot + 1], nhb = p.wcount[3 * slot + 2];
  int status = p.wstatus[3 * slot] | p.wstatus[3 * slot + 1] | p.wstatus[3 * slot + 2];
  int mp = 0, mr = 0;
  if (status == 0) {
    char* wb = ws.walk + ws.slot_walk_bytes * slot;
    const double4* marbles = reinterpret_cast<const double4*>(wb);
    const double4* holes = reinterpret_cast<const double4*>(wb + ws.walk_bytes_prop);
    const double4* holes_b = reinterpret_cast<const double4*>(wb + ws.walk_bytes_prop + ws.walk_bytes_gt);
    Layout L(ws.match + ws.slot_match_bytes * slot);
    const MatchWs mprec = match_ws(L, p);
    const MatchWs mrec = match_ws(L, p);
    // precision: marbles -> holes_bidirection; recall: holes -> marbles
    const bool ok1 = build_csr(marbles, nm, holes_b, nhb, true, p, mprec, s_tot);
    const bool ok2 = build_csr(holes, nh, marbles, nm, false, p, mrec, s_tot);
    if (!ok1 || !ok2) status |= kOverCand;
    __shared__ int s_m[2];
    if (status == 0) {
      if (threadIdx.x == 0) s_m[0] = max_matching(nm, nhb, mprec);
      if (threadIdx.x == 32) s_m[1] = max_matching(nh, nm, mrec);
      __syncthreads();
      mp = s_m[0];
      mr = s_m[1];
    }
  }
  if (threadIdx.x == 0) {
    out[0] = nm;
    out[1] = nh;
    out[2] = nhb;
    out[3] = mp;
    out[4] = mr;
    out[5] = status;
  }
}

}  // namespace

struct samroad_topo_ctx {
  int device = 0;
  SamRoadTopoCaps caps{};
  cudaStream_t stream = nullptr;  // the handle's own non-blocking stream: a run waits for its own work only
  GraphDev g[2];                  // 0 GT, 1 proposal
  DeviceBuffer gbuf[2];           // one allocation per graph, grown on demand and reused across tiles
  DeviceBuffer work;
  size_t layout[3] = {0, 0, 0};   // the walk workspace layout the stamps were cleared for
  uint32_t serial = 0;
};

extern "C" int samroad_topo_create(int device, const SamRoadTopoCaps* caps, samroad_topo_t* out) {
  SRB_REQUIRE(out != nullptr && caps != nullptr, "samroad_topo_create: null argument");
  SRB_REQUIRE(caps->max_marbles >= 2 && caps->max_queue >= 2 && caps->max_covered >= 1 && caps->max_candidates >= 1 &&
                  caps->slots >= 1,
              "samroad_topo_create: capacities must be positive (marbles >= 2, queue >= 2)");
  SRB_REQUIRE(caps->max_marbles <= (1 << 24) && caps->max_queue <= (1 << 26) && caps->max_covered <= (1 << 24) &&
                  caps->max_candidates <= (1 << 28) && caps->slots <= 65535,
              "samroad_topo_create: a capacity is larger than this build supports");
  if (int rc = open_device(device)) return rc;
  cudaStream_t st = nullptr;
  SRB_CUDA_OK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
  samroad_topo_ctx* T = new samroad_topo_ctx();
  T->device = device;
  T->caps = *caps;
  T->stream = st;
  *out = T;
  return 0;
}

extern "C" int samroad_topo_destroy(samroad_topo_t T) {
  if (!T) return 0;
  cudaSetDevice(T->device);
  cudaStreamSynchronize(T->stream);
  cudaStreamDestroy(T->stream);
  delete T;
  return 0;
}

extern "C" int samroad_topo_upload_graph(samroad_topo_t T, int which, int32_t n_nodes, const double* latlon,
                                         const double* cos_lat, const int32_t* link_start, const int32_t* link,
                                         const int32_t* rlink_start, const int32_t* rlink) {
  SRB_REQUIRE(T != nullptr, "samroad_topo_upload_graph: null handle");
  SRB_REQUIRE(which == 0 || which == 1, "samroad_topo_upload_graph: which must be 0 (ground truth) or 1 (proposal)");
  SRB_REQUIRE(n_nodes >= 0, "samroad_topo_upload_graph: negative node count");
  SRB_REQUIRE(n_nodes == 0 || (latlon && cos_lat && link_start && rlink_start),
              "samroad_topo_upload_graph: null argument");
  if (n_nodes > 0) {
    if (int rc = check_csr("samroad_topo_upload_graph", n_nodes, link_start, link)) return rc;
    if (int rc = check_csr("samroad_topo_upload_graph", n_nodes, rlink_start, rlink)) return rc;
  }
  for (int32_t i = 0; i < n_nodes; ++i) {
    SRB_REQUIRE(std::isfinite(latlon[2 * i]) && std::isfinite(latlon[2 * i + 1]) && std::isfinite(cos_lat[i]),
                "samroad_topo_upload_graph: node %d has a coordinate that is not finite", i);
    for (int32_t k = link_start[i]; k < link_start[i + 1]; ++k) {
      const int32_t j = link[k];
      SRB_REQUIRE(!(latlon[2 * i] == latlon[2 * j] && latlon[2 * i + 1] == latlon[2 * j + 1]),
                  "samroad_topo_upload_graph: edge %d -> %d has length zero", i, j);
    }
  }
  SRB_CUDA_OK(cudaSetDevice(T->device));
  T->g[which].n = 0;
  if (n_nodes == 0) return 0;
  const size_t n = static_cast<size_t>(n_nodes);
  const size_t m0 = link_start[n_nodes], m1 = rlink_start[n_nodes];
  const size_t sizes[] = {16 * n, 8 * n, 4 * (n + 1), 4 * m0, 4 * (n + 1), 4 * m1};
  const void* src[] = {latlon, cos_lat, link_start, link, rlink_start, rlink};
  // each array gets a region of at least one byte
  auto carve = [&](void* base, void** dst) {
    Layout L(base);
    for (int i = 0; i < 6; ++i) dst[i] = L.take<char>(std::max<size_t>(sizes[i], 1));
    return L.bytes();
  };
  void* dst[6];
  // runs are synchronous, so nothing of this handle still reads the old buffer
  if (T->gbuf[which].reserve(carve(nullptr, dst), "samroad_topo_upload_graph")) return 1;
  carve(T->gbuf[which].get(), dst);
  for (int i = 0; i < 6; ++i)
    if (sizes[i]) SRB_CUDA_OK(cudaMemcpyAsync(dst[i], src[i], sizes[i], cudaMemcpyHostToDevice, T->stream));
  SRB_CUDA_OK(cudaStreamSynchronize(T->stream));
  GraphDev g;
  g.ll = static_cast<const double*>(dst[0]);
  g.cosl = static_cast<const double*>(dst[1]);
  g.ls = static_cast<const int32_t*>(dst[2]);
  g.li = static_cast<const int32_t*>(dst[3]);
  g.rs = static_cast<const int32_t*>(dst[4]);
  g.ri = static_cast<const int32_t*>(dst[5]);
  g.n = n_nodes;
  T->g[which] = g;
  return 0;
}

extern "C" int samroad_topo_run(samroad_topo_t T, int32_t n_pairs, const int32_t* pair_nodes,
                                const double* pair_dists, double r, double step, double threshold, double cos40,
                                int32_t* counts) {
  const char* what = "samroad_topo_run";
  SRB_REQUIRE(T != nullptr, "%s: null handle", what);
  SRB_REQUIRE(n_pairs >= 0, "%s: negative pair count", what);
  if (n_pairs == 0) return 0;
  SRB_REQUIRE(pair_nodes && pair_dists && counts, "%s: null argument", what);
  SRB_REQUIRE(T->g[0].n > 0 && T->g[1].n > 0, "%s: both graphs must be uploaded and non-empty", what);
  SRB_REQUIRE(std::isfinite(r) && std::isfinite(step) && step > 0.0 && std::isfinite(threshold) &&
                  std::isfinite(cos40),
              "%s: r, step, threshold must be finite and step positive", what);
  for (int32_t i = 0; i < n_pairs; ++i) {
    for (int k = 0; k < 4; ++k) {
      const int32_t nmax = T->g[k < 2 ? 1 : 0].n;
      SRB_REQUIRE(pair_nodes[4 * i + k] >= 0 && pair_nodes[4 * i + k] < nmax,
                  "%s: pair %d names node %d, outside its graph", what, i, pair_nodes[4 * i + k]);
      SRB_REQUIRE(std::isfinite(pair_dists[4 * i + k]), "%s: pair %d has a distance that is not finite", what, i);
    }
    SRB_REQUIRE(pair_nodes[4 * i] != pair_nodes[4 * i + 1] && pair_nodes[4 * i + 2] != pair_nodes[4 * i + 3],
                "%s: pair %d names an edge from a node to itself", what, i);
  }
  SRB_CUDA_OK(cudaSetDevice(T->device));
  const SamRoadTopoCaps& c = T->caps;
  Params p;
  p.gt = T->g[0];
  p.prop = T->g[1];
  p.r = r;
  p.step = step;
  p.threshold = threshold;
  p.cos40 = cos40;
  p.cap_marbles = c.max_marbles;
  p.cap_queue = c.max_queue;
  p.cap_covered = c.max_covered;
  p.hash_size = 1;
  while (p.hash_size < 2 * c.max_covered) p.hash_size <<= 1;
  p.cap_cand = c.max_candidates;
  p.npairs = n_pairs;
  const int slots = std::min(n_pairs, c.slots);
  auto walk_bytes = [&](int32_t n) {
    Layout L(nullptr);
    walk_ws(L, p, n);
    return L.bytes();
  };
  Ws ws;
  ws.walk_bytes_prop = walk_bytes(p.prop.n);
  ws.walk_bytes_gt = walk_bytes(p.gt.n);
  ws.slot_walk_bytes = ws.walk_bytes_prop + 2 * ws.walk_bytes_gt;
  Layout match(nullptr);
  match_ws(match, p);
  match_ws(match, p);
  ws.slot_match_bytes = match.bytes();
  // the run's workspace: every slot's walks, every slot's matchings, the pairs in, the counts and walk status out
  int32_t* d_pn = nullptr;
  double* d_pd = nullptr;
  auto carve = [&](void* base) {
    Layout L(base);
    ws.walk = L.take<char>(ws.slot_walk_bytes * slots);
    ws.match = L.take<char>(ws.slot_match_bytes * slots);
    d_pn = L.take<int32_t>(4ull * n_pairs);
    d_pd = L.take<double>(4ull * n_pairs);
    p.out = L.take<int32_t>(6ull * n_pairs);
    p.wcount = L.take<int32_t>(3ull * slots);
    p.wstatus = L.take<int32_t>(3ull * slots);
    return L.bytes();
  };
  const size_t need = carve(nullptr);
  const bool fresh = need > T->work.capacity();
  // the previous run has finished: runs are synchronous
  if (T->work.reserve(need, what)) {
    set_last_error("%s: out of device memory (%zu bytes for %d pair slots); lower the slot count", what, need, slots);
    return 1;
  }
  carve(T->work.get());
  p.pn = d_pn;
  p.pd = d_pd;
  // the stamps of the dense distance maps and covered-edge tables must start below every serial in use
  const int chunks = (n_pairs + slots - 1) / slots;
  const size_t layout[3] = {ws.walk_bytes_prop, ws.walk_bytes_gt, static_cast<size_t>(slots)};
  if (fresh || !std::equal(layout, layout + 3, T->layout) || T->serial > 0xFFFFFFF0u - static_cast<uint32_t>(chunks)) {
    SRB_CUDA_OK(cudaMemsetAsync(T->work.get(), 0, ws.slot_walk_bytes * slots, T->stream));
    std::copy(layout, layout + 3, T->layout);
    T->serial = 0;
  }
  cudaStream_t st = T->stream;
  SRB_CUDA_OK(cudaMemcpyAsync(d_pn, pair_nodes, 16ull * n_pairs, cudaMemcpyHostToDevice, st));
  SRB_CUDA_OK(cudaMemcpyAsync(d_pd, pair_dists, 32ull * n_pairs, cudaMemcpyHostToDevice, st));
  for (int ch = 0; ch < chunks; ++ch) {
    p.first_pair = ch * slots;
    p.serial = ++T->serial;
    SRB_LAUNCH(walk_kernel, dim3(slots, 3), 32, 0, st, p, ws);
    SRB_LAUNCH(match_kernel, slots, kMatchThreads, 0, st, p, ws);
  }
  SRB_CUDA_OK(cudaMemcpyAsync(counts, p.out, 24ull * n_pairs, cudaMemcpyDeviceToHost, st));
  SRB_CUDA_OK(cudaStreamSynchronize(st));
  for (int32_t i = 0; i < n_pairs; ++i) {
    const int32_t s = counts[6 * i + 5];
    if (s == 0) continue;
    SRB_REQUIRE(!(s & kOverMarbles), "%s: pair %d: a walk placed more than %d marbles", what, i, c.max_marbles);
    SRB_REQUIRE(!(s & kOverQueue), "%s: pair %d: a walk queued more than %d nodes at once", what, i, c.max_queue);
    SRB_REQUIRE(!(s & kOverCovered), "%s: pair %d: a walk covered more than %d directed edges", what, i,
                c.max_covered);
    SRB_REQUIRE(!(s & kOverCand), "%s: pair %d: more than %d candidate marble-hole edges", what, i,
                c.max_candidates);
  }
  return 0;
}
