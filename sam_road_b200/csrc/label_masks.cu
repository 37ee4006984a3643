// sam_road_b200 :: the keypoint and road label masks of the datasets (DESIGN.md §16).
//
// Reference: cityscale/generate_labels.py and spacenet/generate_labels.py, which draw every keypoint with
// cv2.circle(img, p, KEYPOINT_RADIUS, 255, -1) and every edge with cv2.line(img, p0, p1, 255, ROAD_WIDTH).  The
// masks are pixel-identical to OpenCV 4.x's (oracle/label_mask_oracle.py restates its loops):
//
//   circle, filled      Circle(): the spans of the integer midpoint walk, clipped to the image.
//   line, thickness t>1 the segment clipped (clipLine, whole pixels) to the image grown by t on every side; then
//                       ThickLine(): the quad p0 +- d, p1 -+ d in 16-bit fixed point with d = cvRound of the unit
//                       normal times (t + (t & 1)) / 2 pixels, filled by FillConvexPoly(LINE_8, shift 16) (outline
//                       by Line2, then one span per scanline), and Circle(p, (t + 1) / 2) at both ends.
//
// One warp per keypoint and one per edge.  OpenCV accumulates the scanline x and the Line2 step row by row;
// both are x0 + k * dx in int64, so every lane computes its own rows and points in closed form and no result
// depends on another lane's.  Every write is a plain store of 255: overlapping shapes race benignly and the
// masks do not depend on the schedule or the drawing order.
#include "../../include/samroad_b200.h"

#include <cuda_runtime.h>

#include <algorithm>

#include "common.cuh"

using namespace srb;

namespace {

constexpr int kXYShift = 16;
constexpr int64_t kXYOne = int64_t(1) << kXYShift;
constexpr int kWarps = 8;                  // warps per block
constexpr int kTargetBlocks = 1056;        // 8 blocks per SM of an H100 SXM
constexpr int kMaxThickness = 32767;       // OpenCV's MAX_THICKNESS
constexpr int kMaxRadius = 32767;          // keeps the midpoint walk's int arithmetic exact

struct Img {
  uint8_t* p;
  int size;
  __device__ void put(int64_t x, int64_t y) const {
    if (x >= 0 && x < size && y >= 0 && y < size) p[y * size + x] = 255;
  }
  __device__ void hline(int64_t y, int64_t x1, int64_t x2) const {
    for (int64_t x = x1; x <= x2; ++x) p[y * size + x] = 255;
  }
};

// (int64)((double)num0 * (double)num1 / (double)den), as clipLine evaluates it (no contraction).
__device__ __forceinline__ int64_t clip_step(int64_t num0, int64_t num1, int64_t den) {
  return __double2ll_rz(__ddiv_rn(__dmul_rn(__ll2double_rn(num0), __ll2double_rn(num1)), __ll2double_rn(den)));
}

// clipLine(Size2l(w, h), p1, p2): Cohen-Sutherland; false when nothing of the segment is inside.
__device__ bool clip_line(int64_t w, int64_t h, int64_t& x1, int64_t& y1, int64_t& x2, int64_t& y2) {
  const int64_t right = w - 1, bottom = h - 1;
  int c1 = (x1 < 0) + (x1 > right) * 2 + (y1 < 0) * 4 + (y1 > bottom) * 8;
  int c2 = (x2 < 0) + (x2 > right) * 2 + (y2 < 0) * 4 + (y2 > bottom) * 8;
  if ((c1 & c2) == 0 && (c1 | c2) != 0) {
    if (c1 & 12) {
      const int64_t a = c1 < 8 ? 0 : bottom;
      x1 += clip_step(a - y1, x2 - x1, y2 - y1);
      y1 = a;
      c1 = (x1 < 0) + (x1 > right) * 2;
    }
    if (c2 & 12) {
      const int64_t a = c2 < 8 ? 0 : bottom;
      x2 += clip_step(a - y2, x2 - x1, y2 - y1);
      y2 = a;
      c2 = (x2 < 0) + (x2 > right) * 2;
    }
    if ((c1 & c2) == 0 && (c1 | c2) != 0) {
      if (c1) {
        const int64_t a = c1 == 1 ? 0 : right;
        y1 += clip_step(a - x1, y2 - y1, x2 - x1);
        x1 = a;
        c1 = 0;
      }
      if (c2) {
        const int64_t a = c2 == 1 ? 0 : right;
        y2 += clip_step(a - x2, y2 - y1, x2 - x1);
        x2 = a;
        c2 = 0;
      }
    }
  }
  return (c1 | c2) == 0;
}

// Circle(img, (cx, cy), r, fill=1).  Every lane runs the midpoint walk; the lanes share each step's spans.
__device__ void circle_fill(const Img& img, int cx, int cy, int r, int lane) {
  int err = 0, dx = r, dy = 0, plus = 1, minus = (r << 1) - 1;
  while (dx >= dy) {
#pragma unroll
    for (int s = 0; s < 2; ++s) {
      const int h = s ? dx : dy, half = s ? dy : dx;   // rows cy -+ h span cx -+ half
      const int64_t xa = max(int64_t(cx) - half, int64_t(0));
      const int64_t xb = min(int64_t(cx) + half, int64_t(img.size) - 1);
      for (int64_t x = xa + lane; x <= xb; x += 32) {
        img.put(x, int64_t(cy) - h);
        img.put(x, int64_t(cy) + h);
      }
    }
    dy++;
    err += plus;
    plus += 2;
    const int mask = (err <= 0) - 1;
    err -= minus & mask;
    dx += mask;
    minus -= mask & 2;
  }
}

// Line2(img, p1, p2) in 16-bit fixed point: point k of the DDA is (x1 + k, (y1 + k * y_step) >> 16) along x
// (or the transpose), one point per lane, plus the rounded end point.
__device__ void line2(const Img& img, int64_t x1, int64_t y1, int64_t x2, int64_t y2, int lane) {
  const int64_t scaled = int64_t(img.size) << kXYShift;
  if (!clip_line(scaled, scaled, x1, y1, x2, y2)) return;
  int64_t dx = x2 - x1, dy = y2 - y1;
  const int64_t ax = dx < 0 ? -dx : dx, ay = dy < 0 ? -dy : dy;
  const bool along_x = ax > ay;
  if (along_x ? dx < 0 : dy < 0) {
    dx = -dx;
    dy = -dy;
    int64_t t = x1; x1 = x2; x2 = t;
    t = y1; y1 = y2; y2 = t;
  }
  if (lane == 0) img.put((x2 + (kXYOne >> 1)) >> kXYShift, (y2 + (kXYOne >> 1)) >> kXYShift);
  if (along_x) {
    const int64_t y_step = (dy << kXYShift) / (ax | 1), ecount = (x2 - x1) >> kXYShift;
    const int64_t x0 = (x1 + (kXYOne >> 1)) >> kXYShift, y0 = y1 + (kXYOne >> 1);
    for (int64_t k = lane; k <= ecount; k += 32) img.put(x0 + k, (y0 + k * y_step) >> kXYShift);
  } else {
    const int64_t x_step = (dx << kXYShift) / (ay | 1), ecount = (y2 - y1) >> kXYShift;
    const int64_t x0 = x1 + (kXYOne >> 1), y0 = (y1 + (kXYOne >> 1)) >> kXYShift;
    for (int64_t k = lane; k <= ecount; k += 32) img.put((x0 + k * x_step) >> kXYShift, y0 + k);
  }
}

// FillConvexPoly(img, v, 4, LINE_8, shift 16).  OpenCV walks the left and right chains from the top vertex
// with one budget of 4 edges between them: at row y a chain whose edge ends (y >= ye) takes the next edge
// whose rounded end row lies below y, with x = its start vertex's x and the rounded per-row step dx; the fill
// stops before the first row at which the budget runs out.  The walk changes state at no more than 5 rows, so
// every lane replays it into at most 5 row ranges of constant state and then draws its own rows.
__device__ void fill_quad(const Img& img, const int64_t (&vx)[4], const int64_t (&vy)[4], int lane) {
  constexpr int n = 4;
  const int64_t delta = kXYOne >> 1;
  int imin = 0;
  int64_t xmin = vx[0], xmax = vx[0], ymin = vy[0], ymax = vy[0];
  for (int i = 0; i < n; ++i) {
    if (vy[i] < ymin) {
      ymin = vy[i];
      imin = i;
    }
    ymax = max(ymax, vy[i]);
    xmax = max(xmax, vx[i]);
    xmin = min(xmin, vx[i]);
    line2(img, vx[(i + n - 1) % n], vy[(i + n - 1) % n], vx[i], vy[i], lane);
  }
  xmin = (xmin + delta) >> kXYShift;
  xmax = (xmax + delta) >> kXYShift;
  ymin = (ymin + delta) >> kXYShift;
  ymax = (ymax + delta) >> kXYShift;
  if (xmax < 0 || ymax < 0 || xmin >= img.size || ymin >= img.size) return;
  ymax = min(ymax, int64_t(img.size) - 1);

  constexpr int kRanges = n + 1;
  int64_t r_begin[kRanges], r_x[kRanges][2], r_dx[kRanges][2], r_ya[kRanges][2];
  int ranges = 0;
  int64_t stop = ymax + 1;                  // first row not drawn
  int idx[2] = {imin, imin}, edges = n;
  int64_t ye[2] = {ymin, ymin}, ex[2] = {-kXYOne, -kXYOne}, edx[2] = {0, 0}, ya[2] = {ymin, ymin};
  for (int64_t y = ymin; y <= ymax;) {
    for (int i = 0; i < 2; ++i) {
      if (y < ye[i]) continue;
      const int di = i ? n - 1 : 1;
      int idx0 = idx[i], j = (idx0 + di) % n;
      while (edges-- > 0) {
        const int64_t ty = (vy[j] + delta) >> kXYShift;
        if (ty > y) {
          ye[i] = ty;
          edx[i] = ((vx[j] - vx[idx0]) * 2 + (ty - y)) / (2 * (ty - y));
          ex[i] = vx[idx0];
          ya[i] = y;
          idx[i] = j;
          break;
        }
        idx0 = j;
        j = (j + di) % n;
      }
    }
    if (edges < 0) {
      stop = y;
      break;
    }
    r_begin[ranges] = y;
    for (int i = 0; i < 2; ++i) {
      r_x[ranges][i] = ex[i];
      r_dx[ranges][i] = edx[i];
      r_ya[ranges][i] = ya[i];
    }
    ++ranges;
    y = min(ye[0], ye[1]);
  }

  for (int64_t y = max(ymin, int64_t(0)) + lane; y < stop; y += 32) {
    int r = 0;
    while (r + 1 < ranges && r_begin[r + 1] <= y) ++r;
    const int64_t x0 = r_x[r][0] + (y - r_ya[r][0]) * r_dx[r][0];
    const int64_t x1 = r_x[r][1] + (y - r_ya[r][1]) * r_dx[r][1];
    int64_t xx1 = (min(x0, x1) + delta) >> kXYShift;
    int64_t xx2 = (max(x0, x1) + delta) >> kXYShift;
    if (xx2 >= 0 && xx1 < img.size) img.hline(y, max(xx1, int64_t(0)), min(xx2, int64_t(img.size) - 1));
  }
}

// cv2.line(img, p0, p1, 255, thickness) for thickness >= 2.
__device__ void thick_line(const Img& img, int64_t x0, int64_t y0, int64_t x1, int64_t y1, int thickness,
                           int lane) {
  const int64_t grown = int64_t(img.size) + 2 * thickness;
  x0 += thickness; y0 += thickness; x1 += thickness; y1 += thickness;
  if (!clip_line(grown, grown, x0, y0, x1, y1)) return;
  x0 -= thickness; y0 -= thickness; x1 -= thickness; y1 -= thickness;

  const double dx = __ll2double_rn(x0 - x1), dy = __ll2double_rn(y1 - y0);
  double r = __dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy));
  const int t = thickness << (kXYShift - 1);
  if (r > 2.220446049250313e-16) {          // fabs(r) > DBL_EPSILON
    r = __ddiv_rn(__dadd_rn(double(t), double((thickness & 1) * kXYOne) * 0.5), __dsqrt_rn(r));
    const int64_t dpx = __double2int_rn(__dmul_rn(dy, r)), dpy = __double2int_rn(__dmul_rn(dx, r));
    const int64_t ax = x0 << kXYShift, ay = y0 << kXYShift, bx = x1 << kXYShift, by = y1 << kXYShift;
    const int64_t vx[4] = {ax + dpx, ax - dpx, bx - dpx, bx + dpx};
    const int64_t vy[4] = {ay + dpy, ay - dpy, by - dpy, by + dpy};
    fill_quad(img, vx, vy, lane);
  }
  const int cap = static_cast<int>((int64_t(t) + (kXYOne >> 1)) >> kXYShift);
  circle_fill(img, static_cast<int>(x0), static_cast<int>(y0), cap, lane);
  circle_fill(img, static_cast<int>(x1), static_cast<int>(y1), cap, lane);
}

// grid (T, blocks per tile): the warps of a tile's blocks take its keypoints, then its edges.
__global__ void __launch_bounds__(kWarps * 32) label_masks_kernel(
    int size, const int32_t* __restrict__ nodes_xy, const int64_t* __restrict__ node_off,
    const int32_t* __restrict__ edges_xyxy, const int64_t* __restrict__ edge_off, int keypoint_radius,
    int road_width, uint8_t* keypoint_mask, uint8_t* road_mask) {
  const int tile = blockIdx.x, lane = threadIdx.x & 31;
  const int64_t pixels = int64_t(size) * size;
  const Img kp{keypoint_mask + tile * pixels, size}, road{road_mask + tile * pixels, size};
  const int64_t n0 = node_off[tile], nk = node_off[tile + 1] - n0;
  const int64_t e0 = edge_off[tile], ne = edge_off[tile + 1] - e0;
  const int64_t stride = int64_t(gridDim.y) * kWarps;
  for (int64_t w = int64_t(blockIdx.y) * kWarps + (threadIdx.x >> 5); w < nk + ne; w += stride) {
    if (w < nk) {
      const int32_t* p = nodes_xy + 2 * (n0 + w);
      circle_fill(kp, p[0], p[1], keypoint_radius, lane);
    } else {
      const int32_t* e = edges_xyxy + 4 * (e0 + w - nk);
      thick_line(road, e[0], e[1], e[2], e[3], road_width, lane);
    }
  }
}

}  // namespace

extern "C" int samroad_label_masks(int T, int size, const int32_t* nodes_xy, const int64_t* node_off,
                                   const int32_t* edges_xyxy, const int64_t* edge_off, int keypoint_radius,
                                   int road_width, uint8_t* keypoint_mask, uint8_t* road_mask, void* stream) {
  SRB_REQUIRE(T >= 0, "samroad_label_masks: tile count must be >= 0 (got %d)", T);
  SRB_REQUIRE(size >= 1, "samroad_label_masks: size must be >= 1 (got %d)", size);
  SRB_REQUIRE(road_width >= 2 && road_width <= kMaxThickness,
              "samroad_label_masks: road_width must be in [2, %d] (got %d)", kMaxThickness, road_width);
  SRB_REQUIRE(keypoint_radius >= 0 && keypoint_radius <= kMaxRadius,
              "samroad_label_masks: keypoint_radius must be in [0, %d] (got %d)", kMaxRadius, keypoint_radius);
  SRB_REQUIRE(nodes_xy && node_off && edges_xyxy && edge_off && keypoint_mask && road_mask,
              "samroad_label_masks: null pointer");
  if (T == 0) return 0;
  auto s = static_cast<cudaStream_t>(stream);
  const size_t bytes = size_t(T) * size_t(size) * size_t(size);
  SRB_CUDA_OK(cudaMemsetAsync(keypoint_mask, 0, bytes, s));
  SRB_CUDA_OK(cudaMemsetAsync(road_mask, 0, bytes, s));
  const dim3 grid(T, std::min(65535, std::max(1, blocks_for(kTargetBlocks, T))));
  SRB_LAUNCH(label_masks_kernel, grid, kWarps * 32, 0, s, size, nodes_xy, node_off, edges_xyxy, edge_off,
             keypoint_radius, road_width, keypoint_mask, road_mask);
  return 0;
}
