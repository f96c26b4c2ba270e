// overlay.cuh -- draw_person_pose (pose_detector.py:520-553) on the device, bit-exact with OpenCV's rasteriser.
//
// The reference draws, per person, 17 limbs with cv2.line(canvas, p1, p2, color, 2) (ear-shoulder limbs 9 and 13 are
// skipped) and then, per person, up to 18 joints with cv2.circle(canvas, (x, y), 3, color, -1); later primitives
// overwrite earlier ones.  OpenCV (imgproc/drawing.cpp, 4.13) rasterises them as
//   line, thickness 2, LINE_8   ThickLine: half-width vector dp = (cvRound(dy*r), cvRound(dx*r)), r = 2^16/|p1-p0| in
//                               16.16 fixed point; FillConvexPoly of the 4-corner polygon (its edges with the
//                               fixed-point DDA `Line2` after clipLine, then the scan-line fill with 16.16 edge
//                               walkers), then a filled circle of radius 1 at both end points;
//   circle, radius 3, filled    the midpoint circle's horizontal spans, clipped to the image.
// Here every primitive is rasterised by ONE thread with the same integer / double operation sequence (single IEEE
// operations, no contraction) into a per-pixel PRIORITY plane (atomicMax of the primitive's 1-based index in the
// reference's drawing order); a second kernel paints each covered pixel with the colour of its highest-priority
// primitive -- exactly the pixel the sequential overwrite order leaves.  All joints are inside the image by
// construction (they are scaled peak positions), which is the case OpenCV's own pre-clipping leaves untouched; the entry
// point rejects joints outside the image.
//
// The whole-body picture of demo.py:28-57 extends the same scheme.  After the skeleton primitives come the face / hand
// parts in the caller's order, each part owning OV_PART_STRIDE consecutive priorities:
//   face (face_detector.py:79-97)   70 dots cv2.circle(radius 2, filled), then the 63 face_line_indices segments
//                                   cv2.line(thickness 1), then the crop rectangle;
//   hand (hand_detector.py:89-117)  per finger and segment: dot a, dot b (radius 3), the segment (thickness 1), all in
//                                   the finger's colour; then the crop rectangle;
//   rectangle                       cv2.rectangle(thickness 1): PolyLine of the four closed edges with thickness 1.
// A 1-px line is ThickLine with thickness <= 1, LINE_8 and shift 0, i.e. drawing.cpp Line(): LineIterator(img, p0, p1,
// 8, leftToRight = true) -- clipLine on the unscaled image size when an end point lies outside, then Bresenham.  Parts
// may lie partly or wholly outside the frame.  The paint pass composes cv2.addWeighted(img, 0.6, skeleton, 0.4, 0):
// a pixel whose top primitive is a part takes the part's colour, a skeleton pixel blend(img, skeleton colour), any
// other pixel keeps img (blend(a, a) == a for every uint8 a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace opb {

constexpr int OV_SHIFT = 16;
constexpr long long OV_ONE = 1ll << OV_SHIFT;
constexpr int OV_LIMBS = 19, OV_JOINTS = 18;
constexpr int OV_FACE_POINTS = 70, OV_FACE_LINES = 63, OV_HAND_POINTS = 21, OV_FINGERS = 5, OV_FINGER_SEGS = 4;
constexpr int OV_HAND_PRIMS = OV_FINGERS * OV_FINGER_SEGS * 3;                 // dot a, dot b, segment
constexpr int OV_PART_STRIDE = OV_FACE_POINTS + OV_FACE_LINES + 1;             // the larger part, rectangle included
constexpr int OV_PART_FACE = 0, OV_PART_HAND = 1;

struct OverlayTables {
  int limb_a[OV_LIMBS], limb_b[OV_LIMBS];      // params['limbs_point'] (entity.py:85-105)
  uint8_t limb_color[OV_LIMBS][3];             // pose_detector.py:524-529 (written to channels 0,1,2 as given)
  uint8_t joint_color[OV_JOINTS][3];           // :531-535
  uint8_t face_line[OV_FACE_LINES][2];         // params['face_line_indices'] (entity.py:130-141)
  uint8_t finger[OV_FINGERS][OV_FINGER_SEGS][2];  // params['fingers_indices'] (entity.py:145-151)
  uint8_t finger_color[OV_FINGERS][3];         // hand_detector.py:93-99
  uint8_t face_color[3], rect_color[3];        // face_detector.py:86,95; demo.py:40,50,57
};

struct OvPart {                                // == opb_part (include/opb.h)
  int kind, left, top, right, bottom, first_point;
};

struct OvCanvas {
  unsigned int* prio;
  int H, W;
  unsigned int tag;
  __device__ __forceinline__ void put(long long x, long long y) const {
    if (x >= 0 && x < W && y >= 0 && y < H) atomicMax(prio + static_cast<size_t>(y) * W + x, tag);
  }
  __device__ __forceinline__ void hline(int y, int xa, int xb) const {   // caller guarantees 0 <= y < H and clipped xa..xb
    for (int x = xa; x <= xb; ++x) atomicMax(prio + static_cast<size_t>(y) * W + x, tag);
  }
};

// cv::clipLine(Size2l, Point2l&, Point2l&) on the 16.16-scaled image rectangle
__device__ inline bool ov_clip_line(long long Ws, long long Hs, long long& x1, long long& y1, long long& x2, long long& y2) {
  const long long right = Ws - 1, bottom = Hs - 1;
  if (Ws <= 0 || Hs <= 0) return false;
  int c1 = (x1 < 0) + (x1 > right) * 2 + (y1 < 0) * 4 + (y1 > bottom) * 8;
  int c2 = (x2 < 0) + (x2 > right) * 2 + (y2 < 0) * 4 + (y2 > bottom) * 8;
  if ((c1 & c2) == 0 && (c1 | c2) != 0) {
    long long a;
    if (c1 & 12) {
      a = c1 < 8 ? 0 : bottom;
      x1 += static_cast<long long>(__ddiv_rn(__dmul_rn(static_cast<double>(a - y1), static_cast<double>(x2 - x1)), static_cast<double>(y2 - y1)));
      y1 = a;
      c1 = (x1 < 0) + (x1 > right) * 2;
    }
    if (c2 & 12) {
      a = c2 < 8 ? 0 : bottom;
      x2 += static_cast<long long>(__ddiv_rn(__dmul_rn(static_cast<double>(a - y2), static_cast<double>(x2 - x1)), static_cast<double>(y2 - y1)));
      y2 = a;
      c2 = (x2 < 0) + (x2 > right) * 2;
    }
    if ((c1 & c2) == 0 && (c1 | c2) != 0) {
      if (c1) {
        a = c1 == 1 ? 0 : right;
        y1 += static_cast<long long>(__ddiv_rn(__dmul_rn(static_cast<double>(a - x1), static_cast<double>(y2 - y1)), static_cast<double>(x2 - x1)));
        x1 = a;
        c1 = 0;
      }
      if (c2) {
        a = c2 == 1 ? 0 : right;
        y2 += static_cast<long long>(__ddiv_rn(__dmul_rn(static_cast<double>(a - x2), static_cast<double>(y2 - y1)), static_cast<double>(x2 - x1)));
        x2 = a;
        c2 = 0;
      }
    }
  }
  return (c1 | c2) == 0;
}

// drawing.cpp Line2: fixed-point DDA between two 16.16 points
__device__ inline void ov_line2(const OvCanvas& cv, long long x1, long long y1, long long x2, long long y2) {
  if (!ov_clip_line(static_cast<long long>(cv.W) << OV_SHIFT, static_cast<long long>(cv.H) << OV_SHIFT, x1, y1, x2, y2)) return;
  long long dx = x2 - x1, dy = y2 - y1;
  const long long ax = dx < 0 ? -dx : dx, ay = dy < 0 ? -dy : dy;
  long long x_step, y_step;
  int ecount;
  if (ax > ay) {
    if (dx < 0) {
      dy = -dy;
      long long t = x1; x1 = x2; x2 = t;
      t = y1; y1 = y2; y2 = t;
    }
    x_step = OV_ONE;
    y_step = (dy * OV_ONE) / (ax | 1);       // (dy << XY_SHIFT) / (ax | 1), C++ truncating division
    ecount = static_cast<int>((x2 - x1) >> OV_SHIFT);
  } else {
    if (dy < 0) {
      dx = -dx;
      long long t = x1; x1 = x2; x2 = t;
      t = y1; y1 = y2; y2 = t;
    }
    x_step = (dx * OV_ONE) / (ay | 1);
    y_step = OV_ONE;
    ecount = static_cast<int>((y2 - y1) >> OV_SHIFT);
  }
  x1 += OV_ONE >> 1;
  y1 += OV_ONE >> 1;
  cv.put((x2 + (OV_ONE >> 1)) >> OV_SHIFT, (y2 + (OV_ONE >> 1)) >> OV_SHIFT);
  if (ax > ay) {
    x1 >>= OV_SHIFT;
    while (ecount >= 0) {
      cv.put(x1, y1 >> OV_SHIFT);
      x1++;
      y1 += y_step;
      ecount--;
    }
  } else {
    y1 >>= OV_SHIFT;
    while (ecount >= 0) {
      cv.put(x1 >> OV_SHIFT, y1);
      x1 += x_step;
      y1++;
      ecount--;
    }
  }
  (void)x_step;
}

// drawing.cpp Line(img, p1, p2, color, 8): LineIterator(img, p1, p2, 8, leftToRight = true), every pixel it visits.
// Coordinates are bounded by the entry point (|v| <= 2^20), so the int arithmetic below cannot overflow.
__device__ inline void ov_line1(const OvCanvas& cv, int x1, int y1, int x2, int y2) {
  if (static_cast<unsigned>(x1) >= static_cast<unsigned>(cv.W) || static_cast<unsigned>(x2) >= static_cast<unsigned>(cv.W) ||
      static_cast<unsigned>(y1) >= static_cast<unsigned>(cv.H) || static_cast<unsigned>(y2) >= static_cast<unsigned>(cv.H)) {
    long long a1 = x1, b1 = y1, a2 = x2, b2 = y2;    // clipLine(Size, Point&, Point&) widens to Point2l
    if (!ov_clip_line(cv.W, cv.H, a1, b1, a2, b2)) return;
    x1 = static_cast<int>(a1); y1 = static_cast<int>(b1);
    x2 = static_cast<int>(a2); y2 = static_cast<int>(b2);
  }
  int dx = x2 - x1, dy = y2 - y1, delta_y = 1;
  if (dx < 0) {                                      // leftToRight: walk from the other end
    dx = -dx;
    dy = -dy;
    x1 = x2;
    y1 = y2;
  }
  if (dy < 0) {
    dy = -dy;
    delta_y = -1;
  }
  const bool vert = dy > dx;
  if (vert) { const int t = dx; dx = dy; dy = t; }
  // 8-connectivity: the major axis advances every step, the minor one when err < 0
  int err = dx - (dy + dy);
  const int plus_delta = dx + dx, minus_delta = -(dy + dy);
  int x = x1, y = y1;
  for (int i = 0; i <= dx; ++i) {
    cv.put(x, y);
    const int mask = err < 0 ? -1 : 0;
    err += minus_delta + (plus_delta & mask);
    if (vert) { y += delta_y; x += 1 & mask; }
    else { x += 1; y += delta_y & mask; }
  }
}

// drawing.cpp rectangle(img, pt1, pt2, color, 1): PolyLine of the closed quad (l,t) (r,t) (r,b) (l,b), starting with
// the closing edge, each edge a 1-px Line()
__device__ inline void ov_rect1(const OvCanvas& cv, int l, int t, int r, int b) {
  ov_line1(cv, l, b, l, t);
  ov_line1(cv, l, t, r, t);
  ov_line1(cv, r, t, r, b);
  ov_line1(cv, r, b, l, b);
}

// drawing.cpp FillConvexPoly(img, v, 4, color, LINE_8, XY_SHIFT)
__device__ inline void ov_fill_convex4(const OvCanvas& cv, const long long (&vx)[4], const long long (&vy)[4]) {
  constexpr int npts = 4;
  const long long delta = OV_ONE >> 1;
  long long xmin = vx[0], xmax = vx[0], ymin = vy[0], ymax = vy[0];
  int imin = 0;
  long long px = vx[npts - 1], py = vy[npts - 1];
  for (int i = 0; i < npts; ++i) {
    if (vy[i] < ymin) { ymin = vy[i]; imin = i; }
    ymax = vy[i] > ymax ? vy[i] : ymax;
    xmax = vx[i] > xmax ? vx[i] : xmax;
    xmin = vx[i] < xmin ? vx[i] : xmin;
    ov_line2(cv, px, py, vx[i], vy[i]);
    px = vx[i];
    py = vy[i];
  }
  xmin = (xmin + delta) >> OV_SHIFT;
  xmax = (xmax + delta) >> OV_SHIFT;
  ymin = (ymin + delta) >> OV_SHIFT;
  ymax = (ymax + delta) >> OV_SHIFT;
  if (xmax < 0 || ymax < 0 || xmin >= cv.W || ymin >= cv.H) return;
  if (ymax > cv.H - 1) ymax = cv.H - 1;
  int e_idx[2] = {imin, imin}, e_di[2] = {1, npts - 1}, e_ye[2] = {static_cast<int>(ymin), static_cast<int>(ymin)};
  long long e_x[2] = {-OV_ONE, -OV_ONE}, e_dx[2] = {0, 0};
  int y = static_cast<int>(ymin), edges = npts;
  do {
    for (int i = 0; i < 2; ++i) {
      if (y >= e_ye[i]) {
        int idx0 = e_idx[i];
        const int di = e_di[i];
        int idx = idx0 + di;
        if (idx >= npts) idx -= npts;
        for (; edges-- > 0;) {
          const int ty = static_cast<int>((vy[idx] + delta) >> OV_SHIFT);
          if (ty > y) {
            const long long xs = vx[idx0], xe = vx[idx];
            e_ye[i] = ty;
            e_dx[i] = ((xe - xs) * 2 + (ty - y)) / (2 * (ty - y));
            e_x[i] = xs;
            e_idx[i] = idx;
            break;
          }
          idx0 = idx;
          idx += di;
          if (idx >= npts) idx -= npts;
        }
      }
    }
    if (edges < 0) break;
    if (y >= 0) {
      int left = 0, right = 1;
      if (e_x[0] > e_x[1]) { left = 1; right = 0; }
      int xx1 = static_cast<int>((e_x[left] + delta) >> OV_SHIFT);
      int xx2 = static_cast<int>((e_x[right] + delta) >> OV_SHIFT);
      if (xx2 >= 0 && xx1 < cv.W) {
        if (xx1 < 0) xx1 = 0;
        if (xx2 >= cv.W) xx2 = cv.W - 1;
        cv.hline(y, xx1, xx2);
      }
    }
    e_x[0] += e_dx[0];
    e_x[1] += e_dx[1];
  } while (++y <= static_cast<int>(ymax));
}

// drawing.cpp Circle(img, center, radius, color, fill = 1)
__device__ inline void ov_circle_fill(const OvCanvas& cv, int cx, int cy, int radius) {
  int err = 0, dx = radius, dy = 0, plus = 1, minus = (radius << 1) - 1;
  const int W = cv.W, H = cv.H;
  while (dx >= dy) {
    const int y11 = cy - dy, y12 = cy + dy, y21 = cy - dx, y22 = cy + dx;
    int x11 = cx - dx, x12 = cx + dx, x21 = cx - dy, x22 = cx + dy;
    if (x11 < W && x12 >= 0 && y21 < H && y22 >= 0) {
      x11 = max(x11, 0);
      x12 = min(x12, W - 1);
      if (static_cast<unsigned>(y11) < static_cast<unsigned>(H)) cv.hline(y11, x11, x12);
      if (static_cast<unsigned>(y12) < static_cast<unsigned>(H)) cv.hline(y12, x11, x12);
      if (x21 < W && x22 >= 0) {
        x21 = max(x21, 0);
        x22 = min(x22, W - 1);
        if (static_cast<unsigned>(y21) < static_cast<unsigned>(H)) cv.hline(y21, x21, x22);
        if (static_cast<unsigned>(y22) < static_cast<unsigned>(H)) cv.hline(y22, x21, x22);
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

// drawing.cpp ThickLine(img, p0, p1, color, thickness = 2, LINE_8, flags = 3, shift = 0)
__device__ inline void ov_thick_line2(const OvCanvas& cv, int x0, int y0, int x1, int y1) {
  const long long p0x = static_cast<long long>(x0) << OV_SHIFT, p0y = static_cast<long long>(y0) << OV_SHIFT;
  const long long p1x = static_cast<long long>(x1) << OV_SHIFT, p1y = static_cast<long long>(y1) << OV_SHIFT;
  const double inv = 1.0 / 65536.0;
  const double dx = __dmul_rn(static_cast<double>(p0x - p1x), inv), dy = __dmul_rn(static_cast<double>(p1y - p0y), inv);
  double r = __dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy));
  const long long th = 2ll << (OV_SHIFT - 1);
  if (fabs(r) > 2.220446049250313e-16) {
    r = __ddiv_rn(static_cast<double>(th), __dsqrt_rn(r));
    const long long dpx = __double2ll_rn(__dmul_rn(dy, r)), dpy = __double2ll_rn(__dmul_rn(dx, r));
    const long long vx[4] = {p0x + dpx, p0x - dpx, p1x - dpx, p1x + dpx};
    const long long vy[4] = {p0y + dpy, p0y - dpy, p1y - dpy, p1y + dpy};
    ov_fill_convex4(cv, vx, vy);
  }
  const int rad = static_cast<int>((th + (OV_ONE >> 1)) >> OV_SHIFT);
  ov_circle_fill(cv, x0, y0, rad);
  ov_circle_fill(cv, x1, y1, rad);
}

// records of the pipeline -> the reference's `poses.round().astype('i')` (:513-514 then :539):
// x = rint(double(peak x) * sx), y likewise, v = 2 for a present joint; absent joints are (0, 0, 0).  Joint j of
// record p -> poses row i.
__device__ __forceinline__ void ov_pose_joint(const int* __restrict__ rec_x, const int* __restrict__ rec_y,
                                              const int* __restrict__ rec_id, int person_stride_ints, size_t p, int j,
                                              double sx, double sy, int* __restrict__ poses, size_t i) {
  const bool has = rec_id[p * person_stride_ints + j] >= 0;
  poses[3 * i + 0] = has ? __double2int_rn(__dmul_rn(static_cast<double>(rec_x[p * person_stride_ints + j]), sx)) : 0;
  poses[3 * i + 1] = has ? __double2int_rn(__dmul_rn(static_cast<double>(rec_y[p * person_stride_ints + j]), sy)) : 0;
  poses[3 * i + 2] = has ? 2 : 0;
}

__global__ void overlay_poses_from_records_kernel(const int* __restrict__ rec_x, const int* __restrict__ rec_y,
                                                  const int* __restrict__ rec_id, int person_stride_ints, int n_persons,
                                                  double sx, double sy, int* __restrict__ poses) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_persons * OV_JOINTS) return;
  const int p = i / OV_JOINTS, j = i - p * OV_JOINTS;
  ov_pose_joint(rec_x, rec_y, rec_id, person_stride_ints, static_cast<size_t>(p), j, sx, sy, poses, static_cast<size_t>(i));
}

// primitive j (< OV_PART_STRIDE) of one face / hand part; pts: the part's (x, y, present) rows in crop coordinates
__device__ inline void ov_part_primitive(const OvCanvas& cv, const OverlayTables& tb, const OvPart& pt, const int* pts, int j) {
  if (pt.kind == OV_PART_FACE) {
    if (j < OV_FACE_POINTS) {
      const int* a = pts + 3 * j;
      if (a[2]) ov_circle_fill(cv, a[0] + pt.left, a[1] + pt.top, 2);
    } else if (j < OV_FACE_POINTS + OV_FACE_LINES) {
      const int* a = pts + 3 * tb.face_line[j - OV_FACE_POINTS][0];
      const int* b = pts + 3 * tb.face_line[j - OV_FACE_POINTS][1];
      if (a[2] && b[2]) ov_line1(cv, a[0] + pt.left, a[1] + pt.top, b[0] + pt.left, b[1] + pt.top);
    } else {
      ov_rect1(cv, pt.left, pt.top, pt.right, pt.bottom);
    }
  } else if (j < OV_HAND_PRIMS) {
    const int f = j / (OV_FINGER_SEGS * 3), r = j - f * (OV_FINGER_SEGS * 3), s = r / 3, step = r - 3 * s;
    const int* a = pts + 3 * tb.finger[f][s][0];
    const int* b = pts + 3 * tb.finger[f][s][1];
    if (step == 0) {
      if (a[2]) ov_circle_fill(cv, a[0] + pt.left, a[1] + pt.top, 3);
    } else if (step == 1) {
      if (b[2]) ov_circle_fill(cv, b[0] + pt.left, b[1] + pt.top, 3);
    } else if (a[2] && b[2]) {
      ov_line1(cv, a[0] + pt.left, a[1] + pt.top, b[0] + pt.left, b[1] + pt.top);
    }
  } else if (j == OV_HAND_PRIMS) {
    ov_rect1(cv, pt.left, pt.top, pt.right, pt.bottom);
  }
}

// primitive i of one picture's index space [n_poses * 19 limbs | n_poses * 18 joints | n_parts * OV_PART_STRIDE part
// primitives] in the reference's drawing order, drawn with priority i + 1.  `bad` is raised when a drawn joint lies
// outside the image.
__device__ inline void ov_raster_primitive(const int* __restrict__ poses, int n_poses, const OverlayTables& tb,
                                           unsigned int* __restrict__ prio, int H, int W, int* __restrict__ bad,
                                           const OvPart* __restrict__ parts, const int* __restrict__ points, int i) {
  const int n_limb = n_poses * OV_LIMBS, n_skel = n_limb + n_poses * OV_JOINTS;
  OvCanvas cv{prio, H, W, static_cast<unsigned int>(i) + 1u};
  if (i < n_limb) {
    const int p = i / OV_LIMBS, l = i - p * OV_LIMBS;
    if (l == 9 || l == 13) return;
    const int* a = poses + (static_cast<size_t>(p) * OV_JOINTS + tb.limb_a[l]) * 3;
    const int* b = poses + (static_cast<size_t>(p) * OV_JOINTS + tb.limb_b[l]) * 3;
    if (a[2] == 0 || b[2] == 0) return;
    if (a[0] < 0 || a[0] >= W || a[1] < 0 || a[1] >= H || b[0] < 0 || b[0] >= W || b[1] < 0 || b[1] >= H) { atomicOr(bad, 1); return; }
    ov_thick_line2(cv, a[0], a[1], b[0], b[1]);
  } else if (i < n_skel) {
    const int k = i - n_limb;
    const int* a = poses + static_cast<size_t>(k) * 3;
    if (a[2] == 0) return;
    if (a[0] < 0 || a[0] >= W || a[1] < 0 || a[1] >= H) { atomicOr(bad, 1); return; }
    ov_circle_fill(cv, a[0], a[1], 3);
  } else {
    const int q = i - n_skel, p = q / OV_PART_STRIDE;
    const OvPart pt = parts[p];
    ov_part_primitive(cv, tb, pt, points + static_cast<size_t>(pt.first_point) * 3, q - p * OV_PART_STRIDE);
  }
}

// one thread per potential primitive of one picture
__global__ void overlay_raster_kernel(const int* __restrict__ poses, int n_poses, OverlayTables tb, unsigned int* __restrict__ prio,
                                      int H, int W, int* __restrict__ bad, const OvPart* __restrict__ parts, int n_parts,
                                      const int* __restrict__ points) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_poses * (OV_LIMBS + OV_JOINTS) + n_parts * OV_PART_STRIDE) return;
  ov_raster_primitive(poses, n_poses, tb, prio, H, W, bad, parts, points, i);
}

// ---- n pictures of equally sized frames in one raster and one paint launch (opb_whole_body_batch) ----
// Frame f keeps its own 1-based priority index space [limbs | joints | parts] and its own priority plane
// prio + f * H * W.  Its primitives are prim0 .. prim0 + n_poses * 37 + n_parts * OV_PART_STRIDE - 1 of the launch;
// its poses start at person f * pose_stride of `poses`, its parts at parts + part0 (first_point indexes the shared points).
struct OvFrame {
  int prim0, n_poses, part0, n_parts;
};

// The frame that owns primitive t: the last of frames[0..n) with prim0 <= t (prim0 ascending, frames[0].prim0 == 0);
// a frame without primitives shares its prim0 with the next one and is never returned for a t it does not own.
__device__ __forceinline__ int ov_find_frame(const OvFrame* __restrict__ frames, int n, int t) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (frames[mid].prim0 <= t) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// the records of n_frames frames, max_persons (= cap) each, frame f's persons at f * cap: joint rows of the first
// frames[f].n_poses persons of every frame go to poses [n_frames][cap][18][3]; grid over n_frames * cap * 18 threads
__global__ void overlay_poses_from_records_batch_kernel(const int* __restrict__ rec_x, const int* __restrict__ rec_y,
                                                        const int* __restrict__ rec_id, int person_stride_ints, int cap,
                                                        const OvFrame* __restrict__ frames, int n_frames, double sx,
                                                        double sy, int* __restrict__ poses) {
  const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= static_cast<size_t>(n_frames) * cap * OV_JOINTS) return;
  const size_t p = i / OV_JOINTS;
  const int j = static_cast<int>(i - p * OV_JOINTS), f = static_cast<int>(p / cap);
  if (static_cast<int>(p - static_cast<size_t>(f) * cap) >= frames[f].n_poses) return;
  ov_pose_joint(rec_x, rec_y, rec_id, person_stride_ints, p, j, sx, sy, poses, i);
}

// one thread per potential primitive of all n_frames pictures (n_prim in all); pose_stride: persons per frame in poses
__global__ void overlay_raster_batch_kernel(const int* __restrict__ poses, int pose_stride, const OvFrame* __restrict__ frames,
                                            int n_frames, int n_prim, OverlayTables tb, unsigned int* __restrict__ prio,
                                            int H, int W, int* __restrict__ bad, const OvPart* __restrict__ parts,
                                            const int* __restrict__ points) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_prim) return;
  const int f = ov_find_frame(frames, n_frames, i);
  const OvFrame fr = frames[f];
  ov_raster_primitive(poses + static_cast<size_t>(f) * pose_stride * OV_JOINTS * 3, fr.n_poses, tb,
                      prio + static_cast<size_t>(f) * H * W, H, W, bad, parts + fr.part0, points, i - fr.prim0);
}

// cv2.addWeighted(a, 0.6, b, 0.4, 0) on uint8: saturate_cast<uchar>(a*0.6f + (b*0.4f + 0.f)) in float32, rounded half
// to even (the same bits with or without a fused multiply-add for every (a, b) pair)
__device__ __forceinline__ uint8_t ov_blend(uint8_t a, uint8_t b) {
  const float r = __fadd_rn(__fmul_rn(static_cast<float>(a), 0.6f), __fadd_rn(__fmul_rn(static_cast<float>(b), 0.4f), 0.f));
  const int v = __float2int_rn(r);
  return static_cast<uint8_t>(v < 0 ? 0 : (v > 255 ? 255 : v));
}

// canvas = orig_img.copy(), then every covered pixel takes the colour of its last primitive.  blend != 0 (whole-body
// picture): skeleton pixels take blend(img, skeleton colour) instead; part pixels always take the part's colour.
// Pixel i of one picture.
__device__ __forceinline__ void ov_paint_pixel(const uint8_t* __restrict__ img, const unsigned int* __restrict__ prio,
                                               int n_poses, const OverlayTables& tb, uint8_t* __restrict__ out,
                                               const OvPart* __restrict__ parts, int blend, size_t i) {
  const unsigned int t = prio[i];
  uint8_t c0 = img[3 * static_cast<size_t>(i)], c1 = img[3 * static_cast<size_t>(i) + 1], c2 = img[3 * static_cast<size_t>(i) + 2];
  if (t) {
    const int k = static_cast<int>(t) - 1, n_limb = n_poses * OV_LIMBS, n_skel = n_limb + n_poses * OV_JOINTS;
    if (k < n_skel) {
      const uint8_t* col = (k < n_limb) ? tb.limb_color[k % OV_LIMBS] : tb.joint_color[(k - n_limb) % OV_JOINTS];
      if (blend) {
        c0 = ov_blend(c0, col[0]); c1 = ov_blend(c1, col[1]); c2 = ov_blend(c2, col[2]);
      } else {
        c0 = col[0]; c1 = col[1]; c2 = col[2];
      }
    } else {
      const int q = k - n_skel, p = q / OV_PART_STRIDE, j = q - p * OV_PART_STRIDE;
      const uint8_t* col;
      if (parts[p].kind == OV_PART_FACE) col = j < OV_FACE_POINTS + OV_FACE_LINES ? tb.face_color : tb.rect_color;
      else col = j < OV_HAND_PRIMS ? tb.finger_color[j / (OV_FINGER_SEGS * 3)] : tb.rect_color;
      c0 = col[0]; c1 = col[1]; c2 = col[2];
    }
  }
  out[3 * static_cast<size_t>(i)] = c0;
  out[3 * static_cast<size_t>(i) + 1] = c1;
  out[3 * static_cast<size_t>(i) + 2] = c2;
}

__global__ void __launch_bounds__(256)
overlay_paint_kernel(const uint8_t* __restrict__ img, const unsigned int* __restrict__ prio, int n_pix, int n_poses,
                     OverlayTables tb, uint8_t* __restrict__ out, const OvPart* __restrict__ parts, int blend) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_pix) return;
  ov_paint_pixel(img, prio, n_poses, tb, out, parts, blend, static_cast<size_t>(i));
}

// n_frames whole-body pictures [n_frames][n_pix] (blend on): a thread finds its frame from its pixel index
__global__ void __launch_bounds__(256)
overlay_paint_batch_kernel(const uint8_t* __restrict__ imgs, const unsigned int* __restrict__ prio, int n_pix,
                           const OvFrame* __restrict__ frames, int n_frames, OverlayTables tb, uint8_t* __restrict__ out,
                           const OvPart* __restrict__ parts) {
  const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= static_cast<size_t>(n_frames) * n_pix) return;
  const int f = static_cast<int>(i / static_cast<size_t>(n_pix));
  const OvFrame fr = frames[f];
  ov_paint_pixel(imgs, prio, fr.n_poses, tb, out, parts + fr.part0, 1, i);
}

}  // namespace opb
