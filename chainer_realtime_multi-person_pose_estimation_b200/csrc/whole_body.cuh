// whole_body.cuh -- the per-person crop boxes of demo.py:31-57 on the device, from the result records of the last
// detect: PoseDetector.get_unit_length (compute_limbs_length + compute_unit_length, pose_detector.py:267-297),
// crop_face and crop_hands (:354-392) in float64, exactly as the host helpers compute them from _poses_from_records'
// poses:
//   joint j = (fl(x * sx), fl(y * sy)) when peak_id >= 0, else (0, 0).  compute_limbs_length never sees None (a pose
//     row is an array), so EVERY limb is measured, a missing joint counting as the origin.
//   limb length = np.linalg.norm(b - a) = sqrt(fma(dy, dy, fl(dx * dx))) (NumPy's 2-element dot).
//   unit length: limbs [14, 3, 0, 13, 9] with ratios (0.85, 2.2, 2.2, 0.85, 0.85) when any of them is positive,
//     summed left to right; else every positive limb over the 19-entry ratio table, summed as np.sum does (pairwise:
//     from 8 terms up, 8 accumulators over blocks of 8, combined ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)), then the
//     remainder one by one); then divided by the count.
//   face box (nose present): int(nx - u), int(ny - fl(u*1.2)), int(nx + u), int(ny + fl(u*0.8)).
//   hand box (hand present): c = hand + fl(0.3 * fl(hand - elbow)) when the elbow is present, cs = fl(u * 0.95),
//     int(c - cs), int(c + cs) per axis.
// int() truncates toward zero; a value outside int32 is reported (status), never converted.  Every product is rounded
// on its own (__dmul_rn / __dadd_rn / __dsub_rn: nvcc would otherwise contract a*b + c into an FMA); the norm's one
// FMA is explicit.
//
// Skipping policy of the one-call path (the demo would raise instead): a person whose unit length is not finite (no
// limb of positive length: 0/0) gets no part; a box of non-positive width or height is not a part.  The kept parts are
// compacted in the demo's order (per person: face, left hand, right hand) into the face table, the hand table
// (flip = 1 for left hands) and the part list.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "paf.cuh"

namespace opb {

constexpr int WB_THREADS = 256;
constexpr int WB_FACE = 0, WB_LEFT = 1, WB_RIGHT = 2;
constexpr int WB_ERR_RANGE = -6;      // OPB_ERR_UNSUPPORTED: a box edge does not fit int32

struct WbCrop { int left, top, right, bottom, flip, reserved; };  // == opb_crop
struct WbPart { int side, person, row, reserved; };              // row: index into the face or the hand table
struct WbCounts { int status, n_face, n_hand, n_parts; };

struct WbOut {
  WbCounts* counts;
  double* unit;     // [cap]        unit length per person (NaN when no limb is positive)
  int* box;         // [cap][3][4]  face, left hand, right hand (valid where the present bit is set)
  int* present;     // [cap]        bit k: the helper returns box k (joint present, unit length finite)
  WbCrop* face;     // [cap]
  WbCrop* hand;     // [2 cap]
  WbPart* parts;    // [3 cap]
};

__device__ __forceinline__ bool wb_trunc(double v, int* out) {
  if (!(v > -2147483649.0 && v < 2147483648.0)) return false;   // also false for NaN
  *out = static_cast<int>(v);                                   // in range: truncation toward zero, as int()
  return true;
}

// ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)) of NumPy's pairwise_sum
__device__ __forceinline__ double wb_combine8(const double (&r)[8]) {
  return __dadd_rn(__dadd_rn(__dadd_rn(r[0], r[1]), __dadd_rn(r[2], r[3])),
                   __dadd_rn(__dadd_rn(r[4], r[5]), __dadd_rn(r[6], r[7])));
}

// One person: unit length, the three boxes, the present bits and the kept bits.  Returns false when a box edge does
// not fit int32.
__device__ __forceinline__ bool wb_person(const PersonOut& rec, double sx, double sy, double* unit_out, int box[3][4],
                          int* present_out, int* keep_out) {
  double jx[18], jy[18];
#pragma unroll
  for (int j = 0; j < 18; ++j) {
    const bool has = rec.peak_id[j] >= 0;
    jx[j] = has ? __dmul_rn(static_cast<double>(rec.x[j]), sx) : 0.0;
    jy[j] = has ? __dmul_rn(static_cast<double>(rec.y[j]), sy) : 0.0;
  }
  // params['limbs_point'] (entity.py:85-105): the helpers always use these, whatever limbs the context was created with
  const int limb_a[19] = {1, 8, 9, 1, 11, 12, 1, 2, 3, 2, 1, 5, 6, 5, 1, 0, 0, 14, 15};
  const int limb_b[19] = {8, 9, 10, 11, 12, 13, 2, 3, 4, 16, 5, 6, 7, 17, 0, 14, 15, 16, 17};
  double len[19];
#pragma unroll
  for (int l = 0; l < 19; ++l) {
    const double dx = __dsub_rn(jx[limb_b[l]], jx[limb_a[l]]), dy = __dsub_rn(jy[limb_b[l]], jy[limb_a[l]]);
    len[l] = __dsqrt_rn(fma(dy, dy, __dmul_rn(dx, dx)));
  }
  double u;
  {
    const int pick[5] = {14, 3, 0, 13, 9};
    const double ratio[5] = {0.85, 2.2, 2.2, 0.85, 0.85};
    double s = 0.0;
    int n = 0;
#pragma unroll
    for (int k = 0; k < 5; ++k)
      if (len[pick[k]] > 0.0) { s = __dadd_rn(s, __ddiv_rn(len[pick[k]], ratio[k])); ++n; }
    if (n > 0) {
      u = __ddiv_rn(s, static_cast<double>(n));
    } else {
      const double ratio19[19] = {2.2, 1.7, 1.7, 2.2, 1.7, 1.7, 0.6, 0.93, 0.65, 0.85, 0.6, 0.93, 0.65, 0.85, 1.0, 0.2,
                                  0.2, 0.25, 0.25};
#pragma unroll
      for (int l = 0; l < 19; ++l) n += len[l] > 0.0;
      const int full = n >= 8 ? n - n % 8 : 0;   // terms [0, full) go through the 8 accumulators
      double r[8] = {0, 0, 0, 0, 0, 0, 0, 0};
      s = 0.0;
      int k = 0;
#pragma unroll
      for (int l = 0; l < 19; ++l) {
        if (!(len[l] > 0.0)) continue;
        const double t = __ddiv_rn(len[l], ratio19[l]);
        if (k < full) {
#pragma unroll
          for (int q = 0; q < 8; ++q)
            if ((k & 7) == q) r[q] = k < 8 ? t : __dadd_rn(r[q], t);
        } else {
          if (k == full && full > 0) s = wb_combine8(r);
          s = __dadd_rn(s, t);
        }
        ++k;
      }
      if (full > 0 && full == n) s = wb_combine8(r);
      u = __ddiv_rn(s, static_cast<double>(n));    // 0 / 0 = NaN without a positive limb
    }
  }
  *unit_out = u;
  int present = 0, keep = 0;
  bool ok = true;
  if (u - u == 0.0) {                             // finite (NaN and inf give NaN)
    double e[3][4];
    if (rec.peak_id[0] >= 0) {                    // JointType.Nose
      const double nx = jx[0], ny = jy[0];
      e[0][0] = __dsub_rn(nx, u);
      e[0][1] = __dsub_rn(ny, __dmul_rn(u, 1.2));
      e[0][2] = __dadd_rn(nx, u);
      e[0][3] = __dadd_rn(ny, __dmul_rn(u, 0.8));
      present |= 1;
    }
    const double cs = __dmul_rn(u, 0.95);
    const int hand_j[2] = {7, 4}, elbow_j[2] = {6, 3};   // LeftHand / LeftElbow, RightHand / RightElbow
#pragma unroll
    for (int s = 0; s < 2; ++s) {
      const int hj = hand_j[s], ej = elbow_j[s];
      if (rec.peak_id[hj] < 0) continue;
      double cx = jx[hj], cy = jy[hj];
      if (rec.peak_id[ej] >= 0) {
        cx = __dadd_rn(cx, __dmul_rn(0.3, __dsub_rn(jx[hj], jx[ej])));
        cy = __dadd_rn(cy, __dmul_rn(0.3, __dsub_rn(jy[hj], jy[ej])));
      }
      e[1 + s][0] = __dsub_rn(cx, cs);
      e[1 + s][1] = __dsub_rn(cy, cs);
      e[1 + s][2] = __dadd_rn(cx, cs);
      e[1 + s][3] = __dadd_rn(cy, cs);
      present |= 2 << s;
    }
#pragma unroll
    for (int p = 0; p < 3; ++p) {
      if (!(present >> p & 1)) continue;
#pragma unroll
      for (int c = 0; c < 4; ++c) ok = wb_trunc(e[p][c], &box[p][c]) && ok;
      if (box[p][2] > box[p][0] && box[p][3] > box[p][1]) keep |= 1 << p;
    }
  }
  *present_out = present;
  *keep_out = ok ? keep : 0;
  return ok;
}

// Grid n, one block of WB_THREADS per frame: block f reads hd[f] and persons[f * cap ..] and writes the frame's
// section of every output (counts[f]; unit, box, present and the face table from f * cap; the hand table from
// f * 2 cap; the part list from f * 3 cap), persons in chunks of WB_THREADS, a block scan of each chunk's kept faces
// and hands placing them in the demo's order.  A frame with an error status or without peaks contributes nothing.
__global__ void __launch_bounds__(WB_THREADS)
whole_body_boxes_kernel(const ImageHeader* __restrict__ hd, const PersonOut* __restrict__ persons, int cap, double sx,
                        double sy, WbOut out) {
  __shared__ int scan[2][WB_THREADS];
  __shared__ int base_face, base_hand, bad;
  const int tid = threadIdx.x;
  const size_t f = blockIdx.x, fc = f * static_cast<size_t>(cap);
  persons += fc;
  out.counts += f;
  out.unit += fc;
  out.box += fc * 12;
  out.present += fc;
  out.face += fc;
  out.hand += 2 * fc;
  out.parts += 3 * fc;
  const ImageHeader h = hd[f];
  if (h.status != 0) {
    if (tid == 0) *out.counts = WbCounts{h.status, 0, 0, 0};
    return;
  }
  const int n = h.n_peaks == 0 ? 0 : min(h.n_persons, cap);   // _poses_from_records: no peaks, no persons
  if (tid == 0) { base_face = 0; base_hand = 0; bad = 0; }
  __syncthreads();
  for (int p0 = 0; p0 < n; p0 += WB_THREADS) {
    const int p = p0 + tid;
    int keep = 0;
    int box[3][4] = {};
    if (p < n) {
      int present = 0;
      double u;
      if (!wb_person(persons[p], sx, sy, &u, box, &present, &keep)) bad = 1;
      out.unit[p] = u;
      out.present[p] = present;
#pragma unroll
      for (int q = 0; q < 3; ++q)
#pragma unroll
        for (int c = 0; c < 4; ++c) out.box[(p * 3 + q) * 4 + c] = box[q][c];
    }
    // inclusive scan of (faces | hands << 16) over the chunk
    const int mine = (keep & 1) + ((((keep >> 1) & 1) + ((keep >> 2) & 1)) << 16);
    int buf = 0;
    scan[0][tid] = mine;
    __syncthreads();
    for (int d = 1; d < WB_THREADS; d <<= 1) {
      const int v = scan[buf][tid] + (tid >= d ? scan[buf][tid - d] : 0);
      scan[buf ^ 1][tid] = v;
      buf ^= 1;
      __syncthreads();
    }
    const int excl = scan[buf][tid] - mine;
    int f = base_face + (excl & 0xffff), hh = base_hand + (excl >> 16);
    if (p < n && keep) {
      int part = f + hh;                           // parts before this person's = faces + hands before it
      if (keep & 1) {
        out.face[f] = WbCrop{box[0][0], box[0][1], box[0][2], box[0][3], 0, 0};
        out.parts[part++] = WbPart{WB_FACE, p, f, 0};
        ++f;
      }
#pragma unroll
      for (int s = 0; s < 2; ++s) {
        if (!(keep >> (1 + s) & 1)) continue;
        out.hand[hh] = WbCrop{box[1 + s][0], box[1 + s][1], box[1 + s][2], box[1 + s][3], s == 0 ? 1 : 0, 0};
        out.parts[part++] = WbPart{s == 0 ? WB_LEFT : WB_RIGHT, p, hh, 0};
        ++hh;
      }
    }
    __syncthreads();
    if (tid == WB_THREADS - 1) { base_face += scan[buf][tid] & 0xffff; base_hand += scan[buf][tid] >> 16; }
    __syncthreads();
  }
  if (tid == 0) {
    *out.counts = bad ? WbCounts{WB_ERR_RANGE, 0, 0, 0} : WbCounts{0, base_face, base_hand, base_face + base_hand};
  }
}

}  // namespace opb
