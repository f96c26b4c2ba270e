// cascade.cuh -- cv2.CascadeClassifier.detectMultiScale for stump-based HAAR cascades on the device, bit-exact
// (objdetect/cascadedetect.cpp of OpenCV 4.x; pinned in NumPy by tests/haar_ref.py, DESIGN.md "Haar cascade").
//
// Every pyramid layer lives in one buffer with one pitch P, as OpenCV keeps them, so a feature's rectangle corners are
// the same offsets from a window's top-left at every scale: the stump table carries them, built on the host per P.
//   layer i: (h_i + 1) x (w_i + 1) integral rows starting at row row0_i; layer image pixel (y, x) at (row0_i + y + 1)*P
//   + x + 1 of the uint8 plane (the integral's own position), so the row scan reads it in place.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace opb {

struct CascadeLayer {
  int h, w;           // layer size: cvRound(H / sc), cvRound(W / sc)
  int row0;           // first integral row of the layer in the shared buffer
  int ystep;          // 2 if sc < 2, else 1
  int nx, ny;         // windows per row / rows of windows (x, y over the working size in ystep)
  int win0;           // first window of the layer in the flat enumeration
  int xtab, ytab;     // first entry of the layer's column / row interpolation records
  float scale;
};

struct CascadeAxis {  // INTER_LINEAR_EXACT, one output column or row: s0, s1 (clamped), c1 (of 256)
  int s0, s1, c1, pad;
};

struct CascadeStump { // one stump with its feature's rect corners as offsets from the window's top-left
  int ofs[3][4];      // p0 - p1 - p2 + p3 of rect r: (y)P+x, (y)P+x+w, (y+h)P+x, (y+h)P+x+w
  float w[3];         // rect weights (w[2] == 0: two rects)
  float thr, left, right;
};

struct CascadeStage {
  int first, ntrees;
  float thr;          // stageThreshold - 1e-5f (THRESHOLD_EPS, applied at load)
  int pad;
};

struct CascadeWindowSetup {
  int nofs[4];        // normrect (1, 1, winW-2, winH-2) corners
  double area;
};

constexpr int kCascadeSmemStumps = 128;   // stumps of the first stages held in shared memory (frontalface_alt: 3 + 16
                                          // + 21 + 39 + 33 = 112 cover the stages that see most windows)
constexpr int kCascadeMaxStages = 64;

__device__ __forceinline__ uint32_t cascade_gray(const uint8_t* __restrict__ f, int fw, int ch, int y, int x) {
  if (ch == 1) return f[static_cast<size_t>(y) * fw + x];
  const uint8_t* p = f + (static_cast<size_t>(y) * fw + x) * 3;   // cvtColor(BGR2GRAY): fixed point, 15 bits
  return (p[0] * 3735u + p[1] * 19235u + p[2] * 9798u + (1u << 14)) >> 15;
}

// Gray conversion and every INTER_LINEAR_EXACT layer in one launch: grid (ceil(maxw/32), ceil(maxh/8), layers).
// Horizontal sums in 8.8, vertical in 16.16, (v + 2^15) >> 16.  Block (0,0,0) also resets the candidate count.
__global__ void __launch_bounds__(256)
cascade_pyramid_kernel(const uint8_t* __restrict__ frame, int fh, int fw, int ch, const CascadeLayer* __restrict__ layers,
                       const CascadeAxis* __restrict__ axes, uint8_t* __restrict__ img, int pitch, int* cand_count) {
  if (blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == 0 && threadIdx.x == 0 && threadIdx.y == 0) *cand_count = 0;
  const CascadeLayer L = layers[blockIdx.z];
  const int x = blockIdx.x * 32 + threadIdx.x, y = blockIdx.y * 8 + threadIdx.y;
  if (x >= L.w || y >= L.h) return;
  const CascadeAxis ax = axes[L.xtab + x], ay = axes[L.ytab + y];
  const uint32_t a1 = ax.c1, a0 = 256 - a1, b1 = ay.c1, b0 = 256 - b1;
  const uint32_t h0 = cascade_gray(frame, fw, ch, ay.s0, ax.s0) * a0 + cascade_gray(frame, fw, ch, ay.s0, ax.s1) * a1;
  const uint32_t h1 = cascade_gray(frame, fw, ch, ay.s1, ax.s0) * a0 + cascade_gray(frame, fw, ch, ay.s1, ax.s1) * a1;
  img[static_cast<size_t>(L.row0 + y + 1) * pitch + x + 1] = static_cast<uint8_t>((h0 * b0 + h1 * b1 + (1u << 15)) >> 16);
}

// Row prefix sums of pixel and pixel^2 (uint32: OpenCV's int32 sqsum wraps, only differences are used), one warp per
// integral row; row 0 and column 0 of every layer are zero.  grid (ceil((maxh+1)/8), layers), block (32, 8).
__global__ void __launch_bounds__(256)
cascade_row_scan_kernel(const CascadeLayer* __restrict__ layers, const uint8_t* __restrict__ img, int pitch,
                        uint32_t* __restrict__ sum, uint32_t* __restrict__ sq) {
  const CascadeLayer L = layers[blockIdx.y];
  const int r = blockIdx.x * 8 + threadIdx.y, lane = threadIdx.x;
  if (r > L.h) return;
  const size_t row = static_cast<size_t>(L.row0 + r) * pitch;
  uint32_t cs = 0, cq = 0;
  for (int x0 = 0; x0 <= L.w; x0 += 32) {
    const int x = x0 + lane;
    uint32_t v = (r > 0 && x > 0 && x <= L.w) ? img[row + x] : 0u;
    uint32_t s = v, q = v * v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const uint32_t ts = __shfl_up_sync(0xffffffffu, s, d), tq = __shfl_up_sync(0xffffffffu, q, d);
      if (lane >= d) { s += ts; q += tq; }
    }
    if (x <= L.w) { sum[row + x] = cs + s; sq[row + x] = cq + q; }
    cs += __shfl_sync(0xffffffffu, s, 31);
    cq += __shfl_sync(0xffffffffu, q, 31);
  }
}

// Column prefix sums in place: one thread per integral column.  grid (ceil(maxw+1 / 128), layers), block 128.
__global__ void __launch_bounds__(128)
cascade_col_scan_kernel(const CascadeLayer* __restrict__ layers, int pitch, uint32_t* __restrict__ sum,
                        uint32_t* __restrict__ sq) {
  const CascadeLayer L = layers[blockIdx.y];
  const int x = blockIdx.x * 128 + threadIdx.x;
  if (x > L.w) return;
  size_t p = static_cast<size_t>(L.row0 + 1) * pitch + x;
  uint32_t cs = 0, cq = 0;
  for (int r = 1; r <= L.h; ++r, p += pitch) {
    cs += sum[p]; cq += sq[p];
    sum[p] = cs; sq[p] = cq;
  }
}

__device__ __forceinline__ int cascade_rect(const uint32_t* __restrict__ p, const int (&o)[4]) {
  return static_cast<int>(p[o[0]] - p[o[1]] - p[o[2]] + p[o[3]]);
}

// One thread per window of every layer (before the skip rule): code -1 (variance test fails), -k (stage k rejects), or
// 1 (passes); with `sums`, also the final stage sum.  Single IEEE operations throughout, so nothing is contracted.
__global__ void __launch_bounds__(128)
cascade_eval_kernel(const CascadeLayer* __restrict__ layers, int n_layers, int n_windows, int pitch,
                    const uint32_t* __restrict__ sum, const uint32_t* __restrict__ sq,
                    const CascadeStage* __restrict__ stages, int n_stages, const CascadeStump* __restrict__ stumps,
                    int n_stumps, CascadeWindowSetup ws, int* __restrict__ codes, double* __restrict__ sums) {
  __shared__ CascadeStage s_stage[kCascadeMaxStages];
  __shared__ CascadeStump s_stump[kCascadeSmemStumps];
  const int n_smem = min(n_stumps, kCascadeSmemStumps);
  for (int i = threadIdx.x; i < n_stages; i += blockDim.x) s_stage[i] = stages[i];
  for (int i = threadIdx.x; i < n_smem; i += blockDim.x) s_stump[i] = stumps[i];
  __syncthreads();
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n_windows) return;
  int lo = 0, hi = n_layers - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (__ldg(&layers[mid].win0) <= k) lo = mid; else hi = mid - 1;
  }
  const CascadeLayer L = layers[lo];
  const int j = k - L.win0, wy = (j / L.nx) * L.ystep, wx = (j % L.nx) * L.ystep;
  const size_t base = static_cast<size_t>(L.row0 + wy) * pitch + wx;
  const uint32_t* ps = sum + base;
  const uint32_t* pq = sq + base;
  const double vs = static_cast<double>(cascade_rect(ps, ws.nofs));
  const double vq = static_cast<double>(static_cast<uint32_t>(cascade_rect(pq, ws.nofs)));
  const double nf = __dsub_rn(__dmul_rn(ws.area, vq), __dmul_rn(vs, vs));
  int code = 1;
  double acc = 0.0;
  float vnf = 1.f;
  if (nf > 0.0) vnf = __double2float_rn(__ddiv_rn(1.0, __dsqrt_rn(nf)));
  if (!(nf > 0.0) || !(__dmul_rn(ws.area, static_cast<double>(vnf)) < 0.1)) {
    code = -1;
  } else {
    for (int s = 0; s < n_stages; ++s) {
      const CascadeStage st = s_stage[s];
      acc = 0.0;
      for (int t = st.first; t < st.first + st.ntrees; ++t) {
        const CascadeStump& u = t < kCascadeSmemStumps ? s_stump[t] : stumps[t];
        float ret = __fadd_rn(__fmul_rn(u.w[0], static_cast<float>(cascade_rect(ps, u.ofs[0]))),
                              __fmul_rn(u.w[1], static_cast<float>(cascade_rect(ps, u.ofs[1]))));
        if (u.w[2] != 0.f) ret = __fadd_rn(ret, __fmul_rn(u.w[2], static_cast<float>(cascade_rect(ps, u.ofs[2]))));
        const float value = __fmul_rn(ret, vnf);
        acc = __dadd_rn(acc, static_cast<double>(value < u.thr ? u.left : u.right));
      }
      if (acc < static_cast<double>(st.thr)) { code = -s; break; }
    }
  }
  codes[k] = code;
  if (sums) sums[k] = acc;
}

// CascadeClassifierInvoker's scan of one row of windows: x restarts at 0, and a window rejected by stage 0 (code 0)
// skips the next x.  Passing windows visited by that scan are appended as (layer, x, y) after the count in cand[0].
// One warp per row of windows: the lanes load 32 codes, lane 0 resolves the skip chain on the ballot bits.
// grid (ceil(max ny / 4), layers), block (32, 4).
__global__ void __launch_bounds__(128)
cascade_compact_kernel(const CascadeLayer* __restrict__ layers, const int* __restrict__ codes, int* __restrict__ cand,
                       int cap) {
  const CascadeLayer L = layers[blockIdx.y];
  const int row = blockIdx.x * 4 + threadIdx.y, lane = threadIdx.x;
  if (row >= L.ny) return;
  const int* c = codes + L.win0 + static_cast<size_t>(row) * L.nx;
  bool skip = false;   // the previous visited window was rejected by stage 0
  for (int i0 = 0; i0 < L.nx; i0 += 32) {
    const int i = i0 + lane;
    const int v = i < L.nx ? c[i] : -1;
    const unsigned zero = __ballot_sync(0xffffffffu, v == 0);
    unsigned visited = 0;
    if (lane == 0) {
      for (int b = 0; b < 32; ++b) {
        if (!skip) { visited |= 1u << b; skip = (zero >> b) & 1u; }
        else skip = false;
      }
    }
    visited = __shfl_sync(0xffffffffu, visited, 0);
    skip = __shfl_sync(0xffffffffu, skip, 0);
    if (((visited >> lane) & 1u) && v > 0) {
      const int slot = atomicAdd(cand, 1);
      if (slot < cap) {
        cand[1 + 3 * slot] = blockIdx.y;
        cand[2 + 3 * slot] = i * L.ystep;
        cand[3 + 3 * slot] = row * L.ystep;
      }
    }
  }
}

}  // namespace opb
