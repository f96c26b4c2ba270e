// conv_first.cuh -- conv1_1 (3 -> 64, 3x3, pad 1) + ReLU (models/CocoPoseNet.py:136) fused with
// preprocess (pose_detector.py:426-431: float32, /255, -0.5, BGR kept).  K = 27 is too small for
// a tensor-core tile, and the tensor cores would change the result bits: a direct fp32 CUDA-core
// kernel writing NHWC fp16 (plus the lo plane in parity mode, the correction bytes in compensated
// mode).  Every output channel is exactly `acc = bias; for r, s, c: acc = fmaf(x, w, acc)`.
//
// The layer is bound by its output (64 channels x 128 or 256 B per pixel, ~2 GB at batch 32 x
// 368 x 656 in the two-plane precisions) and by its 1728 FMAs per pixel, so the kernel is built
// around both:
// * Block = 8 x 32 output pixels, 8 warps.  Warp w computes output channels (w & 3) * 16 .. +15 of
//   tile rows (w >> 2) * 4 .. +3; a lane owns 4 horizontally adjacent pixels of one row.  Each
//   broadcast weight load (LDS.128, warp-uniform address) feeds 16 FMAs, and the 18 inputs of one
//   filter row are reused by 3 taps x 16 channels.
// * The uint8 halo tile is normalised once through a 256-entry look-up table (exactly
//   float32(v)/255 - 0.5, as the reference computes it) into shared memory.  Its rows are padded
//   to an odd pitch so that the 32 lanes of an input load hit 32 different banks.
// * The finished bytes of the whole tile (hi fp16 | lo fp16 or correction bytes) are staged in
//   shared memory in the output's NHWC layout, then written with 16-byte lanes: a tile row is one
//   contiguous run of 32 x 256 B (two-plane) or 32 x 128 B (fast) in global memory.  Staged 16-byte
//   chunks are XOR-swizzled within their pixel so that both the staging and the read-out are free
//   of bank conflicts.
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "conv_wgmma.cuh"   // compensated-precision byte helpers

namespace opb {

constexpr int CF_TH = 8, CF_TW = 32, CF_THREADS = 256;
constexpr int CF_IN_PITCH = (CF_TW + 2) * 3 + 1;                   // floats per halo row (odd: conflict-free loads)
constexpr int CF_W_BYTES = 27 * 64 * 4, CF_B_BYTES = 64 * 4, CF_LUT_BYTES = 256 * 4;
constexpr int CF_IN_BYTES = ((CF_TH + 2) * CF_IN_PITCH * 4 + 15) / 16 * 16;
constexpr int CF_STAGE_OFF = CF_W_BYTES + CF_B_BYTES + CF_LUT_BYTES + CF_IN_BYTES;

enum ConvFirstMode { CF_FAST = 0, CF_PARITY = 1, CF_COMP = 2 };

// bytes per output pixel: [hi 64 halves] (fast), [hi 64 halves | lo 64 halves] (parity),
// [hi 64 halves | fp8(lo * 2^11) 64 B | fp8(v) 64 B] (compensated)
__host__ __device__ constexpr int conv_first_pix_bytes(int mode) { return mode == CF_FAST ? 128 : 256; }
__host__ __device__ constexpr int conv_first_smem_bytes(int mode) {
  return CF_STAGE_OFF + CF_TH * CF_TW * conv_first_pix_bytes(mode);
}

// wt: [27][64] fp32 (k = (r*3+s)*3 + c), bias [64].
// x_u8: [N][H][W][3] uint8 BGR, or x_f32: [N][3][H][W] float32 (already preprocessed).
// out: [N][H][W] pixels of conv_first_pix_bytes(MODE) bytes.
template <int MODE>
__global__ void __launch_bounds__(CF_THREADS, 2)
conv_first_kernel(const uint8_t* __restrict__ x_u8, const float* __restrict__ x_f32, const float* __restrict__ wt,
                  const float* __restrict__ bias, uint8_t* __restrict__ out, int N, int H, int W, float u8_denom) {
  constexpr int PIX = conv_first_pix_bytes(MODE);
  constexpr int PIX_CHUNKS = PIX / 16;
  extern __shared__ __align__(16) uint8_t cf_smem[];
  float* s_w = reinterpret_cast<float*>(cf_smem);
  float* s_b = reinterpret_cast<float*>(cf_smem + CF_W_BYTES);
  float* s_lut = reinterpret_cast<float*>(cf_smem + CF_W_BYTES + CF_B_BYTES);
  float* s_in = reinterpret_cast<float*>(cf_smem + CF_W_BYTES + CF_B_BYTES + CF_LUT_BYTES);
  uint8_t* s_out = cf_smem + CF_STAGE_OFF;
  const int tid = threadIdx.x;
  for (int i = tid; i < 27 * 64; i += CF_THREADS) s_w[i] = wt[i];
  if (tid < 64) s_b[tid] = bias[tid];
  s_lut[tid] = __fsub_rn(__fdiv_rn(static_cast<float>(tid), u8_denom), 0.5f);   // 255: pose (:429), 256: face / hand
  const int tiles_x = (W + CF_TW - 1) / CF_TW, tiles_y = (H + CF_TH - 1) / CF_TH;
  const int warp = tid >> 5, lane = tid & 31;
  const int cg = warp & 3;                        // output channels cg*16 .. +15 (warp-uniform: broadcast weight loads)
  const int py = (warp >> 2) * 4 + (lane >> 3);   // tile row 0..7
  const int px = (lane & 7) * 4;                  // first of 4 tile columns
  const int total_tiles = N * tiles_y * tiles_x;
  constexpr int IN_ELEMS = (CF_TH + 2) * (CF_TW + 2) * 3;
  constexpr int PER_THREAD = (IN_ELEMS + CF_THREADS - 1) / CF_THREADS;
  float pre[PER_THREAD];   // next tile's (raw) inputs, in flight while this tile computes
  auto prefetch = [&](int tile) {
    const int n = tile / (tiles_y * tiles_x);
    const int rem = tile - n * (tiles_y * tiles_x);
    const int y0 = (rem / tiles_x) * CF_TH, x0 = (rem % tiles_x) * CF_TW;
#pragma unroll
    for (int e = 0; e < PER_THREAD; ++e) {
      const int i = tid + e * CF_THREADS;
      float v = 0.f;
      if (i < IN_ELEMS) {
        const int c = i % 3;
        const int q = i / 3;
        const int xx = x0 - 1 + q % (CF_TW + 2), yy = y0 - 1 + q / (CF_TW + 2);
        if (yy >= 0 && yy < H && xx >= 0 && xx < W) {
          if (x_u8) v = __int_as_float(static_cast<int>(x_u8[((static_cast<size_t>(n) * H + yy) * W + xx) * 3 + c]));
          else v = x_f32[((static_cast<size_t>(n) * 3 + c) * H + yy) * W + xx];
        } else {
          v = x_u8 ? __int_as_float(-1) : 0.f;   // -1 marks zero padding on the uint8 path
        }
      }
      pre[e] = v;
    }
  };
  if (static_cast<int>(blockIdx.x) < total_tiles) prefetch(blockIdx.x);
  for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
    const int n = tile / (tiles_y * tiles_x);
    const int rem = tile - n * (tiles_y * tiles_x);
    const int y0 = (rem / tiles_x) * CF_TH, x0 = (rem % tiles_x) * CF_TW;
    __syncthreads();   // LUT / weights ready; previous tile's s_in consumed and its staged bytes written out
#pragma unroll
    for (int e = 0; e < PER_THREAD; ++e) {
      const int i = tid + e * CF_THREADS;
      if (i < IN_ELEMS) {
        float v = pre[e];
        if (x_u8) { const int b = __float_as_int(v); v = (b < 0) ? 0.f : s_lut[b]; }
        const int row = i / ((CF_TW + 2) * 3);
        s_in[row * CF_IN_PITCH + i - row * ((CF_TW + 2) * 3)] = v;
      }
    }
    __syncthreads();
    if (tile + static_cast<int>(gridDim.x) < total_tiles) prefetch(tile + gridDim.x);
    float acc[4][16];   // [pixel px + p][channel cg*16 + j]
    {
      const float4* b4 = reinterpret_cast<const float4*>(s_b + cg * 16);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float4 bv = b4[j];
#pragma unroll
        for (int p = 0; p < 4; ++p) {
          acc[p][4 * j + 0] = bv.x; acc[p][4 * j + 1] = bv.y; acc[p][4 * j + 2] = bv.z; acc[p][4 * j + 3] = bv.w;
        }
      }
    }
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      float in[6 * 3];   // row py + r, columns px .. px+5 of the halo tile, 3 channels each
      const float* src = s_in + (py + r) * CF_IN_PITCH + px * 3;
#pragma unroll
      for (int q = 0; q < 18; ++q) in[q] = src[q];
#pragma unroll
      for (int s = 0; s < 3; ++s) {
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          const float4* w4 = reinterpret_cast<const float4*>(s_w + ((r * 3 + s) * 3 + c) * 64 + cg * 16);
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const float4 wv = w4[j];
#pragma unroll
            for (int p = 0; p < 4; ++p) {
              const float a = in[(p + s) * 3 + c];
              acc[p][4 * j + 0] = fmaf(a, wv.x, acc[p][4 * j + 0]);
              acc[p][4 * j + 1] = fmaf(a, wv.y, acc[p][4 * j + 1]);
              acc[p][4 * j + 2] = fmaf(a, wv.z, acc[p][4 * j + 2]);
              acc[p][4 * j + 3] = fmaf(a, wv.w, acc[p][4 * j + 3]);
            }
          }
        }
      }
    }
    // stage the finished bytes: 16-byte chunk k of tile pixel t lives at t * PIX + 16 * (k ^ ((t >> 2) & 7))
#pragma unroll
    for (int p = 0; p < 4; ++p) {
      const int t = py * CF_TW + px + p;
      uint8_t* o = s_out + t * PIX;
      const int sw = (t >> 2) & 7;
#pragma unroll
      for (int g = 0; g < 2; ++g) {   // channels cg*16 + g*8 .. +7
        uint32_t hi[4], lo[4];   // fp16 pairs, lower channel in the low half
        float v[8], l[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = fmaxf(acc[p][g * 8 + j], 0.f);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const __half2 h = __floats2half2_rn(v[2 * j], v[2 * j + 1]);
          hi[j] = *reinterpret_cast<const uint32_t*>(&h);
          const float h0 = __low2float(h), h1 = __high2float(h);
          if (MODE == CF_PARITY) {
            const __half2 q = __floats2half2_rn(v[2 * j] - h0, v[2 * j + 1] - h1);
            lo[j] = *reinterpret_cast<const uint32_t*>(&q);
          }
          if (MODE == CF_COMP) { l[2 * j] = (v[2 * j] - h0) * kCompLoScale; l[2 * j + 1] = (v[2 * j + 1] - h1) * kCompLoScale; }
        }
        *reinterpret_cast<uint4*>(o + 16 * ((cg * 2 + g) ^ sw)) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
        if (MODE == CF_PARITY) *reinterpret_cast<uint4*>(o + 16 * ((8 + cg * 2 + g) ^ sw)) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
        if (MODE == CF_COMP) {   // correction plane [fp8(lo * 2^11) 64 B | fp8(v) 64 B] of the single 64-channel chunk
          *reinterpret_cast<uint2*>(o + 16 * ((8 + cg) ^ sw) + 8 * g) =
              make_uint2(f32x4_to_act8x4(l[0], l[1], l[2], l[3]), f32x4_to_act8x4(l[4], l[5], l[6], l[7]));
          *reinterpret_cast<uint2*>(o + 16 * ((12 + cg) ^ sw) + 8 * g) =
              make_uint2(f32x4_to_act8x4(v[0], v[1], v[2], v[3]), f32x4_to_act8x4(v[4], v[5], v[6], v[7]));
        }
      }
    }
    __syncthreads();
    // write out: every 8 consecutive threads store one 128-byte run of a pixel row
    constexpr int ROW_CHUNKS = CF_TW * PIX_CHUNKS;
#pragma unroll 4
    for (int it = 0; it < CF_TH * ROW_CHUNKS / CF_THREADS; ++it) {
      const int id = tid + it * CF_THREADS;
      const int row = id / ROW_CHUNKS, col = (id % ROW_CHUNKS) / PIX_CHUNKS, k = id % PIX_CHUNKS;
      const int y = y0 + row, x = x0 + col;
      if (y < H && x < W) {
        const int t = row * CF_TW + col;
        const uint4 v = *reinterpret_cast<const uint4*>(s_out + t * PIX + 16 * (k ^ ((t >> 2) & 7)));
        *reinterpret_cast<uint4*>(out + ((static_cast<size_t>(n) * H + y) * W + x) * PIX + 16 * k) = v;
      }
    }
  }
}

}  // namespace opb
