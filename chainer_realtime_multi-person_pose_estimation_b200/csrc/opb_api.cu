// opb_api.cu -- C ABI of libopb.so (see include/opb.h).  Host-side orchestration of the
// sm_90a kernels: weight repacking, activation buffers, TMA tensor maps, the 92-conv chain of
// models/CocoPoseNet.py:132-262 as ~60 launches, and the post-process of
// pose_detector.py:501-517.  No CPU compute fallback exists in this file.
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <dlfcn.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <memory>
#include <string>
#include <queue>
#include <vector>

#include "../../include/opb.h"
#include "cascade.cuh"
#include "conv_first.cuh"
#include "ingest.cuh"
#include "overlay.cuh"
#include "keypoints.cuh"
#include "conv_wgmma.cuh"
#include "paf.cuh"
#include "peaks.cuh"
#include "peaks_sep.cuh"
#include "pool.cuh"
#include "upsample.cuh"
#include "whole_body.cuh"

using namespace opb;

static_assert(sizeof(opb_person) == sizeof(PersonOut), "opb_person layout");
static_assert(sizeof(opb_person) == 240, "opb_person size");
static_assert(sizeof(opb_image_header) == sizeof(ImageHeader), "opb_image_header layout");
static_assert(sizeof(opb_crop) == 24, "opb_crop size");
static_assert(sizeof(opb_part) == 24, "opb_part size");
static_assert(sizeof(opb_wb_part) == 32, "opb_wb_part size");
static_assert(sizeof(opb_crop) == sizeof(WbCrop), "opb_crop layout");

namespace {

struct OpbNcclId { char internal[128]; };   // == ncclUniqueId (passed BY VALUE to ncclCommInitRank)

thread_local std::string g_create_error;

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

struct HostLayer {
  int cin = 0, cout = 0, ks = 0;
  std::vector<float> W, b;
};

struct PackedW {          // one "B" operand: [cout_pad][ks*ks][k_per_tap] fp16
  __half* w = nullptr;
  float* bias = nullptr;  // [cout_pad]
  int cout_pad = 0, k_per_tap = 0, cin_pad = 0, ks = 0;
  float acc_scale = 1.f;  // compensated precision: 2^-S (the fp16 weights are stored pre-scaled by 2^S)
};

struct Act {              // NHWC fp16 activation tensor, channels [hi C | lo C]
  __half* p = nullptr;
  int N = 0, H = 0, W = 0, C = 0, Ctot = 0;
  size_t bytes() const { return static_cast<size_t>(N) * H * W * Ctot * sizeof(__half); }
};

enum OpKind { OP_FIRST, OP_CONV, OP_POOL };

struct ConvRec {          // what one problem of a conv op was built from (read back by the test hooks only)
  Act in, out;
  int in_coff = 0, out_coff = 0, cout_valid = 0, relu = 0, pool = 0;
  float* out32 = nullptr;
  std::string wkey;
};

struct Op {
  OpKind kind;
  std::string tag;
  // OP_CONV
  int ks = 0, bn = 0;
  bool drain = false;
  CUtensorMap tmA[2], tmB[2];
  ConvParams P;
  int grid = 0;
  ConvRec rec[2];
  // OP_FIRST / OP_POOL
  const __half* in = nullptr;
  __half* out = nullptr;
  int N = 0, H = 0, W = 0, C = 0, cstride = 0, lo_off = 0;
};

struct Chain {            // everything cached for one (N, H, W)
  int N = 0, H = 0, W = 0;
  std::vector<Op> ops;
  std::vector<void*> allocs;
  float* paf_lo = nullptr;   // [N][38][h][w]
  float* heat_lo = nullptr;  // [N][19][h][w]  (keypoint nets: [N][kp_out][h][w])
  uint8_t* img_u8 = nullptr;
  float* img_f32 = nullptr;
  const uint8_t* img_u8_src = nullptr;   // where conv1_1 reads uint8 frames (img_u8, or the caller's device buffer)
};

struct PostWs {           // post-process workspace for (N, map_h, map_w)
  int N = 0, H = 0, W = 0;
  float* pafs = nullptr;      // [N][38][H][W]
  float* heat = nullptr;      // [N][19][H][W]
  PeakKey* keys = nullptr;    // [N][max_peaks]
  float* tile_max = nullptr;  // cell maxima [N*18][ceil(H/8)][ceil(W/8)]
  int* peak_counts = nullptr; // [N]
  PeakD* peaks = nullptr;     // [N][max_peaks]
  int* idx_list = nullptr;
  int* type_start = nullptr;  // [N][19]
  int* status = nullptr;      // [N]
  Candidate* cands = nullptr; // [N][19][max_cand]
  Candidate* cands_alt = nullptr;  // ping-pong partner of cands for limb_assign's per-round compaction
  int* cand_counts = nullptr; // [N][19]
  Connection* conns = nullptr;  // [N][19][conn_cap]
  int* conn_counts = nullptr;
  double* subsets_out = nullptr;
  ImageHeader* headers = nullptr;
  PersonOut* persons = nullptr;
  const float* last_paf_lo = nullptr;   // low-res maps the last opb_detect_batch upsampled (network or injected)
  const float* last_heat_lo = nullptr;
  int last_h8 = 0, last_w8 = 0;         // their size
  float* sep_wy = nullptr;              // smooth_nms_sep_kernel: per-row / per-column operator records ([H][8], [W][8] floats)
  float* sep_wx = nullptr;
  int sep_h = 0, sep_w = 0;             // low-resolution size the records were built for (0: none); -1: not representable
  float* lo_stage = nullptr;            // opb_postprocess_batch: device copy of host low-res maps [N][57][h8][w8]
  size_t lo_cap = 0;                    // floats
  double last_img_len = 0;
  std::vector<void*> allocs;
};

struct KpWs {             // face / hand post-process workspace (grown on demand)
  size_t cap = 0;             // floats per buffer
  int records = 0;            // capacity of res / h_res
  int n_crops = 0;            // capacity of crops
  float* up = nullptr;        // upsampled maps, ragged: crop i's [planes][h_i][w_i] at KpCrop::off
  float* tmp = nullptr;       // after the axis-0 pass
  ChannelMax* res = nullptr;  // [crops][planes]
  ChannelMax* h_res = nullptr;  // pinned
  KpCrop* crops = nullptr;    // crop table of the current call
};

}  // namespace

struct CascadeState;

struct opb_ctx {
  int device = 0;
  int num_sms = 132;
  cudaStream_t stream = nullptr;
  cudaStream_t own_stream = nullptr;
  opb_params prm;
  PafConsts pc;
  GaussTaps taps;
  std::string err;
  int64_t launches = 0;
  EncodeTiledFn encode = nullptr;
  int precision = -1;
  int kp_out = 0;            // 0: CocoPoseNet; 71 / 22: FaceNet / HandNet (channels of the final 1x1, incl. background)
  float u8_denom = 255.f;    // uint8 normalisation: /255 (pose_detector.py:429) or /256 (face_detector.py:32)
  KpWs* kp_ws = nullptr;
  CascadeState* cascade = nullptr;   // opb_cascade_load
  std::map<std::string, HostLayer> host_layers;
  std::map<std::string, PackedW> packed;
  float* w_first = nullptr;  // conv1_1 [27][64] fp32
  float* b_first = nullptr;
  std::vector<void*> weight_allocs;
  std::map<long long, Chain*> chains;
  Chain* last_chain = nullptr;
  std::map<long long, PostWs*> posts;
  PostWs* last_post = nullptr;
  uint8_t* ingest_buf = nullptr;   // staging for the original frame(s) of opb_detect_image
  float* precise_mid = nullptr;    // x8 cubic intermediate of the precise path
  uint8_t* ov_buf = nullptr;       // overlay scratch: [frame in | frame out | priority plane | int poses | flag]
  size_t ov_bytes = 0;
  uint8_t* wb_buf = nullptr;       // opb_whole_body_frame: box-kernel outputs (whole_body.cuh) ...
  uint8_t* wb_host = nullptr;      // ... and their pinned host copy, preceded by the record block
  size_t wb_bytes = 0, wb_host_bytes = 0;
  size_t precise_mid_cap = 0;
  size_t ingest_bytes = 0;
  // streaming mode (opb_stream_submit / opb_stream_collect): two slots, pinned staging, a copy stream
  struct StreamSlot {
    uint8_t* d_frames = nullptr; size_t d_bytes = 0;     // device copy of the submitted frames (original size)
    uint8_t* h_frames = nullptr; size_t h_bytes = 0;     // pinned staging for pageable caller buffers
    uint8_t* h_result = nullptr; size_t r_bytes = 0;     // pinned [headers | persons] of the slot
    cudaEvent_t h2d_done = nullptr, done = nullptr;
    int n = 0; bool busy = false;
    const void* post = nullptr;                          // PostWs of the submitted batch (record block of opb_allgather_results)
    // CUDA-graph replay of the slot's pipeline: the launch sequence of one (shape, buffers) combination is captured
    // the second time it is submitted and replayed afterwards
    struct Key {
      int n, oh, ow, ih, iw, mh, mw; double img_len; const void *ip, *ih_, *frames, *result, *chain, *post;
      uint64_t epoch;
      bool operator==(const Key& o) const {
        return n == o.n && oh == o.oh && ow == o.ow && ih == o.ih && iw == o.iw && mh == o.mh && mw == o.mw &&
               img_len == o.img_len && ip == o.ip && ih_ == o.ih_ && frames == o.frames && result == o.result &&
               chain == o.chain && post == o.post && epoch == o.epoch;
      }
    } key{};
    int key_seen = 0;               // consecutive submits with `key`
    cudaGraphExec_t gexec = nullptr;
    int64_t graph_launches = 0;
  } slots[2];
  cudaStream_t copy_stream = nullptr;
  int cur_slot = 0;                // streaming slot whose chain / workspace get_chain / get_post hand out
  cudaStream_t stream_b = nullptr; // compute stream of streaming slot 1 (slot 0 uses `stream`)
  uint64_t cache_epoch = 0;        // bumped whenever cached chains / workspaces / weights are freed (invalidates graphs)
  int two_streams = 1;             // OPB_TWO_STREAMS=0: both streaming slots share `stream` and one set of buffers
  int use_graphs = 1;              // OPB_GRAPH=0: streaming mode launches kernel by kernel
  // Post-process variants (bit-exact against the oracle in every combination):
  int fused_peaks = 3;             // OPB_FUSED_PEAKS=1: the peak kernel interpolates its tiles from the low-res heat maps;
                                   // =3: candidates from the separable (bilinear o Gaussian) operator on the low-res maps (peaks_sep.cuh);
                                   // =2: materialised maps, but the tile-skip bound comes from the low-res maps (no cell_max pass)
  int paf_lowres = 1;              // OPB_PAF_LOWRES=1: PAF line integrals sample the low-res PAFs on demand
  int peaks_v2 = 0;                // OPB_PEAKS_V2=1 (with OPB_FUSED_PEAKS=2): smoothing passes spread over all 256 threads
  int conn_cap = kAssignMaxType;
  bool profile = false;                       // OPB_PROFILE=1: cudaEvent after every launch of a batch
  std::vector<std::pair<std::string, cudaEvent_t>> marks;
};

namespace {

#define OPB_CUDA(ctx, expr)                                                                       \
  do {                                                                                            \
    cudaError_t e__ = (expr);                                                                     \
    if (e__ != cudaSuccess) {                                                                     \
      (ctx)->err = std::string(#expr) + ": " + cudaGetErrorString(e__) + " (" __FILE__ ":" +      \
                   std::to_string(__LINE__) + ")";                                                \
      return OPB_ERR_CUDA;                                                                        \
    }                                                                                             \
  } while (0)

#define OPB_FAIL(ctx, code, msg) \
  do {                           \
    (ctx)->err = (msg);          \
    return (code);               \
  } while (0)

int round_up(int v, int m) { return (v + m - 1) / m * m; }

void prof_mark(opb_ctx* ctx, const std::string& name) {
  if (!ctx->profile) return;
  cudaEvent_t e;
  cudaEventCreate(&e);
  cudaEventRecord(e, ctx->stream);
  ctx->marks.emplace_back(name, e);
}

void prof_report(opb_ctx* ctx) {
  if (!ctx->profile || ctx->marks.size() < 2) return;
  cudaStreamSynchronize(ctx->stream);
  std::map<std::string, std::pair<int, float>> agg;
  std::vector<std::string> order;
  float total = 0.f;
  for (size_t i = 1; i < ctx->marks.size(); ++i) {
    float ms = 0.f;
    cudaEventElapsedTime(&ms, ctx->marks[i - 1].second, ctx->marks[i].second);
    auto& a = agg[ctx->marks[i].first];
    if (a.first == 0) order.push_back(ctx->marks[i].first);
    a.first++;
    a.second += ms;
    total += ms;
  }
  fprintf(stderr, "[opb profile] total %.3f ms\n", total);
  for (auto& k : order) fprintf(stderr, "[opb profile] %-16s n=%3d %9.3f ms %5.1f%%\n", k.c_str(), agg[k].first, agg[k].second, 100.f * agg[k].second / total);
  for (auto& m : ctx->marks) cudaEventDestroy(m.second);
  ctx->marks.clear();
}

template <typename T>
int dev_alloc(opb_ctx* ctx, T** p, size_t count, std::vector<void*>& owner, bool zero = true) {
  void* q = nullptr;
  OPB_CUDA(ctx, cudaMalloc(&q, std::max<size_t>(count * sizeof(T), 256)));
  if (zero) OPB_CUDA(ctx, cudaMemsetAsync(q, 0, std::max<size_t>(count * sizeof(T), 256), ctx->stream));
  owner.push_back(q);
  *p = static_cast<T*>(q);
  return OPB_OK;
}

void free_all(std::vector<void*>& v) {
  for (void* p : v) cudaFree(p);
  v.clear();
}

// ------------------------------------------------------------------ tensor maps
int make_act_map(opb_ctx* ctx, CUtensorMap* tm, const Act& a, int coff, int ks, int box_w = 8) {
  cuuint64_t dims[4] = {static_cast<cuuint64_t>(a.Ctot - coff), static_cast<cuuint64_t>(a.W),
                        static_cast<cuuint64_t>(a.H), static_cast<cuuint64_t>(a.N)};
  cuuint64_t strides[3] = {static_cast<cuuint64_t>(a.Ctot) * 2, static_cast<cuuint64_t>(a.W) * a.Ctot * 2,
                           static_cast<cuuint64_t>(a.H) * a.W * a.Ctot * 2};
  cuuint32_t box[4] = {64, static_cast<cuuint32_t>(box_w), static_cast<cuuint32_t>(16 + ks - 1), 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = ctx->encode(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, a.p + coff, dims, strides, box, estr,
                           CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                           CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) OPB_FAIL(ctx, OPB_ERR_CUDA, "cuTensorMapEncodeTiled(activation) failed: " + std::to_string(r));
  return OPB_OK;
}

int make_w_map(opb_ctx* ctx, CUtensorMap* tm, const PackedW& w, int bn) {
  const cuuint64_t ktot = static_cast<cuuint64_t>(w.ks) * w.ks * w.k_per_tap;
  cuuint64_t dims[2] = {ktot, static_cast<cuuint64_t>(w.cout_pad)};
  cuuint64_t strides[1] = {ktot * 2};
  cuuint32_t box[2] = {64, static_cast<cuuint32_t>(bn)};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = ctx->encode(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, w.w, dims, strides, box, estr,
                           CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                           CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) OPB_FAIL(ctx, OPB_ERR_CUDA, "cuTensorMapEncodeTiled(weights) failed: " + std::to_string(r));
  return OPB_OK;
}

// ------------------------------------------------------------------ conv launch
template <int KS, int BN, bool DRAIN>
int launch_conv_t(opb_ctx* ctx, const Op& op) {
  using Cfg = ConvCfg<KS, BN>;
  auto kern = conv_wgmma_kernel<KS, BN, DRAIN>;
  static bool attr_set[64] = {};
  if (!attr_set[ctx->device & 63]) {
    OPB_CUDA(ctx, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
    attr_set[ctx->device & 63] = true;
  }
  kern<<<op.grid, kConvThreads, Cfg::SMEM_BYTES, ctx->stream>>>(op.tmA[0], op.tmB[0], op.tmA[1], op.tmB[1], op.P);
  ctx->launches++;
  OPB_CUDA(ctx, cudaGetLastError());
  return OPB_OK;
}

template <int KS>
int launch_conv_ks(opb_ctx* ctx, const Op& op) {
  if (op.P.comp && !op.drain) OPB_FAIL(ctx, OPB_ERR_UNSUPPORTED, "compensated precision needs two-level accumulation");
  switch (op.bn * 2 + (op.drain ? 1 : 0)) {
    case 128 * 2: return launch_conv_t<KS, 128, false>(ctx, op);
    case 128 * 2 + 1: return launch_conv_t<KS, 128, true>(ctx, op);
    case 64 * 2: return launch_conv_t<KS, 64, false>(ctx, op);
    case 64 * 2 + 1: return launch_conv_t<KS, 64, true>(ctx, op);
    case 48 * 2: return launch_conv_t<KS, 48, false>(ctx, op);
    case 48 * 2 + 1: return launch_conv_t<KS, 48, true>(ctx, op);
    default: OPB_FAIL(ctx, OPB_ERR_UNSUPPORTED, "no conv kernel variant for ks " + std::to_string(KS) + " bn " + std::to_string(op.bn));
  }
}

int launch_conv(opb_ctx* ctx, const Op& op) {
  if (op.ks == 7) return launch_conv_ks<7>(ctx, op);
  if (op.ks == 3) return launch_conv_ks<3>(ctx, op);
  if (op.ks == 1) return launch_conv_ks<1>(ctx, op);
  OPB_FAIL(ctx, OPB_ERR_UNSUPPORTED, "no conv kernel variant for ks " + std::to_string(op.ks));
}

template <int MODE>
int launch_first_t(opb_ctx* ctx, const Chain* ch, const Op& op) {
  auto kern = conv_first_kernel<MODE>;
  constexpr int smem = conv_first_smem_bytes(MODE);
  static bool attr_set[64] = {};
  if (!attr_set[ctx->device & 63]) {
    OPB_CUDA(ctx, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    attr_set[ctx->device & 63] = true;
  }
  // persistent: two resident blocks per SM (register bound), each walking the tiles with a grid stride
  const int tiles = op.N * ((op.H + CF_TH - 1) / CF_TH) * ((op.W + CF_TW - 1) / CF_TW);
  const int grid = std::min(tiles, ctx->num_sms * 2);
  kern<<<grid, CF_THREADS, smem, ctx->stream>>>(op.C == 1 ? (ch->img_u8_src ? ch->img_u8_src : ch->img_u8) : nullptr,
                                                op.C == 1 ? nullptr : ch->img_f32, ctx->w_first, ctx->b_first,
                                                reinterpret_cast<uint8_t*>(op.out), op.N, op.H, op.W, ctx->u8_denom);
  ctx->launches++;
  OPB_CUDA(ctx, cudaGetLastError());
  return OPB_OK;
}

int launch_op(opb_ctx* ctx, const Chain* ch, const Op& op) {
  if (op.kind == OP_CONV) return launch_conv(ctx, op);
  if (op.kind == OP_POOL) {
    const size_t total = static_cast<size_t>(op.N) * (op.H / 2) * (op.W / 2) * (op.C / 8);
    const int grid = static_cast<int>(std::min<size_t>((total + 255) / 256, static_cast<size_t>(ctx->num_sms) * 16));
    maxpool2x2_kernel<<<grid, 256, 0, ctx->stream>>>(op.in, op.out, op.N, op.H, op.W, op.C, op.cstride, op.lo_off);
    ctx->launches++;
    OPB_CUDA(ctx, cudaGetLastError());
    return OPB_OK;
  }
  // OP_FIRST
  const int mode = op.lo_off == 0 ? CF_FAST : ctx->precision == OPB_PRECISION_COMP ? CF_COMP : CF_PARITY;
  if (op.cstride * 2 != conv_first_pix_bytes(mode) || (mode != CF_FAST && op.lo_off != 64))
    OPB_FAIL(ctx, OPB_ERR_UNSUPPORTED, "conv1_1 output must be a dense 64-channel activation tensor");
  switch (mode) {
    case CF_FAST: return launch_first_t<CF_FAST>(ctx, ch, op);
    case CF_PARITY: return launch_first_t<CF_PARITY>(ctx, ch, op);
    default: return launch_first_t<CF_COMP>(ctx, ch, op);
  }
}

// ------------------------------------------------------------------ weight packing
// rows: list of (layer, n_rows_pad); cin_map[d] = reference input channel of device channel d
// (or -1 = zero).  Output [sum rows_pad][ks*ks][cin_pad * (split ? 2 : 1)].
// Compensated precision (prec == OPB_PRECISION_COMP): per tap [W_hi * 2^S : cin_pad halves][per 64-channel chunk:
// e4m3(W * 2^kW) 64 B | e4m3(W_lo * 2^S) 64 B], S = kW + 11, 2^kW * max|W| in (8, 16] (one power of two per packed matrix).
int pack_weights(opb_ctx* ctx, const std::string& key, const std::vector<std::pair<std::string, int>>& rows,
                 const std::vector<int>& cin_map, int ks, int prec) {
  const bool split = prec == OPB_PRECISION_PARITY, comp = prec == OPB_PRECISION_COMP;
  const int cin_pad = static_cast<int>(cin_map.size());
  const int kpt = cin_pad * ((split || comp) ? 2 : 1);
  int cout_pad = 0;
  for (auto& r : rows) cout_pad += r.second;
  const size_t ktot = static_cast<size_t>(ks) * ks * kpt;
  std::vector<__half> hw(static_cast<size_t>(cout_pad) * ktot, __float2half(0.f));
  std::vector<float> hb(cout_pad, 0.f);
  int kW = 0, S = 0;
  if (comp) {
    float mx = 0.f;
    for (auto& r : rows) {
      auto it = ctx->host_layers.find(r.first);
      if (it == ctx->host_layers.end()) OPB_FAIL(ctx, OPB_ERR_STATE, "weights for layer " + r.first + " were not loaded");
      for (float v : it->second.W) mx = std::max(mx, std::fabs(v));
    }
    if (mx > 0.f && std::isfinite(mx)) {
      kW = static_cast<int>(std::floor(std::log2(16.0 / static_cast<double>(mx))));
      kW = std::max(-100, std::min(100, kW));
      S = kW + 11;
    }
  }
  int row0 = 0;
  for (auto& r : rows) {
    auto it = ctx->host_layers.find(r.first);
    if (it == ctx->host_layers.end()) OPB_FAIL(ctx, OPB_ERR_STATE, "weights for layer " + r.first + " were not loaded");
    const HostLayer& L = it->second;
    if (L.ks != ks) OPB_FAIL(ctx, OPB_ERR_ARG, "ksize mismatch for " + r.first);
    for (int o = 0; o < L.cout; ++o) {
      hb[row0 + o] = L.b[o];
      for (int t = 0; t < ks * ks; ++t) {
        __half* dst = hw.data() + (static_cast<size_t>(row0 + o) * ks * ks + t) * kpt;
        for (int d = 0; d < cin_pad; ++d) {
          const int c = cin_map[d];
          if (c < 0 || c >= L.cin) continue;
          const float v = L.W[(static_cast<size_t>(o) * L.cin + c) * ks * ks + t];
          if (comp) {
            const __half hs = __float2half_rn(std::ldexp(v, S));                     // W_hi * 2^S (exact scaling)
            dst[d] = hs;
            const double lo_s = std::ldexp(static_cast<double>(v), S) - static_cast<double>(__half2float(hs));   // W_lo * 2^S
            uint8_t* cb = reinterpret_cast<uint8_t*>(dst + cin_pad) + comp_byte_off(d);
            cb[0] = f32_to_e4m3(std::ldexp(v, kW));
            cb[64] = f32_to_e4m3(static_cast<float>(lo_s));
            continue;
          }
          const __half hi = __float2half_rn(v);
          dst[d] = hi;
          if (split) dst[cin_pad + d] = __float2half_rn(v - __half2float(hi));
        }
      }
    }
    row0 += r.second;
  }
  PackedW pw;
  pw.cout_pad = cout_pad;
  pw.k_per_tap = kpt;
  pw.cin_pad = cin_pad;
  pw.ks = ks;
  pw.acc_scale = comp ? std::ldexp(1.f, -S) : 1.f;
  int rc = dev_alloc(ctx, &pw.w, hw.size(), ctx->weight_allocs, false);
  if (rc) return rc;
  rc = dev_alloc(ctx, &pw.bias, hb.size() + 64, ctx->weight_allocs, true);
  if (rc) return rc;
  OPB_CUDA(ctx, cudaMemcpyAsync(pw.w, hw.data(), hw.size() * sizeof(__half), cudaMemcpyHostToDevice, ctx->stream));
  OPB_CUDA(ctx, cudaMemcpyAsync(pw.bias, hb.data(), hb.size() * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
  OPB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));  // host vectors die here
  ctx->packed[key] = pw;
  return OPB_OK;
}

std::vector<int> identity_map(int cin, int cin_pad) {
  std::vector<int> m(cin_pad, -1);
  for (int i = 0; i < cin; ++i) m[i] = i;
  return m;
}

// ------------------------------------------------------------------ chain construction
struct ConvSpec {
  const Act* in[2];
  int in_coff[2];
  std::string wkey[2];
  const Act* out[2];
  int out_coff[2];
  int cout_valid[2];
  float* out32[2];
  int n_problems;
  int relu;
  int pool;
};

int add_conv(opb_ctx* ctx, Chain* ch, const std::string& tag, const ConvSpec& s) {
  Op op;
  op.kind = OP_CONV;
  op.tag = tag;
  const PackedW& w0 = ctx->packed.at(s.wkey[0]);
  const bool split = ctx->precision == OPB_PRECISION_PARITY;
  const bool comp = ctx->precision == OPB_PRECISION_COMP;
  op.ks = w0.ks;
  const int per_problem_cout_pad = w0.cout_pad;
  // two-level accumulation in the precisions that claim the 1e-3 map tolerance: the tensor core's truncating accumulate
  // over long MMA chains (and an 8-bit wgmma's ~14-bit view of the accumulator it adds to) would otherwise dominate
  // their remaining map error
  op.drain = split || comp;
  // channel block: a consumer warpgroup holds 64 x BN fp32 accumulators in registers (two sets when draining)
  op.bn = std::min(per_problem_cout_pad, 128);
  const Act& a0 = *s.in[0];
  if (a0.H < 16 + op.ks - 1 || a0.W < 8)
    OPB_FAIL(ctx, OPB_ERR_UNSUPPORTED, "feature map smaller than one TMA box (min 22 x 8); image too small");
  {  // Small batches (one camera frame): a launch that fills less than half a wave halves its channel block (down to 64)
     // while it still fits one wave, trading operand reuse for parallelism.  OPB_SMALL_BATCH=0 disables.
    const char* e = getenv("OPB_SMALL_BATCH");
    const long long m_tiles = static_cast<long long>(a0.N) * ((a0.H + 15) / 16) * ((a0.W + 7) / 8);
    const long long tiles = s.n_problems * (per_problem_cout_pad / op.bn) * m_tiles;
    if (!(e && atoi(e) == 0) && op.bn == 128 && !s.pool && tiles * 4 <= ctx->num_sms) op.bn = 64;
  }
  std::memset(&op.P, 0, sizeof(op.P));
  ConvParams& P = op.P;
  P.N = a0.N; P.H = a0.H; P.W = a0.W;
  P.tiles_x = (a0.W + 7) / 8;
  P.tiles_y = (a0.H + 15) / 16;
  P.n_blocks = per_problem_cout_pad / op.bn;
  P.n_problems = s.n_problems;
  P.b_tap_stride = w0.k_per_tap;
  const int chunks = w0.cin_pad / 64;
  int np = 0;
  for (int i = 0; i < chunks; ++i) {
    P.a_off[np] = i * 64; P.b_off[np] = i * 64; ++np;
    if (split) {
      P.a_off[np] = a0.C + i * 64; P.b_off[np] = i * 64; ++np;             // lo * Whi
      P.a_off[np] = i * 64; P.b_off[np] = w0.cin_pad + i * 64; ++np;        // hi * Wlo
    }
    if (comp) {   // odd pairs: the 128-byte 8-bit-float correction row of chunk i (addressed as 64 halves)
      P.a_off[np] = a0.C + i * 64; P.b_off[np] = w0.cin_pad + i * 64; ++np;
    }
  }
  P.comp = comp ? 1 : 0;
  if (np > kMaxPairs) OPB_FAIL(ctx, OPB_ERR_UNSUPPORTED, "too many K chunk pairs");
  P.n_pairs = np;
  for (int p = 0; p < s.n_problems; ++p) {
    const PackedW& w = ctx->packed.at(s.wkey[p]);
    if (w.ks != op.ks || w.cout_pad != per_problem_cout_pad || w.k_per_tap != w0.k_per_tap)
      OPB_FAIL(ctx, OPB_ERR_ARG, "grouped problems must share a shape");
    if ((split || comp) && s.in[p]->C != a0.C) OPB_FAIL(ctx, OPB_ERR_ARG, "grouped problems must share the lo-plane offset");
    int rc = make_act_map(ctx, &op.tmA[p], *s.in[p], s.in_coff[p], op.ks);
    if (rc) return rc;
    rc = make_w_map(ctx, &op.tmB[p], w, op.bn);
    if (rc) return rc;
    ConvProblem& pr = P.prob[p];
    pr.out = s.out[p] ? s.out[p]->p : nullptr;
    pr.out32 = s.out32[p];
    pr.bias = w.bias;
    pr.out_cstride = s.out[p] ? s.out[p]->Ctot : 0;
    pr.out_coff = s.out_coff[p];
    pr.out_lo_off = ((split || comp) && s.out[p]) ? s.out[p]->C : 0;
    pr.cout_valid = s.cout_valid[p];
    pr.relu = s.relu;
    pr.pool = s.pool;
    pr.acc_scale = w.acc_scale;
    ConvRec& rec = op.rec[p];
    rec.in = *s.in[p];
    if (s.out[p]) rec.out = *s.out[p];
    rec.in_coff = s.in_coff[p];
    rec.out_coff = s.out_coff[p];
    rec.cout_valid = s.cout_valid[p];
    rec.relu = s.relu;
    rec.pool = s.pool;
    rec.out32 = s.out32[p];
    rec.wkey = s.wkey[p];
  }
  if (s.n_problems == 1) { op.tmA[1] = op.tmA[0]; op.tmB[1] = op.tmB[0]; P.prob[1] = P.prob[0]; }
  const int total_tiles = P.n_problems * P.n_blocks * P.N * P.tiles_y * P.tiles_x;
  op.grid = std::min(total_tiles, ctx->num_sms);
  ch->ops.push_back(op);
  return OPB_OK;
}

int alloc_act(opb_ctx* ctx, Chain* ch, Act* a, int N, int H, int W, int C) {
  a->N = N; a->H = H; a->W = W; a->C = C;
  a->Ctot = C * (ctx->precision == OPB_PRECISION_FAST ? 1 : 2);   // parity: [hi | lo] fp16; compensated: [hi fp16 | 2C correction bytes]
  return dev_alloc(ctx, &a->p, a->bytes() / sizeof(__half), ch->allocs, true);
}

int build_chain_keypoint(opb_ctx* ctx, Chain* ch, int N, int H, int W);

int build_chain(opb_ctx* ctx, Chain* ch, int N, int H, int W) {
  if (ctx->kp_out) return build_chain_keypoint(ctx, ch, N, H, W);
  ch->N = N; ch->H = H; ch->W = W;
  const bool split = ctx->precision != OPB_PRECISION_FAST;   // two planes per activation tensor (parity: lo; compensated: correction bytes)
  const int h8 = H / 8, w8 = W / 8;
  int rc;
#define RC(x) do { rc = (x); if (rc) return rc; } while (0)
  RC(dev_alloc(ctx, &ch->img_u8, static_cast<size_t>(N) * H * W * 3, ch->allocs, false));
  RC(dev_alloc(ctx, &ch->img_f32, static_cast<size_t>(N) * H * W * 3, ch->allocs, false));
  RC(dev_alloc(ctx, &ch->paf_lo, static_cast<size_t>(N) * 38 * h8 * w8, ch->allocs, true));
  RC(dev_alloc(ctx, &ch->heat_lo, static_cast<size_t>(N) * 19 * h8 * w8, ch->allocs, true));
  // activation buffers (kept alive for the lifetime of the chain; 180 GB of HBM make reuse
  // games unnecessary at batch 32: ~4.5 GB fast, ~9 GB parity)
  Act B0, B1, P1, B2, B3, P2, B4, B5, P3, B6, B7, B8, CAT, SA, SB, S512;   // ops keep raw pointers only
  RC(alloc_act(ctx, ch, &B0, N, H, W, 64));
  RC(alloc_act(ctx, ch, &B1, N, H, W, 64));
  RC(alloc_act(ctx, ch, &P1, N, H / 2, W / 2, 64));
  RC(alloc_act(ctx, ch, &B2, N, H / 2, W / 2, 128));
  RC(alloc_act(ctx, ch, &B3, N, H / 2, W / 2, 128));
  RC(alloc_act(ctx, ch, &P2, N, H / 4, W / 4, 128));
  RC(alloc_act(ctx, ch, &B4, N, H / 4, W / 4, 256));
  RC(alloc_act(ctx, ch, &B5, N, H / 4, W / 4, 256));
  RC(alloc_act(ctx, ch, &P3, N, h8, w8, 256));
  RC(alloc_act(ctx, ch, &B6, N, h8, w8, 512));
  RC(alloc_act(ctx, ch, &B7, N, h8, w8, 512));
  RC(alloc_act(ctx, ch, &B8, N, h8, w8, 256));
  RC(alloc_act(ctx, ch, &CAT, N, h8, w8, 192));
  RC(alloc_act(ctx, ch, &SA, N, h8, w8, 256));
  RC(alloc_act(ctx, ch, &SB, N, h8, w8, 256));
  RC(alloc_act(ctx, ch, &S512, N, h8, w8, 1024));

  auto first = [&]() {
    Op op; op.kind = OP_FIRST; op.tag = "conv1_1"; op.out = B0.p; op.N = N; op.H = H; op.W = W; op.C = 1;
    op.cstride = B0.Ctot; op.lo_off = split ? B0.C : 0;
    ch->ops.push_back(op);
  };
  auto pool = [&](const char* tag, const Act& in, const Act& out) {
    Op op; op.kind = OP_POOL; op.tag = tag; op.in = in.p; op.out = out.p; op.N = N; op.H = in.H; op.W = in.W;
    op.C = in.Ctot /* hi and lo planes are pooled as one channel range in fast mode */; op.cstride = in.Ctot;
    op.lo_off = split ? in.C : 0;
    if (split) op.C = in.C;
    ch->ops.push_back(op);
  };
  auto conv1 = [&](const std::string& layer, const Act& in, const Act& out, int out_coff, int cout,
                   int fuse_pool = 0) -> int {
    ConvSpec s{};
    s.in[0] = &in; s.in_coff[0] = 0; s.wkey[0] = layer; s.out[0] = &out; s.out_coff[0] = out_coff;
    s.cout_valid[0] = cout; s.out32[0] = nullptr; s.n_problems = 1; s.relu = 1; s.pool = fuse_pool;
    return add_conv(ctx, ch, layer, s);
  };
  const bool fuse = ctx->precision == OPB_PRECISION_COMP ||   // (the stand-alone pool kernel has no compensated variant)
                    !(getenv("OPB_NO_POOL_FUSION") && atoi(getenv("OPB_NO_POOL_FUSION")));   // debug knob
  auto conv2 = [&](const std::string& tag, const std::string& l1, const std::string& l2, const Act& in, int ic1,
                   int ic2, const Act& out, int oc1, int oc2, int cv1, int cv2, int relu, float* o32a,
                   float* o32b) -> int {
    ConvSpec s{};
    s.in[0] = &in; s.in[1] = &in; s.in_coff[0] = ic1; s.in_coff[1] = ic2; s.wkey[0] = l1; s.wkey[1] = l2;
    s.out[0] = &out; s.out[1] = &out; s.out_coff[0] = oc1; s.out_coff[1] = oc2; s.cout_valid[0] = cv1;
    s.cout_valid[1] = cv2; s.out32[0] = o32a; s.out32[1] = o32b; s.n_problems = 2; s.relu = relu;
    return add_conv(ctx, ch, tag, s);
  };

  first();
  // F.max_pooling_2d(2,2) (models/CocoPoseNet.py:138,141,146) is fused into the producing conv's epilogue
  if (fuse) { RC(conv1("conv1_2", B0, P1, 0, 64, 1)); } else { RC(conv1("conv1_2", B0, B1, 0, 64)); pool("pool1", B1, P1); }
  RC(conv1("conv2_1", P1, B2, 0, 128));
  if (fuse) { RC(conv1("conv2_2", B2, P2, 0, 128, 1)); } else { RC(conv1("conv2_2", B2, B3, 0, 128)); pool("pool2", B3, P2); }
  RC(conv1("conv3_1", P2, B4, 0, 256));
  RC(conv1("conv3_2", B4, B5, 0, 256));
  RC(conv1("conv3_3", B5, B4, 0, 256));
  if (fuse) { RC(conv1("conv3_4", B4, P3, 0, 256, 1)); } else { RC(conv1("conv3_4", B4, B5, 0, 256)); pool("pool3", B5, P3); }
  RC(conv1("conv4_1", P3, B6, 0, 512));
  RC(conv1("conv4_2", B6, B7, 0, 512));
  RC(conv1("conv4_3_CPM", B7, B8, 0, 256));
  RC(conv1("conv4_4_CPM", B8, CAT, 0, 128));
  // stage 1 (models/CocoPoseNet.py:154-165): both branches as 2-problem grouped launches
  RC(conv2("conv5_1", "conv5_1_CPM_L1", "conv5_1_CPM_L2", CAT, 0, 0, SA, 0, 128, 128, 128, 1, nullptr, nullptr));
  RC(conv2("conv5_2", "conv5_2_CPM_L1", "conv5_2_CPM_L2", SA, 0, 128, SB, 0, 128, 128, 128, 1, nullptr, nullptr));
  RC(conv2("conv5_3", "conv5_3_CPM_L1", "conv5_3_CPM_L2", SB, 0, 128, SA, 0, 128, 128, 128, 1, nullptr, nullptr));
  RC(conv2("conv5_4", "conv5_4_CPM_L1", "conv5_4_CPM_L2", SA, 0, 128, S512, 0, 512, 512, 512, 1, nullptr, nullptr));
  RC(conv2("conv5_5", "conv5_5_CPM_L1", "conv5_5_CPM_L2", S512, 0, 512, CAT, 128, 166, 38, 19, 0, nullptr, nullptr));
  for (int st = 2; st <= 6; ++st) {
    const std::string S = "_stage" + std::to_string(st);
    {  // Mconv1: both branches read the same concat tensor -> one N=256 GEMM (:168-169,176)
      ConvSpec s{};
      s.in[0] = &CAT; s.in_coff[0] = 0; s.wkey[0] = "Mconv1" + S + "_fused"; s.out[0] = &SA; s.out_coff[0] = 0;
      s.cout_valid[0] = 256; s.n_problems = 1; s.relu = 1;
      RC(add_conv(ctx, ch, "Mconv1", s));
    }
    RC(conv2("Mconv7x7", "Mconv2" + S + "_L1", "Mconv2" + S + "_L2", SA, 0, 128, SB, 0, 128, 128, 128, 1, nullptr, nullptr));
    RC(conv2("Mconv7x7", "Mconv3" + S + "_L1", "Mconv3" + S + "_L2", SB, 0, 128, SA, 0, 128, 128, 128, 1, nullptr, nullptr));
    RC(conv2("Mconv7x7", "Mconv4" + S + "_L1", "Mconv4" + S + "_L2", SA, 0, 128, SB, 0, 128, 128, 128, 1, nullptr, nullptr));
    RC(conv2("Mconv7x7", "Mconv5" + S + "_L1", "Mconv5" + S + "_L2", SB, 0, 128, SA, 0, 128, 128, 128, 1, nullptr, nullptr));
    RC(conv2("Mconv6", "Mconv6" + S + "_L1", "Mconv6" + S + "_L2", SA, 0, 128, SB, 0, 128, 128, 128, 1, nullptr, nullptr));
    RC(conv2("Mconv7", "Mconv7" + S + "_L1", "Mconv7" + S + "_L2", SB, 0, 128, CAT, 128, 166, 38, 19, 0,
             st == 6 ? ch->paf_lo : nullptr, st == 6 ? ch->heat_lo : nullptr));
  }
#undef RC
  return OPB_OK;
}

// FaceNet / HandNet (models/FaceNet.py:78-161, models/HandNet.py): one branch, VGG front to conv5_2, conv5_3_CPM -> 128
// features, stage 1 = two 1x1 convs, stages 2-6 on concat(previous maps, features).  Device concat layout:
// [features 0..127 | maps 128..128+kp_out-1 | 0 pad] (the Mconv1 weights are permuted to match).
int build_chain_keypoint(opb_ctx* ctx, Chain* ch, int N, int H, int W) {
  ch->N = N; ch->H = H; ch->W = W;
  const bool split = ctx->precision != OPB_PRECISION_FAST;
  const int h8 = H / 8, w8 = W / 8, KC = ctx->kp_out;
  int rc;
#define RC(x) do { rc = (x); if (rc) return rc; } while (0)
  RC(dev_alloc(ctx, &ch->img_u8, static_cast<size_t>(N) * H * W * 3, ch->allocs, false));
  RC(dev_alloc(ctx, &ch->img_f32, static_cast<size_t>(N) * H * W * 3, ch->allocs, false));
  RC(dev_alloc(ctx, &ch->paf_lo, 64, ch->allocs, true));
  RC(dev_alloc(ctx, &ch->heat_lo, static_cast<size_t>(N) * KC * h8 * w8, ch->allocs, true));
  Act B0, P1, B2, P2, B4, B5, P3, B6, B7, CAT, SA, SB, S512;
  RC(alloc_act(ctx, ch, &B0, N, H, W, 64));
  RC(alloc_act(ctx, ch, &P1, N, H / 2, W / 2, 64));
  RC(alloc_act(ctx, ch, &B2, N, H / 2, W / 2, 128));
  RC(alloc_act(ctx, ch, &P2, N, H / 4, W / 4, 128));
  RC(alloc_act(ctx, ch, &B4, N, H / 4, W / 4, 256));
  RC(alloc_act(ctx, ch, &B5, N, H / 4, W / 4, 256));
  RC(alloc_act(ctx, ch, &P3, N, h8, w8, 256));
  RC(alloc_act(ctx, ch, &B6, N, h8, w8, 512));
  RC(alloc_act(ctx, ch, &B7, N, h8, w8, 512));
  RC(alloc_act(ctx, ch, &CAT, N, h8, w8, round_up(128 + KC, 64)));
  RC(alloc_act(ctx, ch, &SA, N, h8, w8, 128));
  RC(alloc_act(ctx, ch, &SB, N, h8, w8, 128));
  RC(alloc_act(ctx, ch, &S512, N, h8, w8, 512));
  {
    Op op; op.kind = OP_FIRST; op.tag = "conv1_1"; op.out = B0.p; op.N = N; op.H = H; op.W = W; op.C = 1;
    op.cstride = B0.Ctot; op.lo_off = split ? B0.C : 0;
    ch->ops.push_back(op);
  }
  auto conv = [&](const std::string& layer, const Act& in, const Act& out, int out_coff, int cout, int relu = 1,
                  int fuse_pool = 0, float* o32 = nullptr) -> int {
    ConvSpec s{};
    s.in[0] = &in; s.in_coff[0] = 0; s.wkey[0] = layer; s.out[0] = &out; s.out_coff[0] = out_coff;
    s.cout_valid[0] = cout; s.out32[0] = o32; s.n_problems = 1; s.relu = relu; s.pool = fuse_pool;
    return add_conv(ctx, ch, layer.rfind("Mconv", 0) == 0 ? layer.substr(0, 6) : layer, s);
  };
  RC(conv("conv1_2", B0, P1, 0, 64, 1, 1));      // max-pools (models/FaceNet.py:83,86,91) fused into the producers
  RC(conv("conv2_1", P1, B2, 0, 128));
  RC(conv("conv2_2", B2, P2, 0, 128, 1, 1));
  RC(conv("conv3_1", P2, B4, 0, 256));
  RC(conv("conv3_2", B4, B5, 0, 256));
  RC(conv("conv3_3", B5, B4, 0, 256));
  RC(conv("conv3_4", B4, P3, 0, 256, 1, 1));
  RC(conv("conv4_1", P3, B6, 0, 512));
  RC(conv("conv4_2", B6, B7, 0, 512));
  RC(conv("conv4_3", B7, B6, 0, 512));
  RC(conv("conv4_4", B6, B7, 0, 512));
  RC(conv("conv5_1", B7, B6, 0, 512));
  RC(conv("conv5_2", B6, B7, 0, 512));
  RC(conv("conv5_3_CPM", B7, CAT, 0, 128));
  RC(conv("conv6_1_CPM", CAT, S512, 0, 512));
  RC(conv("conv6_2_CPM", S512, CAT, 128, KC, 0));
  for (int st = 2; st <= 6; ++st) {
    const std::string S = "_stage" + std::to_string(st);
    RC(conv("Mconv1" + S, CAT, SA, 0, 128));
    RC(conv("Mconv2" + S, SA, SB, 0, 128));
    RC(conv("Mconv3" + S, SB, SA, 0, 128));
    RC(conv("Mconv4" + S, SA, SB, 0, 128));
    RC(conv("Mconv5" + S, SB, SA, 0, 128));
    RC(conv("Mconv6" + S, SA, SB, 0, 128));
    RC(conv("Mconv7" + S, SB, CAT, 128, KC, 0, 0, st == 6 ? ch->heat_lo : nullptr));
  }
#undef RC
  return OPB_OK;
}

long long shape_key(int n, int h, int w) { return (static_cast<long long>(n) << 40) | (static_cast<long long>(h) << 20) | w; }
// streaming slot 1 owns its own activations / workspaces so that the two slots can run on two streams
long long slot_key(const opb_ctx* ctx, int n, int h, int w) { return shape_key(n, h, w) | (static_cast<long long>(ctx->cur_slot) << 62); }

int get_chain(opb_ctx* ctx, int n, int h, int w, Chain** out) {
  if (ctx->precision < 0) OPB_FAIL(ctx, OPB_ERR_STATE, "opb_finalize_weights has not been called");
  if (n <= 0 || h <= 0 || w <= 0 || (h % 8) || (w % 8)) OPB_FAIL(ctx, OPB_ERR_ARG, "H and W must be positive multiples of 8");
  const long long key = slot_key(ctx, n, h, w);
  auto it = ctx->chains.find(key);
  if (it != ctx->chains.end()) { *out = it->second; ctx->last_chain = it->second; return OPB_OK; }
  // keep at most a few cached shapes (the precise path cycles through 4)
  if (ctx->chains.size() >= 10) {
    cudaDeviceSynchronize();   // both streaming slots may still be running on their chains
    for (auto& kv : ctx->chains) { free_all(kv.second->allocs); delete kv.second; }
    ctx->chains.clear();
    ctx->cache_epoch++;
    ctx->last_chain = nullptr;
  }
  Chain* ch = new Chain();
  int rc = build_chain(ctx, ch, n, h, w);
  if (rc) { free_all(ch->allocs); delete ch; return rc; }
  ctx->chains[key] = ch;
  ctx->last_chain = ch;
  *out = ch;
  return OPB_OK;
}

int run_chain(opb_ctx* ctx, Chain* ch, bool u8_input) {
  for (Op& op : ch->ops) {
    if (op.kind == OP_FIRST) op.C = u8_input ? 1 : 0;
    int rc = launch_op(ctx, ch, op);
    if (rc) return rc;
    prof_mark(ctx, op.tag);
  }
  return OPB_OK;
}

// ------------------------------------------------------------------ post-process
int get_post(opb_ctx* ctx, int n, int H, int W, PostWs** out) {
  const long long key = slot_key(ctx, n, H, W);
  auto it = ctx->posts.find(key);
  if (it != ctx->posts.end()) { *out = it->second; ctx->last_post = it->second; return OPB_OK; }
  if (ctx->posts.size() >= 6) {
    cudaDeviceSynchronize();
    for (auto& kv : ctx->posts) { free_all(kv.second->allocs); delete kv.second; }
    ctx->posts.clear();
    ctx->cache_epoch++;
    ctx->last_post = nullptr;
  }
  PostWs* ws = new PostWs();
  ws->N = n; ws->H = H; ws->W = W;
  const opb_params& p = ctx->prm;
  int rc = 0;
#define RC(x) do { rc = (x); if (rc) { free_all(ws->allocs); delete ws; return rc; } } while (0)
  RC(dev_alloc(ctx, &ws->pafs, static_cast<size_t>(n) * 38 * H * W, ws->allocs, false));
  RC(dev_alloc(ctx, &ws->heat, static_cast<size_t>(n) * 19 * H * W, ws->allocs, false));
  RC(dev_alloc(ctx, &ws->keys, static_cast<size_t>(n) * p.max_peaks, ws->allocs));
  RC(dev_alloc(ctx, &ws->tile_max, static_cast<size_t>(n) * 18 * ((H + PK_CELL - 1) / PK_CELL) * ((W + PK_CELL - 1) / PK_CELL), ws->allocs));
  RC(dev_alloc(ctx, &ws->peak_counts, n + 1, ws->allocs));     // [n] counts + the peak kernel's work counter
  RC(dev_alloc(ctx, &ws->peaks, static_cast<size_t>(n) * p.max_peaks, ws->allocs));
  RC(dev_alloc(ctx, &ws->idx_list, static_cast<size_t>(n) * p.max_peaks, ws->allocs));
  RC(dev_alloc(ctx, &ws->type_start, static_cast<size_t>(n) * 19, ws->allocs));
  RC(dev_alloc(ctx, &ws->status, n, ws->allocs));
  RC(dev_alloc(ctx, &ws->cands, static_cast<size_t>(n) * 19 * p.max_candidates, ws->allocs, false));
  RC(dev_alloc(ctx, &ws->cands_alt, static_cast<size_t>(n) * 19 * p.max_candidates, ws->allocs, false));
  RC(dev_alloc(ctx, &ws->cand_counts, static_cast<size_t>(n) * 19, ws->allocs));
  RC(dev_alloc(ctx, &ws->conns, static_cast<size_t>(n) * 19 * ctx->conn_cap, ws->allocs, false));
  RC(dev_alloc(ctx, &ws->conn_counts, static_cast<size_t>(n) * 19, ws->allocs));
  RC(dev_alloc(ctx, &ws->subsets_out, static_cast<size_t>(n) * p.max_persons * 20, ws->allocs, false));
  {  // ONE contiguous record block [n headers | n x max_persons persons]: the payload of opb_allgather_results
    static_assert(sizeof(ImageHeader) % 16 == 0, "persons must stay 16-byte aligned behind the headers");
    uint8_t* rec = nullptr;
    RC(dev_alloc(ctx, &rec, static_cast<size_t>(n) * (sizeof(ImageHeader) + sizeof(PersonOut) * p.max_persons), ws->allocs));
    ws->headers = reinterpret_cast<ImageHeader*>(rec);
    ws->persons = reinterpret_cast<PersonOut*>(rec + static_cast<size_t>(n) * sizeof(ImageHeader));
  }
#undef RC
  ctx->posts[key] = ws;
  ctx->last_post = ws;
  *out = ws;
  return OPB_OK;
}

int launch_upsample(opb_ctx* ctx, const float* in, int planes, int h, int w, float* out, int H, int W) {
  const int ppb = 19;
  dim3 block(32, 8);
  const bool v4 = (W % 4 == 0) && ((reinterpret_cast<uintptr_t>(out) & 15) == 0);
  dim3 grid(v4 ? (W + 127) / 128 : (W + 31) / 32, (H + 7) / 8, (planes + ppb - 1) / ppb);
  if (grid.z > 65535) OPB_FAIL(ctx, OPB_ERR_ARG, "too many planes");
  if (v4) upsample_bilinear_ac_v4_kernel<<<grid, block, 0, ctx->stream>>>(in, planes, h, w, out, H, W, ppb);
  else upsample_bilinear_ac_kernel<<<grid, block, 0, ctx->stream>>>(in, planes, h, w, out, H, W, ppb);
  ctx->launches++;
  OPB_CUDA(ctx, cudaGetLastError());
  return OPB_OK;
}

// One axis of the combined (align-corners bilinear upsample, then Gaussian with scipy's 'reflect' border) operator of
// csrc/peaks_sep.cuh: rec[i] = {w0..w5, first input index (int bits), 0}.  false if some output depends on more than
// PKS_TAPS inputs or the first indices are not non-decreasing (the kernel's sliding window needs both).
bool build_sep_axis(int n_in, int n_out, const GaussTaps& taps, std::vector<float>& rec) {
  if (n_in < PKS_TAPS || n_out < 1) return false;
  const int R = taps.radius;
  const double step = (n_out > 1) ? static_cast<double>(n_in - 1) / static_cast<double>(n_out - 1) : 0.0;
  rec.assign(static_cast<size_t>(n_out) * 8, 0.f);
  std::vector<double> c(n_in);
  int prev_base = 0;
  for (int i = 0; i < n_out; ++i) {
    std::fill(c.begin(), c.end(), 0.0);
    for (int j = -R; j <= R; ++j) {
      int ii = i + j;
      while (ii < 0 || ii >= n_out) { if (ii < 0) ii = -ii - 1; if (ii >= n_out) ii = 2 * n_out - 1 - ii; }
      const double u = (n_out == 1) ? 0.0 : (ii == n_out - 1) ? static_cast<double>(n_in - 1) : ii * step;
      int k = static_cast<int>(std::floor(u));
      k = std::max(0, std::min(k, n_in - 2));
      c[k] += taps.w[j + R] * (static_cast<double>(k + 1) - u);
      c[k + 1] += taps.w[j + R] * (u - static_cast<double>(k));
    }
    int lo = 0, hi = n_in - 1;
    while (lo < n_in - 1 && c[lo] == 0.0) ++lo;
    while (hi > lo && c[hi] == 0.0) --hi;
    if (hi - lo + 1 > PKS_TAPS) return false;
    int base = std::max(0, std::min(lo, n_in - PKS_TAPS));
    base = std::max(base, prev_base);                    // keep the window monotone (it still has to cover [lo, hi])
    if (base > lo || base + PKS_TAPS - 1 < hi) return false;
    prev_base = base;
    for (int k = 0; k < PKS_TAPS; ++k) rec[static_cast<size_t>(i) * 8 + k] = static_cast<float>(c[base + k]);
    std::memcpy(&rec[static_cast<size_t>(i) * 8 + 6], &base, sizeof(int));
  }
  return true;
}

// (re)builds the operator records of workspace `ws` for low-resolution size (h_lo, w_lo); *ok = usable
int ensure_sep_axes(opb_ctx* ctx, PostWs* ws, int h_lo, int w_lo, bool* ok) {
  if (ws->sep_h == h_lo && ws->sep_w == w_lo) { *ok = true; return OPB_OK; }
  if (ws->sep_h == -h_lo - 1 && ws->sep_w == -w_lo - 1) { *ok = false; return OPB_OK; }
  std::vector<float> ry, rx;
  const bool good = ctx->taps.radius == PK_R_FAST && ws->H <= 4096 && build_sep_axis(h_lo, ws->H, ctx->taps, ry) &&
                    build_sep_axis(w_lo, ws->W, ctx->taps, rx) &&
                    smooth_nms_sep_smem_bytes(ws->H, PKS_MAX_WARPS) <= 200 * 1024;
  if (!good) { ws->sep_h = -h_lo - 1; ws->sep_w = -w_lo - 1; *ok = false; return OPB_OK; }
  if (!ws->sep_wy) {
    int rc = dev_alloc(ctx, &ws->sep_wy, static_cast<size_t>(ws->H) * 8, ws->allocs, false);
    if (rc) return rc;
    if ((rc = dev_alloc(ctx, &ws->sep_wx, static_cast<size_t>(ws->W) * 8, ws->allocs, false))) return rc;
  }
  OPB_CUDA(ctx, cudaMemcpyAsync(ws->sep_wy, ry.data(), ry.size() * 4, cudaMemcpyHostToDevice, ctx->stream));
  OPB_CUDA(ctx, cudaMemcpyAsync(ws->sep_wx, rx.data(), rx.size() * 4, cudaMemcpyHostToDevice, ctx->stream));
  OPB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));   // the host vectors die here
  ws->sep_h = h_lo; ws->sep_w = w_lo;
  *ok = true;
  return OPB_OK;
}

// heat: [n][c_total][H][W]; fills ws->peaks / idx_list / type_start / peak_counts.
// h_lo > 0: `heat` is the network-resolution map [n][c_total][h_lo][w_lo] and the peak kernel interpolates its tiles
// from it (smooth_nms_lowres_kernel): the same peaks as upsampling to (H, W) first, without the full-resolution map.
// heat_full != nullptr (with h_lo > 0): the materialised maps are read as usual and only the tile-skip bound comes from the
// low-resolution maps (smooth_nms_loskip_kernel).
int launch_peaks(opb_ctx* ctx, PostWs* ws, const float* heat, int n, int c_total, int H, int W, int h_lo = 0,
                 int w_lo = 0, const float* heat_full = nullptr) {
  const opb_params& p = ctx->prm;
  OPB_CUDA(ctx, cudaMemsetAsync(ws->peak_counts, 0, sizeof(int) * (n + 1), ctx->stream));
  OPB_CUDA(ctx, cudaMemsetAsync(ws->status, 0, sizeof(int) * n, ctx->stream));
  const int c_use = c_total - 1;   // background channel dropped, pose_detector.py:78
  const size_t smem = smooth_nms_smem_bytes(ctx->taps.radius);
  // function attributes are per device: key the one-time flags by device like the conv launchers do
  static bool attr1_d[64] = {}, attr2_d[64] = {}, attr3_d[64] = {}, attr4_d[64] = {};
  bool &attr1 = attr1_d[ctx->device & 63], &attr2 = attr2_d[ctx->device & 63], &attr3 = attr3_d[ctx->device & 63],
       &attr4 = attr4_d[ctx->device & 63];
  if (!attr1) {
    OPB_CUDA(ctx, cudaFuncSetAttribute(smooth_nms_kernel<PK_R_FAST>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
    OPB_CUDA(ctx, cudaFuncSetAttribute(smooth_nms_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
    attr1 = true;
  }
  dim3 grid((W + PK_TX - 1) / PK_TX, (H + PK_TY - 1) / PK_TY, n * c_use);
  if (grid.z > 65535) OPB_FAIL(ctx, OPB_ERR_ARG, "batch too large for the peaks grid");
  if (h_lo > 0) {
    if (!attr3) {
      OPB_CUDA(ctx, cudaFuncSetAttribute(smooth_nms_lowres_kernel<PK_R_FAST>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
      OPB_CUDA(ctx, cudaFuncSetAttribute(smooth_nms_lowres_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
      OPB_CUDA(ctx, cudaFuncSetAttribute(smooth_nms_loskip_kernel<PK_R_FAST>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
      OPB_CUDA(ctx, cudaFuncSetAttribute(smooth_nms_loskip_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
      attr3 = true;
    }
    if (h_lo < 2 || w_lo < 2) OPB_FAIL(ctx, OPB_ERR_ARG, "low-resolution maps need at least 2 x 2 samples");
    bool sep = false;
    if (!heat_full && ctx->fused_peaks == 3 && H == ws->H && W == ws->W) {   // separable-operator candidate search (peaks_sep.cuh)
      int rc = ensure_sep_axes(ctx, ws, h_lo, w_lo, &sep);
      if (rc) return rc;
    }
    if (sep) {
      // one block per plane; its warps pull 30-column x 32-row cells from a shared counter (no lockstep between warps)
      const int n_cells = ((W + 29) / 30) * ((H + PKS_SEG - 1) / PKS_SEG);
      const int nw = std::max(1, std::min(PKS_MAX_WARPS, n_cells));
      static bool attr5_d[64] = {};
      if (!attr5_d[ctx->device & 63]) {
        OPB_CUDA(ctx, cudaFuncSetAttribute(smooth_nms_sep_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
        attr5_d[ctx->device & 63] = true;
      }
      // persistent blocks (as many as fit: registers / 75 KB of shared memory allow 3 per SM); warps pull (plane, cell)
      // items from a global counter, so there is no tail of half-empty waves
      const long long n_items = static_cast<long long>(n) * c_use * n_cells;
      dim3 gs(static_cast<unsigned>(std::min<long long>((n_items + nw - 1) / nw, 3LL * ctx->num_sms)), 1, 1);
      SepAxes axes{ws->sep_wy, ws->sep_wx};
      smooth_nms_sep_kernel<<<gs, nw * 32, smooth_nms_sep_smem_bytes(H, nw), ctx->stream>>>(
          heat, c_total, c_use, n * c_use, h_lo, w_lo, H, W, ctx->taps, static_cast<float>(p.heatmap_peak_thresh), axes, ws->keys,
          ws->peak_counts, p.max_peaks, ws->peak_counts + n);
    } else if (heat_full && ctx->peaks_v2 && ctx->taps.radius == PK_R_FAST) {   // + both smoothing passes on all threads
      if (!attr4) {
        OPB_CUDA(ctx, cudaFuncSetAttribute(smooth_nms_loskip_kernel_v2<PK_R_FAST>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
        attr4 = true;
      }
      smooth_nms_loskip_kernel_v2<PK_R_FAST><<<grid, PK_THREADS, smem, ctx->stream>>>(
          heat_full, heat, c_total, c_use, h_lo, w_lo, H, W, ctx->taps, static_cast<float>(p.heatmap_peak_thresh),
          ws->keys, ws->peak_counts, p.max_peaks);
    } else if (heat_full) {   // materialised maps, tile-skip bound from the low-resolution maps (no cell_max pass)
      if (ctx->taps.radius == PK_R_FAST)
        smooth_nms_loskip_kernel<PK_R_FAST><<<grid, PK_THREADS, smem, ctx->stream>>>(
            heat_full, heat, c_total, c_use, h_lo, w_lo, H, W, ctx->taps, static_cast<float>(p.heatmap_peak_thresh),
            ws->keys, ws->peak_counts, p.max_peaks);
      else
        smooth_nms_loskip_kernel<0><<<grid, PK_THREADS, smem, ctx->stream>>>(
            heat_full, heat, c_total, c_use, h_lo, w_lo, H, W, ctx->taps, static_cast<float>(p.heatmap_peak_thresh),
            ws->keys, ws->peak_counts, p.max_peaks);
    } else if (ctx->taps.radius == PK_R_FAST)
      smooth_nms_lowres_kernel<PK_R_FAST><<<grid, PK_THREADS, smem, ctx->stream>>>(
          heat, c_total, c_use, h_lo, w_lo, H, W, ctx->taps, static_cast<float>(p.heatmap_peak_thresh), ws->keys,
          ws->peak_counts, p.max_peaks);
    else
      smooth_nms_lowres_kernel<0><<<grid, PK_THREADS, smem, ctx->stream>>>(
          heat, c_total, c_use, h_lo, w_lo, H, W, ctx->taps, static_cast<float>(p.heatmap_peak_thresh), ws->keys,
          ws->peak_counts, p.max_peaks);
  } else {
  cell_max_kernel<<<grid, 256, 0, ctx->stream>>>(heat, c_total, c_use, H, W, ws->tile_max, (H + PK_CELL - 1) / PK_CELL,
                                                 (W + PK_CELL - 1) / PK_CELL);
  ctx->launches++;
  prof_mark(ctx, "tile_max");
  if (ctx->taps.radius == PK_R_FAST)
    smooth_nms_kernel<PK_R_FAST><<<grid, PK_THREADS, smem, ctx->stream>>>(heat, c_total, c_use, H, W, ctx->taps,
                                                                   static_cast<float>(p.heatmap_peak_thresh), ws->keys,
                                                                   ws->peak_counts, p.max_peaks, ws->tile_max);
  else
    smooth_nms_kernel<0><<<grid, PK_THREADS, smem, ctx->stream>>>(heat, c_total, c_use, H, W, ctx->taps,
                                                           static_cast<float>(p.heatmap_peak_thresh), ws->keys,
                                                           ws->peak_counts, p.max_peaks, ws->tile_max);
  }
  ctx->launches++;
  OPB_CUDA(ctx, cudaGetLastError());
  prof_mark(ctx, "smooth_nms");
  int npow = 1;
  while (npow < p.max_peaks) npow <<= 1;
  const size_t smem2 = static_cast<size_t>(npow) * 8;
  if (!attr2) {
    OPB_CUDA(ctx, cudaFuncSetAttribute(sort_peaks_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    attr2 = true;
  }
  sort_peaks_kernel<<<n, 1024, smem2, ctx->stream>>>(ws->keys, ws->peak_counts, p.max_peaks, H, W, 18, ws->peaks,
                                                     ws->idx_list, ws->type_start, ws->status);
  ctx->launches++;
  OPB_CUDA(ctx, cudaGetLastError());
  return OPB_OK;
}

// h_lo > 0: `pafs` is the network-resolution map [n][38][h_lo][w_lo]; the line integrals sample it on demand
// (paf_candidates_lowres_kernel) at the positions of the (H, W) map the reference upsamples to.
int launch_connections(opb_ctx* ctx, PostWs* ws, const float* pafs, int n, int H, int W, double img_len, int h_lo = 0,
                       int w_lo = 0) {
  const opb_params& p = ctx->prm;
  OPB_CUDA(ctx, cudaMemsetAsync(ws->cand_counts, 0, sizeof(int) * n * 19, ctx->stream));
  dim3 g1(8, 19, n);
  if (h_lo > 0) {
    if (h_lo < 2 || w_lo < 2) OPB_FAIL(ctx, OPB_ERR_ARG, "low-resolution maps need at least 2 x 2 samples");
    paf_candidates_lowres_kernel<<<g1, 128, 0, ctx->stream>>>(pafs, h_lo, w_lo, H, W, ws->peaks, ws->idx_list,
                                                              ws->type_start, p.max_peaks, 18, ctx->pc, img_len,
                                                              ws->cands, ws->cand_counts, p.max_candidates);
  } else {
  paf_candidates_kernel<<<g1, 128, 0, ctx->stream>>>(pafs, H, W, ws->peaks, ws->idx_list, ws->type_start,
                                                     p.max_peaks, 18, ctx->pc, img_len, ws->cands, ws->cand_counts,
                                                     p.max_candidates);
  }
  ctx->launches++;
  OPB_CUDA(ctx, cudaGetLastError());
  prof_mark(ctx, "paf_candidates");
  dim3 g2(19, n);
  limb_assign_kernel<<<g2, kAssignThreads, 0, ctx->stream>>>(ws->peaks, ws->idx_list, ws->type_start, p.max_peaks, 18,
                                                             ctx->pc, ws->cands, ws->cands_alt, ws->cand_counts,
                                                             p.max_candidates, ws->conns, ws->conn_counts, ctx->conn_cap,
                                                             ws->status);
  ctx->launches++;
  OPB_CUDA(ctx, cudaGetLastError());
  return OPB_OK;
}

int launch_group(opb_ctx* ctx, PostWs* ws, int n, bool with_counts) {
  // peak ids fit int16 (max_peaks <= 16384); the subset table takes 52 B of shared memory per row
  const size_t table_bytes = group_smem_bytes(ctx->prm.max_persons, ctx->prm.max_peaks);
  if (table_bytes > 48 * 1024)
    OPB_CUDA(ctx, cudaFuncSetAttribute(group_persons_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       static_cast<int>(table_bytes)));
  group_persons_kernel<<<n, 32, table_bytes, ctx->stream>>>(
      ws->peaks, with_counts ? ws->peak_counts : nullptr, ctx->prm.max_peaks, ctx->pc, ws->conns, ws->conn_counts,
      ctx->conn_cap, ctx->prm.max_persons, ws->status, ws->headers, ws->persons, ws->subsets_out);
  ctx->launches++;
  OPB_CUDA(ctx, cudaGetLastError());
  return OPB_OK;
}

int copy_in(opb_ctx* ctx, void* dst, const void* src, size_t bytes, int loc) {
  OPB_CUDA(ctx, cudaMemcpyAsync(dst, src, bytes, loc == OPB_HOST ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice,
                                ctx->stream));
  return OPB_OK;
}
int copy_out(opb_ctx* ctx, void* dst, const void* src, size_t bytes, int loc) {
  OPB_CUDA(ctx, cudaMemcpyAsync(dst, src, bytes, loc == OPB_HOST ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice,
                                ctx->stream));
  return OPB_OK;
}

// host peak table [n,5] float64 -> device PeakD + per-type stable index lists
int upload_peaks(opb_ctx* ctx, PostWs* ws, const double* peaks, int n_peaks) {
  if (n_peaks > ctx->prm.max_peaks) OPB_FAIL(ctx, OPB_ERR_CAPACITY, "peak table larger than opb_params.max_peaks");
  std::vector<PeakD> pk(n_peaks);
  std::vector<int> idx(n_peaks), ts(19, 0);
  std::vector<int> cnt(19, 0);
  for (int i = 0; i < n_peaks; ++i) {
    pk[i].type = static_cast<int>(peaks[i * 5 + 0]);
    pk[i].x = peaks[i * 5 + 1];
    pk[i].y = peaks[i * 5 + 2];
    pk[i].score = static_cast<float>(peaks[i * 5 + 3]);
    if (pk[i].type < 0 || pk[i].type >= 18) OPB_FAIL(ctx, OPB_ERR_ARG, "peak type out of range");
    cnt[pk[i].type + 1]++;
  }
  for (int t = 1; t < 19; ++t) ts[t] = ts[t - 1] + cnt[t];
  std::vector<int> fill(ts.begin(), ts.end());
  for (int i = 0; i < n_peaks; ++i) idx[fill[pk[i].type]++] = i;
  OPB_CUDA(ctx, cudaMemcpyAsync(ws->peaks, pk.data(), sizeof(PeakD) * n_peaks, cudaMemcpyHostToDevice, ctx->stream));
  OPB_CUDA(ctx, cudaMemcpyAsync(ws->idx_list, idx.data(), sizeof(int) * n_peaks, cudaMemcpyHostToDevice, ctx->stream));
  OPB_CUDA(ctx, cudaMemcpyAsync(ws->type_start, ts.data(), sizeof(int) * 19, cudaMemcpyHostToDevice, ctx->stream));
  OPB_CUDA(ctx, cudaMemcpyAsync(ws->peak_counts, &n_peaks, sizeof(int), cudaMemcpyHostToDevice, ctx->stream));
  OPB_CUDA(ctx, cudaMemsetAsync(ws->status, 0, sizeof(int), ctx->stream));
  OPB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return OPB_OK;
}

}  // namespace

// ====================================================================== C ABI
extern "C" {

int opb_version(void) { return 1; }

const char* opb_last_error(const opb_ctx* ctx) { return ctx ? ctx->err.c_str() : g_create_error.c_str(); }

int opb_create(opb_ctx** out, int device, const opb_params* params) {
  if (!out || !params) { g_create_error = "null argument"; return OPB_ERR_ARG; }
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0) {
    g_create_error = std::string("no CUDA device: ") + cudaGetErrorString(e) + " (libopb has no CPU fallback)";
    return OPB_ERR_CUDA;
  }
  if (device < 0) device = 0;   // reference: device<0 means CPU; here it means GPU 0 (no CPU path)
  if (device >= ndev) { g_create_error = "device id out of range"; return OPB_ERR_ARG; }
  cudaDeviceProp prop;
  cudaGetDeviceProperties(&prop, device);
  if (prop.major != 9 || prop.minor != 0) {   // sm_90a code (wgmma) loads on compute capability 9.0 only
    g_create_error = "libopb is built for sm_90a (H100) only; found sm_" + std::to_string(prop.major * 10 + prop.minor);
    return OPB_ERR_UNSUPPORTED;
  }
  if (params->n_integ_points != 10 || params->gauss_radius < 1 || params->gauss_radius > PK_R_MAX ||
      params->max_peaks < 32 || params->max_peaks > 16384 || params->max_candidates < 32 || params->max_persons < 1 || params->max_persons > 4096) {
    g_create_error = "unsupported opb_params (n_integ_points must be 10, gauss_radius 1..16, max_peaks 32..16384, max_persons 1..4096)";
    return OPB_ERR_ARG;
  }
  opb_ctx* ctx = new opb_ctx();
  ctx->device = device;
  ctx->num_sms = prop.multiProcessorCount;
  ctx->prm = *params;
  cudaSetDevice(device);
  if (cudaStreamCreateWithFlags(&ctx->own_stream, cudaStreamNonBlocking) != cudaSuccess) {
    g_create_error = "cudaStreamCreate failed";
    delete ctx;
    return OPB_ERR_CUDA;
  }
  ctx->stream = ctx->own_stream;
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult qres;
  e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres);
  if (e != cudaSuccess || !fn) {
    g_create_error = "cuTensorMapEncodeTiled driver entry point not found";
    delete ctx;
    return OPB_ERR_CUDA;
  }
  ctx->encode = reinterpret_cast<EncodeTiledFn>(fn);
  std::memset(&ctx->pc, 0, sizeof(ctx->pc));
  for (int l = 0; l < 19; ++l) { ctx->pc.limbs[l][0] = params->limbs[l][0]; ctx->pc.limbs[l][1] = params->limbs[l][1]; }
  ctx->pc.inner_product_thresh = params->inner_product_thresh;
  ctx->pc.limb_length_ratio = params->limb_length_ratio;
  ctx->pc.length_penalty_value = params->length_penalty_value;
  ctx->pc.n_subset_limbs_thresh = params->n_subset_limbs_thresh;
  ctx->pc.subset_score_thresh = params->subset_score_thresh;
  ctx->pc.n_integ_points_thresh = params->n_integ_points_thresh;
  ctx->taps.radius = params->gauss_radius;
  for (int i = 0; i < 2 * params->gauss_radius + 1; ++i) ctx->taps.w[i] = params->gauss_taps[i];
  ctx->conn_cap = kAssignMaxType;
  ctx->profile = getenv("OPB_PROFILE") && atoi(getenv("OPB_PROFILE")) > 0;
  if (const char* g = getenv("OPB_GRAPH")) ctx->use_graphs = atoi(g);
  if (const char* g = getenv("OPB_TWO_STREAMS")) ctx->two_streams = atoi(g);
  if (const char* g = getenv("OPB_FUSED_PEAKS")) ctx->fused_peaks = atoi(g);
  if (const char* g = getenv("OPB_PAF_LOWRES")) ctx->paf_lowres = atoi(g);
  if (const char* g = getenv("OPB_PEAKS_V2")) ctx->peaks_v2 = atoi(g);
  *out = ctx;
  return OPB_OK;
}

void opb_destroy(opb_ctx* ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  cudaDeviceSynchronize();
  for (auto& kv : ctx->chains) { free_all(kv.second->allocs); delete kv.second; }
  for (auto& kv : ctx->posts) { free_all(kv.second->allocs); delete kv.second; }
  free_all(ctx->weight_allocs);
  if (ctx->ingest_buf) cudaFree(ctx->ingest_buf);
  if (ctx->precise_mid) cudaFree(ctx->precise_mid);
  if (ctx->ov_buf) cudaFree(ctx->ov_buf);
  if (ctx->wb_buf) cudaFree(ctx->wb_buf);
  if (ctx->wb_host) cudaFreeHost(ctx->wb_host);
  if (ctx->kp_ws) {
    cudaFree(ctx->kp_ws->up); cudaFree(ctx->kp_ws->tmp); cudaFree(ctx->kp_ws->res); cudaFreeHost(ctx->kp_ws->h_res);
    cudaFree(ctx->kp_ws->crops);
    delete ctx->kp_ws;
  }
  delete ctx->cascade;
  for (auto& sl : ctx->slots) {
    if (sl.d_frames) cudaFree(sl.d_frames);
    if (sl.h_frames) cudaFreeHost(sl.h_frames);
    if (sl.h_result) cudaFreeHost(sl.h_result);
    if (sl.gexec) cudaGraphExecDestroy(sl.gexec);
    if (sl.h2d_done) cudaEventDestroy(sl.h2d_done);
    if (sl.done) cudaEventDestroy(sl.done);
  }
  if (ctx->copy_stream) cudaStreamDestroy(ctx->copy_stream);
  if (ctx->stream_b) cudaStreamDestroy(ctx->stream_b);
  if (ctx->own_stream) cudaStreamDestroy(ctx->own_stream);
  delete ctx;
}

int opb_set_stream(opb_ctx* ctx, void* cuda_stream) {
  if (!ctx) return OPB_ERR_ARG;
  ctx->stream = cuda_stream ? static_cast<cudaStream_t>(cuda_stream) : ctx->own_stream;
  return OPB_OK;
}

int opb_synchronize(opb_ctx* ctx) {
  if (!ctx) return OPB_ERR_ARG;
  OPB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (ctx->stream_b) OPB_CUDA(ctx, cudaStreamSynchronize(ctx->stream_b));   // streaming slot 1
  return OPB_OK;
}

int64_t opb_launch_count(const opb_ctx* ctx) { return ctx ? ctx->launches : 0; }

int opb_load_weights(opb_ctx* ctx, const char* layer, const float* W, const int64_t shape[4], const float* b) {
  if (!ctx || !layer || !W || !shape || !b) return OPB_ERR_ARG;
  if (shape[2] != shape[3] || (shape[2] != 1 && shape[2] != 3 && shape[2] != 7))
    OPB_FAIL(ctx, OPB_ERR_ARG, std::string("unsupported kernel shape for layer ") + layer);
  HostLayer L;
  L.cout = static_cast<int>(shape[0]);
  L.cin = static_cast<int>(shape[1]);
  L.ks = static_cast<int>(shape[2]);
  const size_t n = static_cast<size_t>(L.cout) * L.cin * L.ks * L.ks;
  L.W.assign(W, W + n);
  L.b.assign(b, b + L.cout);
  ctx->host_layers[layer] = std::move(L);
  return OPB_OK;
}

int opb_finalize_weights(opb_ctx* ctx, int precision_mode) {
  if (!ctx) return OPB_ERR_ARG;
  if (precision_mode != OPB_PRECISION_FAST && precision_mode != OPB_PRECISION_PARITY && precision_mode != OPB_PRECISION_COMP)
    OPB_FAIL(ctx, OPB_ERR_ARG, "bad precision mode");
  cudaSetDevice(ctx->device);
  // drop everything derived from older weights
  OPB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  for (auto& kv : ctx->chains) { free_all(kv.second->allocs); delete kv.second; }
  ctx->chains.clear();
  ctx->cache_epoch++;
  ctx->last_chain = nullptr;
  free_all(ctx->weight_allocs);
  ctx->packed.clear();
  ctx->precision = precision_mode;
  const int split = precision_mode;   // pack_weights' precision argument
  int rc;
  // conv1_1: [27][64] fp32, k = (r*3+s)*3 + c
  {
    auto it = ctx->host_layers.find("conv1_1");
    if (it == ctx->host_layers.end()) OPB_FAIL(ctx, OPB_ERR_STATE, "weights for layer conv1_1 were not loaded");
    const HostLayer& L = it->second;
    if (L.cin != 3 || L.cout != 64 || L.ks != 3) OPB_FAIL(ctx, OPB_ERR_ARG, "conv1_1 must be 3->64, 3x3");
    std::vector<float> wt(27 * 64);
    for (int o = 0; o < 64; ++o)
      for (int c = 0; c < 3; ++c)
        for (int t = 0; t < 9; ++t) wt[(t * 3 + c) * 64 + o] = L.W[(static_cast<size_t>(o) * 3 + c) * 9 + t];
    if ((rc = dev_alloc(ctx, &ctx->w_first, wt.size(), ctx->weight_allocs, false))) return rc;
    if ((rc = dev_alloc(ctx, &ctx->b_first, 64, ctx->weight_allocs, false))) return rc;
    OPB_CUDA(ctx, cudaMemcpyAsync(ctx->w_first, wt.data(), wt.size() * 4, cudaMemcpyHostToDevice, ctx->stream));
    OPB_CUDA(ctx, cudaMemcpyAsync(ctx->b_first, L.b.data(), 64 * 4, cudaMemcpyHostToDevice, ctx->stream));
    OPB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  }
  auto simple = [&](const std::string& name, int cin, int cout, int ks) -> int {
    return pack_weights(ctx, name, {{name, cout}}, identity_map(cin, round_up(cin, 64)), ks, split);
  };
  ctx->kp_out = 0;
  ctx->u8_denom = 255.f;
  if (ctx->host_layers.count("conv6_2_CPM")) {
    // FaceNet / HandNet (models/FaceNet.py:10-76): 52 layers, single branch; uint8 input is /256 - 0.5
    const int KC = ctx->host_layers.at("conv6_2_CPM").cout;
    if (KC < 2 || KC > 128) OPB_FAIL(ctx, OPB_ERR_ARG, "conv6_2_CPM must have 2..128 output channels");
    const int kc_pad = KC <= 48 ? 48 : KC <= 64 ? 64 : 128;
    const struct { const char* n; int cin, cout; } vgg[] = {
        {"conv1_2", 64, 64},   {"conv2_1", 64, 128},  {"conv2_2", 128, 128}, {"conv3_1", 128, 256}, {"conv3_2", 256, 256},
        {"conv3_3", 256, 256}, {"conv3_4", 256, 256}, {"conv4_1", 256, 512}, {"conv4_2", 512, 512}, {"conv4_3", 512, 512},
        {"conv4_4", 512, 512}, {"conv5_1", 512, 512}, {"conv5_2", 512, 512}, {"conv5_3_CPM", 512, 128}};
    for (auto& b : vgg)
      if ((rc = simple(b.n, b.cin, b.cout, 3))) return rc;
    if ((rc = simple("conv6_1_CPM", 128, 512, 1))) return rc;
    if ((rc = pack_weights(ctx, "conv6_2_CPM", {{"conv6_2_CPM", kc_pad}}, identity_map(512, 512), 1, split))) return rc;
    // device concat [features 0..127 | maps 128..128+KC-1]; reference order is (h, feature_map) (models/FaceNet.py:108)
    std::vector<int> cat_map(round_up(128 + KC, 64), -1);
    for (int d = 0; d < 128; ++d) cat_map[d] = KC + d;
    for (int d = 0; d < KC; ++d) cat_map[128 + d] = d;
    for (int st = 2; st <= 6; ++st) {
      const std::string S = "_stage" + std::to_string(st);
      if ((rc = pack_weights(ctx, "Mconv1" + S, {{"Mconv1" + S, 128}}, cat_map, 7, split))) return rc;
      for (int i = 2; i <= 5; ++i)
        if ((rc = simple("Mconv" + std::to_string(i) + S, 128, 128, 7))) return rc;
      if ((rc = simple("Mconv6" + S, 128, 128, 1))) return rc;
      if ((rc = pack_weights(ctx, "Mconv7" + S, {{"Mconv7" + S, kc_pad}}, identity_map(128, 128), 1, split))) return rc;
    }
    ctx->kp_out = KC;
    ctx->u8_denom = 256.f;
    return OPB_OK;
  }
  const struct { const char* n; int cin, cout; } backbone[] = {
      {"conv1_2", 64, 64},    {"conv2_1", 64, 128},   {"conv2_2", 128, 128},     {"conv3_1", 128, 256},
      {"conv3_2", 256, 256},  {"conv3_3", 256, 256},  {"conv3_4", 256, 256},     {"conv4_1", 256, 512},
      {"conv4_2", 512, 512},  {"conv4_3_CPM", 512, 256}, {"conv4_4_CPM", 256, 128}};
  for (auto& b : backbone)
    if ((rc = simple(b.n, b.cin, b.cout, 3))) return rc;
  for (const char* br : {"L1", "L2"}) {
    const std::string B(br);
    for (int i = 1; i <= 3; ++i)
      if ((rc = simple("conv5_" + std::to_string(i) + "_CPM_" + B, 128, 128, 3))) return rc;
    if ((rc = simple("conv5_4_CPM_" + B, 128, 512, 1))) return rc;
    if ((rc = pack_weights(ctx, "conv5_5_CPM_" + B, {{"conv5_5_CPM_" + B, 48}}, identity_map(512, 512), 1, split)))
      return rc;
  }
  // concat order on the device: [feature_map 0..127 | PAF 128..165 | heat 166..184 | 0 x 7];
  // reference order is (h1[38], h2[19], feature_map[128]) (models/CocoPoseNet.py:168)
  std::vector<int> cat_map(192, -1);
  for (int d = 0; d < 128; ++d) cat_map[d] = 57 + d;
  for (int d = 0; d < 38; ++d) cat_map[128 + d] = d;
  for (int d = 0; d < 19; ++d) cat_map[166 + d] = 38 + d;
  for (int st = 2; st <= 6; ++st) {
    const std::string S = "_stage" + std::to_string(st);
    if ((rc = pack_weights(ctx, "Mconv1" + S + "_fused", {{"Mconv1" + S + "_L1", 128}, {"Mconv1" + S + "_L2", 128}},
                           cat_map, 7, split)))
      return rc;
    for (const char* br : {"L1", "L2"}) {
      const std::string B = std::string("_") + br;
      for (int i = 2; i <= 5; ++i)
        if ((rc = simple("Mconv" + std::to_string(i) + S + B, 128, 128, 7))) return rc;
      if ((rc = simple("Mconv6" + S + B, 128, 128, 1))) return rc;
      if ((rc = pack_weights(ctx, "Mconv7" + S + B, {{"Mconv7" + S + B, 48}}, identity_map(128, 128), 1, split)))
        return rc;
    }
  }
  return OPB_OK;
}

int opb_forward(opb_ctx* ctx, const void* x, int x_format, int x_loc, int n, int h, int w, float* paf_out,
                float* heat_out, int out_loc) {
  if (!ctx || !x) return OPB_ERR_ARG;
  cudaSetDevice(ctx->device);
  Chain* ch = nullptr;
  int rc = get_chain(ctx, n, h, w, &ch);
  if (rc) return rc;
  const size_t px = static_cast<size_t>(n) * h * w * 3;
  ch->img_u8_src = nullptr;
  if (x_format == OPB_U8_NHWC_BGR) {
    if ((rc = copy_in(ctx, ch->img_u8, x, px, x_loc))) return rc;
  } else if (x_format == OPB_F32_NCHW) {
    if ((rc = copy_in(ctx, ch->img_f32, x, px * 4, x_loc))) return rc;
  } else {
    OPB_FAIL(ctx, OPB_ERR_ARG, "bad x_format");
  }
  if ((rc = run_chain(ctx, ch, x_format == OPB_U8_NHWC_BGR))) return rc;
  const size_t lo = static_cast<size_t>(n) * (h / 8) * (w / 8);
  if (paf_out && !ctx->kp_out && (rc = copy_out(ctx, paf_out, ch->paf_lo, lo * 38 * 4, out_loc))) return rc;
  if (heat_out && (rc = copy_out(ctx, heat_out, ch->heat_lo, lo * (ctx->kp_out ? ctx->kp_out : 19) * 4, out_loc))) return rc;
  OPB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return OPB_OK;
}

int opb_upsample(opb_ctx* ctx, int mode, const float* in, int in_loc, int planes, int h, int w, float* out,
                 int out_loc, int out_h, int out_w) {
  if (!ctx || !in || !out || planes <= 0) return OPB_ERR_ARG;
  cudaSetDevice(ctx->device);
  std::vector<void*> tmp;
  const float* d_in = in;
  float* d_out = out;
  int rc;
  if (in_loc == OPB_HOST) {
    float* t;
    if ((rc = dev_alloc(ctx, &t, static_cast<size_t>(planes) * h * w, tmp, false))) { free_all(tmp); return rc; }
    if ((rc = copy_in(ctx, t, in, static_cast<size_t>(planes) * h * w * 4, OPB_HOST))) { free_all(tmp); return rc; }
    d_in = t;
  }
  if (out_loc == OPB_HOST) {
    if ((rc = dev_alloc(ctx, &d_out, static_cast<size_t>(planes) * out_h * out_w, tmp, false))) { free_all(tmp); return rc; }
  }
  if (mode == OPB_UPSAMPLE_BILINEAR_AC) {
    if (h < 2 || w < 2) { free_all(tmp); OPB_FAIL(ctx, OPB_ERR_ARG, "bilinear upsample needs h, w >= 2"); }
    rc = launch_upsample(ctx, d_in, planes, h, w, d_out, out_h, out_w);
  } else if (mode == OPB_UPSAMPLE_BICUBIC) {
    dim3 grid((out_w + 31) / 32, (out_h + 7) / 8, std::min(planes, 64)), block(32, 8);
    resize_cubic_kernel<<<grid, block, 0, ctx->stream>>>(d_in, planes, h, w, d_out, out_h, out_w, out_h, out_w, 0, 0.f);
    ctx->launches++;
    rc = OPB_OK;
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { ctx->err = cudaGetErrorString(e); rc = OPB_ERR_CUDA; }
  } else {
    ctx->err = "bad upsample mode";
    rc = OPB_ERR_ARG;
  }
  if (!rc && out_loc == OPB_HOST) rc = copy_out(ctx, out, d_out, static_cast<size_t>(planes) * out_h * out_w * 4, OPB_HOST);
  cudaError_t e = cudaStreamSynchronize(ctx->stream);
  if (!rc && e != cudaSuccess) { ctx->err = cudaGetErrorString(e); rc = OPB_ERR_CUDA; }
  free_all(tmp);
  return rc;
}

int opb_peaks(opb_ctx* ctx, const float* heat, int heat_loc, int c_plus_1, int h, int w, double* peaks_out,
              int peaks_cap, int* n_peaks) {
  if (!ctx || !heat || !peaks_out || !n_peaks) return OPB_ERR_ARG;
  if (c_plus_1 != 19) OPB_FAIL(ctx, OPB_ERR_ARG, "heatmaps must have 19 channels (18 joints + background)");
  cudaSetDevice(ctx->device);
  PostWs* ws;
  int rc = get_post(ctx, 1, h, w, &ws);
  if (rc) return rc;
  const float* d_heat = heat;
  if (heat_loc == OPB_HOST) {
    if ((rc = copy_in(ctx, ws->heat, heat, static_cast<size_t>(19) * h * w * 4, OPB_HOST))) return rc;
    d_heat = ws->heat;
  }
  if ((rc = launch_peaks(ctx, ws, d_heat, 1, 19, h, w))) return rc;
  int cnt = 0, st = 0;
  OPB_CUDA(ctx, cudaMemcpyAsync(&cnt, ws->peak_counts, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
  OPB_CUDA(ctx, cudaMemcpyAsync(&st, ws->status, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
  OPB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (st) OPB_FAIL(ctx, OPB_ERR_CAPACITY, "more peaks than opb_params.max_peaks");
  if (cnt > peaks_cap) OPB_FAIL(ctx, OPB_ERR_CAPACITY, "peaks_out too small");
  std::vector<PeakD> pk(cnt);
  if (cnt) {
    OPB_CUDA(ctx, cudaMemcpyAsync(pk.data(), ws->peaks, sizeof(PeakD) * cnt, cudaMemcpyDeviceToHost, ctx->stream));
    OPB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  }
  for (int i = 0; i < cnt; ++i) {
    peaks_out[i * 5 + 0] = pk[i].type;
    peaks_out[i * 5 + 1] = pk[i].x;
    peaks_out[i * 5 + 2] = pk[i].y;
    peaks_out[i * 5 + 3] = static_cast<double>(pk[i].score);
    peaks_out[i * 5 + 4] = i;
  }
  *n_peaks = cnt;
  return OPB_OK;
}

static int download_connections(opb_ctx* ctx, PostWs* ws, int img, double* conn_out, int conn_cap, int* conn_counts) {
  std::vector<int> cc(19);
  OPB_CUDA(ctx, cudaMemcpyAsync(cc.data(), ws->conn_counts + img * 19, sizeof(int) * 19, cudaMemcpyDeviceToHost,
                                ctx->stream));
  std::vector<Connection> all(static_cast<size_t>(19) * ctx->conn_cap);
  OPB_CUDA(ctx, cudaMemcpyAsync(all.data(), ws->conns + static_cast<size_t>(img) * 19 * ctx->conn_cap,
                                sizeof(Connection) * all.size(), cudaMemcpyDeviceToHost, ctx->stream));
  OPB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  int o = 0;
  for (int l = 0; l < 19; ++l) {
    conn_counts[l] = cc[l];
    for (int k = 0; k < cc[l]; ++k) {
      if (o >= conn_cap) OPB_FAIL(ctx, OPB_ERR_CAPACITY, "conn_out too small");
      const Connection& c = all[static_cast<size_t>(l) * ctx->conn_cap + k];
      conn_out[o * 3 + 0] = c.id_a;
      conn_out[o * 3 + 1] = c.id_b;
      conn_out[o * 3 + 2] = c.score;
      ++o;
    }
  }
  return OPB_OK;
}

int opb_connections(opb_ctx* ctx, const float* paf, int paf_loc, int h, int w, const double* peaks, int n_peaks,
                    double img_len, double* conn_out, int conn_cap, int* conn_counts) {
  if (!ctx || !paf || !conn_out || !conn_counts || (n_peaks > 0 && !peaks)) return OPB_ERR_ARG;
  cudaSetDevice(ctx->device);
  PostWs* ws;
  int rc = get_post(ctx, 1, h, w, &ws);
  if (rc) return rc;
  const float* d_paf = paf;
  if (paf_loc == OPB_HOST) {
    if ((rc = copy_in(ctx, ws->pafs, paf, static_cast<size_t>(38) * h * w * 4, OPB_HOST))) return rc;
    d_paf = ws->pafs;
  }
  if ((rc = upload_peaks(ctx, ws, peaks, n_peaks))) return rc;
  if ((rc = launch_connections(ctx, ws, d_paf, 1, h, w, img_len))) return rc;
  int st = 0;
  OPB_CUDA(ctx, cudaMemcpyAsync(&st, ws->status, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
  OPB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (st) OPB_FAIL(ctx, OPB_ERR_CAPACITY, "candidate / per-type capacity exceeded (status " + std::to_string(st) +
                                              "); raise opb_params.max_candidates");
  return download_connections(ctx, ws, 0, conn_out, conn_cap, conn_counts);
}

int opb_candidates(opb_ctx* ctx, const float* paf, int h, int w, const double* cand_a, int n_a, const double* cand_b,
                   int n_b, double img_len, double* out, int out_cap, int* n_out) {
  if (!ctx || !paf || !out || !n_out || (n_a > 0 && !cand_a) || (n_b > 0 && !cand_b)) return OPB_ERR_ARG;
  cudaSetDevice(ctx->device);
  PostWs* ws;
  int rc = get_post(ctx, 1, h, w, &ws);
  if (rc) return rc;
  *n_out = 0;
  if (n_a == 0 || n_b == 0) return OPB_OK;
  // limb 0 of the table joins joint types limbs[0][0] -> limbs[0][1]; its PAF channels are 0 and 1
  const int ja = ctx->pc.limbs[0][0], jb = ctx->pc.limbs[0][1];
  std::vector<double> pk(static_cast<size_t>(n_a + n_b) * 5);
  for (int i = 0; i < n_a + n_b; ++i) {
    const double* src = (i < n_a) ? cand_a + i * 4 : cand_b + (i - n_a) * 4;
    pk[i * 5 + 0] = (i < n_a) ? ja : jb;
    pk[i * 5 + 1] = src[0]; pk[i * 5 + 2] = src[1]; pk[i * 5 + 3] = src[2]; pk[i * 5 + 4] = i;
  }
  if ((rc = upload_peaks(ctx, ws, pk.data(), n_a + n_b))) return rc;
  OPB_CUDA(ctx, cudaMemsetAsync(ws->pafs, 0, sizeof(float) * 38 * static_cast<size_t>(h) * w, ctx->stream));
  if ((rc = copy_in(ctx, ws->pafs, paf, sizeof(float) * 2 * static_cast<size_t>(h) * w, OPB_HOST))) return rc;
  OPB_CUDA(ctx, cudaMemsetAsync(ws->cand_counts, 0, sizeof(int) * 19, ctx->stream));
  dim3 g1(8, 1, 1);
  paf_candidates_kernel<<<g1, 128, 0, ctx->stream>>>(ws->pafs, h, w, ws->peaks, ws->idx_list, ws->type_start,
                                                     ctx->prm.max_peaks, 18, ctx->pc, img_len, ws->cands,
                                                     ws->cand_counts, ctx->prm.max_candidates);
  ctx->launches++;
  OPB_CUDA(ctx, cudaGetLastError());
  int cnt = 0;
  OPB_CUDA(ctx, cudaMemcpyAsync(&cnt, ws->cand_counts, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
  OPB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (cnt > ctx->prm.max_candidates) OPB_FAIL(ctx, OPB_ERR_CAPACITY, "more candidates than opb_params.max_candidates");
  if (cnt > out_cap) OPB_FAIL(ctx, OPB_ERR_CAPACITY, "out too small");
  std::vector<Candidate> cd(cnt);
  if (cnt) {
    OPB_CUDA(ctx, cudaMemcpyAsync(cd.data(), ws->cands, sizeof(Candidate) * cnt, cudaMemcpyDeviceToHost, ctx->stream));
    OPB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  }
  // presentation order only (the scores were computed on the device): descending score, ties in
  // generation order (a-major, b-minor) = Python's stable sorted(..., reverse=True)
  std::sort(cd.begin(), cd.end(), [](const Candidate& x, const Candidate& y) {
    return x.score > y.score || (x.score == y.score && x.pair < y.pair);
  });
  for (int i = 0; i < cnt; ++i) {
    const int a = cd[i].pair / n_b, b = cd[i].pair % n_b;
    out[i * 3 + 0] = static_cast<double>(static_cast<int>(cand_a[a * 4 + 3]));
    out[i * 3 + 1] = static_cast<double>(static_cast<int>(cand_b[b * 4 + 3]));
    out[i * 3 + 2] = cd[i].score;
  }
  *n_out = cnt;
  return OPB_OK;
}

int opb_group(opb_ctx* ctx, const double* conns, const int* conn_counts, const double* peaks, int n_peaks,
              double* subsets_out, int subsets_cap, int* n_subsets) {
  if (!ctx || !conn_counts || !subsets_out || !n_subsets || (n_peaks > 0 && !peaks)) return OPB_ERR_ARG;
  cudaSetDevice(ctx->device);
  PostWs* ws;
  int rc = get_post(ctx, 1, 8, 8, &ws);
  if (rc) return rc;
  if ((rc = upload_peaks(ctx, ws, peaks, n_peaks))) return rc;
  std::vector<Connection> all(static_cast<size_t>(19) * ctx->conn_cap);
  int o = 0;
  for (int l = 0; l < 19; ++l) {
    if (conn_counts[l] > ctx->conn_cap) OPB_FAIL(ctx, OPB_ERR_CAPACITY, "too many connections for one limb");
    for (int k = 0; k < conn_counts[l]; ++k, ++o) {
      Connection& c = all[static_cast<size_t>(l) * ctx->conn_cap + k];
      c.id_a = static_cast<int>(conns[o * 3 + 0]);
      c.id_b = static_cast<int>(conns[o * 3 + 1]);
      c.score = conns[o * 3 + 2];
      if (c.id_a < 0 || c.id_a >= n_peaks || c.id_b < 0 || c.id_b >= n_peaks) OPB_FAIL(ctx, OPB_ERR_ARG, "connection id out of range");
    }
  }
  OPB_CUDA(ctx, cudaMemcpyAsync(ws->conns, all.data(), sizeof(Connection) * all.size(), cudaMemcpyHostToDevice, ctx->stream));
  OPB_CUDA(ctx, cudaMemcpyAsync(ws->conn_counts, conn_counts, sizeof(int) * 19, cudaMemcpyHostToDevice, ctx->stream));
  if ((rc = launch_group(ctx, ws, 1, true))) return rc;
  ImageHeader hd;
  OPB_CUDA(ctx, cudaMemcpyAsync(&hd, ws->headers, sizeof(hd), cudaMemcpyDeviceToHost, ctx->stream));
  OPB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (hd.status == OPB_ERR_INDEX) OPB_FAIL(ctx, OPB_ERR_INDEX, "list assignment index out of range");
  if (hd.status) OPB_FAIL(ctx, OPB_ERR_CAPACITY, "more live subsets than opb_params.max_persons");
  if (hd.n_persons > subsets_cap) OPB_FAIL(ctx, OPB_ERR_CAPACITY, "subsets_out too small");
  if (hd.n_persons) {
    OPB_CUDA(ctx, cudaMemcpyAsync(subsets_out, ws->subsets_out, sizeof(double) * 20 * hd.n_persons,
                                  cudaMemcpyDeviceToHost, ctx->stream));
    OPB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  }
  *n_subsets = hd.n_persons;
  return OPB_OK;
}

// upsample + peaks + connections + grouping of n images' network outputs (device pointers, [n][38|19][h8][w8]):
// pose_detector.py:501-512.  OPB_PAF_LOWRES / OPB_FUSED_PEAKS skip the materialised full-resolution PAFs / heat maps.
static int run_postprocess(opb_ctx* ctx, PostWs* ws, int n, int h8, int w8, int map_h, int map_w, double img_len,
                           const float* paf_lo, const float* heat_lo) {
  int rc;
  ws->last_paf_lo = paf_lo; ws->last_heat_lo = heat_lo; ws->last_img_len = img_len;
  ws->last_h8 = h8; ws->last_w8 = w8;
  if (!ctx->paf_lowres) {
    if ((rc = launch_upsample(ctx, paf_lo, n * 38, h8, w8, ws->pafs, map_h, map_w))) return rc;
    prof_mark(ctx, "upsample_paf");
  }
  if (ctx->fused_peaks == 1 || ctx->fused_peaks == 3) {
    if ((rc = launch_peaks(ctx, ws, heat_lo, n, 19, map_h, map_w, h8, w8))) return rc;
  } else if (ctx->fused_peaks == 2) {
    if ((rc = launch_upsample(ctx, heat_lo, n * 19, h8, w8, ws->heat, map_h, map_w))) return rc;
    prof_mark(ctx, "upsample_heat");
    if ((rc = launch_peaks(ctx, ws, heat_lo, n, 19, map_h, map_w, h8, w8, ws->heat))) return rc;
  } else {
    if ((rc = launch_upsample(ctx, heat_lo, n * 19, h8, w8, ws->heat, map_h, map_w))) return rc;
    prof_mark(ctx, "upsample_heat");
    if ((rc = launch_peaks(ctx, ws, ws->heat, n, 19, map_h, map_w))) return rc;
  }
  prof_mark(ctx, "peaks");
  if (ctx->paf_lowres) rc = launch_connections(ctx, ws, paf_lo, n, map_h, map_w, img_len, h8, w8);
  else rc = launch_connections(ctx, ws, ws->pafs, n, map_h, map_w, img_len);
  if (rc) return rc;
  prof_mark(ctx, "connections");
  if ((rc = launch_group(ctx, ws, n, true))) return rc;
  prof_mark(ctx, "group");
  return OPB_OK;
}

// conv chain + upsample + peaks + connections + grouping for the frames ch->img_u8_src points at (all on ctx->stream,
// no host synchronisation): the device-resident body of PoseDetector.__call__ (pose_detector.py:495-512)
static int run_pipeline(opb_ctx* ctx, Chain* ch, PostWs* ws, int n, int h, int w, int map_h, int map_w, double img_len,
                        const float* inject_paf, const float* inject_heat) {
  int rc;
  if (ctx->kp_out) OPB_FAIL(ctx, OPB_ERR_STATE, "this context holds a face / hand net: use opb_keypoints_detect");
  if ((rc = run_chain(ctx, ch, true))) return rc;
  return run_postprocess(ctx, ws, n, h / 8, w / 8, map_h, map_w, img_len, inject_paf ? inject_paf : ch->paf_lo,
                         inject_heat ? inject_heat : ch->heat_lo);
}

int opb_detect_batch(opb_ctx* ctx, const uint8_t* imgs, int imgs_loc, int n, int h, int w, int map_h, int map_w,
                     double img_len, const float* inject_paf, const float* inject_heat, opb_image_header* headers_out,
                     opb_person* persons_out, int out_loc) {
  if (!ctx || !imgs || !headers_out || !persons_out) return OPB_ERR_ARG;
  cudaSetDevice(ctx->device);
  Chain* ch = nullptr;
  PostWs* ws = nullptr;
  int rc;
  if ((rc = get_chain(ctx, n, h, w, &ch))) return rc;
  if ((rc = get_post(ctx, n, map_h, map_w, &ws))) return rc;
  prof_mark(ctx, "begin");
  if (imgs_loc == OPB_DEVICE) {
    ch->img_u8_src = imgs;            // frames already resident in HBM: conv1_1 reads them in place
  } else {
    ch->img_u8_src = nullptr;
    if ((rc = copy_in(ctx, ch->img_u8, imgs, static_cast<size_t>(n) * h * w * 3, imgs_loc))) return rc;
  }
  prof_mark(ctx, "copy_in");
  if ((rc = run_pipeline(ctx, ch, ws, n, h, w, map_h, map_w, img_len, inject_paf, inject_heat))) return rc;
  if ((rc = copy_out(ctx, headers_out, ws->headers, sizeof(ImageHeader) * n, out_loc))) return rc;
  if ((rc = copy_out(ctx, persons_out, ws->persons, sizeof(PersonOut) * n * ctx->prm.max_persons, out_loc))) return rc;
  prof_mark(ctx, "copy_out");
  OPB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  prof_report(ctx);
  return OPB_OK;
}

int opb_postprocess_batch(opb_ctx* ctx, const float* paf_lo, const float* heat_lo, int maps_loc, int n, int h8, int w8,
                          int map_h, int map_w, double img_len, opb_image_header* headers_out, opb_person* persons_out,
                          int out_loc) {
  if (!ctx || !paf_lo || !heat_lo || !headers_out || !persons_out || n <= 0 || h8 < 2 || w8 < 2 || map_h <= 0 || map_w <= 0)
    return OPB_ERR_ARG;
  cudaSetDevice(ctx->device);
  PostWs* ws = nullptr;
  int rc;
  if ((rc = get_post(ctx, n, map_h, map_w, &ws))) return rc;
  const size_t plane = static_cast<size_t>(h8) * w8;
  if (maps_loc == OPB_HOST) {
    if (ws->lo_cap < static_cast<size_t>(n) * 57 * plane) {   // grows only; earlier blocks stay owned by the workspace
      if ((rc = dev_alloc(ctx, &ws->lo_stage, static_cast<size_t>(n) * 57 * plane, ws->allocs, false))) return rc;
      ws->lo_cap = static_cast<size_t>(n) * 57 * plane;
    }
    if ((rc = copy_in(ctx, ws->lo_stage, paf_lo, sizeof(float) * n * 38 * plane, OPB_HOST))) return rc;
    if ((rc = copy_in(ctx, ws->lo_stage + n * 38 * plane, heat_lo, sizeof(float) * n * 19 * plane, OPB_HOST))) return rc;
    paf_lo = ws->lo_stage;
    heat_lo = ws->lo_stage + n * 38 * plane;
  }
  if ((rc = run_postprocess(ctx, ws, n, h8, w8, map_h, map_w, img_len, paf_lo, heat_lo))) return rc;
  if ((rc = copy_out(ctx, headers_out, ws->headers, sizeof(ImageHeader) * n, out_loc))) return rc;
  if ((rc = copy_out(ctx, persons_out, ws->persons, sizeof(PersonOut) * n * ctx->prm.max_persons, out_loc))) return rc;
  OPB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return OPB_OK;
}

int opb_get_image_detail(opb_ctx* ctx, int img, double* peaks_out, int peaks_cap, int* n_peaks, double* conn_out,
                         int conn_cap, int* conn_counts, double* subsets_out, int subsets_cap, int* n_subsets) {
  if (!ctx) return OPB_ERR_ARG;
  PostWs* ws = ctx->last_post;
  if (!ws || img < 0 || img >= ws->N) OPB_FAIL(ctx, OPB_ERR_STATE, "no post-process result for that image");
  cudaSetDevice(ctx->device);
  ImageHeader hd;
  OPB_CUDA(ctx, cudaMemcpyAsync(&hd, ws->headers + img, sizeof(hd), cudaMemcpyDeviceToHost, ctx->stream));
  OPB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (n_peaks) *n_peaks = hd.n_peaks;
  if (peaks_out) {
    if (hd.n_peaks > peaks_cap) OPB_FAIL(ctx, OPB_ERR_CAPACITY, "peaks_out too small");
    std::vector<PeakD> pk(hd.n_peaks);
    if (hd.n_peaks) {
      OPB_CUDA(ctx, cudaMemcpyAsync(pk.data(), ws->peaks + static_cast<size_t>(img) * ctx->prm.max_peaks,
                                    sizeof(PeakD) * hd.n_peaks, cudaMemcpyDeviceToHost, ctx->stream));
      OPB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    }
    for (int i = 0; i < hd.n_peaks; ++i) {
      peaks_out[i * 5 + 0] = pk[i].type; peaks_out[i * 5 + 1] = pk[i].x; peaks_out[i * 5 + 2] = pk[i].y;
      peaks_out[i * 5 + 3] = static_cast<double>(pk[i].score); peaks_out[i * 5 + 4] = i;
    }
  }
  if (conn_out && conn_counts) {
    int rc = download_connections(ctx, ws, img, conn_out, conn_cap, conn_counts);
    if (rc) return rc;
  }
  if (n_subsets) *n_subsets = hd.n_persons;
  if (subsets_out) {
    if (hd.n_persons > subsets_cap) OPB_FAIL(ctx, OPB_ERR_CAPACITY, "subsets_out too small");
    if (hd.n_persons) {
      OPB_CUDA(ctx, cudaMemcpyAsync(subsets_out, ws->subsets_out + static_cast<size_t>(img) * ctx->prm.max_persons * 20,
                                    sizeof(double) * 20 * hd.n_persons, cudaMemcpyDeviceToHost, ctx->stream));
      OPB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    }
  }
  return OPB_OK;
}

int opb_precise_begin(opb_ctx* ctx, int orig_h, int orig_w) {
  if (!ctx || orig_h <= 0 || orig_w <= 0) return OPB_ERR_ARG;
  cudaSetDevice(ctx->device);
  PostWs* ws;
  return get_post(ctx, 1, orig_h, orig_w, &ws);
}

static int ensure_ingest(opb_ctx* ctx, size_t bytes);
static int launch_resize_u8(opb_ctx* ctx, const uint8_t* d_src, int n, int h0, int w0, uint8_t* d_dst, int h, int w,
                            bool cubic = false);

// forward + both cubic resizes + accumulate for the padded frame already in ch->img_u8 (:447-467)
static int precise_accumulate(opb_ctx* ctx, PostWs* ws, Chain* ch, int ph, int pw, int pad_h, int pad_w, int scale_index,
                              int n_scales) {
  int rc;
  ch->img_u8_src = nullptr;
  if ((rc = run_chain(ctx, ch, true))) return rc;
  const int h8 = ph / 8, w8 = pw / 8;
  const int ch_h = ph - pad_h, ch_w = pw - pad_w;   // crop after the x8 resize (:462,:466)
  const size_t need = static_cast<size_t>(38) * ch_h * ch_w;
  if (ctx->precise_mid_cap < need) {                 // x8 intermediate, kept across scales and calls
    if (ctx->precise_mid) { OPB_CUDA(ctx, cudaStreamSynchronize(ctx->stream)); cudaFree(ctx->precise_mid); ctx->precise_mid = nullptr; }
    OPB_CUDA(ctx, cudaMalloc(reinterpret_cast<void**>(&ctx->precise_mid), need * sizeof(float)));
    ctx->precise_mid_cap = need;
  }
  float* mid = ctx->precise_mid;
  const float scale = (scale_index == n_scales - 1) ? static_cast<float>(n_scales) : 0.f;   // divisor of the last pass (0 = none)
  for (int which = 0; which < 2; ++which) {
    const int C = which ? 19 : 38;
    const float* lo = which ? ch->heat_lo : ch->paf_lo;
    float* acc = which ? ws->heat : ws->pafs;
    dim3 block(32, 8);
    dim3 g1((ch_w + 31) / 32, (ch_h + 7) / 8, C);
    resize_cubic_kernel<<<g1, block, 0, ctx->stream>>>(lo, C, h8, w8, mid, ph, pw, ch_h, ch_w, 0, 0.f);
    dim3 g2((ws->W + 31) / 32, (ws->H + 7) / 8, C);
    resize_cubic_kernel<<<g2, block, 0, ctx->stream>>>(mid, C, ch_h, ch_w, acc, ws->H, ws->W, ws->H, ws->W,
                                                       scale_index > 0 ? 1 : 0, scale);
    ctx->launches += 2;
  }
  OPB_CUDA(ctx, cudaGetLastError());
  return OPB_OK;
}

int opb_precise_add_scale(opb_ctx* ctx, const uint8_t* img, int img_loc, int ph, int pw, int pad_h, int pad_w,
                          int scale_index, int n_scales) {
  if (!ctx || !img) return OPB_ERR_ARG;
  PostWs* ws = ctx->last_post;
  if (!ws || ws->N != 1) OPB_FAIL(ctx, OPB_ERR_STATE, "opb_precise_begin was not called");
  cudaSetDevice(ctx->device);
  Chain* ch = nullptr;
  int rc = get_chain(ctx, 1, ph, pw, &ch);
  if (rc) return rc;
  if ((rc = copy_in(ctx, ch->img_u8, img, static_cast<size_t>(ph) * pw * 3, img_loc))) return rc;
  return precise_accumulate(ctx, ws, ch, ph, pw, pad_h, pad_w, scale_index, n_scales);
}

int opb_precise_add_scale_unpadded(opb_ctx* ctx, const uint8_t* img, int img_loc, int h, int w, int stride,
                                   const uint8_t pad_value[3], int scale_index, int n_scales) {
  if (!ctx || !img || !pad_value || h <= 0 || w <= 0 || stride <= 0) return OPB_ERR_ARG;
  PostWs* ws = ctx->last_post;
  if (!ws || ws->N != 1) OPB_FAIL(ctx, OPB_ERR_STATE, "opb_precise_begin was not called");
  cudaSetDevice(ctx->device);
  const int pad_h = (stride - h % stride) % stride, pad_w = (stride - w % stride) % stride;     // :50-51
  const int ph = h + pad_h, pw = w + pad_w;
  Chain* ch = nullptr;
  int rc = get_chain(ctx, 1, ph, pw, &ch);
  if (rc) return rc;
  const size_t in_b = static_cast<size_t>(h) * w * 3;
  const uint8_t* d_src = img;
  if (img_loc == OPB_HOST) {
    if ((rc = ensure_ingest(ctx, in_b + 512))) return rc;
    if ((rc = copy_in(ctx, ctx->ingest_buf, img, in_b, OPB_HOST))) return rc;
    d_src = ctx->ingest_buf;
  }
  dim3 block(32, 8), grid((pw + 31) / 32, (ph + 7) / 8);
  pad_image_u8_kernel<<<grid, block, 0, ctx->stream>>>(d_src, h, w, ch->img_u8, ph, pw, pad_value[0], pad_value[1],
                                                       pad_value[2]);
  ctx->launches++;
  OPB_CUDA(ctx, cudaGetLastError());
  return precise_accumulate(ctx, ws, ch, ph, pw, pad_h, pad_w, scale_index, n_scales);
}

int opb_precise_add_scale_orig(opb_ctx* ctx, const uint8_t* orig, int img_loc, int orig_h, int orig_w, int h, int w,
                               int stride, const uint8_t pad_value[3], int scale_index, int n_scales) {
  if (!ctx || !orig || !pad_value || orig_h <= 0 || orig_w <= 0 || h <= 0 || w <= 0 || stride <= 0) return OPB_ERR_ARG;
  PostWs* ws = ctx->last_post;
  if (!ws || ws->N != 1) OPB_FAIL(ctx, OPB_ERR_STATE, "opb_precise_begin was not called");
  cudaSetDevice(ctx->device);
  const size_t in_b = static_cast<size_t>(orig_h) * orig_w * 3, mid_b = static_cast<size_t>(h) * w * 3;
  const size_t mid_off = (in_b + 255) & ~size_t(255);
  int rc = ensure_ingest(ctx, mid_off + mid_b + 512);
  if (rc) return rc;
  const uint8_t* d_src = orig;
  if (img_loc == OPB_HOST) {
    if ((rc = copy_in(ctx, ctx->ingest_buf, orig, in_b, OPB_HOST))) return rc;
    d_src = ctx->ingest_buf;
  }
  uint8_t* d_mid = ctx->ingest_buf + mid_off;
  if ((rc = launch_resize_u8(ctx, d_src, 1, orig_h, orig_w, d_mid, h, w, true))) return rc;   // :443
  return opb_precise_add_scale_unpadded(ctx, d_mid, OPB_DEVICE, h, w, stride, pad_value, scale_index, n_scales);
}

int opb_precise_finish(opb_ctx* ctx, double img_len, opb_image_header* header_out, opb_person* persons_out,
                       int out_loc) {
  if (!ctx || !header_out || !persons_out) return OPB_ERR_ARG;
  PostWs* ws = ctx->last_post;
  if (!ws || ws->N != 1) OPB_FAIL(ctx, OPB_ERR_STATE, "opb_precise_begin was not called");
  cudaSetDevice(ctx->device);
  int rc;
  if ((rc = launch_peaks(ctx, ws, ws->heat, 1, 19, ws->H, ws->W))) return rc;
  if ((rc = launch_connections(ctx, ws, ws->pafs, 1, ws->H, ws->W, img_len))) return rc;
  if ((rc = launch_group(ctx, ws, 1, true))) return rc;
  if ((rc = copy_out(ctx, header_out, ws->headers, sizeof(ImageHeader), out_loc))) return rc;
  if ((rc = copy_out(ctx, persons_out, ws->persons, sizeof(PersonOut) * ctx->prm.max_persons, out_loc))) return rc;
  OPB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return OPB_OK;
}

int opb_download_maps(opb_ctx* ctx, float* pafs_out, float* heat_out, int out_loc) {
  if (!ctx) return OPB_ERR_ARG;
  PostWs* ws = ctx->last_post;
  if (!ws) OPB_FAIL(ctx, OPB_ERR_STATE, "no post-process workspace");
  cudaSetDevice(ctx->device);
  int rc;
  const size_t plane = static_cast<size_t>(ws->H) * ws->W * 4;
  if (pafs_out && (rc = copy_out(ctx, pafs_out, ws->pafs, plane * 38, out_loc))) return rc;
  if (heat_out && (rc = copy_out(ctx, heat_out, ws->heat, plane * 19, out_loc))) return rc;
  OPB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return OPB_OK;
}

// ---- draw_person_pose on the device (pose_detector.py:520-553; csrc/overlay.cuh) -------------------------------
static OverlayTables overlay_tables(const opb_ctx* ctx) {
  // limb_colors / joint_colors of pose_detector.py:523-535, written into channels 0,1,2 as given
  static const uint8_t kLimb[OV_LIMBS][3] = {
      {0, 255, 0}, {0, 255, 85}, {0, 255, 170}, {0, 255, 255}, {0, 170, 255}, {0, 85, 255}, {255, 0, 0},
      {255, 85, 0}, {255, 170, 0}, {255, 255, 0}, {255, 0, 85}, {170, 255, 0}, {85, 255, 0}, {170, 0, 255},
      {0, 0, 255}, {0, 0, 255}, {255, 0, 255}, {170, 0, 255}, {255, 0, 170}};
  static const uint8_t kJoint[OV_JOINTS][3] = {
      {255, 0, 0}, {255, 85, 0}, {255, 170, 0}, {255, 255, 0}, {170, 255, 0}, {85, 255, 0}, {0, 255, 0},
      {0, 255, 85}, {0, 255, 170}, {0, 255, 255}, {0, 170, 255}, {0, 85, 255}, {0, 0, 255}, {85, 0, 255},
      {170, 0, 255}, {255, 0, 255}, {255, 0, 170}, {255, 0, 85}};
  OverlayTables tb;
  for (int l = 0; l < OV_LIMBS; ++l) {
    tb.limb_a[l] = ctx->prm.limbs[l][0];
    tb.limb_b[l] = ctx->prm.limbs[l][1];
    for (int c = 0; c < 3; ++c) tb.limb_color[l][c] = kLimb[l][c];
  }
  for (int j = 0; j < OV_JOINTS; ++j)
    for (int c = 0; c < 3; ++c) tb.joint_color[j][c] = kJoint[j][c];
  // params['face_line_indices'] (entity.py:130-140): polylines over keypoint ranges, the eyes and lips closed
  static const int kFaceChains[9][3] = {{0, 16, 0}, {17, 21, 0}, {22, 26, 0}, {27, 30, 0}, {31, 35, 0},
                                        {36, 41, 1}, {42, 47, 1}, {48, 59, 1}, {60, 67, 1}};
  int n = 0;
  for (const auto& ch : kFaceChains) {
    for (int k = ch[0]; k < ch[1]; ++k, ++n) { tb.face_line[n][0] = static_cast<uint8_t>(k); tb.face_line[n][1] = static_cast<uint8_t>(k + 1); }
    if (ch[2]) { tb.face_line[n][0] = static_cast<uint8_t>(ch[1]); tb.face_line[n][1] = static_cast<uint8_t>(ch[0]); ++n; }
  }
  // params['fingers_indices'] (entity.py:145-151): wrist 0, then four joints per finger; finger_colors of
  // hand_detector.py:93-99, the face colour of face_detector.py:86,95, the box colour of demo.py:40
  static const uint8_t kFinger[OV_FINGERS][3] = {{0, 0, 255}, {0, 255, 255}, {0, 255, 0}, {255, 0, 0}, {255, 0, 255}};
  for (int f = 0; f < OV_FINGERS; ++f) {
    for (int s = 0; s < OV_FINGER_SEGS; ++s) {
      tb.finger[f][s][0] = static_cast<uint8_t>(s == 0 ? 0 : 4 * f + s);
      tb.finger[f][s][1] = static_cast<uint8_t>(4 * f + s + 1);
    }
    for (int c = 0; c < 3; ++c) tb.finger_color[f][c] = kFinger[f][c];
  }
  for (int c = 0; c < 3; ++c) {
    tb.face_color[c] = c < 2 ? 255 : 0;
    tb.rect_color[c] = 255;
  }
  return tb;
}

static int ov_reserve(opb_ctx* ctx, size_t need) {
  if (ctx->ov_bytes >= need) return OPB_OK;
  if (ctx->ov_buf) { cudaStreamSynchronize(ctx->stream); cudaFree(ctx->ov_buf); ctx->ov_buf = nullptr; ctx->ov_bytes = 0; }
  OPB_CUDA(ctx, cudaMalloc(reinterpret_cast<void**>(&ctx->ov_buf), need));
  ctx->ov_bytes = need;
  return OPB_OK;
}

// poses: device int [n_poses][18][3] when from_records == nullptr; otherwise the records of one image are converted first
static int overlay_run(opb_ctx* ctx, const uint8_t* img, int img_loc, int h, int w, const int32_t* host_poses, int n_poses,
                       const PersonOut* d_records, double sx, double sy, uint8_t* out, int out_loc) {
  cudaSetDevice(ctx->device);
  const size_t px = static_cast<size_t>(h) * w, img_b = (px * 3 + 255) & ~size_t(255);
  const size_t prio_b = (px * 4 + 255) & ~size_t(255), poses_b = (static_cast<size_t>(n_poses > 0 ? n_poses : 1) * OV_JOINTS * 3 * 4 + 255) & ~size_t(255);
  const size_t need = 2 * img_b + prio_b + poses_b + 256;
  int rc;
  if ((rc = ov_reserve(ctx, need))) return rc;
  uint8_t* d_in = ctx->ov_buf;
  uint8_t* d_out = ctx->ov_buf + img_b;
  unsigned int* d_prio = reinterpret_cast<unsigned int*>(ctx->ov_buf + 2 * img_b);
  int* d_poses = reinterpret_cast<int*>(ctx->ov_buf + 2 * img_b + prio_b);
  int* d_bad = reinterpret_cast<int*>(ctx->ov_buf + 2 * img_b + prio_b + poses_b);
  const uint8_t* d_src = img;
  if (img_loc == OPB_HOST) {
    if ((rc = copy_in(ctx, d_in, img, px * 3, OPB_HOST))) return rc;
    d_src = d_in;
  }
  uint8_t* d_dst = (out_loc == OPB_HOST) ? d_out : out;
  OPB_CUDA(ctx, cudaMemsetAsync(d_prio, 0, px * 4, ctx->stream));
  OPB_CUDA(ctx, cudaMemsetAsync(d_bad, 0, 4, ctx->stream));
  const OverlayTables tb = overlay_tables(ctx);
  if (n_poses > 0) {
    if (d_records) {
      const int* base = reinterpret_cast<const int*>(d_records);
      const int stride = static_cast<int>(sizeof(PersonOut) / 4), off_id = 4, off_x = 4 + OPB_N_JOINTS, off_y = 4 + 2 * OPB_N_JOINTS;
      overlay_poses_from_records_kernel<<<(n_poses * OV_JOINTS + 127) / 128, 128, 0, ctx->stream>>>(
          base + off_x, base + off_y, base + off_id, stride, n_poses, sx, sy, d_poses);
      ctx->launches++;
    } else {
      if ((rc = copy_in(ctx, d_poses, host_poses, static_cast<size_t>(n_poses) * OV_JOINTS * 3 * 4, OPB_HOST))) return rc;
    }
    const int n_prim = n_poses * (OV_LIMBS + OV_JOINTS);
    overlay_raster_kernel<<<(n_prim + 63) / 64, 64, 0, ctx->stream>>>(d_poses, n_poses, tb, d_prio, h, w, d_bad, nullptr, 0,
                                                                         nullptr);
    ctx->launches++;
  }
  overlay_paint_kernel<<<static_cast<unsigned>((px + 255) / 256), 256, 0, ctx->stream>>>(d_src, d_prio, static_cast<int>(px), n_poses, tb, d_dst,
                                                                                        nullptr, 0);
  ctx->launches++;
  OPB_CUDA(ctx, cudaGetLastError());
  int bad = 0;
  OPB_CUDA(ctx, cudaMemcpyAsync(&bad, d_bad, 4, cudaMemcpyDeviceToHost, ctx->stream));
  if (out_loc == OPB_HOST && (rc = copy_out(ctx, out, d_dst, px * 3, OPB_HOST))) return rc;
  OPB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (bad) OPB_FAIL(ctx, OPB_ERR_ARG, "draw_person_pose: a joint lies outside the image");
  return OPB_OK;
}

int opb_draw_person_pose(opb_ctx* ctx, const uint8_t* img, int img_loc, int h, int w, const int32_t* poses, int n_poses,
                         uint8_t* out, int out_loc) {
  if (!ctx || !img || !out || h <= 0 || w <= 0 || n_poses < 0 || (n_poses > 0 && !poses)) return OPB_ERR_ARG;
  return overlay_run(ctx, img, img_loc, h, w, poses, n_poses, nullptr, 1.0, 1.0, out, out_loc);
}

int opb_draw_last_result(opb_ctx* ctx, int image_index, const uint8_t* img, int img_loc, int h, int w, double sx, double sy,
                         uint8_t* out, int out_loc) {
  if (!ctx || !img || !out || h <= 0 || w <= 0) return OPB_ERR_ARG;
  PostWs* ws = ctx->last_post;
  if (!ws || image_index < 0 || image_index >= ws->N) OPB_FAIL(ctx, OPB_ERR_STATE, "no result for that image");
  cudaSetDevice(ctx->device);
  ImageHeader hd;
  OPB_CUDA(ctx, cudaMemcpyAsync(&hd, ws->headers + image_index, sizeof(hd), cudaMemcpyDeviceToHost, ctx->stream));
  OPB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (hd.status != 0) OPB_FAIL(ctx, hd.status, "the image's result carries an error status");
  return overlay_run(ctx, img, img_loc, h, w, nullptr, hd.n_persons,
                     ws->persons + static_cast<size_t>(image_index) * ctx->prm.max_persons, sx, sy, out, out_loc);
}

// Every part's kind, point range, box and present keypoints checked before the raster kernel reads them unchecked:
// OPB_ERR_ARG for an unknown kind, points past n_points, or a box or drawn keypoint coordinate beyond 2^20.
static int check_parts(opb_ctx* ctx, const opb_part* parts, int n_parts, const int32_t* points, int n_points) {
  auto big = [](long long v) { return v < -(1ll << 20) || v > (1ll << 20); };   // keeps the rasterisers' ints in range
  for (int p = 0; p < n_parts; ++p) {
    const opb_part& pt = parts[p];
    const int count = pt.kind == OPB_PART_FACE ? OV_FACE_POINTS : pt.kind == OPB_PART_HAND ? OV_HAND_POINTS : -1;
    if (count < 0) OPB_FAIL(ctx, OPB_ERR_ARG, "draw_whole_body: unknown part kind");
    if (pt.first_point < 0 || static_cast<long long>(pt.first_point) + count > n_points)
      OPB_FAIL(ctx, OPB_ERR_ARG, "draw_whole_body: a part's points run past the point table");
    if (big(pt.left) || big(pt.top) || big(pt.right) || big(pt.bottom))
      OPB_FAIL(ctx, OPB_ERR_ARG, "draw_whole_body: a box coordinate exceeds 2^20 in magnitude");
    for (int k = 0; k < count; ++k) {
      const int32_t* a = points + 3 * (static_cast<long long>(pt.first_point) + k);
      if (a[2] != 0 && (big(a[0]) || big(a[1]) || big(static_cast<long long>(a[0]) + pt.left) ||
                        big(static_cast<long long>(a[1]) + pt.top)))
        OPB_FAIL(ctx, OPB_ERR_ARG, "draw_whole_body: a keypoint coordinate exceeds 2^20 in magnitude");
    }
  }
  return OPB_OK;
}

// ---- the whole-body picture of demo.py:28-57 on the device (face_detector.py:79-97, hand_detector.py:89-117;
// csrc/overlay.cuh): one upload of the frame and of the tables, one raster and one paint launch, one download
int opb_draw_whole_body(opb_ctx* ctx, const uint8_t* img, int img_loc, int h, int w, const int32_t* poses, int n_poses,
                        const opb_part* parts, int n_parts, const int32_t* points, int n_points, uint8_t* out, int out_loc) {
  if (!ctx) return OPB_ERR_ARG;
  if (!img || !out || h <= 0 || w <= 0 || n_poses < 0 || n_parts < 0 || n_points < 0 || (n_poses > 0 && !poses) ||
      (n_parts > 0 && !parts) || (n_points > 0 && !points))
    OPB_FAIL(ctx, OPB_ERR_ARG, "draw_whole_body: bad image, pose, part or point arguments");
  const long long n_prim = static_cast<long long>(n_poses) * (OV_LIMBS + OV_JOINTS) + static_cast<long long>(n_parts) * OV_PART_STRIDE;
  if (n_prim > (1ll << 30)) OPB_FAIL(ctx, OPB_ERR_ARG, "draw_whole_body: too many poses / parts");
  // the raster kernel reads everything below without bounds checks: validate it all before anything is enqueued
  for (long long k = 0; k < static_cast<long long>(n_poses) * OV_JOINTS; ++k) {
    const int32_t* a = poses + 3 * k;
    if (a[2] != 0 && (a[0] < 0 || a[0] >= w || a[1] < 0 || a[1] >= h))
      OPB_FAIL(ctx, OPB_ERR_ARG, "draw_whole_body: a joint lies outside the image");
  }
  int rc;
  if ((rc = check_parts(ctx, parts, n_parts, points, n_points))) return rc;
  cudaSetDevice(ctx->device);
  // scratch: [frame in | frame out | priority plane | tables: int poses | parts | points]
  const size_t px = static_cast<size_t>(h) * w, img_b = (px * 3 + 255) & ~size_t(255), prio_b = (px * 4 + 255) & ~size_t(255);
  const size_t poses_n = static_cast<size_t>(n_poses) * OV_JOINTS * 3, parts_n = static_cast<size_t>(n_parts) * 6;
  const size_t tab_n = poses_n + parts_n + static_cast<size_t>(n_points) * 3;
  static_assert(sizeof(opb_part) == 6 * sizeof(int32_t) && sizeof(OvPart) == sizeof(opb_part), "opb_part layout");
  if ((rc = ov_reserve(ctx, 2 * img_b + prio_b + tab_n * 4 + 256))) return rc;
  uint8_t* d_in = ctx->ov_buf;
  uint8_t* d_out = ctx->ov_buf + img_b;
  unsigned int* d_prio = reinterpret_cast<unsigned int*>(ctx->ov_buf + 2 * img_b);
  int* d_tab = reinterpret_cast<int*>(ctx->ov_buf + 2 * img_b + prio_b);
  int* d_bad = d_tab + tab_n;                 // never raised: the joints were checked above
  const uint8_t* d_src = img;
  if (img_loc == OPB_HOST) {
    if ((rc = copy_in(ctx, d_in, img, px * 3, OPB_HOST))) return rc;
    d_src = d_in;
  }
  uint8_t* d_dst = (out_loc == OPB_HOST) ? d_out : out;
  if (tab_n) {
    std::vector<int32_t> tab(tab_n);
    std::copy(poses, poses + poses_n, tab.begin());
    if (parts_n) std::memcpy(tab.data() + poses_n, parts, parts_n * 4);
    std::copy(points, points + static_cast<size_t>(n_points) * 3, tab.begin() + poses_n + parts_n);
    if ((rc = copy_in(ctx, d_tab, tab.data(), tab_n * 4, OPB_HOST))) return rc;
  }
  const int* d_poses = d_tab;
  const OvPart* d_parts = reinterpret_cast<const OvPart*>(d_tab + poses_n);
  const int* d_points = d_tab + poses_n + parts_n;
  OPB_CUDA(ctx, cudaMemsetAsync(d_prio, 0, px * 4, ctx->stream));
  const OverlayTables tb = overlay_tables(ctx);
  if (n_prim > 0) {
    overlay_raster_kernel<<<static_cast<unsigned>((n_prim + 63) / 64), 64, 0, ctx->stream>>>(d_poses, n_poses, tb, d_prio, h, w, d_bad,
                                                                                          d_parts, n_parts, d_points);
    ctx->launches++;
  }
  overlay_paint_kernel<<<static_cast<unsigned>((px + 255) / 256), 256, 0, ctx->stream>>>(d_src, d_prio, static_cast<int>(px), n_poses, tb, d_dst,
                                                                                        d_parts, 1);
  ctx->launches++;
  OPB_CUDA(ctx, cudaGetLastError());
  if (out_loc == OPB_HOST && (rc = copy_out(ctx, out, d_dst, px * 3, OPB_HOST))) return rc;
  OPB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return OPB_OK;
}

static int launch_resize_u8(opb_ctx* ctx, const uint8_t* d_src, int n, int h0, int w0, uint8_t* d_dst, int h, int w,
                            bool cubic) {
  if (h0 == h && w0 == w) {
    OPB_CUDA(ctx, cudaMemcpyAsync(d_dst, d_src, static_cast<size_t>(n) * h * w * 3, cudaMemcpyDeviceToDevice, ctx->stream));
    return OPB_OK;
  }
  const double sx = 1.0 / (static_cast<double>(w) / w0), sy = 1.0 / (static_cast<double>(h) / h0);
  dim3 grid((w + 31) / 32, (h + 7) / 8, n), block(32, 8);
  if (cubic) resize_cubic_u8_kernel<<<grid, block, 0, ctx->stream>>>(d_src, h0, w0, d_dst, h, w, sx, sy);
  else resize_linear_u8_kernel<<<grid, block, 0, ctx->stream>>>(d_src, h0, w0, d_dst, h, w, sx, sy);
  ctx->launches++;
  OPB_CUDA(ctx, cudaGetLastError());
  return OPB_OK;
}

static int ensure_ingest(opb_ctx* ctx, size_t bytes) {
  if (ctx->ingest_bytes >= bytes) return OPB_OK;
  if (ctx->ingest_buf) { cudaStreamSynchronize(ctx->stream); cudaFree(ctx->ingest_buf); ctx->ingest_buf = nullptr; }
  OPB_CUDA(ctx, cudaMalloc(reinterpret_cast<void**>(&ctx->ingest_buf), bytes));
  ctx->ingest_bytes = bytes;
  return OPB_OK;
}

static int resize_u8_entry(opb_ctx* ctx, const uint8_t* src, int src_loc, int n, int h0, int w0, uint8_t* dst,
                           int dst_loc, int h, int w, bool cubic);

int opb_resize_linear_u8(opb_ctx* ctx, const uint8_t* src, int src_loc, int n, int h0, int w0, uint8_t* dst,
                         int dst_loc, int h, int w) {
  return resize_u8_entry(ctx, src, src_loc, n, h0, w0, dst, dst_loc, h, w, false);
}

int opb_resize_cubic_u8(opb_ctx* ctx, const uint8_t* src, int src_loc, int n, int h0, int w0, uint8_t* dst,
                        int dst_loc, int h, int w) {
  return resize_u8_entry(ctx, src, src_loc, n, h0, w0, dst, dst_loc, h, w, true);
}

static int resize_u8_entry(opb_ctx* ctx, const uint8_t* src, int src_loc, int n, int h0, int w0, uint8_t* dst,
                           int dst_loc, int h, int w, bool cubic) {
  if (!ctx || !src || !dst || n <= 0 || h0 <= 0 || w0 <= 0 || h <= 0 || w <= 0) return OPB_ERR_ARG;
  cudaSetDevice(ctx->device);
  const size_t in_b = static_cast<size_t>(n) * h0 * w0 * 3, out_b = static_cast<size_t>(n) * h * w * 3;
  int rc = ensure_ingest(ctx, in_b + out_b + 512);
  if (rc) return rc;
  const uint8_t* d_src = src;
  if (src_loc == OPB_HOST) {
    if ((rc = copy_in(ctx, ctx->ingest_buf, src, in_b, OPB_HOST))) return rc;
    d_src = ctx->ingest_buf;
  }
  uint8_t* d_dst = (dst_loc == OPB_HOST) ? ctx->ingest_buf + ((in_b + 255) & ~size_t(255)) : dst;
  if ((rc = launch_resize_u8(ctx, d_src, n, h0, w0, d_dst, h, w, cubic))) return rc;
  if (dst_loc == OPB_HOST && (rc = copy_out(ctx, dst, d_dst, out_b, OPB_HOST))) return rc;
  OPB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return OPB_OK;
}

int opb_detect_image(opb_ctx* ctx, const uint8_t* img, int img_loc, int orig_h, int orig_w, int in_h, int in_w,
                     int map_h, int map_w, double img_len, opb_image_header* header_out, opb_person* persons_out,
                     int out_loc) {
  if (!ctx || !img || !header_out || !persons_out) return OPB_ERR_ARG;
  cudaSetDevice(ctx->device);
  Chain* ch = nullptr;
  int rc = get_chain(ctx, 1, in_h, in_w, &ch);
  if (rc) return rc;
  const size_t in_b = static_cast<size_t>(orig_h) * orig_w * 3;
  const uint8_t* d_src = img;
  if (img_loc == OPB_HOST) {
    if ((rc = ensure_ingest(ctx, in_b + 512))) return rc;
    if ((rc = copy_in(ctx, ctx->ingest_buf, img, in_b, OPB_HOST))) return rc;
    d_src = ctx->ingest_buf;
  }
  if ((rc = launch_resize_u8(ctx, d_src, 1, orig_h, orig_w, ch->img_u8, in_h, in_w))) return rc;
  // frames are now resident at network-input size: reuse the batch path in place
  return opb_detect_batch(ctx, ch->img_u8, OPB_DEVICE, 1, in_h, in_w, map_h, map_w, img_len, nullptr, nullptr, header_out,
                          persons_out, out_loc);
}

int opb_stream_submit(opb_ctx* ctx, const uint8_t* frames, int frames_loc, int n, int orig_h, int orig_w, int in_h, int in_w,
                      int map_h, int map_w, double img_len, const float* inject_paf, const float* inject_heat, int slot) {
  if (!ctx || !frames || n <= 0 || slot < 0 || slot > 1) return OPB_ERR_ARG;
  cudaSetDevice(ctx->device);
  auto& sl = ctx->slots[slot];
  if (sl.busy) OPB_FAIL(ctx, OPB_ERR_ARG, "opb_stream_submit: slot still holds an uncollected batch");
  Chain* ch = nullptr;
  PostWs* ws = nullptr;
  int rc;
  if (slot == 1 && ctx->two_streams && !ctx->stream_b)
    OPB_CUDA(ctx, cudaStreamCreateWithFlags(&ctx->stream_b, cudaStreamNonBlocking));
  // slot 1 runs on its own stream with its own activations, so the tail / launch gaps of one slot's kernels are
  // filled by the other slot's; everything below launches on ctx->stream, which is swapped for the call
  struct SlotScope {
    opb_ctx* c; cudaStream_t saved; int saved_slot;
    SlotScope(opb_ctx* c_, int slot_) : c(c_), saved(c_->stream), saved_slot(c_->cur_slot) {
      if (slot_ == 1 && c->two_streams) { c->stream = c->stream_b; c->cur_slot = 1; }
    }
    ~SlotScope() { c->stream = saved; c->cur_slot = saved_slot; }
  } scope(ctx, slot);
  if ((rc = get_chain(ctx, n, in_h, in_w, &ch))) return rc;
  if ((rc = get_post(ctx, n, map_h, map_w, &ws))) return rc;
  if (!ctx->copy_stream) OPB_CUDA(ctx, cudaStreamCreateWithFlags(&ctx->copy_stream, cudaStreamNonBlocking));
  if (!sl.done) {
    OPB_CUDA(ctx, cudaEventCreateWithFlags(&sl.h2d_done, cudaEventDisableTiming));
    OPB_CUDA(ctx, cudaEventCreateWithFlags(&sl.done, cudaEventDisableTiming));
  }
  const size_t in_b = static_cast<size_t>(n) * orig_h * orig_w * 3;
  const size_t res_b = n * (sizeof(ImageHeader) + sizeof(PersonOut) * static_cast<size_t>(ctx->prm.max_persons));
  const bool resident = frames_loc == OPB_DEVICE;   // frames already in HBM: used in place, no upload
  if (!resident && sl.d_bytes < in_b) {
    if (sl.d_frames) { OPB_CUDA(ctx, cudaStreamSynchronize(ctx->stream)); cudaFree(sl.d_frames); sl.d_frames = nullptr; }
    OPB_CUDA(ctx, cudaMalloc(reinterpret_cast<void**>(&sl.d_frames), in_b));
    sl.d_bytes = in_b;
  }
  if (sl.r_bytes < res_b) {
    if (sl.h_result) cudaFreeHost(sl.h_result);
    OPB_CUDA(ctx, cudaMallocHost(reinterpret_cast<void**>(&sl.h_result), res_b));
    sl.r_bytes = res_b;
  }
  // pageable caller memory goes through the slot's pinned staging buffer so the H2D copy is truly asynchronous
  const uint8_t* h_src = frames;
  cudaPointerAttributes at{};
  const bool pinned = resident || (cudaPointerGetAttributes(&at, frames) == cudaSuccess && at.type == cudaMemoryTypeHost);
  cudaGetLastError();
  if (!pinned) {
    if (sl.h_bytes < in_b) {
      if (sl.h_frames) cudaFreeHost(sl.h_frames);
      OPB_CUDA(ctx, cudaMallocHost(reinterpret_cast<void**>(&sl.h_frames), in_b));
      sl.h_bytes = in_b;
    }
    memcpy(sl.h_frames, frames, in_b);
    h_src = sl.h_frames;
  }
  // the slot's previous batch was collected (sl.done reached), so its device frames are free to overwrite
  const uint8_t* d_frames = resident ? frames : sl.d_frames;
  if (!resident) {
    OPB_CUDA(ctx, cudaMemcpyAsync(sl.d_frames, h_src, in_b, cudaMemcpyHostToDevice, ctx->copy_stream));
    OPB_CUDA(ctx, cudaEventRecord(sl.h2d_done, ctx->copy_stream));
    OPB_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, sl.h2d_done, 0));
  }
  // everything between the upload and the `done` event: [resize] + pipeline + record download
  auto body = [&]() -> int {
    int r;
    if (orig_h == in_h && orig_w == in_w) {
      ch->img_u8_src = d_frames;
    } else {
      if ((r = launch_resize_u8(ctx, d_frames, n, orig_h, orig_w, ch->img_u8, in_h, in_w))) return r;
      ch->img_u8_src = nullptr;
    }
    if ((r = run_pipeline(ctx, ch, ws, n, in_h, in_w, map_h, map_w, img_len, inject_paf, inject_heat))) return r;
    if ((r = copy_out(ctx, sl.h_result, ws->headers, sizeof(ImageHeader) * n, OPB_HOST))) return r;
    return copy_out(ctx, sl.h_result + sizeof(ImageHeader) * n, ws->persons,
                    sizeof(PersonOut) * n * static_cast<size_t>(ctx->prm.max_persons), OPB_HOST);
  };
  const opb_ctx::StreamSlot::Key key{n, orig_h, orig_w, in_h, in_w, map_h, map_w, img_len, inject_paf, inject_heat,
                                     d_frames, sl.h_result, ch, ws, ctx->cache_epoch};
  const bool graphs = ctx->use_graphs && !ctx->profile;
  if (!(key == sl.key)) {
    if (sl.gexec) { cudaGraphExecDestroy(sl.gexec); sl.gexec = nullptr; }
    sl.key = key;
    sl.key_seen = 0;
  }
  if (graphs && sl.gexec) {
    OPB_CUDA(ctx, cudaGraphLaunch(sl.gexec, ctx->stream));
    ctx->launches += sl.graph_launches;
  } else if (graphs && sl.key_seen >= 1) {
    // second submit of this combination: capture the launch sequence, then run it as a graph
    const int64_t l0 = ctx->launches;
    OPB_CUDA(ctx, cudaStreamBeginCapture(ctx->stream, cudaStreamCaptureModeRelaxed));
    rc = body();
    cudaGraph_t graph = nullptr;
    const cudaError_t ce = cudaStreamEndCapture(ctx->stream, &graph);
    if (rc) { if (graph) cudaGraphDestroy(graph); return rc; }
    if (ce != cudaSuccess || !graph) OPB_FAIL(ctx, OPB_ERR_CUDA, std::string("stream capture failed: ") + cudaGetErrorString(ce));
    const cudaError_t ie = cudaGraphInstantiate(&sl.gexec, graph, 0);
    cudaGraphDestroy(graph);
    if (ie != cudaSuccess) { sl.gexec = nullptr; OPB_FAIL(ctx, OPB_ERR_CUDA, std::string("cudaGraphInstantiate: ") + cudaGetErrorString(ie)); }
    sl.graph_launches = ctx->launches - l0;
    OPB_CUDA(ctx, cudaGraphLaunch(sl.gexec, ctx->stream));
  } else {
    if ((rc = body())) return rc;
  }
  sl.key_seen++;
  OPB_CUDA(ctx, cudaEventRecord(sl.done, ctx->stream));
  sl.n = n;
  sl.post = ws;
  sl.busy = true;
  return OPB_OK;
}

// ---- the one collective of the path (SURVEY.md 8e): all-gather of the fixed-size result records --------------------
// NCCL is resolved at run time from the library the process already carries (torch loads libnccl.so.2; a stand-alone
// C program links or preloads it): no link-time dependency, and a box without NCCL can still use everything else.
namespace {
struct NcclApi {
  int (*GetUniqueId)(void*) = nullptr;
  int (*CommInitRank)(void**, int, OpbNcclId, int) = nullptr;
  int (*CommDestroy)(void*) = nullptr;
  int (*AllGather)(const void*, void*, size_t, int, void*, cudaStream_t) = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
  bool ok = false;
  std::string why;
};
NcclApi& nccl_api() {
  static NcclApi api;
  static bool tried = false;
  if (tried) return api;
  tried = true;
  void* h = nullptr;
  const char* names[] = {getenv("OPB_NCCL_LIB"), "libnccl.so.2", "libnccl.so"};
  for (const char* n : names) {
    if (!n || !*n) continue;
    h = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
    if (h) break;
  }
  if (!h) { api.why = "libnccl.so.2 not found (set OPB_NCCL_LIB)"; return api; }
  api.GetUniqueId = reinterpret_cast<int (*)(void*)>(dlsym(h, "ncclGetUniqueId"));
  api.CommInitRank = reinterpret_cast<int (*)(void**, int, OpbNcclId, int)>(dlsym(h, "ncclCommInitRank"));
  api.CommDestroy = reinterpret_cast<int (*)(void*)>(dlsym(h, "ncclCommDestroy"));
  api.AllGather = reinterpret_cast<int (*)(const void*, void*, size_t, int, void*, cudaStream_t)>(dlsym(h, "ncclAllGather"));
  api.GetErrorString = reinterpret_cast<const char* (*)(int)>(dlsym(h, "ncclGetErrorString"));
  api.ok = api.GetUniqueId && api.CommInitRank && api.CommDestroy && api.AllGather;
  if (!api.ok) api.why = "libnccl lacks ncclGetUniqueId / ncclCommInitRank / ncclCommDestroy / ncclAllGather";
  return api;
}
}  // namespace

int opb_nccl_unique_id(uint8_t id_out[128]) {
  if (!id_out) return OPB_ERR_ARG;
  NcclApi& a = nccl_api();
  if (!a.ok) { g_create_error = a.why; return OPB_ERR_UNSUPPORTED; }
  OpbNcclId id;
  const int r = a.GetUniqueId(&id);
  if (r) { g_create_error = std::string("ncclGetUniqueId: ") + (a.GetErrorString ? a.GetErrorString(r) : "error"); return OPB_ERR_CUDA; }
  std::memcpy(id_out, id.internal, 128);
  return OPB_OK;
}

int opb_nccl_comm_init(opb_ctx* ctx, void** comm_out, int world, int rank, const uint8_t id[128]) {
  if (!ctx || !comm_out || !id || world < 1 || rank < 0 || rank >= world) return OPB_ERR_ARG;
  NcclApi& a = nccl_api();
  if (!a.ok) OPB_FAIL(ctx, OPB_ERR_UNSUPPORTED, a.why);
  cudaSetDevice(ctx->device);
  OpbNcclId uid;
  std::memcpy(uid.internal, id, 128);
  void* comm = nullptr;
  const int r = a.CommInitRank(&comm, world, uid, rank);
  if (r) OPB_FAIL(ctx, OPB_ERR_CUDA, std::string("ncclCommInitRank: ") + (a.GetErrorString ? a.GetErrorString(r) : "error"));
  *comm_out = comm;
  return OPB_OK;
}

int opb_nccl_comm_destroy(void* comm) {
  NcclApi& a = nccl_api();
  if (!a.ok || !comm) return OPB_ERR_ARG;
  return a.CommDestroy(comm) ? OPB_ERR_CUDA : OPB_OK;
}

size_t opb_record_block_bytes(const opb_ctx* ctx, int n) {
  return ctx ? static_cast<size_t>(n) * (sizeof(ImageHeader) + sizeof(PersonOut) * static_cast<size_t>(ctx->prm.max_persons)) : 0;
}

int opb_allgather_results(opb_ctx* ctx, void* nccl_comm, int slot, void* gathered_dev) {
  if (!ctx || !nccl_comm || !gathered_dev || slot < 0 || slot > 1) return OPB_ERR_ARG;
  NcclApi& a = nccl_api();
  if (!a.ok) OPB_FAIL(ctx, OPB_ERR_UNSUPPORTED, a.why);
  cudaSetDevice(ctx->device);
  auto& sl = ctx->slots[slot];
  if (!sl.busy || !sl.post) OPB_FAIL(ctx, OPB_ERR_STATE, "opb_allgather_results: nothing submitted on this slot");
  cudaStream_t st = (slot == 1 && ctx->two_streams && ctx->stream_b) ? ctx->stream_b : ctx->stream;
  const PostWs* ws = static_cast<const PostWs*>(sl.post);
  // device-resident [headers | persons] of the slot's batch -> every rank's block, in rank order; no host hop
  const int r = a.AllGather(ws->headers, gathered_dev, opb_record_block_bytes(ctx, sl.n), 1 /* ncclUint8 */, nccl_comm, st);
  if (r) OPB_FAIL(ctx, OPB_ERR_CUDA, std::string("ncclAllGather: ") + (a.GetErrorString ? a.GetErrorString(r) : "error"));
  ctx->launches++;
  OPB_CUDA(ctx, cudaEventRecord(sl.done, st));       // opb_stream_collect / opb_stream_join now also cover the collective
  return OPB_OK;
}

int opb_stream_join(opb_ctx* ctx) {
  if (!ctx) return OPB_ERR_ARG;
  cudaSetDevice(ctx->device);
  for (auto& sl : ctx->slots)
    if (sl.busy && sl.done) OPB_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, sl.done, 0));
  return OPB_OK;
}

int opb_stream_collect(opb_ctx* ctx, int slot, opb_image_header* headers_out, opb_person* persons_out) {
  if (!ctx || slot < 0 || slot > 1 || !headers_out || !persons_out) return OPB_ERR_ARG;
  cudaSetDevice(ctx->device);
  auto& sl = ctx->slots[slot];
  if (!sl.busy) OPB_FAIL(ctx, OPB_ERR_ARG, "opb_stream_collect: nothing submitted on this slot");
  OPB_CUDA(ctx, cudaEventSynchronize(sl.done));
  sl.busy = false;
  memcpy(headers_out, sl.h_result, sizeof(ImageHeader) * sl.n);
  memcpy(persons_out, sl.h_result + sizeof(ImageHeader) * sl.n, sizeof(PersonOut) * sl.n * static_cast<size_t>(ctx->prm.max_persons));
  return OPB_OK;
}

// Grows the face / hand workspace to at least `floats` per map buffer, `records` arg-max records and `n_crops` table
// entries (keeping the larger of the old and the requested sizes).
static int kp_workspace(opb_ctx* ctx, size_t floats, int records, int n_crops, KpWs** out) {
  if (!ctx->kp_ws) ctx->kp_ws = new KpWs();
  KpWs* ws = ctx->kp_ws;
  if (ws->cap < floats || ws->records < records || ws->n_crops < n_crops) {
    OPB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    cudaFree(ws->up); cudaFree(ws->tmp); cudaFree(ws->res); cudaFreeHost(ws->h_res); cudaFree(ws->crops);
    ws->up = ws->tmp = nullptr; ws->res = nullptr; ws->h_res = nullptr; ws->crops = nullptr;
    const size_t cap = std::max(ws->cap, floats);
    const int rec = std::max(ws->records, records), nc = std::max(ws->n_crops, n_crops);
    ws->cap = 0; ws->records = 0; ws->n_crops = 0;
    OPB_CUDA(ctx, cudaMalloc(reinterpret_cast<void**>(&ws->up), cap * 4));
    OPB_CUDA(ctx, cudaMalloc(reinterpret_cast<void**>(&ws->tmp), cap * 4));
    OPB_CUDA(ctx, cudaMalloc(reinterpret_cast<void**>(&ws->res), sizeof(ChannelMax) * rec));
    OPB_CUDA(ctx, cudaMallocHost(reinterpret_cast<void**>(&ws->h_res), sizeof(ChannelMax) * rec));
    OPB_CUDA(ctx, cudaMalloc(reinterpret_cast<void**>(&ws->crops), sizeof(KpCrop) * nc));
    ws->cap = cap; ws->records = rec; ws->n_crops = nc;
  }
  *out = ws;
  return OPB_OK;
}

// Lays out the ragged workspace for `table` (h, w set): map offsets and tile numbers from host prefix sums.
// Returns the number of 32x8 tiles and the floats the maps of `planes` channels need.
static void kp_layout(std::vector<KpCrop>& table, int planes, long long* tiles, size_t* floats) {
  size_t off = 0;
  long long t = 0;
  for (KpCrop& c : table) {
    c.off = static_cast<long long>(off);
    c.tile0 = static_cast<int>(std::min<long long>(t, INT32_MAX));   // callers reject tables with more than 2^30 tiles
    off += static_cast<size_t>(planes) * c.h * c.w;
    t += static_cast<long long>((c.w + 31) / 32) * ((c.h + 7) / 8);
  }
  *tiles = t;
  *floats = off;
}

// One crop's arg-max records -> (x, y, conf) / valid, read the way compute_peaks_from_heatmaps reads them
// (face_detector.py:55-67).  Shared by the single-crop and the batched entry points.
static void kp_records_to_keypoints(const ChannelMax* res, int planes, int W, double thresh, double* out, int32_t* valid) {
  const float th = static_cast<float>(thresh);      // `max_value > thresh` with a float32 max_value compares in float32
  for (int c = 0; c < planes; ++c) {
    const ChannelMax& r = res[c];
    valid[c] = r.value > th ? 1 : 0;
    // np.array(np.where(g == m)).flatten() = [y0..yk-1, x0..xk-1]; the reference reads [1] as x and [0] as y
    const int y0 = r.key0 / W, x0 = r.key0 - y0 * W;
    out[c * 3 + 0] = r.count >= 2 ? static_cast<double>(r.key1 / W) : static_cast<double>(x0);
    out[c * 3 + 1] = static_cast<double>(y0);
    out[c * 3 + 2] = static_cast<double>(r.value);
  }
}

// Smooths the ragged maps in ws->up (both passes), takes every (crop, plane) maximum and enqueues the copy of the
// records to the pinned ws->h_res, without waiting.  ws->crops must already hold `table`.
static int kp_peaks_enqueue(opb_ctx* ctx, KpWs* ws, const std::vector<KpCrop>& table, int planes, int tiles) {
  const int n = static_cast<int>(table.size());
  dim3 block(32, 8), grid(tiles, planes);
  gauss_pass_ragged_kernel<0><<<grid, block, 0, ctx->stream>>>(ws->up, ws->tmp, ws->crops, n, ctx->taps);
  gauss_pass_ragged_kernel<1><<<grid, block, 0, ctx->stream>>>(ws->tmp, ws->up, ws->crops, n, ctx->taps);
  channel_argmax_ragged_kernel<<<dim3(planes, n), 256, 0, ctx->stream>>>(ws->up, ws->crops, ws->res);
  ctx->launches += 3;
  OPB_CUDA(ctx, cudaGetLastError());
  OPB_CUDA(ctx, cudaMemcpyAsync(ws->h_res, ws->res, sizeof(ChannelMax) * planes * n, cudaMemcpyDeviceToHost, ctx->stream));
  return OPB_OK;
}

// Waits for the records kp_peaks_enqueue asked for (one synchronisation), then the host conversion.
static int kp_peaks_collect(opb_ctx* ctx, KpWs* ws, const std::vector<KpCrop>& table, int planes, double thresh,
                            double* out, int32_t* valid) {
  OPB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  for (size_t i = 0; i < table.size(); ++i)
    kp_records_to_keypoints(ws->h_res + i * planes, planes, table[i].w, thresh, out + i * planes * 3,
                            valid + i * planes);
  return OPB_OK;
}

// Both halves: one copy of the records to the host, one synchronisation, then the host conversion.
static int kp_peaks(opb_ctx* ctx, KpWs* ws, const std::vector<KpCrop>& table, int planes, int tiles, double thresh,
                    double* out, int32_t* valid) {
  int rc = kp_peaks_enqueue(ctx, ws, table, planes, tiles);
  return rc ? rc : kp_peaks_collect(ctx, ws, table, planes, thresh, out, valid);
}

// Workspace and device crop table for the single-crop entry points: one [planes][h][w] map set at offset 0.
static int kp_single(opb_ctx* ctx, int planes, int h, int w, int mirror, std::vector<KpCrop>& table, int* tiles,
                     KpWs** ws) {
  KpCrop c{};
  c.h = h; c.w = w; c.flip = mirror ? 1 : 0;
  table.assign(1, c);
  size_t floats = 0;
  long long t = 0;
  kp_layout(table, planes, &t, &floats);
  if (t > (1 << 30)) OPB_FAIL(ctx, OPB_ERR_ARG, "maps too large");
  *tiles = static_cast<int>(t);
  int rc = kp_workspace(ctx, floats, planes, 1, ws);
  if (rc) return rc;
  OPB_CUDA(ctx, cudaMemcpyAsync((*ws)->crops, table.data(), sizeof(KpCrop), cudaMemcpyHostToDevice, ctx->stream));
  return OPB_OK;
}

int opb_keypoints_from_heatmaps(opb_ctx* ctx, const float* heat, int heat_loc, int planes, int h, int w, int mirror,
                                double thresh, double* out, int32_t* valid) {
  if (!ctx || !heat || !out || !valid || planes <= 0 || h <= 0 || w <= 0) return OPB_ERR_ARG;
  cudaSetDevice(ctx->device);
  KpWs* ws = nullptr;
  std::vector<KpCrop> table;
  int tiles = 0;
  int rc = kp_single(ctx, planes, h, w, mirror, table, &tiles, &ws);
  if (rc) return rc;
  if ((rc = copy_in(ctx, ws->up, heat, static_cast<size_t>(planes) * h * w * 4, heat_loc))) return rc;
  return kp_peaks(ctx, ws, table, planes, tiles, thresh, out, valid);
}

int opb_keypoints_detect(opb_ctx* ctx, const uint8_t* img, int img_loc, int img_h, int img_w, int net_size, int mirror,
                         double thresh, double* out, int32_t* valid, float* maps_out) {
  if (!ctx || !img || !out || !valid || img_h <= 0 || img_w <= 0) return OPB_ERR_ARG;
  if (!ctx->kp_out) OPB_FAIL(ctx, OPB_ERR_STATE, "this context holds the pose net: load FaceNet / HandNet weights first");
  cudaSetDevice(ctx->device);
  Chain* ch = nullptr;
  int rc = get_chain(ctx, 1, net_size, net_size, &ch);
  if (rc) return rc;
  const size_t in_b = static_cast<size_t>(img_h) * img_w * 3;
  const uint8_t* d_src = img;
  if (img_loc == OPB_HOST) {
    if ((rc = ensure_ingest(ctx, in_b + 512))) return rc;
    if ((rc = copy_in(ctx, ctx->ingest_buf, img, in_b, OPB_HOST))) return rc;
    d_src = ctx->ingest_buf;
  }
  // cv2.resize(crop, (368, 368)) (face_detector.py:31), bit-exact uint8 INTER_LINEAR on the device
  if ((rc = launch_resize_u8(ctx, d_src, 1, img_h, img_w, ch->img_u8, net_size, net_size))) return rc;
  ch->img_u8_src = nullptr;
  if ((rc = run_chain(ctx, ch, true))) return rc;
  const int planes = ctx->kp_out - 1;              // the last channel is background (face_detector.py:59)
  KpWs* ws = nullptr;
  std::vector<KpCrop> table;
  int tiles = 0;
  if ((rc = kp_single(ctx, planes, img_h, img_w, mirror, table, &tiles, &ws))) return rc;
  // F.resize_images(hs[-1], (crop_h, crop_w)) (face_detector.py:38)
  if ((rc = launch_upsample(ctx, ch->heat_lo, planes, net_size / 8, net_size / 8, ws->up, img_h, img_w))) return rc;
  if (maps_out && (rc = copy_out(ctx, maps_out, ws->up, static_cast<size_t>(planes) * img_h * img_w * 4, OPB_HOST))) return rc;
  return kp_peaks(ctx, ws, table, planes, tiles, thresh, out, valid);
}

// Batch slots of the next forward chunk for `remaining` crops: full chunks of kKpMaxChunk, then the remainder rounded
// up to a power of two, so that at most log2(kKpMaxChunk) + 1 chain shapes are ever built per net size.
static const int kKpMaxChunk = 16;
static int kp_chunk_slots(int remaining) {
  if (remaining >= kKpMaxChunk) return kKpMaxChunk;
  int p = 1;
  while (p < remaining) p <<= 1;
  return p;
}

// Fills in cv2.resize's inverse scales (canvas -> net_size, as launch_resize_u8 forms them) and the ragged layout of
// `table` (top, left, h, w, flip, vh, vw, frame set).  *tiles: the table's 32x8 tiles; *floats: its maps of `planes`.
static int kp_prepare_table(opb_ctx* ctx, std::vector<KpCrop>& table, int net_size, int planes, int* tiles,
                            size_t* floats) {
  for (KpCrop& c : table) {
    c.sx = 1.0 / (static_cast<double>(net_size) / c.w);
    c.sy = 1.0 / (static_cast<double>(net_size) / c.h);
  }
  long long t = 0;
  kp_layout(table, planes, &t, floats);
  if (t > (1 << 30) || *floats / planes > (1ull << 31)) OPB_FAIL(ctx, OPB_ERR_ARG, "crops too large for one call");
  *tiles = static_cast<int>(t);
  return OPB_OK;
}

// crop_image + flip + cv2.resize(crop, (net, net)) straight from the frames (face_detector.py:31) of the nc crops at
// d_crops (device table) into dst [slots][net][net][3]; the padding slots nc..slots-1 are zeroed.
static int kp_canvas_enqueue(opb_ctx* ctx, const uint8_t* d_frames, int frame_h, int frame_w, const KpCrop* d_crops,
                             int nc, int slots, uint8_t* dst, int net_size) {
  dim3 rgrid((net_size + 31) / 32, (net_size + 7) / 8, slots);
  crop_resize_linear_u8_kernel<<<rgrid, dim3(32, 8), 0, ctx->stream>>>(d_frames, frame_h, frame_w, d_crops, nc, dst,
                                                                       net_size);
  ctx->launches++;
  OPB_CUDA(ctx, cudaGetLastError());
  return OPB_OK;
}

// F.resize_images(hs[-1], (crop_h, crop_w)) (face_detector.py:38) of the chunk table[first, first + nc): slot i of the
// chunk reads planes [0, planes) of heat_lo + i * kp_out * h8 * h8 (channel `planes` and up, the background, are never
// read) and writes crop first + i's ragged maps in `up`.  d_crops holds `table` on the device.
static int kp_upsample_enqueue(opb_ctx* ctx, const float* heat_lo, int kp_out, int planes, int h8,
                               const std::vector<KpCrop>& table, const KpCrop* d_crops, int first, int nc, int tiles,
                               float* up) {
  const int n = static_cast<int>(table.size());
  const int tile_end = first + nc < n ? table[first + nc].tile0 : tiles;
  const int ppb = 19;
  dim3 ugrid(tile_end - table[first].tile0, (planes + ppb - 1) / ppb);
  upsample_bilinear_ac_ragged_kernel<<<ugrid, dim3(32, 8), 0, ctx->stream>>>(
      heat_lo, static_cast<size_t>(kp_out) * h8 * h8, planes, h8, h8, d_crops + first, nc, table[first].tile0, up, ppb);
  ctx->launches++;
  OPB_CUDA(ctx, cudaGetLastError());
  return OPB_OK;
}

// Crops of `table` (top, left, h, w, flip, vh, vw set) of a frame already on the device, through FaceNet / HandNet in
// chunks of kp_chunk_slots: one crop-table upload, then per chunk a crop + resize launch, the chain and a ragged
// upsample; then kp_peaks_enqueue.  Nothing waits: kp_peaks_collect(ctx, ctx->kp_ws, table, ...) collects the result.
static int kp_enqueue_table(opb_ctx* ctx, const uint8_t* d_frame, int frame_h, int frame_w, std::vector<KpCrop>& table,
                            int net_size) {
  const int n = static_cast<int>(table.size());
  const int planes = ctx->kp_out - 1;              // the last channel is background (face_detector.py:59)
  int tiles = 0, rc;
  size_t floats = 0;
  if ((rc = kp_prepare_table(ctx, table, net_size, planes, &tiles, &floats))) return rc;
  KpWs* ws = nullptr;
  if ((rc = kp_workspace(ctx, floats, planes * n, n, &ws))) return rc;
  OPB_CUDA(ctx, cudaMemcpyAsync(ws->crops, table.data(), sizeof(KpCrop) * n, cudaMemcpyHostToDevice, ctx->stream));
  for (int first = 0; first < n;) {
    const int slots = kp_chunk_slots(n - first), nc = std::min(slots, n - first);
    Chain* ch = nullptr;
    if ((rc = get_chain(ctx, slots, net_size, net_size, &ch))) return rc;
    if ((rc = kp_canvas_enqueue(ctx, d_frame, frame_h, frame_w, ws->crops + first, nc, slots, ch->img_u8, net_size)))
      return rc;
    ch->img_u8_src = nullptr;
    if ((rc = run_chain(ctx, ch, true))) return rc;
    if ((rc = kp_upsample_enqueue(ctx, ch->heat_lo, ctx->kp_out, planes, net_size / 8, table, ws->crops, first, nc,
                                  tiles, ws->up)))
      return rc;
    first += nc;
  }
  return kp_peaks_enqueue(ctx, ws, table, planes, tiles);
}

// kp_enqueue_table, then kp_peaks_collect (one download, one synchronisation).  Keypoints of crop i in crop i's canvas
// coordinates.
static int kp_detect_table(opb_ctx* ctx, const uint8_t* d_frame, int frame_h, int frame_w, std::vector<KpCrop>& table,
                           int net_size, double thresh, double* out, int32_t* valid) {
  int rc = kp_enqueue_table(ctx, d_frame, frame_h, frame_w, table, net_size);
  return rc ? rc : kp_peaks_collect(ctx, ctx->kp_ws, table, ctx->kp_out - 1, thresh, out, valid);
}

int opb_keypoints_detect_crops(opb_ctx* ctx, const uint8_t* frame, int frame_loc, int frame_h, int frame_w,
                               const opb_crop* crops, int n, int net_size, double thresh, double* out, int32_t* valid) {
  if (!ctx) return OPB_ERR_ARG;
  if (!ctx->kp_out) OPB_FAIL(ctx, OPB_ERR_STATE, "this context holds the pose net: load FaceNet / HandNet weights first");
  if (n < 0 || n > 65535) OPB_FAIL(ctx, OPB_ERR_ARG, "crop count must be in [0, 65535]");
  if (n == 0) return OPB_OK;
  if (!frame || !crops || !out || !valid || frame_h <= 0 || frame_w <= 0) OPB_FAIL(ctx, OPB_ERR_ARG, "bad frame or output");
  if (net_size <= 0 || net_size % 8) OPB_FAIL(ctx, OPB_ERR_ARG, "net_size must be a positive multiple of 8");
  std::vector<KpCrop> table(n);
  for (int i = 0; i < n; ++i) {
    const opb_crop& b = crops[i];
    const long long w = static_cast<long long>(b.right) - b.left, h = static_cast<long long>(b.bottom) - b.top;
    if (w <= 0 || h <= 0 || w > (1 << 20) || h > (1 << 20))
      OPB_FAIL(ctx, OPB_ERR_ARG, "crop " + std::to_string(i) + " has a non-positive (or huge) width or height");
    KpCrop& c = table[i];
    c.top = b.top; c.left = b.left; c.h = static_cast<int>(h); c.w = static_cast<int>(w); c.flip = b.flip ? 1 : 0;
    c.vh = c.h; c.vw = c.w;
  }
  cudaSetDevice(ctx->device);
  int rc;
  const uint8_t* d_frame = frame;
  if (frame_loc == OPB_HOST) {
    const size_t in_b = static_cast<size_t>(frame_h) * frame_w * 3;
    if ((rc = ensure_ingest(ctx, in_b + 512))) return rc;
    if ((rc = copy_in(ctx, ctx->ingest_buf, frame, in_b, OPB_HOST))) return rc;
    d_frame = ctx->ingest_buf;
  }
  return kp_detect_table(ctx, d_frame, frame_h, frame_w, table, net_size, thresh, out, valid);
}

// ---------------------------------------------------------------- Haar cascade (csrc/cascade.cuh)
namespace {

const float kCascadeThresholdEps = 1e-5f;   // OpenCV's THRESHOLD_EPS, subtracted from stage thresholds at load
const int kCascadeMaxRaw = 8192;            // raw candidates per frame (before grouping)

int cv_round(double v) { return static_cast<int>(std::nearbyint(v)); }   // cvRound: half to even

}  // namespace

struct CascadeState {
  int win_w = 0, win_h = 0;
  std::vector<CascadeStage> stages;
  std::vector<int> feat;                        // per stump
  std::vector<float> sthr, sleft, sright;
  std::vector<int> rects;                       // [F][3][4]
  std::vector<float> weights;                   // [F][3]
  CascadeStage* d_stages = nullptr;
  CascadeStump* d_stumps = nullptr;
  int stump_pitch = -1;                         // pitch the stump offsets were built for
  // plan of the last (h, w, scale_factor, min, max)
  struct Key { int h, w, min_w, min_h, max_w, max_h; double sf; } key{-1, -1, 0, 0, 0, 0, 0.0};
  std::vector<CascadeLayer> layers;
  int pitch = 0, rows = 0, n_windows = 0, max_h = 0, max_w = 0, max_ny = 0;
  CascadeLayer* d_layers = nullptr;
  CascadeAxis* d_axes = nullptr;
  uint8_t* d_img = nullptr;
  uint32_t *d_sum = nullptr, *d_sq = nullptr;
  int* d_codes = nullptr;
  double* d_sums = nullptr; size_t sums_cap = 0;
  std::vector<void*> plan_allocs;
  uint8_t* d_frame = nullptr; size_t frame_cap = 0;
  int* d_cand = nullptr;
  int* h_cand = nullptr;                        // pinned [1 + 3 * kCascadeMaxRaw]
  void release_plan() { free_all(plan_allocs); d_layers = nullptr; d_axes = nullptr; d_img = nullptr; d_sum = d_sq = nullptr; d_codes = nullptr; key.h = -1; }
  ~CascadeState() {
    release_plan();
    cudaFree(d_stages); cudaFree(d_stumps); cudaFree(d_sums); cudaFree(d_frame); cudaFree(d_cand); cudaFreeHost(h_cand);
  }
};

namespace {

// The float32 scale list of detectMultiScaleNoGrouping: factor *= scale_factor in double while cvRound(win * factor)
// fits the frame and the maximum size; factors whose window is below the minimum size are skipped.
std::vector<float> cascade_scales(const CascadeState* cs, int h, int w, double sf, int min_w, int min_h, int max_w,
                                  int max_h) {
  if (max_w == 0 || max_h == 0) { max_w = w; max_h = h; }
  std::vector<float> out;
  for (double factor = 1.0;; factor *= sf) {
    const int ww = cv_round(cs->win_w * factor), wh = cv_round(cs->win_h * factor);
    if (ww > max_w || wh > max_h || ww > w || wh > h) break;
    if (ww < min_w || wh < min_h) continue;
    out.push_back(static_cast<float>(factor));
  }
  return out;
}

void cascade_axis(int dst_n, int src_n, std::vector<CascadeAxis>& out) {
  const double scale = 1.0 / (static_cast<double>(dst_n) / src_n);
  for (int d = 0; d < dst_n; ++d) {
    const double f = (d + 0.5) * scale - 0.5;
    const double s = std::floor(f);
    const int c1 = cv_round((f - s) * 256);
    const int si = static_cast<int>(s);
    out.push_back(CascadeAxis{std::min(std::max(si, 0), src_n - 1), std::min(std::max(si + 1, 0), src_n - 1), c1, 0});
  }
}

// Layers, interpolation records and buffers for one (h, w, scale_factor, min, max); reused while the key holds.
int cascade_plan(opb_ctx* ctx, CascadeState* cs, int h, int w, double sf, int min_w, int min_h, int max_w, int max_h) {
  CascadeState::Key k{h, w, min_w, min_h, max_w, max_h, sf};
  if (cs->key.h == k.h && cs->key.w == k.w && cs->key.min_w == k.min_w && cs->key.min_h == k.min_h &&
      cs->key.max_w == k.max_w && cs->key.max_h == k.max_h && cs->key.sf == k.sf)
    return OPB_OK;
  OPB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  cs->release_plan();
  const std::vector<float> sc = cascade_scales(cs, h, w, sf, min_w, min_h, max_w, max_h);
  cs->layers.clear();
  std::vector<CascadeAxis> axes;
  int row = 0, win = 0;
  cs->max_h = cs->max_w = cs->max_ny = 0;
  for (float s : sc) {
    CascadeLayer L{};
    L.scale = s;
    L.w = cv_round(static_cast<float>(w) / s);
    L.h = cv_round(static_cast<float>(h) / s);
    L.ystep = s >= 2.f ? 1 : 2;
    const int ww = L.w + 1 - cs->win_w, wh = L.h + 1 - cs->win_h;
    L.nx = ww > 0 ? (ww + L.ystep - 1) / L.ystep : 0;
    L.ny = wh > 0 ? (wh + L.ystep - 1) / L.ystep : 0;
    if (L.nx == 0) L.ny = 0;
    L.row0 = row;
    L.win0 = win;
    L.xtab = static_cast<int>(axes.size());
    cascade_axis(L.w, w, axes);
    L.ytab = static_cast<int>(axes.size());
    cascade_axis(L.h, h, axes);
    row += L.h + 1;
    if (static_cast<long long>(win) + static_cast<long long>(L.nx) * L.ny > (1ll << 30))
      OPB_FAIL(ctx, OPB_ERR_ARG, "too many cascade windows for one frame");
    win += L.nx * L.ny;
    cs->max_h = std::max(cs->max_h, L.h);
    cs->max_w = std::max(cs->max_w, L.w);
    cs->max_ny = std::max(cs->max_ny, L.ny);
    cs->layers.push_back(L);
  }
  cs->pitch = cs->max_w + 1;
  cs->rows = row;
  cs->n_windows = win;
  if (cs->layers.empty()) { cs->key = k; return OPB_OK; }
  if (cs->layers.size() > 65535) OPB_FAIL(ctx, OPB_ERR_ARG, "too many cascade scales");
  const size_t cells = static_cast<size_t>(cs->pitch) * cs->rows;
  int rc;
  if ((rc = dev_alloc(ctx, &cs->d_layers, cs->layers.size(), cs->plan_allocs, false))) return rc;
  if ((rc = dev_alloc(ctx, &cs->d_axes, axes.size(), cs->plan_allocs, false))) return rc;
  if ((rc = dev_alloc(ctx, &cs->d_img, cells, cs->plan_allocs, false))) return rc;
  if ((rc = dev_alloc(ctx, &cs->d_sum, cells, cs->plan_allocs, false))) return rc;
  if ((rc = dev_alloc(ctx, &cs->d_sq, cells, cs->plan_allocs, false))) return rc;
  if ((rc = dev_alloc(ctx, &cs->d_codes, std::max(win, 1), cs->plan_allocs, false))) return rc;
  OPB_CUDA(ctx, cudaMemcpyAsync(cs->d_layers, cs->layers.data(), sizeof(CascadeLayer) * cs->layers.size(),
                                cudaMemcpyHostToDevice, ctx->stream));
  OPB_CUDA(ctx, cudaMemcpyAsync(cs->d_axes, axes.data(), sizeof(CascadeAxis) * axes.size(), cudaMemcpyHostToDevice,
                                ctx->stream));
  if (cs->stump_pitch != cs->pitch) {   // rect corners as offsets in this pitch
    const int P = cs->pitch, T = static_cast<int>(cs->feat.size());
    std::vector<CascadeStump> st(T);
    for (int t = 0; t < T; ++t) {
      CascadeStump& u = st[t];
      for (int r = 0; r < 3; ++r) {
        const int* q = &cs->rects[(static_cast<size_t>(cs->feat[t]) * 3 + r) * 4];
        u.ofs[r][0] = q[1] * P + q[0];
        u.ofs[r][1] = q[1] * P + q[0] + q[2];
        u.ofs[r][2] = (q[1] + q[3]) * P + q[0];
        u.ofs[r][3] = (q[1] + q[3]) * P + q[0] + q[2];
        u.w[r] = cs->weights[static_cast<size_t>(cs->feat[t]) * 3 + r];
      }
      u.thr = cs->sthr[t]; u.left = cs->sleft[t]; u.right = cs->sright[t];
    }
    OPB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    cudaFree(cs->d_stumps);
    cs->d_stumps = nullptr;
    cs->stump_pitch = -1;
    OPB_CUDA(ctx, cudaMalloc(reinterpret_cast<void**>(&cs->d_stumps), sizeof(CascadeStump) * std::max(T, 1)));
    OPB_CUDA(ctx, cudaMemcpyAsync(cs->d_stumps, st.data(), sizeof(CascadeStump) * T, cudaMemcpyHostToDevice, ctx->stream));
    cs->stump_pitch = P;
  }
  cs->key = k;
  return OPB_OK;
}

int cascade_check(opb_ctx* ctx, const uint8_t* img, int h, int w, int channels, double sf, int min_w, int min_h,
                  int max_w, int max_h) {
  if (!ctx->cascade) OPB_FAIL(ctx, OPB_ERR_STATE, "no cascade loaded: call opb_cascade_load first");
  if (!img || h <= 0 || w <= 0) OPB_FAIL(ctx, OPB_ERR_ARG, "bad frame");
  if (channels != 1 && channels != 3) OPB_FAIL(ctx, OPB_ERR_ARG, "channels must be 1 (gray) or 3 (BGR)");
  if (!(sf > 1.0) || !std::isfinite(sf)) OPB_FAIL(ctx, OPB_ERR_ARG, "scale_factor must be a finite number > 1");
  if (min_w < 0 || min_h < 0 || max_w < 0 || max_h < 0) OPB_FAIL(ctx, OPB_ERR_ARG, "sizes must not be negative");
  if (h > 32767 || w > 32767) OPB_FAIL(ctx, OPB_ERR_ARG, "frame larger than 32767 pixels on a side");
  return OPB_OK;
}

// Uploads the frame and runs the four pyramid / integral / window launches; `sums` (optional) receives stage sums.
int cascade_run(opb_ctx* ctx, CascadeState* cs, const uint8_t* img, int img_loc, int h, int w, int channels,
                double* sums, const uint8_t** d_frame_out) {
  const size_t bytes = static_cast<size_t>(h) * w * channels;
  const uint8_t* d_frame = img;
  if (img_loc == OPB_HOST) {
    if (cs->frame_cap < bytes) {
      OPB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
      cudaFree(cs->d_frame);
      cs->d_frame = nullptr;
      cs->frame_cap = 0;
      OPB_CUDA(ctx, cudaMalloc(reinterpret_cast<void**>(&cs->d_frame), bytes));
      cs->frame_cap = bytes;
    }
    if (int rc = copy_in(ctx, cs->d_frame, img, bytes, OPB_HOST)) return rc;
    d_frame = cs->d_frame;
  }
  if (d_frame_out) *d_frame_out = d_frame;
  if (!cs->d_cand) {
    OPB_CUDA(ctx, cudaMalloc(reinterpret_cast<void**>(&cs->d_cand), sizeof(int) * (1 + 3 * kCascadeMaxRaw)));
    OPB_CUDA(ctx, cudaMallocHost(reinterpret_cast<void**>(&cs->h_cand), sizeof(int) * (1 + 3 * kCascadeMaxRaw)));
  }
  const int nl = static_cast<int>(cs->layers.size());
  if (nl == 0) return OPB_OK;
  const int P = cs->pitch;
  cascade_pyramid_kernel<<<dim3((cs->max_w + 31) / 32, (cs->max_h + 7) / 8, nl), dim3(32, 8), 0, ctx->stream>>>(
      d_frame, h, w, channels, cs->d_layers, cs->d_axes, cs->d_img, P, cs->d_cand);
  cascade_row_scan_kernel<<<dim3((cs->max_h + 1 + 7) / 8, nl), dim3(32, 8), 0, ctx->stream>>>(cs->d_layers, cs->d_img, P,
                                                                                              cs->d_sum, cs->d_sq);
  cascade_col_scan_kernel<<<dim3((cs->max_w + 1 + 127) / 128, nl), 128, 0, ctx->stream>>>(cs->d_layers, P, cs->d_sum,
                                                                                          cs->d_sq);
  ctx->launches += 3;
  OPB_CUDA(ctx, cudaGetLastError());
  if (cs->n_windows == 0) return OPB_OK;
  CascadeWindowSetup ws{};
  const int nw = cs->win_w - 2, nh = cs->win_h - 2;
  ws.nofs[0] = P + 1; ws.nofs[1] = P + 1 + nw; ws.nofs[2] = (1 + nh) * P + 1; ws.nofs[3] = (1 + nh) * P + 1 + nw;
  ws.area = static_cast<double>(nw * nh);
  cascade_eval_kernel<<<(cs->n_windows + 127) / 128, 128, 0, ctx->stream>>>(
      cs->d_layers, nl, cs->n_windows, P, cs->d_sum, cs->d_sq, cs->d_stages, static_cast<int>(cs->stages.size()),
      cs->d_stumps, static_cast<int>(cs->feat.size()), ws, cs->d_codes, sums);
  ctx->launches++;
  OPB_CUDA(ctx, cudaGetLastError());
  return OPB_OK;
}

struct CvRect { int x, y, w, h; };

bool rect_less(const CvRect& a, const CvRect& b) {
  if (a.y != b.y) return a.y < b.y;
  if (a.x != b.x) return a.x < b.x;
  if (a.w != b.w) return a.w < b.w;
  return a.h < b.h;
}

// cv::groupRectangles(rects, group_threshold, 0.2) as detectMultiScale applies it (partition with SimilarRects,
// float averaging, the inside-a-bigger-class filter).  The set it returns does not depend on the input order.
std::vector<CvRect> group_rectangles(const std::vector<CvRect>& in, int thr) {
  const double eps = 0.2;
  if (thr <= 0 || in.empty()) return in;
  const int n = static_cast<int>(in.size());
  std::vector<int> parent(n);
  for (int i = 0; i < n; ++i) parent[i] = i;
  auto find = [&](int i) { while (parent[i] != i) { parent[i] = parent[parent[i]]; i = parent[i]; } return i; };
  for (int i = 0; i < n; ++i)
    for (int j = i + 1; j < n; ++j) {
      const CvRect &a = in[i], &b = in[j];
      const double delta = eps * (std::min(a.w, b.w) + std::min(a.h, b.h)) * 0.5;
      if (std::abs(a.x - b.x) <= delta && std::abs(a.y - b.y) <= delta && std::abs(a.x + a.w - b.x - b.w) <= delta &&
          std::abs(a.y + a.h - b.y - b.h) <= delta) {
        const int ra = find(i), rb = find(j);
        if (ra != rb) parent[rb] = ra;
      }
    }
  std::map<int, int> cls;
  std::vector<long long> sx, sy, sw, sh;
  std::vector<int> cnt;
  for (int i = 0; i < n; ++i) {
    const int r = find(i);
    auto it = cls.find(r);
    int c;
    if (it == cls.end()) { c = static_cast<int>(cnt.size()); cls[r] = c; sx.push_back(0); sy.push_back(0); sw.push_back(0); sh.push_back(0); cnt.push_back(0); }
    else c = it->second;
    sx[c] += in[i].x; sy[c] += in[i].y; sw[c] += in[i].w; sh[c] += in[i].h; cnt[c]++;
  }
  const int nc = static_cast<int>(cnt.size());
  std::vector<CvRect> avg(nc);
  for (int c = 0; c < nc; ++c) {
    const float s = 1.f / static_cast<float>(cnt[c]);
    avg[c] = CvRect{cv_round(static_cast<float>(sx[c]) * s), cv_round(static_cast<float>(sy[c]) * s),
                    cv_round(static_cast<float>(sw[c]) * s), cv_round(static_cast<float>(sh[c]) * s)};
  }
  std::vector<CvRect> out;
  for (int i = 0; i < nc; ++i) {
    const CvRect r1 = avg[i];
    const int n1 = cnt[i];
    if (n1 <= thr) continue;
    int j = 0;
    for (; j < nc; ++j) {
      const int n2 = cnt[j];
      if (j == i || n2 <= thr) continue;
      const CvRect r2 = avg[j];
      const int dx = cv_round(r2.w * eps), dy = cv_round(r2.h * eps);
      if (r1.x >= r2.x - dx && r1.y >= r2.y - dy && r1.x + r1.w <= r2.x + r2.w + dx && r1.y + r1.h <= r2.y + r2.h + dy &&
          (n2 > std::max(3, n1) || n1 < 3))
        break;
    }
    if (j == nc) out.push_back(r1);
  }
  return out;
}

// The full detectMultiScale: upload, five launches, one candidate download and synchronisation, host grouping.
int cascade_detect(opb_ctx* ctx, const uint8_t* img, int img_loc, int h, int w, int channels, double sf, int min_nb,
                   int min_w, int min_h, int max_w, int max_h, std::vector<CvRect>& out, const uint8_t** d_frame) {
  CascadeState* cs = ctx->cascade;
  int rc;
  if ((rc = cascade_plan(ctx, cs, h, w, sf, min_w, min_h, max_w, max_h))) return rc;
  if ((rc = cascade_run(ctx, cs, img, img_loc, h, w, channels, nullptr, d_frame))) return rc;
  out.clear();
  if (cs->n_windows == 0) return OPB_OK;
  const int nl = static_cast<int>(cs->layers.size());
  cascade_compact_kernel<<<dim3((cs->max_ny + 3) / 4, nl), dim3(32, 4), 0, ctx->stream>>>(cs->d_layers, cs->d_codes,
                                                                                        cs->d_cand, kCascadeMaxRaw);
  ctx->launches++;
  OPB_CUDA(ctx, cudaGetLastError());
  OPB_CUDA(ctx, cudaMemcpyAsync(cs->h_cand, cs->d_cand, sizeof(int) * (1 + 3 * kCascadeMaxRaw), cudaMemcpyDeviceToHost,
                                ctx->stream));
  OPB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  const int n = cs->h_cand[0];
  if (n > kCascadeMaxRaw) OPB_FAIL(ctx, OPB_ERR_CAPACITY, "more than 8192 raw cascade candidates in one frame");
  std::vector<CvRect> raw(n);
  for (int i = 0; i < n; ++i) {
    const CascadeLayer& L = cs->layers[cs->h_cand[1 + 3 * i]];
    const float s = L.scale;
    const int x = cv_round(static_cast<float>(cs->h_cand[2 + 3 * i]) * s);
    const int y = cv_round(static_cast<float>(cs->h_cand[3 + 3 * i]) * s);
    const int rw = cv_round(static_cast<float>(cs->win_w) * s), rh = cv_round(static_cast<float>(cs->win_h) * s);
    raw[i] = CvRect{x, y, std::min(x + rw, w) - x, std::min(y + rh, h) - y};   // clipped to the frame, as cv2 4.13
  }
  out = group_rectangles(raw, min_nb);
  std::sort(out.begin(), out.end(), rect_less);
  return OPB_OK;
}

int cascade_write_rects(opb_ctx* ctx, const std::vector<CvRect>& r, int32_t* rects_out, int cap, int* n_out) {
  *n_out = static_cast<int>(r.size());
  if (static_cast<int>(r.size()) > cap) OPB_FAIL(ctx, OPB_ERR_CAPACITY, "more detections than rects_out holds");
  for (size_t i = 0; i < r.size(); ++i) {
    rects_out[i * 4 + 0] = r[i].x; rects_out[i * 4 + 1] = r[i].y; rects_out[i * 4 + 2] = r[i].w; rects_out[i * 4 + 3] = r[i].h;
  }
  return OPB_OK;
}

}  // namespace

int opb_cascade_load(opb_ctx* ctx, int win_w, int win_h, int n_stages, const int32_t* stage_ntrees,
                     const float* stage_threshold, int n_stumps, const int32_t* stump_feature,
                     const float* stump_threshold, const float* stump_left, const float* stump_right, int n_features,
                     const int32_t* rects, const float* weights) {
  if (!ctx) return OPB_ERR_ARG;
  if (win_w < 3 || win_h < 3 || win_w > 1024 || win_h > 1024) OPB_FAIL(ctx, OPB_ERR_ARG, "window size out of range");
  if (n_stages <= 0 || n_stages > kCascadeMaxStages) OPB_FAIL(ctx, OPB_ERR_ARG, "stage count must be in [1, 64]");
  if (n_stumps <= 0 || n_features <= 0 || !stage_ntrees || !stage_threshold || !stump_feature || !stump_threshold ||
      !stump_left || !stump_right || !rects || !weights)
    OPB_FAIL(ctx, OPB_ERR_ARG, "empty or missing cascade tables");
  auto cs = std::unique_ptr<CascadeState>(new CascadeState());
  cs->win_w = win_w; cs->win_h = win_h;
  long long first = 0;
  for (int s = 0; s < n_stages; ++s) {
    if (stage_ntrees[s] <= 0) OPB_FAIL(ctx, OPB_ERR_ARG, "a stage without stumps");
    cs->stages.push_back(CascadeStage{static_cast<int>(first), stage_ntrees[s], stage_threshold[s] - kCascadeThresholdEps, 0});
    first += stage_ntrees[s];
  }
  if (first != n_stumps) OPB_FAIL(ctx, OPB_ERR_ARG, "stage tree counts do not add up to the stump count");
  for (int t = 0; t < n_stumps; ++t)
    if (stump_feature[t] < 0 || stump_feature[t] >= n_features) OPB_FAIL(ctx, OPB_ERR_ARG, "stump feature index out of range");
  for (int f = 0; f < n_features; ++f)
    for (int r = 0; r < 3; ++r) {
      const int32_t* q = rects + (static_cast<size_t>(f) * 3 + r) * 4;
      if (weights[f * 3 + r] == 0.f && r > 0) continue;
      if (q[0] < 0 || q[1] < 0 || q[2] < 0 || q[3] < 0 || q[0] + q[2] > win_w || q[1] + q[3] > win_h)
        OPB_FAIL(ctx, OPB_ERR_ARG, "feature " + std::to_string(f) + " has a rect outside the window");
    }
  cs->feat.assign(stump_feature, stump_feature + n_stumps);
  cs->sthr.assign(stump_threshold, stump_threshold + n_stumps);
  cs->sleft.assign(stump_left, stump_left + n_stumps);
  cs->sright.assign(stump_right, stump_right + n_stumps);
  cs->rects.assign(rects, rects + static_cast<size_t>(n_features) * 12);
  cs->weights.assign(weights, weights + static_cast<size_t>(n_features) * 3);
  for (int f = 0; f < n_features; ++f)     // an absent rect reads nothing: point it at the window origin
    for (int r = 1; r < 3; ++r)
      if (cs->weights[f * 3 + r] == 0.f) std::fill_n(&cs->rects[(static_cast<size_t>(f) * 3 + r) * 4], 4, 0);
  cudaSetDevice(ctx->device);
  OPB_CUDA(ctx, cudaMalloc(reinterpret_cast<void**>(&cs->d_stages), sizeof(CascadeStage) * n_stages));
  OPB_CUDA(ctx, cudaMemcpyAsync(cs->d_stages, cs->stages.data(), sizeof(CascadeStage) * n_stages, cudaMemcpyHostToDevice,
                                ctx->stream));
  OPB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  delete ctx->cascade;
  ctx->cascade = cs.release();
  return OPB_OK;
}

int opb_cascade_detect(opb_ctx* ctx, const uint8_t* img, int img_loc, int h, int w, int channels, double scale_factor,
                       int min_neighbors, int min_w, int min_h, int max_w, int max_h, int32_t* rects_out, int cap,
                       int* n_out) {
  if (!ctx) return OPB_ERR_ARG;
  int rc;
  if ((rc = cascade_check(ctx, img, h, w, channels, scale_factor, min_w, min_h, max_w, max_h))) return rc;
  if (min_neighbors < 0 || cap < 0 || !n_out || (cap > 0 && !rects_out)) OPB_FAIL(ctx, OPB_ERR_ARG, "bad output or min_neighbors");
  cudaSetDevice(ctx->device);
  std::vector<CvRect> r;
  if ((rc = cascade_detect(ctx, img, img_loc, h, w, channels, scale_factor, min_neighbors, min_w, min_h, max_w, max_h, r,
                           nullptr)))
    return rc;
  return cascade_write_rects(ctx, r, rects_out, cap, n_out);
}

int opb_face_detect_frame(opb_ctx* ctx, const uint8_t* frame, int frame_loc, int h, int w, double scale_factor,
                          int min_neighbors, int min_w, int min_h, int max_w, int max_h, double crop_scale,
                          int net_size, double thresh, int32_t* rects_out, int cap, int* n_out, double* out,
                          int32_t* valid, int32_t* left_top) {
  if (!ctx) return OPB_ERR_ARG;
  int rc;
  if ((rc = cascade_check(ctx, frame, h, w, 3, scale_factor, min_w, min_h, max_w, max_h))) return rc;
  if (!ctx->kp_out) OPB_FAIL(ctx, OPB_ERR_STATE, "this context holds the pose net: load FaceNet weights first");
  if (min_neighbors < 0 || cap < 0 || !n_out || (cap > 0 && (!rects_out || !out || !valid || !left_top)))
    OPB_FAIL(ctx, OPB_ERR_ARG, "bad output or min_neighbors");
  if (!(crop_scale > 0.0) || !std::isfinite(crop_scale)) OPB_FAIL(ctx, OPB_ERR_ARG, "crop_scale must be positive");
  if (net_size <= 0 || net_size % 8) OPB_FAIL(ctx, OPB_ERR_ARG, "net_size must be a positive multiple of 8");
  cudaSetDevice(ctx->device);
  std::vector<CvRect> r;
  const uint8_t* d_frame = nullptr;
  if ((rc = cascade_detect(ctx, frame, frame_loc, h, w, 3, scale_factor, min_neighbors, min_w, min_h, max_w, max_h, r,
                           &d_frame)))
    return rc;
  if ((rc = cascade_write_rects(ctx, r, rects_out, cap, n_out))) return rc;
  if (r.empty()) return OPB_OK;
  // crop_face of camera_face_demo.py:10-24: int() truncates toward zero; right / bottom clamp to w / h; the crop is
  // zero-padded at the bottom and right to an edge x edge square
  std::vector<KpCrop> table(r.size());
  for (size_t i = 0; i < r.size(); ++i) {
    const double cx = r[i].x + r[i].w / 2.0, cy = r[i].y + r[i].h / 2.0;
    const double cw = r[i].w * crop_scale, chh = r[i].h * crop_scale;
    const int left = std::max(0, static_cast<int>(cx - cw / 2)), top = std::max(0, static_cast<int>(cy - chh / 2));
    const int right = std::min(w, static_cast<int>(cx + cw / 2)), bottom = std::min(h, static_cast<int>(cy + chh / 2));
    if (right <= left || bottom <= top) OPB_FAIL(ctx, OPB_ERR_ARG, "a face rect gives an empty crop");
    KpCrop& c = table[i];
    c.top = top; c.left = left; c.vh = bottom - top; c.vw = right - left;
    c.h = c.w = std::max(c.vh, c.vw);
    c.flip = 0;
    left_top[i * 2 + 0] = left;
    left_top[i * 2 + 1] = top;
  }
  return kp_detect_table(ctx, d_frame, h, w, table, net_size, thresh, out, valid);
}

int opb_test_cascade_windows(opb_ctx* ctx, const uint8_t* img, int img_loc, int h, int w, int channels,
                             double scale_factor, int min_w, int min_h, int max_w, int max_h, int32_t* codes_out,
                             double* sums_out, int cap, int* n_out) {
  if (!ctx) return OPB_ERR_ARG;
  int rc;
  if ((rc = cascade_check(ctx, img, h, w, channels, scale_factor, min_w, min_h, max_w, max_h))) return rc;
  if (!n_out || cap < 0 || (cap > 0 && (!codes_out || !sums_out))) OPB_FAIL(ctx, OPB_ERR_ARG, "bad output");
  cudaSetDevice(ctx->device);
  CascadeState* cs = ctx->cascade;
  if ((rc = cascade_plan(ctx, cs, h, w, scale_factor, min_w, min_h, max_w, max_h))) return rc;
  *n_out = cs->n_windows;
  if (cs->n_windows > cap) OPB_FAIL(ctx, OPB_ERR_CAPACITY, "more windows than the output holds");
  if (cs->sums_cap < static_cast<size_t>(cs->n_windows)) {
    OPB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    cudaFree(cs->d_sums);
    cs->d_sums = nullptr;
    cs->sums_cap = 0;
    OPB_CUDA(ctx, cudaMalloc(reinterpret_cast<void**>(&cs->d_sums), sizeof(double) * std::max(cs->n_windows, 1)));
    cs->sums_cap = cs->n_windows;
  }
  if ((rc = cascade_run(ctx, cs, img, img_loc, h, w, channels, cs->d_sums, nullptr))) return rc;
  if (cs->n_windows == 0) return OPB_OK;
  if ((rc = copy_out(ctx, codes_out, cs->d_codes, sizeof(int) * cs->n_windows, OPB_HOST))) return rc;
  if ((rc = copy_out(ctx, sums_out, cs->d_sums, sizeof(double) * cs->n_windows, OPB_HOST))) return rc;
  OPB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return OPB_OK;
}

// ---------------------------------------------------------------- the whole-body frame of demo.py (csrc/whole_body.cuh)
namespace {

// Device block of the box kernel's outputs for `n` frames of `cap` persons, in the order the frame call downloads it:
// the counts and the three compacted tables first, then the per-person unit lengths, boxes and present bits (test
// hooks only).  Frame f's section of each array starts at f * cap persons (whole_body_boxes_kernel).
struct WbLayout {
  size_t counts, face, hand, parts, tables_end, unit, box, present, total;
};

WbLayout wb_layout(int cap, int n = 1) {
  auto al = [](size_t v) { return (v + 255) & ~size_t(255); };
  const size_t c = static_cast<size_t>(cap) * n;
  WbLayout L;
  L.counts = 0;
  L.face = al(sizeof(WbCounts) * n);
  L.hand = L.face + al(sizeof(WbCrop) * c);
  L.parts = L.hand + al(sizeof(WbCrop) * 2 * c);
  L.tables_end = L.parts + al(sizeof(WbPart) * 3 * c);
  L.unit = L.tables_end;
  L.box = L.unit + al(sizeof(double) * c);
  L.present = L.box + al(sizeof(int) * 12 * c);
  L.total = L.present + al(sizeof(int) * c);
  return L;
}

// Grows ctx->wb_buf to the layout of `n` frames of `cap` persons plus `extra` bytes after it, and the pinned
// ctx->wb_host to `host_bytes`.
int wb_reserve(opb_ctx* ctx, int cap, int n, size_t extra, size_t host_bytes, WbOut* out) {
  const WbLayout L = wb_layout(cap, n);
  if (ctx->wb_bytes < L.total + extra) {
    if (ctx->wb_buf) { OPB_CUDA(ctx, cudaStreamSynchronize(ctx->stream)); cudaFree(ctx->wb_buf); ctx->wb_buf = nullptr; }
    ctx->wb_bytes = 0;
    OPB_CUDA(ctx, cudaMalloc(reinterpret_cast<void**>(&ctx->wb_buf), L.total + extra));
    ctx->wb_bytes = L.total + extra;
  }
  if (ctx->wb_host_bytes < host_bytes) {
    if (ctx->wb_host) { cudaFreeHost(ctx->wb_host); ctx->wb_host = nullptr; }
    ctx->wb_host_bytes = 0;
    OPB_CUDA(ctx, cudaMallocHost(reinterpret_cast<void**>(&ctx->wb_host), host_bytes));
    ctx->wb_host_bytes = host_bytes;
  }
  uint8_t* b = ctx->wb_buf;
  out->counts = reinterpret_cast<WbCounts*>(b + L.counts);
  out->face = reinterpret_cast<WbCrop*>(b + L.face);
  out->hand = reinterpret_cast<WbCrop*>(b + L.hand);
  out->parts = reinterpret_cast<WbPart*>(b + L.parts);
  out->unit = reinterpret_cast<double*>(b + L.unit);
  out->box = reinterpret_cast<int*>(b + L.box);
  out->present = reinterpret_cast<int*>(b + L.present);
  return OPB_OK;
}

// Ragged-map budget per net of one group of frames in opb_whole_body_batch: 2^30 floats, i.e. 4 GiB for each of the
// two map buffers
constexpr size_t kWbGroupFloats = size_t(1) << 30;

// One launch for n frames: headers d_hd[n], persons d_persons[n][cap]
int wb_launch(opb_ctx* ctx, const ImageHeader* d_hd, const PersonOut* d_persons, int n, int cap, double sx, double sy,
              const WbOut& out) {
  whole_body_boxes_kernel<<<n, WB_THREADS, 0, ctx->stream>>>(d_hd, d_persons, cap, sx, sy, out);
  ctx->launches++;
  OPB_CUDA(ctx, cudaGetLastError());
  return OPB_OK;
}

// opb_crop rows of frame `frame` -> KpCrop rows appended to the table of opb_keypoints_detect_crops
int wb_kp_table(opb_ctx* ctx, const WbCrop* crops, int n, int frame, std::vector<KpCrop>& table) {
  for (int i = 0; i < n; ++i) {
    const WbCrop& b = crops[i];
    const long long w = static_cast<long long>(b.right) - b.left, h = static_cast<long long>(b.bottom) - b.top;
    if (w <= 0 || h <= 0 || w > (1 << 20) || h > (1 << 20))
      OPB_FAIL(ctx, OPB_ERR_ARG, "whole_body_batch: a crop is wider or taller than 2^20");
    KpCrop c{};
    c.top = b.top; c.left = b.left; c.h = static_cast<int>(h); c.w = static_cast<int>(w); c.flip = b.flip;
    c.vh = c.h; c.vw = c.w; c.frame = frame;
    table.push_back(c);
  }
  return OPB_OK;
}

}  // namespace

int opb_whole_body_batch(opb_ctx* pose, opb_ctx* face, opb_ctx* hand, const uint8_t* frames, int frames_loc, int n,
                         int orig_h, int orig_w, int in_h, int in_w, int map_h, int map_w, double img_len,
                         const float* inject_paf, const float* inject_heat, int face_net_size, double face_thresh,
                         int hand_net_size, double hand_thresh, opb_image_header* headers_out, opb_person* persons_out,
                         opb_wb_part* parts_out, int parts_cap, int* n_parts, int* frame_parts, double* face_out,
                         int32_t* face_valid, double* hand_out, int32_t* hand_valid, uint8_t* pictures_out) {
  if (!pose) return OPB_ERR_ARG;
  // everything is checked before the first enqueue
  if (!face || !hand) OPB_FAIL(pose, OPB_ERR_ARG, "whole_body_batch: a FaceNet and a HandNet context are required");
  if (pose->kp_out != 0) OPB_FAIL(pose, OPB_ERR_STATE, "whole_body_batch: the first context must hold the pose net");
  if (face->kp_out != 71) OPB_FAIL(pose, OPB_ERR_STATE, "whole_body_batch: the face context does not hold FaceNet");
  if (hand->kp_out != 22) OPB_FAIL(pose, OPB_ERR_STATE, "whole_body_batch: the hand context does not hold HandNet");
  if (pose->precision < 0 || face->precision < 0 || hand->precision < 0)
    OPB_FAIL(pose, OPB_ERR_STATE, "whole_body_batch: opb_finalize_weights has not been called on every context");
  if (face->device != pose->device || hand->device != pose->device)
    OPB_FAIL(pose, OPB_ERR_ARG, "whole_body_batch: the three contexts must be on the same device");
  if (n < 1) OPB_FAIL(pose, OPB_ERR_ARG, "whole_body_batch: the batch must hold at least one frame");
  if (!frames || orig_h <= 0 || orig_w <= 0 || in_h <= 0 || in_w <= 0 || in_h % 8 || in_w % 8 || map_h <= 0 || map_w <= 0)
    OPB_FAIL(pose, OPB_ERR_ARG, "whole_body_batch: bad frame, input or map size");
  const size_t px = static_cast<size_t>(orig_h) * orig_w;
  if (static_cast<unsigned long long>(n) * px > (1ull << 31) - 256)
    OPB_FAIL(pose, OPB_ERR_ARG, "whole_body_batch: more than 2^31 pixels in one batch");
  if (face_net_size <= 0 || face_net_size % 8 || hand_net_size <= 0 || hand_net_size % 8)
    OPB_FAIL(pose, OPB_ERR_ARG, "whole_body_batch: net sizes must be positive multiples of 8");
  if (!headers_out || !persons_out || !n_parts || !frame_parts || parts_cap < 0 ||
      (parts_cap > 0 && (!parts_out || !face_out || !face_valid || !hand_out || !hand_valid)))
    OPB_FAIL(pose, OPB_ERR_ARG, "whole_body_batch: bad output arguments");
  *n_parts = 0;
  cudaSetDevice(pose->device);
  const double sx = static_cast<double>(orig_w) / map_w, sy = static_cast<double>(orig_h) / map_h;  // :513-514
  const int cap = pose->prm.max_persons;
  const size_t rec_b = static_cast<size_t>(n) * (sizeof(ImageHeader) + sizeof(PersonOut) * static_cast<size_t>(cap));
  const WbLayout L = wb_layout(cap, n);
  int rc;
  // (1) one upload of all frames, one device resize of the batch and the pipeline at batch n, the launch sequence of
  // opb_stream_submit for n frames
  Chain* ch = nullptr;
  PostWs* ws = nullptr;
  if ((rc = get_chain(pose, n, in_h, in_w, &ch))) return rc;
  if ((rc = get_post(pose, n, map_h, map_w, &ws))) return rc;
  WbOut wo;
  if ((rc = wb_reserve(pose, cap, n, 0, rec_b + L.tables_end, &wo))) return rc;
  const size_t in_b = px * 3 * n;
  const uint8_t* d_frames = frames;
  if (frames_loc == OPB_HOST) {
    if ((rc = ensure_ingest(pose, in_b + 512))) return rc;
    if ((rc = copy_in(pose, pose->ingest_buf, frames, in_b, OPB_HOST))) return rc;
    d_frames = pose->ingest_buf;
  }
  if ((rc = launch_resize_u8(pose, d_frames, n, orig_h, orig_w, ch->img_u8, in_h, in_w))) return rc;
  ch->img_u8_src = nullptr;
  // (2) inject_* replace the network output, as in opb_detect_batch
  if ((rc = run_pipeline(pose, ch, ws, n, in_h, in_w, map_h, map_w, img_len, inject_paf, inject_heat))) return rc;
  // (3) the crop boxes of every frame in one launch, then one download of the records and the tables and one
  // synchronisation
  if ((rc = wb_launch(pose, ws->headers, ws->persons, n, cap, sx, sy, wo))) return rc;
  static_assert(sizeof(ImageHeader) % 16 == 0, "the persons follow the headers in the record block");
  OPB_CUDA(pose, cudaMemcpyAsync(pose->wb_host, ws->headers, rec_b, cudaMemcpyDeviceToHost, pose->stream));
  OPB_CUDA(pose, cudaMemcpyAsync(pose->wb_host + rec_b, pose->wb_buf, L.tables_end, cudaMemcpyDeviceToHost, pose->stream));
  OPB_CUDA(pose, cudaStreamSynchronize(pose->stream));
  const uint8_t* hb = pose->wb_host;
  const ImageHeader* hds = reinterpret_cast<const ImageHeader*>(hb);
  std::memcpy(headers_out, hb, sizeof(ImageHeader) * n);
  std::memcpy(persons_out, hb + sizeof(ImageHeader) * n, sizeof(PersonOut) * static_cast<size_t>(cap) * n);
  for (int f = 0; f < n; ++f)
    if (hds[f].status != 0)
      OPB_FAIL(pose, hds[f].status, "whole_body_batch: frame " + std::to_string(f) + "'s result carries an error status");
  const WbCounts* cnt = reinterpret_cast<const WbCounts*>(hb + rec_b + L.counts);
  for (int f = 0; f < n; ++f)
    if (cnt[f].status != 0)
      OPB_FAIL(pose, cnt[f].status, "whole_body_batch: a crop box edge of frame " + std::to_string(f) + " does not fit int32");
  const WbCrop* h_face = reinterpret_cast<const WbCrop*>(hb + rec_b + L.face);
  const WbCrop* h_hand = reinterpret_cast<const WbCrop*>(hb + rec_b + L.hand);
  const WbPart* h_parts = reinterpret_cast<const WbPart*>(hb + rec_b + L.parts);
  long long total = 0;
  frame_parts[0] = 0;
  for (int f = 0; f < n; ++f) {
    total += cnt[f].n_parts;
    frame_parts[f + 1] = static_cast<int>(std::min<long long>(total, INT32_MAX));
  }
  *n_parts = static_cast<int>(std::min<long long>(total, INT32_MAX));
  if (total > parts_cap) OPB_FAIL(pose, OPB_ERR_CAPACITY, "whole_body_batch: more parts than parts_cap");
  // the sections of every frame, concatenated frame by frame: face / hand rows run over the whole batch
  std::vector<KpCrop> ftab, htab;
  std::vector<int> face_first(n + 1, 0), hand_first(n + 1, 0);
  for (int f = 0; f < n; ++f) {
    const size_t fc = static_cast<size_t>(f) * cap;
    const int face0 = static_cast<int>(ftab.size()), hand0 = static_cast<int>(htab.size());
    face_first[f] = face0;
    hand_first[f] = hand0;
    if ((rc = wb_kp_table(pose, h_face + fc, cnt[f].n_face, f, ftab))) return rc;
    if ((rc = wb_kp_table(pose, h_hand + 2 * fc, cnt[f].n_hand, f, htab))) return rc;
    for (int i = 0; i < cnt[f].n_parts; ++i) {
      const WbPart& p = h_parts[3 * fc + i];
      const WbCrop& b = p.side == WB_FACE ? h_face[fc + p.row] : h_hand[2 * fc + p.row];
      parts_out[frame_parts[f] + i] =
          opb_wb_part{p.side == WB_FACE ? OPB_PART_FACE : OPB_PART_HAND, b.left, b.top, b.right, b.bottom,
                      p.row + (p.side == WB_FACE ? face0 : hand0), p.person, p.side};
    }
  }
  face_first[n] = static_cast<int>(ftab.size());
  hand_first[n] = static_cast<int>(htab.size());
  // (4) FaceNet on the face stream and HandNet on the hand stream, both reading the frames in place; both chains are
  // enqueued before either is collected, so they overlap, and their chunks cross frame boundaries.  The ragged maps of
  // a call hold every crop at its own size, so frames go through the nets in groups of whole frames whose maps stay
  // under kWbGroupFloats per net (a group holds at least one frame): a batch needs no more map workspace than the
  // budget or its largest frame.  Groups after the first start a new chunk sequence.
  const int face_pl = face->kp_out - 1, hand_pl = hand->kp_out - 1;
  auto area = [](const std::vector<KpCrop>& t, int a, int b) {
    size_t v = 0;
    for (int i = a; i < b; ++i) v += static_cast<size_t>(t[i].h) * t[i].w;
    return v;
  };
  for (int g0 = 0; g0 < n;) {
    size_t ff = area(ftab, face_first[g0], face_first[g0 + 1]) * face_pl;
    size_t hf = area(htab, hand_first[g0], hand_first[g0 + 1]) * hand_pl;
    int g1 = g0 + 1;
    for (; g1 < n; ++g1) {
      const size_t nf = ff + area(ftab, face_first[g1], face_first[g1 + 1]) * face_pl;
      const size_t nh = hf + area(htab, hand_first[g1], hand_first[g1 + 1]) * hand_pl;
      if (nf > kWbGroupFloats || nh > kWbGroupFloats) break;
      ff = nf;
      hf = nh;
    }
    std::vector<KpCrop> fg(ftab.begin() + face_first[g0], ftab.begin() + face_first[g1]);
    std::vector<KpCrop> hg(htab.begin() + hand_first[g0], htab.begin() + hand_first[g1]);
    if (!fg.empty() && (rc = kp_enqueue_table(face, d_frames, orig_h, orig_w, fg, face_net_size))) {
      pose->err = face->err;
      cudaGetLastError();
      return rc;
    }
    if (!hg.empty() && (rc = kp_enqueue_table(hand, d_frames, orig_h, orig_w, hg, hand_net_size))) {
      pose->err = hand->err;
      cudaGetLastError();
      cudaStreamSynchronize(face->stream);
      return rc;
    }
    const size_t fr0 = face_first[g0], hr0 = hand_first[g0];
    int rc_face = OPB_OK, rc_hand = OPB_OK;
    if (!fg.empty())
      rc_face = kp_peaks_collect(face, face->kp_ws, fg, face_pl, face_thresh, face_out + fr0 * face_pl * 3,
                                 face_valid + fr0 * face_pl);
    if (!hg.empty())
      rc_hand = kp_peaks_collect(hand, hand->kp_ws, hg, hand_pl, hand_thresh, hand_out + hr0 * hand_pl * 3,
                                 hand_valid + hr0 * hand_pl);
    if (rc_face) { pose->err = face->err; return rc_face; }
    if (rc_hand) { pose->err = hand->err; return rc_hand; }
    g0 = g1;
  }
  if (!pictures_out) return OPB_OK;
  // (5) the pictures of opb_draw_whole_body on the resident frames, the skeletons from the device records: one table
  // upload, one records -> poses launch, one raster and one paint launch for all n pictures, one download
  const int n_all = *n_parts;
  std::vector<int32_t> tab(static_cast<size_t>(n) * 4 + static_cast<size_t>(n_all) * 6);   // [frames | parts | points]
  std::vector<int32_t> pts;
  long long n_prim = 0;
  int total_poses = 0;
  for (int f = 0; f < n; ++f) {
    const int n_poses = hds[f].n_peaks == 0 ? 0 : std::min(hds[f].n_persons, cap);
    const int np = frame_parts[f + 1] - frame_parts[f];
    const int32_t fr[4] = {static_cast<int32_t>(n_prim), n_poses, frame_parts[f], np};
    std::copy(fr, fr + 4, tab.begin() + 4 * f);
    n_prim += static_cast<long long>(n_poses) * (OV_LIMBS + OV_JOINTS) + static_cast<long long>(np) * OV_PART_STRIDE;
    total_poses += n_poses;
    if (n_prim > (1ll << 30)) OPB_FAIL(pose, OPB_ERR_ARG, "whole_body_batch: too many poses / parts to draw");
  }
  static_assert(sizeof(OvFrame) == 16, "OvFrame rows are four ints");
  int32_t* tparts = tab.data() + 4 * n;
  for (int i = 0; i < n_all; ++i) {
    const opb_wb_part& p = parts_out[i];
    const bool is_face = p.kind == OPB_PART_FACE;
    const int count = is_face ? face_pl : hand_pl;
    const double* o = (is_face ? face_out : hand_out) + static_cast<size_t>(p.row) * count * 3;
    const int32_t* v = (is_face ? face_valid : hand_valid) + static_cast<size_t>(p.row) * count;
    const int32_t row[6] = {p.kind, p.left, p.top, p.right, p.bottom, static_cast<int32_t>(pts.size() / 3)};
    std::copy(row, row + 6, tparts + 6 * i);
    for (int k = 0; k < count; ++k) {
      pts.push_back(v[k] ? static_cast<int32_t>(o[3 * k]) : 0);
      pts.push_back(v[k] ? static_cast<int32_t>(o[3 * k + 1]) : 0);
      pts.push_back(v[k] ? 1 : 0);
    }
  }
  const int n_points = static_cast<int>(pts.size() / 3);
  if ((rc = check_parts(pose, reinterpret_cast<const opb_part*>(tparts), n_all, pts.data(), n_points))) return rc;
  tab.insert(tab.end(), pts.begin(), pts.end());
  const size_t img_b = (px * 3 * n + 255) & ~size_t(255), prio_b = (px * 4 * n + 255) & ~size_t(255);
  const size_t poses_b = (static_cast<size_t>(n) * cap * OV_JOINTS * 3 * 4 + 255) & ~size_t(255);
  const size_t tab_b = (tab.size() * 4 + 255) & ~size_t(255);
  // scratch: [pictures | priority planes | int poses [n][cap] | frames, parts and points | flag]
  if ((rc = ov_reserve(pose, img_b + prio_b + poses_b + tab_b + 256))) return rc;
  uint8_t* d_out = pose->ov_buf;
  unsigned int* d_prio = reinterpret_cast<unsigned int*>(pose->ov_buf + img_b);
  int* d_poses = reinterpret_cast<int*>(pose->ov_buf + img_b + prio_b);
  int* d_tab = reinterpret_cast<int*>(pose->ov_buf + img_b + prio_b + poses_b);
  int* d_bad = reinterpret_cast<int*>(pose->ov_buf + img_b + prio_b + poses_b + tab_b);
  if ((rc = copy_in(pose, d_tab, tab.data(), tab.size() * 4, OPB_HOST))) return rc;
  OPB_CUDA(pose, cudaMemsetAsync(d_prio, 0, px * 4 * n, pose->stream));
  OPB_CUDA(pose, cudaMemsetAsync(d_bad, 0, 4, pose->stream));
  const OverlayTables tb = overlay_tables(pose);
  const OvFrame* d_fr = reinterpret_cast<const OvFrame*>(d_tab);
  const OvPart* d_parts = reinterpret_cast<const OvPart*>(d_tab + 4 * n);
  const int* d_points = d_tab + 4 * n + static_cast<size_t>(n_all) * 6;
  if (total_poses > 0) {
    const int* base = reinterpret_cast<const int*>(ws->persons);
    const int stride = static_cast<int>(sizeof(PersonOut) / 4), off_id = 4, off_x = 4 + OPB_N_JOINTS, off_y = 4 + 2 * OPB_N_JOINTS;
    const size_t threads = static_cast<size_t>(n) * cap * OV_JOINTS;
    overlay_poses_from_records_batch_kernel<<<static_cast<unsigned>((threads + 127) / 128), 128, 0, pose->stream>>>(
        base + off_x, base + off_y, base + off_id, stride, cap, d_fr, n, sx, sy, d_poses);
    pose->launches++;
  }
  if (n_prim > 0) {
    overlay_raster_batch_kernel<<<static_cast<unsigned>((n_prim + 63) / 64), 64, 0, pose->stream>>>(
        d_poses, cap, d_fr, n, static_cast<int>(n_prim), tb, d_prio, orig_h, orig_w, d_bad, d_parts, d_points);
    pose->launches++;
  }
  overlay_paint_batch_kernel<<<static_cast<unsigned>((px * n + 255) / 256), 256, 0, pose->stream>>>(
      d_frames, d_prio, static_cast<int>(px), d_fr, n, tb, d_out, d_parts);
  pose->launches++;
  OPB_CUDA(pose, cudaGetLastError());
  int bad = 0;
  OPB_CUDA(pose, cudaMemcpyAsync(&bad, d_bad, 4, cudaMemcpyDeviceToHost, pose->stream));
  if ((rc = copy_out(pose, pictures_out, d_out, px * 3 * n, OPB_HOST))) return rc;
  OPB_CUDA(pose, cudaStreamSynchronize(pose->stream));
  if (bad) OPB_FAIL(pose, OPB_ERR_ARG, "whole_body_batch: a joint lies outside the image");
  return OPB_OK;
}

int opb_whole_body_frame(opb_ctx* pose, opb_ctx* face, opb_ctx* hand, const uint8_t* img, int img_loc, int orig_h,
                         int orig_w, int in_h, int in_w, int map_h, int map_w, double img_len, const float* inject_paf,
                         const float* inject_heat, int face_net_size, double face_thresh, int hand_net_size,
                         double hand_thresh, opb_image_header* header_out, opb_person* persons_out,
                         opb_wb_part* parts_out, int parts_cap, int* n_parts, double* face_out, int32_t* face_valid,
                         double* hand_out, int32_t* hand_valid, uint8_t* picture_out) {
  int frame_parts[2];
  return opb_whole_body_batch(pose, face, hand, img, img_loc, 1, orig_h, orig_w, in_h, in_w, map_h, map_w, img_len,
                              inject_paf, inject_heat, face_net_size, face_thresh, hand_net_size, hand_thresh, header_out,
                              persons_out, parts_out, parts_cap, n_parts, frame_parts, face_out, face_valid, hand_out,
                              hand_valid, picture_out);
}

int opb_test_whole_body_boxes(opb_ctx* ctx, const opb_person* persons, int n, double sx, double sy, double* unit_out,
                              int32_t* boxes_out, int32_t* present_out, int32_t* parts_out, int* n_parts) {
  if (!ctx) return OPB_ERR_ARG;
  if (n < 0 || n > (1 << 16) || (n > 0 && (!persons || !unit_out || !boxes_out || !present_out || !parts_out)) ||
      !n_parts || !std::isfinite(sx) || !std::isfinite(sy))
    OPB_FAIL(ctx, OPB_ERR_ARG, "test_whole_body_boxes: bad arguments");
  cudaSetDevice(ctx->device);
  const int cap = std::max(n, 1);
  const WbLayout L = wb_layout(cap);
  const size_t rec_b = sizeof(ImageHeader) + sizeof(PersonOut) * static_cast<size_t>(cap);
  WbOut wo;
  int rc;
  if ((rc = wb_reserve(ctx, cap, 1, rec_b, L.total, &wo))) return rc;
  ImageHeader* d_hd = reinterpret_cast<ImageHeader*>(ctx->wb_buf + L.total);
  PersonOut* d_persons = reinterpret_cast<PersonOut*>(ctx->wb_buf + L.total + sizeof(ImageHeader));
  const ImageHeader hd{1, n, 0, 0};
  if ((rc = copy_in(ctx, d_hd, &hd, sizeof(hd), OPB_HOST))) return rc;
  if (n > 0 && (rc = copy_in(ctx, d_persons, persons, sizeof(PersonOut) * n, OPB_HOST))) return rc;
  if ((rc = wb_launch(ctx, d_hd, d_persons, 1, cap, sx, sy, wo))) return rc;
  OPB_CUDA(ctx, cudaMemcpyAsync(ctx->wb_host, ctx->wb_buf, L.total, cudaMemcpyDeviceToHost, ctx->stream));
  OPB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  const uint8_t* hb = ctx->wb_host;
  const WbCounts cnt = *reinterpret_cast<const WbCounts*>(hb + L.counts);
  if (cnt.status != 0) OPB_FAIL(ctx, cnt.status, "test_whole_body_boxes: a crop box edge does not fit int32");
  if (n > 0) {
    std::memcpy(unit_out, hb + L.unit, sizeof(double) * n);
    std::memcpy(boxes_out, hb + L.box, sizeof(int) * 12 * n);
    std::memcpy(present_out, hb + L.present, sizeof(int) * n);
  }
  const WbPart* parts = reinterpret_cast<const WbPart*>(hb + L.parts);
  for (int i = 0; i < cnt.n_parts; ++i) {
    parts_out[2 * i] = parts[i].person;
    parts_out[2 * i + 1] = parts[i].side;
  }
  *n_parts = cnt.n_parts;
  return OPB_OK;
}

int opb_test_whole_body_boxes_batch(opb_ctx* ctx, const opb_image_header* headers, const opb_person* persons, int n,
                                    int cap, double sx, double sy, int32_t* counts_out, double* unit_out,
                                    int32_t* boxes_out, int32_t* present_out, opb_crop* face_out, opb_crop* hand_out,
                                    int32_t* parts_out) {
  if (!ctx) return OPB_ERR_ARG;
  if (n < 1 || cap < 1 || static_cast<long long>(n) * cap > (1 << 16) || !headers || !persons || !counts_out ||
      !unit_out || !boxes_out || !present_out || !face_out || !hand_out || !parts_out || !std::isfinite(sx) ||
      !std::isfinite(sy))
    OPB_FAIL(ctx, OPB_ERR_ARG, "test_whole_body_boxes_batch: bad arguments");
  cudaSetDevice(ctx->device);
  const size_t c = static_cast<size_t>(n) * cap;
  const WbLayout L = wb_layout(cap, n);
  const size_t hd_b = (sizeof(ImageHeader) * n + 255) & ~size_t(255);
  WbOut wo;
  int rc;
  if ((rc = wb_reserve(ctx, cap, n, hd_b + sizeof(PersonOut) * c, L.total, &wo))) return rc;
  ImageHeader* d_hd = reinterpret_cast<ImageHeader*>(ctx->wb_buf + L.total);
  PersonOut* d_persons = reinterpret_cast<PersonOut*>(ctx->wb_buf + L.total + hd_b);
  if ((rc = copy_in(ctx, d_hd, headers, sizeof(ImageHeader) * n, OPB_HOST))) return rc;
  if ((rc = copy_in(ctx, d_persons, persons, sizeof(PersonOut) * c, OPB_HOST))) return rc;
  // outputs a frame does not write (error status, no peaks, persons past n_persons) read back as zero
  OPB_CUDA(ctx, cudaMemsetAsync(ctx->wb_buf, 0, L.total, ctx->stream));
  if ((rc = wb_launch(ctx, d_hd, d_persons, n, cap, sx, sy, wo))) return rc;
  OPB_CUDA(ctx, cudaMemcpyAsync(ctx->wb_host, ctx->wb_buf, L.total, cudaMemcpyDeviceToHost, ctx->stream));
  OPB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  const uint8_t* hb = ctx->wb_host;
  std::memcpy(counts_out, hb + L.counts, sizeof(WbCounts) * n);
  std::memcpy(unit_out, hb + L.unit, sizeof(double) * c);
  std::memcpy(boxes_out, hb + L.box, sizeof(int) * 12 * c);
  std::memcpy(present_out, hb + L.present, sizeof(int) * c);
  std::memcpy(face_out, hb + L.face, sizeof(WbCrop) * c);
  std::memcpy(hand_out, hb + L.hand, sizeof(WbCrop) * 2 * c);
  std::memcpy(parts_out, hb + L.parts, sizeof(WbPart) * 3 * c);
  return OPB_OK;
}

void* opb_device_buffer(opb_ctx* ctx, int which) {
  if (!ctx) return nullptr;
  Chain* ch = ctx->last_chain;
  PostWs* ws = ctx->last_post;
  switch (which) {
    case 0: return ch ? ch->paf_lo : nullptr;
    case 1: return ch ? ch->heat_lo : nullptr;
    case 2: return ws ? ws->pafs : nullptr;
    case 3: return ws ? ws->heat : nullptr;
    case 4: return ws ? ws->headers : nullptr;
    case 5: return ws ? ws->persons : nullptr;
    case 6: return ws ? ws->peaks : nullptr;
    default: return nullptr;
  }
}

int opb_time_stage(opb_ctx* ctx, const char* stage, int reps, float* ms) {
  if (!ctx || !stage || !ms || reps <= 0) return OPB_ERR_ARG;
  cudaSetDevice(ctx->device);
  Chain* ch = ctx->last_chain;
  PostWs* ws = ctx->last_post;
  const std::string s(stage);
  cudaEvent_t e0, e1;
  OPB_CUDA(ctx, cudaEventCreate(&e0));
  OPB_CUDA(ctx, cudaEventCreate(&e1));
  int rc = OPB_OK;
  int n_launch = 0;
  auto run_once = [&]() -> int {
    if (s == "upsample_paf" || s == "upsample_heat" || s == "peaks" || s == "paf_integral" || s == "limb_assign" ||
        s == "group") {
      if (!ws || (!ch && !ws->last_paf_lo)) { ctx->err = "no cached pipeline to time"; return OPB_ERR_STATE; }
      const int n = ws->N, h8 = ws->last_h8 ? ws->last_h8 : ch->H / 8, w8 = ws->last_w8 ? ws->last_w8 : ch->W / 8;
      const float* plo = ws->last_paf_lo ? ws->last_paf_lo : ch->paf_lo;     // same maps as the last batch
      const float* hlo = ws->last_heat_lo ? ws->last_heat_lo : ch->heat_lo;
      const double ilen = ws->last_img_len > 0 ? ws->last_img_len : ws->W;
      if (s == "upsample_paf") { ++n_launch; return launch_upsample(ctx, plo, n * 38, h8, w8, ws->pafs, ws->H, ws->W); }
      if (s == "upsample_heat") { ++n_launch; return launch_upsample(ctx, hlo, n * 19, h8, w8, ws->heat, ws->H, ws->W); }
      if (s == "peaks") {
        if (ctx->fused_peaks == 1 || ctx->fused_peaks == 3) { n_launch += 2; return launch_peaks(ctx, ws, hlo, n, 19, ws->H, ws->W, h8, w8); }
        if (ctx->fused_peaks == 2) { n_launch += 2; return launch_peaks(ctx, ws, hlo, n, 19, ws->H, ws->W, h8, w8, ws->heat); }
        n_launch += 3;
        return launch_peaks(ctx, ws, ws->heat, n, 19, ws->H, ws->W);
      }
      if (s == "paf_integral") {
        n_launch += 2;
        if (ctx->paf_lowres) return launch_connections(ctx, ws, plo, n, ws->H, ws->W, ilen, h8, w8);
        return launch_connections(ctx, ws, ws->pafs, n, ws->H, ws->W, ilen);
      }
      if (s == "limb_assign") {
        ++n_launch;
        dim3 g2(19, n);
        limb_assign_kernel<<<g2, kAssignThreads, 0, ctx->stream>>>(ws->peaks, ws->idx_list, ws->type_start,
                                                                   ctx->prm.max_peaks, 18, ctx->pc, ws->cands, ws->cands_alt,
                                                                   ws->cand_counts, ctx->prm.max_candidates, ws->conns,
                                                                   ws->conn_counts, ctx->conn_cap, ws->status);
        return OPB_OK;
      }
      ++n_launch;
      return launch_group(ctx, ws, n, true);
    }
    if (!ch) { ctx->err = "no cached conv chain to time"; return OPB_ERR_STATE; }
    bool any = false;
    for (Op& op : ch->ops) {
      if (s == "conv_chain" || op.tag == s) {
        any = true;
        ++n_launch;
        int r = launch_op(ctx, ch, op);
        if (r) return r;
      }
    }
    if (!any) { ctx->err = "unknown stage " + s; return OPB_ERR_ARG; }
    return OPB_OK;
  };
  rc = run_once();  // warm-up
  if (!rc) {
    n_launch = 0;
    cudaEventRecord(e0, ctx->stream);
    for (int i = 0; i < reps && !rc; ++i) rc = run_once();
    cudaEventRecord(e1, ctx->stream);
    cudaError_t e = cudaEventSynchronize(e1);
    if (e != cudaSuccess && !rc) { ctx->err = cudaGetErrorString(e); rc = OPB_ERR_CUDA; }
    float t = 0.f;
    cudaEventElapsedTime(&t, e0, e1);
    *ms = t / reps;
  }
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  return rc;
}

int opb_test_conv(opb_ctx* ctx, const float* x, int n, int h, int w, int cin, const float* W, const float* b, int cout,
                  int ksize, int relu, int precision_mode, float* y) {
  if (!ctx || !x || !W || !b || !y) return OPB_ERR_ARG;
  cudaSetDevice(ctx->device);
  const bool split = precision_mode == OPB_PRECISION_PARITY, comp = precision_mode == OPB_PRECISION_COMP;
  const int saved_precision = ctx->precision;
  ctx->precision = precision_mode;
  const int pool = (relu >> 1) & 1;   // bit 1 of `relu`: fuse the 2x2 max-pool (y is then [N,H/2,W/2,Cout])
  relu &= 1;
  if (pool && ((h | w) & 1)) { ctx->precision = saved_precision; OPB_FAIL(ctx, OPB_ERR_ARG, "pooled test conv needs even H, W"); }
  const int oh = pool ? h / 2 : h, ow = pool ? w / 2 : w;
  Chain tmp;
  int rc = OPB_OK;
  const int cin_pad = round_up(cin, 64);
  const int cout_pad = cout <= 48 ? 48 : round_up(cout, 64);
  if (cout_pad > 256 && cout_pad % 256) { ctx->precision = saved_precision; OPB_FAIL(ctx, OPB_ERR_ARG, "test conv: cout must be <=256 or a multiple of 256"); }
  HostLayer L;
  L.cin = cin; L.cout = cout; L.ks = ksize;
  L.W.assign(W, W + static_cast<size_t>(cout) * cin * ksize * ksize);
  L.b.assign(b, b + cout);
  ctx->host_layers["__test__"] = L;
  Act in, out;
  std::vector<__half> hx;
  std::vector<__half> hy;
  do {
    if ((rc = pack_weights(ctx, "__test__", {{"__test__", cout_pad}}, identity_map(cin, cin_pad), ksize, precision_mode))) break;
    if ((rc = alloc_act(ctx, &tmp, &in, n, h, w, cin_pad))) break;
    // (the correction plane of the compensated precision is laid out in whole 64-channel chunks)
    if ((rc = alloc_act(ctx, &tmp, &out, n, oh, ow, comp ? round_up(cout_pad, 64) : cout_pad))) break;
    hx.assign(static_cast<size_t>(n) * h * w * in.Ctot, __float2half(0.f));
    for (size_t pix = 0; pix < static_cast<size_t>(n) * h * w; ++pix)
      for (int c = 0; c < cin; ++c) {
        const float v = x[pix * cin + c];
        const __half hi = __float2half_rn(v);
        hx[pix * in.Ctot + c] = hi;
        if (split) hx[pix * in.Ctot + in.C + c] = __float2half_rn(v - __half2float(hi));
        if (comp) {
          uint8_t* cb = reinterpret_cast<uint8_t*>(&hx[pix * in.Ctot + in.C]) + comp_byte_off(c);
          cb[0] = f32_to_act8((v - __half2float(hi)) * kCompLoScale);
          cb[64] = f32_to_act8(v);
        }
      }
    cudaError_t e = cudaMemcpyAsync(in.p, hx.data(), hx.size() * 2, cudaMemcpyHostToDevice, ctx->stream);
    if (e != cudaSuccess) { ctx->err = cudaGetErrorString(e); rc = OPB_ERR_CUDA; break; }
    ConvSpec s{};
    s.in[0] = &in; s.in_coff[0] = 0; s.wkey[0] = "__test__"; s.out[0] = &out; s.out_coff[0] = 0;
    s.cout_valid[0] = cout; s.n_problems = 1; s.relu = relu; s.pool = pool;
    if ((rc = add_conv(ctx, &tmp, "__test__", s))) break;
    if ((rc = launch_op(ctx, &tmp, tmp.ops[0]))) break;
    hy.resize(static_cast<size_t>(n) * oh * ow * out.Ctot);
    e = cudaMemcpyAsync(hy.data(), out.p, hy.size() * 2, cudaMemcpyDeviceToHost, ctx->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    if (e != cudaSuccess) { ctx->err = std::string("test conv: ") + cudaGetErrorString(e); rc = OPB_ERR_CUDA; break; }
    for (size_t pix = 0; pix < static_cast<size_t>(n) * oh * ow; ++pix)
      for (int c = 0; c < cout; ++c) {
        float v = __half2float(hy[pix * out.Ctot + c]);
        if (split) v += __half2float(hy[pix * out.Ctot + out.C + c]);
        if (comp)   // hi + the 8-bit-float lo
          v += act8_to_f32(reinterpret_cast<const uint8_t*>(&hy[pix * out.Ctot + out.C])[comp_byte_off(c)]) / kCompLoScale;
        y[pix * cout + c] = v;
      }
  } while (0);
  cudaStreamSynchronize(ctx->stream);
  free_all(tmp.allocs);
  ctx->host_layers.erase("__test__");
  ctx->packed.erase("__test__");
  ctx->precision = saved_precision;
  return rc;
}

int opb_test_conv_first(opb_ctx* ctx, const void* x, int x_is_u8, int n, int h, int w, float u8_denom, const float* W,
                        const float* b, int precision_mode, uint8_t* out) {
  if (!ctx || !x || !W || !b || !out || n <= 0 || h <= 0 || w <= 0) return OPB_ERR_ARG;
  if (precision_mode != OPB_PRECISION_FAST && precision_mode != OPB_PRECISION_PARITY && precision_mode != OPB_PRECISION_COMP)
    return OPB_ERR_ARG;
  cudaSetDevice(ctx->device);
  const size_t pixels = static_cast<size_t>(n) * h * w;
  std::vector<float> wt(27 * 64);   // [27][64], k = (r*3+s)*3 + c, as load_weights packs conv1_1
  for (int o = 0; o < 64; ++o)
    for (int c = 0; c < 3; ++c)
      for (int t = 0; t < 9; ++t) wt[(t * 3 + c) * 64 + o] = W[(static_cast<size_t>(o) * 3 + c) * 9 + t];
  const int saved_precision = ctx->precision;
  float* const saved_w = ctx->w_first;
  float* const saved_b = ctx->b_first;
  const float saved_denom = ctx->u8_denom;
  Chain tmp;
  Act y;
  int rc = OPB_OK;
  do {
    ctx->precision = precision_mode;
    if ((rc = dev_alloc(ctx, &ctx->w_first, wt.size(), tmp.allocs, false))) break;
    if ((rc = dev_alloc(ctx, &ctx->b_first, 64, tmp.allocs, false))) break;
    if (x_is_u8) { if ((rc = dev_alloc(ctx, &tmp.img_u8, pixels * 3, tmp.allocs, false))) break; }
    else if ((rc = dev_alloc(ctx, &tmp.img_f32, pixels * 3, tmp.allocs, false))) break;
    if ((rc = alloc_act(ctx, &tmp, &y, n, h, w, 64))) break;
    ctx->u8_denom = u8_denom;
    cudaError_t e = cudaMemcpyAsync(ctx->w_first, wt.data(), wt.size() * 4, cudaMemcpyHostToDevice, ctx->stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(ctx->b_first, b, 64 * 4, cudaMemcpyHostToDevice, ctx->stream);
    if (e == cudaSuccess)
      e = x_is_u8 ? cudaMemcpyAsync(tmp.img_u8, x, pixels * 3, cudaMemcpyHostToDevice, ctx->stream)
                  : cudaMemcpyAsync(tmp.img_f32, x, pixels * 3 * 4, cudaMemcpyHostToDevice, ctx->stream);
    if (e != cudaSuccess) { ctx->err = cudaGetErrorString(e); rc = OPB_ERR_CUDA; break; }
    Op op; op.kind = OP_FIRST; op.tag = "conv1_1"; op.out = y.p; op.N = n; op.H = h; op.W = w; op.C = x_is_u8 ? 1 : 0;
    op.cstride = y.Ctot; op.lo_off = precision_mode == OPB_PRECISION_FAST ? 0 : y.C;
    if ((rc = launch_op(ctx, &tmp, op))) break;
    e = cudaMemcpyAsync(out, y.p, y.bytes(), cudaMemcpyDeviceToHost, ctx->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    if (e != cudaSuccess) { ctx->err = std::string("test conv_first: ") + cudaGetErrorString(e); rc = OPB_ERR_CUDA; break; }
  } while (0);
  cudaStreamSynchronize(ctx->stream);
  free_all(tmp.allocs);
  ctx->precision = saved_precision;
  ctx->w_first = saved_w;
  ctx->b_first = saved_b;
  ctx->u8_denom = saved_denom;
  return rc;
}

static_assert(sizeof(opb_conv_problem) == 72, "opb_conv_problem size");
static_assert(sizeof(opb_conv_record) == 32 + 96 + 32 + 2 * 72, "opb_conv_record size");

static void copy_name(char* dst, size_t cap, const std::string& s) {
  std::memset(dst, 0, cap);
  std::memcpy(dst, s.data(), std::min(s.size(), cap - 1));
}

int opb_test_chain_convs(opb_ctx* ctx, int n, int h, int w, opb_conv_record* out, int cap, int* count) {
  if (!ctx || !count || cap < 0 || (cap && !out)) return OPB_ERR_ARG;
  cudaSetDevice(ctx->device);
  Chain* ch = nullptr;
  int rc = get_chain(ctx, n, h, w, &ch);
  if (rc) return rc;
  int k = 0;
  for (const Op& op : ch->ops) {
    if (op.kind != OP_CONV) continue;
    if (k < cap) {
      opb_conv_record& r = out[k];
      std::memset(&r, 0, sizeof(r));
      copy_name(r.tag, sizeof(r.tag), op.tag);
      r.ks = op.ks; r.bn = op.bn; r.drain = op.drain; r.comp = op.P.comp; r.n_problems = op.P.n_problems;
      r.grid = op.grid;
      r.shared_in = op.P.n_problems == 2 && op.rec[0].in.p == op.rec[1].in.p;
      for (int p = 0; p < op.P.n_problems; ++p) {
        const ConvRec& c = op.rec[p];
        const PackedW& pw = ctx->packed.at(c.wkey);
        copy_name(r.wkey[p], sizeof(r.wkey[p]), c.wkey);
        opb_conv_problem& q = r.prob[p];
        q.in_h = c.in.H; q.in_w = c.in.W; q.in_c = c.in.C; q.in_ctot = c.in.Ctot; q.in_coff = c.in_coff;
        q.out_h = c.out.H; q.out_w = c.out.W; q.out_c = c.out.C; q.out_ctot = c.out.Ctot; q.out_coff = c.out_coff;
        q.cout_valid = c.cout_valid; q.relu = c.relu; q.pool = c.pool; q.has_out32 = c.out32 != nullptr;
        q.cin_pad = pw.cin_pad; q.cout_pad = pw.cout_pad; q.acc_scale = pw.acc_scale;
      }
    }
    ++k;
  }
  *count = k;
  if (k > cap) OPB_FAIL(ctx, OPB_ERR_CAPACITY, "test chain convs: " + std::to_string(k) + " records, capacity " + std::to_string(cap));
  return OPB_OK;
}

int opb_test_chain_conv_run(opb_ctx* ctx, int n, int h, int w, int index, const void* in0, const void* in1,
                            void* out_io, float* out32_0, float* out32_1) {
  if (!ctx || !in0 || !out_io) return OPB_ERR_ARG;
  cudaSetDevice(ctx->device);
  Chain* ch = nullptr;
  int rc = get_chain(ctx, n, h, w, &ch);
  if (rc) return rc;
  const Op* op = nullptr;
  int k = 0;
  for (const Op& o : ch->ops) {
    if (o.kind != OP_CONV) continue;
    if (k++ == index) { op = &o; break; }
  }
  if (!op) OPB_FAIL(ctx, OPB_ERR_ARG, "test chain conv run: no conv launch " + std::to_string(index));
  const int np = op->P.n_problems;
  const ConvRec* rec = op->rec;
  const Act& out = rec[0].out;
  if (!out.p) OPB_FAIL(ctx, OPB_ERR_UNSUPPORTED, "test chain conv run: the op writes no activation tensor");
  float* const o32[2] = {out32_0, out32_1};
  for (int p = 0; p < np; ++p) {
    if (rec[p].out.p != out.p) OPB_FAIL(ctx, OPB_ERR_UNSUPPORTED, "test chain conv run: the problems write two tensors");
    if (rec[p].in.p == out.p) OPB_FAIL(ctx, OPB_ERR_UNSUPPORTED, "test chain conv run: the op reads its own output");
    if (rec[p].out32 && !o32[p]) OPB_FAIL(ctx, OPB_ERR_ARG, "test chain conv run: missing fp32 map buffer");
  }
  const bool second_in = np == 2 && rec[1].in.p != rec[0].in.p;
  if (second_in && !in1) OPB_FAIL(ctx, OPB_ERR_ARG, "test chain conv run: problem 1 reads its own input tensor");
  auto planes_bytes = [&](int p) { return static_cast<size_t>(out.N) * rec[p].cout_valid * out.H * out.W * sizeof(float); };
  OPB_CUDA(ctx, cudaMemcpyAsync(rec[0].in.p, in0, rec[0].in.bytes(), cudaMemcpyHostToDevice, ctx->stream));
  if (second_in) OPB_CUDA(ctx, cudaMemcpyAsync(rec[1].in.p, in1, rec[1].in.bytes(), cudaMemcpyHostToDevice, ctx->stream));
  OPB_CUDA(ctx, cudaMemcpyAsync(out.p, out_io, out.bytes(), cudaMemcpyHostToDevice, ctx->stream));
  for (int p = 0; p < np; ++p)
    if (rec[p].out32) OPB_CUDA(ctx, cudaMemcpyAsync(rec[p].out32, o32[p], planes_bytes(p), cudaMemcpyHostToDevice, ctx->stream));
  if ((rc = launch_op(ctx, ch, *op))) return rc;
  OPB_CUDA(ctx, cudaMemcpyAsync(out_io, out.p, out.bytes(), cudaMemcpyDeviceToHost, ctx->stream));
  for (int p = 0; p < np; ++p)
    if (rec[p].out32) OPB_CUDA(ctx, cudaMemcpyAsync(o32[p], rec[p].out32, planes_bytes(p), cudaMemcpyDeviceToHost, ctx->stream));
  OPB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return OPB_OK;
}

static_assert(sizeof(opb_kp_stage_crop) == 32, "opb_kp_stage_crop size");
static_assert(sizeof(opb_channel_max) == sizeof(ChannelMax), "opb_channel_max mirrors ChannelMax");

int opb_test_keypoint_stages(opb_ctx* ctx, const uint8_t* frames, int n_frames, int frame_h, int frame_w,
                             const opb_kp_stage_crop* crops, int n, int net_size, int planes, const float* maps,
                             double thresh, uint8_t* canvas_out, size_t canvas_cap, float* up_out, float* tmp_out,
                             float* smooth_out, size_t map_cap, opb_channel_max* records_out, size_t records_cap,
                             double* out, int32_t* valid, int64_t* sizes_out) {
  if (!ctx) return OPB_ERR_ARG;
  if (!frames || !crops || !maps || !sizes_out) OPB_FAIL(ctx, OPB_ERR_ARG, "test_keypoint_stages: missing input");
  if (n < 1 || n > 65535 || n_frames < 1 || frame_h <= 0 || frame_w <= 0)
    OPB_FAIL(ctx, OPB_ERR_ARG, "test_keypoint_stages: bad crop count or frame size");
  if (net_size < 16 || net_size > 4096 || net_size % 8)
    OPB_FAIL(ctx, OPB_ERR_ARG, "test_keypoint_stages: net_size must be a multiple of 8 in [16, 4096]");
  if (planes < 1 || planes > 1024) OPB_FAIL(ctx, OPB_ERR_ARG, "test_keypoint_stages: planes must be in [1, 1024]");
  std::vector<KpCrop> table(n);
  for (int i = 0; i < n; ++i) {
    const opb_kp_stage_crop& b = crops[i];
    const long long w = static_cast<long long>(b.right) - b.left, h = static_cast<long long>(b.bottom) - b.top;
    if (w <= 0 || h <= 0 || w > (1 << 20) || h > (1 << 20) || (b.flip != 0 && b.flip != 1) || b.frame < 0 ||
        b.frame >= n_frames || b.vh < 0 || b.vh > h || b.vw < 0 || b.vw > w)
      OPB_FAIL(ctx, OPB_ERR_ARG, "test_keypoint_stages: bad crop row " + std::to_string(i));
    KpCrop& c = table[i];
    c.top = b.top; c.left = b.left; c.h = static_cast<int>(h); c.w = static_cast<int>(w); c.flip = b.flip;
    c.vh = b.vh; c.vw = b.vw; c.frame = b.frame;
  }
  int tiles = 0, rc;
  size_t floats = 0;
  if ((rc = kp_prepare_table(ctx, table, net_size, planes, &tiles, &floats))) return rc;
  size_t slots_total = 0;
  for (int first = 0; first < n; first += std::min(kp_chunk_slots(n - first), n - first))
    slots_total += kp_chunk_slots(n - first);
  const size_t canvas_b = slots_total * net_size * net_size * 3, records = static_cast<size_t>(n) * planes;
  sizes_out[0] = static_cast<int64_t>(canvas_b);
  sizes_out[1] = static_cast<int64_t>(floats);
  sizes_out[2] = static_cast<int64_t>(records);
  if (canvas_cap < canvas_b || map_cap < floats || records_cap < records)
    OPB_FAIL(ctx, OPB_ERR_CAPACITY, "test_keypoint_stages: output capacity below the sizes in sizes_out");
  if (!canvas_out || !up_out || !tmp_out || !smooth_out || !records_out || !out || !valid)
    OPB_FAIL(ctx, OPB_ERR_ARG, "test_keypoint_stages: missing output");
  cudaSetDevice(ctx->device);
  const int h8 = net_size / 8;
  const size_t frame_b = static_cast<size_t>(n_frames) * frame_h * frame_w * 3;
  const size_t maps_in = static_cast<size_t>(n) * (planes + 1) * h8 * h8;
  // sentinels: a NaN bit pattern in every 32-bit word of the float and record buffers, 0xA5 in every canvas byte
  const uint32_t kWord = 0x7FA5A5A5u;
  std::vector<uint32_t> fill(std::max(map_cap, records_cap * 4), kWord);
  std::vector<void*> allocs;
  uint8_t *d_frames = nullptr, *d_canvas = nullptr;
  float *d_maps = nullptr, *d_up = nullptr, *d_tmp = nullptr;
  ChannelMax* d_res = nullptr;
  KpCrop* d_crops = nullptr;
  auto run = [&]() -> int {
    int r;
    if ((r = dev_alloc(ctx, &d_frames, frame_b, allocs, false)) || (r = dev_alloc(ctx, &d_canvas, canvas_cap, allocs, false)) ||
        (r = dev_alloc(ctx, &d_maps, maps_in, allocs, false)) || (r = dev_alloc(ctx, &d_up, map_cap, allocs, false)) ||
        (r = dev_alloc(ctx, &d_tmp, map_cap, allocs, false)) || (r = dev_alloc(ctx, &d_res, records_cap, allocs, false)) ||
        (r = dev_alloc(ctx, &d_crops, table.size(), allocs, false)))
      return r;
    OPB_CUDA(ctx, cudaMemcpyAsync(d_frames, frames, frame_b, cudaMemcpyHostToDevice, ctx->stream));
    OPB_CUDA(ctx, cudaMemcpyAsync(d_maps, maps, maps_in * 4, cudaMemcpyHostToDevice, ctx->stream));
    OPB_CUDA(ctx, cudaMemcpyAsync(d_crops, table.data(), sizeof(KpCrop) * n, cudaMemcpyHostToDevice, ctx->stream));
    OPB_CUDA(ctx, cudaMemsetAsync(d_canvas, 0xA5, canvas_cap, ctx->stream));
    OPB_CUDA(ctx, cudaMemcpyAsync(d_up, fill.data(), map_cap * 4, cudaMemcpyHostToDevice, ctx->stream));
    OPB_CUDA(ctx, cudaMemcpyAsync(d_tmp, fill.data(), map_cap * 4, cudaMemcpyHostToDevice, ctx->stream));
    OPB_CUDA(ctx, cudaMemcpyAsync(d_res, fill.data(), sizeof(ChannelMax) * records_cap, cudaMemcpyHostToDevice, ctx->stream));
    // the chunks of kp_enqueue_table, with the injected maps in place of each chunk's network output
    size_t slot0 = 0;
    for (int first = 0; first < n;) {
      const int slots = kp_chunk_slots(n - first), nc = std::min(slots, n - first);
      if ((r = kp_canvas_enqueue(ctx, d_frames, frame_h, frame_w, d_crops + first, nc, slots,
                                 d_canvas + slot0 * net_size * net_size * 3, net_size)))
        return r;
      if ((r = kp_upsample_enqueue(ctx, d_maps + static_cast<size_t>(first) * (planes + 1) * h8 * h8, planes + 1, planes,
                                   h8, table, d_crops, first, nc, tiles, d_up)))
        return r;
      slot0 += slots;
      first += nc;
    }
    OPB_CUDA(ctx, cudaMemcpyAsync(up_out, d_up, map_cap * 4, cudaMemcpyDeviceToHost, ctx->stream));
    KpWs ws;
    ws.up = d_up; ws.tmp = d_tmp; ws.res = d_res; ws.crops = d_crops;
    ws.h_res = reinterpret_cast<ChannelMax*>(records_out);
    if ((r = kp_peaks_enqueue(ctx, &ws, table, planes, tiles))) return r;
    OPB_CUDA(ctx, cudaMemcpyAsync(records_out + records, d_res + records, sizeof(ChannelMax) * (records_cap - records),
                                  cudaMemcpyDeviceToHost, ctx->stream));
    OPB_CUDA(ctx, cudaMemcpyAsync(canvas_out, d_canvas, canvas_cap, cudaMemcpyDeviceToHost, ctx->stream));
    OPB_CUDA(ctx, cudaMemcpyAsync(tmp_out, d_tmp, map_cap * 4, cudaMemcpyDeviceToHost, ctx->stream));
    OPB_CUDA(ctx, cudaMemcpyAsync(smooth_out, d_up, map_cap * 4, cudaMemcpyDeviceToHost, ctx->stream));
    OPB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    for (int i = 0; i < n; ++i)
      kp_records_to_keypoints(ws.h_res + static_cast<size_t>(i) * planes, planes, table[i].w, thresh,
                              out + static_cast<size_t>(i) * planes * 3, valid + static_cast<size_t>(i) * planes);
    return OPB_OK;
  };
  rc = run();
  cudaStreamSynchronize(ctx->stream);
  free_all(allocs);
  return rc;
}

}  // extern "C"
