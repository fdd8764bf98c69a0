// superpoint.cu - SuperPoint extraction (dimb_sp_*), replacing SuperPointExtractor._extract
// (reference extractors/superpoint.py:107-132) and the MagicLeap graph it drives
// (thirdparty/SuperGluePretrainedNetwork/models/superpoint.py:160-227).
//
// Data layout in HBM: activations are NHWC fp16 in two planes (hi, lo) so that each 3x3 conv is an
// implicit GEMM whose A tile for one filter tap is a plain 4D TMA box (see gemm.cuh); weights are
// [Cout][tap*Cin + c] fp16 hi/lo.  Pipeline per call (B images):
//   sp_conv1a (CUDA cores, Cin=1)        -> a1   64@HxW
//   conv1b  +ReLU+pool (wgmma)           -> a1p  64@H/2
//   conv2a, conv2b+pool                  -> a2p  64@H/4
//   conv3a, conv3b+pool                  -> a3p 128@H/8
//   conv4a, conv4b                       -> feat 128@h x w
//   convPa (3x3) -> convPb (1x1, fp32 logits) -> sp_softmax_d2s -> scores 8h x 8w
//   sp_nms (2 refinement rounds, exact ==) -> sp_count/scan/compact -> sp_select (radix select + bitonic)
//   convDa (3x3) -> convDb (1x1, fp32)   -> sp_describe (normalise, bilinear, normalise)
#include <algorithm>
#include <memory>
#include <cmath>
#include <cstring>

#include "conv3x3.cuh"
#include "detect.cuh"
#include "gemm.cuh"
#include "sp_head.cuh"

namespace {

// ------------------------------------------------------------------ conv1a: Cin = 1, direct, CUDA cores
// block = 16x16 pixels, one thread per pixel; two passes of 32 output channels (low register count -> 3 CTAs/SM).
// The normalised (image / 255) halo tile and the tap-major weights live in shared memory (weights are read as
// broadcast float4); results are staged in swizzled shared memory and written out as 512 B contiguous runs.
// conv1a weights [9 taps][64] + bias [64] travel as a __grid_constant__ kernel parameter: parameters live in the constant
// bank, the compiler pulls them into uniform registers (LDCU) and every FMA takes its weight as a uniform-register operand -
// no per-thread load instruction (the kernel is bound by the L1 / shared-memory pipe) - and, unlike a __constant__ symbol,
// each launch carries the weights of its own handle (same SASS as the symbol version: 591 FFMA + 163 LDCU).
struct Conv1aW {
  float v[576 + 64];
};

__global__ void __launch_bounds__(256, 3) sp_conv1a_kernel(const __grid_constant__ Conv1aW c_w, const float* __restrict__ img,
                                                           __half* __restrict__ hi, __half* __restrict__ lo, int H, int W) {
  const float* c_conv1a = c_w.v;
  extern __shared__ __align__(16) uint8_t c1smem[];
  float (*tin)[18] = reinterpret_cast<float (*)[18]>(c1smem);  // [18][18]
  uint8_t* sthi = c1smem + 4096;                            // [256 px][128 B], 16B chunks XOR-swizzled by (px & 7)
  uint8_t* stlo = sthi + 256 * 128;
  const int tid = threadIdx.y * 16 + threadIdx.x;
  const int b = blockIdx.z, y0 = blockIdx.y * 16, x0 = blockIdx.x * 16;
  const float* im = img + static_cast<size_t>(b) * H * W;
  for (int i = tid; i < 18 * 18; i += 256) {
    const int yy = y0 + i / 18 - 1, xx = x0 + i % 18 - 1;
    tin[i / 18][i % 18] = (yy >= 0 && yy < H && xx >= 0 && xx < W) ? __fdiv_rn(im[static_cast<size_t>(yy) * W + xx], 255.f) : 0.f;
  }
  __syncthreads();
  float a[9];
#pragma unroll
  for (int t = 0; t < 9; ++t) a[t] = tin[threadIdx.y + t / 3][threadIdx.x + t % 3];
#pragma unroll
  for (int pass = 0; pass < 2; ++pass) {
    float acc[32];
#pragma unroll
    for (int c = 0; c < 32; ++c) acc[c] = c_conv1a[576 + pass * 32 + c];
#pragma unroll
    for (int t = 0; t < 9; ++t) {
#pragma unroll
      for (int c = 0; c < 32; ++c) acc[c] = fmaf(a[t], c_conv1a[t * 64 + pass * 32 + c], acc[c]);
    }
#pragma unroll
    for (int g8 = 0; g8 < 4; ++g8) {
      __half2 h[4], l[4];
#pragma unroll
      for (int j = 0; j < 4; ++j)
        split2_f32(fmaxf(acc[g8 * 8 + 2 * j], 0.f), fmaxf(acc[g8 * 8 + 2 * j + 1], 0.f), h[j], l[j]);
      const int chunk = pass * 4 + g8;
      const uint32_t off = static_cast<uint32_t>(tid * 128 + (((chunk ^ tid) & 7) << 4));
      *reinterpret_cast<uint4*>(sthi + off) = *reinterpret_cast<uint4*>(h);
      *reinterpret_cast<uint4*>(stlo + off) = *reinterpret_cast<uint4*>(l);
    }
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int L = i * 256 + tid;
    const int ty = L >> 7, rem = L & 127, tx = rem >> 3, chunk = rem & 7;
    const int y = y0 + ty, x = x0 + tx, px = ty * 16 + tx;
    if (y >= H || x >= W) continue;
    const uint32_t off = static_cast<uint32_t>(px * 128 + (((chunk ^ px) & 7) << 4));
    const size_t g = ((static_cast<size_t>(b) * H + y) * W + x) * 64 + chunk * 8;
    *reinterpret_cast<uint4*>(hi + g) = *reinterpret_cast<const uint4*>(sthi + off);
    if (lo) *reinterpret_cast<uint4*>(lo + g) = *reinterpret_cast<const uint4*>(stlo + off);
  }
}

}  // namespace

struct dimb_sp {
  std::vector<void*> mem;  // device memory owned by this handle
  dimb_ctx* ctx;
  dimb_sp_conf conf;
  // weights
  Conv1aW w1a;  // conv1a weights, tap-major [9][64] + bias [64] (host copy: passed by value with every launch)
  ConvLayer L[11];  // conv1b conv2a conv2b conv3a conv3b conv4a conv4b convPa convPb convDa convDb
  // workspace (sized for max_batch x max_height x max_width)
  float* img = nullptr;
  __half *a1h, *a1l, *a1ph, *a1pl, *a2h, *a2l, *a2ph, *a2pl, *a3h, *a3l, *a3ph, *a3pl, *a4h, *a4l, *fth, *ftl, *pah, *pal,
      *dah, *dal;
  float *logits, *ddesc, *scores, *nms, *cand_score, *sel_score;
  int *cand_idx, *chunk_count, *chunk_off, *cand_count, *sel_idx = nullptr;
  float *o_kpts = nullptr, *o_scores = nullptr, *o_desc = nullptr;
  int* o_counts = nullptr;
  int o_cap = 0, sel_cap = 0;
  TopkScratch topk;  // grid-wide top-k (max_keypoints > kMaxTopK)
  // last-call geometry (debug taps)
  int lastB = 0, lastH = 0, lastW = 0;
};

namespace {

enum { L1B = 0, L2A, L2B, L3A, L3B, L4A, L4B, LPA, LPB, LDA, LDB };

// 1x1 conv = GEMM over cells, fp32 output [cells][ldc]
int run_conv1_f32(dimb_sp* sp, cudaStream_t st, const ConvLayer& L, const __half* inh, const __half* inl, float* out, int cells,
                  int ldc, const char* tag) {
  dimb_ctx* ctx = sp->ctx;
  TcOperands ops;
  DIMB_TRY(dimb_tmap_2d(ctx, &ops.Ah, inh, cells, L.cin, L.cin, kTileM));
  DIMB_TRY(dimb_tmap_2d(ctx, &ops.Al, inl, cells, L.cin, L.cin, kTileM));
  ops.Bh = L.tmBh;
  ops.Bl = L.tmBl;
  GemmArgs g{};
  g.num_kb = L.cin / 64;
  g.M = cells;
  g.N = L.cout;
  EpiStoreF32 epi;
  epi.out = out;
  epi.bias = L.bias;
  epi.ldc = ldc;
  epi.n_valid = L.cout;
  epi.m_valid = cells;
  epi.scale = 1.f;
  return launch_gemm<128, false>(ctx, st, ops, g, epi, ceil_div(cells, kTileM), L.cout_pad, tag);
}

}  // namespace

extern "C" {

int dimb_sp_create(dimb_ctx* ctx, const float* weights, size_t n_floats, const dimb_sp_conf* conf, dimb_sp** out) {
  if (!ctx || !weights || !conf || !out) return DIMB_ERR_ARG;
  *out = nullptr;
  DIMB_CUDA_OK(ctx, cudaSetDevice(ctx->device));
  static const int shp[12][3] = {{64, 1, 3},    {64, 64, 3},   {64, 64, 3},   {64, 64, 3},   {128, 64, 3},  {128, 128, 3},
                                 {128, 128, 3}, {128, 128, 3}, {256, 128, 3}, {65, 256, 1},  {256, 128, 3}, {256, 256, 1}};
  size_t need = 0;
  for (auto& s : shp) need += static_cast<size_t>(s[0]) * s[1] * s[2] * s[2] + s[0];
  if (n_floats != need) {
    dimb_set_error(ctx, "dimb_sp_create: weight blob has " + std::to_string(n_floats) + " floats, expected " + std::to_string(need));
    return DIMB_ERR_ARG;
  }
  if (conf->nms_radius < 0 || conf->nms_radius > 8 || conf->max_keypoints == 0 || conf->max_keypoints < -1 || conf->max_batch < 1 || conf->max_height < 16 || conf->max_width < 16) {
    dimb_set_error(ctx, "dimb_sp_create: unsupported configuration (\"max_keypoints\" must be positive or -1)");
    return DIMB_ERR_ARG;
  }
  dimb_sp* sp = new dimb_sp();
  sp->ctx = ctx;
  std::unique_ptr<dimb_sp, void (*)(dimb_sp*)> guard(sp, dimb_sp_destroy);  // a failed create releases what it built
  OwnerScope own(ctx, &sp->mem);
  sp->conf = *conf;
  const float* p = weights;
  // conv1a stays fp32 on CUDA cores
  {  // conv1a: [64][9] -> tap-major [9][64], bias appended (the layout of c_conv1a)
    float* t = sp->w1a.v;
    for (int i = 0; i < 576; ++i) t[(i % 9) * 64 + i / 9] = p[i];
    for (int i = 0; i < 64; ++i) t[576 + i] = p[576 + i];
  }
  p += 640;
  for (int i = 1; i < 12; ++i) {
    const int co = shp[i][0], ci = shp[i][1], ks = shp[i][2];
    const int bn = conv_bn(co);
    const size_t nw = static_cast<size_t>(co) * ci * ks * ks;
    DIMB_TRY(make_conv_layer(ctx, sp->L[i - 1], p, p + nw, co, ci, ks, bn));
    p += nw + co;
  }
  const size_t B = conf->max_batch, H = conf->max_height, W = conf->max_width;
  const size_t h = H / 8, w = W / 8;
  auto act = [&](__half** hi, __half** lo, size_t n) -> int {
    DIMB_TRY(dimb_alloc_t(ctx, hi, n));
    DIMB_TRY(dimb_alloc_t(ctx, lo, n));
    return (int)DIMB_OK;
  };
  DIMB_TRY(dimb_alloc_t(ctx, &sp->img, B * H * W));
  DIMB_TRY(act(&sp->a1h, &sp->a1l, B * H * W * 64));
  DIMB_TRY(act(&sp->a1ph, &sp->a1pl, B * (H / 2) * (W / 2) * 64));
  DIMB_TRY(act(&sp->a2h, &sp->a2l, B * (H / 2) * (W / 2) * 64));
  DIMB_TRY(act(&sp->a2ph, &sp->a2pl, B * (H / 4) * (W / 4) * 64));
  DIMB_TRY(act(&sp->a3h, &sp->a3l, B * (H / 4) * (W / 4) * 128));
  DIMB_TRY(act(&sp->a3ph, &sp->a3pl, B * h * w * 128));
  DIMB_TRY(act(&sp->a4h, &sp->a4l, B * h * w * 128));
  DIMB_TRY(act(&sp->fth, &sp->ftl, B * h * w * 128));
  DIMB_TRY(act(&sp->pah, &sp->pal, B * h * w * 256));
  DIMB_TRY(act(&sp->dah, &sp->dal, B * h * w * 256));
  DIMB_TRY(dimb_alloc_t(ctx, &sp->logits, B * h * w * 65));
  DIMB_TRY(dimb_alloc_t(ctx, &sp->ddesc, B * h * w * 256));
  DIMB_TRY(dimb_alloc_t(ctx, &sp->scores, B * H * W));
  DIMB_TRY(dimb_alloc_t(ctx, &sp->nms, B * H * W));
  DIMB_TRY(dimb_alloc_t(ctx, &sp->cand_idx, B * H * W));
  DIMB_TRY(dimb_alloc_t(ctx, &sp->cand_score, B * H * W));
  const size_t nch = ceil_div(static_cast<int>(H * W), kChunk);
  DIMB_TRY(dimb_alloc_t(ctx, &sp->chunk_count, B * nch));
  DIMB_TRY(dimb_alloc_t(ctx, &sp->chunk_off, B * nch));
  DIMB_TRY(dimb_alloc_t(ctx, &sp->cand_count, B));
  if (conf->max_keypoints > kMaxTopK) DIMB_TRY(topk_reserve(ctx, sp->topk, static_cast<int>(B), static_cast<int>(H * W), conf->max_keypoints));
  *out = guard.release();
  return DIMB_OK;
}

void dimb_sp_destroy(dimb_sp* sp) {
  if (!sp) return;
  dimb_release(sp->ctx, sp->mem);
  delete sp;
}

int dimb_sp_extract_dev(dimb_sp* sp, const float* d_images, int B, int H, int W, float* d_kpts, float* d_scores, float* d_desc,
                        int* d_counts, int cap, void* stream) {
  if (!sp) return DIMB_ERR_ARG;
  dimb_ctx* ctx = sp->ctx;
  OwnerScope own(ctx, &sp->mem);
  const dimb_sp_conf& cf = sp->conf;
  if (B < 1 || B > cf.max_batch || H > cf.max_height || W > cf.max_width || H < 16 || W < 16 || cap < 1) {
    dimb_set_error(ctx, "dimb_sp_extract: batch/size outside the workspace given at create time");
    return DIMB_ERR_ARG;
  }
  if (cf.max_keypoints > 0 && cap < cf.max_keypoints) {
    dimb_set_error(ctx, "dimb_sp_extract: cap < max_keypoints");
    return DIMB_ERR_ARG;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const bool exact = ctx->precision == DIMB_PRECISION_EXACT;
  const int H2 = H / 2, W2 = W / 2, H4 = H2 / 2, W4 = W2 / 2, h = H4 / 2, w = W4 / 2;
  const int H8 = h * 8, W8 = w * 8;
  sp->lastB = B;
  sp->lastH = H;
  sp->lastW = W;
  {
    ProfScope prof(ctx, st, "sp.conv1a");
    constexpr int c1smem = 4096 + 2 * 256 * 128;
    DIMB_TRY(dimb_func_smem(ctx, sp_conv1a_kernel, c1smem));
    sp_conv1a_kernel<<<dim3(ceil_div(W, 16), ceil_div(H, 16), B), dim3(16, 16), c1smem, st>>>(sp->w1a, d_images, sp->a1h,
                                                                                           exact ? sp->a1l : nullptr, H, W);
    DIMB_LAUNCH_CHECK(ctx);
  }
  DIMB_TRY((run_conv3<64, true>(sp->ctx, st, sp->L[L1B], sp->a1h, sp->a1l, sp->a1ph, sp->a1pl, B, H, W, "sp.conv1b")));
  DIMB_TRY((run_conv3<64, false>(sp->ctx, st, sp->L[L2A], sp->a1ph, sp->a1pl, sp->a2h, sp->a2l, B, H2, W2, "sp.conv2a")));
  DIMB_TRY((run_conv3<64, true>(sp->ctx, st, sp->L[L2B], sp->a2h, sp->a2l, sp->a2ph, sp->a2pl, B, H2, W2, "sp.conv2b")));
  DIMB_TRY((run_conv3<128, false>(sp->ctx, st, sp->L[L3A], sp->a2ph, sp->a2pl, sp->a3h, sp->a3l, B, H4, W4, "sp.conv3a")));
  DIMB_TRY((run_conv3<128, true>(sp->ctx, st, sp->L[L3B], sp->a3h, sp->a3l, sp->a3ph, sp->a3pl, B, H4, W4, "sp.conv3b")));
  DIMB_TRY((run_conv3<128, false>(sp->ctx, st, sp->L[L4A], sp->a3ph, sp->a3pl, sp->a4h, sp->a4l, B, h, w, "sp.conv4a")));
  DIMB_TRY((run_conv3<128, false>(sp->ctx, st, sp->L[L4B], sp->a4h, sp->a4l, sp->fth, sp->ftl, B, h, w, "sp.conv4b")));
  DIMB_TRY((run_conv3<128, false>(sp->ctx, st, sp->L[LPA], sp->fth, sp->ftl, sp->pah, sp->pal, B, h, w, "sp.convPa")));
  DIMB_TRY((run_conv3<128, false>(sp->ctx, st, sp->L[LDA], sp->fth, sp->ftl, sp->dah, sp->dal, B, h, w, "sp.convDa")));
  const int cells = B * h * w;
  DIMB_TRY(run_conv1_f32(sp, st, sp->L[LPB], sp->pah, sp->pal, sp->logits, cells, 65, "sp.convPb"));
  DIMB_TRY(run_conv1_f32(sp, st, sp->L[LDB], sp->dah, sp->dal, sp->ddesc, cells, 256, "sp.convDb"));
  {
    ProfScope prof(ctx, st, "sp.softmax");
    DIMB_TRY(launch_sp_softmax(ctx, st, sp->logits, sp->scores, B, h, w));
  }
  {
    ProfScope prof(ctx, st, "sp.nms");
    DIMB_TRY(launch_nms(ctx, st, sp->scores, sp->nms, B, H8, W8, cf.nms_radius, kNmsProductionVer));
  }
  ProfScope prof_sel(ctx, st, "sp.select+describe");
  const CandBufs cand{sp->chunk_count, sp->chunk_off, sp->cand_count, sp->cand_idx, sp->cand_score};
  DIMB_TRY(launch_candidates(ctx, st, sp->nms, cand, B, H8, W8, cf.keypoint_threshold, cf.remove_borders, nullptr, true));
  if (sp->sel_cap < cap) {  // selection scratch [max_batch][cap]; the smaller buffers of an earlier call are released
    dimb_free(ctx, sp->sel_idx);
    dimb_free(ctx, sp->sel_score);
    DIMB_TRY(dimb_alloc_t(ctx, &sp->sel_idx, static_cast<size_t>(cf.max_batch) * cap));
    DIMB_TRY(dimb_alloc_t(ctx, &sp->sel_score, static_cast<size_t>(cf.max_batch) * cap));
    sp->sel_cap = cap;
  }
  DIMB_TRY(launch_select(ctx, st, cand, sp->sel_idx, sp->sel_score, d_counts, B, H8 * W8, cf.max_keypoints, cap, &sp->topk,
                         false));
  return launch_sp_describe(ctx, st, sp->sel_idx, sp->sel_score, d_counts, sp->ddesc, d_kpts, d_scores, d_desc, B, h, w, cap,
                            cf.fix_sampling);
}

int dimb_sp_extract(dimb_sp* sp, const float* images, int B, int H, int W, float* kpts, float* scores, float* desc, int* counts,
                    int cap) {
  if (!sp || !images || !kpts || !scores || !desc || !counts) return DIMB_ERR_ARG;
  dimb_ctx* ctx = sp->ctx;
  OwnerScope own(ctx, &sp->mem);
  DIMB_CUDA_OK(ctx, cudaSetDevice(ctx->device));
  if (B < 1 || B > sp->conf.max_batch || H > sp->conf.max_height || W > sp->conf.max_width) {
    dimb_set_error(ctx, "dimb_sp_extract: batch/size outside the workspace given at create time");
    return DIMB_ERR_ARG;
  }
  if (!sp->o_kpts || sp->o_cap < cap) {
    for (void* old : {static_cast<void*>(sp->o_kpts), static_cast<void*>(sp->o_scores), static_cast<void*>(sp->o_desc), static_cast<void*>(sp->o_counts)})
      dimb_free(ctx, old);
    DIMB_TRY(dimb_alloc_t(ctx, &sp->o_kpts, static_cast<size_t>(sp->conf.max_batch) * cap * 2));
    DIMB_TRY(dimb_alloc_t(ctx, &sp->o_scores, static_cast<size_t>(sp->conf.max_batch) * cap));
    DIMB_TRY(dimb_alloc_t(ctx, &sp->o_desc, static_cast<size_t>(sp->conf.max_batch) * cap * 256));
    DIMB_TRY(dimb_alloc_t(ctx, &sp->o_counts, sp->conf.max_batch));
    sp->o_cap = cap;
  }
  cudaStream_t st = 0;
  DIMB_CUDA_OK(ctx, cudaMemcpyAsync(sp->img, images, static_cast<size_t>(B) * H * W * sizeof(float), cudaMemcpyHostToDevice, st));
  DIMB_TRY(dimb_sp_extract_dev(sp, sp->img, B, H, W, sp->o_kpts, sp->o_scores, sp->o_desc, sp->o_counts, cap, st));
  DIMB_CUDA_OK(ctx, cudaMemcpyAsync(counts, sp->o_counts, B * sizeof(int), cudaMemcpyDeviceToHost, st));
  DIMB_CUDA_OK(ctx, cudaMemcpyAsync(kpts, sp->o_kpts, static_cast<size_t>(B) * cap * 2 * sizeof(float), cudaMemcpyDeviceToHost, st));
  DIMB_CUDA_OK(ctx, cudaMemcpyAsync(scores, sp->o_scores, static_cast<size_t>(B) * cap * sizeof(float), cudaMemcpyDeviceToHost, st));
  DIMB_CUDA_OK(ctx, cudaMemcpyAsync(desc, sp->o_desc, static_cast<size_t>(B) * cap * 256 * sizeof(float), cudaMemcpyDeviceToHost, st));
  DIMB_CUDA_OK(ctx, cudaStreamSynchronize(st));
  for (int b = 0; b < B; ++b)
    if (counts[b] > cap) {
      dimb_set_error(ctx, "dimb_sp_extract: image " + std::to_string(b) + " has " + std::to_string(counts[b]) +
                              " keypoints > cap " + std::to_string(cap));
      return DIMB_ERR_CAPACITY;
    }
  return DIMB_OK;
}

int dimb_sp_debug_read(dimb_sp* sp, int which, float* out, size_t n_floats) {
  if (!sp || !out) return DIMB_ERR_ARG;
  dimb_ctx* ctx = sp->ctx;
  const int H = sp->lastH, W = sp->lastW, h = H / 8, w = W / 8;
  DIMB_CUDA_OK(ctx, cudaDeviceSynchronize());
  if (which == 0 || which == 1) {
    const size_t n = static_cast<size_t>(h) * 8 * w * 8;
    if (n_floats < n) return DIMB_ERR_ARG;
    DIMB_CUDA_OK(ctx, cudaMemcpy(out, which == 0 ? sp->scores : sp->nms, n * sizeof(float), cudaMemcpyDeviceToHost));
    return DIMB_OK;
  }
  if (which == 2) {
    const size_t n = static_cast<size_t>(h) * w * 128;
    if (n_floats < n) return DIMB_ERR_ARG;
    std::vector<__half> hh(n), ll(n);
    DIMB_CUDA_OK(ctx, cudaMemcpy(hh.data(), sp->fth, n * sizeof(__half), cudaMemcpyDeviceToHost));
    DIMB_CUDA_OK(ctx, cudaMemcpy(ll.data(), sp->ftl, n * sizeof(__half), cudaMemcpyDeviceToHost));
    const bool exact = ctx->precision == DIMB_PRECISION_EXACT;
    for (size_t i = 0; i < n; ++i) out[i] = __half2float(hh[i]) + (exact ? __half2float(ll[i]) : 0.f);
    return DIMB_OK;
  }
  if (which == 3) {
    const size_t n = static_cast<size_t>(h) * w * 256;
    if (n_floats < n) return DIMB_ERR_ARG;
    DIMB_CUDA_OK(ctx, cudaMemcpy(out, sp->ddesc, n * sizeof(float), cudaMemcpyDeviceToHost));
    return DIMB_OK;
  }
  return DIMB_ERR_ARG;
}

}  // extern "C"

extern "C" dimb_ctx* dimb_sp_ctx(dimb_sp* sp) { return sp ? sp->ctx : nullptr; }
