// selftest.cu - test infrastructure of libdimb200_selftest.so, used by tests/ to validate kernels in isolation from the model code:
//   dimb_selftest_gemm / dimb_selftest_conv3x3: the persistent tensor-core GEMM (gemm.cuh) through its production launch, as a plain
//     C = A B^T and as the SuperPoint 3x3 conv layer (conv3x3.cuh);
//   dimb_selftest_gemm_plan: the launch plan of the persistent kernel, host only;
//   dimb_selftest_attention: the flash-attention kernels through their production launches;
//   dimb_selftest_detect: simple_nms, candidate compaction and top-k (detect.cuh) through their production launches;
//   dimb_selftest_nms_plan: the launch plan of simple_nms, host only;
//   dimb_selftest_sp_softmax / dimb_selftest_sp_describe: the SuperPoint head kernels (sp_head.cuh) through their production launches;
//   dimb_selftest_lg_assign / dimb_selftest_lg_tail: the LightGlue assignment and per-layer tail (lg_assign.cuh) through their launch
//     helpers; dimb_selftest_lgx_assign: the shape-generic LightGlue assignment and filter (lgx_assign.cuh) through its launch helper;
//     dimb_selftest_sg_sinkhorn: SuperGlue's Sinkhorn and mutual-max matching (sg_assign.cuh);
//   dimb_selftest_sift_extrema / _ori / _select / _desc: the SIFT extremum refinement, orientation, selection and descriptor kernels
//     (sift_kernels.cuh) through their launch helpers, on caller-given levels, candidates and records;
//   dimb_selftest_aliked_conv_plan / _conv3x3 / _conv1x1 / _avgpool / _pad / _crop / _deform / _fuse / _dkd / _sddh / _threshold: the
//     ALIKED stages (aliked_kernels.cuh) through their launch helpers, on caller-given maps, weights and keypoints;
//   dimb_selftest_nn_stats / _select: the brute-force NN engine (nn_kernels.cuh) through the pieces nn_run calls: prep, top-2 GEMM and
//     merge of both directions on caller-given device sides, and the mode logic and compaction on planted row statistics;
//   dimb_gv_host / dimb_gv_lo_host / dimb_gv_degensac_host / dimb_gv_seven_point_host: the RANSAC arithmetic of gv.cu on the host
//     (ransac8, lo-ransac, degensac, the 7-point solver); dimb_gv_h_from_f3_host / _degenerate_host / _plane_parallax_host: degensac's
//     H from F and three points, dominant-plane test and plane-and-parallax F.
#include <algorithm>
#include <cstring>
#include <vector>

#include "conv3x3.cuh"
#include "gemm.cuh"

extern "C" int dimb_selftest_gemm_plan(int conv, int bn, int split, int const_b, int num_kb, int m_tiles, int n_tiles, int num_sms,
                                       int* out);

namespace {
// run_conv3 on the tile shape of gemm.cuh CONV mode `conv` (1: 8 x 16, 2: 16 x 16, BN 64 only)
template <int BN, bool POOL>
int run_conv3_mode(dimb_ctx* ctx, const ConvLayer& L, const __half* xh, const __half* xl, __half* oh, __half* ol, int B, int H, int W,
                   int conv, const char* tag) {
  if constexpr (BN == 64) {
    if (conv == 2) return run_conv3_tiles<64, POOL, 2>(ctx, 0, L, xh, xl, oh, ol, B, H, W, tag);
  }
  return run_conv3_tiles<BN, POOL, 1>(ctx, 0, L, xh, xl, oh, ol, B, H, W, tag);
}

// gemm.cuh CONV mode of a conv3x3 self-test call: tile 0 = the production choice (conv_mode), 8 = 8 x 16 tiles, 16 = 16 x 16 tiles
// (cout 64 only); -1 when the tile cannot run
int selftest_conv_mode(dimb_ctx* ctx, int tile, int cout, int B, int H, int W) {
  if (tile == 0) return conv_mode(cout, B, H, W, ctx->num_sms);
  if (tile == 8) return 1;
  if (tile == 16 && conv_bn(cout) == 64) return 2;
  return -1;
}

// hash of (seed, i) -> a value in [-1, 1) with 15 significant bits, split into fp16 hi / lo planes (lo null: hi only)
__global__ void fill_split_kernel(__half* __restrict__ hi, __half* __restrict__ lo, size_t n, unsigned seed) {
  for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    uint32_t h = static_cast<uint32_t>(i) * 0x9E3779B1u ^ static_cast<uint32_t>(i >> 32) * 0x85EBCA77u ^ seed;
    h ^= h >> 15;
    h *= 0x2C1B3C6Du;
    h ^= h >> 12;
    const float v = static_cast<float>(h & 0xFFFFu) * (1.f / 32768.f) - 1.f;
    __half a, b;
    split_f32(v, a, b);
    hi[i] = a;
    if (lo) lo[i] = b;
  }
}
__global__ void split_rows_kernel(const float* __restrict__ src, __half* __restrict__ hi, __half* __restrict__ lo, size_t n) {
  const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  __half h, l;
  split_f32(src[i], h, l);
  hi[i] = h;
  lo[i] = l;
}

// temporary device buffers of one self-test call, freed on every return path
struct DevTmp {
  dimb_ctx* ctx;
  std::vector<void*> p;
  ~DevTmp() {
    cudaDeviceSynchronize();
    for (void* q : p) cudaFree(q);
  }
  template <class T>
  int get(T** out, size_t n) {
    DIMB_CUDA_OK(ctx, cudaMalloc(reinterpret_cast<void**>(out), sizeof(T) * (n ? n : 1)));
    p.push_back(*out);
    return DIMB_OK;
  }
  template <class T>
  int upload(T** out, const std::vector<T>& h) {
    DIMB_TRY(get(out, h.size()));
    DIMB_CUDA_OK(ctx, cudaMemcpy(*out, h.data(), sizeof(T) * h.size(), cudaMemcpyHostToDevice));
    return DIMB_OK;
  }
  // fp32 host values -> fp16 hi / lo planes on the device (lo may be null: FAST)
  int split(const std::vector<float>& h, __half** hi, __half** lo) {
    float* d;
    DIMB_TRY(upload(&d, h));
    DIMB_TRY(get(hi, h.size()));
    DIMB_TRY(get(lo, h.size()));
    split_rows_kernel<<<ceil_div(static_cast<int>(h.size()), 256), 256>>>(d, *hi, *lo, h.size());
    DIMB_CUDA_OK(ctx, cudaGetLastError());
    return DIMB_OK;
  }
};

__global__ void join_rows_kernel(const __half* __restrict__ hi, const __half* __restrict__ lo, float* __restrict__ out, size_t n) {
  const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < n) out[i] = __half2float(hi[i]) + (lo ? __half2float(lo[i]) : 0.f);
}

int sync_call(dimb_ctx* ctx, const char* what) {
  cudaError_t ce = cudaGetLastError();
  if (ce == cudaSuccess) ce = cudaDeviceSynchronize();
  if (ce != cudaSuccess) {
    dimb_set_error(ctx, std::string(what) + ": " + cudaGetErrorString(ce));
    return DIMB_ERR_CUDA;
  }
  return DIMB_OK;
}

// out[5] = {resb, sa, sb, smem_bytes, grid} of pers_plan for one instantiation of the kernel
template <int BN, int CONV>
void plan_of(bool split, bool const_b, int num_kb, int m_tiles, int n_tiles, int num_sms, int* out) {
  const PersPlan p = split ? pers_plan<BN, true, CONV>(const_b, num_kb, m_tiles, n_tiles, num_sms)
                           : pers_plan<BN, false, CONV>(const_b, num_kb, m_tiles, n_tiles, num_sms);
  out[0] = p.resb;
  out[1] = p.cfg.sa;
  out[2] = p.cfg.sb;
  out[3] = p.cfg.smem_bytes;
  out[4] = p.grid;
}

// the plan the persistent kernel of ctx runs with
void launch_plan(dimb_ctx* ctx, int conv, int bn, bool const_b, int num_kb, int m_tiles, int n_tiles, int* out) {
  if (!out) return;
  dimb_selftest_gemm_plan(conv, bn, ctx->precision == DIMB_PRECISION_EXACT, const_b, num_kb, m_tiles, n_tiles, ctx->num_sms, out);
}
}  // namespace

// Launch plan of the persistent kernel (gemm.cuh pers_plan, as launch_gemm computes it) for one call shape, host only: no context, no
// device.  conv: 0 plain GEMM (bn 64 / 128 / 256), 1 3x3 conv on 8 x 16 tiles (bn 64 / 128), 2 3x3 conv on 16 x 16 tiles (bn 64),
// 3 32-wide K blocks (bn 256); split: EXACT operands
// (hi / lo planes); const_b: Epi::kConstB of the epilogue; num_kb: B tiles per output tile.  out[5] = {resb, sa, sb, smem_bytes, grid}.
extern "C" int dimb_selftest_gemm_plan(int conv, int bn, int split, int const_b, int num_kb, int m_tiles, int n_tiles, int num_sms,
                                       int* out) {
  if (!out || num_kb < 1 || m_tiles < 1 || n_tiles < 1 || num_sms < 1) return DIMB_ERR_ARG;
  const bool s = split != 0, cb = const_b != 0;
  if (conv == 0 && bn == 64) plan_of<64, 0>(s, cb, num_kb, m_tiles, n_tiles, num_sms, out);
  else if (conv == 0 && bn == 128) plan_of<128, 0>(s, cb, num_kb, m_tiles, n_tiles, num_sms, out);
  else if (conv == 0 && bn == 256) plan_of<256, 0>(s, cb, num_kb, m_tiles, n_tiles, num_sms, out);
  else if (conv == 1 && bn == 64) plan_of<64, 1>(s, cb, num_kb, m_tiles, n_tiles, num_sms, out);
  else if (conv == 1 && bn == 128) plan_of<128, 1>(s, cb, num_kb, m_tiles, n_tiles, num_sms, out);
  else if (conv == 2 && bn == 64) plan_of<64, 2>(s, cb, num_kb, m_tiles, n_tiles, num_sms, out);
  else if (conv == 3 && bn == 256) plan_of<256, 3>(s, cb, num_kb, m_tiles, n_tiles, num_sms, out);
  else return DIMB_ERR_ARG;
  return DIMB_OK;
}

// C = A B^T (+ bias) through launch_gemm with the fp32 store epilogue (EpiStoreF32), precision of the context.
//   A [M][K], B [N][K] host fp32, K a multiple of 64; bias [N] or null; ldc = N.  bn: 64, 128 or 256 (CTA tile width); k32: 32-wide K
//   blocks on SWIZZLE_64B maps (gemm.cuh CONV 3, bn 256), as the LightGlue linears run with DIMB_K32=1.
//   The tensor maps have exactly M and N rows, over allocations padded to whole tiles whose extra rows hold `guard`: rows past M / N
//   reach the MMAs only as TMA out-of-bounds fill.  C [M + 128][N] starts as `guard` everywhere: the M output rows, then a tail that
//   must stay untouched.  plan[5] (may be null): {resb, sa, sb, smem_bytes, grid} of the launch.
extern "C" int dimb_selftest_gemm(dimb_ctx* ctx, const float* A, const float* B, const float* bias, float* C, int M, int N, int K, int bn,
                                  int k32, float guard, int* plan) {
  if (!ctx || !A || !B || !C || K < 64 || K % 64 || M < 1 || N < 1) return DIMB_ERR_ARG;
  if ((bn != 64 && bn != 128 && bn != 256) || (k32 && bn != 256)) return DIMB_ERR_ARG;
  DIMB_CUDA_OK(ctx, cudaSetDevice(ctx->device));
  const int Mp = round_up(M, kTileM), Np = round_up(N, 256), n_pad = round_up(N, bn), mt = Mp / kTileM;
  std::vector<float> a(static_cast<size_t>(Mp) * K, guard), b(static_cast<size_t>(Np) * K, guard);
  std::copy(A, A + static_cast<size_t>(M) * K, a.begin());
  std::copy(B, B + static_cast<size_t>(N) * K, b.begin());
  DevTmp t{ctx, {}};
  __half *ah, *al, *bh, *bl;
  float *d_bias = nullptr, *dC;
  DIMB_TRY(t.split(a, &ah, &al));
  DIMB_TRY(t.split(b, &bh, &bl));
  if (bias) DIMB_TRY(t.upload(&d_bias, std::vector<float>(bias, bias + N)));
  const size_t nc = static_cast<size_t>(M + kTileM) * N;
  DIMB_TRY(t.upload(&dC, std::vector<float>(nc, guard)));
  auto tmap = k32 ? dimb_tmap_2d_sw64 : dimb_tmap_2d;
  TcOperands ops;
  DIMB_TRY(tmap(ctx, &ops.Ah, ah, M, K, K, kTileM));
  DIMB_TRY(tmap(ctx, &ops.Al, al, M, K, K, kTileM));
  DIMB_TRY(tmap(ctx, &ops.Bh, bh, N, K, K, bn));
  DIMB_TRY(tmap(ctx, &ops.Bl, bl, N, K, K, bn));
  GemmArgs g{};
  g.num_kb = K / (k32 ? 32 : 64);
  g.M = M;
  g.N = N;
  EpiStoreF32 e;
  e.out = dC;
  e.bias = d_bias;
  e.ldc = N;
  e.n_valid = N;
  e.m_valid = M;
  e.scale = 1.f;
  if (k32)
    DIMB_TRY((launch_gemm<256, 3>(ctx, 0, ops, g, e, mt, n_pad)));
  else if (bn == 64)
    DIMB_TRY((launch_gemm<64, false>(ctx, 0, ops, g, e, mt, n_pad)));
  else if (bn == 128)
    DIMB_TRY((launch_gemm<128, false>(ctx, 0, ops, g, e, mt, n_pad)));
  else
    DIMB_TRY((launch_gemm<256, false>(ctx, 0, ops, g, e, mt, n_pad)));
  DIMB_TRY(sync_call(ctx, "dimb_selftest_gemm"));
  DIMB_CUDA_OK(ctx, cudaMemcpy(C, dC, sizeof(float) * nc, cudaMemcpyDeviceToHost));
  launch_plan(ctx, k32 ? 3 : 0, bn, EpiStoreF32::kConstB, g.num_kb, mt, n_pad / bn, plan);
  return DIMB_OK;
}

// One SuperPoint 3x3 conv layer (zero padding 1, bias, ReLU, optional 2x2 max pool) through make_conv_layer and run_conv3
// (conv3x3.cuh), precision of the context.
//   x: NHWC fp32 [B][H][W][cin]; w: OIHW fp32 [cout][cin][3][3]; bias [cout]; cin a multiple of 64, cout 64 or a multiple of 128.
//   The input allocation holds one more image of `guard` after the B images, outside the tensor map (B x H x W pixels): a halo read
//   past the last image, or across the image boundary, would bring it in.  `guard` must be finite: the ReLU turns NaN into 0.
//   out: [B + 1][Ho][Wo][cout] with Ho, Wo = H / 2, W / 2 under pool: the B output images joined from their hi + lo planes (hi only in
//   FAST), then one image of tail; every element starts as `sentinel` (fp16-exact), so unwritten and stray writes show.
//   tile: 0 = the tile shape production picks for this call (conv3x3.cuh conv_mode), 8 = 8 x 16 pixels, 16 = 16 x 16 pixels
//   (cout 64 only).
//   plan[6] (may be null): as dimb_selftest_gemm, then the gemm.cuh CONV mode that ran (1 or 2).
extern "C" int dimb_selftest_conv3x3(dimb_ctx* ctx, const float* x, const float* w, const float* bias, float* out, int B, int H, int W,
                                     int cin, int cout, int pool, int tile, float guard, float sentinel, int* plan) {
  if (!ctx || !x || !w || !bias || !out || B < 1 || H < 1 || W < 1 || cin < 64 || cin % 64) return DIMB_ERR_ARG;
  if ((cout != 64 && (cout < 128 || cout % 128)) || (pool && (H < 2 || W < 2))) return DIMB_ERR_ARG;
  const int mode = selftest_conv_mode(ctx, tile, cout, B, H, W);
  if (mode < 0) return DIMB_ERR_ARG;
  DIMB_CUDA_OK(ctx, cudaSetDevice(ctx->device));
  const bool exact = ctx->precision == DIMB_PRECISION_EXACT;
  const int Ho = pool ? H / 2 : H, Wo = pool ? W / 2 : W;
  const size_t img = static_cast<size_t>(H) * W * cin, nout = static_cast<size_t>(B + 1) * Ho * Wo * cout;
  std::vector<float> xin(img * (B + 1), guard);
  std::copy(x, x + img * B, xin.begin());
  DevTmp t{ctx, {}};
  __half *xh, *xl, *oh, *ol;
  float* d_out;
  DIMB_TRY(t.split(xin, &xh, &xl));
  DIMB_TRY(t.split(std::vector<float>(nout, sentinel), &oh, &ol));
  DIMB_TRY(t.get(&d_out, nout));
  ConvLayer L;
  {
    OwnerScope own(ctx, &t.p);  // the layer's weights and bias are this call's temporaries
    DIMB_TRY(make_conv_layer(ctx, L, w, bias, cout, cin, 3, conv_bn(cout)));
  }
  const int bn = conv_bn(cout);
  const char* tag = "selftest.conv3x3";
  if (tile == 0) {  // the production entry itself
    if (bn == 64)
      DIMB_TRY(pool ? (run_conv3<64, true>(ctx, 0, L, xh, xl, oh, ol, B, H, W, tag)) : (run_conv3<64, false>(ctx, 0, L, xh, xl, oh, ol, B, H, W, tag)));
    else
      DIMB_TRY(pool ? (run_conv3<128, true>(ctx, 0, L, xh, xl, oh, ol, B, H, W, tag))
                    : (run_conv3<128, false>(ctx, 0, L, xh, xl, oh, ol, B, H, W, tag)));
  } else if (bn == 64) {
    DIMB_TRY(pool ? (run_conv3_mode<64, true>(ctx, L, xh, xl, oh, ol, B, H, W, mode, tag))
                  : (run_conv3_mode<64, false>(ctx, L, xh, xl, oh, ol, B, H, W, mode, tag)));
  } else {
    DIMB_TRY(pool ? (run_conv3_mode<128, true>(ctx, L, xh, xl, oh, ol, B, H, W, mode, tag))
                  : (run_conv3_mode<128, false>(ctx, L, xh, xl, oh, ol, B, H, W, mode, tag)));
  }
  join_rows_kernel<<<ceil_div(static_cast<int>(nout), 256), 256>>>(oh, exact ? ol : nullptr, d_out, nout);
  DIMB_TRY(sync_call(ctx, "dimb_selftest_conv3x3"));
  DIMB_CUDA_OK(ctx, cudaMemcpy(out, d_out, sizeof(float) * nout, cudaMemcpyDeviceToHost));
  launch_plan(ctx, mode, bn, EpiConvRelu<false>::kConstB, 9 * (cin / 64), conv_m_tiles(B, H, W, mode), L.cout_pad / bn, plan);
  if (plan) plan[5] = mode;
  return DIMB_OK;
}

// Host only: the gemm.cuh CONV mode (tile shape) run_conv3 picks for a conv of B images of H x W with `cout` output channels on a
// device with num_sms SMs (conv3x3.cuh conv_mode), either precision.
extern "C" int dimb_selftest_conv_mode(int cout, int B, int H, int W, int num_sms, int* out) {
  if (!out || B < 1 || H < 1 || W < 1 || num_sms < 1 || cout < 1) return DIMB_ERR_ARG;
  *out = conv_mode(cout, B, H, W, num_sms);
  return DIMB_OK;
}

// Device time of one 3x3 conv layer at a production size, precision of the context: device-generated activations
// [B][H][W][cin] (hi / lo planes), seeded weights, `warm` untimed calls, then `iters` calls between CUDA events.  tile as
// dimb_selftest_conv3x3.  ms: milliseconds per call.  plan[6] (may be null): as dimb_selftest_conv3x3.
extern "C" int dimb_selftest_conv3x3_time(dimb_ctx* ctx, int B, int H, int W, int cin, int cout, int pool, int tile, int warm, int iters,
                                          float* ms, int* plan) {
  if (!ctx || !ms || B < 1 || H < 2 || W < 2 || cin < 64 || cin % 64 || warm < 0 || iters < 1) return DIMB_ERR_ARG;
  if (cout != 64 && (cout < 128 || cout % 128)) return DIMB_ERR_ARG;
  const int mode = selftest_conv_mode(ctx, tile, cout, B, H, W);
  if (mode < 0) return DIMB_ERR_ARG;
  DIMB_CUDA_OK(ctx, cudaSetDevice(ctx->device));
  const bool exact = ctx->precision == DIMB_PRECISION_EXACT;
  const int Ho = pool ? H / 2 : H, Wo = pool ? W / 2 : W;
  const size_t nin = static_cast<size_t>(B) * H * W * cin, nout = static_cast<size_t>(B) * Ho * Wo * cout;
  DevTmp t{ctx, {}};
  __half *xh, *xl, *oh, *ol;
  DIMB_TRY(t.get(&xh, nin));
  DIMB_TRY(t.get(&xl, nin));
  DIMB_TRY(t.get(&oh, nout));
  DIMB_TRY(t.get(&ol, nout));
  fill_split_kernel<<<4 * ctx->num_sms, 256>>>(xh, exact ? xl : nullptr, nin, 12345u);
  DIMB_CUDA_OK(ctx, cudaGetLastError());
  std::vector<float> w(static_cast<size_t>(cout) * cin * 9), bias(cout);
  uint32_t s = 1;
  for (float& v : w) v = static_cast<float>((s = s * 1664525u + 1013904223u) >> 8) * (0.1f / 16777216.f) - 0.05f;
  for (float& v : bias) v = static_cast<float>((s = s * 1664525u + 1013904223u) >> 8) * (0.2f / 16777216.f) - 0.1f;
  ConvLayer L;
  {
    OwnerScope own(ctx, &t.p);
    DIMB_TRY(make_conv_layer(ctx, L, w.data(), bias.data(), cout, cin, 3, conv_bn(cout)));
  }
  const int bn = conv_bn(cout);
  auto run = [&]() {
    const char* tag = "selftest.conv3x3_time";
    if (bn == 64)
      return pool ? run_conv3_mode<64, true>(ctx, L, xh, xl, oh, ol, B, H, W, mode, tag)
                  : run_conv3_mode<64, false>(ctx, L, xh, xl, oh, ol, B, H, W, mode, tag);
    return pool ? run_conv3_mode<128, true>(ctx, L, xh, xl, oh, ol, B, H, W, mode, tag)
                : run_conv3_mode<128, false>(ctx, L, xh, xl, oh, ol, B, H, W, mode, tag);
  };
  for (int i = 0; i < warm; ++i) DIMB_TRY(run());
  cudaEvent_t e0, e1;
  DIMB_CUDA_OK(ctx, cudaEventCreate(&e0));
  DIMB_CUDA_OK(ctx, cudaEventCreate(&e1));
  auto cuda_ok = [&](cudaError_t ce, const char* what) -> int {
    if (ce == cudaSuccess) return DIMB_OK;
    dimb_set_error(ctx, std::string("dimb_selftest_conv3x3_time: ") + what + ": " + cudaGetErrorString(ce));
    return DIMB_ERR_CUDA;
  };
  int rc = cuda_ok(cudaEventRecord(e0, 0), "cudaEventRecord");
  for (int i = 0; i < iters && rc == DIMB_OK; ++i) rc = run();
  if (rc == DIMB_OK) rc = cuda_ok(cudaEventRecord(e1, 0), "cudaEventRecord");
  if (rc == DIMB_OK) rc = sync_call(ctx, "dimb_selftest_conv3x3_time");
  float total = 0.f;
  if (rc == DIMB_OK) rc = cuda_ok(cudaEventElapsedTime(&total, e0, e1), "cudaEventElapsedTime");
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  DIMB_TRY(rc);
  *ms = total / iters;
  launch_plan(ctx, mode, bn, EpiConvRelu<false>::kConstB, 9 * (cin / 64), conv_m_tiles(B, H, W, mode), L.cout_pad / bn, plan);
  if (plan) plan[5] = mode;
  return DIMB_OK;
}

// ------------------------------------------------------------------ attention self-test
#include "attn_hd128.cuh"
#include "lg_kernels.cuh"

namespace {
// LightGlue / SuperGlue attention (lg_kernels.cuh) on operands packed as lightglue.cu packs them
int selftest_attention_lg(dimb_ctx* ctx, const float* Q, const float* K, const float* V, float* out, int S, int NP, const int* n,
                          const int* stopped, int cross, float lazy, float pad, float out_pad) {
  const bool exact = ctx->precision == DIMB_PRECISION_EXACT;
  const size_t nel = static_cast<size_t>(S) * kHeads * NP * kHd, R = static_cast<size_t>(S) * NP;
  std::vector<float> q(nel), k(cross ? 0 : nel), vt(nel);  // q / k [S][4][NP][64], V^T [S][4][64][NP]
  for (int s = 0; s < S; ++s)
    for (int h = 0; h < kHeads; ++h)
      for (int r = 0; r < NP; ++r)
        for (int d = 0; d < kHd; ++d) {
          const size_t i = ((static_cast<size_t>(s) * kHeads + h) * NP + r) * kHd + d;
          const bool live = r < n[s];
          q[i] = live ? Q[i] : pad;
          if (!cross) k[i] = live ? K[i] : pad;
          vt[((static_cast<size_t>(s) * kHeads + h) * kHd + d) * NP + r] = live ? V[i] : pad;
        }
  DevTmp t{ctx, {}};
  __half *qh, *ql, *kh = nullptr, *kl = nullptr, *vh, *vl, *ch, *cl;
  int *d_n, *d_stop;
  DIMB_TRY(t.split(q, &qh, &ql));
  if (!cross) DIMB_TRY(t.split(k, &kh, &kl));
  DIMB_TRY(t.split(vt, &vh, &vl));
  DIMB_TRY(t.split(std::vector<float>(R * kD, out_pad), &ch, &cl));
  DIMB_TRY(t.upload(&d_n, std::vector<int>(n, n + S)));
  DIMB_TRY(t.upload(&d_stop, std::vector<int>(stopped, stopped + S / 2)));
  AttnArgs a;
  a.rows = LgRows{d_n, d_stop, NP};
  a.cross = cross;
  a.ctx_h = ch;
  a.ctx_l = exact ? cl : nullptr;
  a.scale = 0.125f;  // hd^-0.5
  a.lazy = lazy;
  const __half *kh_ = cross ? qh : kh, *kl_ = cross ? ql : kl;  // cross: keys = the q rows of the other side (shared to_qk)
  CUtensorMap mq[2], mk[2], mv[2];  // as lightglue.cu builds them: Q box 128 rows, K box 64 rows, V^T box 64 rows
  const uint64_t rows = static_cast<uint64_t>(S) * kHeads * NP;
  for (int pl = 0; pl < 2; ++pl) {
    DIMB_TRY(dimb_tmap_2d(ctx, &mq[pl], pl ? ql : qh, rows, kHd, kHd, kTileM));
    DIMB_TRY(dimb_tmap_2d(ctx, &mk[pl], pl ? kl_ : kh_, rows, kHd, kHd, kBlkK));
    DIMB_TRY(dimb_tmap_2d(ctx, &mv[pl], pl ? vl : vh, static_cast<uint64_t>(S) * kHeads * kHd, NP, NP, kHd));
  }
  DIMB_TRY(launch_lg_attention(ctx, 0, dim3(1, kHeads, S), mq, mk, mv, a, exact));
  float* d_out;
  DIMB_TRY(t.get(&d_out, R * kD));
  join_rows_kernel<<<ceil_div(static_cast<int>(R * kD), 256), 256>>>(ch, exact ? cl : nullptr, d_out, R * kD);
  DIMB_TRY(sync_call(ctx, "dimb_selftest_attention"));
  DIMB_CUDA_OK(ctx, cudaMemcpy(out, d_out, sizeof(float) * R * kD, cudaMemcpyDeviceToHost));
  return DIMB_OK;
}

// shape-generic attention (attn_hd128.cuh) through hd128_attend, on one pair of two sides of NPp rows (NP rounded up to the query tile):
// side 0 holds Q as its q rows, side 1 K as its q rows and V as its v rows, and side 0 attends to side 1 in the cross form.  With
// n[0] == n[1] side 0 holds K and V itself and attends to its own keys (the self form), side 1 is empty.
int selftest_attention_hd128(dimb_ctx* ctx, const float* Q, const float* K, const float* V, float* out, int H, int hd, int NP, const int* n,
                             float lazy, float pad, float out_pad) {
  const int NPp = round_up(NP, kAttnTile), ld = H * hd, self = n[0] == n[1];
  const size_t side = static_cast<size_t>(NPp) * ld, pl_el = 2 * static_cast<size_t>(H) * NPp * kXHd;
  std::vector<float> q(2 * side, pad), k(2 * side, pad), v(2 * side, pad);  // rows past the live counts: `pad`, not read by the packers
  std::copy(Q, Q + static_cast<size_t>(n[0]) * ld, q.begin());
  std::copy(K, K + static_cast<size_t>(n[1]) * ld, self ? k.begin() : q.begin() + side);
  std::copy(V, V + static_cast<size_t>(n[1]) * ld, self ? v.begin() : v.begin() + side);
  DevTmp t{ctx, {}};
  float *fq, *fk, *fv, *d_out;
  int *d_n, *d_stop;
  Hd128Ops o;
  o.S = 2, o.h = H, o.d = ld, o.hd = hd, o.NP = NPp, o.NPp = NPp;
  DIMB_TRY(t.upload(&fq, q));
  DIMB_TRY(t.upload(&fk, k));
  DIMB_TRY(t.upload(&fv, v));
  DIMB_TRY(t.upload(&d_out, std::vector<float>(2 * side, out_pad)));
  DIMB_TRY(t.upload(&d_n, std::vector<int>{n[0], self ? 0 : n[1]}));
  DIMB_TRY(t.upload(&d_stop, std::vector<int>{0}));
  for (int pl = 0; pl < 2; ++pl)
    for (__half** p : {&o.q[pl], &o.k[pl], &o.vt[pl]}) DIMB_TRY(t.get(p, pl_el));
  DIMB_TRY(hd128_maps(ctx, o));
  DIMB_TRY(hd128_attend(ctx, 0, o, 2, fq, fk, fv, !self, d_n, d_stop, lazy, d_out));
  DIMB_TRY(sync_call(ctx, "dimb_selftest_attention"));
  DIMB_CUDA_OK(ctx, cudaMemcpy(out, d_out, sizeof(float) * side, cudaMemcpyDeviceToHost));
  return DIMB_OK;
}
}  // namespace

// Flash attention (attention.cuh) through its production launches, on host fp32 operands; precision from ctx.
//   variant 0: lg_attn_kernel (LightGlue / SuperGlue, H = 4 heads of hd = 64) via launch_lg_attention.  Q, K, V [S][4][NP][64] (S even,
//     NP a multiple of 128), live rows n[S], stopped[S / 2]
//     (nonzero: the pair is stopped); cross: the keys of side s are the q rows of side s ^ 1 (K unused, may be null).  out: the
//     context buffer [S * NP][256], hi + lo planes (hi only in FAST), every row.
//   variant 1: lgx_attn_tc_kernel (head dim hd <= 128, even, padded to 128) via hd128_attend, which packs the operands
//     (lgx_pack_rows_kernel / lgx_pack_vt_kernel) as the shape-generic LightGlue runs them: the cross form, or the self form when
//     n[0] == n[1].  Q [n[0]][H * hd], K / V [n[1]][H * hd], NP >= n[0], n[1]; S, stopped and cross unused.  out: [NPp][H * hd] fp32
//     with NPp = NP rounded up to 128.
// Every Q / K / V row past the live counts holds `pad` (stale values of earlier layers in production), and the output
// buffer starts as `out_pad`, so rows the kernel must not write can be checked.  lazy: rescale threshold in log2 units, in
// [0, kAttnLazyMax]; negative = the context's (DIMB_ATTN_LAZY).
extern "C" int dimb_selftest_attention(dimb_ctx* ctx, int variant, const float* Q, const float* K, const float* V, float* out, int S,
                                       int H, int hd, int NP, const int* n, const int* stopped, int cross, float lazy, float pad,
                                       float out_pad) {
  if (!ctx || !Q || !V || !out || !n || NP < 1) return DIMB_ERR_ARG;
  if (lazy < 0.f)
    lazy = ctx->attn_lazy;
  else if (!(lazy <= kAttnLazyMax))  // NaN and inf included
    return DIMB_ERR_ARG;
  DIMB_CUDA_OK(ctx, cudaSetDevice(ctx->device));
  if (variant == 0) {
    if (!stopped || (!cross && !K) || H != kHeads || hd != kHd || S < 2 || S % 2 || NP % kAttnTile) return DIMB_ERR_ARG;
    for (int s = 0; s < S; ++s)
      if (n[s] < 0 || n[s] > NP) return DIMB_ERR_ARG;
    return selftest_attention_lg(ctx, Q, K, V, out, S, NP, n, stopped, cross, lazy, pad, out_pad);
  }
  if (variant == 1) {
    if (!K || H < 1 || hd < 2 || hd > kXHd || hd % 2 || n[0] < 0 || n[1] < 0 || n[0] > NP || n[1] > NP) return DIMB_ERR_ARG;
    return selftest_attention_hd128(ctx, Q, K, V, out, H, hd, NP, n, lazy, pad, out_pad);
  }
  return DIMB_ERR_ARG;
}

// ------------------------------------------------------------------ keypoint detection and the SuperPoint head kernels
#include <climits>

#include "detect.cuh"
#include "sp_head.cuh"

namespace {
constexpr int kDetTail = 1024;  // elements past the last valid one in every output buffer of these entries

// nms_plan version of a self-test cut: 0 = the production choice (kNmsProductionVer), 1 = first cut, 2 = bit-mask kernel
// (radii 1..5 only); -1 when the cut cannot run at radius r
int version_of_cut(int r, int cut) {
  if (r < 0 || r > 8) return -1;
  if (cut == 0) return kNmsProductionVer;
  if (cut == 1) return 1;
  if (cut == 2 && r >= 1 && r <= 5) return 2;
  return -1;
}

void plan_out(const NmsPlan& p, int* out) {
  out[0] = p.kernel;
  out[1] = p.tile;
  out[2] = p.threads;
  out[3] = p.smem;
}

// int buffers start as the bit pattern of the float sentinel
int sentinel_bits(float sentinel) {
  int v;
  memcpy(&v, &sentinel, sizeof v);
  return v;
}

template <class T>
int download(dimb_ctx* ctx, T* host, const T* dev, size_t n) {
  DIMB_CUDA_OK(ctx, cudaMemcpy(host, dev, sizeof(T) * n, cudaMemcpyDeviceToHost));
  return DIMB_OK;
}
}  // namespace

// Launch plan of simple_nms at radius r (detect.cuh nms_plan), host only.  cut 0: the production choice (bit-mask kernel for radii
// 1..5, first cut otherwise), 1: the first cut (sp_nms_kernel, radii 0..8), 2: the bit-mask kernel (sp_nms2_kernel,
// radii 1..5).  out[4] = {kernel (1 first cut, 2 bit-mask), tile, threads, dynamic shared memory bytes}.
extern "C" int dimb_selftest_nms_plan(int r, int cut, int* out) {
  const int ver = version_of_cut(r, cut);
  if (!out || ver < 0) return DIMB_ERR_ARG;
  plan_out(nms_plan(r, ver), out);
  return DIMB_OK;
}

// simple_nms, candidate compaction and top-k (detect.cuh) through the launch helpers SuperPoint and ALIKED run, on host fp32 scores
// [B][H][W] (positive: the select kernel orders scores by their bits).
//   r, cut: radius and kernel as dimb_selftest_nms_plan.
//   thr >= 0: candidates are nms > thr; thr_per_image [B] (may be null) replaces it through the device-threshold argument, as ALIKED
//   passes its threshold.  border: candidates lie at least `border` pixels inside the image.  K: top-k (-1 keeps every candidate, in
//   row-major order), 1..kMaxTopK; cap >= K: selection slots per image.
// Every output buffer holds kDetTail more elements after the valid ones, and starts as `sentinel` (int buffers: its bit pattern):
//   nms [B H W], cand_count [B], cand_idx / cand_score [B][H W] (image b's first cand_count[b] entries are valid), sel_idx / sel_score
//   [B][cap] (image b's first min(sel_count[b], cap)), sel_count [B].  plan[4] (may be null): the simple_nms plan that ran.
extern "C" int dimb_selftest_detect(dimb_ctx* ctx, const float* scores, int B, int H, int W, int r, int cut, float thr,
                                    const float* thr_per_image, int border, int K, int cap, float sentinel, float* nms, int* cand_count,
                                    int* cand_idx, float* cand_score, int* sel_idx, float* sel_score, int* sel_count, int* plan) {
  if (!ctx || !scores || !nms || !cand_count || !cand_idx || !cand_score || !sel_idx || !sel_score || !sel_count) return DIMB_ERR_ARG;
  if (B < 1 || H < 1 || W < 1 || static_cast<long long>(B) * H * W > INT_MAX || border < 0 || !(thr >= 0.f)) return DIMB_ERR_ARG;
  if (K == 0 || K < -1 || K > kMaxTopK || cap < 1 || K > cap) return DIMB_ERR_ARG;
  if (thr_per_image)
    for (int b = 0; b < B; ++b)
      if (!(thr_per_image[b] >= 0.f)) return DIMB_ERR_ARG;
  const int ver = version_of_cut(r, cut);
  if (ver < 0) return DIMB_ERR_ARG;
  DIMB_CUDA_OK(ctx, cudaSetDevice(ctx->device));
  const int HW = H * W, nch = ceil_div(HW, kChunk);
  const size_t npix = static_cast<size_t>(B) * HW, nsel = static_cast<size_t>(B) * cap;
  const int isent = sentinel_bits(sentinel);
  DevTmp t{ctx, {}};
  float *d_scores, *d_nms, *d_cs, *d_ss, *d_thr = nullptr;
  int *d_cc, *d_ci, *d_si, *d_sc;
  CandBufs c;
  DIMB_TRY(t.upload(&d_scores, std::vector<float>(scores, scores + npix)));
  DIMB_TRY(t.upload(&d_nms, std::vector<float>(npix + kDetTail, sentinel)));
  DIMB_TRY(t.upload(&d_cc, std::vector<int>(B + kDetTail, isent)));
  DIMB_TRY(t.upload(&d_ci, std::vector<int>(npix + kDetTail, isent)));
  DIMB_TRY(t.upload(&d_cs, std::vector<float>(npix + kDetTail, sentinel)));
  DIMB_TRY(t.upload(&d_si, std::vector<int>(nsel + kDetTail, isent)));
  DIMB_TRY(t.upload(&d_ss, std::vector<float>(nsel + kDetTail, sentinel)));
  DIMB_TRY(t.upload(&d_sc, std::vector<int>(B + kDetTail, isent)));
  DIMB_TRY(t.get(&c.chunk_count, static_cast<size_t>(B) * nch));
  DIMB_TRY(t.get(&c.chunk_off, static_cast<size_t>(B) * nch));
  if (thr_per_image) DIMB_TRY(t.upload(&d_thr, std::vector<float>(thr_per_image, thr_per_image + B)));
  c.cand_count = d_cc;
  c.cand_idx = d_ci;
  c.cand_score = d_cs;
  DIMB_TRY(launch_nms(ctx, 0, d_scores, d_nms, B, H, W, r, ver));
  DIMB_TRY(launch_candidates(ctx, 0, d_nms, c, B, H, W, thr, border, d_thr, true));
  DIMB_TRY(launch_select(ctx, 0, c, d_si, d_ss, d_sc, B, HW, K, cap, nullptr, false));
  DIMB_TRY(sync_call(ctx, "dimb_selftest_detect"));
  DIMB_TRY(download(ctx, nms, d_nms, npix + kDetTail));
  DIMB_TRY(download(ctx, cand_count, d_cc, B + kDetTail));
  DIMB_TRY(download(ctx, cand_idx, d_ci, npix + kDetTail));
  DIMB_TRY(download(ctx, cand_score, d_cs, npix + kDetTail));
  DIMB_TRY(download(ctx, sel_idx, d_si, nsel + kDetTail));
  DIMB_TRY(download(ctx, sel_score, d_ss, nsel + kDetTail));
  DIMB_TRY(download(ctx, sel_count, d_sc, B + kDetTail));
  if (plan) plan_out(nms_plan(r, ver), plan);
  return DIMB_OK;
}

// dimb_selftest_detect with the selection of any K: the same arguments and buffers, and
//   K >= 1, cap >= K; sort_all: ALIKED's top-k mode (sorted even when count <= K, slots count .. K-1 filled with the first pixels
//   that are not candidates; needs K <= H W); path 0: the selection production runs for K (sp_select_kernel up to kMaxTopK, the
//   grid-wide path above), 1: the grid-wide path at any K.
//   iters > 0: afterwards the selection alone runs `iters` more times on the same candidates; ms = device milliseconds per run.
extern "C" int dimb_selftest_select(dimb_ctx* ctx, const float* scores, int B, int H, int W, int r, int cut, float thr,
                                    const float* thr_per_image, int border, int K, int cap, int sort_all, int path, float sentinel,
                                    float* nms, int* cand_count, int* cand_idx, float* cand_score, int* sel_idx, float* sel_score,
                                    int* sel_count, int iters, float* ms) {
  if (!ctx || !scores || !nms || !cand_count || !cand_idx || !cand_score || !sel_idx || !sel_score || !sel_count) return DIMB_ERR_ARG;
  if (B < 1 || H < 1 || W < 1 || static_cast<long long>(B) * H * W > INT_MAX || border < 0 || !(thr >= 0.f)) return DIMB_ERR_ARG;
  if (K < 1 || cap < K || (sort_all && K > H * W) || (path != 0 && path != 1) || iters < 0 || (iters > 0 && !ms)) return DIMB_ERR_ARG;
  if (thr_per_image)
    for (int b = 0; b < B; ++b)
      if (!(thr_per_image[b] >= 0.f)) return DIMB_ERR_ARG;
  const int ver = version_of_cut(r, cut);
  if (ver < 0) return DIMB_ERR_ARG;
  DIMB_CUDA_OK(ctx, cudaSetDevice(ctx->device));
  const int HW = H * W, nch = ceil_div(HW, kChunk);
  const size_t npix = static_cast<size_t>(B) * HW, nsel = static_cast<size_t>(B) * cap;
  const int isent = sentinel_bits(sentinel);
  DevTmp t{ctx, {}};
  float *d_scores, *d_nms, *d_cs, *d_ss, *d_thr = nullptr;
  int *d_cc, *d_ci, *d_si, *d_sc;
  CandBufs c;
  DIMB_TRY(t.upload(&d_scores, std::vector<float>(scores, scores + npix)));
  DIMB_TRY(t.upload(&d_nms, std::vector<float>(npix + kDetTail, sentinel)));
  DIMB_TRY(t.upload(&d_cc, std::vector<int>(B + kDetTail, isent)));
  DIMB_TRY(t.upload(&d_ci, std::vector<int>(npix + kDetTail, isent)));
  DIMB_TRY(t.upload(&d_cs, std::vector<float>(npix + kDetTail, sentinel)));
  DIMB_TRY(t.upload(&d_si, std::vector<int>(nsel + kDetTail, isent)));
  DIMB_TRY(t.upload(&d_ss, std::vector<float>(nsel + kDetTail, sentinel)));
  DIMB_TRY(t.upload(&d_sc, std::vector<int>(B + kDetTail, isent)));
  DIMB_TRY(t.get(&c.chunk_count, static_cast<size_t>(B) * nch));
  DIMB_TRY(t.get(&c.chunk_off, static_cast<size_t>(B) * nch));
  if (thr_per_image) DIMB_TRY(t.upload(&d_thr, std::vector<float>(thr_per_image, thr_per_image + B)));
  c.cand_count = d_cc;
  c.cand_idx = d_ci;
  c.cand_score = d_cs;
  // scratch of the grid-wide path, the sizes topk_reserve gives it (the dirty contents production meets after earlier calls: 0xff)
  TopkScratch tk;
  const TopkSizes z = topk_sizes(B, HW, K);
  DIMB_TRY(t.get(&tk.hist, z.hist));
  DIMB_TRY(t.get(&tk.state, z.state));
  DIMB_TRY(t.get(&tk.chunk_cnt, z.chunks));
  DIMB_TRY(t.get(&tk.gt_off, z.chunks));
  DIMB_TRY(t.get(&tk.tie_off, z.chunks));
  DIMB_TRY(t.get(&tk.digit_off, z.digits));
  DIMB_TRY(t.get(&tk.keys0, z.keys));
  DIMB_TRY(t.get(&tk.keys1, z.keys));
  DIMB_CUDA_OK(ctx, cudaMemset(tk.hist, 0xff, z.hist * sizeof(unsigned)));
  DIMB_CUDA_OK(ctx, cudaMemset(tk.digit_off, 0xff, z.digits * sizeof(int)));
  DIMB_CUDA_OK(ctx, cudaMemset(tk.keys0, 0xff, z.keys * sizeof(unsigned long long)));
  DIMB_CUDA_OK(ctx, cudaMemset(tk.keys1, 0xff, z.keys * sizeof(unsigned long long)));
  tk.B = B, tk.HW = HW, tk.K = K;
  auto select = [&]() { return launch_select(ctx, 0, c, d_si, d_ss, d_sc, B, HW, K, cap, &tk, sort_all != 0, path == 1); };
  DIMB_TRY(launch_nms(ctx, 0, d_scores, d_nms, B, H, W, r, ver));
  DIMB_TRY(launch_candidates(ctx, 0, d_nms, c, B, H, W, thr, border, d_thr, true));
  DIMB_TRY(select());
  DIMB_TRY(sync_call(ctx, "dimb_selftest_select"));
  DIMB_TRY(download(ctx, nms, d_nms, npix + kDetTail));
  DIMB_TRY(download(ctx, cand_count, d_cc, B + kDetTail));
  DIMB_TRY(download(ctx, cand_idx, d_ci, npix + kDetTail));
  DIMB_TRY(download(ctx, cand_score, d_cs, npix + kDetTail));
  DIMB_TRY(download(ctx, sel_idx, d_si, nsel + kDetTail));
  DIMB_TRY(download(ctx, sel_score, d_ss, nsel + kDetTail));
  DIMB_TRY(download(ctx, sel_count, d_sc, B + kDetTail));
  if (iters > 0) {
    DIMB_TRY(select());  // warm-up
    cudaEvent_t e0, e1;
    DIMB_CUDA_OK(ctx, cudaEventCreate(&e0));
    DIMB_CUDA_OK(ctx, cudaEventCreate(&e1));
    int rc = cudaEventRecord(e0, 0) == cudaSuccess ? DIMB_OK : DIMB_ERR_CUDA;
    for (int i = 0; i < iters && rc == DIMB_OK; ++i) rc = select();
    if (rc == DIMB_OK && cudaEventRecord(e1, 0) != cudaSuccess) rc = DIMB_ERR_CUDA;
    if (rc == DIMB_OK) rc = sync_call(ctx, "dimb_selftest_select (timing)");
    float total = 0.f;
    if (rc == DIMB_OK && cudaEventElapsedTime(&total, e0, e1) != cudaSuccess) rc = DIMB_ERR_CUDA;
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    DIMB_TRY(rc);
    *ms = total / iters;
  }
  return DIMB_OK;
}

// sp_softmax_d2s_kernel through its production launch: logits [B h w][65] fp32 -> scores [B][8h][8w] (+ kDetTail, starting as
// `sentinel`).
extern "C" int dimb_selftest_sp_softmax(dimb_ctx* ctx, const float* logits, int B, int h, int w, float sentinel, float* scores) {
  if (!ctx || !logits || !scores || B < 1 || h < 1 || w < 1 || static_cast<long long>(B) * h * w * 64 > INT_MAX) return DIMB_ERR_ARG;
  DIMB_CUDA_OK(ctx, cudaSetDevice(ctx->device));
  const size_t cells = static_cast<size_t>(B) * h * w, n = cells * 64 + kDetTail;
  DevTmp t{ctx, {}};
  float *d_logits, *d_scores;
  DIMB_TRY(t.upload(&d_logits, std::vector<float>(logits, logits + cells * 65)));
  DIMB_TRY(t.upload(&d_scores, std::vector<float>(n, sentinel)));
  DIMB_TRY(launch_sp_softmax(ctx, 0, d_logits, d_scores, B, h, w));
  DIMB_TRY(sync_call(ctx, "dimb_selftest_sp_softmax"));
  return download(ctx, scores, d_scores, n);
}

// sp_describe_kernel through its production launch.  sel_idx / sel_score [B][cap]: selected pixels of the 8h x 8w score map (the first
// min(sel_count[b], cap) of image b are read, and must lie in the map); dense [B][h w][256] fp32 (convDb output, not normalised).
// Outputs start as `sentinel` and hold kDetTail more elements: kpts [B][cap][2] (x, y), scores [B][cap], desc [B][256][cap].
extern "C" int dimb_selftest_sp_describe(dimb_ctx* ctx, const int* sel_idx, const float* sel_score, const int* sel_count, const float* dense,
                                         int B, int h, int w, int cap, int fix_sampling, float sentinel, float* kpts, float* scores,
                                         float* desc) {
  if (!ctx || !sel_idx || !sel_score || !sel_count || !dense || !kpts || !scores || !desc) return DIMB_ERR_ARG;
  if (B < 1 || h < 1 || w < 1 || cap < 1 || static_cast<long long>(B) * h * w * 256 > INT_MAX || static_cast<long long>(B) * cap * 256 > INT_MAX)
    return DIMB_ERR_ARG;
  for (int b = 0; b < B; ++b) {
    if (sel_count[b] < 0) return DIMB_ERR_ARG;
    for (int k = 0; k < std::min(sel_count[b], cap); ++k) {
      const int p = sel_idx[static_cast<size_t>(b) * cap + k];
      if (p < 0 || p >= h * w * 64) return DIMB_ERR_ARG;
    }
  }
  DIMB_CUDA_OK(ctx, cudaSetDevice(ctx->device));
  const size_t nsel = static_cast<size_t>(B) * cap;
  DevTmp t{ctx, {}};
  int *d_si, *d_sc;
  float *d_ss, *d_dense, *d_kpts, *d_scores, *d_desc;
  DIMB_TRY(t.upload(&d_si, std::vector<int>(sel_idx, sel_idx + nsel)));
  DIMB_TRY(t.upload(&d_ss, std::vector<float>(sel_score, sel_score + nsel)));
  DIMB_TRY(t.upload(&d_sc, std::vector<int>(sel_count, sel_count + B)));
  DIMB_TRY(t.upload(&d_dense, std::vector<float>(dense, dense + static_cast<size_t>(B) * h * w * 256)));
  DIMB_TRY(t.upload(&d_kpts, std::vector<float>(nsel * 2 + kDetTail, sentinel)));
  DIMB_TRY(t.upload(&d_scores, std::vector<float>(nsel + kDetTail, sentinel)));
  DIMB_TRY(t.upload(&d_desc, std::vector<float>(nsel * 256 + kDetTail, sentinel)));
  DIMB_TRY(launch_sp_describe(ctx, 0, d_si, d_ss, d_sc, d_dense, d_kpts, d_scores, d_desc, B, h, w, cap, fix_sampling));
  DIMB_TRY(sync_call(ctx, "dimb_selftest_sp_describe"));
  DIMB_TRY(download(ctx, kpts, d_kpts, nsel * 2 + kDetTail));
  DIMB_TRY(download(ctx, scores, d_scores, nsel + kDetTail));
  return download(ctx, desc, d_desc, nsel * 256 + kDetTail);
}

// ------------------------------------------------------------------ CPU drive of the RANSAC arithmetic of gv.cu (gv_math.cuh)
// The same host/device functions, run sequentially on the host: lets tests/ check the estimators without a GPU.  Sums run in a
// different order than on the device, so results agree statistically, not bitwise.
#include "gv_math.cuh"
namespace {
void gv_host_norms(const float* k0, const float* k1, int n, gv::Norm nm[2]) {
  for (int s = 0; s < 2; ++s) {
    const float* k = s ? k1 : k0;
    double mx = 0, my = 0, d = 0;
    for (int i = 0; i < n; ++i) mx += k[2 * i], my += k[2 * i + 1];
    mx /= n, my /= n;
    for (int i = 0; i < n; ++i) d += sqrt((k[2 * i] - mx) * (k[2 * i] - mx) + (k[2 * i + 1] - my) * (k[2 * i + 1] - my));
    nm[s] = gv::Norm{static_cast<float>(mx), static_cast<float>(my), static_cast<float>(1.41421356 * n / d)};
  }
}

// the matches within thr2 of f: their count, and with `ids` their indices in order
int gv_host_count(const float* f, const float* k0, const float* k1, int n, float thr2, std::vector<int>* ids = nullptr) {
  int c = 0;
  if (ids) ids->clear();
  for (int i = 0; i < n; ++i)
    if (gv::sampson2(f, k0[2 * i], k0[2 * i + 1], k1[2 * i], k1[2 * i + 1]) < thr2) {
      ++c;
      if (ids) ids->push_back(i);
    }
  return c;
}

// least-squares fit on the matches `ids` (at least 8)
bool gv_host_lsq(const std::vector<int>& ids, const float* k0, const float* k1, const gv::Norm nm[2], float f[9]) {
  if (ids.size() < 8) return false;
  float N[9][9] = {};
  for (int i : ids) {
    float a[9];
    gv::normal_row(k0[2 * i], k0[2 * i + 1], k1[2 * i], k1[2 * i + 1], nm[0], nm[1], a);
    for (int p = 0; p < 9; ++p)
      for (int q = 0; q < 9; ++q) N[p][q] += a[p] * a[q];
  }
  return gv::refit_from_normal(N, nm[0], nm[1], f);
}

// the finalize step: two least-squares refits of bf on its inliers (kept unless they lose inliers), then F and the mask
void gv_host_finish(float bf[9], const float* k0, const float* k1, int n, float thr2, const gv::Norm nm[2], float* F, unsigned char* mask) {
  for (int round = 0; round < 2; ++round) {
    float N[9][9] = {};
    int c = 0;
    for (int i = 0; i < n; ++i)
      if (gv::sampson2(bf, k0[2 * i], k0[2 * i + 1], k1[2 * i], k1[2 * i + 1]) < thr2) {
        const float u0 = (k0[2 * i] - nm[0].cx) * nm[0].s, v0 = (k0[2 * i + 1] - nm[0].cy) * nm[0].s;
        const float u1 = (k1[2 * i] - nm[1].cx) * nm[1].s, v1 = (k1[2 * i + 1] - nm[1].cy) * nm[1].s;
        const float a[9] = {u1 * u0, u1 * v0, u1, v1 * u0, v1 * v0, v1, u0, v0, 1.f};
        for (int p = 0; p < 9; ++p)
          for (int q = 0; q < 9; ++q) N[p][q] += a[p] * a[q];
        ++c;
      }
    float f[9];
    if (c >= 8 && gv::refit_from_normal(N, nm[0], nm[1], f)) {
      int cn = 0;
      for (int i = 0; i < n; ++i) cn += gv::sampson2(f, k0[2 * i], k0[2 * i + 1], k1[2 * i], k1[2 * i + 1]) < thr2;
      if (cn >= c)
        for (int j = 0; j < 9; ++j) bf[j] = f[j];
    }
  }
  for (int j = 0; j < 9; ++j) F[j] = bf[j];
  for (int i = 0; i < n; ++i) mask[i] = gv::sampson2(bf, k0[2 * i], k0[2 * i + 1], k1[2 * i], k1[2 * i + 1]) < thr2;
}

// the local optimisation of gv_lo_kernel on the model bf adopted after wave `wave` with count best (both updated)
void gv_host_lo(float bf[9], int& best, int wave, unsigned seed, const float* k0, const float* k1, int n, float thr2, const gv::Norm nm[2]) {
  std::vector<int> in;
  for (int it = 0; it < 20; ++it) {
    gv_host_count(bf, k0, k1, n, 4.f * thr2, &in);
    if (in.size() < 16) break;
    int pos[16];
    gv::lo_sample16(seed, wave, it, static_cast<int>(in.size()), pos);
    std::vector<int> sub(16);
    for (int k = 0; k < 16; ++k) sub[k] = in[pos[k]];
    float f[9], g[9];
    if (!gv_host_lsq(sub, k0, k1, nm, f)) continue;
    for (int r = 0; r < 4; ++r) {
      gv_host_count(f, k0, k1, n, thr2, &in);
      if (!gv_host_lsq(in, k0, k1, nm, g)) break;
      for (int j = 0; j < 9; ++j) f[j] = g[j];
    }
    const int c = gv_host_count(f, k0, k1, n, thr2);
    if (c > best) {
      best = c;
      for (int j = 0; j < 9; ++j) bf[j] = f[j];
    }
  }
}
}  // namespace

extern "C" int dimb_gv_host(const float* k0, const float* k1, int n, float threshold, int iters, unsigned seed, float* F, unsigned char* mask) {
  if (!k0 || !k1 || !F || !mask || n < 8) return DIMB_ERR_ARG;
  gv::Norm nm[2];
  gv_host_norms(k0, k1, n, nm);
  const float thr2 = threshold * threshold;
  int best = -1;
  float bf[9] = {0};
  for (int h = 0; h < iters; ++h) {
    int idx[8];
    float f[9];
    gv::sample8(seed, h, n, idx);
    if (!gv::eight_point(k0, k1, idx, nm[0], nm[1], f)) continue;
    const int c = gv_host_count(f, k0, k1, n, thr2);
    if (c > best) {
      best = c;
      for (int j = 0; j < 9; ++j) bf[j] = f[j];
    }
  }
  if (best < 8) return DIMB_ERR_UNSUPPORTED;
  gv_host_finish(bf, k0, k1, n, thr2, nm, F, mask);
  return DIMB_OK;
}

// lo-ransac of gv.cu in wave order on the host: the wave's best hypothesis (highest count, then lowest 3 h + root), its local
// optimisation when it beats the pair's best, confidence stopping, the finalize step.  n_hyp: the hypotheses that ran.  n < 8 or no
// model: DIMB_ERR_UNSUPPORTED (the device keeps every match then).
extern "C" int dimb_gv_lo_host(const float* k0, const float* k1, int n, float threshold, int max_iters, float confidence, unsigned seed,
                               float* F, unsigned char* mask, int* n_hyp) {
  if (!k0 || !k1 || !F || !mask || !n_hyp || n < 8 || max_iters < 1 || !(confidence > 0.f && confidence < 1.f)) return DIMB_ERR_ARG;
  constexpr int W = 1024;
  gv::Norm nm[2];
  gv_host_norms(k0, k1, n, nm);
  const float thr2 = threshold * threshold;
  const int H = std::min(max_iters, 65536);
  int best = 0, lim = H, run = 0;
  float bf[9] = {0};
  for (int wave = 0; run < lim; ++wave) {
    int wb = -1;
    float wf[9] = {0};
    const int end = std::min(lim, (wave + 1) * W);
    for (int h = wave * W; h < end; ++h) {
      int idx[7];
      float M[3][9];
      gv::sample7(seed, h, n, idx);
      const int m = gv::seven_point(k0, k1, idx, nm[0], nm[1], M);
      for (int r = 0; r < m; ++r) {
        const int c = gv_host_count(M[r], k0, k1, n, thr2);
        if (c > wb) {
          wb = c;
          for (int j = 0; j < 9; ++j) wf[j] = M[r][j];
        }
      }
    }
    run = end;
    if (wb > best) {
      best = wb;
      for (int j = 0; j < 9; ++j) bf[j] = wf[j];
      gv_host_lo(bf, best, wave, seed, k0, k1, n, thr2, nm);
    }
    lim = std::min(lim, gv::lo_needed(best, n, confidence, H));
  }
  *n_hyp = run;
  if (best < 8) return DIMB_ERR_UNSUPPORTED;
  gv_host_finish(bf, k0, k1, n, thr2, nm, F, mask);
  return DIMB_OK;
}

namespace {
// correspondence i in the normalised coordinates (x, y, x', y')
void gv_host_unit(const float* k0, const float* k1, int i, const gv::Norm nm[2], float u[4]) {
  u[0] = (k0[2 * i] - nm[0].cx) * nm[0].s, u[1] = (k0[2 * i + 1] - nm[0].cy) * nm[0].s;
  u[2] = (k1[2 * i] - nm[1].cx) * nm[1].s, u[3] = (k1[2 * i + 1] - nm[1].cy) * nm[1].s;
}

// the matches within the squared transfer error t2 (pixels) of H (pixels)
int gv_host_count_h(const float* H, const float* k0, const float* k1, int n, float t2, std::vector<int>* outside = nullptr) {
  int c = 0;
  if (outside) outside->clear();
  for (int i = 0; i < n; ++i) {
    const bool in = gv::transfer2(H, k0[2 * i], k0[2 * i + 1], k1[2 * i], k1[2 * i + 1]) < t2;
    c += in;
    if (outside && !in) outside->push_back(i);
  }
  return c;
}

// the plane-and-parallax step of gv_pp_kernel after wave `wave`: the matches outside the plane Hn (normalised) in order, up to
// gv::kPpMax pairs of them drawn in chunks with confidence stopping on the off-plane inlier fraction, F = [e']_x H of each, the best by
// Sampson count (lowest draw on ties) into pf.  Returns its count, -1 when fewer than 2 matches are off the plane or no draw gave a model.
int gv_host_pp(const float Hn[9], int wave, unsigned seed, const float* k0, const float* k1, int n, float thr2, const gv::Norm nm[2],
               float confidence, float pf[9]) {
  float Hp[9];
  if (!gv::h_denormalise(Hn, nm[0], nm[1], Hp)) return -1;
  std::vector<int> off;
  gv_host_count_h(Hp, k0, k1, n, gv::kDegHFactor * gv::kDegHFactor * thr2, &off);
  const int m = static_cast<int>(off.size());
  if (m < 2) return -1;
  int bc = -1, need = gv::kPpMax;
  for (int base = 0; base < need; base += gv::kPpChunk) {
    for (int d = base; d < base + gv::kPpChunk; ++d) {
      int pos[2];
      gv::pp_sample2(seed, wave, d, m, pos);
      float a[4], b[4], f[9], Fp[9];
      gv_host_unit(k0, k1, off[pos[0]], nm, a);
      gv_host_unit(k0, k1, off[pos[1]], nm, b);
      if (!gv::plane_parallax(Hn, a, b, f) || !gv::denormalise(f, nm[0], nm[1], Fp)) continue;
      const int c = gv_host_count(Fp, k0, k1, n, thr2);
      if (c > bc) {
        bc = c;
        for (int j = 0; j < 9; ++j) pf[j] = Fp[j];
      }
    }
    need = gv::ransac_needed<2>(std::max(0, bc - (n - m)), m, confidence, gv::kPpMax);
  }
  return bc;
}
}  // namespace

// degensac of gv.cu in wave order on the host: lo-ransac's waves, where a 7-point model that DEGENSAC's test finds dominated by a plane
// also has its H scored (matches within gv::kDegHFactor * threshold transfer error; the first such model of a hypothesis, highest
// count then lowest 3 h + root per wave).  When a wave's best H beats the pair's best H, the plane-and-parallax step runs on it, and
// its F is adopted (and locally optimised) if it explains at least as many matches as the pair's best and the wave's best 7-point
// model; otherwise the wave's best model is adopted as in lo-ransac.  Confidence stopping and the finalize step as lo-ransac.
extern "C" int dimb_gv_degensac_host(const float* k0, const float* k1, int n, float threshold, int max_iters, float confidence, unsigned seed,
                                     float* F, unsigned char* mask, int* n_hyp) {
  if (!k0 || !k1 || !F || !mask || !n_hyp || n < 8 || max_iters < 1 || !(confidence > 0.f && confidence < 1.f)) return DIMB_ERR_ARG;
  constexpr int W = 1024;
  gv::Norm nm[2];
  gv_host_norms(k0, k1, n, nm);
  const float thr2 = threshold * threshold, tH2 = gv::kDegHFactor * gv::kDegHFactor * thr2, t2n = gv::deg_t2n(thr2, nm[1]);
  const int H = std::min(max_iters, 65536);
  int best = 0, lim = H, run = 0, hbest = 0;
  float bf[9] = {0};
  for (int wave = 0; run < lim; ++wave) {
    int wb = -1, hb = -1;
    float wf[9] = {0}, wh[9] = {0};
    const int end = std::min(lim, (wave + 1) * W);
    for (int h = wave * W; h < end; ++h) {
      int idx[7];
      float M[3][9], Mn[3][9], u[7][4];
      gv::sample7(seed, h, n, idx);
      const int m = gv::seven_point(k0, k1, idx, nm[0], nm[1], M);
      for (int r = 0; r < m; ++r) gv::normalise_f(M[r], nm[0], nm[1], Mn[r]);
      for (int r = 0; r < m; ++r) {
        const int c = gv_host_count(M[r], k0, k1, n, thr2);
        if (c > wb) {
          wb = c;
          for (int j = 0; j < 9; ++j) wf[j] = M[r][j];
        }
      }
      for (int k = 0; k < 7; ++k) gv_host_unit(k0, k1, idx[k], nm, u[k]);
      for (int r = 0; r < m; ++r) {
        float Hn[9], Hp[9];
        if (gv::degenerate7(Mn[r], u, t2n, Hn) < 0) continue;
        if (gv::h_denormalise(Hn, nm[0], nm[1], Hp)) {
          const int c = gv_host_count_h(Hp, k0, k1, n, tH2);
          if (c > hb) {
            hb = c;
            for (int j = 0; j < 9; ++j) wh[j] = Hn[j];
          }
        }
        break;
      }
    }
    run = end;
    int pc = -1;
    float pf[9];
    if (hb > hbest) {
      hbest = hb;
      pc = gv_host_pp(wh, wave, seed, k0, k1, n, thr2, nm, confidence, pf);
    }
    const float* adopt = nullptr;
    if (pc >= 8 && pc >= best && pc >= wb) {
      best = pc;
      adopt = pf;
    } else if (wb > best) {
      best = wb;
      adopt = wf;
    }
    if (adopt) {
      for (int j = 0; j < 9; ++j) bf[j] = adopt[j];
      gv_host_lo(bf, best, wave, seed, k0, k1, n, thr2, nm);
    }
    lim = std::min(lim, gv::lo_needed(best, n, confidence, H));
  }
  *n_hyp = run;
  if (best < 8) return DIMB_ERR_UNSUPPORTED;
  gv_host_finish(bf, k0, k1, n, thr2, nm, F, mask);
  return DIMB_OK;
}

namespace {
void gv_mul3(const double a[9], const double b[9], double c[9]) {
  for (int r = 0; r < 3; ++r)
    for (int k = 0; k < 3; ++k) c[3 * r + k] = a[3 * r] * b[k] + a[3 * r + 1] * b[3 + k] + a[3 * r + 2] * b[6 + k];
}

// L X R for 3 x 3 matrices (X float, in double), into out (float)
void gv_sandwich(const double L[9], const float* X, const double R[9], float out[9]) {
  double x[9], t[9], o[9];
  for (int k = 0; k < 9; ++k) x[k] = X[k];
  gv_mul3(L, x, t);
  gv_mul3(t, R, o);
  for (int k = 0; k < 9; ++k) out[k] = static_cast<float>(o[k]);
}

// a matrix in pixels in the normalised coordinates: F -> T1^-T F T0^-1 (`fundamental`), H -> T1 H T0^-1, T = the Hartley normalisation
void gv_host_normalise(const float* X, bool fundamental, const gv::Norm nm[2], float out[9]) {
  const double s0 = nm[0].s, s1 = nm[1].s;
  const double T0i[9] = {1 / s0, 0, nm[0].cx, 0, 1 / s0, nm[0].cy, 0, 0, 1};
  const double T1[9] = {s1, 0, -s1 * nm[1].cx, 0, s1, -s1 * nm[1].cy, 0, 0, 1};
  const double T1it[9] = {1 / s1, 0, 0, 0, 1 / s1, 0, nm[1].cx, nm[1].cy, 1};
  gv_sandwich(fundamental ? T1it : T1, X, T0i, out);
}
}  // namespace

// gv::h_from_f3 on F (pixels) and the correspondences idx[0..2] of k0[i] <-> k1[i] (n of them, which set the Hartley normalisations as
// in the estimator): H in pixels (unit norm).  Returns 1, or 0 when h_from_f3 rejects the triplet.
extern "C" int dimb_gv_h_from_f3_host(const float* F, const float* k0, const float* k1, int n, const int* idx, float* H) {
  if (!F || !k0 || !k1 || !idx || !H || n < 3) return DIMB_ERR_ARG;
  gv::Norm nm[2];
  gv_host_norms(k0, k1, n, nm);
  float Fn[9], c[3][4], Hn[9];
  gv_host_normalise(F, true, nm, Fn);
  for (int i = 0; i < 3; ++i) gv_host_unit(k0, k1, idx[i], nm, c[i]);
  if (!gv::h_from_f3(Fn, c, Hn)) return 0;
  return gv::h_denormalise(Hn, nm[0], nm[1], H) ? 1 : 0;
}

// gv::degenerate7 on the 7-point model F (pixels) of the sample idx[0..6] at the estimator's H threshold (gv::kDegHFactor *
// threshold): the triplet found (0 .. 4; H in pixels, unit norm) or -1.
extern "C" int dimb_gv_degenerate_host(const float* F, const float* k0, const float* k1, int n, const int* idx, float threshold, float* H) {
  if (!F || !k0 || !k1 || !idx || !H || n < 7 || !(threshold > 0.f)) return DIMB_ERR_ARG;
  gv::Norm nm[2];
  gv_host_norms(k0, k1, n, nm);
  float Fn[9], u[7][4], Hn[9];
  gv_host_normalise(F, true, nm, Fn);
  for (int k = 0; k < 7; ++k) gv_host_unit(k0, k1, idx[k], nm, u[k]);
  const int t = gv::degenerate7(Fn, u, gv::deg_t2n(threshold * threshold, nm[1]), Hn);
  if (t >= 0) gv::h_denormalise(Hn, nm[0], nm[1], H);
  return t;
}

// gv::plane_parallax on H (pixels) and the correspondences i, j of k0 <-> k1 (n of them, for the normalisations): F in pixels (unit
// norm).  Returns 1, or 0 when the parallax lines do not define an epipole.
extern "C" int dimb_gv_plane_parallax_host(const float* H, const float* k0, const float* k1, int n, int i, int j, float* F) {
  if (!H || !k0 || !k1 || !F || n < 2 || i < 0 || j < 0 || i >= n || j >= n) return DIMB_ERR_ARG;
  gv::Norm nm[2];
  gv_host_norms(k0, k1, n, nm);
  float Hn[9], a[4], b[4], f[9];
  gv_host_normalise(H, false, nm, Hn);
  gv_host_unit(k0, k1, i, nm, a);
  gv_host_unit(k0, k1, j, nm, b);
  if (!gv::plane_parallax(Hn, a, b, f)) return 0;
  return gv::denormalise(f, nm[0], nm[1], F) ? 1 : 0;
}

// gv::seven_point on 7 correspondences k0[i] <-> k1[i] (pixels) with the Hartley normalisations of those 7 points: the models in
// F [3][9], their number returned
extern "C" int dimb_gv_seven_point_host(const float* k0, const float* k1, float* F) {
  if (!k0 || !k1 || !F) return DIMB_ERR_ARG;
  gv::Norm nm[2];
  gv_host_norms(k0, k1, 7, nm);
  const int idx[7] = {0, 1, 2, 3, 4, 5, 6};
  return gv::seven_point(k0, k1, idx, nm[0], nm[1], reinterpret_cast<float(*)[9]>(F));
}

// ------------------------------------------------------------------ matching heads: LightGlue assignment and tail, SuperGlue Sinkhorn
#include <limits>

#include "lg_assign.cuh"
#include "lgx_assign.cuh"
#include "sg_assign.cuh"

namespace {
// logsigmoid of the shape-generic path, as lgx_assign_kernel evaluates it
__global__ void log_sigmoid_kernel(const float* __restrict__ z, float* __restrict__ out, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = log_sigmoid(z[i]);
}

// dst[p] = src[p]^T for P square NP x NP blocks: grid (NP / 32, NP / 32, P), block (32, 8)
__global__ void transpose_blocks_kernel(const float* __restrict__ src, float* __restrict__ dst, int NP) {
  __shared__ float tile[32][33];
  const size_t off = static_cast<size_t>(blockIdx.z) * NP * NP;
  const int x0 = blockIdx.x * 32, y0 = blockIdx.y * 32;
  for (int k = threadIdx.y; k < 32; k += 8) tile[k][threadIdx.x] = src[off + static_cast<size_t>(y0 + k) * NP + x0 + threadIdx.x];
  __syncthreads();
  for (int k = threadIdx.y; k < 32; k += 8) dst[off + static_cast<size_t>(x0 + k) * NP + y0 + threadIdx.x] = tile[threadIdx.x][k];
}

bool counts_ok(const int* c, int len, int hi) {
  for (int k = 0; k < len; ++k)
    if (c[k] < 0 || c[k] > hi) return false;
  return true;
}
}  // namespace

// The LightGlue assignment (lg_assign.cuh launch_lg_assign) on P pairs in the production layout, host fp32 inputs.
//   sim [P][NP][NP] (NP a multiple of 128; pair p live nf[2p] x nf[2p + 1], the rest as given: padding is read only by a wrong kernel),
//   nf / n_orig [2P], layer [P], indf [2P][NP], z [2P][NP] = logsigmoid(matchability); th: filter threshold; cap >= 1.
// Every output starts as `sentinel` (int buffers: its bit pattern, matches: that int sign-extended) and holds kDetTail more elements:
//   smax / slog / best / arg [2P][NP] (row statistics, row maxima and row argmaxes at side 2p; column statistics and argmaxes at side
//   2p + 1), matches [P][cap][2], mscores [P][cap], n_matches / stop_layer [P].
extern "C" int dimb_selftest_lg_assign(dimb_ctx* ctx, int P, int NP, const float* sim, const int* nf, const int* n_orig, const int* layer,
                                       const int* indf, const float* z, float th, int cap, float sentinel, float* smax, float* slog,
                                       float* best, int* arg, int64_t* matches, float* mscores, int* n_matches, int* stop_layer) {
  if (!ctx || !sim || !nf || !n_orig || !layer || !indf || !z || !smax || !slog || !best || !arg || !matches || !mscores || !n_matches ||
      !stop_layer)
    return DIMB_ERR_ARG;
  if (P < 1 || NP < 128 || NP % 128 || cap < 1 || !counts_ok(nf, 2 * P, NP) || !counts_ok(n_orig, 2 * P, INT_MAX)) return DIMB_ERR_ARG;
  DIMB_CUDA_OK(ctx, cudaSetDevice(ctx->device));
  const size_t R = static_cast<size_t>(2) * P * NP, nt = static_cast<size_t>(P) * cap;
  const int isent = sentinel_bits(sentinel);
  DevTmp t{ctx, {}};
  float *d_sim, *d_z, *d_smax, *d_slog, *d_best, *d_ms;
  int *d_nf, *d_no, *d_layer, *d_indf, *d_arg, *d_nm, *d_sl;
  long long* d_m;
  DIMB_TRY(t.upload(&d_sim, std::vector<float>(sim, sim + static_cast<size_t>(P) * NP * NP)));
  DIMB_TRY(t.upload(&d_z, std::vector<float>(z, z + R)));
  DIMB_TRY(t.upload(&d_nf, std::vector<int>(nf, nf + 2 * P)));
  DIMB_TRY(t.upload(&d_no, std::vector<int>(n_orig, n_orig + 2 * P)));
  DIMB_TRY(t.upload(&d_layer, std::vector<int>(layer, layer + P)));
  DIMB_TRY(t.upload(&d_indf, std::vector<int>(indf, indf + R)));
  DIMB_TRY(t.upload(&d_smax, std::vector<float>(R + kDetTail, sentinel)));
  DIMB_TRY(t.upload(&d_slog, std::vector<float>(R + kDetTail, sentinel)));
  DIMB_TRY(t.upload(&d_best, std::vector<float>(R + kDetTail, sentinel)));
  DIMB_TRY(t.upload(&d_arg, std::vector<int>(R + kDetTail, isent)));
  DIMB_TRY(t.upload(&d_m, std::vector<long long>(2 * nt + kDetTail, isent)));
  DIMB_TRY(t.upload(&d_ms, std::vector<float>(nt + kDetTail, sentinel)));
  DIMB_TRY(t.upload(&d_nm, std::vector<int>(P + kDetTail, isent)));
  DIMB_TRY(t.upload(&d_sl, std::vector<int>(P + kDetTail, isent)));
  DIMB_TRY(launch_lg_assign(ctx, 0, P, NP, d_sim, d_nf, d_no, d_layer, d_z, d_indf, th, d_smax, d_slog, d_best, d_arg, d_m, d_ms, d_nm, d_sl,
                            cap));
  DIMB_TRY(sync_call(ctx, "dimb_selftest_lg_assign"));
  DIMB_TRY(download(ctx, smax, d_smax, R + kDetTail));
  DIMB_TRY(download(ctx, slog, d_slog, R + kDetTail));
  DIMB_TRY(download(ctx, best, d_best, R + kDetTail));
  DIMB_TRY(download(ctx, arg, d_arg, R + kDetTail));
  DIMB_TRY(download(ctx, reinterpret_cast<long long*>(matches), d_m, 2 * nt + kDetTail));
  DIMB_TRY(download(ctx, mscores, d_ms, nt + kDetTail));
  DIMB_TRY(download(ctx, n_matches, d_nm, P + kDetTail));
  return download(ctx, stop_layer, d_sl, P + kDetTail);
}

// The LightGlue per-layer tail (lg_assign.cuh) on P pairs, side s = rows [s NP, (s + 1) NP), live rows n_act [2P], n_orig [2P],
// stopped_in / counter_in [P] (the state before the call).
//   x32 [2P NP][256] given: launch_lg_tail - lg_conf_kernel (confidence weights wt / bt, matchability weights wm / bm) then
//   lg_decide_kernel; tok and mat start as `sentinel`.  x32 null: launch_lg_decide alone on the given tok_in / mat_in [2P NP].
//   thr: this layer's confidence threshold; depth_conf, keep_thr = 1 - width_confidence, do_stop, do_prune, prune_min as production.
// Outputs hold kDetTail more elements: tok / mat / map [2P NP], n_next [2P] (int buffers start as the sentinel's bits), counter /
// stopped [P] (start as counter_in / stopped_in).
extern "C" int dimb_selftest_lg_tail(dimb_ctx* ctx, int P, int NP, const float* x32, const float* wt, float bt, const float* wm, float bm,
                                     const float* tok_in, const float* mat_in, const int* n_act, const int* n_orig, const int* stopped_in,
                                     const int* counter_in, int layer, float thr, float depth_conf, float keep_thr, int do_stop,
                                     int do_prune, int prune_min, float sentinel, float* tok, float* mat, int* counter, int* stopped, int* map,
                                     int* n_next) {
  if (!ctx || !n_act || !n_orig || !stopped_in || !counter_in || !tok || !mat || !counter || !stopped || !map || !n_next) return DIMB_ERR_ARG;
  if (x32 ? (!wt || !wm) : (!tok_in || !mat_in)) return DIMB_ERR_ARG;
  if (P < 1 || NP < 1 || layer < 0 || !counts_ok(n_act, 2 * P, NP) || !counts_ok(n_orig, 2 * P, INT_MAX)) return DIMB_ERR_ARG;
  DIMB_CUDA_OK(ctx, cudaSetDevice(ctx->device));
  const size_t R = static_cast<size_t>(2) * P * NP;
  const int isent = sentinel_bits(sentinel);
  DevTmp t{ctx, {}};
  float *d_tok, *d_mat;
  int *d_na, *d_no, *d_st, *d_cnt, *d_map, *d_nn;
  std::vector<float> ht(R + kDetTail, sentinel), hm(R + kDetTail, sentinel);
  if (!x32) {
    std::copy(tok_in, tok_in + R, ht.begin());
    std::copy(mat_in, mat_in + R, hm.begin());
  }
  std::vector<int> hs(P + kDetTail, isent), hc(P + kDetTail, isent);
  std::copy(stopped_in, stopped_in + P, hs.begin());
  std::copy(counter_in, counter_in + P, hc.begin());
  DIMB_TRY(t.upload(&d_tok, ht));
  DIMB_TRY(t.upload(&d_mat, hm));
  DIMB_TRY(t.upload(&d_st, hs));
  DIMB_TRY(t.upload(&d_cnt, hc));
  DIMB_TRY(t.upload(&d_na, std::vector<int>(n_act, n_act + 2 * P)));
  DIMB_TRY(t.upload(&d_no, std::vector<int>(n_orig, n_orig + 2 * P)));
  DIMB_TRY(t.upload(&d_map, std::vector<int>(R + kDetTail, isent)));
  DIMB_TRY(t.upload(&d_nn, std::vector<int>(2 * P + kDetTail, isent)));
  if (x32) {
    float *d_x, *d_wt, *d_wm;
    DIMB_TRY(t.upload(&d_x, std::vector<float>(x32, x32 + R * kD)));
    DIMB_TRY(t.upload(&d_wt, std::vector<float>(wt, wt + kD)));
    DIMB_TRY(t.upload(&d_wm, std::vector<float>(wm, wm + kD)));
    DIMB_TRY(launch_lg_tail(ctx, 0, P, LgRows{d_na, d_st, NP}, d_x, d_wt, bt, d_wm, bm, d_tok, d_mat, d_nn, d_no, d_st, d_cnt, d_map, layer,
                            thr, depth_conf, keep_thr, do_stop, do_prune, prune_min));
  } else {
    DIMB_TRY(launch_lg_decide(ctx, 0, P, NP, d_na, d_nn, d_no, d_st, d_cnt, d_tok, d_mat, d_map, layer, thr, depth_conf, keep_thr, do_stop,
                              do_prune, prune_min));
  }
  DIMB_TRY(sync_call(ctx, "dimb_selftest_lg_tail"));
  DIMB_TRY(download(ctx, tok, d_tok, R + kDetTail));
  DIMB_TRY(download(ctx, mat, d_mat, R + kDetTail));
  DIMB_TRY(download(ctx, counter, d_cnt, P + kDetTail));
  DIMB_TRY(download(ctx, stopped, d_st, P + kDetTail));
  DIMB_TRY(download(ctx, map, d_map, R + kDetTail));
  return download(ctx, n_next, d_nn, 2 * P + kDetTail);
}

// The assignment of the shape-generic LightGlue for one pair through launch_lgx_assign (lgx_assign.cuh), with P = 1 in the production
// layout at row stride NP = max(m, ld) + kDetTail: log-sum-exp, maxima and argmaxes in both directions, then the device filter.
// sim [m][ld] (ld >= n; m, n >= 1), raw matchability logits z0 [m] / z1 [n], original indices ind0 [m] / ind1 [n]; the cells of the
// layout outside sim hold NaN.  Outputs hold kDetTail more elements and start as `sentinel` (int buffers: its bit pattern, matches: that
// int sign-extended): rlse / ls0 / best0 / arg0 [m], clse / ls1 / best1 / arg1 [n] (ls = logsigmoid(z) as the device evaluates it),
// matches [cap][2], mscores [cap]; n_matches [1] the full count.
extern "C" int dimb_selftest_lgx_assign(dimb_ctx* ctx, int m, int n, int ld, const float* sim, const float* z0, const float* z1, const int* ind0,
                                        const int* ind1, float th, int cap, float sentinel, float* rlse, float* clse, float* ls0, float* ls1,
                                        float* best0, int* arg0, float* best1, int* arg1, int64_t* matches, float* mscores, int* n_matches) {
  if (!ctx || !sim || !z0 || !z1 || !ind0 || !ind1 || !rlse || !clse || !ls0 || !ls1 || !best0 || !arg0 || !best1 || !arg1 || !matches ||
      !mscores || !n_matches)
    return DIMB_ERR_ARG;
  if (m < 1 || n < 1 || ld < n || cap < 1) return DIMB_ERR_ARG;
  DIMB_CUDA_OK(ctx, cudaSetDevice(ctx->device));
  const int isent = sentinel_bits(sentinel), NP = std::max(m, ld) + kDetTail;  // side 0's tails end before side 1's rows
  const size_t nm = static_cast<size_t>(m) + kDetTail, nn = static_cast<size_t>(n) + kDetTail, R = 2 * static_cast<size_t>(NP);
  const float nan = std::numeric_limits<float>::quiet_NaN();
  std::vector<float> hsim(static_cast<size_t>(NP) * NP, nan), hz(R, nan);
  std::vector<int> hind(R, -1);
  for (size_t r = 0; r < static_cast<size_t>(m); ++r) std::copy(sim + r * ld, sim + (r + 1) * ld, hsim.begin() + r * NP);
  std::copy(z0, z0 + m, hz.begin());
  std::copy(z1, z1 + n, hz.begin() + NP);
  std::copy(ind0, ind0 + m, hind.begin());
  std::copy(ind1, ind1 + n, hind.begin() + NP);
  DevTmp t{ctx, {}};
  float *d_sim, *d_z, *d_rl, *d_cl, *d_l0, *d_l1, *d_best, *d_ms;
  int *d_nf, *d_stop, *d_ind, *d_arg, *d_nm, *d_sl;
  long long* d_m;
  DIMB_TRY(t.upload(&d_sim, hsim));
  DIMB_TRY(t.upload(&d_z, hz));
  DIMB_TRY(t.upload(&d_ind, hind));
  DIMB_TRY(t.upload(&d_nf, std::vector<int>{m, n}));
  DIMB_TRY(t.upload(&d_stop, std::vector<int>{0}));
  for (float** b : {&d_rl, &d_cl}) DIMB_TRY(t.upload(b, std::vector<float>(NP + kDetTail, sentinel)));
  for (float** b : {&d_l0, &d_l1}) DIMB_TRY(t.upload(b, std::vector<float>(NP, sentinel)));
  DIMB_TRY(t.upload(&d_best, std::vector<float>(R + kDetTail, sentinel)));
  DIMB_TRY(t.upload(&d_arg, std::vector<int>(R + kDetTail, isent)));
  DIMB_TRY(t.upload(&d_m, std::vector<long long>(2 * static_cast<size_t>(cap) + kDetTail, isent)));
  DIMB_TRY(t.upload(&d_ms, std::vector<float>(static_cast<size_t>(cap) + kDetTail, sentinel)));
  DIMB_TRY(t.upload(&d_nm, std::vector<int>(1, isent)));
  DIMB_TRY(t.upload(&d_sl, std::vector<int>(1, isent)));
  DIMB_TRY(launch_lgx_assign(ctx, 0, 1, NP, d_sim, d_nf, d_z, d_stop, 1, d_ind, th, d_rl, d_cl, d_best, d_arg, d_m, d_ms, d_nm, d_sl, cap));
  log_sigmoid_kernel<<<ceil_div(m, 256), 256>>>(d_z, d_l0, m);
  log_sigmoid_kernel<<<ceil_div(n, 256), 256>>>(d_z + NP, d_l1, n);
  DIMB_TRY(sync_call(ctx, "dimb_selftest_lgx_assign"));
  DIMB_TRY(download(ctx, rlse, d_rl, nm));
  DIMB_TRY(download(ctx, clse, d_cl, nn));
  DIMB_TRY(download(ctx, ls0, d_l0, nm));
  DIMB_TRY(download(ctx, ls1, d_l1, nn));
  DIMB_TRY(download(ctx, best0, d_best, nm));
  DIMB_TRY(download(ctx, arg0, d_arg, nm));
  DIMB_TRY(download(ctx, best1, d_best + NP, nn));
  DIMB_TRY(download(ctx, arg1, d_arg + NP, nn));
  DIMB_TRY(download(ctx, reinterpret_cast<long long*>(matches), d_m, 2 * static_cast<size_t>(cap) + kDetTail));
  DIMB_TRY(download(ctx, mscores, d_ms, static_cast<size_t>(cap) + kDetTail));
  return download(ctx, n_matches, d_nm, 1);
}

// SuperGlue's optimal-transport head (sg_assign.cuh) on P pairs: launch_sg_sinkhorn, then launch_sg_matches.
//   scores: the P score blocks one after the other, block p [m[p]][n[p]] row-major; a pair with an empty side counts as 0 x 0, as
//   superglue.cu's input kernel makes it.  They are laid out as production lays them: [P][NPt][NPt] with NPt = max(m, n, 1) rounded up
//   to 128, padding `pad`, and the transposes built on the device.  alpha: bin score.  u_in / v_in [P][NPt + 1] (null: zeros, as
//   production starts): the duals before the first half step.  wave >= 1: pairs per launch; half_steps >= 0: row pass, column pass,
//   row pass, ... (production: 2 x sinkhorn_iterations).  th, cap: match threshold and table rows per pair.
// Outputs hold kDetTail more elements and start as `sentinel` (int buffers: its bit pattern, matches: that int sign-extended): pc [P][4]
// (sg_pair_consts; the fourth entry stays), u / v [P][NPt + 1], best0 / arg0 / arg1 [P][NPt], matches [P][cap][2], mscores [P][cap],
// n_matches [P].
extern "C" int dimb_selftest_sg_sinkhorn(dimb_ctx* ctx, int P, const int* m, const int* n, const float* scores, float alpha, float pad,
                                         const float* u_in, const float* v_in, int wave, int half_steps, float th, int cap, float sentinel,
                                         float* pc, float* u, float* v, float* best0, int* arg0, int* arg1, int64_t* matches, float* mscores,
                                         int* n_matches) {
  if (!ctx || !m || !n || !scores || !pc || !u || !v || !best0 || !arg0 || !arg1 || !matches || !mscores || !n_matches) return DIMB_ERR_ARG;
  if (P < 1 || wave < 1 || half_steps < 0 || cap < 1 || !counts_ok(m, P, 1 << 14) || !counts_ok(n, P, 1 << 14)) return DIMB_ERR_ARG;
  int mx = 1;
  for (int p = 0; p < P; ++p) mx = std::max(mx, std::max(m[p], n[p]));
  const int NPt = round_up(mx, 128), vld = NPt + 1;
  const size_t ps = static_cast<size_t>(NPt) * NPt, nv = static_cast<size_t>(P) * vld, nb = static_cast<size_t>(P) * NPt,
               nt = static_cast<size_t>(P) * cap;
  std::vector<float> hs(P * ps, pad), hpc(4 * P + kDetTail, sentinel);
  std::vector<int> na(2 * P);
  size_t off = 0;
  for (int p = 0; p < P; ++p) {
    for (int i = 0; i < m[p]; ++i) std::copy(scores + off + static_cast<size_t>(i) * n[p], scores + off + static_cast<size_t>(i + 1) * n[p],
                                             hs.begin() + p * ps + static_cast<size_t>(i) * NPt);
    off += static_cast<size_t>(m[p]) * n[p];
    const bool empty = m[p] == 0 || n[p] == 0;
    na[2 * p] = empty ? 0 : m[p];
    na[2 * p + 1] = empty ? 0 : n[p];
    sg_pair_consts(na[2 * p], na[2 * p + 1], &hpc[4 * p]);
  }
  DIMB_CUDA_OK(ctx, cudaSetDevice(ctx->device));
  const int isent = sentinel_bits(sentinel);
  std::vector<float> hu(nv + kDetTail, sentinel), hv(nv + kDetTail, sentinel);
  std::fill(hu.begin(), hu.begin() + nv, 0.f);
  std::fill(hv.begin(), hv.begin() + nv, 0.f);
  if (u_in) std::copy(u_in, u_in + nv, hu.begin());
  if (v_in) std::copy(v_in, v_in + nv, hv.begin());
  DevTmp t{ctx, {}};
  float *d_sim, *d_simT, *d_alpha, *d_pc, *d_u, *d_v, *d_b0, *d_ms;
  int *d_na, *d_a0, *d_a1, *d_nm;
  long long* d_m;
  DIMB_TRY(t.upload(&d_sim, hs));
  DIMB_TRY(t.get(&d_simT, hs.size()));
  DIMB_TRY(t.upload(&d_alpha, std::vector<float>{alpha}));
  DIMB_TRY(t.upload(&d_pc, hpc));
  DIMB_TRY(t.upload(&d_na, na));
  DIMB_TRY(t.upload(&d_u, hu));
  DIMB_TRY(t.upload(&d_v, hv));
  DIMB_TRY(t.upload(&d_b0, std::vector<float>(nb + kDetTail, sentinel)));
  DIMB_TRY(t.upload(&d_a0, std::vector<int>(nb + kDetTail, isent)));
  DIMB_TRY(t.upload(&d_a1, std::vector<int>(nb + kDetTail, isent)));
  DIMB_TRY(t.upload(&d_m, std::vector<long long>(2 * nt + kDetTail, isent)));
  DIMB_TRY(t.upload(&d_ms, std::vector<float>(nt + kDetTail, sentinel)));
  DIMB_TRY(t.upload(&d_nm, std::vector<int>(P + kDetTail, isent)));
  transpose_blocks_kernel<<<dim3(NPt / 32, NPt / 32, P), dim3(32, 8)>>>(d_sim, d_simT, NPt);
  DIMB_CUDA_OK(ctx, cudaGetLastError());
  DIMB_TRY(launch_sg_sinkhorn(ctx, 0, P, wave, half_steps, d_sim, d_simT, NPt, d_na, d_alpha, d_u, d_v, vld, d_pc));
  DIMB_TRY(launch_sg_matches(ctx, 0, P, d_sim, NPt, ps, NPt, d_na, d_u, d_v, vld, d_pc, th, d_b0, d_a0, d_a1, d_m, d_ms, d_nm, cap));
  DIMB_TRY(sync_call(ctx, "dimb_selftest_sg_sinkhorn"));
  std::copy(hpc.begin(), hpc.end(), pc);
  DIMB_TRY(download(ctx, u, d_u, nv + kDetTail));
  DIMB_TRY(download(ctx, v, d_v, nv + kDetTail));
  DIMB_TRY(download(ctx, best0, d_b0, nb + kDetTail));
  DIMB_TRY(download(ctx, arg0, d_a0, nb + kDetTail));
  DIMB_TRY(download(ctx, arg1, d_a1, nb + kDetTail));
  DIMB_TRY(download(ctx, reinterpret_cast<long long*>(matches), d_m, 2 * nt + kDetTail));
  DIMB_TRY(download(ctx, mscores, d_ms, nt + kDetTail));
  return download(ctx, n_matches, d_nm, P + kDetTail);
}

#include "sift_kernels.cuh"

namespace {
// Geo of B images, L layers and n_oct octaves of h[o] x w[o], laid out as sift.cu's make_layout does ([levels][B][h][w] per octave:
// L + 3 Gaussian levels, then L + 2 DoG levels); false on sizes production cannot hold.  sigma <= 16: the first blur of a larger
// sigma needs more than the 127 taps sift_run takes, and the orientation kernel's sample disc grows with it.
bool sift_geo(int B, int L, int n_oct, const int* h, const int* w, float contrast, float edge, float sigma, Geo& g, size_t& total) {
  if (!h || !w || B < 1 || L < 1 || L > 32 || B * L > 65535 || n_oct < 1 || n_oct > 16) return false;
  if (!(contrast >= 0.f) || !(edge > 0.f) || !(sigma > 0.f && sigma <= 16.f) || !std::isfinite(edge)) return false;
  g.B = B, g.L = L, g.n_oct = n_oct, g.contrast = contrast, g.edge = edge, g.sigma = sigma;
  total = 0;
  for (int o = 0; o < n_oct; ++o) {
    if (h[o] < 1 || w[o] < 1 || h[o] > 32768 || w[o] > 32768) return false;
    g.h[o] = h[o], g.w[o] = w[o];
    const size_t plane = static_cast<size_t>(h[o]) * w[o] * B;
    g.gauss[o] = total;
    total += plane * (L + 3);
    g.dog[o] = total;
    total += plane * (L + 2);
  }
  return total <= (size_t{1} << 31);
}

// the production pyramid buffer with one kind of level (is_dog) copied from the caller's concatenated octaves and NaN elsewhere
int sift_stage(DevTmp& t, const Geo& g, size_t total, const float* levels, bool is_dog, float** d_pyr) {
  std::vector<float> pyr(total, std::nanf(""));
  size_t src = 0;
  for (int o = 0; o < g.n_oct; ++o) {
    const size_t n = static_cast<size_t>(g.h[o]) * g.w[o] * g.B * (g.L + (is_dog ? 2 : 3));
    std::copy(levels + src, levels + src + n, pyr.begin() + (is_dog ? g.dog[o] : g.gauss[o]));
    src += n;
  }
  return t.upload(d_pyr, pyr);
}

// int buffer of n elements starting as 0 (atomic counters) or `fill`, and kDetTail more holding `tail`
std::vector<int> sift_ibuf(size_t n, int fill, int tail) {
  std::vector<int> v(n + kDetTail, tail);
  std::fill(v.begin(), v.begin() + n, fill);
  return v;
}
}  // namespace

// SIFT (sift_kernels.cuh) stage by stage, through the launch helpers sift_run calls, on caller-given levels in the production layout.
// Levels: for each octave o < n_oct in turn, [levels][B][h[o]][w[o]] (L + 2 DoG levels or L + 3 Gaussian levels); the other kind of
// level holds NaN.  Outputs start as `sentinel` (int buffers: its bit pattern; counters: 0) and hold kDetTail more elements.
// Candidates are Cand records as 6 ints: octave << 8 | layer, row << 16 | column, then the float bits of xc, xr, xi, contr.

// sift.extrema at findScaleSpaceExtrema's threshold for contrast and L: cand [B][ccap][6] (image b's first min(count[b], ccap) valid,
// in atomic order), count [B] (every survivor, stored or not).
extern "C" int dimb_selftest_sift_extrema(dimb_ctx* ctx, const float* dog, int B, int L, int n_oct, const int* h, const int* w, float contrast,
                                          float edge, float sigma, int ccap, float sentinel, int* cand, int* count) {
  Geo g{};
  size_t total;
  if (!ctx || !dog || !cand || !count || ccap < 1 || !sift_geo(B, L, n_oct, h, w, contrast, edge, sigma, g, total)) return DIMB_ERR_ARG;
  if (static_cast<size_t>(B) * ccap * 6 > INT_MAX) return DIMB_ERR_ARG;
  DIMB_CUDA_OK(ctx, cudaSetDevice(ctx->device));
  const int isent = sentinel_bits(sentinel);
  const size_t nc = static_cast<size_t>(B) * ccap * 6;
  DevTmp t{ctx, {}};
  float* d_pyr;
  int *d_cand, *d_count;
  DIMB_TRY(sift_stage(t, g, total, dog, true, &d_pyr));
  DIMB_TRY(t.upload(&d_cand, sift_ibuf(nc, isent, isent)));
  DIMB_TRY(t.upload(&d_count, sift_ibuf(B, 0, isent)));
  DIMB_TRY(launch_sift_extrema(ctx, 0, d_pyr, g, sift_extrema_thr(contrast, L), reinterpret_cast<Cand*>(d_cand), d_count, ccap));
  DIMB_TRY(sync_call(ctx, "dimb_selftest_sift_extrema"));
  DIMB_TRY(download(ctx, cand, d_cand, nc + kDetTail));
  return download(ctx, count, d_count, B + kDetTail);
}

// sift.ori on Gaussian levels and caller-given candidates cand [B][ccap][6] (image b's first min(cand_count[b], ccap) are read: octave
// < n_oct, layer 1..L, row < h, column < w, offsets within 1): records rec [B][6][kcap] (x, y, size, angle, response, then the packed
// octave's bits; image b's first min(kp_count[b], kcap) valid, in atomic order), kp_count [B] (every keypoint, stored or not).
extern "C" int dimb_selftest_sift_ori(dimb_ctx* ctx, const float* gauss, int B, int L, int n_oct, const int* h, const int* w, float sigma,
                                      const int* cand, const int* cand_count, int ccap, int kcap, float sentinel, float* rec, int* kp_count) {
  Geo g{};
  size_t total;
  if (!ctx || !gauss || !cand || !cand_count || !rec || !kp_count || ccap < 1 || kcap < 1) return DIMB_ERR_ARG;
  if (!sift_geo(B, L, n_oct, h, w, 0.f, 1.f, sigma, g, total) || static_cast<size_t>(B) * std::max(ccap, kcap) * 6 > INT_MAX) return DIMB_ERR_ARG;
  for (int b = 0; b < B; ++b)
    if (cand_count[b] < 0) return DIMB_ERR_ARG;
  std::vector<Cand> cv(static_cast<size_t>(B) * ccap);
  memcpy(cv.data(), cand, cv.size() * sizeof(Cand));
  for (int b = 0; b < B; ++b) {
    for (int i = 0; i < std::min(cand_count[b], ccap); ++i) {
      const Cand& c = cv[static_cast<size_t>(b) * ccap + i];
      const int o = c.ol >> 8, layer = c.ol & 255, r = c.rc >> 16, col = c.rc & 0xffff;
      if (o >= n_oct || layer < 1 || layer > L || r >= h[o] || col >= w[o]) return DIMB_ERR_ARG;
      if (!(std::fabs(c.xc) <= 1.f && std::fabs(c.xr) <= 1.f && std::fabs(c.xi) <= 1.f && std::isfinite(c.contr))) return DIMB_ERR_ARG;
    }
  }
  DIMB_CUDA_OK(ctx, cudaSetDevice(ctx->device));
  const size_t nr = static_cast<size_t>(B) * kNumFields * kcap;
  DevTmp t{ctx, {}};
  float *d_pyr, *d_rec;
  Cand* d_cand;
  int *d_cc, *d_kc;
  DIMB_TRY(sift_stage(t, g, total, gauss, false, &d_pyr));
  DIMB_TRY(t.upload(&d_cand, cv));
  DIMB_TRY(t.upload(&d_cc, std::vector<int>(cand_count, cand_count + B)));
  DIMB_TRY(t.upload(&d_rec, std::vector<float>(nr + kDetTail, sentinel)));
  DIMB_TRY(t.upload(&d_kc, sift_ibuf(B, 0, sentinel_bits(sentinel))));
  DIMB_TRY(launch_sift_ori(ctx, 0, d_pyr, g, d_cand, d_cc, ccap, d_rec, d_kc, kcap));
  DIMB_TRY(sync_call(ctx, "dimb_selftest_sift_ori"));
  DIMB_TRY(download(ctx, rec, d_rec, nr + kDetTail));
  return download(ctx, kp_count, d_kc, B + kDetTail);
}

// sift.select on caller-given records rec [B][6][kcap] (sift_ori's layout; x, y, size, angle and response >= 0 in image b's first
// min(kp_count[b], kcap)); kp_count [B] >= 0, above kcap: the overflow path (count -1).  n_features 0 keeps all.  Outputs: sel_out
// [B][cap] (the record index of each output row), kpts [B][cap][2], frames [B][cap][3] (size, angle, response), octave [B][cap], counts
// [B].  The sort and selection scratch starts dirty (0xff bytes), as production leaves it between calls.
extern "C" int dimb_selftest_sift_select(dimb_ctx* ctx, const float* rec, const int* kp_count, int B, int kcap, int n_features, int cap,
                                         float sentinel, int* sel_out, float* kpts, float* frames, int* octave, int* counts) {
  if (!ctx || !rec || !kp_count || !sel_out || !kpts || !frames || !octave || !counts) return DIMB_ERR_ARG;
  if (B < 1 || B > 65535 || kcap < 1 || n_features < 0 || cap < 1 || static_cast<size_t>(B) * kNumFields * std::max(kcap, cap) > INT_MAX)
    return DIMB_ERR_ARG;
  for (int b = 0; b < B; ++b) {
    if (kp_count[b] < 0) return DIMB_ERR_ARG;
    for (int f = kFx; f <= kFresp; ++f)
      for (int i = 0; i < std::min(kp_count[b], kcap); ++i) {
        const float v = rec[(static_cast<size_t>(b) * kNumFields + f) * kcap + i];
        if (!(v >= 0.f) || std::signbit(v)) return DIMB_ERR_ARG;
      }
  }
  DIMB_CUDA_OK(ctx, cudaSetDevice(ctx->device));
  const int isent = sentinel_bits(sentinel);
  const size_t nr = static_cast<size_t>(B) * kNumFields * kcap, nk = static_cast<size_t>(B) * kcap, no = static_cast<size_t>(B) * cap;
  const size_t nch = ceil_div(kcap, kChunk), nblk = ceil_div(kcap, kSortTile);
  DevTmp t{ctx, {}};
  float *d_rec, *d_kpts, *d_frames;
  int *d_cc, *d_kc, *d_selo, *d_oct, *d_counts;
  SiftSelectBufs s;
  DIMB_TRY(t.upload(&d_rec, std::vector<float>(rec, rec + nr)));
  DIMB_TRY(t.upload(&d_cc, std::vector<int>(B, 0)));
  DIMB_TRY(t.upload(&d_kc, std::vector<int>(kp_count, kp_count + B)));
  DIMB_TRY(t.upload(&d_selo, sift_ibuf(no, isent, isent)));
  DIMB_TRY(t.upload(&d_kpts, std::vector<float>(no * 2 + kDetTail, sentinel)));
  DIMB_TRY(t.upload(&d_frames, std::vector<float>(no * 3 + kDetTail, sentinel)));
  DIMB_TRY(t.upload(&d_oct, sift_ibuf(no, isent, isent)));
  DIMB_TRY(t.upload(&d_counts, sift_ibuf(B, isent, isent)));
  DIMB_TRY(t.get(&s.n_sorted, B));
  DIMB_TRY(t.get(&s.n_dedup, B));
  DIMB_TRY(t.get(&s.ovf, B));
  DIMB_TRY(t.get(&s.dummy, B));
  DIMB_TRY(t.get(&s.sel, nk));
  DIMB_TRY(t.get(&s.chunk, B * nch));
  DIMB_TRY(t.get(&s.digit_off, B * nblk * 256));
  DIMB_TRY(t.get(&s.resp, nk));
  DIMB_TRY(t.get(&s.state, static_cast<size_t>(B) * kTkState));
  DIMB_TRY(t.get(&s.hist, static_cast<size_t>(B) * 256));
  DIMB_TRY(t.get(&s.keys0, nk));
  DIMB_TRY(t.get(&s.keys1, nk));
  s.sel_out = d_selo;
  DIMB_CUDA_OK(ctx, cudaMemset(s.sel, 0xff, nk * sizeof(int)));
  DIMB_CUDA_OK(ctx, cudaMemset(s.resp, 0xff, nk * sizeof(float)));
  DIMB_CUDA_OK(ctx, cudaMemset(s.chunk, 0xff, B * nch * sizeof(int)));
  DIMB_CUDA_OK(ctx, cudaMemset(s.digit_off, 0xff, B * nblk * 256 * sizeof(int)));
  DIMB_CUDA_OK(ctx, cudaMemset(s.state, 0xff, static_cast<size_t>(B) * kTkState * sizeof(unsigned)));
  DIMB_CUDA_OK(ctx, cudaMemset(s.hist, 0xff, static_cast<size_t>(B) * 256 * sizeof(unsigned)));
  DIMB_CUDA_OK(ctx, cudaMemset(s.keys0, 0xff, nk * sizeof(unsigned long long)));
  DIMB_CUDA_OK(ctx, cudaMemset(s.keys1, 0xff, nk * sizeof(unsigned long long)));
  const SiftOut out{d_kpts, nullptr, d_frames, d_oct, d_counts, cap};
  DIMB_TRY(launch_sift_select(ctx, 0, B, d_rec, d_cc, d_kc, kcap, kcap, n_features, s, out));
  DIMB_TRY(sync_call(ctx, "dimb_selftest_sift_select"));
  DIMB_TRY(download(ctx, sel_out, d_selo, no + kDetTail));
  DIMB_TRY(download(ctx, kpts, d_kpts, no * 2 + kDetTail));
  DIMB_TRY(download(ctx, frames, d_frames, no * 3 + kDetTail));
  DIMB_TRY(download(ctx, octave, d_oct, no + kDetTail));
  return download(ctx, counts, d_counts, B + kDetTail);
}

// sift.desc on Gaussian levels at caller-given output rows (sift_select's outputs): rows [B][n][4] (x, y, size, angle: finite, |x|,
// |y| <= 1e6, 0 < size <= 1e4, 0 <= angle <= 360), octave [B][n] (output packing: octave - 1 in the low byte, a level 0..L + 2 of an
// octave < n_oct), counts [B] (0..n).  The rows go back into records as sift.select read them; desc [B][128][cap] holds image b's
// first min(counts[b], cap) rows.
extern "C" int dimb_selftest_sift_desc(dimb_ctx* ctx, const float* gauss, int B, int L, int n_oct, const int* h, const int* w,
                                       const float* rows, const int* octave, const int* counts, int n, int cap, float sentinel, float* desc) {
  Geo g{};
  size_t total;
  if (!ctx || !gauss || !rows || !octave || !counts || !desc || n < 1 || cap < 1) return DIMB_ERR_ARG;
  if (!sift_geo(B, L, n_oct, h, w, 0.f, 1.f, 1.f, g, total) || static_cast<size_t>(B) * std::max(n * kNumFields, cap * 128) > INT_MAX)
    return DIMB_ERR_ARG;
  std::vector<float> rec(static_cast<size_t>(B) * kNumFields * n, 0.f);
  std::vector<int> sel(static_cast<size_t>(B) * cap, 0);
  for (int b = 0; b < B; ++b) {
    if (counts[b] < 0 || counts[b] > n) return DIMB_ERR_ARG;
    for (int i = 0; i < counts[b]; ++i) {
      const float* r = rows + (static_cast<size_t>(b) * n + i) * 4;
      const int oc = octave[static_cast<size_t>(b) * n + i], o = ((oc & 255) + 1) & 255, layer = (oc >> 8) & 255;
      if (!(std::fabs(r[0]) <= 1e6f && std::fabs(r[1]) <= 1e6f && r[2] > 0.f && r[2] <= 1e4f && r[3] >= 0.f && r[3] <= 360.f)) return DIMB_ERR_ARG;
      if (o >= n_oct || layer > L + 2) return DIMB_ERR_ARG;
      float* rb = rec.data() + static_cast<size_t>(b) * kNumFields * n;
      rb[kFx * static_cast<size_t>(n) + i] = r[0] * 2.f;
      rb[kFy * static_cast<size_t>(n) + i] = r[1] * 2.f;
      rb[kFsize * static_cast<size_t>(n) + i] = r[2] * 2.f;
      rb[kFangle * static_cast<size_t>(n) + i] = r[3];
      const int packed = (oc & ~255) | o;
      memcpy(&rb[kFoct * static_cast<size_t>(n) + i], &packed, sizeof packed);
      if (i < cap) sel[static_cast<size_t>(b) * cap + i] = i;
    }
  }
  DIMB_CUDA_OK(ctx, cudaSetDevice(ctx->device));
  const size_t nd = static_cast<size_t>(B) * 128 * cap;
  DevTmp t{ctx, {}};
  float *d_pyr, *d_rec, *d_desc;
  int *d_sel, *d_counts;
  DIMB_TRY(sift_stage(t, g, total, gauss, false, &d_pyr));
  DIMB_TRY(t.upload(&d_rec, rec));
  DIMB_TRY(t.upload(&d_sel, sel));
  DIMB_TRY(t.upload(&d_counts, std::vector<int>(counts, counts + B)));
  DIMB_TRY(t.upload(&d_desc, std::vector<float>(nd + kDetTail, sentinel)));
  const SiftOut out{nullptr, d_desc, nullptr, nullptr, d_counts, cap};
  DIMB_TRY(launch_sift_desc(ctx, 0, d_pyr, g, d_rec, d_sel, n, out));
  DIMB_TRY(sync_call(ctx, "dimb_selftest_sift_desc"));
  return download(ctx, desc, d_desc, nd + kDetTail);
}

#include "aliked_kernels.cuh"

namespace {
// caller's n floats followed by kDetTail NaN: a read past the logical end turns an output into NaN
std::vector<float> al_nan_tail(const float* p, size_t n) {
  std::vector<float> v(n + kDetTail, std::nanf(""));
  std::copy(p, p + n, v.begin());
  return v;
}
// n + kDetTail floats holding `sentinel`
std::vector<float> al_sent(size_t n, float sentinel) { return std::vector<float>(n + kDetTail, sentinel); }
// a staged input, or null when the caller gives none
int al_up_opt(DevTmp& t, const float* p, size_t n, float** d) {
  *d = nullptr;
  return p ? t.upload(d, al_nan_tail(p, n)) : DIMB_OK;
}
bool al_sizes_ok(int H, int W, int c) {
  return H >= 1 && W >= 1 && c >= 1 && H <= 16384 && W <= 16384 && static_cast<size_t>(H) * W * c <= (size_t{1} << 30);
}
}  // namespace

// ALIKED (aliked_kernels.cuh) stage by stage, through the launch helpers dimb_aliked_extract_dev calls, on caller-given inputs in the
// production layout.  Inputs are staged with kDetTail NaN after them; every output buffer holds kDetTail more elements after the valid
// ones and starts as `sentinel`.  Bad arguments return DIMB_ERR_ARG (DIMB_ERR_UNSUPPORTED: a deformable shape production has no
// kernel for) before any CUDA call.

// The al_conv3x3_kernel instantiation conv3 picks for an H x W map with cout output channels: out[0] = 1 (<8,1>), 2 (<16,4>) or 3
// (<8,4>).  Host only.
extern "C" int dimb_selftest_aliked_conv_plan(int H, int W, int cout, int* out) {
  if (!out || H < 1 || W < 1 || cout < 1) return DIMB_ERR_ARG;
  out[0] = al_conv3_plan(H, W, cout);
  return DIMB_OK;
}

// conv3: out [cout][H][W] = act(alpha * conv3x3(x [cin][H][W], w [cout][cin][3][3], zero padding 1) + beta (+ resid [cout][H][W])).
// alpha, beta [cout] and resid may be null; act 0 none, 1 SELU, 2 sigmoid.  variant 0: the production rule (al_conv3_plan), 1..3 that
// instantiation.  plan[0] (may be null): the instantiation that ran.
extern "C" int dimb_selftest_aliked_conv3x3(dimb_ctx* ctx, int variant, const float* x, int cin, int H, int W, const float* w,
                                            const float* alpha, const float* beta, const float* resid, int cout, int act, float sentinel,
                                            float* out, int* plan) {
  if (!ctx || !x || !w || !out || variant < 0 || variant > 3 || act < 0 || act > 2 || cin < 1 || cout < 1 || cin > 1024 || cout > 1024 ||
      !al_sizes_ok(H, W, std::max(cin, cout)))
    return DIMB_ERR_ARG;
  const int pl = variant ? variant : al_conv3_plan(H, W, cout);
  if (plan) plan[0] = pl;
  DIMB_CUDA_OK(ctx, cudaSetDevice(ctx->device));
  const size_t hw = static_cast<size_t>(H) * W;
  DevTmp t{ctx, {}};
  float *d_x, *d_w, *d_a, *d_b, *d_r, *d_o;
  DIMB_TRY(t.upload(&d_x, al_nan_tail(x, hw * cin)));
  DIMB_TRY(t.upload(&d_w, al_nan_tail(w, static_cast<size_t>(cout) * cin * 9)));
  DIMB_TRY(al_up_opt(t, alpha, cout, &d_a));
  DIMB_TRY(al_up_opt(t, beta, cout, &d_b));
  DIMB_TRY(al_up_opt(t, resid, hw * cout, &d_r));
  DIMB_TRY(t.upload(&d_o, al_sent(hw * cout, sentinel)));
  DIMB_TRY(conv3_as(ctx, 0, pl, d_x, cin, H, W, d_w, d_a, d_b, d_r, d_o, cout, act));
  DIMB_TRY(sync_call(ctx, "dimb_selftest_aliked_conv3x3"));
  return download(ctx, out, d_o, hw * cout + kDetTail);
}

// conv1: out [cout][P] = act(w [cout][cin] x [cin][P] + bias [cout] (may be null)); cin <= 512
extern "C" int dimb_selftest_aliked_conv1x1(dimb_ctx* ctx, const float* x, int cin, int P, const float* w, const float* bias, int cout,
                                            int act, float sentinel, float* out) {
  if (!ctx || !x || !w || !out || act < 0 || act > 2 || cin < 1 || cout < 1 || cin > 512 || cout > 1024 || !al_sizes_ok(1, P, std::max(cin, cout)))
    return DIMB_ERR_ARG;
  DIMB_CUDA_OK(ctx, cudaSetDevice(ctx->device));
  DevTmp t{ctx, {}};
  float *d_x, *d_w, *d_b, *d_o;
  DIMB_TRY(t.upload(&d_x, al_nan_tail(x, static_cast<size_t>(P) * cin)));
  DIMB_TRY(t.upload(&d_w, al_nan_tail(w, static_cast<size_t>(cout) * cin)));
  DIMB_TRY(al_up_opt(t, bias, cout, &d_b));
  DIMB_TRY(t.upload(&d_o, al_sent(static_cast<size_t>(P) * cout, sentinel)));
  DIMB_TRY(conv1(ctx, 0, d_x, cin, P, d_w, d_b, d_o, cout, act));
  DIMB_TRY(sync_call(ctx, "dimb_selftest_aliked_conv1x1"));
  return download(ctx, out, d_o, static_cast<size_t>(P) * cout + kDetTail);
}

// k x k average pooling, stride k: x [C][H][W] -> out [C][H / k][W / k]; 1 <= k <= min(H, W)
extern "C" int dimb_selftest_aliked_avgpool(dimb_ctx* ctx, const float* x, int C, int H, int W, int k, float sentinel, float* out) {
  if (!ctx || !x || !out || !al_sizes_ok(H, W, C) || k < 1 || k > H || k > W) return DIMB_ERR_ARG;
  DIMB_CUDA_OK(ctx, cudaSetDevice(ctx->device));
  const size_t no = static_cast<size_t>(C) * (H / k) * (W / k);
  DevTmp t{ctx, {}};
  float *d_x, *d_o;
  DIMB_TRY(t.upload(&d_x, al_nan_tail(x, static_cast<size_t>(C) * H * W)));
  DIMB_TRY(t.upload(&d_o, al_sent(no, sentinel)));
  DIMB_TRY(launch_al_avgpool(ctx, 0, d_x, C, H, W, k, d_o));
  DIMB_TRY(sync_call(ctx, "dimb_selftest_aliked_avgpool"));
  return download(ctx, out, d_o, no + kDetTail);
}

// InputPadder and al_pad_kernel: image [H][W][channels] (channels 1 or 3, 0..255) -> out [3][Hp][Wp]; geo[4] = {Hp, Wp, top, left}.
// out holds 3 (H + 31) (W + 31) elements and kDetTail more: the padded size is not known to the caller in advance.
extern "C" int dimb_selftest_aliked_pad(dimb_ctx* ctx, const float* img, int H, int W, int channels, float sentinel, float* out, int* geo) {
  if (!ctx || !img || !out || !geo || (channels != 1 && channels != 3) || !al_sizes_ok(H, W, 3)) return DIMB_ERR_ARG;
  int Hp, Wp, top, left;
  al_input_padder(H, W, Hp, Wp, top, left);
  geo[0] = Hp, geo[1] = Wp, geo[2] = top, geo[3] = left;
  DIMB_CUDA_OK(ctx, cudaSetDevice(ctx->device));
  const size_t no = static_cast<size_t>(3) * (H + 31) * (W + 31);
  DevTmp t{ctx, {}};
  float *d_i, *d_o;
  DIMB_TRY(t.upload(&d_i, al_nan_tail(img, static_cast<size_t>(H) * W * channels)));
  DIMB_TRY(t.upload(&d_o, al_sent(no, sentinel)));
  DIMB_TRY(launch_al_pad(ctx, 0, d_i, H, W, channels, d_o, Hp, Wp, top, left));
  DIMB_TRY(sync_call(ctx, "dimb_selftest_aliked_pad"));
  return download(ctx, out, d_o, no + kDetTail);
}

// al_crop_kernel: one plane [Hp][Wp] -> out [H][W] = rows top.., columns left..
extern "C" int dimb_selftest_aliked_crop(dimb_ctx* ctx, const float* in, int Hp, int Wp, int top, int left, int H, int W, float sentinel,
                                         float* out) {
  if (!ctx || !in || !out || !al_sizes_ok(Hp, Wp, 1) || H < 1 || W < 1 || top < 0 || left < 0 || top + H > Hp || left + W > Wp)
    return DIMB_ERR_ARG;
  DIMB_CUDA_OK(ctx, cudaSetDevice(ctx->device));
  const size_t no = static_cast<size_t>(H) * W;
  DevTmp t{ctx, {}};
  float *d_i, *d_o;
  DIMB_TRY(t.upload(&d_i, al_nan_tail(in, static_cast<size_t>(Hp) * Wp)));
  DIMB_TRY(t.upload(&d_o, al_sent(no, sentinel)));
  DIMB_TRY(launch_al_crop(ctx, 0, d_i, Hp, Wp, top, left, d_o, H, W));
  DIMB_TRY(sync_call(ctx, "dimb_selftest_aliked_crop"));
  return download(ctx, out, d_o, no + kDetTail);
}

// Deformable 3x3 conv + eval BatchNorm (+ resid [cout][H][W], may be null) + act on x [cin][H][W]; cin a multiple of 8 up to 128, cout
// 64 or 128.  w [cout][cin][3][3] (the state_dict layout) and bn [4][cout] (gamma, beta, running mean, running var) go through the
// transforms dimb_aliked_create applies.  Mode A (offs given): offsets [18][H][W] ((dy, dx) per tap) clamped to +-max_off.  Mode B (offs
// null): the dcn helper, offsets = offset_conv(x) with offw [18][cin][3][3] and offb [18], max_off = max(H, W) / 4; off_out [18][H][W]
// (may be null) receives them.  out [cout][H][W].
extern "C" int dimb_selftest_aliked_deform(dimb_ctx* ctx, const float* x, int cin, int H, int W, const float* offs, float max_off,
                                           const float* offw, const float* offb, const float* w, const float* bn, const float* resid, int cout,
                                           int act, float sentinel, float* out, float* off_out) {
  if (!ctx || !x || !w || !bn || !out || (!offs && (!offw || !offb)) || act < 0 || act > 2 || !al_sizes_ok(H, W, 128) || cin < 1 ||
      cout < 1 || (offs && !(max_off >= 0.f && std::isfinite(max_off))))
    return DIMB_ERR_ARG;
  if (cin % 8 || cin > 128 || (cout != 64 && cout != 128)) return DIMB_ERR_UNSUPPORTED;
  DIMB_CUDA_OK(ctx, cudaSetDevice(ctx->device));
  const size_t hw = static_cast<size_t>(H) * W;
  std::vector<float> al, be;
  al_bn_fold(bn, bn + cout, bn + 2 * cout, bn + 3 * cout, cout, al, be);
  const std::vector<float> wt = al_dcn_weight(w, cout, cin);
  DevTmp t{ctx, {}};
  BnConv c;
  c.cin = cin, c.cout = cout;
  float *d_x, *d_off, *d_r, *d_o;
  DIMB_TRY(t.upload(&d_x, al_nan_tail(x, hw * cin)));
  DIMB_TRY(t.upload(&c.w, wt));
  DIMB_TRY(t.upload(&c.alpha, al));
  DIMB_TRY(t.upload(&c.beta, be));
  DIMB_TRY(al_up_opt(t, resid, hw * cout, &d_r));
  DIMB_TRY(t.upload(&d_o, al_sent(hw * cout, sentinel)));
  if (offs) {
    DIMB_TRY(t.upload(&d_off, al_nan_tail(offs, hw * 18)));
    DIMB_TRY(launch_al_deform(ctx, 0, d_x, cin, H, W, d_off, max_off, c, d_r, d_o, act));
  } else {
    float *d_ow, *d_ob;
    DIMB_TRY(t.upload(&d_ow, al_nan_tail(offw, static_cast<size_t>(18) * cin * 9)));
    DIMB_TRY(t.upload(&d_ob, al_nan_tail(offb, 18)));
    DIMB_TRY(t.upload(&d_off, al_sent(hw * 18, sentinel)));
    DIMB_TRY(dcn(ctx, 0, d_x, cin, H, W, d_ow, d_ob, d_off, c, d_r, d_o, act));
  }
  DIMB_TRY(sync_call(ctx, "dimb_selftest_aliked_deform"));
  if (!offs && off_out) DIMB_TRY(download(ctx, off_out, d_off, hw * 18 + kDetTail));
  return download(ctx, out, d_o, hw * cout + kDetTail);
}

// al_fuse_kernel on a padded Hp x Wp map (multiples of 32): x1 [16][Hp][Wp] (block 1's output), the lateral outputs l2o [32][Hp/2][Wp/2],
// l3o [32][Hp/8][Wp/8], l4o [32][Hp/32][Wp/32], l1 = conv1.weight [32][16], s0 = score_head.0.weight [8][128].  Outputs sh0 [8][Hp][Wp]
// and feat [H][W][128], the crop at (top, left).
extern "C" int dimb_selftest_aliked_fuse(dimb_ctx* ctx, const float* x1, const float* l2o, const float* l3o, const float* l4o, const float* l1,
                                         const float* s0, int Hp, int Wp, int top, int left, int H, int W, float sentinel, float* sh0,
                                         float* feat) {
  if (!ctx || !x1 || !l2o || !l3o || !l4o || !l1 || !s0 || !sh0 || !feat || !al_sizes_ok(Hp, Wp, 128) || Hp % 32 || Wp % 32 || H < 1 ||
      W < 1 || top < 0 || left < 0 || top + H > Hp || left + W > Wp)
    return DIMB_ERR_ARG;
  DIMB_CUDA_OK(ctx, cudaSetDevice(ctx->device));
  const size_t P = static_cast<size_t>(Hp) * Wp, nf = static_cast<size_t>(H) * W * 128;
  DevTmp t{ctx, {}};
  float *d_x1, *d_l2, *d_l3, *d_l4, *d_w1, *d_s0, *d_sh, *d_f;
  DIMB_TRY(t.upload(&d_x1, al_nan_tail(x1, P * 16)));
  DIMB_TRY(t.upload(&d_l2, al_nan_tail(l2o, P / 4 * 32)));
  DIMB_TRY(t.upload(&d_l3, al_nan_tail(l3o, P / 64 * 32)));
  DIMB_TRY(t.upload(&d_l4, al_nan_tail(l4o, P / 1024 * 32)));
  DIMB_TRY(t.upload(&d_w1, al_nan_tail(l1, 32 * 16)));
  DIMB_TRY(t.upload(&d_s0, al_nan_tail(s0, 8 * 128)));
  DIMB_TRY(t.upload(&d_sh, al_sent(P * 8, sentinel)));
  DIMB_TRY(t.upload(&d_f, al_sent(nf, sentinel)));
  DIMB_TRY(launch_al_fuse(ctx, 0, d_x1, d_w1, d_l2, d_l3, d_l4, d_s0, Hp, Wp, top, left, H, W, d_sh, d_f));
  DIMB_TRY(sync_call(ctx, "dimb_selftest_aliked_fuse"));
  DIMB_TRY(download(ctx, sh0, d_sh, P * 8 + kDetTail));
  return download(ctx, feat, d_f, nf + kDetTail);
}

// DKD refinement at radius r (1..5) on score [H][W] (H, W >= 2) at the pixels sel_idx [min(count, cap)] (each < H W): kxy [cap][2]
// normalised, disp [cap], kscore [cap]; entries from min(count, cap) on are not written.
extern "C" int dimb_selftest_aliked_dkd(dimb_ctx* ctx, const float* score, int H, int W, int r, const int* sel_idx, int count, int cap,
                                        float sentinel, float* kxy, float* disp, float* kscore) {
  if (!ctx || !score || !kxy || !disp || !kscore || (count > 0 && !sel_idx) || !al_sizes_ok(H, W, 1) || H < 2 || W < 2 || r < 1 || r > 5 ||
      count < 0 || cap < 1 || cap > (1 << 24))
    return DIMB_ERR_ARG;
  const int n = std::min(count, cap);
  for (int i = 0; i < n; ++i)
    if (sel_idx[i] < 0 || sel_idx[i] >= H * W) return DIMB_ERR_ARG;
  DIMB_CUDA_OK(ctx, cudaSetDevice(ctx->device));
  DevTmp t{ctx, {}};
  float *d_s, *d_kxy, *d_disp, *d_ks;
  int *d_idx, *d_cnt;
  std::vector<int> idx(static_cast<size_t>(n) + kDetTail, 0);
  std::copy(sel_idx, sel_idx + n, idx.begin());
  DIMB_TRY(t.upload(&d_s, al_nan_tail(score, static_cast<size_t>(H) * W)));
  DIMB_TRY(t.upload(&d_idx, idx));
  DIMB_TRY(t.upload(&d_cnt, std::vector<int>{count}));
  DIMB_TRY(t.upload(&d_kxy, al_sent(static_cast<size_t>(cap) * 2, sentinel)));
  DIMB_TRY(t.upload(&d_disp, al_sent(cap, sentinel)));
  DIMB_TRY(t.upload(&d_ks, al_sent(cap, sentinel)));
  DIMB_TRY(launch_al_dkd(ctx, 0, d_s, H, W, r, d_idx, d_cnt, cap, d_kxy, d_disp, d_ks));
  DIMB_TRY(sync_call(ctx, "dimb_selftest_aliked_dkd"));
  DIMB_TRY(download(ctx, kxy, d_kxy, static_cast<size_t>(cap) * 2 + kDetTail));
  DIMB_TRY(download(ctx, disp, d_disp, cap + kDetTail));
  return download(ctx, kscore, d_ks, cap + kDetTail);
}

// The SDDH descriptor head in the context's precision on feat [H][W][128] (H, W >= 8) at normalised keypoints kxy [min(count, cap)][2]
// (within [-1, 1]).  Weights in the state_dict layout: w0 [32][128][3][3], b0 [32], w2 [32][32], b2 [32], sf [128][128], agg
// [16][128][128].  off_in [min(count, cap)][32] (may be null; finite): offsets (16 x, then 16 y) that replace the offsets stage's for the
// samples.  Outputs kpts_px [cap][2] and off [cap][32] of the offsets stage, and desc [128][cap].
extern "C" int dimb_selftest_aliked_sddh(dimb_ctx* ctx, const float* feat, int H, int W, const float* kxy, int count, int cap, const float* w0,
                                         const float* b0, const float* w2, const float* b2, const float* sf, const float* agg,
                                         const float* off_in, float sentinel, float* kpts_px, float* off, float* desc) {
  if (!ctx || !feat || !w0 || !b0 || !w2 || !b2 || !sf || !agg || !kpts_px || !off || !desc || (count > 0 && !kxy) ||
      !al_sizes_ok(H, W, 128) || H < 8 || W < 8 || count < 0 || cap < 1 || cap > (1 << 20))
    return DIMB_ERR_ARG;
  const int n = std::min(count, cap);
  for (int i = 0; i < 2 * n; ++i)
    if (!(std::fabs(kxy[i]) <= 1.f)) return DIMB_ERR_ARG;
  if (off_in)
    for (int i = 0; i < 32 * n; ++i)
      if (!std::isfinite(off_in[i])) return DIMB_ERR_ARG;
  DIMB_CUDA_OK(ctx, cudaSetDevice(ctx->device));
  const bool exact = ctx->precision == DIMB_PRECISION_EXACT;
  const size_t rows = static_cast<size_t>(round_up(cap, kTileM)) * 16;
  DevTmp t{ctx, {}};
  float *d_feat, *d_kxy, *d_w0T, *d_b0, *d_w2, *d_b2, *d_kp, *d_off, *d_offs, *d_dsc, *d_desc;
  __half *sfh, *sfl, *agh, *agl, *fsh, *fsl, *f2h, *f2l;
  int* d_cnt;
  CUtensorMap m_sf[2], m_ag[2], m_fs[2], m_f2[2];
  std::vector<__half> h, l;
  al_split_host(sf, static_cast<size_t>(128) * 128, h, l);
  DIMB_TRY(t.upload(&sfh, h));
  DIMB_TRY(t.upload(&sfl, l));
  const std::vector<float> agt = al_sddh_agg(agg);
  al_split_host(agt.data(), agt.size(), h, l);
  DIMB_TRY(t.upload(&agh, h));
  DIMB_TRY(t.upload(&agl, l));
  DIMB_TRY(dimb_tmap_2d(ctx, &m_sf[0], sfh, 128, 128, 128, 128));
  DIMB_TRY(dimb_tmap_2d(ctx, &m_sf[1], sfl, 128, 128, 128, 128));
  DIMB_TRY(dimb_tmap_2d(ctx, &m_ag[0], agh, 128, 2048, 2048, 128));
  DIMB_TRY(dimb_tmap_2d(ctx, &m_ag[1], agl, 128, 2048, 2048, 128));
  DIMB_TRY(t.get(&fsh, rows * 128));
  DIMB_TRY(t.get(&fsl, rows * 128));
  DIMB_TRY(t.get(&f2h, rows * 128));
  DIMB_TRY(t.get(&f2l, rows * 128));
  DIMB_TRY(dimb_tmap_2d(ctx, &m_fs[0], fsh, rows, 128, 128, kTileM));
  DIMB_TRY(dimb_tmap_2d(ctx, &m_fs[1], fsl, rows, 128, 128, kTileM));
  DIMB_TRY(dimb_tmap_2d(ctx, &m_f2[0], f2h, rows / 16, 2048, 2048, kTileM));
  DIMB_TRY(dimb_tmap_2d(ctx, &m_f2[1], f2l, rows / 16, 2048, 2048, kTileM));
  DIMB_TRY(t.get(&d_dsc, static_cast<size_t>(round_up(cap, kTileM)) * 128));
  DIMB_TRY(t.upload(&d_feat, al_nan_tail(feat, static_cast<size_t>(H) * W * 128)));
  DIMB_TRY(t.upload(&d_kxy, al_nan_tail(kxy, static_cast<size_t>(2) * n)));
  DIMB_TRY(t.upload(&d_w0T, al_sddh_w0T(w0)));
  DIMB_TRY(t.upload(&d_b0, al_nan_tail(b0, 32)));
  DIMB_TRY(t.upload(&d_w2, al_nan_tail(w2, 32 * 32)));
  DIMB_TRY(t.upload(&d_b2, al_nan_tail(b2, 32)));
  DIMB_TRY(t.upload(&d_cnt, std::vector<int>{count}));
  DIMB_TRY(t.upload(&d_kp, al_sent(static_cast<size_t>(cap) * 2, sentinel)));
  DIMB_TRY(t.upload(&d_off, al_sent(static_cast<size_t>(cap) * 32, sentinel)));
  DIMB_TRY(t.upload(&d_desc, al_sent(static_cast<size_t>(cap) * 128, sentinel)));
  d_offs = d_off;
  if (off_in) DIMB_TRY(t.upload(&d_offs, al_nan_tail(off_in, static_cast<size_t>(32) * n)));
  DIMB_TRY(launch_al_sddh_offsets(ctx, 0, d_feat, H, W, d_kxy, d_cnt, cap, d_w0T, d_b0, d_w2, d_b2, d_kp, d_off));
  DIMB_TRY(launch_al_sddh_sample(ctx, 0, d_feat, H, W, d_kxy, d_cnt, cap, d_offs, fsh, exact ? fsl : nullptr));
  DIMB_TRY(launch_al_sddh_sf_gemm(ctx, 0, m_fs, m_sf, f2h, exact ? f2l : nullptr, d_cnt, cap));
  DIMB_TRY(launch_al_sddh_agg_gemm(ctx, 0, m_f2, m_ag, d_dsc, d_cnt, cap));
  DIMB_TRY(launch_al_sddh_norm(ctx, 0, d_dsc, d_cnt, cap, d_desc));
  DIMB_TRY(sync_call(ctx, "dimb_selftest_aliked_sddh"));
  DIMB_TRY(download(ctx, kpts_px, d_kp, static_cast<size_t>(cap) * 2 + kDetTail));
  DIMB_TRY(download(ctx, off, d_off, static_cast<size_t>(cap) * 32 + kDetTail));
  return download(ctx, desc, d_desc, static_cast<size_t>(cap) * 128 + kDetTail);
}

// al_threshold_kernel on score [HW]: cand_count (may be null: mean mode) points at the candidate count above thr.  thr_out [1].
extern "C" int dimb_selftest_aliked_threshold(dimb_ctx* ctx, const float* score, int HW, const int* cand_count, float thr, float sentinel,
                                              float* thr_out) {
  if (!ctx || !score || !thr_out || HW < 1 || HW > (1 << 28) || (cand_count && *cand_count < 0)) return DIMB_ERR_ARG;
  DIMB_CUDA_OK(ctx, cudaSetDevice(ctx->device));
  DevTmp t{ctx, {}};
  float *d_s, *d_o;
  int* d_c = nullptr;
  DIMB_TRY(t.upload(&d_s, al_nan_tail(score, HW)));
  if (cand_count) DIMB_TRY(t.upload(&d_c, std::vector<int>{*cand_count}));
  DIMB_TRY(t.upload(&d_o, al_sent(1, sentinel)));
  DIMB_TRY(launch_al_threshold(ctx, 0, d_s, HW, d_c, thr, d_o));
  DIMB_TRY(sync_call(ctx, "dimb_selftest_aliked_threshold"));
  return download(ctx, thr_out, d_o, 1 + kDetTail);
}

// ------------------------------------------------------------------ brute-force NN matcher
#include "nn_kernels.cuh"

namespace {
// the engine's sides of P pairs as dimb_nn_match_batch_dev resolves them (descriptors, n, n_cap, desc_ld, f16, round_fp16 read); host:
// n unused, n_cap rows (the host-count entries).  False for a side the entries refuse.
bool nn_sides(int P, const dimb_feats_dev* f0, const dimb_feats_dev* f1, bool host, std::vector<NNSideIn>& sides, int& max_cap) {
  sides.resize(2 * P);
  max_cap = 0;
  for (int p = 0; p < P; ++p)
    for (int sd = 0; sd < 2; ++sd) {
      const dimb_feats_dev& f = sd ? f1[p] : f0[p];
      if (!f.descriptors || (!host && !f.n) || f.n_cap < 0 || f.desc_layout != 0 || f.desc_ld < 0) return false;
      sides[2 * p + sd] = NNSideIn{f.descriptors, host ? nullptr : f.n, f.n_cap, f.desc_ld ? f.desc_ld : f.n_cap, f.f16 ? 1 : 0,
                                   f.round_fp16 ? 1 : 0};
      max_cap = std::max(max_cap, f.n_cap);
    }
  return true;
}
}  // namespace

// The NN engine (nn_kernels.cuh) up to its row statistics: prep, then top-2 GEMM and merge in both directions (whatever the mode, which
// only decides the sides kornia leaves empty), through the pieces nn_run calls.  f0 / f1 [P]: device sides as dimb_nn_match_batch_dev
// reads them.  host_counts 1 (P = 1): the host-count engine of dimb_nn_match_dev / dimb_nn_match (EpiNNTop2, n_cap rows, n unused;
// a pair kornia leaves empty is refused, as those entries return before the engine); 0: device counts (EpiNNTop2Batch).  split: 1 / 0 =
// three / one MMA per product, whatever the context's precision.  NPp: the caller's row pitch of the outputs, which must be the
// engine's (the largest n_cap rounded up to 128, at least 128).
// Outputs hold kDetTail more elements and start as `sentinel` (int buffers: its bit pattern): n_live [2P]; d1 / d2 / i1 [2P][NPp], the
// merged best and second distance and the argbest of side s's row r at s * NPp + r (the rows of side 2p + 1 are the backward
// direction).  plan[10]: {resb, sa, sb, smem_bytes, grid} of the top-2 GEMM of each direction, as dimb_selftest_gemm_plan gives it for
// the row tiles and padded columns of the engine's NNShape (what nn_direction launches; the plan is not read back from the launch).
extern "C" int dimb_selftest_nn_stats(dimb_ctx* ctx, int P, const dimb_feats_dev* f0, const dimb_feats_dev* f1, int D, int mode, int split,
                                      int host_counts, int NPp, float sentinel, int* n_live, float* d1, float* d2, int* i1, int* plan) {
  std::vector<NNSideIn> sides;
  int max_cap = 0;
  if (!ctx || !f0 || !f1 || !n_live || !d1 || !d2 || !i1 || !plan || P < 1 || D < 1 || mode < 0 || mode > 3 || split < 0 || split > 1 ||
      host_counts < 0 || host_counts > 1 || (host_counts && P != 1) || !nn_sides(P, f0, f1, host_counts, sides, max_cap))
    return DIMB_ERR_ARG;
  const int hn[2] = {sides[0].n_cap, sides[1].n_cap};
  if (host_counts && nn_trivially_empty(hn[0], hn[1], mode)) return DIMB_ERR_ARG;
  const NNShape sh = nn_shape(P, max_cap, host_counts ? hn : nullptr);
  if (NPp != sh.NPp || static_cast<size_t>(2 * P) * NPp > INT_MAX) return DIMB_ERR_ARG;
  const int const_b = host_counts ? EpiNNTop2::kConstB : EpiNNTop2Batch::kConstB, num_kb = round_up(D, 64) / 64;
  for (int d = 0; d < 2; ++d)
    if (dimb_selftest_gemm_plan(0, kNnBN, split, const_b, num_kb, std::max(sh.P * sh.tps[d], 1), sh.npad[d] / kNnBN, ctx->num_sms,
                                plan + 5 * d) != DIMB_OK)
      return DIMB_ERR_ARG;
  DIMB_CUDA_OK(ctx, cudaSetDevice(ctx->device));
  NNWork w;
  DIMB_TRY(nn_workspace(ctx, sh, D, split != 0, &w));
  // the outputs replace the workspace's statistics buffers, so that rows the engine must not write keep the sentinel
  const size_t rows = static_cast<size_t>(2 * P) * NPp;
  const int isent = sentinel_bits(sentinel);
  DevTmp t{ctx, {}};
  DIMB_TRY(t.upload(&w.n_live, std::vector<int>(2 * P + kDetTail, isent)));
  DIMB_TRY(t.upload(&w.d1, std::vector<float>(rows + kDetTail, sentinel)));
  DIMB_TRY(t.upload(&w.d2, std::vector<float>(rows + kDetTail, sentinel)));
  DIMB_TRY(t.upload(&w.i1, std::vector<int>(rows + kDetTail, isent)));
  DIMB_CUDA_OK(ctx, cudaMemcpy(w.sides, sides.data(), sides.size() * sizeof(NNSideIn), cudaMemcpyHostToDevice));
  nn_prep_kernel<<<dim3(sh.NPp / 32, 2 * P), dim3(32, 8)>>>(w.sides, mode, D, w.Dp, sh.NPp, w.hi, w.lo, w.norm, w.n_live, nullptr);
  DIMB_CUDA_OK(ctx, cudaGetLastError());
  for (int d = 0; d < 2; ++d)
    if (sh.tps[d] > 0) DIMB_TRY(nn_direction(ctx, 0, w, sh, d, split != 0));
  DIMB_TRY(sync_call(ctx, "dimb_selftest_nn_stats"));
  DIMB_TRY(download(ctx, n_live, w.n_live, 2 * P + kDetTail));
  DIMB_TRY(download(ctx, d1, w.d1, rows + kDetTail));
  DIMB_TRY(download(ctx, d2, w.d2, rows + kDetTail));
  return download(ctx, i1, w.i1, rows + kDetTail);
}

// nn_select_kernel, as nn_run launches it, on planted row statistics: n_live [2P] (0..NPp), d1 / d2 / i1 [2P][NPp] (side s's row r at
// s * NPp + r; only live rows are read, and their i1 must lie in [0, NPp)).  th: the ratio threshold of snn / smnn.  Outputs hold
// kDetTail more elements and start as `sentinel` (idx: (long long) sentinel, count: its bit pattern): idx [P][cap][2], dist [P][cap],
// count [P] (the full count; only the first cap rows of a pair are written).
extern "C" int dimb_selftest_nn_select(dimb_ctx* ctx, int mode, float th, int P, int NPp, const int* n_live, const float* d1, const float* d2,
                                       const int* i1, int cap, float sentinel, int64_t* idx, float* dist, int* count) {
  if (!ctx || !n_live || !d1 || !d2 || !i1 || !idx || !dist || !count || mode < 0 || mode > 3 || P < 1 || NPp < 1 || cap < 1 ||
      static_cast<size_t>(2 * P) * NPp > INT_MAX || static_cast<size_t>(P) * cap * 2 > INT_MAX)
    return DIMB_ERR_ARG;
  for (int s = 0; s < 2 * P; ++s) {
    if (n_live[s] < 0 || n_live[s] > NPp) return DIMB_ERR_ARG;
    for (int r = 0; r < n_live[s]; ++r)
      if (i1[static_cast<size_t>(s) * NPp + r] < 0 || i1[static_cast<size_t>(s) * NPp + r] >= NPp) return DIMB_ERR_ARG;
  }
  DIMB_CUDA_OK(ctx, cudaSetDevice(ctx->device));
  const size_t rows = static_cast<size_t>(2 * P) * NPp, out = static_cast<size_t>(P) * cap;
  DevTmp t{ctx, {}};
  int *d_live, *d_i1, *d_count;
  float *d_d1, *d_d2, *d_dist;
  long long* d_idx;
  DIMB_TRY(t.upload(&d_live, std::vector<int>(n_live, n_live + 2 * P)));
  DIMB_TRY(t.upload(&d_d1, al_nan_tail(d1, rows)));
  DIMB_TRY(t.upload(&d_d2, al_nan_tail(d2, rows)));
  DIMB_TRY(t.upload(&d_i1, std::vector<int>(i1, i1 + rows)));
  DIMB_TRY(t.upload(&d_idx, std::vector<long long>(2 * out + kDetTail, static_cast<long long>(sentinel))));
  DIMB_TRY(t.upload(&d_dist, al_sent(out, sentinel)));
  DIMB_TRY(t.upload(&d_count, std::vector<int>(P + kDetTail, sentinel_bits(sentinel))));
  nn_select_kernel<<<P, 1024>>>(mode, th, d_live, NPp, d_d1, d_d2, d_i1, d_idx, d_dist, d_count, cap);
  DIMB_TRY(sync_call(ctx, "dimb_selftest_nn_select"));
  DIMB_TRY(download(ctx, reinterpret_cast<long long*>(idx), d_idx, 2 * out + kDetTail));
  DIMB_TRY(download(ctx, dist, d_dist, out + kDetTail));
  return download(ctx, count, d_count, P + kDetTail);
}
