// selftest.cu - dimb_selftest_gemm: C = A * B^T through the production tensor-core GEMM (or its SIMT twin),
// used by tests/ to validate the wgmma/TMA plumbing in isolation from the model code.
#include <vector>

#include "gemm.cuh"

namespace {
__global__ void split_rows_kernel(const float* __restrict__ src, __half* __restrict__ hi, __half* __restrict__ lo, size_t n) {
  const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  __half h, l;
  split_f32(src[i], h, l);
  hi[i] = h;
  lo[i] = l;
}
}  // namespace

// A [M][K], B [N][K], C [M][N] host fp32; K multiple of 64. bn: 64, 128 or 256 (CTA tile width).
extern "C" int dimb_selftest_gemm(dimb_ctx* ctx, const float* A, const float* B, float* C, int M, int N, int K, int bn) {
  if (!ctx || !A || !B || !C || K % 64 || M < 1 || N < 1) return DIMB_ERR_ARG;
  DIMB_CUDA_OK(ctx, cudaSetDevice(ctx->device));
  const int Mp = round_up(M, 128), Np = round_up(N, 256);
  float *dA, *dB, *dC;
  __half *ah, *al, *bh, *bl;
  std::vector<void*> tmp;
  auto alloc = [&](void** p, size_t b) -> int {
    DIMB_CUDA_OK(ctx, cudaMalloc(p, b));
    tmp.push_back(*p);
    DIMB_CUDA_OK(ctx, cudaMemset(*p, 0, b));
    return static_cast<int>(DIMB_OK);
  };
  int rc = DIMB_OK;
  do {
    if ((rc = alloc((void**)&dA, sizeof(float) * Mp * K))) break;
    if ((rc = alloc((void**)&dB, sizeof(float) * Np * K))) break;
    if ((rc = alloc((void**)&dC, sizeof(float) * Mp * N))) break;
    if ((rc = alloc((void**)&ah, sizeof(__half) * Mp * K))) break;
    if ((rc = alloc((void**)&al, sizeof(__half) * Mp * K))) break;
    if ((rc = alloc((void**)&bh, sizeof(__half) * Np * K))) break;
    if ((rc = alloc((void**)&bl, sizeof(__half) * Np * K))) break;
    cudaMemcpy(dA, A, sizeof(float) * M * K, cudaMemcpyHostToDevice);
    cudaMemcpy(dB, B, sizeof(float) * N * K, cudaMemcpyHostToDevice);
    split_rows_kernel<<<ceil_div(Mp * K, 256), 256>>>(dA, ah, al, static_cast<size_t>(Mp) * K);
    split_rows_kernel<<<ceil_div(Np * K, 256), 256>>>(dB, bh, bl, static_cast<size_t>(Np) * K);
    TcOperands ops;
    if ((rc = dimb_tmap_2d(ctx, &ops.Ah, ah, Mp, K, K, kTileM))) break;
    if ((rc = dimb_tmap_2d(ctx, &ops.Al, al, Mp, K, K, kTileM))) break;
    if ((rc = dimb_tmap_2d(ctx, &ops.Bh, bh, Np, K, K, bn))) break;
    if ((rc = dimb_tmap_2d(ctx, &ops.Bl, bl, Np, K, K, bn))) break;
    GemmArgs g{};
    g.num_kb = K / 64;
    g.M = M;
    g.N = N;
    g.Ah = ah;
    g.Al = al;
    g.Bh = bh;
    g.Bl = bl;
    g.lda = K;
    g.ldb = K;
    EpiStoreF32 e;
    e.out = dC;
    e.bias = nullptr;
    e.ldc = N;
    e.n_valid = N;
    e.m_valid = M;
    e.scale = 1.f;
    const int mt = Mp / 128;
    if (bn == 64)
      rc = launch_gemm<64, false>(ctx, 0, ops, g, e, mt, round_up(N, 64));
    else if (bn == 128)
      rc = launch_gemm<128, false>(ctx, 0, ops, g, e, mt, round_up(N, 128));
    else if (bn == 256)
      rc = launch_gemm<256, false>(ctx, 0, ops, g, e, mt, round_up(N, 256));
    else
      rc = DIMB_ERR_ARG;
    if (rc) break;
    cudaError_t ce = cudaDeviceSynchronize();
    if (ce != cudaSuccess) {
      dimb_set_error(ctx, std::string("dimb_selftest_gemm: ") + cudaGetErrorString(ce));
      rc = DIMB_ERR_CUDA;
      break;
    }
    cudaMemcpy(C, dC, sizeof(float) * M * N, cudaMemcpyDeviceToHost);
  } while (0);
  for (void* p : tmp) cudaFree(p);
  return rc;
}

// ------------------------------------------------------------------ CPU drive of the RANSAC arithmetic of gv.cu (gv_math.cuh)
// The same host/device functions, run sequentially on the host: lets tests/ check the estimator without a GPU.
#include "gv_math.cuh"
extern "C" int dimb_gv_host(const float* k0, const float* k1, int n, float threshold, int iters, unsigned seed, float* F, unsigned char* mask) {
  if (!k0 || !k1 || !F || !mask || n < 8) return DIMB_ERR_ARG;
  gv::Norm nm[2];
  for (int s = 0; s < 2; ++s) {
    const float* k = s ? k1 : k0;
    double mx = 0, my = 0, d = 0;
    for (int i = 0; i < n; ++i) mx += k[2 * i], my += k[2 * i + 1];
    mx /= n, my /= n;
    for (int i = 0; i < n; ++i) d += sqrt((k[2 * i] - mx) * (k[2 * i] - mx) + (k[2 * i + 1] - my) * (k[2 * i + 1] - my));
    nm[s] = gv::Norm{static_cast<float>(mx), static_cast<float>(my), static_cast<float>(1.41421356 * n / d)};
  }
  const float thr2 = threshold * threshold;
  int best = -1;
  float bf[9] = {0};
  for (int h = 0; h < iters; ++h) {
    int idx[8];
    float f[9];
    gv::sample8(seed, h, n, idx);
    if (!gv::eight_point(k0, k1, idx, nm[0], nm[1], f)) continue;
    int c = 0;
    for (int i = 0; i < n; ++i) c += gv::sampson2(f, k0[2 * i], k0[2 * i + 1], k1[2 * i], k1[2 * i + 1]) < thr2;
    if (c > best) {
      best = c;
      for (int j = 0; j < 9; ++j) bf[j] = f[j];
    }
  }
  if (best < 8) return DIMB_ERR_UNSUPPORTED;
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
  return DIMB_OK;
}
