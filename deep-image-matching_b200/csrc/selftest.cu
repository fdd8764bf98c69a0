// selftest.cu - dimb_selftest_gemm: C = A * B^T through the production tensor-core GEMM (or its SIMT twin), and
// dimb_selftest_attention: the flash-attention kernels through their production launches; used by tests/ to validate the
// wgmma/TMA plumbing in isolation from the model code.
#include <algorithm>
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

// ------------------------------------------------------------------ attention self-test
#include "attn_hd128.cuh"
#include "lg_kernels.cuh"

namespace {
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

int sync_call(dimb_ctx* ctx) {
  cudaError_t ce = cudaGetLastError();
  if (ce == cudaSuccess) ce = cudaDeviceSynchronize();
  if (ce != cudaSuccess) {
    dimb_set_error(ctx, std::string("dimb_selftest_attention: ") + cudaGetErrorString(ce));
    return DIMB_ERR_CUDA;
  }
  return DIMB_OK;
}

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
  if (ctx->use_tc) {  // tensor maps as lightglue.cu builds them: Q box 128 rows, K box 64 rows, V^T box 64 rows
    CUtensorMap mq[2], mk[2], mv[2];
    const uint64_t rows = static_cast<uint64_t>(S) * kHeads * NP;
    for (int pl = 0; pl < 2; ++pl) {
      DIMB_TRY(dimb_tmap_2d(ctx, &mq[pl], pl ? ql : qh, rows, kHd, kHd, kTileM));
      DIMB_TRY(dimb_tmap_2d(ctx, &mk[pl], pl ? kl_ : kh_, rows, kHd, kHd, kBlkK));
      DIMB_TRY(dimb_tmap_2d(ctx, &mv[pl], pl ? vl : vh, static_cast<uint64_t>(S) * kHeads * kHd, NP, NP, kHd));
    }
    DIMB_TRY(launch_lg_attention(ctx, 0, dim3(1, kHeads, S), mq, mk, mv, a, exact));
  } else {
    lg_attn_simt_kernel<<<dim3(ceil_div(NP * 32, 256), kHeads, S), 256>>>(a, qh, exact ? ql : nullptr, kh_, exact ? kl_ : nullptr, vh,
                                                                          exact ? vl : nullptr);
  }
  float* d_out;
  DIMB_TRY(t.get(&d_out, R * kD));
  join_rows_kernel<<<ceil_div(static_cast<int>(R * kD), 256), 256>>>(ch, exact ? cl : nullptr, d_out, R * kD);
  DIMB_TRY(sync_call(ctx));
  DIMB_CUDA_OK(ctx, cudaMemcpy(out, d_out, sizeof(float) * R * kD, cudaMemcpyDeviceToHost));
  return DIMB_OK;
}

// shape-generic attention (attn_hd128.cuh) on operands packed by the production packers at NP rounded up to the query tile
int selftest_attention_hd128(dimb_ctx* ctx, const float* Q, const float* K, const float* V, float* out, int H, int hd, int NP, const int* n,
                             float lazy, float pad, float out_pad) {
  if (!ctx->use_tc) {
    dimb_set_error(ctx, "dimb_selftest_attention: variant 1 is the tensor-core kernel (DIMB_TC=0 runs the fp32 kernel of the generic path)");
    return DIMB_ERR_UNSUPPORTED;
  }
  const bool exact = ctx->precision == DIMB_PRECISION_EXACT;
  const int NPp = round_up(NP, kAttnTile), ld = H * hd;
  const size_t nel = static_cast<size_t>(NPp) * ld, pl_el = static_cast<size_t>(H) * NPp * kXHd;
  std::vector<float> q(nel, pad), k(nel, pad), v(nel, pad);  // rows past the live counts hold `pad`: the packers copy all NPp rows
  std::copy(Q, Q + static_cast<size_t>(n[0]) * ld, q.begin());
  std::copy(K, K + static_cast<size_t>(n[1]) * ld, k.begin());
  std::copy(V, V + static_cast<size_t>(n[1]) * ld, v.begin());
  DevTmp t{ctx, {}};
  float *fq, *fk, *fv, *d_out;
  __half *qp[2], *kp[2], *vp[2];
  DIMB_TRY(t.upload(&fq, q));
  DIMB_TRY(t.upload(&fk, k));
  DIMB_TRY(t.upload(&fv, v));
  DIMB_TRY(t.upload(&d_out, std::vector<float>(nel, out_pad)));
  for (int pl = 0; pl < 2; ++pl) {
    DIMB_TRY(t.get(&qp[pl], pl_el));
    DIMB_TRY(t.get(&kp[pl], pl_el));
    DIMB_TRY(t.get(&vp[pl], pl_el));
  }
  gx_pack_rows_kernel<<<dim3(NPp, H), kXHd>>>(fq, ld, NPp, hd, NPp, qp[0], exact ? qp[1] : nullptr);
  gx_pack_rows_kernel<<<dim3(NPp, H), kXHd>>>(fk, ld, NPp, hd, NPp, kp[0], exact ? kp[1] : nullptr);
  gx_pack_vt_kernel<<<dim3(NPp / 32, kXHd / 32, H), dim3(32, 8)>>>(fv, ld, NPp, hd, NPp, vp[0], exact ? vp[1] : nullptr);
  DIMB_CUDA_OK(ctx, cudaGetLastError());
  CUtensorMap mq[2], mk[2], mv[2];  // as lightglue_generic.cu: Q box 128 rows, K box 64 rows, V^T box 128 rows
  for (int pl = 0; pl < 2; ++pl) {
    DIMB_TRY(dimb_tmap_2d(ctx, &mq[pl], qp[pl], static_cast<uint64_t>(H) * NPp, kXHd, kXHd, kAttnTile));
    DIMB_TRY(dimb_tmap_2d(ctx, &mk[pl], kp[pl], static_cast<uint64_t>(H) * NPp, kXHd, kXHd, kAttnBlk));
    DIMB_TRY(dimb_tmap_2d(ctx, &mv[pl], vp[pl], static_cast<uint64_t>(H) * kXHd, NPp, NPp, kXHd));
  }
  AttnXArgs a;
  a.nq = n[0], a.nk = n[1], a.NP = NPp, a.hd = hd;
  a.scale = 1.f / sqrtf(static_cast<float>(hd));
  a.lazy = lazy;
  a.out = d_out, a.ldo = ld;
  DIMB_TRY(launch_attn_hd128(ctx, 0, mq, mk, mv, H, a, exact));
  DIMB_TRY(sync_call(ctx));
  DIMB_CUDA_OK(ctx, cudaMemcpy(out, d_out, sizeof(float) * nel, cudaMemcpyDeviceToHost));
  return DIMB_OK;
}
}  // namespace

// Flash attention (attention.cuh) through its production launches, on host fp32 operands; precision from ctx.
//   variant 0: lg_attn_kernel (LightGlue / SuperGlue, H = 4 heads of hd = 64) via launch_lg_attention, or its SIMT twin
//     lg_attn_simt_kernel when ctx->use_tc == 0.  Q, K, V [S][4][NP][64] (S even, NP a multiple of 128), live rows n[S], stopped[S / 2]
//     (nonzero: the pair is stopped); cross: the keys of side s are the q rows of side s ^ 1 (K unused, may be null).  out: the
//     context buffer [S * NP][256], hi + lo planes (hi only in FAST), every row.
//   variant 1: gx_attn_tc_kernel (head dim hd <= 128, even, padded to 128) via launch_attn_hd128, operands packed by
//     gx_pack_rows_kernel / gx_pack_vt_kernel.  Q [n[0]][H * hd], K / V [n[1]][H * hd], NP >= n[0], n[1]; S, stopped and cross unused.
//     out: [NPp][H * hd] fp32 with NPp = NP rounded up to 128.
// Every Q / K row and V^T column past the live counts holds `pad` (stale values of earlier layers in production), and the output
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
