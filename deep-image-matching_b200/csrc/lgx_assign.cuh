// lgx_assign.cuh - the assignment head of the shape-generic LightGlue (lightglue_generic.cu): row / column log-sum-exp, maxima and first
// argmaxes of each pair's similarity, and filter_matches (lightglue.py:246-297) on the device, through launch_lgx_assign; glibc_expf and
// host_sigmoid, which the per-layer decisions share.  Included by lightglue_generic.cu and by the self-test library.
#pragma once
#include "generic_kernels.cuh"

namespace {

// glibc's expf (sysdeps/ieee754/flt-32/e_expf.c, the FMA build x86-64 CPUs with FMA run): exp(x) = 2^(k/32) * 2^(r/32) with
// k = round(x * 32 / ln 2), 2^(k/32) from a 32-entry table and 2^(r/32) a cubic, all in double.  It reproduces the host's
// std::exp(float) bit for bit (checked against glibc 2.39 over every float with |x| < 87), which plain (float)exp((double)x) does not
// (it is correctly rounded, glibc is not quite: 0.502 ulp).  This path's match scores exp(max) and its confidence / matchability
// sigmoid decisions were defined on the host with glibc, and the current outputs and goldens are those; expf would change them.
__constant__ unsigned long long kExp2fTab[32] = {
    0x3ff0000000000000ull, 0x3fefd9b0d3158574ull, 0x3fefb5586cf9890full, 0x3fef9301d0125b51ull, 0x3fef72b83c7d517bull, 0x3fef54873168b9aaull,
    0x3fef387a6e756238ull, 0x3fef1e9df51fdee1ull, 0x3fef06fe0a31b715ull, 0x3feef1a7373aa9cbull, 0x3feedea64c123422ull, 0x3feece086061892dull,
    0x3feebfdad5362a27ull, 0x3feeb42b569d4f82ull, 0x3feeab07dd485429ull, 0x3feea47eb03a5585ull, 0x3feea09e667f3bcdull, 0x3fee9f75e8ec5f74ull,
    0x3feea11473eb0187ull, 0x3feea589994cce13ull, 0x3feeace5422aa0dbull, 0x3feeb737b0cdc5e5ull, 0x3feec49182a3f090ull, 0x3feed503b23e255dull,
    0x3feee89f995ad3adull, 0x3feeff76f2fb5e47ull, 0x3fef199bdd85529cull, 0x3fef3720dcef9069ull, 0x3fef5818dcfba487ull, 0x3fef7c97337b9b5full,
    0x3fefa4afa2a490daull, 0x3fefd0765b6e4540ull};

__device__ __forceinline__ float glibc_expf(float x) {
  if (x != x) return x + x;
  if (x > 0x1.62e42ep6f) return INFINITY;
  if (x < -0x1.9fe368p6f) return 0.f;
  const double inv_ln2_n = 0x1.71547652b82fep+0 * 32, shift = 0x1.8p+52;
  const double c0 = 0x1.c6af84b912394p-5 / 32 / 32 / 32, c1 = 0x1.ebfce50fac4f3p-3 / 32 / 32, c2 = 0x1.62e42ff0c52d6p-1 / 32;
  const double xd = static_cast<double>(x);
  double kd = __fma_rn(inv_ln2_n, xd, shift);
  const unsigned long long ki = static_cast<unsigned long long>(__double_as_longlong(kd));
  kd = __dsub_rn(kd, shift);
  const double r = __fma_rn(inv_ln2_n, xd, -kd);
  const unsigned long long t = kExp2fTab[ki % 32] + (ki << 47);
  const double s = __longlong_as_double(static_cast<long long>(t));
  const double z = __fma_rn(c0, r, c1), r2 = __dmul_rn(r, r);
  double y = __fma_rn(c2, r, 1.0);
  y = __fma_rn(z, r2, y);
  return __double2float_rn(__dmul_rn(y, s));
}
// 1.f / (1.f + std::exp(-z)) as the host evaluates it
__device__ __forceinline__ float host_sigmoid(float z) { return __fdiv_rn(1.f, __fadd_rn(1.f, glibc_expf(-z))); }

// warp per (pair, row or column): log-sum-exp (what = 0) or maximum / first argmax of the log assignment (what = 1), dir 0 rows, 1 columns
__global__ void lgx_assign_kernel(int what, int dir, const float* __restrict__ sim, int NP, const int* __restrict__ nf,
                                  float* __restrict__ rlse, float* __restrict__ clse, const float* __restrict__ z, float* __restrict__ best,
                                  int* __restrict__ arg, int P) {
  const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  const int p = gw / NP, i = gw - p * NP;
  if (p >= P) return;
  const int m = nf[2 * p], n = nf[2 * p + 1];
  if (m == 0 || n == 0 || i >= (dir == 0 ? m : n)) return;
  const float* s = sim + static_cast<size_t>(p) * NP * NP;
  const size_t o = static_cast<size_t>(p) * NP;
  if (what == 0) {
    gx_lse_one(s, NP, m, n, dir, (dir == 0 ? rlse : clse) + o, i, lane);
  } else {
    gx_argmax_one(s, NP, m, n, rlse + o, clse + o, z + 2 * o, z + 2 * o + NP, dir, best + 2 * o + (dir ? NP : 0), arg + 2 * o + (dir ? NP : 0),
                  i, lane);
  }
}

// block (1024) per pair: filter_matches - mutual argmax, exp(max) > th, matches in row order (first cap written, full count reported) -
// and the stop layer (1 for a pair with an empty side)
__global__ void __launch_bounds__(1024) lgx_filter_kernel(const int* __restrict__ nf, const int* __restrict__ stopped, int L, int NP,
                                                          const float* __restrict__ best, const int* __restrict__ arg, const int* __restrict__ indf,
                                                          float th, long long* __restrict__ matches, float* __restrict__ mscores,
                                                          int* __restrict__ n_matches, int* __restrict__ stop_layer, int cap) {
  const int p = blockIdx.x, tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const int st = stopped[p], n0 = nf[2 * p], n1 = nf[2 * p + 1];
  const bool run = n0 > 0 && n1 > 0;
  __shared__ int wsum[32], total;
  const size_t o = static_cast<size_t>(2 * p) * NP;
  const float* b0 = best + o;
  const int *a0 = arg + o, *a1 = arg + o + NP;
  int base = 0;
  for (int r0 = 0; run && r0 < n0; r0 += blockDim.x) {
    const int r = r0 + tid;
    int c = -1;
    float e = 0.f;
    bool ok = false;
    if (r < n0) {
      c = a0[r];
      if (c >= 0 && c < n1 && a1[c] == r) {
        e = glibc_expf(b0[r]);
        ok = e > th;
      }
    }
    const unsigned bal = __ballot_sync(0xffffffffu, ok);
    if (lane == 0) wsum[w] = __popc(bal);
    __syncthreads();
    if (w == 0) {
      const int nw = blockDim.x >> 5;
      int v = lane < nw ? wsum[lane] : 0, incl = v;
#pragma unroll
      for (int of = 1; of < 32; of <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, incl, of);
        if (lane >= of) incl += t;
      }
      if (lane < nw) wsum[lane] = incl - v;
      if (lane == 31) total = incl;
    }
    __syncthreads();
    const int pos = base + wsum[w] + __popc(bal & ((1u << lane) - 1u));
    if (ok && pos < cap) {
      const size_t q = static_cast<size_t>(p) * cap + pos;
      matches[2 * q] = indf[o + r];
      matches[2 * q + 1] = indf[o + NP + c];
      mscores[q] = e;
    }
    base += total;
    __syncthreads();
  }
  if (tid == 0) {
    n_matches[p] = base;
    stop_layer[p] = st ? st : L;
  }
}

// The assignment of P pairs: sim [P][NP][NP] (pair p: nf[2p] x nf[2p + 1] live, row stride NP), raw matchability logits z [2P][NP],
// original indices indf [2P][NP], stopped [P] (0: the pair ran all L layers, else its stop layer).  Writes rlse / clse [P][NP], the row
// maxima / argmaxes at best / arg [2p][NP] and the column ones at [2p + 1][NP], matches [P][cap][2], mscores [P][cap], n_matches and
// stop_layer [P].
inline int launch_lgx_assign(dimb_ctx* ctx, cudaStream_t st, int P, int NP, const float* sim, const int* nf, const float* z, const int* stopped,
                             int L, const int* indf, float th, float* rlse, float* clse, float* best, int* arg, long long* matches,
                             float* mscores, int* n_matches, int* stop_layer, int cap) {
  const int pair_rows = ceil_div(P * NP * 32, 256);
  for (int what = 0; what < 2; ++what)
    for (int dir = 0; dir < 2; ++dir) {
      lgx_assign_kernel<<<pair_rows, 256, 0, st>>>(what, dir, sim, NP, nf, rlse, clse, z, best, arg, P);
      DIMB_LAUNCH_CHECK(ctx);
    }
  lgx_filter_kernel<<<P, 1024, 0, st>>>(nf, stopped, L, NP, best, arg, indf, th, matches, mscores, n_matches, stop_layer, cap);
  DIMB_LAUNCH_CHECK(ctx);
  return DIMB_OK;
}

}  // namespace
