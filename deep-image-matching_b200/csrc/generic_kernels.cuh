// generic_kernels.cuh - plain fp32 CUDA-core kernel bodies of the shape-generic LightGlue (lightglue_generic.cu, lgx_assign.cuh) and
// SuperGlue (superglue.cu) paths: tiled linear layer, warp-per-query online-softmax attention, LayerNorm+GELU, row dot products,
// log-sum-exp / argmax over a score matrix.  The kernels that launch them add a grid dimension over the sides or pairs.  They trade speed
// for generality; the tensor-core kernels live in gemm.cuh / lightglue.cu.
#pragma once
#include "common.cuh"

namespace {

// C[m][n] = act((sum_k A[m*lda + k] * W[n*ldw + k] + bias[n]) * scale) (+ resid[m*ldr + n]), act = ReLU or identity; 64 x 64 tile, 256 threads, 4 x 4 outputs
// per thread, K streamed through shared memory 16 at a time (k ascending per output: deterministic summation order).
// The tile body is shared with SuperGlue's batched keypoint encoder (one more grid dimension over the sides).
__device__ __forceinline__ void gx_linear_tile(const float* __restrict__ A, int lda, const float* __restrict__ W, int ldw,
                                               const float* __restrict__ bias, float* __restrict__ C, int ldc, int M, int N, int K,
                                               float scale, const float* __restrict__ resid, int ldr, int relu, int m0) {
  __shared__ float sa[16][64 + 4], sb[16][64 + 4];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4, n0 = blockIdx.x * 64;
  float acc[4][4] = {};
  for (int k0 = 0; k0 < K; k0 += 16) {
    for (int e = threadIdx.x; e < 64 * 16; e += 256) {
      const int r = e >> 4, k = e & 15;
      sa[k][r] = (m0 + r < M && k0 + k < K) ? A[static_cast<size_t>(m0 + r) * lda + k0 + k] : 0.f;
      sb[k][r] = (n0 + r < N && k0 + k < K) ? W[static_cast<size_t>(n0 + r) * ldw + k0 + k] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 16; ++k) {
      const float4 a = *reinterpret_cast<const float4*>(&sa[k][ty * 4]);
      const float4 b = *reinterpret_cast<const float4*>(&sb[k][tx * 4]);
      const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty * 4 + i;
    if (m >= M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx * 4 + j;
      if (n >= N) continue;
      float v = (acc[i][j] + (bias ? bias[n] : 0.f)) * scale;
      if (relu) v = fmaxf(v, 0.f);
      if (resid) v += resid[static_cast<size_t>(m) * ldr + n];
      C[static_cast<size_t>(m) * ldc + n] = v;
    }
  }
}

// keypoint normalisation (lightglue.py:24-34) + Fourier encoding (:57-70): enc [2][N][hd] = cos / sin, each frequency twice
// (one keypoint i, one frequency f; shared with the batched prep of lightglue_generic.cu)
__device__ __forceinline__ void gx_posenc_one(const float* __restrict__ kpts, int i, int f, float size0, float size1,
                                              const float* __restrict__ Wr, int hd, float* __restrict__ enc, int np) {
  const float sc = fmaxf(size0, size1) / 2.f;
  const float x = (kpts[2 * i] - size0 / 2.f) / sc, y = (kpts[2 * i + 1] - size1 / 2.f) / sc;
  const float pr = x * Wr[2 * f] + y * Wr[2 * f + 1];
  const float c = cosf(pr), s = sinf(pr);
  float* e0 = enc + static_cast<size_t>(i) * hd + 2 * f;
  e0[0] = c, e0[1] = c;
  e0[static_cast<size_t>(np) * hd] = s, e0[static_cast<size_t>(np) * hd + 1] = s;
}

// Wqkv output [N][3d] interleaved as (h, hd, 3) (lightglue.py:153-154) -> q, k (rotary applied, :47-54), v, each [N][d]
__device__ __forceinline__ void gx_qkv_rotary_one(const float* __restrict__ qkv, int i, int c, int d, int hd, const float* __restrict__ enc,
                                                  int np, float* __restrict__ q, float* __restrict__ k, float* __restrict__ v) {
  const float* r = qkv + static_cast<size_t>(i) * 3 * d;
  const int dd = c % hd;  // position inside the head: the encoding is shared by the heads
  const float c0 = enc[static_cast<size_t>(i) * hd + dd], c1 = enc[static_cast<size_t>(i) * hd + dd + 1];
  const float s0 = enc[(static_cast<size_t>(np) + i) * hd + dd], s1 = enc[(static_cast<size_t>(np) + i) * hd + dd + 1];
  const float q0 = r[c * 3], q1 = r[(c + 1) * 3], k0 = r[c * 3 + 1], k1 = r[(c + 1) * 3 + 1];
  const size_t o = static_cast<size_t>(i) * d + c;
  q[o] = q0 * c0 + (-q1) * s0;  // rotate_half: (x0, x1) -> (-x1, x0)
  q[o + 1] = q1 * c1 + q0 * s1;
  k[o] = k0 * c0 + (-k1) * s0;
  k[o + 1] = k1 * c1 + k0 * s1;
  v[o] = r[c * 3 + 2];
  v[o + 1] = r[(c + 1) * 3 + 2];
}

// softmax(q k^T * hd^-0.5) v, fp32.  CTA = 8 warps = 8 queries of one head sharing 32-key tiles of K and V in shared memory;
// lane = key of the tile for the logits, lane = channel (mod 32) for the output.  Online softmax.  HDP = hd rounded up to 32.
// The CTA body takes its query block and head explicitly (the batched path adds a grid dimension over the sides).
template <int HDP>
__device__ __forceinline__ void gx_attention_block(const float* __restrict__ q, const float* __restrict__ k, const float* __restrict__ v,
                                                   int nq, int nk, int d, int hd, float* __restrict__ out, int ldo, int qblk, int head) {
  __shared__ float sk[32][HDP + 1], sv[32][HDP], sq[8][HDP];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31, qi = qblk * 8 + w;
  const int co = head * hd;
  for (int c = lane; c < HDP; c += 32) sq[w][c] = (qi < nq && c < hd) ? q[static_cast<size_t>(qi) * d + co + c] : 0.f;
  const float scale = 1.f / sqrtf(static_cast<float>(hd));
  float mx = -INFINITY, l = 0.f, o[HDP / 32];
#pragma unroll
  for (int j = 0; j < HDP / 32; ++j) o[j] = 0.f;
  for (int k0 = 0; k0 < nk; k0 += 32) {
    __syncthreads();
    for (int e = threadIdx.x; e < 32 * HDP; e += 256) {
      const int r = e / HDP, c = e - r * HDP;
      const bool ok = k0 + r < nk && c < hd;
      sk[r][c] = ok ? k[static_cast<size_t>(k0 + r) * d + co + c] : 0.f;
      sv[r][c] = ok ? v[static_cast<size_t>(k0 + r) * d + co + c] : 0.f;
    }
    __syncthreads();
    float s = 0.f;
#pragma unroll 8
    for (int c = 0; c < HDP; ++c) s = fmaf(sq[w][c], sk[lane][c], s);
    s = (k0 + lane < nk) ? s * scale : -INFINITY;
    float tm = s;
#pragma unroll
    for (int of = 16; of; of >>= 1) tm = fmaxf(tm, __shfl_xor_sync(0xffffffffu, tm, of));
    const float mn = fmaxf(mx, tm), corr = expf(mx - mn), p = expf(s - mn);
    float ps = p;
#pragma unroll
    for (int of = 16; of; of >>= 1) ps += __shfl_xor_sync(0xffffffffu, ps, of);
    l = l * corr + ps;
#pragma unroll
    for (int j = 0; j < HDP / 32; ++j) o[j] *= corr;
    for (int r = 0; r < 32; ++r) {
      const float pr = __shfl_sync(0xffffffffu, p, r);
#pragma unroll
      for (int j = 0; j < HDP / 32; ++j) o[j] = fmaf(pr, sv[r][lane + 32 * j], o[j]);
    }
    mx = mn;
  }
  if (qi >= nq) return;
#pragma unroll
  for (int j = 0; j < HDP / 32; ++j) {
    const int c = lane + 32 * j;
    if (c < hd) out[static_cast<size_t>(qi) * ldo + co + c] = nk > 0 ? o[j] / l : 0.f;  // empty key set -> zeros (lightglue.py:103-104)
  }
}

// y = gelu(layer_norm(x)) over the n features of a row, eps 1e-5, exact (erf) GELU; warp per row
__device__ __forceinline__ void gx_ln_gelu_row(const float* __restrict__ x, int row, int lane, int n, const float* __restrict__ g,
                                               const float* __restrict__ b, float* __restrict__ y) {
  const float* r = x + static_cast<size_t>(row) * n;
  float s = 0.f;
  for (int c = lane; c < n; c += 32) s += r[c];
#pragma unroll
  for (int of = 16; of; of >>= 1) s += __shfl_xor_sync(0xffffffffu, s, of);
  const float mean = s / n;
  float vs = 0.f;
  for (int c = lane; c < n; c += 32) {
    const float dlt = r[c] - mean;
    vs = fmaf(dlt, dlt, vs);
  }
#pragma unroll
  for (int of = 16; of; of >>= 1) vs += __shfl_xor_sync(0xffffffffu, vs, of);
  const float inv = rsqrtf(vs / n + 1e-5f);
  for (int c = lane; c < n; c += 32) {
    const float t = (r[c] - mean) * inv * g[c] + b[c];
    y[static_cast<size_t>(row) * n + c] = 0.5f * t * (1.f + erff(t * 0.70710678118654752440f));
  }
}

// z[row] = x[row] . w + b (token confidence / matchability logits); warp per row
__device__ __forceinline__ void gx_rowdot_row(const float* __restrict__ x, int ldx, int row, int lane, int n, const float* __restrict__ w,
                                              const float* __restrict__ b, float* __restrict__ z) {
  float s = 0.f;
  for (int c = lane; c < n; c += 32) s = fmaf(x[static_cast<size_t>(row) * ldx + c], w[c], s);
#pragma unroll
  for (int of = 16; of; of >>= 1) s += __shfl_xor_sync(0xffffffffu, s, of);
  if (lane == 0) z[row] = s + b[0];
}


// log-sum-exp of the rows (dir 0) or columns (dir 1) of sim [m][n] (row stride ld); warp per row / column
__device__ __forceinline__ void gx_lse_one(const float* __restrict__ sim, int ld, int m, int n, int dir, float* __restrict__ lse, int i,
                                           int lane) {
  const int len = dir == 0 ? n : m;
  float mx = -INFINITY;
  for (int j = lane; j < len; j += 32) mx = fmaxf(mx, dir == 0 ? sim[static_cast<size_t>(i) * ld + j] : sim[static_cast<size_t>(j) * ld + i]);
#pragma unroll
  for (int of = 16; of; of >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, of));
  float s = 0.f;
  for (int j = lane; j < len; j += 32) s += expf((dir == 0 ? sim[static_cast<size_t>(i) * ld + j] : sim[static_cast<size_t>(j) * ld + i]) - mx);
#pragma unroll
  for (int of = 16; of; of >>= 1) s += __shfl_xor_sync(0xffffffffu, s, of);
  if (lane == 0) lse[i] = mx + logf(s);
}

__device__ __forceinline__ float log_sigmoid(float z) { return fminf(z, 0.f) - log1pf(expf(-fabsf(z))); }

// row (dir 0) / column (dir 1) maximum and first argmax of scores = (sim - rlse) + (sim - clse) + logsig(z0) + logsig(z1)
// in the association of the reference (lightglue.py:246-256: scores0 + scores1 + certainties), torch.max order (argmax_takes)
__device__ __forceinline__ void gx_argmax_one(const float* __restrict__ sim, int ld, int m, int n, const float* __restrict__ rlse,
                                              const float* __restrict__ clse, const float* __restrict__ z0, const float* __restrict__ z1,
                                              int dir, float* __restrict__ best, int* __restrict__ arg, int i, int lane) {
  const int len = dir == 0 ? n : m;
  float bv = -INFINITY;
  int bi = 0x7fffffff;
  for (int j = lane; j < len; j += 32) {
    const int r = dir == 0 ? i : j, c = dir == 0 ? j : i;
    const float sv = sim[static_cast<size_t>(r) * ld + c];
    const float val = ((sv - rlse[r]) + (sv - clse[c])) + (log_sigmoid(z0[r]) + log_sigmoid(z1[c]));
    if (argmax_takes(val, j, bv, bi)) bv = val, bi = j;
  }
#pragma unroll
  for (int of = 16; of; of >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, bv, of);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, of);
    if (argmax_takes(ov, oi, bv, bi)) bv = ov, bi = oi;
  }
  if (lane == 0) best[i] = bv, arg[i] = bi;
}

}  // namespace
