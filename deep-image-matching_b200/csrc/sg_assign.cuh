// sg_assign.cuh - the optimal-transport head of SuperGlue (superglue.cu) behind the launch helpers it calls, so that the self-test
// library runs it on its own: the per-pair Sinkhorn constants, the log-space Sinkhorn sweeps with a virtual dustbin row / column
// (models/superglue.py:155-187), and the mutual-max matching with the threshold and ordered compaction (:278-296).
#pragma once
#include <algorithm>
#include <cmath>

#include "common.cuh"

namespace {

// Sinkhorn constants of a pair with m x n live scores (:177-181): c = {norm = -log(m + n), log n, log m}, each rounded once from double
__host__ __device__ inline void sg_pair_consts(int m, int n, float* c) {
  c[0] = static_cast<float>(-log(static_cast<double>(m) + static_cast<double>(n)));
  c[1] = static_cast<float>(log(static_cast<double>(n)));
  c[2] = static_cast<float>(log(static_cast<double>(m)));
}

// One Sinkhorn half step for the pairs p0 + blockIdx.y of a wave, on the m x n score block S_p (row pitch ld, pairs pstride apart)
// with the dustbin row / column (value alpha, :175-177) kept virtual.  dir 0 = row pass over sim:
// u[i] = log_mu(i) - logsumexp_j(Z(i, j) + v[j]) for i = 0..m (row m = dustbin), j = 0..n; dir 1 = the column pass, the same
// computation over the TRANSPOSED block simT with u and v swapped.  Warp per row, coalesced, one online log-sum-exp pass.
__global__ void sg_sink_rows_kernel(const float* __restrict__ S, int ld, size_t pstride, int p0, const int* __restrict__ n_act, int dir,
                                    const float* __restrict__ alpha_p, const float* __restrict__ add, float* __restrict__ out, int vld,
                                    const float* __restrict__ pc) {
  const int p = p0 + blockIdx.y;
  const int m = n_act[2 * p + dir], n = n_act[2 * p + 1 - dir];
  const int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (m == 0 || i > m) return;
  const float alpha = alpha_p[0];
  const float* row = S + p * pstride + static_cast<size_t>(i) * ld;
  const float* v = add + static_cast<size_t>(p) * vld;
  float mx = -INFINITY, s = 0.f;
  for (int j = lane; j <= n; j += 32) {
    const float x = ((i < m && j < n) ? row[j] : alpha) + v[j];
    if (x > mx) {
      s = s * expf(mx - x) + 1.f;
      mx = x;
    } else {
      s += expf(x - mx);
    }
  }
#pragma unroll
  for (int of = 16; of; of >>= 1) {
    const float om = __shfl_xor_sync(0xffffffffu, mx, of), os = __shfl_xor_sync(0xffffffffu, s, of);
    const float nm = fmaxf(mx, om);
    s = (mx == -INFINITY ? 0.f : s * expf(mx - nm)) + (om == -INFINITY ? 0.f : os * expf(om - nm));
    mx = nm;
  }
  const float norm = pc[4 * p], log_bin = pc[4 * p + 1 + dir];
  if (lane == 0) out[static_cast<size_t>(p) * vld + i] = ((i == m) ? norm + log_bin : norm) - (mx + logf(s));
}

// Row maximum and first argmax of Z[i][j] + u[i] + v[j] - norm over the inner m x n block of every pair (:279-280): warp per row,
// grid (ceil(NPs * 32 / 256), P); results at [p * NPs + i].  torch.max order (argmax_takes): the first NaN, else the first maximum.
__global__ void sg_row_max_kernel(const float* __restrict__ Z, int ld, size_t pstride, const int* __restrict__ n_act, const float* __restrict__ u,
                                  const float* __restrict__ v, int vld, const float* __restrict__ pc, int NPs, float* __restrict__ best,
                                  int* __restrict__ arg) {
  const int p = blockIdx.y, m = n_act[2 * p], n = n_act[2 * p + 1];
  const int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (i >= m) return;
  const float* row = Z + p * pstride + static_cast<size_t>(i) * ld;
  const float ui = u[static_cast<size_t>(p) * vld + i], norm = pc[4 * p];
  const float* vp = v + static_cast<size_t>(p) * vld;
  float bv = -INFINITY;
  int bi = 0x7fffffff;
  for (int j = lane; j < n; j += 32) {
    const float val = ((row[j] + ui) + vp[j]) - norm;
    if (argmax_takes(val, j, bv, bi)) bv = val, bi = j;
  }
#pragma unroll
  for (int of = 16; of; of >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, bv, of);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, of);
    if (argmax_takes(ov, oi, bv, bi)) bv = ov, bi = oi;
  }
  if (lane == 0) best[static_cast<size_t>(p) * NPs + i] = bv, arg[static_cast<size_t>(p) * NPs + i] = bi;
}

// Column first argmax of the same values: block (32, 32) = 32 columns x 32 row strides (coalesced reads), grid (ceil(NPs / 32), P)
__global__ void __launch_bounds__(1024) sg_col_arg_kernel(const float* __restrict__ Z, int ld, size_t pstride, const int* __restrict__ n_act,
                                                          const float* __restrict__ u, const float* __restrict__ v, int vld,
                                                          const float* __restrict__ pc, int NPs, int* __restrict__ arg) {
  const int p = blockIdx.y, m = n_act[2 * p], n = n_act[2 * p + 1];
  const int tx = threadIdx.x, ty = threadIdx.y, j = blockIdx.x * 32 + tx;
  if (blockIdx.x * 32 >= n) return;  // block-uniform
  __shared__ float rv[32][33];
  __shared__ int ri[32][33];
  float bv = -INFINITY;
  int bi = 0x7fffffff;
  if (j < n) {
    const float* up = u + static_cast<size_t>(p) * vld;
    const float vj = v[static_cast<size_t>(p) * vld + j], norm = pc[4 * p];
    const float* col = Z + p * pstride + j;
    for (int i = ty; i < m; i += 32) {
      const float val = ((col[static_cast<size_t>(i) * ld] + up[i]) + vj) - norm;
      if (argmax_takes(val, i, bv, bi)) bv = val, bi = i;
    }
  }
  rv[ty][tx] = bv;
  ri[ty][tx] = bi;
  __syncthreads();
  if (ty == 0 && j < n) {
    for (int k = 1; k < 32; ++k)
      if (argmax_takes(rv[k][tx], ri[k][tx], bv, bi)) bv = rv[k][tx], bi = ri[k][tx];
    arg[static_cast<size_t>(p) * NPs + j] = bi;
  }
}

// Mutual check, exp(max0) > match_threshold and ordered compaction (:281-296, correspondence_matrix_from_matches0): one CTA per
// pair; n_matches[p] is the full count, only the first cap rows are written.  Modelled on lg_matches_kernel.
__global__ void __launch_bounds__(1024) sg_matches_kernel(const int* __restrict__ n_act, int NPs, const float* __restrict__ best,
                                                          const int* __restrict__ arg0, const int* __restrict__ arg1, float th,
                                                          long long* __restrict__ matches, float* __restrict__ mscores,
                                                          int* __restrict__ n_matches, int cap) {
  const int p = blockIdx.x, t = threadIdx.x;
  const int m = n_act[2 * p], n = n_act[2 * p + 1];
  const size_t r0 = static_cast<size_t>(p) * NPs;
  __shared__ int wsum[32];
  __shared__ int s_base;
  if (t == 0) s_base = 0;
  __syncthreads();
  if (m > 0 && n > 0) {
    for (int base = 0; base < m; base += blockDim.x) {
      const int i = base + t;
      bool valid = false;
      int j = 0;
      float sc = 0.f;
      if (i < m) {
        j = arg0[r0 + i];
        sc = expf(best[r0 + i]);
        valid = arg1[r0 + j] == i && sc > th;
      }
      const unsigned bal = __ballot_sync(0xffffffffu, valid);
      if ((t & 31) == 0) wsum[t >> 5] = __popc(bal);
      __syncthreads();
      int before = s_base;
      for (int wv = 0; wv < (t >> 5); ++wv) before += wsum[wv];
      before += __popc(bal & ((1u << (t & 31)) - 1u));
      if (valid && before < cap) {
        matches[(static_cast<size_t>(p) * cap + before) * 2 + 0] = i;
        matches[(static_cast<size_t>(p) * cap + before) * 2 + 1] = j;
        mscores[static_cast<size_t>(p) * cap + before] = sc;
      }
      __syncthreads();
      if (t == 0) {
        int tot = 0;
        for (int wv = 0; wv < 32; ++wv) tot += wsum[wv];
        s_base += tot;
      }
      __syncthreads();
    }
  }
  if (t == 0) n_matches[p] = s_base;
}

// ------------------------------------------------------------------ launch helpers
// `half_steps` Sinkhorn half steps (row pass, column pass, row pass, ...; 2 x sinkhorn_iterations in production) of P pairs, wave
// pairs per launch so that all steps of a wave run while its score blocks are L2-resident.  sim / simT: [P][NPt][NPt] score blocks and
// their transposes, live m x n from n_act [2P]; alpha: device scalar; u / v [P][vld] (vld >= NPt + 1) carry the duals in and out, the
// dustbin at index m / n; pc [P][4] from sg_pair_consts.
inline int launch_sg_sinkhorn(dimb_ctx* ctx, cudaStream_t st, int P, int wave, int half_steps, const float* sim, const float* simT, int NPt,
                              const int* n_act, const float* alpha, float* u, float* v, int vld, const float* pc) {
  const size_t ps = static_cast<size_t>(NPt) * NPt;
  const dim3 blk(256);
  const int gx = ceil_div((NPt + 1) * 32, 256);
  for (int p0 = 0; p0 < P; p0 += wave) {
    const int np = std::min(wave, P - p0);
    for (int h = 0; h < half_steps; ++h) {
      if ((h & 1) == 0)
        sg_sink_rows_kernel<<<dim3(gx, np), blk, 0, st>>>(sim, NPt, ps, p0, n_act, 0, alpha, v, u, vld, pc);
      else
        sg_sink_rows_kernel<<<dim3(gx, np), blk, 0, st>>>(simT, NPt, ps, p0, n_act, 1, alpha, u, v, vld, pc);
      DIMB_LAUNCH_CHECK(ctx);
    }
  }
  return DIMB_OK;
}

// Row / column max and first argmax of the log assignment Z + u + v - norm (score blocks Z of pitch ld, pairs pstride apart; best0 /
// arg0 / arg1 [P][NPs]) and the [P][cap] match tables with the full counts n_matches [P].
inline int launch_sg_matches(dimb_ctx* ctx, cudaStream_t st, int P, const float* Z, int ld, size_t pstride, int NPs, const int* n_act,
                             const float* u, const float* v, int vld, const float* pc, float th, float* best0, int* arg0, int* arg1,
                             long long* matches, float* mscores, int* n_matches, int cap) {
  sg_row_max_kernel<<<dim3(ceil_div(NPs * 32, 256), P), 256, 0, st>>>(Z, ld, pstride, n_act, u, v, vld, pc, NPs, best0, arg0);
  DIMB_LAUNCH_CHECK(ctx);
  sg_col_arg_kernel<<<dim3(ceil_div(NPs, 32), P), dim3(32, 32), 0, st>>>(Z, ld, pstride, n_act, u, v, vld, pc, NPs, arg1);
  DIMB_LAUNCH_CHECK(ctx);
  sg_matches_kernel<<<P, 1024, 0, st>>>(n_act, NPs, best0, arg0, arg1, th, matches, mscores, n_matches, cap);
  DIMB_LAUNCH_CHECK(ctx);
  return DIMB_OK;
}

}  // namespace
