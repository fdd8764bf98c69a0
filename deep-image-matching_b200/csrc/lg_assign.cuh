// lg_assign.cuh - the decision kernels of the tensor-core LightGlue (lightglue.cu), behind the launch helpers it calls, so that the
// self-test library runs them on their own:
//   launch_lg_tail / launch_lg_decide: the per-layer tail - token confidence and matchability, the depth-confidence stop test and the
//     width-confidence pruning with ordered compaction (lightglue.py:586-604);
//   launch_lg_assign: the assignment - row / column log-softmax statistics, row / column first argmax of the log assignment, mutual
//     filter, threshold and ordered compaction into the [P][cap] match tables (lightglue.py:246-297, :540-551).
#pragma once
#include "lg_kernels.cuh"

namespace {

// ------------------------------------------------------------------ per-layer tail
__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + expf(-x)); }

// warp per row: token confidence and matchability; counts low-confidence points per pair
__global__ void lg_conf_kernel(LgRows rows, const float* __restrict__ x32, const float* __restrict__ wt, float bt,
                               const float* __restrict__ wm, float bm, float thr, float* __restrict__ tok,
                               float* __restrict__ mat, int* __restrict__ counter, int R, int do_stop) {
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (row >= R) return;
  const int side = row / rows.NP;
  if (rows.stopped[side >> 1] != 0 || (row - side * rows.NP) >= rows.n_act[side]) return;
  const float* x = x32 + static_cast<size_t>(row) * kD + lane * 8;
  float a = 0.f, b = 0.f;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    a = fmaf(x[j], wt[lane * 8 + j], a);
    b = fmaf(x[j], wm[lane * 8 + j], b);
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    a += __shfl_xor_sync(0xffffffffu, a, o);
    b += __shfl_xor_sync(0xffffffffu, b, o);
  }
  if (lane == 0) {
    const float c = sigmoidf_(a + bt);
    tok[row] = c;
    mat[row] = sigmoidf_(b + bm);
    if (do_stop && c < thr) atomicAdd(&counter[side >> 1], 1);
  }
}

// one CTA per pair: stop test (check_if_stop, lightglue.py:593-604) and pruning masks (:586-591) with ordered
// compaction; writes the gather map and the next live counts.
__global__ void __launch_bounds__(1024)
lg_decide_kernel(const int* __restrict__ n_act, int* __restrict__ n_next, const int* __restrict__ n_orig, int* __restrict__ stopped,
                 int* __restrict__ counter, const float* __restrict__ tok, const float* __restrict__ mat, int* __restrict__ map,
                 int NP, int layer, float thr, float depth_conf, float keep_thr, int do_stop, int do_prune, int prune_min) {
  const int p = blockIdx.x, t = threadIdx.x;
  __shared__ int s_stop;
  __shared__ int wsum[32];
  __shared__ int s_base;
  if (stopped[p] != 0) return;
  if (t == 0) {
    int stop = 0;
    if (do_stop) {
      const float num = static_cast<float>(n_orig[2 * p] + n_orig[2 * p + 1]);
      const float ratio = 1.0f - static_cast<float>(counter[p]) / num;
      stop = ratio > depth_conf;
    }
    counter[p] = 0;
    s_stop = stop;
    if (stop) stopped[p] = layer + 1;
  }
  __syncthreads();
  const bool stop = s_stop != 0;
  for (int sd = 0; sd < 2; ++sd) {
    const int side = 2 * p + sd, n = n_act[side];
    int* mp = map + static_cast<size_t>(side) * NP;
    const bool prune = !stop && do_prune && n > prune_min;
    if (!prune) {
      for (int i = t; i < n; i += blockDim.x) mp[i] = i;
      if (t == 0) n_next[side] = n;
      continue;
    }
    if (t == 0) s_base = 0;
    __syncthreads();
    for (int base = 0; base < n; base += blockDim.x) {
      const int i = base + t;
      bool keep = false;
      if (i < n) {
        const size_t row = static_cast<size_t>(side) * NP + i;
        keep = mat[row] > keep_thr;
        if (do_stop) keep = keep || (tok[row] <= thr);  // low-confidence points are never pruned
      }
      const unsigned bal = __ballot_sync(0xffffffffu, keep);
      if ((t & 31) == 0) wsum[t >> 5] = __popc(bal);
      __syncthreads();
      int before = s_base;
      for (int wv = 0; wv < (t >> 5); ++wv) before += wsum[wv];
      before += __popc(bal & ((1u << (t & 31)) - 1u));
      if (keep) mp[before] = i;
      __syncthreads();
      if (t == 0) {
        int tot = 0;
        for (int wv = 0; wv < 32; ++wv) tot += wsum[wv];
        s_base += tot;
      }
      __syncthreads();
    }
    if (t == 0) n_next[side] = s_base;
    __syncthreads();
  }
}

// ------------------------------------------------------------------ assignment
// row log-softmax statistics: warp per row of sim[p] (n0 x n1): max and log(sum exp(x - max))
__global__ void lg_row_lse_kernel(const float* __restrict__ sim, const int* __restrict__ nf, int NP, float* __restrict__ rmax,
                                  float* __restrict__ rlog) {
  const int p = blockIdx.y;
  const int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  const int m = nf[2 * p], n = nf[2 * p + 1];
  if (i >= m) return;
  const float* s = sim + (static_cast<size_t>(p) * NP + i) * NP;
  float mx = -INFINITY;
  for (int j = lane; j < n; j += 32) mx = fmaxf(mx, s[j]);
#pragma unroll
  for (int o = 16; o; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  float sum = 0.f;
  for (int j = lane; j < n; j += 32) sum += expf(s[j] - mx);
#pragma unroll
  for (int o = 16; o; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  if (lane == 0) {
    rmax[static_cast<size_t>(2 * p) * NP + i] = mx;
    rlog[static_cast<size_t>(2 * p) * NP + i] = logf(sum);
  }
}

// column statistics: block (32 x 32) handles 32 columns, rows strided over threadIdx.y
__global__ void lg_col_lse_kernel(const float* __restrict__ sim, const int* __restrict__ nf, int NP, float* __restrict__ cmax,
                                  float* __restrict__ clog) {
  const int p = blockIdx.y, tx = threadIdx.x, ty = threadIdx.y;
  const int m = nf[2 * p], n = nf[2 * p + 1];
  const int j = blockIdx.x * 32 + tx;
  if (blockIdx.x * 32 >= n) return;
  __shared__ float red[32][33];
  const float* s = sim + static_cast<size_t>(p) * NP * NP;
  float mx = -INFINITY;
  if (j < n)
    for (int i = ty; i < m; i += 32) mx = fmaxf(mx, s[static_cast<size_t>(i) * NP + j]);
  red[ty][tx] = mx;
  __syncthreads();
  mx = -INFINITY;
  for (int k = 0; k < 32; ++k) mx = fmaxf(mx, red[k][tx]);
  __syncthreads();
  float sum = 0.f;
  if (j < n)
    for (int i = ty; i < m; i += 32) sum += expf(s[static_cast<size_t>(i) * NP + j] - mx);
  red[ty][tx] = sum;
  __syncthreads();
  if (ty == 0 && j < n) {
    float tot = 0.f;
    for (int k = 0; k < 32; ++k) tot += red[k][tx];
    cmax[static_cast<size_t>(2 * p + 1) * NP + j] = mx;
    clog[static_cast<size_t>(2 * p + 1) * NP + j] = logf(tot);
  }
}

// log assignment value (sigmoid_log_double_softmax, lightglue.py:246-256), same association as the reference:
// scores0 + scores1 + certainties with scoresX = (x - max) - log(sum)
__device__ __forceinline__ float la_value(float x, float rm, float rl, float cm, float cl, float lz0, float lz1) {
  const float s0 = (x - rm) - rl, s1 = (x - cm) - cl;
  return (s0 + s1) + (lz0 + lz1);
}

// row argmax (warp per row), torch.max order (argmax_takes): the first NaN, else the first maximum
__global__ void lg_row_arg_kernel(const float* __restrict__ sim, const int* __restrict__ nf, int NP, const float* __restrict__ mx,
                                  const float* __restrict__ lg, const float* __restrict__ z, float* __restrict__ best,
                                  int* __restrict__ arg) {
  const int p = blockIdx.y;
  const int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  const int m = nf[2 * p], n = nf[2 * p + 1];
  if (i >= m) return;
  const size_t r0 = static_cast<size_t>(2 * p) * NP, r1 = r0 + NP;
  const float* s = sim + (static_cast<size_t>(p) * NP + i) * NP;
  const float rm = mx[r0 + i], rl = lg[r0 + i], lz0 = z[r0 + i];  // z holds logsigmoid(matchability)
  float bv = -INFINITY;
  int bi = 0x7fffffff;
  for (int j = lane; j < n; j += 32) {
    const float v = la_value(s[j], rm, rl, mx[r1 + j], lg[r1 + j], lz0, z[r1 + j]);
    if (argmax_takes(v, j, bv, bi)) bv = v, bi = j;
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (argmax_takes(ov, oi, bv, bi)) bv = ov, bi = oi;
  }
  if (lane == 0) {
    best[r0 + i] = bv;
    arg[r0 + i] = bi;
  }
}

__global__ void lg_col_arg_kernel(const float* __restrict__ sim, const int* __restrict__ nf, int NP, const float* __restrict__ mx,
                                  const float* __restrict__ lg, const float* __restrict__ z, int* __restrict__ arg) {
  const int p = blockIdx.y, tx = threadIdx.x, ty = threadIdx.y;
  const int m = nf[2 * p], n = nf[2 * p + 1];
  const int j = blockIdx.x * 32 + tx;
  if (blockIdx.x * 32 >= n) return;
  __shared__ float rv[32][33];
  __shared__ int ri[32][33];
  const size_t r0 = static_cast<size_t>(2 * p) * NP, r1 = r0 + NP;
  const float* s = sim + static_cast<size_t>(p) * NP * NP;
  float bv = -INFINITY;
  int bi = 0x7fffffff;
  if (j < n) {
    const float cm = mx[r1 + j], cl = lg[r1 + j], lz1 = z[r1 + j];
    for (int i = ty; i < m; i += 32) {
      const float v = la_value(s[static_cast<size_t>(i) * NP + j], mx[r0 + i], lg[r0 + i], cm, cl, z[r0 + i], lz1);
      if (argmax_takes(v, i, bv, bi)) bv = v, bi = i;
    }
  }
  rv[ty][tx] = bv;
  ri[ty][tx] = bi;
  __syncthreads();
  if (ty == 0 && j < n) {
    for (int k = 1; k < 32; ++k)
      if (argmax_takes(rv[k][tx], ri[k][tx], bv, bi)) bv = rv[k][tx], bi = ri[k][tx];
    arg[r1 + j] = bi;
  }
}

// filter_matches (lightglue.py:281-297) + result assembly (:540-551): one CTA per pair, ordered compaction
__global__ void __launch_bounds__(1024)
lg_matches_kernel(const int* __restrict__ nf, const int* __restrict__ n_orig, const int* __restrict__ layer, int NP,
                  const float* __restrict__ best, const int* __restrict__ arg, const int* __restrict__ indf, float th,
                  long long* __restrict__ matches, float* __restrict__ mscores, int* __restrict__ n_matches,
                  int* __restrict__ stop_layer, int cap) {
  const int p = blockIdx.x, t = threadIdx.x;
  const int m = nf[2 * p], n = nf[2 * p + 1];
  const size_t r0 = static_cast<size_t>(2 * p) * NP, r1 = r0 + NP;
  __shared__ int wsum[32];
  __shared__ int s_base;
  const bool empty = n_orig[2 * p] == 0 || n_orig[2 * p + 1] == 0;  // "no keypoints" return: stop = 1 (lightglue.py:518-538)
  if (t == 0) {
    s_base = 0;
    stop_layer[p] = empty ? 1 : layer[p] + 1;
  }
  __syncthreads();
  if (!empty && m > 0 && n > 0) {
    for (int base = 0; base < m; base += blockDim.x) {
      const int i = base + t;
      bool valid = false;
      int j = 0;
      float sc = 0.f;
      if (i < m) {
        j = arg[r0 + i];
        const bool mutual = arg[r1 + j] == i;
        sc = expf(best[r0 + i]);
        valid = mutual && (sc > th);
      }
      const unsigned bal = __ballot_sync(0xffffffffu, valid);
      if ((t & 31) == 0) wsum[t >> 5] = __popc(bal);
      __syncthreads();
      int before = s_base;
      for (int wv = 0; wv < (t >> 5); ++wv) before += wsum[wv];
      before += __popc(bal & ((1u << (t & 31)) - 1u));
      if (valid && before < cap) {
        matches[(static_cast<size_t>(p) * cap + before) * 2 + 0] = indf[r0 + i];
        matches[(static_cast<size_t>(p) * cap + before) * 2 + 1] = indf[r1 + j];
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
// Stop test and pruning of P pairs (side s = rows [s NP, (s + 1) NP)) from the confidences tok / mat of the live rows: stopped[p],
// counter[p] (reset to 0), map [2P][NP] and n_next [2P] of the pairs still running.
inline int launch_lg_decide(dimb_ctx* ctx, cudaStream_t st, int P, int NP, const int* n_act, int* n_next, const int* n_orig,
                            int* stopped, int* counter, const float* tok, const float* mat, int* map, int layer, float thr, float depth_conf,
                            float keep_thr, int do_stop, int do_prune, int prune_min) {
  lg_decide_kernel<<<P, 1024, 0, st>>>(n_act, n_next, n_orig, stopped, counter, tok, mat, map, NP, layer, thr, depth_conf, keep_thr,
                                       do_stop, do_prune, prune_min);
  DIMB_LAUNCH_CHECK(ctx);
  return DIMB_OK;
}

// The tail of layer `layer`: confidences of the live rows of x32 [2P NP][256] (rows.n_act, rows.stopped), then launch_lg_decide.
inline int launch_lg_tail(dimb_ctx* ctx, cudaStream_t st, int P, const LgRows& rows, const float* x32, const float* wt, float bt,
                          const float* wm, float bm, float* tok, float* mat, int* n_next, const int* n_orig, int* stopped, int* counter,
                          int* map, int layer, float thr, float depth_conf, float keep_thr, int do_stop, int do_prune, int prune_min) {
  const int R = 2 * P * rows.NP;
  lg_conf_kernel<<<ceil_div(R * 32, 256), 256, 0, st>>>(rows, x32, wt, bt, wm, bm, thr, tok, mat, counter, R, do_stop);
  DIMB_LAUNCH_CHECK(ctx);
  return launch_lg_decide(ctx, st, P, rows.NP, rows.n_act, n_next, n_orig, stopped, counter, tok, mat, map, layer, thr, depth_conf,
                          keep_thr, do_stop, do_prune, prune_min);
}

// The assignment of P pairs: sim [P][NP][NP] (pair p: nf[2p] x nf[2p + 1] live), z [2P][NP] = logsigmoid(matchability), indf [2P][NP]
// original keypoint indices.  Row statistics land in smax / slog at side 2p, column statistics at side 2p + 1; best [2P][NP] (rows
// only) and arg [2P][NP] (rows at side 2p, columns at side 2p + 1); then the [P][cap] tables, n_matches (the full count) and
// stop_layer (layer[p] + 1, or 1 for a pair with an empty side: n_orig).
inline int launch_lg_assign(dimb_ctx* ctx, cudaStream_t st, int P, int NP, const float* sim, const int* nf, const int* n_orig,
                            const int* layer, const float* z, const int* indf, float th, float* smax, float* slog, float* best, int* arg,
                            long long* matches, float* mscores, int* n_matches, int* stop_layer, int cap) {
  lg_row_lse_kernel<<<dim3(ceil_div(NP * 32, 256), P), 256, 0, st>>>(sim, nf, NP, smax, slog);
  DIMB_LAUNCH_CHECK(ctx);
  lg_col_lse_kernel<<<dim3(NP / 32, P), dim3(32, 32), 0, st>>>(sim, nf, NP, smax, slog);
  DIMB_LAUNCH_CHECK(ctx);
  lg_row_arg_kernel<<<dim3(ceil_div(NP * 32, 256), P), 256, 0, st>>>(sim, nf, NP, smax, slog, z, best, arg);
  DIMB_LAUNCH_CHECK(ctx);
  lg_col_arg_kernel<<<dim3(NP / 32, P), dim3(32, 32), 0, st>>>(sim, nf, NP, smax, slog, z, arg);
  DIMB_LAUNCH_CHECK(ctx);
  lg_matches_kernel<<<P, 1024, 0, st>>>(nf, n_orig, layer, NP, best, arg, indf, th, matches, mscores, n_matches, stop_layer, cap);
  DIMB_LAUNCH_CHECK(ctx);
  return DIMB_OK;
}

}  // namespace
