// nn_match.cu - brute-force descriptor matcher (dimb_nn_match), replacing KorniaMatcher._match_pairs
// (reference matchers/kornia_matcher.py:27-54 -> kornia.feature.DescriptorMatcher nn/mnn/snn/smnn).
//
// The reference materialises the full n0 x n1 distance matrix (torch.cdist, 268 MB at 8192^2) and runs
// min / topk over it.  Here the distance tile never leaves the SM: the tensor-core GEMM of gemm.cuh
// produces a 128 x 128 tile of dot products in registers and its epilogue turns it into distances
// (|a|^2 + |b|^2 - 2ab, clamped, sqrt) and a per-row running (best, second best, argbest) over each
// 32-column chunk; a small merge kernel reduces the chunk partials.  The column statistics needed by the
// mutual / symmetric modes are the same kernel with the operands swapped.
#include <algorithm>
#include <vector>

#include "gemm.cuh"

namespace {

// 128 x 128 output tiles: with register accumulators a 128 x 256 tile leaves the running top-2 epilogue too few registers
// (it spills), so the wider tile's halved A re-reads are not worth it
constexpr int kNnBN = 128;

struct EpiNNTop2 : EpiBase {
  const float *na, *nb;  // squared norms of A rows / B rows
  float *pd1, *pd2;      // [rows][chunks] best / second best SQUARED distance of each 32-column chunk
  int* pi1;              // [rows][chunks] argbest
  int n_rows, n_cols, chunks;
  // Squared distances |a|^2 + |b|^2 - 2ab are compared as they are: sqrt is monotone, so the order inside a chunk is that of
  // the distances (two columns whose squared distances differ in the last bit but whose square roots round to the same float
  // would be a tie for torch.cdist + min and are an ordered pair here: measure-zero, and the merge kernel compares the
  // chunk partials in the sqrt domain again).  This removes the IEEE sqrt (8 instructions) from the per-element path.
  __device__ void operator()(const TileCoord& tc, int r, int n, float (&v)[32], float*) const {
    const int row = tc.m0 + r;
    if (row >= n_rows) return;
    const float a2 = na[row];
    float d1 = INFINITY, d2 = INFINITY;
    int i1 = 0x7fffffff;
    const float4* nb4 = reinterpret_cast<const float4*>(nb + n);  // nb is padded to a multiple of 256 columns
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const float4 b = __ldg(nb4 + q);
      const float bb[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int j = 4 * q + e;
        float d = fmaf(-2.f, v[j], a2 + bb[e]);
        if (n + j >= n_cols) d = INFINITY;
        if (d < d1) {
          d2 = d1;
          d1 = d;
          i1 = n + j;
        } else if (d < d2) {
          d2 = d;
        }
      }
    }
    const size_t o = static_cast<size_t>(row) * chunks + (n >> 5);
    pd1[o] = d1;
    pd2[o] = d2;
    pi1[o] = i1;
  }
};

// (D,n) descriptors (fp32 or fp16, row pitch ld) -> [n_pad][Dp] fp16 hi/lo + squared norms; block (32,8) transposing 32x32
// tiles.  Dp = D rounded up to 64: the padding columns are zero, which changes no distance (any descriptor size works).
// any_lo is set when some value is not exactly fp16: only then does the GEMM need the lo planes.
template <class T>
__global__ void nn_prep_kernel(const T* __restrict__ d, int D, int Dp, int n, int ld, __half* __restrict__ hi, __half* __restrict__ lo,
                               float* __restrict__ norm, int* __restrict__ any_lo) {
  __shared__ float tile[32][33];
  const int t0 = blockIdx.x * 32, tx = threadIdx.x, ty = threadIdx.y;
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  bool nz = false;
  for (int c0 = 0; c0 < Dp; c0 += 32) {
    for (int k = ty; k < 32; k += 8)
      tile[k][tx] = (t0 + tx < n && c0 + k < D) ? static_cast<float>(d[static_cast<size_t>(c0 + k) * ld + t0 + tx]) : 0.f;
    __syncthreads();
    int q = 0;
    for (int k = ty; k < 32; k += 8, ++q) {
      const float v = tile[tx][k];  // token t0+k, channel c0+tx
      if (t0 + k < n) {
        __half h, l;
        split_f32(v, h, l);
        hi[static_cast<size_t>(t0 + k) * Dp + c0 + tx] = h;
        if (lo) lo[static_cast<size_t>(t0 + k) * Dp + c0 + tx] = l;
        nz |= __half2float(l) != 0.f;
      }
      float sq = v * v;
#pragma unroll
      for (int o = 16; o; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
      acc[q] += sq;
    }
    __syncthreads();
  }
  int q = 0;
  for (int k = ty; k < 32; k += 8, ++q)
    if (tx == 0 && t0 + k < n) norm[t0 + k] = acc[q];
  if (any_lo && __any_sync(0xffffffffu, nz) && tx == 0) atomicOr(any_lo, 1);
}

// warp per row: merge chunk partials -> best, second, arg (first index wins ties); the partials are squared distances, the
// comparison happens on the distances (clamp at 0, IEEE sqrt) like torch.cdist + min / topk
__global__ void nn_merge_kernel(const float* __restrict__ pd1, const float* __restrict__ pd2, const int* __restrict__ pi1, int rows,
                                int chunks, float* __restrict__ d1, float* __restrict__ d2, int* __restrict__ i1) {
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (row >= rows) return;
  float b1 = INFINITY, b2 = INFINITY;
  int bi = 0x7fffffff;
  for (int c = lane; c < chunks; c += 32) {
    const size_t o = static_cast<size_t>(row) * chunks + c;
    const float x1 = sqrtf(fmaxf(pd1[o], 0.f)), x2 = sqrtf(fmaxf(pd2[o], 0.f));
    const int xi = pi1[o];
    if (x1 < b1 || (x1 == b1 && xi < bi)) {
      b2 = fminf(b1, x2);
      b1 = x1;
      bi = xi;
    } else {
      b2 = fminf(b2, x1);
    }
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    const float x1 = __shfl_xor_sync(0xffffffffu, b1, o), x2 = __shfl_xor_sync(0xffffffffu, b2, o);
    const int xi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (x1 < b1 || (x1 == b1 && xi < bi)) {
      b2 = fminf(b1, x2);
      b1 = x1;
      bi = xi;
    } else {
      b2 = fminf(b2, x1);
    }
  }
  if (lane == 0) {
    d1[row] = b1;
    d2[row] = b2;
    i1[row] = bi;
  }
}

// one CTA: apply the kornia mode logic and compact in ascending row order
__global__ void __launch_bounds__(1024)
nn_select_kernel(int mode, float th, int n0, int n1, const float* __restrict__ fd1, const float* __restrict__ fd2,
                 const int* __restrict__ fi1, const float* __restrict__ bd1, const float* __restrict__ bd2, const int* __restrict__ bi1,
                 long long* __restrict__ idx, float* __restrict__ dist, int* __restrict__ count, int cap) {
  __shared__ int wsum[32];
  __shared__ int s_base;
  const int t = threadIdx.x;
  if (t == 0) s_base = 0;
  __syncthreads();
  const int ms = min(n0, n1);
  const bool swapped = (mode == DIMB_NN_MNN) && (n0 > n1);  // kornia match_mnn iterates the smaller side
  const int iters = (mode == DIMB_NN_MNN) ? ms : n0;
  for (int base = 0; base < iters; base += blockDim.x) {
    const int i = base + t;
    bool valid = false;
    long long a = 0, b = 0;
    float dv = 0.f;
    if (i < iters) {
      if (mode == DIMB_NN_NN) {
        valid = true, a = i, b = fi1[i], dv = fd1[i];
      } else if (mode == DIMB_NN_MNN) {
        if (!swapped) {
          const int j = fi1[i];
          valid = bi1[j] == i, a = i, b = j, dv = fd1[i];
        } else {
          const int j = bi1[i];  // i indexes desc2
          valid = fi1[j] == i, a = j, b = i, dv = bd1[i];
        }
      } else if (mode == DIMB_NN_SNN) {
        const float ratio = fd1[i] / fd2[i];
        valid = ratio <= th, a = i, b = fi1[i], dv = ratio;
      } else {  // SMNN
        const float rf = fd1[i] / fd2[i];
        const int j = fi1[i];
        const float rb = bd1[j] / bd2[j];
        valid = (rf <= th) && (rb <= th) && (bi1[j] == i);
        a = i, b = j, dv = fmaxf(rf, rb);
      }
    }
    const unsigned bal = __ballot_sync(0xffffffffu, valid);
    if ((t & 31) == 0) wsum[t >> 5] = __popc(bal);
    __syncthreads();
    int before = s_base;
    for (int wv = 0; wv < (t >> 5); ++wv) before += wsum[wv];
    before += __popc(bal & ((1u << (t & 31)) - 1u));
    if (valid && before < cap) {
      idx[2 * before] = a;
      idx[2 * before + 1] = b;
      dist[before] = dv;
    }
    __syncthreads();
    if (t == 0) {
      int tot = 0;
      for (int wv = 0; wv < 32; ++wv) tot += wsum[wv];
      s_base += tot;
    }
    __syncthreads();
  }
  if (t == 0) *count = s_base;
}

struct NNSide {
  __half *hi, *lo;
  float* norm;
  CUtensorMap mA[2], mB[2];
};

int nn_rowtop2(dimb_ctx* ctx, cudaStream_t st, const NNSide& A, int na, const NNSide& B, int nb, int Dp, bool split, float* pd1, float* pd2,
               int* pi1, float* d1, float* d2, int* i1) {
  EpiNNTop2 e;
  e.na = A.norm;
  e.nb = B.norm;
  e.pd1 = pd1;
  e.pd2 = pd2;
  e.pi1 = pi1;
  e.n_rows = na;
  e.n_cols = nb;
  e.chunks = round_up(nb, kNnBN) / 32;
  TcOperands ops;
  ops.Ah = A.mA[0];
  ops.Al = A.mA[1];
  ops.Bh = B.mB[0];
  ops.Bl = B.mB[1];
  GemmArgs g{};
  g.num_kb = Dp / 64;
  g.M = na;
  g.N = nb;
  g.Ah = A.hi;
  g.Al = A.lo;
  g.Bh = B.hi;
  g.Bl = B.lo;
  g.lda = Dp;
  g.ldb = Dp;
  // descriptors that are exactly fp16 (everything read back from features.h5 is) have zero lo planes: ONE MMA per product is
  // exact, and the 256-descriptor B panel (128 KB) stays resident in shared memory while the A tiles stream
  DIMB_TRY((launch_gemm<kNnBN, false>(ctx, st, ops, g, e, ceil_div(na, kTileM), round_up(nb, kNnBN), "nn.top2_gemm", split ? 1 : 0)));
  ProfScope prof(ctx, st, "nn.merge");
  nn_merge_kernel<<<ceil_div(na * 32, 256), 256, 0, st>>>(pd1, pd2, pi1, na, e.chunks, d1, d2, i1);
  DIMB_LAUNCH_CHECK(ctx);
  return DIMB_OK;
}

struct NNWork {  // grow-only scratch of one matching call (context slots: no cudaMalloc / cudaFree in steady state)
  NNSide s[2];
  float *pd1, *pd2, *fd1, *fd2, *bd1, *bd2;
  int *pi1, *fi1, *bi1, *any_lo;
  int Dp, p0, p1;
};

int nn_workspace(dimb_ctx* ctx, int n0, int n1, int D, NNWork* w) {
  int slot = 8;  // slots 0..7 belong to the host-buffer entry (staging + outputs)
  auto alloc = [&](void* p, size_t bytes) -> int { return dimb_scratch(ctx, slot++, bytes, reinterpret_cast<void**>(p)); };
  w->Dp = round_up(D, 64);
  w->p0 = round_up(n0, kNnBN);
  w->p1 = round_up(n1, kNnBN);
  for (int i = 0; i < 2; ++i) {
    const int pn = i ? w->p1 : w->p0;
    NNSide& sd = w->s[i];
    DIMB_TRY(alloc(&sd.hi, static_cast<size_t>(pn) * w->Dp * sizeof(__half)));
    DIMB_TRY(alloc(&sd.lo, static_cast<size_t>(pn) * w->Dp * sizeof(__half)));
    DIMB_TRY(alloc(&sd.norm, static_cast<size_t>(pn) * sizeof(float)));
    DIMB_TRY(dimb_tmap_2d(ctx, &sd.mA[0], sd.hi, pn, w->Dp, w->Dp, kTileM));
    DIMB_TRY(dimb_tmap_2d(ctx, &sd.mA[1], sd.lo, pn, w->Dp, w->Dp, kTileM));
    DIMB_TRY(dimb_tmap_2d(ctx, &sd.mB[0], sd.hi, pn, w->Dp, w->Dp, kNnBN));  // as B operand: boxes of kNnBN rows
    DIMB_TRY(dimb_tmap_2d(ctx, &sd.mB[1], sd.lo, pn, w->Dp, w->Dp, kNnBN));
  }
  const size_t pm = std::max(w->p0, w->p1), ch = pm / 32;
  DIMB_TRY(alloc(&w->pd1, pm * ch * sizeof(float)));
  DIMB_TRY(alloc(&w->pd2, pm * ch * sizeof(float)));
  DIMB_TRY(alloc(&w->pi1, pm * ch * sizeof(int)));
  DIMB_TRY(alloc(&w->fd1, w->p0 * sizeof(float)));
  DIMB_TRY(alloc(&w->fd2, w->p0 * sizeof(float)));
  DIMB_TRY(alloc(&w->fi1, w->p0 * sizeof(int)));
  DIMB_TRY(alloc(&w->bd1, w->p1 * sizeof(float)));
  DIMB_TRY(alloc(&w->bd2, w->p1 * sizeof(float)));
  DIMB_TRY(alloc(&w->bi1, w->p1 * sizeof(int)));
  DIMB_TRY(alloc(&w->any_lo, sizeof(int)));
  return DIMB_OK;
}

// prep of both sides on `st`; the rows of the padded operands beyond n are left as they are (their distances are never read:
// the epilogue masks columns >= n_cols and rows >= n_rows)
int nn_prep(dimb_ctx* ctx, cudaStream_t st, const NNWork& w, const void* d0, int n0, int ld0, const void* d1, int n1, int ld1, int D,
            int f16, bool want_lo) {
  ProfScope prof(ctx, st, "nn.prep");
  DIMB_CUDA_OK(ctx, cudaMemsetAsync(w.any_lo, 0, sizeof(int), st));
  for (int i = 0; i < 2; ++i) {
    const void* d = i ? d1 : d0;
    const int n = i ? n1 : n0, ld = i ? ld1 : ld0, pn = i ? w.p1 : w.p0;
    const NNSide& sd = w.s[i];
    // zero norms of the padding rows keep the (masked) padded columns finite
    DIMB_CUDA_OK(ctx, cudaMemsetAsync(sd.norm, 0, static_cast<size_t>(pn) * sizeof(float), st));
    if (f16)
      nn_prep_kernel<__half><<<ceil_div(n, 32), dim3(32, 8), 0, st>>>(static_cast<const __half*>(d), D, w.Dp, n, ld, sd.hi, nullptr, sd.norm, nullptr);
    else
      nn_prep_kernel<float><<<ceil_div(n, 32), dim3(32, 8), 0, st>>>(static_cast<const float*>(d), D, w.Dp, n, ld, sd.hi,
                                                                   want_lo ? sd.lo : nullptr, sd.norm, w.any_lo);
    DIMB_LAUNCH_CHECK(ctx);
  }
  return DIMB_OK;
}

int nn_core(dimb_ctx* ctx, cudaStream_t st, const NNWork& w, int n0, int n1, bool split, int mode, float th, long long* d_idx, float* d_dist,
            int* d_n, int cap) {
  DIMB_TRY(nn_rowtop2(ctx, st, w.s[0], n0, w.s[1], n1, w.Dp, split, w.pd1, w.pd2, w.pi1, w.fd1, w.fd2, w.fi1));
  if (mode == DIMB_NN_MNN || mode == DIMB_NN_SMNN)
    DIMB_TRY(nn_rowtop2(ctx, st, w.s[1], n1, w.s[0], n0, w.Dp, split, w.pd1, w.pd2, w.pi1, w.bd1, w.bd2, w.bi1));
  ProfScope prof(ctx, st, "nn.select");
  nn_select_kernel<<<1, 1024, 0, st>>>(mode, th, n0, n1, w.fd1, w.fd2, w.fi1, w.bd1, w.bd2, w.bi1, d_idx, d_dist, d_n, cap);
  DIMB_LAUNCH_CHECK(ctx);
  return DIMB_OK;
}

bool nn_trivially_empty(int n0, int n1, int mode) {
  // kornia: empty inputs / fewer than two candidates for the ratio tests -> no match
  return n0 == 0 || n1 == 0 || (mode == DIMB_NN_SNN && n1 < 2) || (mode == DIMB_NN_SMNN && (n0 < 2 || n1 < 2));
}

}  // namespace

extern "C" {

// Device-resident entry: descriptors (D,n) with row pitch ld in HBM (fp32, or fp16 as the device feature store keeps them),
// results in device buffers, asynchronous on `stream`.  fp16 input takes the single-MMA path (exact: the values ARE fp16).
int dimb_nn_match_dev(dimb_ctx* ctx, const void* d_desc0, int n0, int ld0, const void* d_desc1, int n1, int ld1, int D, int desc_f16,
                      int mode, float th, int64_t* d_idx, float* d_dist, int* d_n, int cap, void* stream) {
  if (!ctx || !d_idx || !d_dist || !d_n || n0 < 0 || n1 < 0 || D < 1 || mode < 0 || mode > 3 || cap < 1) {
    if (ctx) dimb_set_error(ctx, "dimb_nn_match_dev: invalid argument (descriptor dimension >= 1, mode 0..3, cap >= 1)");
    return DIMB_ERR_ARG;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  DIMB_CUDA_OK(ctx, cudaSetDevice(ctx->device));
  if (nn_trivially_empty(n0, n1, mode)) {
    DIMB_CUDA_OK(ctx, cudaMemsetAsync(d_n, 0, sizeof(int), st));
    return DIMB_OK;
  }
  if (!d_desc0 || !d_desc1) return DIMB_ERR_ARG;
  NNWork w;
  DIMB_TRY(nn_workspace(ctx, n0, n1, D, &w));
  const bool split = !desc_f16 && ctx->precision == DIMB_PRECISION_EXACT;  // fp32 input: no host round trip to learn whether lo == 0
  DIMB_TRY(nn_prep(ctx, st, w, d_desc0, n0, ld0 ? ld0 : n0, d_desc1, n1, ld1 ? ld1 : n1, D, desc_f16, split));
  return nn_core(ctx, st, w, n0, n1, split, mode, th, reinterpret_cast<long long*>(d_idx), d_dist, d_n, cap);
}

int dimb_nn_match(dimb_ctx* ctx, const float* d0, int n0, const float* d1, int n1, int D, int mode, float th, int64_t* idx, float* dist,
                  int* n, int cap) {
  if (!ctx || !idx || !dist || !n || n0 < 0 || n1 < 0 || D < 1 || mode < 0 || mode > 3 || cap < 1) {
    if (ctx) dimb_set_error(ctx, "dimb_nn_match: invalid argument (descriptor dimension >= 1, mode nn/mnn/snn/smnn, cap >= 1)");
    return DIMB_ERR_ARG;
  }
  *n = 0;
  if (nn_trivially_empty(n0, n1, mode)) return DIMB_OK;
  if (!d0 || !d1) return DIMB_ERR_ARG;
  DIMB_CUDA_OK(ctx, cudaSetDevice(ctx->device));
  cudaStream_t st = 0;
  float *raw0, *raw1, *o_dist;
  long long* o_idx;
  int* o_n;
  DIMB_TRY(dimb_scratch(ctx, 0, static_cast<size_t>(D) * n0 * sizeof(float), reinterpret_cast<void**>(&raw0)));
  DIMB_TRY(dimb_scratch(ctx, 1, static_cast<size_t>(D) * n1 * sizeof(float), reinterpret_cast<void**>(&raw1)));
  DIMB_TRY(dimb_scratch(ctx, 2, static_cast<size_t>(cap) * 2 * sizeof(long long), reinterpret_cast<void**>(&o_idx)));
  DIMB_TRY(dimb_scratch(ctx, 3, static_cast<size_t>(cap) * sizeof(float), reinterpret_cast<void**>(&o_dist)));
  DIMB_TRY(dimb_scratch(ctx, 4, sizeof(int), reinterpret_cast<void**>(&o_n)));
  NNWork w;
  DIMB_TRY(nn_workspace(ctx, n0, n1, D, &w));
  DIMB_CUDA_OK(ctx, cudaMemcpyAsync(raw0, d0, static_cast<size_t>(D) * n0 * sizeof(float), cudaMemcpyHostToDevice, st));
  DIMB_CUDA_OK(ctx, cudaMemcpyAsync(raw1, d1, static_cast<size_t>(D) * n1 * sizeof(float), cudaMemcpyHostToDevice, st));
  const bool exact = ctx->precision == DIMB_PRECISION_EXACT;
  DIMB_TRY(nn_prep(ctx, st, w, raw0, n0, n0, raw1, n1, n1, D, 0, exact));
  int any_lo = 0;  // descriptors read back from features.h5 are exactly fp16: then the lo planes are zero and one MMA is exact
  if (exact) {
    DIMB_CUDA_OK(ctx, cudaMemcpyAsync(&any_lo, w.any_lo, sizeof(int), cudaMemcpyDeviceToHost, st));
    DIMB_CUDA_OK(ctx, cudaStreamSynchronize(st));
  }
  DIMB_TRY(nn_core(ctx, st, w, n0, n1, exact && any_lo != 0, mode, th, o_idx, o_dist, o_n, cap));
  int cnt = 0;
  DIMB_CUDA_OK(ctx, cudaMemcpyAsync(&cnt, o_n, sizeof(int), cudaMemcpyDeviceToHost, st));
  DIMB_CUDA_OK(ctx, cudaStreamSynchronize(st));
  *n = cnt;
  if (cnt > cap) {
    dimb_set_error(ctx, "dimb_nn_match: more matches than cap");
    return DIMB_ERR_CAPACITY;
  }
  if (cnt > 0) {
    DIMB_CUDA_OK(ctx, cudaMemcpy(idx, o_idx, static_cast<size_t>(cnt) * 2 * sizeof(long long), cudaMemcpyDeviceToHost));
    DIMB_CUDA_OK(ctx, cudaMemcpy(dist, o_dist, static_cast<size_t>(cnt) * sizeof(float), cudaMemcpyDeviceToHost));
  }
  return DIMB_OK;
}

}  // extern "C"
