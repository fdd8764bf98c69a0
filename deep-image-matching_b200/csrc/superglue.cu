// superglue.cu - SuperGlue matching (dimb_sg_*), replacing SuperGlueMatcher._match_pairs
// (reference src/deep_image_matching/matchers/superglue.py:75-106, adapter features_2_sg :8-41) and the model it drives
// (thirdparty/SuperGluePretrainedNetwork/models/superglue.py:51-305: keypoint encoder :73-84, attentional GNN :96-152,
// log-space Sinkhorn :155-187, mutual-max matching :278-296).
//
// SuperGlue's attention shape is 256 / 4 heads x 64 - the shape of LightGlue's tensor-core kernels - so the 18 GNN layers run on the
// shared building blocks of lg_kernels.cuh: per layer ONE q|k GEMM (EpiQK without rotary), the V^T GEMM, the flash-attention kernel
// (self: keys of the same side, cross: keys and values of the other side), merge -> message half of the [x | message] buffer, MLP0
// with the eval-mode BatchNorm folded in and a ReLU / hi-lo-split epilogue, MLP3 + residual; then final_proj and the score matrix as
// wgmma GEMMs, and 100 log-space Sinkhorn sweeps over the L2-resident score matrix with the dustbin row / column kept virtual
// (coalesced row and column passes).  Done once at create time: BatchNorm folding, and the reference's (dim, heads)-interleaved
// channel order of `view(b, dim, heads, n)` (:111-113) permuted to head-major.  The keypoint encoder (3 -> 32 -> 64 -> 128 -> 256 -> 256,
// 0.2 GMAC) stays on the plain fp32 kernels of generic_kernels.cuh; the whole plain-fp32 path remains as the debug twin (DIMB_TC=0).
#include <algorithm>
#include <cmath>
#include <cstring>
#include <memory>
#include <vector>

#include "generic_kernels.cuh"
#include "lg_kernels.cuh"

namespace {

// ---------------------------------------------------------------- tensor-core path helpers
// out = relu(acc + bias) -> fp16 hi/lo planes (MLP0 with the BatchNorm folded into weights and bias), live tiles only
struct EpiSgReluSplit : EpiBase {
  LgRows rows;
  __half *hi, *lo;
  const float* bias;
  int ldc;
  __device__ bool tile_active(const TileCoord& tc) const { return rows.active(tc.m0); }
  __device__ void operator()(const TileCoord& tc, int r, int n, float (&v)[32], float* sc) const {
    const int lane = r & 31, col = n + (lane & 7) * 4;
    const float4 b = __ldg(reinterpret_cast<const float4*>(bias + col));
    float4 f[8];
    warp_transpose32(v, sc, f);
#pragma unroll
    for (int it = 0; it < 8; ++it) {
      const size_t off = static_cast<size_t>(tc.m0 + (r & ~31) + it * 4 + (lane >> 3)) * ldc + col;
      store_split4(hi + off, lo ? lo + off : nullptr,
                   make_float4(fmaxf(f[it].x + b.x, 0.f), fmaxf(f[it].y + b.y, 0.f), fmaxf(f[it].z + b.z, 0.f), fmaxf(f[it].w + b.w, 0.f)));
    }
  }
};

// FeaturesDict inputs -> device layouts: descriptors (D,n) -> token-major [n][ldd] (32 x 32 tile transpose), keypoints / scores ->
// the keypoint encoder's input [n][3] = (normalised x, normalised y, score)  (normalize_keypoints, superglue.py:63-70)
__global__ void sg_input_kernel(const float* __restrict__ desc, int ld, int n, const float* __restrict__ kpts, const float* __restrict__ scores,
                                float cx, float cy, float sc, float* __restrict__ dst, int ldd, float* __restrict__ enc_in) {
  __shared__ float tile[32][33];
  const int t0 = blockIdx.x * 32, c0 = blockIdx.y * 32, tx = threadIdx.x, ty = threadIdx.y;
  for (int k = ty; k < 32; k += 8) tile[k][tx] = (t0 + tx < n) ? desc[static_cast<size_t>(c0 + k) * ld + t0 + tx] : 0.f;
  __syncthreads();
  for (int k = ty; k < 32; k += 8)
    if (t0 + k < n) dst[static_cast<size_t>(t0 + k) * ldd + c0 + tx] = tile[tx][k];
  if (blockIdx.y == 0 && ty == 0 && t0 + tx < n) {
    const int i = t0 + tx;
    enc_in[3 * i] = (kpts[2 * i] - cx) / sc;
    enc_in[3 * i + 1] = (kpts[2 * i + 1] - cy) / sc;
    enc_in[3 * i + 2] = scores[i];
  }
}

// encoder output (fp32 [n][ld]) -> token state of side `side`: fp32 master + fp16 hi/lo first half of the concat buffer
__global__ void sg_pack_kernel(const float* __restrict__ src, int ld, int n, int row0, float* __restrict__ x32, __half* __restrict__ xh,
                               __half* __restrict__ xl) {
  const int i = blockIdx.x, c = threadIdx.x;  // 256 threads = channels
  if (i >= n) return;
  const float v = src[static_cast<size_t>(i) * ld + c];
  const size_t row = static_cast<size_t>(row0) + i;
  x32[row * 256 + c] = v;
  __half h, l;
  split_f32(v, h, l);
  xh[row * 512 + c] = h;
  if (xl) xl[row * 512 + c] = l;
}

// Sinkhorn half steps on the m x n score block S (row pitch ld) with the dustbin row / column (value alpha, :175-177) kept virtual.
// Row pass: u[i] = log_mu(i) - logsumexp_j(Z(i, j) + v[j]) for i = 0..m (row m = dustbin), j = 0..n.  Warp per row, coalesced.
__global__ void sg_sink_rows_kernel(const float* __restrict__ S, int ld, int m, int n, const float* __restrict__ alpha_p, const float* __restrict__ v,
                                    float* __restrict__ u, float norm, float log_bin) {
  const int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (i > m) return;
  const float alpha = alpha_p[0];
  const float* row = S + static_cast<size_t>(i) * ld;
  float mx = -INFINITY, s = 0.f;  // online log-sum-exp: one pass over the row
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
  if (lane == 0) u[i] = ((i == m) ? norm + log_bin : norm) - (mx + logf(s));
}
// The column sweep v[j] = log_nu(j) - logsumexp_i(Z(i, j) + u[i]) is the same kernel on the TRANSPOSED score block (g->simT).

// couplings (:175-177): fill the dustbin row / column of the (m+1) x (n+1) matrix with alpha
__global__ void sg_fill_bins_kernel(float* __restrict__ Z, int ld, int m, int n, const float* __restrict__ alpha) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const float a = alpha[0];
  if (i <= n) Z[static_cast<size_t>(m) * ld + i] = a;
  if (i < m) Z[static_cast<size_t>(i) * ld + n] = a;
}

// One Sinkhorn half step (:158-165): out[i] = log_marg(i) - logsumexp_j(Z[i][j] + add[j]) over rows (dir 0) or columns (dir 1) of
// the (m+1) x (n+1) couplings; log_marg = norm for the regular entries, norm + log(other count) for the dustbin.  Warp per line.
__global__ void sg_sinkhorn_kernel(const float* __restrict__ Z, int ld, int m1, int n1, int dir, const float* __restrict__ add,
                                   float* __restrict__ out, float norm, float log_bin) {
  const int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  const int cnt = dir == 0 ? m1 : n1, len = dir == 0 ? n1 : m1;
  if (i >= cnt) return;
  float mx = -INFINITY;
  for (int j = lane; j < len; j += 32) mx = fmaxf(mx, (dir == 0 ? Z[static_cast<size_t>(i) * ld + j] : Z[static_cast<size_t>(j) * ld + i]) + add[j]);
#pragma unroll
  for (int of = 16; of; of >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, of));
  float s = 0.f;
  for (int j = lane; j < len; j += 32) s += expf((dir == 0 ? Z[static_cast<size_t>(i) * ld + j] : Z[static_cast<size_t>(j) * ld + i]) + add[j] - mx);
#pragma unroll
  for (int of = 16; of; of >>= 1) s += __shfl_xor_sync(0xffffffffu, s, of);
  if (lane == 0) out[i] = ((i == cnt - 1) ? norm + log_bin : norm) - (mx + logf(s));
}

// row (dir 0) / column (dir 1) maximum and first argmax of Z[i][j] + u[i] + v[j] - norm over the inner m x n block (:279-280)
__global__ void sg_argmax_kernel(const float* __restrict__ Z, int ld, int m, int n, const float* __restrict__ u, const float* __restrict__ v,
                                 float norm, int dir, float* __restrict__ best, int* __restrict__ arg) {
  const int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  const int cnt = dir == 0 ? m : n, len = dir == 0 ? n : m;
  if (i >= cnt) return;
  float bv = -INFINITY;
  int bi = 0x7fffffff;
  for (int j = lane; j < len; j += 32) {
    const int r = dir == 0 ? i : j, c = dir == 0 ? j : i;
    const float val = ((Z[static_cast<size_t>(r) * ld + c] + u[r]) + v[c]) - norm;
    if (val > bv) bv = val, bi = j;
  }
#pragma unroll
  for (int of = 16; of; of >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, bv, of);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, of);
    if (ov > bv || (ov == bv && oi < bi)) bv = ov, bi = oi;
  }
  if (lane == 0) best[i] = bv, arg[i] = bi;
}

struct SgLin {
  float *w = nullptr, *b = nullptr;
  int n = 0, k = 0;
};
struct SgTcLin {  // fp16 hi/lo planes [n][k] + fp32 bias + TMA maps (boxes of 128 rows)
  __half *wh = nullptr, *wl = nullptr;
  float* bias = nullptr;
  int n = 0, k = 0;
  CUtensorMap tmh, tml;
};
struct SgTcLayer {
  SgTcLin qkv, merge, mlp0, mlp3;  // qkv = [Wq ; Wk ; Wv] stacked (768 x 256), head-major rows
};
struct SgLayer {
  SgLin q, k, v, merge, mlp0, mlp3;
};

}  // namespace

struct dimb_sg {
  dimb_ctx* ctx;
  std::vector<void*> mem;
  dimb_sg_conf conf;
  int NP, L;
  std::vector<int> cross;  // per GNN layer: 1 = cross, 0 = self
  SgLin kenc[5];
  std::vector<SgLayer> layers;
  SgLin final_proj;
  float* bin_score;
  float *cat[2], *q[2], *k[2], *v[2], *att, *hid, *enc_a, *enc_b, *md[2], *Z, *u, *vv, *best0, *best1;
  int *arg0, *arg1;
  // ---- tensor-core path (sides are rows [s * NPt, (s + 1) * NPt) of every token buffer, NPt = NP rounded up to 128)
  int NPt = 0;
  std::vector<SgTcLayer> tc;
  SgTcLin tc_final;
  float* x32 = nullptr;
  __half *xh, *xl, *qh, *ql, *kh, *kl, *vth, *vtl, *ctxh, *ctxl, *h2h, *h2l, *mdh, *mdl;
  float *sim = nullptr, *simT = nullptr;  // score block and its transpose (both sweeps of a Sinkhorn iteration read rows)
  int *n_act = nullptr, *stopped = nullptr;
  CUtensorMap m_x[2], m_ctx[2], m_h2[2], m_md[2], m_q128[2], m_k64[2], m_vt[2];
};

namespace {

constexpr int kSgD = 256, kSgHeads = 4, kSgHd = 64;

int sg_linear(dimb_sg* g, cudaStream_t st, const float* A, int lda, const SgLin& l, float* C, int ldc, int M, int relu, float scale = 1.f,
              const float* resid = nullptr, int ldr = 0) {
  if (M <= 0) return DIMB_OK;
  dim3 grid(ceil_div(l.n, 64), ceil_div(M, 64));
  gx_linear_kernel<<<grid, 256, 0, st>>>(A, lda, l.w, l.k, l.b, C, ldc, M, l.n, l.k, scale, resid, ldr, relu);
  DIMB_LAUNCH_CHECK(g->ctx);
  return DIMB_OK;
}

// host-side weight preparation: 1x1 conv [n][k] (+ optional eval BatchNorm folded in), optional row / column permutations
struct HostLin {
  std::vector<float> w, b;
  int n, k;
};
HostLin take_conv(const float*& p, int n, int k) {
  HostLin l;
  l.n = n, l.k = k;
  l.w.assign(p, p + static_cast<size_t>(n) * k);
  p += static_cast<size_t>(n) * k;
  l.b.assign(p, p + n);
  p += n;
  return l;
}
void fold_bn(HostLin& l, const float*& p) {  // gamma, beta, running_mean, running_var (eps 1e-5)
  const float *g = p, *be = p + l.n, *mu = p + 2 * l.n, *var = p + 3 * l.n;
  for (int o = 0; o < l.n; ++o) {
    const float a = g[o] / std::sqrt(var[o] + 1e-5f);
    for (int c = 0; c < l.k; ++c) l.w[static_cast<size_t>(o) * l.k + c] *= a;
    l.b[o] = a * (l.b[o] - mu[o]) + be[o];
  }
  p += 4 * l.n;
}
inline int head_major(int c) { return (c % kSgHeads) * kSgHd + c / kSgHeads; }  // reference channel d * heads + h -> h * 64 + d
void permute_rows(HostLin& l) {
  HostLin o = l;
  for (int c = 0; c < l.n; ++c) {
    std::memcpy(&o.w[static_cast<size_t>(head_major(c)) * l.k], &l.w[static_cast<size_t>(c) * l.k], l.k * sizeof(float));
    o.b[head_major(c)] = l.b[c];
  }
  l = o;
}
void permute_cols(HostLin& l) {
  HostLin o = l;
  for (int r = 0; r < l.n; ++r)
    for (int c = 0; c < l.k; ++c) o.w[static_cast<size_t>(r) * l.k + head_major(c)] = l.w[static_cast<size_t>(r) * l.k + c];
  l = o;
}
int upload_tc(dimb_ctx* ctx, SgTcLin& d, const HostLin& h) {
  d.n = h.n, d.k = h.k;
  std::vector<__half> hi(h.w.size()), lo(h.w.size());
  for (size_t i = 0; i < h.w.size(); ++i) {
    hi[i] = __float2half_rn(h.w[i]);
    lo[i] = __float2half_rn(h.w[i] - __half2float(hi[i]));
  }
  DIMB_TRY(dimb_alloc_t(ctx, &d.wh, hi.size(), false));
  DIMB_TRY(dimb_alloc_t(ctx, &d.wl, lo.size(), false));
  DIMB_TRY(dimb_alloc_t(ctx, &d.bias, h.b.size(), false));
  DIMB_CUDA_OK(ctx, cudaMemcpy(d.wh, hi.data(), hi.size() * sizeof(__half), cudaMemcpyHostToDevice));
  DIMB_CUDA_OK(ctx, cudaMemcpy(d.wl, lo.data(), lo.size() * sizeof(__half), cudaMemcpyHostToDevice));
  DIMB_CUDA_OK(ctx, cudaMemcpy(d.bias, h.b.data(), h.b.size() * sizeof(float), cudaMemcpyHostToDevice));
  DIMB_TRY(dimb_tmap_2d(ctx, &d.tmh, d.wh, h.n, h.k, h.k, 128));
  DIMB_TRY(dimb_tmap_2d(ctx, &d.tml, d.wl, h.n, h.k, h.k, 128));
  return DIMB_OK;
}
int upload(dimb_ctx* ctx, SgLin& d, const HostLin& h) {
  d.n = h.n, d.k = h.k;
  DIMB_TRY(dimb_alloc_t(ctx, &d.w, h.w.size(), false));
  DIMB_TRY(dimb_alloc_t(ctx, &d.b, h.b.size(), false));
  DIMB_CUDA_OK(ctx, cudaMemcpy(d.w, h.w.data(), h.w.size() * sizeof(float), cudaMemcpyHostToDevice));
  DIMB_CUDA_OK(ctx, cudaMemcpy(d.b, h.b.data(), h.b.size() * sizeof(float), cudaMemcpyHostToDevice));
  return DIMB_OK;
}

// one GEMM over all 2 * NPt token rows: C = A [R][K] * W^T on the wgmma kernel of gemm.cuh with epilogue `epi`
template <class Epi>
int sg_tc_gemm(dimb_sg* g, cudaStream_t st, const CUtensorMap* A, const __half* Ah, const __half* Al, int lda, const SgTcLin& w, int n_out,
               const Epi& epi, const char* tag) {
  TcOperands ops;
  ops.Ah = A[0];
  ops.Al = A[1];
  ops.Bh = w.tmh;
  ops.Bl = w.tml;
  GemmArgs ga{};
  ga.num_kb = w.k / 64;
  ga.M = 2 * g->NPt;
  ga.N = n_out;
  ga.Ah = Ah;
  ga.Al = Al;
  ga.Bh = w.wh;
  ga.Bl = w.wl;
  ga.lda = lda;
  ga.ldb = w.k;
  return launch_gemm<128, false>(g->ctx, st, ops, ga, epi, 2 * g->NPt / kTileM, n_out, tag);
}

// keypoint-encoded descriptors (g->cat[s], fp32) -> 18 GNN layers, final projection and the m x n score block (g->sim) on the
// tensor-core kernels.  Both sides advance together from the OLD descriptors, as the reference does (superglue.py:147-151).
int sg_gnn_tc(dimb_sg* g, cudaStream_t st, const int n[2]) {
  dimb_ctx* ctx = g->ctx;
  const bool exact = ctx->precision == DIMB_PRECISION_EXACT;
  const int NPt = g->NPt, d = kSgD, R = 2 * NPt;
  const int zero = 0;
  DIMB_CUDA_OK(ctx, cudaMemcpyAsync(g->n_act, n, 2 * sizeof(int), cudaMemcpyHostToDevice, st));
  DIMB_CUDA_OK(ctx, cudaMemcpyAsync(g->stopped, &zero, sizeof(int), cudaMemcpyHostToDevice, st));
  for (int s = 0; s < 2; ++s) {
    sg_pack_kernel<<<n[s], 256, 0, st>>>(g->cat[s], 2 * d, n[s], s * NPt, g->x32, g->xh, exact ? g->xl : nullptr);
    DIMB_LAUNCH_CHECK(ctx);
  }
  const LgRows rows{g->n_act, g->stopped, NPt};
  for (int i = 0; i < g->L; ++i) {
    const SgTcLayer& ly = g->tc[i];
    {  // q | k for every token of both sides (no rotary: EpiQK's cross flag only switches the rotation off)
      EpiQK e;
      e.rows = rows;
      e.bias = ly.qkv.bias;
      e.cs = e.sn = nullptr;
      e.qh = g->qh, e.ql = exact ? g->ql : nullptr, e.kh = g->kh, e.kl = exact ? g->kl : nullptr;
      e.cross = 1;
      DIMB_TRY(sg_tc_gemm(g, st, g->m_x, g->xh, g->xl, 2 * d, ly.qkv, 2 * d, e, "sg.qk"));
    }
    {  // V^T: weights as the A operand (rows 512..767 of the stacked projection), tokens as B
      EpiVT e;
      e.rows = rows;
      e.bias = ly.qkv.bias;
      e.vth = g->vth, e.vtl = exact ? g->vtl : nullptr;
      e.w_row0 = 2 * d;
      TcOperands ops;
      ops.Ah = ly.qkv.tmh, ops.Al = ly.qkv.tml, ops.Bh = g->m_x[0], ops.Bl = g->m_x[1];
      GemmArgs ga{};
      ga.num_kb = d / 64;
      ga.M = ly.qkv.n, ga.N = R;
      ga.Ah = ly.qkv.wh, ga.Al = ly.qkv.wl, ga.Bh = g->xh, ga.Bl = g->xl;
      ga.lda = d, ga.ldb = 2 * d;
      DIMB_TRY((launch_gemm<128, false>(ctx, st, ops, ga, e, 2, R, "sg.vT")));
    }
    {  // attention: self layers attend to their own side, cross layers to the keys AND values of the other side
      AttnArgs a;
      a.rows = rows;
      a.cross = g->cross[i];
      a.ctx_h = g->ctxh, a.ctx_l = exact ? g->ctxl : nullptr;
      a.scale = 0.125f;
      a.lazy = ctx->attn_lazy;
      ProfScope prof(ctx, st, "sg.attention");
      dim3 grid(ceil_div(NPt, 2 * kTileM), kHeads, 2);
      DIMB_TRY(launch_lg_attention(ctx, st, grid, g->m_q128, g->m_k64, g->m_vt, a, exact));
      DIMB_LAUNCH_CHECK(ctx);
    }
    {  // merge -> message half of [x | message]
      EpiLgSplit e;
      e.rows = rows;
      e.hi = g->xh, e.lo = exact ? g->xl : nullptr;
      e.bias = ly.merge.bias;
      e.ldc = 2 * d, e.col_off = d;
      DIMB_TRY(sg_tc_gemm(g, st, g->m_ctx, g->ctxh, g->ctxl, d, ly.merge, d, e, "sg.merge"));
    }
    {  // MLP0 (BatchNorm folded) + ReLU
      EpiSgReluSplit e;
      e.rows = rows;
      e.hi = g->h2h, e.lo = exact ? g->h2l : nullptr;
      e.bias = ly.mlp0.bias;
      e.ldc = 2 * d;
      DIMB_TRY(sg_tc_gemm(g, st, g->m_x, g->xh, g->xl, 2 * d, ly.mlp0, 2 * d, e, "sg.mlp0"));
    }
    {  // x += MLP3(...)
      EpiLgResidual e;
      e.rows = rows;
      e.x32 = g->x32;
      e.xh = g->xh, e.xl = exact ? g->xl : nullptr;
      e.bias = ly.mlp3.bias;
      e.residual = 1;
      DIMB_TRY(sg_tc_gemm(g, st, g->m_h2, g->h2h, g->h2l, 2 * d, ly.mlp3, d, e, "sg.mlp3"));
    }
  }
  {  // mdesc = final_proj(x) / 256^0.25 on each side, so that the score block is mdesc0 . mdesc1^T / sqrt(256) (:262-265)
    EpiStoreSplit e;
    e.hi = g->mdh, e.lo = exact ? g->mdl : nullptr;
    e.bias = g->tc_final.bias;
    e.ldc = d, e.col_off = 0, e.n_valid = d, e.m_valid = R;
    e.scale = 0.25f;
    DIMB_TRY(sg_tc_gemm(g, st, g->m_x, g->xh, g->xl, 2 * d, g->tc_final, d, e, "sg.final_proj"));
  }
  {
    EpiSim e;
    e.nf = g->n_act;
    e.sim = g->sim;
    e.NP = NPt;
    e.tiles_per_side = NPt / kTileM;
    TcOperands ops;
    ops.Ah = g->m_md[0], ops.Al = g->m_md[1], ops.Bh = g->m_md[0], ops.Bl = g->m_md[1];
    GemmArgs ga{};
    ga.num_kb = d / 64;
    ga.M = R, ga.N = R;
    ga.Ah = g->mdh, ga.Al = g->mdl, ga.Bh = g->mdh, ga.Bl = g->mdl;
    ga.lda = d, ga.ldb = d;
    DIMB_TRY((launch_gemm<128, false>(ctx, st, ops, ga, e, NPt / kTileM, NPt, "sg.scores")));
    e.sim = g->simT;  // the same products with the operand roles swapped: scores^T, so that the column sweeps of Sinkhorn read rows
    e.swap = 1;
    DIMB_TRY((launch_gemm<128, false>(ctx, st, ops, ga, e, NPt / kTileM, NPt, "sg.scores")));
  }
  return DIMB_OK;
}

}  // namespace

extern "C" {

size_t dimb_sg_weight_count(int n_layers) {
  const size_t d = kSgD;
  size_t n = 0;
  const int ch[6] = {3, 32, 64, 128, 256, 256};
  for (int i = 0; i < 5; ++i) n += static_cast<size_t>(ch[i + 1]) * ch[i] + ch[i + 1] + (i < 4 ? 4 * ch[i + 1] : 0);
  n += static_cast<size_t>(n_layers) * (4 * (d * d + d) + (2 * d * 2 * d + 2 * d) + 4 * 2 * d + (d * 2 * d + d));
  return n + d * d + d + 1;
}

int dimb_sg_create(dimb_ctx* ctx, const float* weights, size_t n_floats, const dimb_sg_conf* conf, dimb_sg** out) {
  if (!ctx || !weights || !conf || !out) return DIMB_ERR_ARG;
  *out = nullptr;
  if (conf->n_layers < 1 || conf->n_layers > 64 || conf->max_kpts < 1 || conf->sinkhorn_iterations < 0) return DIMB_ERR_ARG;
  if (n_floats != dimb_sg_weight_count(conf->n_layers)) {
    dimb_set_error(ctx, "dimb_sg_create: weight blob has " + std::to_string(n_floats) + " floats, expected " +
                            std::to_string(dimb_sg_weight_count(conf->n_layers)));
    return DIMB_ERR_ARG;
  }
  DIMB_CUDA_OK(ctx, cudaSetDevice(ctx->device));
  dimb_sg* g = new dimb_sg();
  g->ctx = ctx;
  std::unique_ptr<dimb_sg, void (*)(dimb_sg*)> guard(g, dimb_sg_destroy);
  OwnerScope own(ctx, &g->mem);
  g->conf = *conf;
  g->L = conf->n_layers;
  g->NP = conf->max_kpts;
  for (int i = 0; i < g->L; ++i) g->cross.push_back((conf->cross_mask >> i) & 1ull ? 1 : 0);
  const float* p = weights;
  const int ch[6] = {3, 32, 64, 128, 256, 256};
  for (int i = 0; i < 5; ++i) {
    HostLin l = take_conv(p, ch[i + 1], ch[i]);
    if (i < 4) fold_bn(l, p);
    DIMB_TRY(upload(ctx, g->kenc[i], l));
  }
  g->layers.resize(g->L);
  g->tc.resize(g->L);
  for (int i = 0; i < g->L; ++i) {  // state_dict order: attn.merge, attn.proj.0/1/2, mlp.0, mlp.1 (BN), mlp.3
    HostLin merge = take_conv(p, kSgD, kSgD), q = take_conv(p, kSgD, kSgD), k = take_conv(p, kSgD, kSgD), v = take_conv(p, kSgD, kSgD);
    HostLin m0 = take_conv(p, 2 * kSgD, 2 * kSgD);
    fold_bn(m0, p);
    HostLin m3 = take_conv(p, kSgD, 2 * kSgD);
    permute_rows(q), permute_rows(k), permute_rows(v), permute_cols(merge);
    {
      HostLin qkv = q;
      qkv.n = 3 * kSgD;
      qkv.w.insert(qkv.w.end(), k.w.begin(), k.w.end());
      qkv.w.insert(qkv.w.end(), v.w.begin(), v.w.end());
      qkv.b.insert(qkv.b.end(), k.b.begin(), k.b.end());
      qkv.b.insert(qkv.b.end(), v.b.begin(), v.b.end());
      SgTcLayer& t = g->tc[i];
      DIMB_TRY(upload_tc(ctx, t.qkv, qkv));
      DIMB_TRY(upload_tc(ctx, t.merge, merge));
      DIMB_TRY(upload_tc(ctx, t.mlp0, m0));
      DIMB_TRY(upload_tc(ctx, t.mlp3, m3));
    }
    SgLayer& ly = g->layers[i];
    DIMB_TRY(upload(ctx, ly.q, q));
    DIMB_TRY(upload(ctx, ly.k, k));
    DIMB_TRY(upload(ctx, ly.v, v));
    DIMB_TRY(upload(ctx, ly.merge, merge));
    DIMB_TRY(upload(ctx, ly.mlp0, m0));
    DIMB_TRY(upload(ctx, ly.mlp3, m3));
  }
  {
    HostLin fp = take_conv(p, kSgD, kSgD);
    DIMB_TRY(upload(ctx, g->final_proj, fp));
    DIMB_TRY(upload_tc(ctx, g->tc_final, fp));
  }
  DIMB_TRY(dimb_alloc_t(ctx, &g->bin_score, 1, false));
  DIMB_CUDA_OK(ctx, cudaMemcpy(g->bin_score, p, sizeof(float), cudaMemcpyHostToDevice));
  const size_t NP = g->NP;
  for (int s = 0; s < 2; ++s) {
    DIMB_TRY(dimb_alloc_t(ctx, &g->cat[s], NP * 2 * kSgD));
    DIMB_TRY(dimb_alloc_t(ctx, &g->q[s], NP * kSgD));
    DIMB_TRY(dimb_alloc_t(ctx, &g->k[s], NP * kSgD));
    DIMB_TRY(dimb_alloc_t(ctx, &g->v[s], NP * kSgD));
    DIMB_TRY(dimb_alloc_t(ctx, &g->md[s], NP * kSgD));
  }
  DIMB_TRY(dimb_alloc_t(ctx, &g->att, NP * kSgD));
  DIMB_TRY(dimb_alloc_t(ctx, &g->hid, NP * 2 * kSgD));
  DIMB_TRY(dimb_alloc_t(ctx, &g->enc_a, NP * kSgD));
  DIMB_TRY(dimb_alloc_t(ctx, &g->enc_b, NP * kSgD));
  DIMB_TRY(dimb_alloc_t(ctx, &g->Z, (NP + 1) * (NP + 1)));
  DIMB_TRY(dimb_alloc_t(ctx, &g->u, NP + 1));
  DIMB_TRY(dimb_alloc_t(ctx, &g->vv, NP + 1));
  DIMB_TRY(dimb_alloc_t(ctx, &g->best0, NP));
  DIMB_TRY(dimb_alloc_t(ctx, &g->best1, NP));
  DIMB_TRY(dimb_alloc_t(ctx, &g->arg0, NP));
  DIMB_TRY(dimb_alloc_t(ctx, &g->arg1, NP));
  {  // tensor-core path state
    const size_t NPt = round_up(g->NP, 128), R = 2 * NPt, d = kSgD;
    g->NPt = static_cast<int>(NPt);
    DIMB_TRY(dimb_alloc_t(ctx, &g->x32, R * d));
    DIMB_TRY(dimb_alloc_t(ctx, &g->xh, R * 2 * d));
    DIMB_TRY(dimb_alloc_t(ctx, &g->xl, R * 2 * d));
    DIMB_TRY(dimb_alloc_t(ctx, &g->h2h, R * 2 * d));
    DIMB_TRY(dimb_alloc_t(ctx, &g->h2l, R * 2 * d));
    for (__half** b : {&g->qh, &g->ql, &g->kh, &g->kl, &g->vth, &g->vtl, &g->ctxh, &g->ctxl, &g->mdh, &g->mdl}) DIMB_TRY(dimb_alloc_t(ctx, b, R * d));
    DIMB_TRY(dimb_alloc_t(ctx, &g->sim, NPt * NPt));
    DIMB_TRY(dimb_alloc_t(ctx, &g->simT, NPt * NPt));
    DIMB_TRY(dimb_alloc_t(ctx, &g->n_act, 2));
    DIMB_TRY(dimb_alloc_t(ctx, &g->stopped, 1));
    DIMB_TRY(dimb_tmap_2d(ctx, &g->m_x[0], g->xh, R, 2 * d, 2 * d, kTileM));
    DIMB_TRY(dimb_tmap_2d(ctx, &g->m_x[1], g->xl, R, 2 * d, 2 * d, kTileM));
    DIMB_TRY(dimb_tmap_2d(ctx, &g->m_h2[0], g->h2h, R, 2 * d, 2 * d, kTileM));
    DIMB_TRY(dimb_tmap_2d(ctx, &g->m_h2[1], g->h2l, R, 2 * d, 2 * d, kTileM));
    DIMB_TRY(dimb_tmap_2d(ctx, &g->m_ctx[0], g->ctxh, R, d, d, kTileM));
    DIMB_TRY(dimb_tmap_2d(ctx, &g->m_ctx[1], g->ctxl, R, d, d, kTileM));
    DIMB_TRY(dimb_tmap_2d(ctx, &g->m_md[0], g->mdh, R, d, d, kTileM));
    DIMB_TRY(dimb_tmap_2d(ctx, &g->m_md[1], g->mdl, R, d, d, kTileM));
    DIMB_TRY(dimb_tmap_2d(ctx, &g->m_q128[0], g->qh, 2 * kHeads * NPt, kHd, kHd, kTileM));
    DIMB_TRY(dimb_tmap_2d(ctx, &g->m_q128[1], g->ql, 2 * kHeads * NPt, kHd, kHd, kTileM));
    DIMB_TRY(dimb_tmap_2d(ctx, &g->m_k64[0], g->kh, 2 * kHeads * NPt, kHd, kHd, kBlkK));
    DIMB_TRY(dimb_tmap_2d(ctx, &g->m_k64[1], g->kl, 2 * kHeads * NPt, kHd, kHd, kBlkK));
    DIMB_TRY(dimb_tmap_2d(ctx, &g->m_vt[0], g->vth, 2 * kHeads * kHd, NPt, NPt, kHd));
    DIMB_TRY(dimb_tmap_2d(ctx, &g->m_vt[1], g->vtl, 2 * kHeads * kHd, NPt, NPt, kHd));
  }
  *out = guard.release();
  return DIMB_OK;
}

void dimb_sg_destroy(dimb_sg* g) {
  if (!g) return;
  dimb_release(g->ctx, g->mem);
  delete g;
}

// One pair.  Outputs (host): matches [cap][2] int64 ascending in column 0 (correspondence_matrix_from_matches0, superglue.py:44-52),
// mscores [cap] (matching_scores0 of the matched rows), n_matches.
int dimb_sg_match(dimb_sg* g, const dimb_sg_feats* f0, const dimb_sg_feats* f1, int64_t* matches, float* mscores, int* n_matches, int cap) {
  if (!g || !f0 || !f1 || !matches || !mscores || !n_matches || cap < 1) return DIMB_ERR_ARG;
  dimb_ctx* ctx = g->ctx;
  OwnerScope own(ctx, &g->mem);
  DIMB_CUDA_OK(ctx, cudaSetDevice(ctx->device));
  cudaStream_t st = 0;
  const dimb_sg_feats* F[2] = {f0, f1};
  const int n[2] = {f0->n, f1->n}, NP = g->NP, d = kSgD;
  *n_matches = 0;
  if (n[0] > NP || n[1] > NP || n[0] < 0 || n[1] < 0) {
    dimb_set_error(ctx, "dimb_sg_match: more keypoints than max_kpts");
    return DIMB_ERR_ARG;
  }
  if (n[0] == 0 || n[1] == 0) return DIMB_OK;  // "no keypoints" return of the reference (superglue.py:248-256): everything unmatched
  for (int s = 0; s < 2; ++s) {
    const dimb_sg_feats& f = *F[s];
    // descriptors arrive (D,N) like the FeaturesDict: copied as they are, transposed to token-major on the device together with the
    // keypoint encoder's input (normalised x, normalised y, score)
    const float cx = static_cast<float>(f.width) / 2.f, cy = static_cast<float>(f.height) / 2.f;
    const float sc = static_cast<float>(std::max(f.width, f.height)) * 0.7f;
    const int ld = f.desc_ld ? f.desc_ld : f.n;
    float* st_desc = g->hid;  // staging: [256][n] fits the [NP][512] hidden buffer; keypoints / scores behind it
    float* st_kp = g->att;
    DIMB_CUDA_OK(ctx, cudaMemcpy2DAsync(st_desc, static_cast<size_t>(n[s]) * sizeof(float), f.descriptors, static_cast<size_t>(ld) * sizeof(float),
                                        static_cast<size_t>(n[s]) * sizeof(float), d, cudaMemcpyHostToDevice, st));
    DIMB_CUDA_OK(ctx, cudaMemcpyAsync(st_kp, f.keypoints, static_cast<size_t>(n[s]) * 2 * sizeof(float), cudaMemcpyHostToDevice, st));
    DIMB_CUDA_OK(ctx, cudaMemcpyAsync(st_kp + 2 * static_cast<size_t>(NP), f.scores, static_cast<size_t>(n[s]) * sizeof(float), cudaMemcpyHostToDevice, st));
    sg_input_kernel<<<dim3(ceil_div(n[s], 32), d / 32), dim3(32, 8), 0, st>>>(st_desc, n[s], n[s], st_kp, st_kp + 2 * static_cast<size_t>(NP), cx, cy, sc,
                                                                              g->cat[s], 2 * d, g->enc_a);
    DIMB_LAUNCH_CHECK(ctx);
    float *a = g->enc_a, *b = g->enc_b;
    int lda = 3;
    for (int i = 0; i < 5; ++i) {
      if (i < 4) {
        DIMB_TRY(sg_linear(g, st, a, lda, g->kenc[i], b, g->kenc[i].n, n[s], 1));
        std::swap(a, b);
        lda = g->kenc[i].n;
      } else {  // last layer: no BN / ReLU; desc = desc + kenc(...)
        DIMB_TRY(sg_linear(g, st, a, lda, g->kenc[i], g->cat[s], 2 * d, n[s], 0, 1.f, g->cat[s], 2 * d));
      }
    }
    // enc_a / enc_b and the staging buffers are reused by the other side: stream order is enough
  }
  const int m = n[0], nn = n[1];
  const float norm = -std::log(static_cast<float>(m) + static_cast<float>(nn));
  const float* Zs = g->Z;   // score block of the couplings and its row pitch (tensor path: the similarity buffer, virtual dustbins)
  int ld = nn + 1;
  if (ctx->use_tc) {
    DIMB_TRY(sg_gnn_tc(g, st, n));
    Zs = g->sim;
    ld = g->NPt;
    DIMB_CUDA_OK(ctx, cudaMemsetAsync(g->u, 0, (m + 1) * sizeof(float), st));
    DIMB_CUDA_OK(ctx, cudaMemsetAsync(g->vv, 0, (nn + 1) * sizeof(float), st));
    for (int it = 0; it < g->conf.sinkhorn_iterations; ++it) {
      sg_sink_rows_kernel<<<ceil_div((m + 1) * 32, 256), 256, 0, st>>>(Zs, ld, m, nn, g->bin_score, g->vv, g->u, norm, std::log(static_cast<float>(nn)));
      DIMB_LAUNCH_CHECK(ctx);
      // column sweep = row sweep over the transposed block (coalesced, one warp per column)
      sg_sink_rows_kernel<<<ceil_div((nn + 1) * 32, 256), 256, 0, st>>>(g->simT, ld, nn, m, g->bin_score, g->u, g->vv, norm, std::log(static_cast<float>(m)));
      DIMB_LAUNCH_CHECK(ctx);
    }
  } else {
  for (int i = 0; i < g->L; ++i) {  // AttentionalGNN (:132-152): deltas of both sides from the OLD descriptors
    const SgLayer& ly = g->layers[i];
    for (int s = 0; s < 2; ++s) {
      const int src = g->cross[i] ? 1 - s : s;
      DIMB_TRY(sg_linear(g, st, g->cat[s], 2 * d, ly.q, g->q[s], d, n[s], 0));
      DIMB_TRY(sg_linear(g, st, g->cat[src], 2 * d, ly.k, g->k[s], d, n[src], 0));
      DIMB_TRY(sg_linear(g, st, g->cat[src], 2 * d, ly.v, g->v[s], d, n[src], 0));
    }
    for (int s = 0; s < 2; ++s) {
      const int src = g->cross[i] ? 1 - s : s;
      dim3 grid(ceil_div(n[s], 8), kSgHeads);
      gx_attention_kernel<64><<<grid, 256, 0, st>>>(g->q[s], g->k[s], g->v[s], n[s], n[src], d, kSgHd, g->att, d);
      DIMB_LAUNCH_CHECK(ctx);
      DIMB_TRY(sg_linear(g, st, g->att, d, ly.merge, g->cat[s] + d, 2 * d, n[s], 0));  // message -> right half of [x | message]
    }
    for (int s = 0; s < 2; ++s) {  // x += mlp([x | message])
      DIMB_TRY(sg_linear(g, st, g->cat[s], 2 * d, ly.mlp0, g->hid, 2 * d, n[s], 1));
      DIMB_TRY(sg_linear(g, st, g->hid, 2 * d, ly.mlp3, g->cat[s], 2 * d, n[s], 0, 1.f, g->cat[s], 2 * d));
    }
  }
  for (int s = 0; s < 2; ++s) DIMB_TRY(sg_linear(g, st, g->cat[s], 2 * d, g->final_proj, g->md[s], d, n[s], 0));
  {  // scores = mdesc0 . mdesc1^T / sqrt(256) into the top-left block of the couplings
    dim3 grid(ceil_div(nn, 64), ceil_div(m, 64));
    gx_linear_kernel<<<grid, 256, 0, st>>>(g->md[0], d, g->md[1], d, nullptr, g->Z, ld, m, nn, d, 1.f / 16.f, nullptr, 0, 0);
    DIMB_LAUNCH_CHECK(ctx);
  }
  sg_fill_bins_kernel<<<ceil_div(std::max(m, nn) + 1, 256), 256, 0, st>>>(g->Z, ld, m, nn, g->bin_score);
  DIMB_LAUNCH_CHECK(ctx);
  DIMB_CUDA_OK(ctx, cudaMemsetAsync(g->u, 0, (m + 1) * sizeof(float), st));
  DIMB_CUDA_OK(ctx, cudaMemsetAsync(g->vv, 0, (nn + 1) * sizeof(float), st));
  for (int it = 0; it < g->conf.sinkhorn_iterations; ++it) {
    sg_sinkhorn_kernel<<<ceil_div((m + 1) * 32, 256), 256, 0, st>>>(g->Z, ld, m + 1, nn + 1, 0, g->vv, g->u, norm, std::log(static_cast<float>(nn)));
    DIMB_LAUNCH_CHECK(ctx);
    sg_sinkhorn_kernel<<<ceil_div((nn + 1) * 32, 256), 256, 0, st>>>(g->Z, ld, m + 1, nn + 1, 1, g->u, g->vv, norm, std::log(static_cast<float>(m)));
    DIMB_LAUNCH_CHECK(ctx);
  }
  }  // plain fp32 twin
  sg_argmax_kernel<<<ceil_div(m * 32, 256), 256, 0, st>>>(Zs, ld, m, nn, g->u, g->vv, norm, 0, g->best0, g->arg0);
  DIMB_LAUNCH_CHECK(ctx);
  sg_argmax_kernel<<<ceil_div(nn * 32, 256), 256, 0, st>>>(Zs, ld, m, nn, g->u, g->vv, norm, 1, g->best1, g->arg1);
  DIMB_LAUNCH_CHECK(ctx);
  std::vector<float> b0(m);
  std::vector<int> a0(m), a1(nn);
  DIMB_CUDA_OK(ctx, cudaMemcpyAsync(b0.data(), g->best0, m * sizeof(float), cudaMemcpyDeviceToHost, st));
  DIMB_CUDA_OK(ctx, cudaMemcpyAsync(a0.data(), g->arg0, m * sizeof(int), cudaMemcpyDeviceToHost, st));
  DIMB_CUDA_OK(ctx, cudaMemcpyAsync(a1.data(), g->arg1, nn * sizeof(int), cudaMemcpyDeviceToHost, st));
  DIMB_CUDA_OK(ctx, cudaStreamSynchronize(st));
  int cnt = 0;
  for (int r = 0; r < m; ++r) {
    const int c = a0[r];
    if (a1[c] != r) continue;  // mutual
    const float e = std::exp(b0[r]);
    if (!(e > g->conf.match_threshold)) continue;
    if (cnt < cap) {
      matches[2 * cnt] = r;
      matches[2 * cnt + 1] = c;
      mscores[cnt] = e;
    }
    ++cnt;
  }
  *n_matches = cnt;
  if (cnt > cap) {
    dimb_set_error(ctx, "dimb_sg_match: more matches than cap");
    return DIMB_ERR_CAPACITY;
  }
  return DIMB_OK;
}

}  // extern "C"
