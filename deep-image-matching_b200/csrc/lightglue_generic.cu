// lightglue_generic.cu - LightGlue for shapes other than (descriptor_dim 256, 4 heads x 64), i.e. the LighterGlue
// checkpoint the reference ships (thirdparty/accelerated_features/modules/lighterglue.py:12-27: descriptor_dim 96,
// one head, 6 layers, input_dim 64; matcher plugin src/deep_image_matching/matchers/lighterglue.py:78-262).
// Same algorithm as lightglue.cu (thirdparty/LightGlue/lightglue/lightglue.py:24-610) in plain fp32 on the CUDA cores, with the
// attention on the tensor cores for head dims 65..128 (attn_hd128.cuh): the tensor-core kernels of lightglue.cu are specialised for
// head dim 64 / model dim 256 (registers and shared-memory budgets of the attention kernel), this file trades speed for generality.
//
// lgx_match_dev (dimb_lg_match_dev for these shapes; dimb_lg_match stages host pairs into it) runs P pairs at once: the 2P sides share
// one set of token buffers (side s owns rows [s*NP, (s+1)*NP)), every layer's linears, rotary, attention, LayerNorm/GELU and row dots
// run as one launch over all sides, and the live counts, stop layers and pruning maps stay on the device.  The confidence and
// matchability sigmoids and the match scores use glibc_expf (lgx_assign.cuh), glibc's expf on the device.
#include <algorithm>
#include <memory>
#include <cmath>
#include <vector>

#include "generic_kernels.cuh"
#include "attn_hd128.cuh"
#include "lgx_assign.cuh"
#include "lightglue_generic.cuh"

namespace {

struct Lin {
  float *w = nullptr, *b = nullptr;
  int n = 0, k = 0;
};
struct Block {
  Lin qkv, to_qk, to_v, out, ffn0, ffn3;
  float *ln_g = nullptr, *ln_b = nullptr;
};

}  // namespace

// buffers for conf.max_pairs pairs (S = 2 max_pairs sides of NP = max_kpts rows)
struct dimb_lgx {
  dimb_ctx* ctx;
  std::vector<void*> mem;
  dimb_lg_conf conf;
  int d, h, hd, din, L, NP;
  float* Wr;
  Lin input_proj;
  std::vector<Block> self_, cross_;
  std::vector<Lin> matchab, final_proj, token;
  float *cat[2], *enc[2], *kp, *qkv, *q, *k, *v, *hid, *hid2, *xf, *md, *zt, *zm, *sim, *rlse, *clse, *best;
  int *ind[2], *nact[2], *n_orig, *stopped, *idx, *indf, *nf, *layer, *parity, *arg;
  void* in;                               // SideInX [S]
  const float** tab;                      // [4][L]: final_proj w, b, matchability w, b (the final stage picks a pair's layer)
  // head dims 65..128 (LighterGlue: 96): attention on the tensor cores; other head dims run lgx_attention_kernel
  bool tc_attn = false;
  Hd128Ops tc;
};

namespace {

float conf_threshold(int i, int L) {  // lightglue.py:581-584
  return static_cast<float>(std::min(std::max(0.8 + 0.1 * std::exp(-4.0 * i / L), 0.0), 1.0));
}

struct SideInX {  // one side's dimb_feats_dev as the kernels read it
  const void* kpts;
  const void* desc;
  const int* n;
  int n_cap, layout, ld;
  float size0, size1;
  int round_fp16, f16;
  const int* size_dev;
  const float* size_f32;
};

__device__ __forceinline__ float feat_at(const void* p, size_t i, int f16, int r16) {
  const float v = f16 ? __half2float(static_cast<const __half*>(p)[i]) : static_cast<const float*>(p)[i];
  return r16 ? __half2float(__float2half_rn(v)) : v;
}
__device__ __forceinline__ int side_rows(const SideInX& si, int NP) { return min(min(*si.n, si.n_cap), NP); }

// grid (ceil(NP / 32), S), block (32, 8): descriptors -> x rows [S][NP][ldx] (fp32, transposed from (D,n)), keypoints -> kp [S][NP][2],
// identity original indices, live counts; a pair with an empty side is stopped at once (stop 1, no matches: lightglue.py:518-538)
__global__ void lgx_prep_kernel(const SideInX* __restrict__ in, int din, int NP, float* __restrict__ x, int ldx, float* __restrict__ kp,
                                int* __restrict__ ind, int* __restrict__ nact, int* __restrict__ n_orig, int* __restrict__ stopped) {
  const int side = blockIdx.y, t0 = blockIdx.x * 32, tx = threadIdx.x, ty = threadIdx.y;
  const SideInX si = in[side];
  const int n = side_rows(si, NP);
  if (blockIdx.x == 0 && tx == 0 && ty == 0) {
    nact[side] = n;
    n_orig[side] = n;
    if ((side & 1) == 0) stopped[side >> 1] = (n == 0 || side_rows(in[side + 1], NP) == 0) ? 1 : 0;
  }
  if (t0 >= n) return;
  __shared__ float tile[32][33];
  for (int c0 = 0; c0 < din; c0 += 32) {
    for (int k = ty; k < 32; k += 8) {
      if (si.layout == 0) {  // desc[c][tok], coalesced over tok
        const int c = c0 + k, tok = t0 + tx;
        tile[k][tx] = (tok < n && c < din) ? feat_at(si.desc, static_cast<size_t>(c) * si.ld + tok, si.f16, si.round_fp16) : 0.f;
      } else {  // desc[tok][c], coalesced over c
        const int tok = t0 + k, c = c0 + tx;
        tile[tx][k] = (tok < n && c < din) ? feat_at(si.desc, static_cast<size_t>(tok) * si.ld + c, si.f16, si.round_fp16) : 0.f;
      }
    }
    __syncthreads();
    for (int k = ty; k < 32; k += 8) {
      const int tok = t0 + k, c = c0 + tx;
      if (tok < n && c < din) x[(static_cast<size_t>(side) * NP + tok) * ldx + c] = tile[tx][k];
    }
    __syncthreads();
  }
  for (int k = ty; k < 32; k += 8) {
    const int tok = t0 + k;
    if (tok >= n || tx >= 2) continue;
    const size_t row = static_cast<size_t>(side) * NP + tok;
    kp[row * 2 + tx] = feat_at(si.kpts, 2 * static_cast<size_t>(tok) + tx, si.f16, si.round_fp16);
    if (tx == 0) ind[row] = tok;
  }
}

// block (1024) per side: the normalisation size (given, or the keypoints' own extent (1 + max) - min, as dimb_lg_match's
// staging computes it on the host) and the positional encoding of every live row
__global__ void __launch_bounds__(1024) lgx_posenc_kernel(const SideInX* __restrict__ in, const float* __restrict__ kp, const int* __restrict__ nact,
                                                          int NP, const float* __restrict__ Wr, int hd, float* __restrict__ enc) {
  const int side = blockIdx.x, n = nact[side];
  if (n == 0) return;
  const SideInX si = in[side];
  const float* k = kp + static_cast<size_t>(side) * NP * 2;
  float s0 = si.size0, s1 = si.size1;
  if (si.size_f32) {
    s0 = si.size_f32[0], s1 = si.size_f32[1];
  } else if (si.size_dev) {
    s0 = static_cast<float>(si.size_dev[0]), s1 = static_cast<float>(si.size_dev[1]);
  } else if (s0 == 0.f && s1 == 0.f) {
    __shared__ float red[4][32];
    float v[4] = {INFINITY, INFINITY, -INFINITY, -INFINITY};  // min x, min y, max x, max y
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
      v[0] = fminf(v[0], k[2 * i]), v[1] = fminf(v[1], k[2 * i + 1]);
      v[2] = fmaxf(v[2], k[2 * i]), v[3] = fmaxf(v[3], k[2 * i + 1]);
    }
#pragma unroll
    for (int of = 16; of; of >>= 1)
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float o = __shfl_xor_sync(0xffffffffu, v[j], of);
        v[j] = j < 2 ? fminf(v[j], o) : fmaxf(v[j], o);
      }
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
    if (lane == 0)
      for (int j = 0; j < 4; ++j) red[j][w] = v[j];
    __syncthreads();
    for (int j = 0; j < 4; ++j) {
      float r = red[j][0];
      for (int q = 1; q < nw; ++q) r = j < 2 ? fminf(r, red[j][q]) : fmaxf(r, red[j][q]);
      v[j] = r;
    }
    s0 = __fsub_rn(__fadd_rn(1.f, v[2]), v[0]), s1 = __fsub_rn(__fadd_rn(1.f, v[3]), v[1]);
  }
  const int nf = hd / 2;
  float* e = enc + static_cast<size_t>(side) * 2 * NP * hd;
  for (int t = threadIdx.x; t < n * nf; t += blockDim.x) gx_posenc_one(k, t / nf, t % nf, s0, s1, Wr, hd, e, NP);
}

// C rows of every side = A rows . W^T (+ bias, * scale, + resid); grid (ceil(N / 64), ceil(NP / 64), S).  gate: only the live rows of
// running pairs, else all nact rows.  wtab / btab (per layer) + layer (per pair): the weights of the layer each pair ended at.
__global__ void __launch_bounds__(256) lgx_linear_kernel(const float* __restrict__ A, int lda, size_t sA, const float* __restrict__ W,
                                                         const float* __restrict__ bias, float* __restrict__ C, int ldc, size_t sC, int N, int K,
                                                         float scale, const float* __restrict__ resid, const int* __restrict__ nact,
                                                         const int* __restrict__ stopped, int gate, const float* const* __restrict__ wtab,
                                                         const float* const* __restrict__ btab, const int* __restrict__ layer) {
  const int side = blockIdx.z, m0 = blockIdx.y * 64;
  const int M = gate ? live_rows(nact, stopped, side) : nact[side];
  if (m0 >= M) return;
  if (wtab) W = wtab[layer[side >> 1]], bias = btab[layer[side >> 1]];
  gx_linear_tile(A + side * sA, lda, W, K, bias, C + side * sC, ldc, M, N, K, scale, resid ? resid + side * sC : nullptr, ldc, 0, m0);
}

// z[side][row] = x[side][row] . w + b over the rows of every side; warp per row (wtab / btab / layer as lgx_linear_kernel)
__global__ void lgx_rowdot_kernel(const float* __restrict__ x, int ldx, int n, int NP, const float* __restrict__ w, const float* __restrict__ b,
                                  float* __restrict__ z, const int* __restrict__ nact, const int* __restrict__ stopped, int gate,
                                  const float* const* __restrict__ wtab, const float* const* __restrict__ btab, const int* __restrict__ layer,
                                  int S) {
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  const int side = row / NP, j = row - side * NP;
  if (side >= S || j >= (gate ? live_rows(nact, stopped, side) : nact[side])) return;
  if (wtab) w = wtab[layer[side >> 1]], b = btab[layer[side >> 1]];
  gx_rowdot_row(x + static_cast<size_t>(side) * NP * ldx, ldx, j, lane, n, w, b, z + static_cast<size_t>(side) * NP);
}

// grid (NP, S), block max(32, d / 2)
__global__ void lgx_qkv_rotary_kernel(const float* __restrict__ qkv, int d, int hd, const float* __restrict__ enc, int NP, float* __restrict__ q,
                                      float* __restrict__ k, float* __restrict__ v, const int* __restrict__ nact, const int* __restrict__ stopped) {
  const int side = blockIdx.y, i = blockIdx.x, c = threadIdx.x * 2;
  if (i >= live_rows(nact, stopped, side) || c >= d) return;
  const size_t o = static_cast<size_t>(side) * NP * d;
  gx_qkv_rotary_one(qkv + 3 * o, i, c, d, hd, enc + static_cast<size_t>(side) * 2 * NP * hd, NP, q + o, k + o, v + o);
}

// grid (ceil(NP / 8), h, S): side s attends to its own keys (self) or to those of its partner s ^ 1 (cross)
template <int HDP>
__global__ void __launch_bounds__(256) lgx_attention_kernel(const float* __restrict__ q, const float* __restrict__ k, const float* __restrict__ v,
                                                            int NP, int d, int hd, int cross, float* __restrict__ out, const int* __restrict__ nact,
                                                            const int* __restrict__ stopped) {
  const int side = blockIdx.z, ks = cross ? side ^ 1 : side;
  const int nq = live_rows(nact, stopped, side);
  if (static_cast<int>(blockIdx.x) * 8 >= nq) return;
  const size_t so = static_cast<size_t>(side) * NP * d, ko = static_cast<size_t>(ks) * NP * d;
  gx_attention_block<HDP>(q + so, k + ko, v + ko, nq, nact[ks], d, hd, out + so, d, blockIdx.x, blockIdx.y);
}

__global__ void lgx_ln_gelu_kernel(const float* __restrict__ x, int n, int NP, const float* __restrict__ g, const float* __restrict__ b,
                                   float* __restrict__ y, const int* __restrict__ nact, const int* __restrict__ stopped, int S) {
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  const int side = row / NP, j = row - side * NP;
  if (side >= S || j >= live_rows(nact, stopped, side)) return;
  gx_ln_gelu_row(x, row, lane, n, g, b, y);
}

// block (1024) per running pair, after layer i < L - 1: token confidences, the stop test (lightglue.py:593-604), and per side the
// pruning mask (:586-591) compacted in row order into idx (ballot + block prefix; identity when the side is not pruned).  A pair that
// stops keeps stopped = i + 1; one that prunes a side to nothing stops as the reference's next layer would, at min(i + 1, L - 1) + 1.
__global__ void __launch_bounds__(1024) lgx_decide_kernel(int i, int L, int NP, const float* __restrict__ ztok, const float* __restrict__ zmat,
                                                          const int* __restrict__ nact, int* __restrict__ nnext, const int* __restrict__ n_orig,
                                                          int* __restrict__ stopped, int* __restrict__ idx, float thr, float depth_conf,
                                                          float keep_thr, int do_stop, int do_prune, int prune_min) {
  const int p = blockIdx.x, tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  if (stopped[p]) return;
  __shared__ int below, wsum[32], total;
  if (do_stop) {
    if (tid == 0) below = 0;
    __syncthreads();
    int cnt = 0;
    for (int sd = 0; sd < 2; ++sd) {
      const int s = 2 * p + sd;
      for (int j = tid; j < nact[s]; j += blockDim.x) cnt += host_sigmoid(ztok[static_cast<size_t>(s) * NP + j]) < thr;
    }
    atomicAdd(&below, cnt);
    __syncthreads();
    const float ratio = __fsub_rn(1.0f, __fdiv_rn(static_cast<float>(below), static_cast<float>(n_orig[2 * p] + n_orig[2 * p + 1])));
    if (ratio > depth_conf) {
      if (tid == 0) stopped[p] = i + 1;
      return;
    }
  }
  int empty = 0;
  for (int sd = 0; sd < 2; ++sd) {
    const int s = 2 * p + sd, n = nact[s];
    const size_t o = static_cast<size_t>(s) * NP;
    const bool prune = do_prune && n > prune_min;
    int base = 0;
    for (int j0 = 0; j0 < n; j0 += blockDim.x) {
      const int j = j0 + tid;
      bool keep = j < n;
      if (keep && prune) {
        keep = host_sigmoid(zmat[o + j]) > keep_thr;
        if (do_stop) keep = keep || host_sigmoid(ztok[o + j]) <= thr;
      }
      const unsigned bal = __ballot_sync(0xffffffffu, keep);
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
      if (keep) idx[o + base + wsum[w] + __popc(bal & ((1u << lane) - 1u))] = j;
      base += total;
      __syncthreads();
    }
    if (tid == 0) nnext[s] = base;
    empty |= base == 0;
  }
  if (tid == 0 && empty) stopped[p] = min(i + 1, L - 1) + 1;
}

// grid (NP, S), block 128: the rows kept by lgx_decide_kernel into the other ping-pong buffer (state x, both encoding halves, original
// index), for the pairs still running after layer i and those that have just pruned a side to nothing
__global__ void lgx_gather_kernel(int i, const int* __restrict__ stopped, const int* __restrict__ nnext, const int* __restrict__ idx, int NP,
                                  int d, int hd, const float* __restrict__ xs, float* __restrict__ xd, const float* __restrict__ es,
                                  float* __restrict__ ed, const int* __restrict__ is, int* __restrict__ id) {
  const int side = blockIdx.y, j = blockIdx.x, st = stopped[side >> 1];
  if ((st != 0 && st <= i + 1) || j >= nnext[side]) return;
  const size_t base = static_cast<size_t>(side) * NP, src = base + idx[base + j], dst = base + j;
  for (int c = threadIdx.x; c < d; c += blockDim.x) xd[dst * 2 * d + c] = xs[src * 2 * d + c];
  const size_t eb = static_cast<size_t>(side) * 2 * NP * hd;
  const size_t es0 = eb + (src - base) * hd, ed0 = eb + static_cast<size_t>(j) * hd, half = static_cast<size_t>(NP) * hd;
  for (int c = threadIdx.x; c < hd; c += blockDim.x) {
    ed[ed0 + c] = es[es0 + c];
    ed[ed0 + half + c] = es[es0 + half + c];
  }
  if (threadIdx.x == 0) id[dst] = is[src];
}

// thread per pair: the layer a pair ended at (its stop layer, or the last) and the ping-pong buffer holding its state
__global__ void lgx_final_select_kernel(const int* __restrict__ stopped, const int* __restrict__ nact0, const int* __restrict__ nact1,
                                        int* __restrict__ nf, int* __restrict__ layer, int* __restrict__ parity, int P, int L, int adaptive) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  const int st = stopped[p];
  const int par = adaptive ? ((st ? st - 1 : L - 1) & 1) : 0;
  parity[p] = par;
  layer[p] = st ? st - 1 : L - 1;
  const int* na = par ? nact1 : nact0;
  nf[2 * p] = na[2 * p];
  nf[2 * p + 1] = na[2 * p + 1];
}

// grid (NP, S), block 128: the final state x and original indices of every side into fixed buffers
__global__ void lgx_final_gather_kernel(const int* __restrict__ nf, const int* __restrict__ parity, int NP, int d, const float* __restrict__ x0,
                                        const float* __restrict__ x1, const int* __restrict__ i0, const int* __restrict__ i1, float* __restrict__ xf,
                                        int* __restrict__ indf) {
  const int side = blockIdx.y, j = blockIdx.x;
  if (j >= nf[side]) return;
  const int par = parity[side >> 1];
  const size_t row = static_cast<size_t>(side) * NP + j;
  const float* x = (par ? x1 : x0) + row * 2 * d;
  for (int c = threadIdx.x; c < d; c += blockDim.x) xf[row * d + c] = x[c];
  if (threadIdx.x == 0) indf[row] = (par ? i1 : i0)[row];
}

// grid (ceil(NP / 64), ceil(NP / 64), P): sim of pair p [n0][n1] (row stride NP) = md0 . md1^T
__global__ void __launch_bounds__(256) lgx_sim_kernel(const float* __restrict__ md, int d, int NP, const int* __restrict__ nf, float* __restrict__ sim) {
  const int p = blockIdx.z, n0 = nf[2 * p], n1 = nf[2 * p + 1], m0 = blockIdx.y * 64;
  if (m0 >= n0 || static_cast<int>(blockIdx.x) * 64 >= n1) return;
  const size_t o = static_cast<size_t>(2 * p) * NP * d;
  gx_linear_tile(md + o, d, md + o + static_cast<size_t>(NP) * d, d, nullptr, sim + static_cast<size_t>(p) * NP * NP, NP, n0, n1, d, 1.f, nullptr,
                 0, 0, m0);
}

}  // namespace

int lgx_create(dimb_ctx* ctx, const float* weights, size_t n_floats, const dimb_lg_conf* cf, dimb_lgx** out) {
  *out = nullptr;
  const int d = cf->descriptor_dim, h = cf->num_heads, L = cf->n_layers, din = cf->input_dim;
  if (d < 2 || h < 1 || d % h != 0 || (d / h) % 2 != 0 || d / h > 128 || d > 1024 || L < 1 || din < 1 || cf->max_kpts < 1) {
    dimb_set_error(ctx, "dimb_lg_create: unsupported LightGlue shape (head dim must be even and <= 128)");
    return DIMB_ERR_UNSUPPORTED;
  }
  const int hd = d / h;
  size_t need = static_cast<size_t>(hd / 2) * 2;
  if (din != d) need += static_cast<size_t>(d) * din + d;
  const size_t per_layer = (3 * d * d + 3 * d) + (d * d + d) + (4 * d * d + 2 * d) + 4 * d + (2 * d * d + d)  // self
                           + 3 * (static_cast<size_t>(d) * d + d) + (4 * d * d + 2 * d) + 4 * d + (2 * d * d + d);  // cross
  need += per_layer * L + static_cast<size_t>(L) * (d + 1 + d * d + d) + static_cast<size_t>(L - 1) * (d + 1);
  if (n_floats != need) {
    dimb_set_error(ctx, "dimb_lg_create: weight blob has " + std::to_string(n_floats) + " floats, expected " + std::to_string(need));
    return DIMB_ERR_ARG;
  }
  dimb_lgx* g = new dimb_lgx();
  g->ctx = ctx;
  std::unique_ptr<dimb_lgx, void (*)(dimb_lgx*)> guard(g, lgx_destroy);  // a failed create releases what it built
  OwnerScope own(ctx, &g->mem);
  g->conf = *cf;
  g->d = d, g->h = h, g->hd = hd, g->din = din, g->L = L;
  g->NP = cf->max_kpts;
  const float* p = weights;
  auto up = [&](float** dst, size_t n) -> int {
    DIMB_TRY(dimb_alloc_t(ctx, dst, n, false));
    DIMB_CUDA_OK(ctx, cudaMemcpy(*dst, p, n * sizeof(float), cudaMemcpyHostToDevice));
    p += n;
    return static_cast<int>(DIMB_OK);
  };
  auto lin = [&](Lin& l, int n, int k) -> int {
    l.n = n, l.k = k;
    DIMB_TRY(up(&l.w, static_cast<size_t>(n) * k));
    return up(&l.b, n);
  };
  DIMB_TRY(up(&g->Wr, static_cast<size_t>(hd / 2) * 2));
  if (din != d) DIMB_TRY(lin(g->input_proj, d, din));
  g->self_.resize(L), g->cross_.resize(L);
  for (int i = 0; i < L; ++i) {
    Block& s = g->self_[i];
    DIMB_TRY(lin(s.qkv, 3 * d, d));
    DIMB_TRY(lin(s.out, d, d));
    DIMB_TRY(lin(s.ffn0, 2 * d, 2 * d));
    DIMB_TRY(up(&s.ln_g, 2 * d));
    DIMB_TRY(up(&s.ln_b, 2 * d));
    DIMB_TRY(lin(s.ffn3, d, 2 * d));
    Block& c = g->cross_[i];
    DIMB_TRY(lin(c.to_qk, d, d));
    DIMB_TRY(lin(c.to_v, d, d));
    DIMB_TRY(lin(c.out, d, d));
    DIMB_TRY(lin(c.ffn0, 2 * d, 2 * d));
    DIMB_TRY(up(&c.ln_g, 2 * d));
    DIMB_TRY(up(&c.ln_b, 2 * d));
    DIMB_TRY(lin(c.ffn3, d, 2 * d));
  }
  g->matchab.resize(L), g->final_proj.resize(L), g->token.resize(std::max(L - 1, 0));
  for (int i = 0; i < L; ++i) {
    DIMB_TRY(lin(g->matchab[i], 1, d));
    DIMB_TRY(lin(g->final_proj[i], d, d));
  }
  for (int i = 0; i < L - 1; ++i) DIMB_TRY(lin(g->token[i], 1, d));
  const size_t P = cf->max_pairs, S = 2 * P, NP = g->NP, R = S * NP;
  for (int k = 0; k < 2; ++k) {
    DIMB_TRY(dimb_alloc_t(ctx, &g->cat[k], R * 2 * d));
    DIMB_TRY(dimb_alloc_t(ctx, &g->enc[k], R * 2 * hd));
    DIMB_TRY(dimb_alloc_t(ctx, &g->ind[k], R));
    DIMB_TRY(dimb_alloc_t(ctx, &g->nact[k], S));
  }
  DIMB_TRY(dimb_alloc_t(ctx, &g->kp, R * 2));
  DIMB_TRY(dimb_alloc_t(ctx, &g->qkv, R * 3 * d));
  for (float** p : {&g->q, &g->k, &g->v, &g->xf, &g->md}) DIMB_TRY(dimb_alloc_t(ctx, p, R * d));
  DIMB_TRY(dimb_alloc_t(ctx, &g->hid, R * 2 * d));
  DIMB_TRY(dimb_alloc_t(ctx, &g->hid2, R * std::max(2 * d, din)));  // also the input-projection operand
  for (float** p : {&g->zt, &g->zm, &g->best}) DIMB_TRY(dimb_alloc_t(ctx, p, R));
  for (float** p : {&g->rlse, &g->clse}) DIMB_TRY(dimb_alloc_t(ctx, p, P * NP));
  DIMB_TRY(dimb_alloc_t(ctx, &g->sim, P * NP * NP));
  for (int** p : {&g->idx, &g->indf, &g->arg}) DIMB_TRY(dimb_alloc_t(ctx, p, R));
  for (int** p : {&g->n_orig, &g->nf}) DIMB_TRY(dimb_alloc_t(ctx, p, S));
  for (int** p : {&g->stopped, &g->layer, &g->parity}) DIMB_TRY(dimb_alloc_t(ctx, p, P));
  DIMB_TRY(dimb_alloc(ctx, &g->in, S * sizeof(SideInX)));
  std::vector<const float*> tab(4 * static_cast<size_t>(L));
  for (int i = 0; i < L; ++i) {
    tab[i] = g->final_proj[i].w, tab[L + i] = g->final_proj[i].b;
    tab[2 * L + i] = g->matchab[i].w, tab[3 * L + i] = g->matchab[i].b;
  }
  DIMB_TRY(dimb_alloc(ctx, reinterpret_cast<void**>(&g->tab), tab.size() * sizeof(float*)));
  DIMB_CUDA_OK(ctx, cudaMemcpy(g->tab, tab.data(), tab.size() * sizeof(float*), cudaMemcpyHostToDevice));
  g->tc_attn = hd > 64 && hd <= kXHd;
  if (g->tc_attn) {
    Hd128Ops& o = g->tc;
    o.S = static_cast<int>(S), o.h = h, o.d = d, o.hd = hd, o.NP = g->NP, o.NPp = round_up(g->NP, kAttnTile);
    const size_t nel = S * h * o.NPp * kXHd;
    for (int pl = 0; pl < 2; ++pl)
      for (__half** p : {&o.q[pl], &o.k[pl], &o.vt[pl]}) DIMB_TRY(dimb_alloc_t(ctx, p, nel));
    DIMB_TRY(hd128_maps(ctx, o));
  }
  *out = guard.release();
  return DIMB_OK;
}

void lgx_destroy(dimb_lgx* g) {
  if (!g) return;
  dimb_release(g->ctx, g->mem);
  delete g;
}

int lgx_match_dev(dimb_lgx* g, int P, const dimb_feats_dev* f0, const dimb_feats_dev* f1, int64_t* d_matches, float* d_mscores, int* d_n_matches,
                  int* d_stop_layer, int cap, cudaStream_t st) {
  dimb_ctx* ctx = g->ctx;
  const dimb_lg_conf& cf = g->conf;
  const int d = g->d, hd = g->hd, h = g->h, L = g->L, din = g->din, NP = g->NP, S = 2 * P;
  if (!d_matches || !d_mscores || !d_n_matches || !d_stop_layer || P < 1 || P > cf.max_pairs || cap < 1) return DIMB_ERR_ARG;
  std::vector<SideInX> hin(S);
  for (int s = 0; s < S; ++s) {
    const dimb_feats_dev& f = (s & 1) ? f1[s >> 1] : f0[s >> 1];
    if (f.n_cap < 0 || f.n_cap > NP || !f.n || (f.n_cap > 0 && (!f.keypoints || !f.descriptors)) || (f.desc_layout != 0 && f.desc_layout != 1)) {
      dimb_set_error(ctx, "dimb_lg_match_dev: invalid feature set (n_cap above max_kpts, NULL pointer or unknown layout)");
      return DIMB_ERR_ARG;
    }
    SideInX& o = hin[s];
    o.kpts = f.keypoints, o.desc = f.descriptors, o.n = f.n, o.n_cap = f.n_cap, o.layout = f.desc_layout;
    o.ld = f.desc_ld ? f.desc_ld : (f.desc_layout == 0 ? f.n_cap : din);
    o.size0 = f.size0, o.size1 = f.size1, o.round_fp16 = f.round_fp16, o.f16 = f.f16, o.size_dev = f.size_dev, o.size_f32 = f.size_f32_dev;
  }
  DIMB_CUDA_OK(ctx, cudaSetDevice(ctx->device));
  const int do_stop = cf.depth_confidence > 0, do_prune = cf.width_confidence > 0, adaptive = do_stop || do_prune;
  const size_t sRow2 = static_cast<size_t>(NP) * 2 * d, sRow = static_cast<size_t>(NP) * d;
  const int* const stp = g->stopped;
  DIMB_CUDA_OK(ctx, cudaMemcpyAsync(g->in, hin.data(), S * sizeof(SideInX), cudaMemcpyHostToDevice, st));
  auto lin = [&](const float* A, int lda, size_t sA, const Lin& l, float* C, int ldc, size_t sC, const int* nact, bool resid) -> int {
    lgx_linear_kernel<<<dim3(ceil_div(l.n, 64), ceil_div(NP, 64), S), 256, 0, st>>>(A, lda, sA, l.w, l.b, C, ldc, sC, l.n, l.k, 1.f,
                                                                                    resid ? C : nullptr, nact, stp, 1, nullptr, nullptr, nullptr);
    DIMB_LAUNCH_CHECK(ctx);
    return DIMB_OK;
  };
  const int rows_grid = ceil_div(S * NP * 32, 256);
  {  // ---- inputs, input projection, positional encoding
    ProfScope prof(ctx, st, "lgx.prep");
    const SideInX* in = static_cast<const SideInX*>(g->in);
    float* x = din != d ? g->hid2 : g->cat[0];
    lgx_prep_kernel<<<dim3(ceil_div(NP, 32), S), dim3(32, 8), 0, st>>>(in, din, NP, x, din != d ? din : 2 * d, g->kp, g->ind[0], g->nact[0], g->n_orig,
                                                                         g->stopped);
    DIMB_LAUNCH_CHECK(ctx);
    if (din != d) DIMB_TRY(lin(g->hid2, din, static_cast<size_t>(NP) * din, g->input_proj, g->cat[0], 2 * d, sRow2, g->nact[0], false));
    lgx_posenc_kernel<<<S, 1024, 0, st>>>(in, g->kp, g->nact[0], NP, g->Wr, hd, g->enc[0]);
    DIMB_LAUNCH_CHECK(ctx);
  }
  // q / k / v rows of every side -> hid; with tensor cores the packing of the operands comes first (cross: keys = the partner's q rows)
  auto attend = [&](const float* q, const float* k, const float* v, int cross, const int* nact) -> int {
    if (g->tc_attn) {
      ProfScope prof(ctx, st, "lgx.attn_tc");
      return hd128_attend(ctx, st, g->tc, S, q, k, v, cross, nact, stp, ctx->attn_lazy, g->hid);
    }
    ProfScope prof(ctx, st, "lgx.attn");
    const dim3 grid(ceil_div(NP, 8), h, S);
    if (hd <= 32)
      lgx_attention_kernel<32><<<grid, 256, 0, st>>>(q, k, v, NP, d, hd, cross, g->hid, nact, stp);
    else if (hd <= 64)
      lgx_attention_kernel<64><<<grid, 256, 0, st>>>(q, k, v, NP, d, hd, cross, g->hid, nact, stp);
    else if (hd <= 96)
      lgx_attention_kernel<96><<<grid, 256, 0, st>>>(q, k, v, NP, d, hd, cross, g->hid, nact, stp);
    else
      lgx_attention_kernel<128><<<grid, 256, 0, st>>>(q, k, v, NP, d, hd, cross, g->hid, nact, stp);
    DIMB_LAUNCH_CHECK(ctx);
    return DIMB_OK;
  };
  auto ffn = [&](float* cat, const Block& bl, const int* nact) -> int {
    DIMB_TRY(lin(cat, 2 * d, sRow2, bl.ffn0, g->hid, 2 * d, sRow2, nact, false));
    lgx_ln_gelu_kernel<<<rows_grid, 256, 0, st>>>(g->hid, 2 * d, NP, bl.ln_g, bl.ln_b, g->hid2, nact, stp, S);
    DIMB_LAUNCH_CHECK(ctx);
    return lin(g->hid2, 2 * d, sRow2, bl.ffn3, cat, 2 * d, sRow2, nact, true);
  };
  for (int i = 0; i < L; ++i) {
    const int cur = adaptive ? (i & 1) : 0, nxt = cur ^ 1;
    float* cat = g->cat[cur];
    const int* nact = g->nact[cur];
    const Block &sb = g->self_[i], &cb = g->cross_[i];
    {
      ProfScope prof(ctx, st, "lgx.self");
      DIMB_TRY(lin(cat, 2 * d, sRow2, sb.qkv, g->qkv, 3 * d, 3 * sRow, nact, false));
      lgx_qkv_rotary_kernel<<<dim3(NP, S), std::max(32, d / 2), 0, st>>>(g->qkv, d, hd, g->enc[cur], NP, g->q, g->k, g->v, nact, stp);
      DIMB_LAUNCH_CHECK(ctx);
    }
    DIMB_TRY(attend(g->q, g->k, g->v, 0, nact));
    {
      ProfScope prof(ctx, st, "lgx.self");
      DIMB_TRY(lin(g->hid, d, sRow, sb.out, cat + d, 2 * d, sRow2, nact, false));
      DIMB_TRY(ffn(cat, sb, nact));
    }
    {
      ProfScope prof(ctx, st, "lgx.cross");
      DIMB_TRY(lin(cat, 2 * d, sRow2, cb.to_qk, g->q, d, sRow, nact, false));
      DIMB_TRY(lin(cat, 2 * d, sRow2, cb.to_v, g->v, d, sRow, nact, false));
    }
    DIMB_TRY(attend(g->q, g->q, g->v, 1, nact));
    {
      ProfScope prof(ctx, st, "lgx.cross");
      DIMB_TRY(lin(g->hid, d, sRow, cb.out, cat + d, 2 * d, sRow2, nact, false));
      DIMB_TRY(ffn(cat, cb, nact));
    }
    if (i == L - 1 || !adaptive) continue;  // nothing to decide after the last layer, nor in a fixed-work run
    ProfScope prof(ctx, st, "lgx.tail");
    if (do_stop) {
      lgx_rowdot_kernel<<<rows_grid, 256, 0, st>>>(cat, 2 * d, d, NP, g->token[i].w, g->token[i].b, g->zt, nact, stp, 1, nullptr, nullptr, nullptr, S);
      DIMB_LAUNCH_CHECK(ctx);
    }
    if (do_prune) {
      lgx_rowdot_kernel<<<rows_grid, 256, 0, st>>>(cat, 2 * d, d, NP, g->matchab[i].w, g->matchab[i].b, g->zm, nact, stp, 1, nullptr, nullptr, nullptr,
                                                   S);
      DIMB_LAUNCH_CHECK(ctx);
    }
    lgx_decide_kernel<<<P, 1024, 0, st>>>(i, L, NP, g->zt, g->zm, nact, g->nact[nxt], g->n_orig, g->stopped, g->idx, conf_threshold(i, L),
                                          static_cast<float>(cf.depth_confidence), static_cast<float>(1.0 - cf.width_confidence), do_stop, do_prune,
                                          cf.prune_min_kpts);
    DIMB_LAUNCH_CHECK(ctx);
    lgx_gather_kernel<<<dim3(NP, S), 128, 0, st>>>(i, g->stopped, g->nact[nxt], g->idx, NP, d, hd, cat, g->cat[nxt], g->enc[cur], g->enc[nxt],
                                                   g->ind[cur], g->ind[nxt]);
    DIMB_LAUNCH_CHECK(ctx);
  }
  // ---- assignment (lightglue.py:246-275) and filter_matches (:281-297), per pair at the layer it ended at
  ProfScope prof(ctx, st, "lgx.assign");
  lgx_final_select_kernel<<<ceil_div(P, 128), 128, 0, st>>>(g->stopped, g->nact[0], g->nact[1], g->nf, g->layer, g->parity, P, L, adaptive);
  DIMB_LAUNCH_CHECK(ctx);
  lgx_final_gather_kernel<<<dim3(NP, S), 128, 0, st>>>(g->nf, g->parity, NP, d, g->cat[0], g->cat[1], g->ind[0], g->ind[1], g->xf, g->indf);
  DIMB_LAUNCH_CHECK(ctx);
  const float inv = 1.f / std::pow(static_cast<float>(d), 0.25f);
  lgx_linear_kernel<<<dim3(ceil_div(d, 64), ceil_div(NP, 64), S), 256, 0, st>>>(g->xf, d, sRow, nullptr, nullptr, g->md, d, sRow, d, d, inv, nullptr,
                                                                                g->nf, g->stopped, 0, g->tab, g->tab + L, g->layer);
  DIMB_LAUNCH_CHECK(ctx);
  lgx_rowdot_kernel<<<rows_grid, 256, 0, st>>>(g->xf, d, d, NP, nullptr, nullptr, g->zt, g->nf, g->stopped, 0, g->tab + 2 * L, g->tab + 3 * L,
                                               g->layer, S);
  DIMB_LAUNCH_CHECK(ctx);
  lgx_sim_kernel<<<dim3(ceil_div(NP, 64), ceil_div(NP, 64), P), 256, 0, st>>>(g->md, d, NP, g->nf, g->sim);
  DIMB_LAUNCH_CHECK(ctx);
  return launch_lgx_assign(ctx, st, P, NP, g->sim, g->nf, g->zt, g->stopped, L, g->indf, static_cast<float>(cf.filter_threshold), g->rlse, g->clse,
                           g->best, g->arg, reinterpret_cast<long long*>(d_matches), d_mscores, d_n_matches, d_stop_layer, cap);
}
