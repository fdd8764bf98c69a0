// attention.cuh - tensor-core flash attention on sm_90a (wgmma), shared by the 64-dim heads of LightGlue / SuperGlue
// (lg_kernels.cuh) and the padded 128-dim heads of the shape-generic path (attn_hd128.cuh).
//
// One CTA = one 128-row query tile of one head; 288 threads: two consumer warpgroups (query rows 64 wg .. 64 wg + 63) and one TMA
// producer warp that streams 64-key blocks of K and V^T through a two-stage mbarrier ring.  Per key block a warpgroup computes
//   S = Q K^T           wgmma, A = Q and B = K from shared memory, fp32 accumulator in registers
//   online softmax      in the accumulator layout (a row lives in 4 lanes: max by two shuffles), with lazy rescaling: O / l are
//                       rescaled only when a row maximum grows by more than 2^lazy over the reference it was scaled by
//   O += P V            wgmma, A = P straight from registers (the S accumulator of 16 keys IS the A fragment of a 16-deep step),
//                       B = V^T from shared memory
// EXACT mode = fp16 hi / lo planes of Q, K, V and P, three MMAs per product (fp32-class); FAST = hi planes only.
#pragma once
#include "common.cuh"
#include "sm90.cuh"

namespace {

constexpr int kAttnBlk = 64;   // keys per block
constexpr int kAttnTile = 128; // queries per CTA
constexpr int kAttnThreads = 9 * 32;

template <int HD, bool SPLIT>
struct AttnGeom {
  static constexpr int kPl = SPLIT ? 2 : 1;
  static constexpr int kAtoms = HD / 64;                   // [rows x 64 halfs] swizzle atoms along the head dim
  static constexpr int kAtomQ = kAttnTile * 128, kQB = kAtoms * kAtomQ;
  static constexpr int kAtomK = kAttnBlk * 128, kKB = kAtoms * kAtomK;
  static constexpr int kVB = HD * 128;                     // V^T plane: [HD dims x 64 keys]
  static constexpr int kSmem = kPl * (kQB + 2 * (kKB + kVB)) + 256 + 1024;
};

// Maps / rows: Q rows qrow .. qrow + 127 (box 128 rows x 64 halfs), K rows krow + key (box 64 rows), V^T rows vrow .. vrow + HD - 1
// (box HD rows x 64 keys).  `out(row, col, x, y)` receives O[row][col], O[row][col + 1] (row < 128 of the tile, col even); rows
// >= nq are not handed out.  nk == 0 gives zeros (Attention.forward on an empty key set, lightglue.py:103-104).
template <int HD, bool SPLIT, class Out>
__device__ __forceinline__ void attn_tile(const CUtensorMap* tmQh, const CUtensorMap* tmQl, const CUtensorMap* tmKh,
                                          const CUtensorMap* tmKl, const CUtensorMap* tmVh, const CUtensorMap* tmVl, int qrow, int krow,
                                          int vrow, int nq, int nk, float scale, float lazy, const Out& out) {
  using namespace sm90;
  using G = AttnGeom<HD, SPLIT>;
  extern __shared__ uint8_t sm_attn_raw[];
  uint8_t* smem = sm_attn_raw + ((1024u - (smem_u32(sm_attn_raw) & 1023u)) & 1023u);
  uint8_t* sQ = smem;                        // [plane]
  uint8_t* sK = sQ + G::kPl * G::kQB;        // [stage][plane]
  uint8_t* sV = sK + 2 * G::kPl * G::kKB;    // [stage][plane]
  uint64_t* bars = reinterpret_cast<uint64_t*>(sV + 2 * G::kPl * G::kVB);
  uint64_t *bQ = bars, *kFull = bars + 1, *kEmpty = bars + 3, *vFull = bars + 5, *vEmpty = bars + 7;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  if (tid == 0) {
    mbar_init(bQ, 1);
    for (int i = 0; i < 2; ++i) {
      mbar_init(&kFull[i], 1);
      mbar_init(&kEmpty[i], 8);  // one arrival per consumer warp
      mbar_init(&vFull[i], 1);
      mbar_init(&vEmpty[i], 8);
    }
    fence_barrier_init();
  }
  __syncthreads();
  const int nblk = (nk + kAttnBlk - 1) / kAttnBlk;

  if (warp == 8) {  // ---------------- TMA producer (whole warp waits, one elected lane issues)
    if (nblk > 0 && elect_one()) {
      mbar_expect_tx(bQ, G::kPl * G::kQB);
      for (int at = 0; at < G::kAtoms; ++at) {
        tma_load_2d(sQ + at * G::kAtomQ, tmQh, bQ, at * 64, qrow);
        if (SPLIT) tma_load_2d(sQ + G::kQB + at * G::kAtomQ, tmQl, bQ, at * 64, qrow);
      }
    }
    __syncwarp();
    for (int j = 0; j < nblk; ++j) {
      const int s = j & 1;
      const uint32_t ph = (j >> 1) & 1;
      mbar_wait(&kEmpty[s], ph ^ 1);
      if (elect_one()) {
        mbar_expect_tx(&kFull[s], G::kPl * G::kKB);
        for (int at = 0; at < G::kAtoms; ++at) {
          tma_load_2d(sK + s * G::kPl * G::kKB + at * G::kAtomK, tmKh, &kFull[s], at * 64, krow + j * kAttnBlk);
          if (SPLIT) tma_load_2d(sK + s * G::kPl * G::kKB + G::kKB + at * G::kAtomK, tmKl, &kFull[s], at * 64, krow + j * kAttnBlk);
        }
      }
      __syncwarp();
      mbar_wait(&vEmpty[s], ph ^ 1);
      if (elect_one()) {
        mbar_expect_tx(&vFull[s], G::kPl * G::kVB);
        tma_load_2d(sV + s * G::kPl * G::kVB, tmVh, &vFull[s], j * kAttnBlk, vrow);
        if (SPLIT) tma_load_2d(sV + s * G::kPl * G::kVB + G::kVB, tmVl, &vFull[s], j * kAttnBlk, vrow);
      }
      __syncwarp();
    }
    return;
  }
  // ---------------- consumer warpgroup wg
  const int wg = warp >> 2, w4 = warp & 3;
  const int r0 = 64 * wg + 16 * w4 + (lane >> 2);  // this thread's rows r0 and r0 + 8 of the tile
  const uint32_t q_wg = smem_u32(sQ) + wg * 64 * 128;
  float o[HD / 2];
#pragma unroll
  for (int i = 0; i < HD / 2; ++i) o[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};  // l_run: this lane's partial row sums
  const float c2 = scale * 1.4426950408889634f;                   // softmax(scale * s) via exp2
  if (nblk > 0) mbar_wait(bQ, 0);
  for (int j = 0; j < nblk; ++j) {
    const int s = j & 1;
    const uint32_t ph = (j >> 1) & 1;
    float sc[kAttnBlk / 2];
    mbar_wait(&kFull[s], ph);
    {
      const uint32_t kb = smem_u32(sK + s * G::kPl * G::kKB);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 4 * G::kAtoms; ++kk) {
        const uint64_t qh = sdesc_advance_k(make_sdesc_sw128(q_wg + (kk >> 2) * G::kAtomQ), kk & 3);
        const uint64_t kh = sdesc_advance_k(make_sdesc_sw128(kb + (kk >> 2) * G::kAtomK), kk & 3);
        Wgmma<kAttnBlk>::ss(sc, qh, kh, kk != 0);
        if (SPLIT) {
          const uint64_t ql = sdesc_advance_k(make_sdesc_sw128(q_wg + G::kQB + (kk >> 2) * G::kAtomQ), kk & 3);
          const uint64_t kl = sdesc_advance_k(make_sdesc_sw128(kb + G::kKB + (kk >> 2) * G::kAtomK), kk & 3);
          Wgmma<kAttnBlk>::ss(sc, qh, kl, 1);
          Wgmma<kAttnBlk>::ss(sc, ql, kh, 1);
        }
      }
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(sc);
    }
    if (lane == 0) mbar_arrive(&kEmpty[s]);
    // sc[4i + 2h + e]: row r0 + 8h, key j * 64 + 8i + 2 (lane % 4) + e
    const int key0 = j * kAttnBlk + 2 * (lane & 3);
    if (j * kAttnBlk + kAttnBlk > nk) {
#pragma unroll
      for (int i = 0; i < kAttnBlk / 8; ++i)
#pragma unroll
        for (int e = 0; e < 4; ++e)
          if (key0 + 8 * i + (e & 1) >= nk) sc[4 * i + e] = -INFINITY;
    }
    float alpha[2], mc[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float mx = sc[2 * h];
#pragma unroll
      for (int i = 0; i < kAttnBlk / 8; ++i) mx = fmaxf(mx, fmaxf(sc[4 * i + 2 * h], sc[4 * i + 2 * h + 1]));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      // Lazy rescaling: softmax is invariant to the reference subtracted in the exponent, so the running reference only has to stay
      // within 2^lazy of the true maximum (P <= 2^lazy, far inside fp16 / fp32 range; the hi/lo split keeps its RELATIVE precision).
      const float m_blk = fmaxf(m_run[h], mx);
      const bool grow = (m_blk - m_run[h]) * c2 > lazy;  // always true on the first block (m_run = -inf)
      const float m_new = grow ? m_blk : m_run[h];
      alpha[h] = grow ? fast_exp2((m_run[h] - m_new) * c2) : 1.f;  // 0 on the first block
      mc[h] = m_new * c2;
      m_run[h] = m_new;
    }
    float ps[2] = {0.f, 0.f};
#pragma unroll
    for (int i = 0; i < kAttnBlk / 8; ++i)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        sc[4 * i + e] = fast_exp2(fmaf(sc[4 * i + e], c2, -mc[e >> 1]));
        ps[e >> 1] += sc[4 * i + e];
      }
#pragma unroll
    for (int h = 0; h < 2; ++h) l_run[h] = l_run[h] * alpha[h] + ps[h];
#pragma unroll
    for (int i = 0; i < HD / 8; ++i) {
      o[4 * i] *= alpha[0], o[4 * i + 1] *= alpha[0];
      o[4 * i + 2] *= alpha[1], o[4 * i + 3] *= alpha[1];
    }
    // P as the register A operand: k-step kk (keys 16 kk .. 16 kk + 15) = accumulator column blocks 2 kk and 2 kk + 1
    uint32_t ph_[kAttnBlk / 4], pl_[kAttnBlk / 4];
#pragma unroll
    for (int c = 0; c < kAttnBlk / 4; ++c) {
      __half2 h2, l2;
      split2_f32(sc[2 * c], sc[2 * c + 1], h2, l2);
      ph_[c] = *reinterpret_cast<uint32_t*>(&h2);
      pl_[c] = *reinterpret_cast<uint32_t*>(&l2);
    }
    mbar_wait(&vFull[s], ph);
    {
      const uint32_t vb = smem_u32(sV + s * G::kPl * G::kVB);
      const uint64_t v_h = make_sdesc_sw128(vb), v_l = make_sdesc_sw128(vb + G::kVB);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < kAttnBlk / 16; ++kk) {
        const uint32_t ah[4] = {ph_[4 * kk], ph_[4 * kk + 1], ph_[4 * kk + 2], ph_[4 * kk + 3]};
        Wgmma<HD>::rs(o, ah, sdesc_advance_k(v_h, kk), 1);
        if (SPLIT) {
          const uint32_t al[4] = {pl_[4 * kk], pl_[4 * kk + 1], pl_[4 * kk + 2], pl_[4 * kk + 3]};
          Wgmma<HD>::rs(o, ah, sdesc_advance_k(v_l, kk), 1);
          Wgmma<HD>::rs(o, al, sdesc_advance_k(v_h, kk), 1);
        }
      }
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(o);
    }
    if (lane == 0) mbar_arrive(&vEmpty[s]);
  }
  float inv[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float l = l_run[h];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    inv[h] = nblk > 0 ? 1.f / l : 0.f;
  }
#pragma unroll
  for (int i = 0; i < HD / 8; ++i) {
    const int col = 8 * i + 2 * (lane & 3);
    if (r0 < nq) out(r0, col, o[4 * i] * inv[0], o[4 * i + 1] * inv[0]);
    if (r0 + 8 < nq) out(r0 + 8, col, o[4 * i + 2] * inv[1], o[4 * i + 3] * inv[1]);
  }
}

}  // namespace
