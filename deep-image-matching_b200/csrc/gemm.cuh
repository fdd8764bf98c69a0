// gemm.cuh - the tensor-core workhorse of libdimb200.
//
// One kernel template covers every dense contraction on the hot path:
//   C[M,N] = A[M,K] * B[N,K]^T      (LightGlue linears, 1x1 convs, similarity / distance matrices)
//   3x3 convolution as implicit GEMM (SuperPoint VGG encoder and heads): K = 9 taps x Cin, the A tile of a
//   tap is the NHWC activation tile shifted by (dy-1, dx-1), fetched by a 4D TMA whose out-of-bounds
//   fill implements the zero padding.
//
// Structure (sm_90a): 384 threads = 2 consumer warpgroups + 1 producer warpgroup (one warp of it issues the TMA copies).
//   setmaxnreg moves registers from the producer warpgroup (40 per thread) to the consumers (232): a 128 x 256 tile keeps
//   128 fp32 accumulators per consumer thread plus the epilogue's working set without spilling.
//   producer : cp.async.bulk.tensor -> swizzled smem stages, mbarrier full/empty ring
//   consumers: warpgroup g issues wgmma (M = 64 rows 64g..64g+63 of the 128-row tile, N = BN, K = 16) into fp32
//              registers (conv mode 2: rows 128g..128g+127 of a 256-row tile, two M = 64 halves); EXACT mode issues
//              hi*hi + hi*lo + lo*hi per k-step (fp16 split operands).  After the last k-step the warpgroup stages its
//              accumulator through shared memory, 64 columns at a time (mode 2: 16), so that thread r owns output row r
//              and 32 consecutive columns -> fused epilogue functor
//
// The kernel is persistent: one CTA per SM; the producer fills the stages of the next tile while the consumers run the epilogue.
#pragma once
#include "common.cuh"
#include "sm90.cuh"

struct TileCoord {
  int m0;         // GEMM: first global row of this 128-row tile
  int n0;         // first output column of this tile
  int b, y0, x0;  // CONV: image index and top-left pixel of the ConvTile<CONV>::TH x 16 pixel tile
};

// Field order: the kernel reads num_kb, cin_blocks, tiles_x and tiles_y, and each of them shares its 8-byte word with a field it does
// not read.  With tiles_x and tiles_y in one word nvcc loads them as a pair and schedules the 3x3 conv kernels differently: the
// 128 -> 256 channel SuperPoint convolutions (convPa, convDa) then ran about 4 % slower on an H100 SXM at 700 W.
struct GemmArgs {
  int num_kb;      // B tiles per output tile: K / 64 (CONV 3: K / 32)
  int M;           // GEMM: valid rows of A
  int cin_blocks;  // CONV: Cin / 64
  int N;           // valid rows of B (output columns)
  int H;           // CONV: image height
  int tiles_x;     // CONV: tiles per image row / column
  int tiles_y;
  int W;           // CONV: image width
};

constexpr int kTileM = 128;
constexpr int kGemmThreads = 12 * 32;  // warps 0-7: two consumer warpgroups, warps 8-11: producer warpgroup (warp 8 issues)
constexpr int kProducerRegs = 40, kConsumerRegs = 232;  // 128 x 40 + 256 x 232 <= 64 K registers of the SM
// Per-warp shared scratch of the epilogue functors: a 32 x 32 fp32 chunk used to turn "lane = row" into "8 lanes = one row segment"
// so that global accesses are coalesced.  Rows are 128 B with the eight 16-byte chunks XOR-swizzled by (row & 7): conflict-free for
// both the row-wise writes and the transposed reads without padding.
constexpr int kScratchPitch = 32;
constexpr int kScratchFloats = 32 * kScratchPitch;
// Accumulator staging of one consumer warpgroup: [64 rows][64 columns] fp32, rows padded by 4 floats (the float4 row reads of 8
// consecutive lanes hit 8 distinct 16-byte bank groups).  Once every warp holds its 32 x 32 chunk in registers the same bytes are the
// four warps' functor scratch (4 x 4 KB <= 17 KB).
constexpr int kStgCols = 64, kStgPitch = kStgCols + 4;
constexpr int kStgFloats = 64 * kStgPitch;
constexpr int kStgBytes = 2 * kStgFloats * 4;
static_assert(4 * kScratchFloats <= kStgFloats, "functor scratch must fit in the staging buffer of a warpgroup");
// CONV modes of the kernel templates (int CONV):
//   0  plain GEMM
//   1  3x3 conv, tile = 8 rows x 16 pixels, one (8+2) x 16-pixel box of 64 channels per dx (three boxes per channel block);
//      the three dy taps are the same stage at descriptor offsets of one box row (2048 B)
//   2  3x3 conv, tile = 16 rows x 16 pixels, BN 64 only: as mode 1 with a (16+2) x 16-pixel box, so that every weight tile streamed
//      from L2 serves 256 output pixels instead of 128.  A consumer warpgroup owns 128 pixel rows and issues two m64 wgmma per
//      product; its accumulator is staged kStgCols2 columns at a time, which leaves no functor scratch (Epi::kScratch false)
//   3  plain GEMM with 32-wide K blocks (64-byte rows, SWIZZLE_64B): half-size pipeline stages, so that more of them fit next to
//      the 128 x 256 tiles
constexpr int kConvTH = 8, kConvTW = 16;    // mode 1 tile
constexpr int kConvTH2 = 16;                // mode 2 tile height
// mode 2 staging: [64 rows][16 columns] per warpgroup, rows padded by 4 floats (80 B: the float4 row reads of 8 consecutive lanes hit 8
// distinct 16-byte bank groups).  10 KB for both warpgroups instead of 35 KB: two A stages and four B slots fit next to it
constexpr int kStgCols2 = 16, kStgPitch2 = kStgCols2 + 4;
static_assert(32 % kStgCols2 == 0, "a thread's 32 epilogue columns are whole staging chunks");
__host__ __device__ constexpr bool conv_is_3x3(int conv) { return conv == 1 || conv == 2; }
template <int CONV>
struct ConvTile {
  static constexpr int TH = CONV == 2 ? kConvTH2 : kConvTH, TW = kConvTW;
};

template <int CONV>
__device__ __forceinline__ TileCoord make_tile_coord(const GemmArgs& g, int t) {
  TileCoord tc;
  if (conv_is_3x3(CONV)) {
    int per_img = g.tiles_x * g.tiles_y;
    tc.b = t / per_img;
    int rem = t - tc.b * per_img;
    tc.y0 = (rem / g.tiles_x) * ConvTile<CONV>::TH;
    tc.x0 = (rem % g.tiles_x) * ConvTile<CONV>::TW;
    tc.m0 = 0;
    tc.n0 = 0;
  } else {
    tc.m0 = t * kTileM;
    tc.n0 = 0;
    tc.b = tc.y0 = tc.x0 = 0;
  }
  return tc;
}

// ------------------------------------------------------------------ persistent tensor-core kernel
// One CTA per SM loops over output tiles:
//   * A and B have separate smem rings.  CONV modes 1 / 2 fetch the activation tile ONCE per (dx, channel block) as
//     a (TH+2) x 16 pixel box (TH = 8 / 16) and run the three dy taps out of it by advancing the smem descriptor by one box
//     row (16 px * 128 B = 2048 B, swizzle-atom aligned): 3 A loads per channel block instead of 9;
//   * RESB: when all weight tiles of the layer fit (64->64 convs: 9 x 16 KB), they are loaded once per CTA and
//     stay resident; only activations stream.  Otherwise mode 2 releases each dy's B tile as its MMAs retire.
struct PersCfg {
  int sa, sb;        // A / B ring depth (sb unused with RESB)
  int nkb_total;     // B tiles per output tile (RESB: resident tiles)
  int smem_bytes;
};

template <int BN, bool SPLIT, int CONV>
struct PersGeom {
  static constexpr int kPl = SPLIT ? 2 : 1;
  static constexpr int kRowB = CONV == 3 ? 64 : 128;  // bytes per shared-memory operand row (K block of 32 / 64 halfs)
  static constexpr int kABoxTx =  // bytes a TMA box delivers
      conv_is_3x3(CONV) ? (ConvTile<CONV>::TH + 2) * kConvTW * 128 : kTileM * kRowB;
  static constexpr int kABox = (kABoxTx + 1023) / 1024 * 1024;  // plane pitch inside a stage (swizzle-atom aligned)
  static constexpr int kATx = kPl * kABoxTx;
  static constexpr int kAStage = kPl * kABox;
  static constexpr int kBPlane = BN * kRowB;
  static constexpr int kBTile = kPl * kBPlane;
  static constexpr int kStgFloats = CONV == 2 ? 64 * kStgPitch2 : ::kStgFloats;  // accumulator staging per consumer warpgroup
  static constexpr int kStgBytes = 2 * kStgFloats * 4;
  static constexpr int kBudget = kSmemOptin - 1024 - 1024 - kStgBytes;
};

template <int BN, bool SPLIT, int CONV, bool RESB, class Epi>
__global__ void __launch_bounds__(kGemmThreads, 1)
tc_gemm_pers_kernel(const __grid_constant__ CUtensorMap tmAh, const __grid_constant__ CUtensorMap tmAl,
                    const __grid_constant__ CUtensorMap tmBh, const __grid_constant__ CUtensorMap tmBl, GemmArgs g, Epi epi,
                    int m_tiles, int n_tiles, int SA, int SB) {
  using G = PersGeom<BN, SPLIT, CONV>;
  using namespace sm90;
  static_assert(BN % kStgCols == 0, "BN must be a multiple of the staging width");
  static_assert(CONV != 2 || (BN == 64 && !Epi::kScratch), "mode 2: BN 64, and an epilogue without functor scratch");
  extern __shared__ uint8_t smem_raw[];
  // 1024-byte alignment by OFFSET from the __shared__ array (not by integer-casting the pointer): the compiler keeps the shared
  // address space and emits LDS / STS instead of generic LD / ST for every access derived from it
  uint8_t* smem = smem_raw + ((1024u - (sm90::smem_u32(smem_raw) & 1023u)) & 1023u);
  constexpr bool ISCONV = conv_is_3x3(CONV);
  constexpr int MH = CONV == 2 ? 2 : 1;  // 64-row MMA halves per consumer warpgroup
  // mode 2 holds only three B slots: each dy's weight tile is released as soon as its MMAs retire (one commit group per dy)
  constexpr bool EARLY_B = CONV == 2 && !RESB;
  constexpr bool K32 = CONV == 3;
  constexpr int KB_COLS = K32 ? 32 : 64;  // K elements per B tile / A stage
  constexpr int KSTEPS = K32 ? 2 : 4;     // 16-deep MMA steps per K block
  constexpr uint32_t kLayout = K32 ? kLayoutSw64 : kLayoutSw128;
  constexpr uint32_t kSbo = 8 * G::kRowB;
  const int nkb = g.num_kb;  // GEMM: K/64 (CONV 3: K/32).  CONV 1: 9 * cin_blocks
  uint8_t* sA = smem;
  uint8_t* sB = sA + SA * G::kAStage;
  const int nb_slots = RESB ? nkb : SB;
  uint64_t* fullA = reinterpret_cast<uint64_t*>(sB + nb_slots * G::kBTile);
  uint64_t* emptyA = fullA + SA;
  uint64_t* fullB = emptyA + SA;
  uint64_t* emptyB = fullB + nb_slots;
  float* staging = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(fullA) + 1024);  // [2 warpgroups][G::kStgFloats]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int s = 0; s < SA; ++s) {
      mbar_init(&fullA[s], 1);
      mbar_init(&emptyA[s], 8);  // one arrival per consumer warp
    }
    for (int s = 0; s < nb_slots; ++s) {
      mbar_init(&fullB[s], 1);
      mbar_init(&emptyB[s], 8);
    }
    fence_barrier_init();
  }
  __syncthreads();
  const int total = m_tiles * n_tiles;
  const int cinb = ISCONV ? g.cin_blocks : 1;
  // A stages per output tile and B tiles (taps) consumed out of each stage
  const int outer_n = ISCONV ? 3 * cinb : nkb;
  constexpr int inner_n = ISCONV ? 3 : 1;
  // B tile index of tap step `in` of A stage `o`: weights are [Cout][tap * Cin + c]
  auto kb_of = [&](int o, int in) { return ISCONV ? ((in * 3 + o / cinb) * cinb + (o % cinb)) : o; };

  auto tile_coord = [&](int w, int& n0) {
    const int mt = w / n_tiles, nt = w - mt * n_tiles;
    TileCoord tc = make_tile_coord<CONV>(g, mt);
    if (!ISCONV) tc.m0 = epi.m0_of(mt);
    n0 = nt * BN;
    tc.n0 = n0;
    return tc;
  };

  if (warp >= 8) {
    setmaxnreg_dec<kProducerRegs>();
    if (warp == 8) {  // ---------------- TMA producer: the whole warp walks the schedule and waits, one elected lane issues the copies
      if (elect_one()) {
        tma_prefetch_desc(&tmAh);
        tma_prefetch_desc(&tmBh);
        if (SPLIT) {
          tma_prefetch_desc(&tmAl);
          tma_prefetch_desc(&tmBl);
        }
      }
      __syncwarp();
      if (RESB && elect_one()) {  // resident weights: the whole B panel of this CTA's (fixed) n-tile, loaded once
        const int nres = (static_cast<int>(blockIdx.x) % n_tiles) * BN;
        for (int kb = 0; kb < nkb; ++kb) {
          mbar_expect_tx(&fullB[kb], G::kBTile);
          tma_load_2d(sB + kb * G::kBTile, &tmBh, &fullB[kb], kb * KB_COLS, nres);
          if (SPLIT) tma_load_2d(sB + kb * G::kBTile + G::kBPlane, &tmBl, &fullB[kb], kb * KB_COLS, nres);
        }
      }
      __syncwarp();
      uint32_t itA = 0, itB = 0;
      for (int w = blockIdx.x; w < total; w += gridDim.x) {
        int n0;
        const TileCoord tc = tile_coord(w, n0);
        if (!epi.tile_active(tc)) continue;
        const int b_off = epi.b_row_offset(tc);
        const int outer = outer_n;
        if (elect_one()) {  // pull the A operand of the tile this CTA processes two iterations from now into L2
          const int wp = w + 2 * static_cast<int>(gridDim.x);
          if (wp < total) {
            int n0p;
            const TileCoord tp = tile_coord(wp, n0p);
            if ((ISCONV || n0p == 0) && epi.tile_active(tp)) {
              for (int o = 0; o < outer; ++o) {
                if (ISCONV) {
                  const int dx = o / cinb, cb = o - dx * cinb;
                  if (dx != 1) continue;  // the three dx boxes overlap: the centre one plus neighbours' halos cover them
                  tma_prefetch_4d(&tmAh, cb * 64, tp.x0 - 1, tp.y0 - 1, tp.b);
                  if (SPLIT) tma_prefetch_4d(&tmAl, cb * 64, tp.x0 - 1, tp.y0 - 1, tp.b);
                  tma_prefetch_4d(&tmAh, cb * 64, tp.x0 + 1, tp.y0 - 1, tp.b);
                  if (SPLIT) tma_prefetch_4d(&tmAl, cb * 64, tp.x0 + 1, tp.y0 - 1, tp.b);
                } else {
                  tma_prefetch_2d(&tmAh, o * KB_COLS, tp.m0);
                  if (SPLIT) tma_prefetch_2d(&tmAl, o * KB_COLS, tp.m0);
                }
              }
            }
          }
        }
        __syncwarp();
        for (int o = 0; o < outer; ++o) {
          const int s = itA % SA;
          mbar_wait(&emptyA[s], ((itA / SA) & 1) ^ 1);
          uint8_t* st = sA + s * G::kAStage;
          if (elect_one()) {
            mbar_expect_tx(&fullA[s], G::kATx);
            if (ISCONV) {
              const int dx = o / cinb, cb = o - dx * cinb;
              tma_load_4d(st, &tmAh, &fullA[s], cb * 64, tc.x0 + dx - 1, tc.y0 - 1, tc.b);
              if (SPLIT) tma_load_4d(st + G::kABox, &tmAl, &fullA[s], cb * 64, tc.x0 + dx - 1, tc.y0 - 1, tc.b);
            } else {
              tma_load_2d(st, &tmAh, &fullA[s], o * KB_COLS, tc.m0);
              if (SPLIT) tma_load_2d(st + G::kABox, &tmAl, &fullA[s], o * KB_COLS, tc.m0);
            }
          }
          __syncwarp();
          ++itA;
          if (!RESB) {
            for (int dy = 0; dy < inner_n; ++dy) {
              const int kb = kb_of(o, dy);
              const int sb = itB % SB;
              mbar_wait(&emptyB[sb], ((itB / SB) & 1) ^ 1);
              uint8_t* bt = sB + sb * G::kBTile;
              if (elect_one()) {
                mbar_expect_tx(&fullB[sb], G::kBTile);
                tma_load_2d(bt, &tmBh, &fullB[sb], kb * KB_COLS, n0 + b_off);
                if (SPLIT) tma_load_2d(bt + G::kBPlane, &tmBl, &fullB[sb], kb * KB_COLS, n0 + b_off);
              }
              __syncwarp();
              ++itB;
            }
          }
        }
      }
    }
  } else {  // ---------------- consumer warpgroup wg: rows 64 wg .. 64 wg + 63 of every tile
    setmaxnreg_inc<kConsumerRegs>();
    const int wg = warp >> 2, w4 = warp & 3;
    // A rows of this warpgroup start 64 MH rows into the stage: 8 MH swizzle atoms of 8 rows, atom-aligned
    const uint32_t a_wg = static_cast<uint32_t>(wg * 64 * MH * G::kRowB);
    float* stg = staging + wg * G::kStgFloats;
    uint32_t itA = 0, itB = 0;
    bool resb_ready = false;
    float acc[MH][BN / 2];
    for (int w = blockIdx.x; w < total; w += gridDim.x) {
      int n0;
      const TileCoord tc = tile_coord(w, n0);
      if (!epi.tile_active(tc)) continue;
      const int outer = outer_n;
      for (int o = 0; o < outer; ++o) {
        const int s = itA % SA;
        mbar_wait(&fullA[s], (itA / SA) & 1);
        const uint32_t a_base = smem_u32(sA + s * G::kAStage) + a_wg;
        int sb0 = 0;
#pragma unroll
        for (int dy = 0; dy < inner_n; ++dy) {
          const int kb = kb_of(o, dy);
          uint32_t b_base;
          if (RESB) {
            if (!resb_ready) mbar_wait(&fullB[kb], 0);
            b_base = smem_u32(sB + kb * G::kBTile);
          } else {
            const int sb = (itB + dy) % SB;
            if (dy == 0) sb0 = sb;
            mbar_wait(&fullB[sb], ((itB + dy) / SB) & 1);
            b_base = smem_u32(sB + sb * G::kBTile);
          }
          const uint32_t a_tap = a_base + (ISCONV ? dy * (kConvTW * 128) : 0);
          const uint64_t b_h = make_sdesc(b_base, kSbo, kLayout), b_l = make_sdesc(b_base + G::kBPlane, kSbo, kLayout);
          wgmma_fence();
#pragma unroll
          for (int k16 = 0; k16 < KSTEPS; ++k16) {
#pragma unroll
            for (int h = 0; h < MH; ++h) {  // every accumulator sees hi*hi, hi*lo, lo*hi per k16 step, whatever MH is
              const uint32_t a_hh = a_tap + h * 64 * G::kRowB;
              const uint64_t a_h = make_sdesc(a_hh, kSbo, kLayout), a_l = make_sdesc(a_hh + G::kABox, kSbo, kLayout);
              Wgmma<BN>::ss(acc[h], sdesc_advance_k(a_h, k16), sdesc_advance_k(b_h, k16), (o | dy | k16) != 0);
              if (SPLIT) {
                Wgmma<BN>::ss(acc[h], sdesc_advance_k(a_h, k16), sdesc_advance_k(b_l, k16), 1);
                Wgmma<BN>::ss(acc[h], sdesc_advance_k(a_l, k16), sdesc_advance_k(b_h, k16), 1);
              }
            }
          }
          if (EARLY_B) wgmma_commit();
        }
        if (EARLY_B) {  // retire the dy groups in order, handing each weight tile back to the producer as soon as it is read
          wgmma_wait<2>();
          if (lane == 0) mbar_arrive(&emptyB[sb0]);
          wgmma_wait<1>();
          if (lane == 0) mbar_arrive(&emptyB[(sb0 + 1) % SB]);
          wgmma_wait<0>();
        } else {
          wgmma_commit();
          wgmma_wait<0>();
        }
#pragma unroll
        for (int h = 0; h < MH; ++h) wgmma_fence_regs(acc[h]);
        if (lane == 0) {  // this warp is done with the stage and its (remaining) B tiles
          mbar_arrive(&emptyA[s]);
          if (!RESB)
            for (int dy = EARLY_B ? 2 : 0; dy < inner_n; ++dy) mbar_arrive(&emptyB[(sb0 + dy) % SB]);
        }
        ++itA;
        if (!RESB) itB += inner_n;
      }
      resb_ready = true;  // every resident tile has been waited for once
      // epilogue: accumulator -> staging (mode 2: kStgCols2 columns at a time, otherwise 64) -> thread r = row of the tile, 32
      // consecutive columns
      const int rr = 32 * (w4 & 1) + lane, cq = 32 * (w4 >> 1);
      const int lr = 16 * w4 + (lane >> 2);
      if constexpr (CONV == 2) {
        // per 64-row half: stage the 64 columns chunk by chunk; warps 0, 1 collect columns 0-31, warps 2, 3 columns 32-63, then all
        // four warps run the epilogue
        constexpr int NCH = BN / kStgCols2, PER = 32 / kStgCols2;  // chunks per half, chunks per thread's 32 columns
#pragma unroll
        for (int h = 0; h < MH; ++h) {
          float v[32];
#pragma unroll
          for (int c = 0; c < NCH; ++c) {
#pragma unroll
            for (int i = c * kStgCols2 / 8; i < (c + 1) * kStgCols2 / 8; ++i) {
              const int col = 8 * i - c * kStgCols2 + 2 * (lane & 3);
              *reinterpret_cast<float2*>(stg + lr * kStgPitch2 + col) = make_float2(acc[h][4 * i], acc[h][4 * i + 1]);
              *reinterpret_cast<float2*>(stg + (lr + 8) * kStgPitch2 + col) = make_float2(acc[h][4 * i + 2], acc[h][4 * i + 3]);
            }
            named_bar_sync(1 + wg, 128);
            if ((w4 >> 1) == c / PER) {
#pragma unroll
              for (int q = 0; q < kStgCols2 / 4; ++q) {
                const float4 x = *reinterpret_cast<const float4*>(stg + rr * kStgPitch2 + 4 * q);
                const int j = (c % PER) * kStgCols2 + 4 * q;
                v[j] = x.x, v[j + 1] = x.y, v[j + 2] = x.z, v[j + 3] = x.w;
              }
            }
            named_bar_sync(1 + wg, 128);
          }
          epi(tc, 128 * wg + 64 * h + rr, n0 + cq, v, nullptr);
        }
      } else {
#pragma unroll
        for (int c0 = 0; c0 < BN; c0 += kStgCols) {
#pragma unroll
          for (int i = c0 / 8; i < (c0 + kStgCols) / 8; ++i) {
            const int col = 8 * i - c0 + 2 * (lane & 3);
            *reinterpret_cast<float2*>(stg + lr * kStgPitch + col) = make_float2(acc[0][4 * i], acc[0][4 * i + 1]);
            *reinterpret_cast<float2*>(stg + (lr + 8) * kStgPitch + col) = make_float2(acc[0][4 * i + 2], acc[0][4 * i + 3]);
          }
          named_bar_sync(1 + wg, 128);
          float v[32];
#pragma unroll
          for (int q = 0; q < 8; ++q) {
            const float4 x = *reinterpret_cast<const float4*>(stg + rr * kStgPitch + cq + 4 * q);
            v[4 * q] = x.x, v[4 * q + 1] = x.y, v[4 * q + 2] = x.z, v[4 * q + 3] = x.w;
          }
          named_bar_sync(1 + wg, 128);
          epi(tc, 64 * wg + rr, n0 + c0 + cq, v, stg + w4 * kScratchFloats);
          named_bar_sync(1 + wg, 128);
        }
      }
    }
    if (RESB && !resb_ready)  // no active tile: still drain the resident-weight loads before the CTA exits
      for (int kb = 0; kb < nkb; ++kb) mbar_wait(&fullB[kb], 0);
  }
}

// ------------------------------------------------------------------ launch
struct TcOperands {
  CUtensorMap Ah, Al, Bh, Bl;
};

template <int BN, bool SPLIT, int CONV, bool RESB, class Epi>
int launch_pers(dimb_ctx* ctx, cudaStream_t st, const TcOperands& ops, const GemmArgs& g, const Epi& epi, int m_tiles, int n_tiles,
                const PersCfg& cfg, int grid) {
  auto kern = tc_gemm_pers_kernel<BN, SPLIT, CONV, RESB, Epi>;
  DIMB_TRY(dimb_func_smem(ctx, kern, cfg.smem_bytes));
  kern<<<grid, kGemmThreads, cfg.smem_bytes, st>>>(ops.Ah, ops.Al, ops.Bh, ops.Bl, g, epi, m_tiles, n_tiles, cfg.sa, cfg.sb);
  DIMB_LAUNCH_CHECK(ctx);
  return DIMB_OK;
}

// ring depths from the 227 KB shared-memory budget; resb: keep all nkb B tiles resident
template <int BN, bool SPLIT, int CONV>
PersCfg pers_config(int nkb, bool resb) {
  using G = PersGeom<BN, SPLIT, CONV>;
  PersCfg c{};
  c.nkb_total = nkb;
  int budget = G::kBudget;
  if (resb) {
    budget -= nkb * G::kBTile;
    c.sb = 0;
    c.sa = budget / G::kAStage;
  } else if (CONV == 2) {
    // the consumer hands each weight tile back as soon as its dy's MMAs retire, so three B slots already let the producer refill
    // while the stage computes: double-buffer A first, then every B slot that fits (EXACT: 2 A stages, 4 B slots)
    c.sa = budget >= 2 * G::kAStage + 3 * G::kBTile ? 2 : 1;
    c.sb = (budget - c.sa * G::kAStage) / G::kBTile;
  } else {
    // conv consumes 3 B tiles per A stage: give B the deeper ring
    const int per = CONV == 1 ? 3 : 1;
    const int unit = G::kAStage + per * G::kBTile;
    int n = budget / unit;
    if (n < 1) n = 1;
    c.sa = n;
    c.sb = per * n;
    while (c.sa * G::kAStage + (c.sb + 1) * G::kBTile <= budget) ++c.sb;
    while ((c.sa + 1) * G::kAStage + c.sb * G::kBTile <= budget) ++c.sa;
  }
  if (c.sa > 8) c.sa = 8;
  if (c.sb > 12) c.sb = 12;
  c.smem_bytes = c.sa * G::kAStage + (resb ? nkb : c.sb) * G::kBTile + 1024 + 1024 + G::kStgBytes;
  return c;
}

// Launch plan of one persistent-kernel call: resident weights or not, ring depths, shared memory and grid.  Host only, so that
// the plan of every call site can be checked without a GPU (dimb_selftest_gemm_plan).
struct PersPlan {
  bool resb;
  PersCfg cfg;
  int grid;
};

template <int BN, bool SPLIT, int CONV>
PersPlan pers_plan(bool const_b, int num_kb, int m_tiles, int n_tiles, int num_sms) {
  using G = PersGeom<BN, SPLIT, CONV>;
  // resident weights only where a CTA keeps seeing the same B panel (its tiles share the n-tile: the persistent
  // stride = grid size must be a multiple of n_tiles) and >= 2 A stages still fit
  const int total = m_tiles * n_tiles, grid = total < num_sms ? total : num_sms;
  const bool fits = const_b && (G::kBudget - num_kb * G::kBTile) >= 2 * G::kAStage;
  // a grid that is a multiple of n_tiles pins every CTA to one B panel; when the SM count is not such a multiple (the brute-force
  // matcher: 32 panels of 256 descriptors), giving up a few SMs is far cheaper than re-streaming B from L2 for every tile
  int rgrid = grid;
  if (fits && grid % n_tiles != 0 && n_tiles <= grid) rgrid = grid / n_tiles * n_tiles;
  const bool resb = fits && (rgrid % n_tiles == 0) && rgrid * 8 >= grid * 7;
  return PersPlan{resb, pers_config<BN, SPLIT, CONV>(num_kb, resb), resb ? rgrid : grid};
}

template <int BN, bool SPLIT, int CONV, class Epi>
int launch_pers_auto(dimb_ctx* ctx, cudaStream_t st, const TcOperands& ops, const GemmArgs& g, const Epi& epi, int m_tiles, int n_pad) {
  const int n_tiles = n_pad / BN;
  const PersPlan p = pers_plan<BN, SPLIT, CONV>(Epi::kConstB, g.num_kb, m_tiles, n_tiles, ctx->num_sms);
  if (p.resb) return launch_pers<BN, SPLIT, CONV, true, Epi>(ctx, st, ops, g, epi, m_tiles, n_tiles, p.cfg, p.grid);
  return launch_pers<BN, SPLIT, CONV, false, Epi>(ctx, st, ops, g, epi, m_tiles, n_tiles, p.cfg, p.grid);
}

// n_pad: output columns rounded up to a multiple of BN (B operand rows beyond N read as zero via TMA OOB fill).
// CONV 1 / 2: ops.Ah/Al must be NHWC maps with a (ConvTile<CONV>::TH + 2) x kConvTW box (see dimb_tmap_nhwc callers).
template <int BN, int CONV, class Epi>
int launch_gemm(dimb_ctx* ctx, cudaStream_t st, const TcOperands& ops, const GemmArgs& g, const Epi& epi, int m_tiles, int n_pad,
                const char* tag = "gemm", int force_split = -1) {
  // force_split: -1 = by the context's precision; 0 / 1 = operands known to be exactly fp16 (lo planes are zero: one MMA per
  // product IS exact) / to need the split regardless of the precision mode
  if (m_tiles <= 0) return DIMB_OK;
  ProfScope prof(ctx, st, tag);
  const bool exact = force_split < 0 ? ctx->precision == DIMB_PRECISION_EXACT : force_split != 0;
  if (exact) return launch_pers_auto<BN, true, CONV, Epi>(ctx, st, ops, g, epi, m_tiles, n_pad);
  return launch_pers_auto<BN, false, CONV, Epi>(ctx, st, ops, g, epi, m_tiles, n_pad);
}

// ------------------------------------------------------------------ generic epilogues
// Every functor: tile_active(tc) (CTA-uniform) and operator()(tc, r, n, v): row r of the tile, v[j] = C[row][n+j].
// Optional hooks (defaults in EpiBase): m0_of(t) maps the tile index to its first A row; b_row_offset(tc) shifts
// the B rows a tile multiplies with (stacked per-layer weights, or "the other image" for similarity matrices).
struct EpiBase {
  static constexpr bool kConstB = true;       // b_row_offset() == 0 for every tile (B panel may stay resident)
  static constexpr bool kScratch = true;      // operator() uses its per-warp scratch (conv mode 2 has none to give)
  __device__ int m0_of(int t) const { return t * kTileM; }
  __device__ int b_row_offset(const TileCoord&) const { return 0; }
  __device__ bool tile_active(const TileCoord&) const { return true; }
};

// v[j] = chunk[lane][j]  ->  f[it] = chunk[it*4 + lane/8][(lane%8)*4 .. +3]   (it = 0..7)
__device__ __forceinline__ void warp_transpose32(const float (&v)[32], float* sc, float4 (&f)[8]) {
  const int lane = threadIdx.x & 31;
  float4* dst = reinterpret_cast<float4*>(sc + lane * kScratchPitch);
#pragma unroll
  for (int q = 0; q < 8; ++q) dst[q ^ (lane & 7)] = make_float4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]);
  __syncwarp();
#pragma unroll
  for (int it = 0; it < 8; ++it) {
    const int row = it * 4 + (lane >> 3);
    f[it] = *reinterpret_cast<const float4*>(sc + row * kScratchPitch + (((lane & 7) ^ (row & 7)) << 2));
  }
  __syncwarp();
}
// 4 consecutive values -> 4 halfs hi (+ 4 halfs lo), 8-byte stores
__device__ __forceinline__ void store_split4(__half* hi, __half* lo, const float4& x) {
  __half2 h[2], l[2];
  split2_f32(x.x, x.y, h[0], l[0]);
  split2_f32(x.z, x.w, h[1], l[1]);
  *reinterpret_cast<uint2*>(hi) = *reinterpret_cast<const uint2*>(h);
  if (lo) *reinterpret_cast<uint2*>(lo) = *reinterpret_cast<const uint2*>(l);
}

// 16-byte store of 8 consecutive halfs
__device__ __forceinline__ void store_half8(__half* dst, const __half (&h)[8]) {
  *reinterpret_cast<uint4*>(dst) = *reinterpret_cast<const uint4*>(h);
}

// writes 32 consecutive values as fp16 hi (+ lo) planes; dst pointers must be 16B aligned
__device__ __forceinline__ void store_split32(__half* hi, __half* lo, const float (&v)[32]) {
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    __half2 h[4], l[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) split2_f32(v[q * 8 + 2 * j], v[q * 8 + 2 * j + 1], h[j], l[j]);
    *reinterpret_cast<uint4*>(hi + q * 8) = *reinterpret_cast<const uint4*>(h);
    if (lo) *reinterpret_cast<uint4*>(lo + q * 8) = *reinterpret_cast<const uint4*>(l);
  }
}

// v[j] += bias[n + j] with 8 vector loads (bias + n is 128 B aligned: n is a multiple of 32)
__device__ __forceinline__ void add_bias32(float (&v)[32], const float* __restrict__ bias, int n) {
  const float4* b4 = reinterpret_cast<const float4*>(bias + n);
#pragma unroll
  for (int q = 0; q < 8; ++q) {
    const float4 b = __ldg(b4 + q);
    v[4 * q] += b.x;
    v[4 * q + 1] += b.y;
    v[4 * q + 2] += b.z;
    v[4 * q + 3] += b.w;
  }
}

// fp32 store: out[row][n] = (acc + bias[n]) * scale, columns < n_valid, rows < m_valid.
struct EpiStoreF32 : EpiBase {
  float* out;
  const float* bias;  // may be null
  int ldc, n_valid, m_valid;
  float scale;
  __device__ void operator()(const TileCoord& tc, int r, int n, float (&v)[32], float* sc) const {
    const int lane = r & 31, col = n + (lane & 7) * 4;
    float4 b = make_float4(0.f, 0.f, 0.f, 0.f);
    if (bias && col + 3 < n_valid) b = __ldg(reinterpret_cast<const float4*>(bias + col));  // before the transpose's __syncwarp
    float4 f[8];
    warp_transpose32(v, sc, f);
#pragma unroll
    for (int it = 0; it < 8; ++it) {
      const int row = tc.m0 + (r & ~31) + it * 4 + (lane >> 3);
      if (row >= m_valid) continue;
      float* o = out + static_cast<size_t>(row) * ldc + col;
      if (col + 3 < n_valid && (ldc & 3) == 0) {
        *reinterpret_cast<float4*>(o) = make_float4((f[it].x + b.x) * scale, (f[it].y + b.y) * scale, (f[it].z + b.z) * scale,
                                                    (f[it].w + b.w) * scale);
      } else {
        const float e[4] = {f[it].x, f[it].y, f[it].z, f[it].w};
        for (int j = 0; j < 4; ++j)
          if (col + j < n_valid) o[j] = (e[j] + (bias ? bias[col + j] : 0.f)) * scale;
      }
    }
  }
};

// fp16 hi/lo store: out[row][col_off + n] = (acc + bias[n]) * scale   (n_valid multiple of 32)
struct EpiStoreSplit : EpiBase {
  __half *hi, *lo;  // lo may be null (FAST)
  const float* bias;
  int ldc, col_off, n_valid, m_valid;
  float scale;
  __device__ void operator()(const TileCoord& tc, int r, int n, float (&v)[32], float* sc) const {
    const int lane = r & 31, col = n + (lane & 7) * 4;
    const float4 b = (bias && n < n_valid) ? __ldg(reinterpret_cast<const float4*>(bias + col)) : make_float4(0.f, 0.f, 0.f, 0.f);
    float4 f[8];
    warp_transpose32(v, sc, f);
    if (n >= n_valid) return;
#pragma unroll
    for (int it = 0; it < 8; ++it) {
      const int row = tc.m0 + (r & ~31) + it * 4 + (lane >> 3);
      if (row >= m_valid) continue;
      const size_t off = static_cast<size_t>(row) * ldc + col_off + col;
      store_split4(hi + off, lo ? lo + off : nullptr,
                   make_float4((f[it].x + b.x) * scale, (f[it].y + b.y) * scale, (f[it].z + b.z) * scale, (f[it].w + b.w) * scale));
    }
  }
};
