// conv3x3.cuh - the SuperPoint convolutions on the persistent tensor-core kernel (gemm.cuh CONV 1 for 3x3, plain GEMM for 1x1):
// weight layout, bias + ReLU (+ 2x2 max pool) epilogue and launch.  Shared by superpoint.cu and the self-test library, so that the
// self-test runs the production layout, tensor maps and epilogue.
#pragma once
#include <vector>

#include "gemm.cuh"

namespace {

// CTA tile width (output channels) of a SuperPoint convolution: 64 for the 64-channel layers, 128 otherwise.  The weight tensor
// maps are built with this box and run_conv3 must be instantiated with the same BN.
constexpr int conv_bn(int cout) { return cout == 64 ? 64 : 128; }

// ------------------------------------------------------------------ epilogue: conv bias + ReLU (+2x2 max pool) -> NHWC hi/lo
template <bool POOL>
struct EpiConvRelu : EpiBase {
  static constexpr bool kScratch = false;
  static constexpr int TW = kConvTW;  // pixels per tile row (both tile shapes)
  __half *hi, *lo;
  const float* bias;
  int H, W;      // conv resolution
  int Ho, Wo;    // output resolution (H/2, W/2 if POOL)
  int C;         // output channels
  __device__ void operator()(const TileCoord& tc, int r, int n, float (&v)[32], float*) const {
    const int y = tc.y0 + r / TW, x = tc.x0 + r % TW;
    add_bias32(v, bias, n);
#pragma unroll
    for (int j = 0; j < 32; ++j) v[j] = fmaxf(v[j], 0.f);
    int oy = y, ox = x;
    bool write = (y < H) && (x < W);
    if (POOL) {
      // lane = (row % (32 / TW)) * TW + col: the 2x2 window lives in lanes l, l^1, l^TW (gemm.cuh tile shapes)
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        float t = fmaxf(v[j], __shfl_xor_sync(0xffffffffu, v[j], 1));
        v[j] = fmaxf(t, __shfl_xor_sync(0xffffffffu, t, TW));
      }
      oy = y >> 1;
      ox = x >> 1;
      write = ((y & 1) == 0) && ((x & 1) == 0) && (oy < Ho) && (ox < Wo);
    }
    if (!write) return;
    const size_t off = ((static_cast<size_t>(tc.b) * Ho + oy) * Wo + ox) * C + n;
    store_split32(hi + off, lo ? lo + off : nullptr, v);
  }
};

struct ConvLayer {
  int cin, cout;
  __half *wh = nullptr, *wl = nullptr;  // [cout_pad][9*cin] (3x3) or [cout_pad][cin] (1x1)
  float* bias = nullptr;                // [cout_pad]
  int cout_pad, k;
  CUtensorMap tmBh, tmBl;
};

int upload_split(dimb_ctx* ctx, const std::vector<float>& m, __half** hi, __half** lo) {
  std::vector<__half> h(m.size()), l(m.size());
  for (size_t i = 0; i < m.size(); ++i) {
    h[i] = __float2half_rn(m[i]);
    l[i] = __float2half_rn(m[i] - __half2float(h[i]));
  }
  DIMB_TRY(dimb_alloc_t(ctx, hi, m.size(), false));
  DIMB_TRY(dimb_alloc_t(ctx, lo, m.size(), false));
  DIMB_CUDA_OK(ctx, cudaMemcpy(*hi, h.data(), m.size() * sizeof(__half), cudaMemcpyHostToDevice));
  DIMB_CUDA_OK(ctx, cudaMemcpy(*lo, l.data(), m.size() * sizeof(__half), cudaMemcpyHostToDevice));
  return DIMB_OK;
}

// OIHW fp32 -> [cout_pad][tap*cin + c]
int make_conv_layer(dimb_ctx* ctx, ConvLayer& L, const float* w, const float* b, int cout, int cin, int ks, int bn) {
  L.cin = cin;
  L.cout = cout;
  L.cout_pad = round_up(cout, bn);
  L.k = ks * ks * cin;
  std::vector<float> m(static_cast<size_t>(L.cout_pad) * L.k, 0.f), bias(L.cout_pad, 0.f);
  for (int o = 0; o < cout; ++o) {
    bias[o] = b[o];
    for (int c = 0; c < cin; ++c)
      for (int t = 0; t < ks * ks; ++t) m[static_cast<size_t>(o) * L.k + t * cin + c] = w[(static_cast<size_t>(o) * cin + c) * ks * ks + t];
  }
  DIMB_TRY(upload_split(ctx, m, &L.wh, &L.wl));
  DIMB_TRY(dimb_alloc_t(ctx, &L.bias, L.cout_pad, false));
  DIMB_CUDA_OK(ctx, cudaMemcpy(L.bias, bias.data(), bias.size() * sizeof(float), cudaMemcpyHostToDevice));
  DIMB_TRY(dimb_tmap_2d(ctx, &L.tmBh, L.wh, L.cout_pad, L.k, L.k, bn));
  DIMB_TRY(dimb_tmap_2d(ctx, &L.tmBl, L.wl, L.cout_pad, L.k, L.k, bn));
  return DIMB_OK;
}

// tiles of a 3x3 conv over B images of H x W (gemm.cuh CONV 1: 8 x 16 pixels per tile, CONV 2: 16 x 16)
inline int conv_m_tiles(int B, int H, int W, int conv = 1) {
  return B * ceil_div(W, kConvTW) * ceil_div(H, conv == 2 ? kConvTH2 : kConvTH);
}

// Tile shape (gemm.cuh CONV mode) of a 3x3 conv launch.  In EXACT the weights of the 64-channel layers do not fit next to the
// A stages, so every tile streams all nine weight tiles from L2: 16 x 16 tiles cut the bytes fetched per output pixel from 2112 to
// 1440.  FAST keeps those weights resident, and the taller tile still pays off there: fewer halo rows and half the per-tile
// overheads per pixel (conv1b / conv2a / conv2b 1.20 / 1.02 / 1.36 x faster at the bench shapes, DESIGN.md section 4).  They are
// used wherever they still give every SM at least two tiles (fewer, larger tiles would idle SMs on small inputs).
inline int conv_mode(int cout, int B, int H, int W, int num_sms) {
  return conv_bn(cout) == 64 && conv_m_tiles(B, H, W, 2) >= 2 * num_sms ? 2 : 1;
}

// run_conv3 on tiles of one shape (CONV 1 or 2)
template <int BN, bool POOL, int CONV>
int run_conv3_tiles(dimb_ctx* ctx, cudaStream_t st, const ConvLayer& L, const __half* inh, const __half* inl, __half* outh,
                    __half* outl, int B, int H, int W, const char* tag) {
  static_assert(CONV == 1 || (CONV == 2 && BN == 64), "16 x 16 tiles are instantiated for the 64-channel layers only");
  const bool exact = ctx->precision == DIMB_PRECISION_EXACT;
  TcOperands ops;
  GemmArgs g{};
  g.cin_blocks = L.cin / 64;
  g.H = H;
  g.W = W;
  g.N = L.cout;
  auto fill = [&](auto& epi) {
    epi.hi = outh;
    epi.lo = exact ? outl : nullptr;
    epi.bias = L.bias;
    epi.H = H;
    epi.W = W;
    epi.Ho = POOL ? H / 2 : H;
    epi.Wo = POOL ? W / 2 : W;
    epi.C = L.cout;
  };
  // gemm.cuh CONV 1 / 2: one (TH+2)-row halo box per dx serves the three dy taps
  constexpr int TH = ConvTile<CONV>::TH;
  DIMB_TRY(dimb_tmap_nhwc(ctx, &ops.Ah, inh, B, H, W, L.cin, TH + 2, kConvTW));
  DIMB_TRY(dimb_tmap_nhwc(ctx, &ops.Al, inl, B, H, W, L.cin, TH + 2, kConvTW));
  ops.Bh = L.tmBh;
  ops.Bl = L.tmBl;
  g.num_kb = 9 * g.cin_blocks;
  g.tiles_x = ceil_div(W, kConvTW);
  g.tiles_y = ceil_div(H, TH);
  EpiConvRelu<POOL> epi;
  fill(epi);
  return launch_gemm<BN, CONV>(ctx, st, ops, g, epi, conv_m_tiles(B, H, W, CONV), L.cout_pad, tag);
}

// 3x3 conv (zero padding 1) + bias + ReLU (+ 2x2 max pool) of NHWC hi/lo activations [B][H][W][cin] -> [B][Ho][Wo][cout], on the
// tile shape conv_mode picks.  Both shapes give bitwise the same output: every element sees the same MMA sequence.
template <int BN, bool POOL>
int run_conv3(dimb_ctx* ctx, cudaStream_t st, const ConvLayer& L, const __half* inh, const __half* inl, __half* outh, __half* outl,
              int B, int H, int W, const char* tag) {
  if constexpr (BN == 64) {
    if (conv_mode(L.cout, B, H, W, ctx->num_sms) == 2)
      return run_conv3_tiles<BN, POOL, 2>(ctx, st, L, inh, inl, outh, outl, B, H, W, tag);
  }
  return run_conv3_tiles<BN, POOL, 1>(ctx, st, L, inh, inl, outh, outl, B, H, W, tag);
}

}  // namespace
