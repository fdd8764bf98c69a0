// common.cuh - shared host/device utilities of libdimb200 (error handling, context,
// device allocations, fp16 hi/lo split arithmetic, TMA tensor-map encoding).
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <map>
#include <string>
#include <vector>

#include "../../include/dimb200.h"

// ---------------------------------------------------------------- errors
// Largest lazy-rescale threshold of the attention kernel (attention.cuh), in log2 units: the softmax numerators P reach 2^lazy and
// their hi plane is fp16 (largest finite value 65504 < 2^16), so 15 is the last whole threshold that cannot overflow it.
constexpr float kAttnLazyMax = 15.f;
// Opt-in dynamic shared memory per block on sm_90 (cudaDevAttrMaxSharedMemoryPerBlockOptin of the H100).
constexpr int kSmemOptin = 232448;

struct dimb_ctx {
  int device = 0;
  int num_sms = 132;
  int precision = DIMB_PRECISION_EXACT;
  int k32 = 0;            // 32-wide K stages (half-size stages) for the 128 x 256 LightGlue tiles (gemm.cuh CONV 3); DIMB_K32=1
  int bn256 = 0;          // LightGlue q/k projection and FFN0 on 128 x 256 output tiles (DIMB_BN256=1); default 128 x 128: spill-free
  // lazy-rescale threshold of the attention kernel in log2 units (DIMB_ATTN_LAZY; 0 = rescale on every new maximum).  Only finite
  // values in [0, kAttnLazyMax] are taken from the environment, anything else keeps 8: P <= 2^lazy must fit the fp16 hi plane.
  float attn_lazy = 8.f;
  std::string last_error;
  std::vector<void*> allocs;            // device memory owned by the context itself
  std::vector<void*>* owner = nullptr;
  struct Scratch {
    void* p = nullptr;
    size_t bytes = 0;
  };
  std::vector<Scratch> scratch;         // grow-only per-context scratch slots (dimb_scratch), e.g. for dimb_nn_match  // where dimb_alloc records memory right now (an object's list, see OwnerScope)
  // opt-in dynamic shared memory already granted on THIS device, per kernel (the attribute is per device context, so a
  // process-wide static would leave every device after the first without it)
  std::map<const void*, int> func_smem;
  unsigned long long launches = 0;  // kernels launched by this library (bench.py "gpu_launches")
  // optional per-kernel-group CUDA-event profiler (dimb_ctx_profile): tag -> accumulated device time
  int profile = 0;
  struct ProfRec {
    int tag;
    cudaEvent_t e0, e1;
  };
  std::vector<std::string> prof_tags;
  std::vector<ProfRec> prof_recs;
};

// RAII CUDA-event bracket around one kernel (group) on its launching stream; no-op unless profiling is on.
struct ProfScope {
  dimb_ctx* ctx;
  cudaStream_t st;
  int idx = -1;
  ProfScope(dimb_ctx* c, cudaStream_t s, const char* tag);
  ~ProfScope();
};

// Device memory belongs to the handle (dimb_sp / dimb_lg / ...) whose entry point allocated it and is released by
// that handle's destroy; OwnerScope routes dimb_alloc to the handle's list for the duration of one entry point.
struct OwnerScope {
  dimb_ctx* ctx;
  std::vector<void*>* prev;
  OwnerScope(dimb_ctx* c, std::vector<void*>* o) : ctx(c), prev(c->owner) { c->owner = o; }
  ~OwnerScope() { ctx->owner = prev; }
};
void dimb_release(dimb_ctx* ctx, std::vector<void*>& mem);  // synchronises the device, frees every pointer

const char* dimb_set_error(dimb_ctx* ctx, const std::string& msg);

#define DIMB_CUDA_OK(ctx, expr)                                                                         \
  do {                                                                                                  \
    cudaError_t _e = (expr);                                                                            \
    if (_e != cudaSuccess) {                                                                            \
      std::string _m = std::string(#expr) + " failed: " + cudaGetErrorString(_e) + " (" + __FILE__ +    \
                       ":" + std::to_string(__LINE__) + ")";                                            \
      if (_e == cudaErrorMemoryAllocation) _m = "CUDA out of memory. " + _m; /* matcher_base.py:251 */  \
      dimb_set_error(ctx, _m);                                                                          \
      return _e == cudaErrorMemoryAllocation ? DIMB_ERR_OOM : DIMB_ERR_CUDA;                            \
    }                                                                                                   \
  } while (0)

#define DIMB_TRY(expr)            \
  do {                            \
    int _r = (expr);              \
    if (_r != DIMB_OK) return _r; \
  } while (0)

#define DIMB_LAUNCH_CHECK(ctx)                  \
  do {                                          \
    (ctx)->launches++;                          \
    DIMB_CUDA_OK(ctx, cudaGetLastError());      \
  } while (0)

int dimb_alloc(dimb_ctx* ctx, void** p, size_t bytes, bool zero = true);
// cudaFree a pointer dimb_alloc handed out and drop it from its owner list (buffers re-allocated at a larger capacity)
void dimb_free(dimb_ctx* ctx, void* p);
// cudaFuncAttributeMaxDynamicSharedMemorySize >= bytes for `fn` on ctx's device (cached per context)
int dimb_func_smem_raw(dimb_ctx* ctx, const void* fn, int bytes);
template <class F>
int dimb_func_smem(dimb_ctx* ctx, F* fn, int bytes) {
  return dimb_func_smem_raw(ctx, reinterpret_cast<const void*>(fn), bytes);
}
// slot-indexed scratch that survives across calls and only ever grows (no cudaMalloc/cudaFree in steady state)
int dimb_scratch(dimb_ctx* ctx, int slot, size_t bytes, void** p);

template <class T>
int dimb_alloc_t(dimb_ctx* ctx, T** p, size_t n, bool zero = true) {
  return dimb_alloc(ctx, reinterpret_cast<void**>(p), n * sizeof(T), zero);
}

// ---------------------------------------------------------------- fp16 hi/lo split
// x ~= hi + lo with hi = fp16(x), lo = fp16(x - hi): ~22 significant bits.  Three fp16 MMAs
// (hi*hi + hi*lo + lo*hi, fp32 accumulate) then reproduce an fp32 product to ~2^-22 (SURVEY App. C).
__device__ __forceinline__ void split_f32(float x, __half& hi, __half& lo) {
  x = fminf(fmaxf(x, -65504.f), 65504.f);  // keep padding/garbage finite: inf * 0 would poison MMAs
  hi = __float2half_rn(x);
  lo = __float2half_rn(x - __half2float(hi));
}
__device__ __forceinline__ float join_f16(__half hi, __half lo) { return __half2float(hi) + __half2float(lo); }
// Packed variant for kernel-produced values (finite, |x| < 65504): one F2FP per pair, no clamp.
__device__ __forceinline__ void split2_f32(float a, float b, __half2& hi, __half2& lo) {
  hi = __floats2half2_rn(a, b);
  const float2 f = __half22float2(hi);
  lo = __floats2half2_rn(a - f.x, b - f.y);
}

// ---------------------------------------------------------------- first argmax with torch.max semantics
// (v, i) takes the place of the running best (bv, bi): NaN ranks above every number (the first NaN wins), then the larger value, then
// the smaller index.  Starting from (-INFINITY, INT_MAX), a row of -inf therefore yields its first index and a row holding a NaN the
// first NaN, so every index an argmax writes lies inside the row; finite rows give the first maximum, as a plain v > bv scan does.
__device__ __forceinline__ bool argmax_takes(float v, int i, float bv, int bi) {
  const bool vn = isnan(v), bn = isnan(bv);
  if (vn || bn) return vn && (!bn || i < bi);
  return v > bv || (v == bv && i < bi);
}

__host__ __device__ inline int ceil_div(int a, int b) { return (a + b - 1) / b; }
__host__ __device__ inline int round_up(int a, int b) { return ceil_div(a, b) * b; }

// ---------------------------------------------------------------- TMA tensor maps (host)
// 2D fp16 row-major [rows][cols] (pitch ld elements), box = [box_rows][64], SWIZZLE_128B, OOB -> 0.
int dimb_tmap_2d(dimb_ctx* ctx, CUtensorMap* out, const __half* base, uint64_t rows, uint64_t cols, uint64_t ld,
                 uint32_t box_rows);
// 4D fp16 NHWC activation [n][h][w][c], box = [1][box_h][box_w][64], SWIZZLE_128B, OOB -> 0 (conv zero padding).
int dimb_tmap_2d_sw64(dimb_ctx* ctx, CUtensorMap* out, const __half* base, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows);
int dimb_tmap_nhwc(dimb_ctx* ctx, CUtensorMap* out, const __half* base, uint64_t n, uint64_t h, uint64_t w, uint64_t c,
                   uint32_t box_h, uint32_t box_w);
