// common.cu - context, allocation and TMA tensor-map helpers of libdimb200.
#include <map>
#include <mutex>
#include <utility>

#include "common.cuh"

#include <cstdlib>
#include <cstring>

const char* dimb_set_error(dimb_ctx* ctx, const std::string& msg) {
  if (ctx) ctx->last_error = msg;
  return ctx ? ctx->last_error.c_str() : "";
}

void dimb_release(dimb_ctx* ctx, std::vector<void*>& mem) {
  cudaSetDevice(ctx->device);
  cudaDeviceSynchronize();
  for (void* p : mem) cudaFree(p);
  mem.clear();
}

int dimb_scratch(dimb_ctx* ctx, int slot, size_t bytes, void** p) {
  if (slot >= static_cast<int>(ctx->scratch.size())) ctx->scratch.resize(slot + 1);
  dimb_ctx::Scratch& s = ctx->scratch[slot];
  if (s.bytes < bytes) {
    if (s.p) {
      DIMB_CUDA_OK(ctx, cudaDeviceSynchronize());
      DIMB_CUDA_OK(ctx, cudaFree(s.p));
      s.p = nullptr;
      s.bytes = 0;
    }
    const size_t want = bytes + bytes / 4 + 256;
    DIMB_CUDA_OK(ctx, cudaMalloc(&s.p, want));
    s.bytes = want;
  }
  *p = s.p;
  return DIMB_OK;
}

void dimb_free(dimb_ctx* ctx, void* p) {
  if (!p) return;
  std::vector<void*>& list = ctx->owner ? *ctx->owner : ctx->allocs;
  for (size_t i = 0; i < list.size(); ++i)
    if (list[i] == p) {
      list.erase(list.begin() + i);
      break;
    }
  cudaDeviceSynchronize();  // a kernel of an earlier call may still read the buffer
  cudaFree(p);
}

// The attribute belongs to (device, function), not to a context: several contexts on one device (tests with kernel variants, one
// context per stream in a server) share it, so the opt-in is only ever RAISED - a second context asking for less must not lower what the
// first one launches with.  Process-wide table, one mutex; the per-context map is a lock-free fast path.
int dimb_func_smem_raw(dimb_ctx* ctx, const void* fn, int bytes) {
  auto it = ctx->func_smem.find(fn);
  if (it != ctx->func_smem.end() && it->second >= bytes) return DIMB_OK;
  static std::mutex mu;
  static std::map<std::pair<int, const void*>, int> table;
  std::lock_guard<std::mutex> lock(mu);
  int& cur = table[{ctx->device, fn}];
  if (cur < bytes) {
    DIMB_CUDA_OK(ctx, cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
    cur = bytes;
  }
  ctx->func_smem[fn] = cur;
  return DIMB_OK;
}

int dimb_alloc(dimb_ctx* ctx, void** p, size_t bytes, bool zero) {
  *p = nullptr;
  if (bytes == 0) bytes = 16;
  DIMB_CUDA_OK(ctx, cudaMalloc(p, bytes));
  (ctx->owner ? *ctx->owner : ctx->allocs).push_back(*p);
  if (zero) DIMB_CUDA_OK(ctx, cudaMemset(*p, 0, bytes));
  return DIMB_OK;
}

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode(dimb_ctx* ctx) {
  static PFN_encodeTiled fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q);
    if (e != cudaSuccess || q != cudaDriverEntryPointSuccess || !p) {
      dimb_set_error(ctx, "cuTensorMapEncodeTiled not available from the driver");
      return nullptr;
    }
    fn = reinterpret_cast<PFN_encodeTiled>(p);
  }
  return fn;
}

int dimb_tmap_2d(dimb_ctx* ctx, CUtensorMap* out, const __half* base, uint64_t rows, uint64_t cols, uint64_t ld,
                 uint32_t box_rows) {
  PFN_encodeTiled enc = get_encode(ctx);
  if (!enc) return DIMB_ERR_CUDA;
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {ld * sizeof(__half)};
  cuuint32_t box[2] = {64, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<__half*>(base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    dimb_set_error(ctx, "cuTensorMapEncodeTiled(2d) failed: code " + std::to_string(int(r)) + " rows=" +
                            std::to_string(rows) + " cols=" + std::to_string(cols) + " ld=" + std::to_string(ld));
    return DIMB_ERR_CUDA;
  }
  return DIMB_OK;
}

// 2-D map with boxes of 32 halfs (64-byte rows) x box_rows and SWIZZLE_64B: operands of the 32-wide K blocks (gemm.cuh CONV 3)
int dimb_tmap_2d_sw64(dimb_ctx* ctx, CUtensorMap* out, const __half* base, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows) {
  PFN_encodeTiled enc = get_encode(ctx);
  if (!enc) return DIMB_ERR_CUDA;
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {ld * sizeof(__half)};
  cuuint32_t box[2] = {32, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<__half*>(base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    dimb_set_error(ctx, "cuTensorMapEncodeTiled(2d, 64B swizzle) failed: code " + std::to_string(int(r)));
    return DIMB_ERR_CUDA;
  }
  return DIMB_OK;
}

int dimb_tmap_nhwc(dimb_ctx* ctx, CUtensorMap* out, const __half* base, uint64_t n, uint64_t h, uint64_t w, uint64_t c,
                   uint32_t box_h, uint32_t box_w) {
  PFN_encodeTiled enc = get_encode(ctx);
  if (!enc) return DIMB_ERR_CUDA;
  cuuint64_t dims[4] = {c, w, h, n};
  cuuint64_t strides[3] = {c * sizeof(__half), w * c * sizeof(__half), h * w * c * sizeof(__half)};
  cuuint32_t box[4] = {64, box_w, box_h, 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<__half*>(base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    dimb_set_error(ctx, "cuTensorMapEncodeTiled(nhwc) failed: code " + std::to_string(int(r)));
    return DIMB_ERR_CUDA;
  }
  return DIMB_OK;
}

ProfScope::ProfScope(dimb_ctx* c, cudaStream_t s, const char* tag) : ctx(c), st(s) {
  if (!ctx->profile) return;
  int t = -1;
  for (size_t i = 0; i < ctx->prof_tags.size(); ++i)
    if (ctx->prof_tags[i] == tag) t = static_cast<int>(i);
  if (t < 0) {
    ctx->prof_tags.push_back(tag);
    t = static_cast<int>(ctx->prof_tags.size()) - 1;
  }
  dimb_ctx::ProfRec r;
  r.tag = t;
  cudaEventCreate(&r.e0);
  cudaEventCreate(&r.e1);
  cudaEventRecord(r.e0, st);
  ctx->prof_recs.push_back(r);
  idx = static_cast<int>(ctx->prof_recs.size()) - 1;
}
ProfScope::~ProfScope() {
  if (idx >= 0) cudaEventRecord(ctx->prof_recs[idx].e1, st);
}

extern "C" {

int dimb_ctx_profile(dimb_ctx* ctx, int enable) {
  if (!ctx) return DIMB_ERR_ARG;
  cudaDeviceSynchronize();
  for (auto& r : ctx->prof_recs) {
    cudaEventDestroy(r.e0);
    cudaEventDestroy(r.e1);
  }
  ctx->prof_recs.clear();
  ctx->profile = enable ? 1 : 0;
  return DIMB_OK;
}

// JSON object {"tag": [total_ms, launches], ...} of everything recorded since dimb_ctx_profile(ctx, 1)
int dimb_ctx_profile_read(dimb_ctx* ctx, char* buf, size_t n) {
  if (!ctx || !buf || n < 3) return DIMB_ERR_ARG;
  DIMB_CUDA_OK(ctx, cudaDeviceSynchronize());
  std::vector<double> ms(ctx->prof_tags.size(), 0.0);
  std::vector<int> cnt(ctx->prof_tags.size(), 0);
  for (auto& r : ctx->prof_recs) {
    float t = 0.f;
    if (cudaEventElapsedTime(&t, r.e0, r.e1) == cudaSuccess) {
      ms[r.tag] += t;
      cnt[r.tag]++;
    }
  }
  std::string out = "{";
  for (size_t i = 0; i < ms.size(); ++i) {
    if (!cnt[i]) continue;
    if (out.size() > 1) out += ", ";
    out += "\"" + ctx->prof_tags[i] + "\": [" + std::to_string(ms[i]) + ", " + std::to_string(cnt[i]) + "]";
  }
  out += "}";
  if (out.size() + 1 > n) return DIMB_ERR_CAPACITY;
  memcpy(buf, out.c_str(), out.size() + 1);
  return DIMB_OK;
}

// device -> host copy of a library-owned buffer (debug taps / tests: the Python host side has no CUDA runtime of its own)
int dimb_read_dev(dimb_ctx* ctx, void* dst, const void* d_src, size_t bytes) {
  if (!ctx || !dst || !d_src) return DIMB_ERR_ARG;
  DIMB_CUDA_OK(ctx, cudaSetDevice(ctx->device));
  DIMB_CUDA_OK(ctx, cudaDeviceSynchronize());
  DIMB_CUDA_OK(ctx, cudaMemcpy(dst, d_src, bytes, cudaMemcpyDeviceToHost));
  return DIMB_OK;
}

const char* dimb_version(void) { return "dimb200 0.1.0 (sm_90a)"; }

int dimb_ctx_create(int device, dimb_ctx** out) {
  if (!out) return DIMB_ERR_ARG;
  *out = nullptr;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0 || device < 0 || device >= ndev) return DIMB_ERR_CUDA;
  dimb_ctx* ctx = new dimb_ctx();
  ctx->device = device;
  cudaDeviceProp prop;
  if (cudaSetDevice(device) != cudaSuccess || cudaGetDeviceProperties(&prop, device) != cudaSuccess) {
    delete ctx;
    return DIMB_ERR_CUDA;
  }
  if (prop.major != 9) {  // sm_90a cubins only: no compatibility path
    delete ctx;
    return DIMB_ERR_UNSUPPORTED;
  }
  ctx->num_sms = prop.multiProcessorCount;
  const char* lz = getenv("DIMB_ATTN_LAZY");
  if (lz) {  // NaN, inf, out of range or no number at all: keep the default (common.cuh: kAttnLazyMax)
    char* end = nullptr;
    const float v = strtof(lz, &end);
    if (end != lz && v >= 0.f && v <= kAttnLazyMax) ctx->attn_lazy = v;
  }
  const char* k3 = getenv("DIMB_K32");
  if (k3) ctx->k32 = k3[0] == '1';
  const char* b2 = getenv("DIMB_BN256");
  if (b2) ctx->bn256 = b2[0] == '1';
  const char* p = getenv("DIMB_PRECISION");
  if (p && !strcmp(p, "fast")) ctx->precision = DIMB_PRECISION_FAST;
  *out = ctx;
  return DIMB_OK;
}

void dimb_ctx_destroy(dimb_ctx* ctx) {
  if (!ctx) return;
  dimb_release(ctx, ctx->allocs);
  for (auto& s : ctx->scratch) cudaFree(s.p);
  delete ctx;
}

const char* dimb_last_error(dimb_ctx* ctx) { return ctx ? ctx->last_error.c_str() : "null context"; }

int dimb_ctx_set_precision(dimb_ctx* ctx, int precision) {
  if (!ctx || (precision != DIMB_PRECISION_EXACT && precision != DIMB_PRECISION_FAST)) return DIMB_ERR_ARG;
  ctx->precision = precision;
  return DIMB_OK;
}

unsigned long long dimb_ctx_launch_count(dimb_ctx* ctx) { return ctx ? ctx->launches : 0; }

}  // extern "C"
