// Host-side helpers shared by every entry point: error string, device query, TMA tensor maps.
#include "common.cuh"

#include <stdlib.h>
#include <unordered_map>

#include <cudaTypedefs.h>
#include <stdarg.h>
#include <string.h>

namespace oasr {

static thread_local char g_err[512] = "";

void set_last_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int num_sms() {
  static int cached = 0;
  if (cached == 0) {
    int dev = 0, n = 0;
    if (cudaGetDevice(&dev) == cudaSuccess &&
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && n > 0)
      cached = n;
    else
      cached = 132;
  }
  return cached;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                  CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                  CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  if (fn == nullptr) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    // resolved at run time so the library links without libcuda (it is built on a GPU-less box)
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

static CUtensorMapDataType dtype_of(int elt_bytes, bool fp16) {
  if (elt_bytes == 1) return CU_TENSOR_MAP_DATA_TYPE_UINT8;   // fp8 operands (TMA copies bytes; wgmma reads the format)
  if (elt_bytes == 2) return fp16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  return CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
}

// Host-side cache of encoded tensor maps.  A training step encodes ~3000 of them (3-7 per GEMM / attention launch) and the
// same (pointer, shape, stride, box) tuples come back every step because the caching allocator hands out the same blocks;
// a descriptor is a pure function of that tuple, so a hit is a 128-byte copy instead of a driver call.
// OASR_TMAP_CACHE=0 disables it (A/B of the host enqueue time).
namespace {
struct TmapKey {
  uintptr_t base;
  uint64_t d0, d1, d2, s1, s2;
  uint32_t b0, b1, b2;
  int32_t dtype, swz, rank;   // dtype: the CUtensorMapDataType
  bool operator==(const TmapKey& o) const {
    return base == o.base && d0 == o.d0 && d1 == o.d1 && d2 == o.d2 && s1 == o.s1 && s2 == o.s2 && b0 == o.b0 && b1 == o.b1 &&
           b2 == o.b2 && dtype == o.dtype && swz == o.swz && rank == o.rank;
  }
};
struct TmapKeyHash {
  size_t operator()(const TmapKey& k) const {
    uint64_t h = 0x9E3779B97F4A7C15ull;
    auto mix = [&h](uint64_t v) { h ^= v + 0x9E3779B97F4A7C15ull + (h << 6) + (h >> 2); };
    mix(k.base); mix(k.d0); mix(k.d1); mix(k.d2); mix(k.s1); mix(k.s2);
    mix((uint64_t(k.b0) << 32) | k.b1); mix((uint64_t(k.b2) << 32) | uint32_t(k.dtype));
    mix((uint64_t(uint32_t(k.swz)) << 32) | uint32_t(k.rank));
    return static_cast<size_t>(h);
  }
};
bool tmap_cache_enabled() {
  static const bool on = [] { const char* e = getenv("OASR_TMAP_CACHE"); return !(e && e[0] == '0'); }();
  return on;
}
std::unordered_map<TmapKey, CUtensorMap, TmapKeyHash>& tmap_cache() {
  static thread_local std::unordered_map<TmapKey, CUtensorMap, TmapKeyHash> cache;
  return cache;
}
bool tmap_lookup(const TmapKey& k, CUtensorMap* out) {
  if (!tmap_cache_enabled()) return false;
  auto& c = tmap_cache();
  auto it = c.find(k);
  if (it == c.end()) return false;
  *out = it->second;
  return true;
}
void tmap_store(const TmapKey& k, const CUtensorMap& m) {
  if (!tmap_cache_enabled()) return;
  auto& c = tmap_cache();
  if (c.size() >= 16384) c.clear();   // bounded: shapes of a few models / batch sizes fit many times over
  c.emplace(k, m);
}
}  // namespace

int make_tmap_2d(CUtensorMap* out, const void* base, int elt_bytes, uint64_t inner, uint64_t outer,
                 uint64_t row_stride_bytes, uint32_t box_inner, uint32_t box_outer, bool swizzle128, bool fp16) {
  return make_tmap_2d_sw(out, base, elt_bytes, inner, outer, row_stride_bytes, box_inner, box_outer, swizzle128 ? 128 : 0, fp16);
}

int make_tmap_2d_sw(CUtensorMap* out, const void* base, int elt_bytes, uint64_t inner, uint64_t outer,
                    uint64_t row_stride_bytes, uint32_t box_inner, uint32_t box_outer, int swizzle_bytes, bool fp16) {
  EncodeTiledFn enc = get_encode();
  OASR_REQUIRE(enc != nullptr, "cuTensorMapEncodeTiled not available from the driver");
  OASR_REQUIRE((row_stride_bytes & 15) == 0, "tensor map: row stride %llu B not a multiple of 16",
               (unsigned long long)row_stride_bytes);
  OASR_REQUIRE((reinterpret_cast<uintptr_t>(base) & 15) == 0, "tensor map: base not 16-byte aligned");
  const TmapKey key{reinterpret_cast<uintptr_t>(base), inner, outer, 0, row_stride_bytes, 0, box_inner, box_outer, 0,
                    (int32_t)dtype_of(elt_bytes, fp16), swizzle_bytes, 2};
  if (tmap_lookup(key, out)) return OASR_OK;
  cuuint64_t dims[2] = {inner, outer};
  cuuint64_t strides[1] = {row_stride_bytes};
  cuuint32_t box[2] = {box_inner, box_outer};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(out, dtype_of(elt_bytes, fp16), 2, const_cast<void*>(base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE,
                   swizzle_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B
                                        : (swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_NONE),
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  OASR_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(2d) failed: CUresult %d (inner=%llu outer=%llu stride=%llu box=%ux%u)",
               (int)r, (unsigned long long)inner, (unsigned long long)outer,
               (unsigned long long)row_stride_bytes, box_inner, box_outer);
  tmap_store(key, *out);
  return OASR_OK;
}

int make_tmap_3d(CUtensorMap* out, const void* base, int elt_bytes, uint64_t d0, uint64_t d1, uint64_t d2,
                 uint64_t stride1_bytes, uint64_t stride2_bytes, uint32_t b0, uint32_t b1, uint32_t b2,
                 bool swizzle128) {
  EncodeTiledFn enc = get_encode();
  OASR_REQUIRE(enc != nullptr, "cuTensorMapEncodeTiled not available from the driver");
  OASR_REQUIRE((stride1_bytes & 15) == 0 && (stride2_bytes & 15) == 0, "tensor map: strides must be multiples of 16 B");
  const TmapKey key{reinterpret_cast<uintptr_t>(base), d0, d1, d2, stride1_bytes, stride2_bytes, b0, b1, b2, (int32_t)dtype_of(elt_bytes, false),
                    swizzle128 ? 128 : 0, 3};
  if (tmap_lookup(key, out)) return OASR_OK;
  cuuint64_t dims[3] = {d0, d1, d2};
  cuuint64_t strides[2] = {stride1_bytes, stride2_bytes};
  cuuint32_t box[3] = {b0, b1, b2};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(out, dtype_of(elt_bytes, false), 3, const_cast<void*>(base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE,
                   swizzle128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  OASR_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(3d) failed: CUresult %d", (int)r);
  tmap_store(key, *out);
  return OASR_OK;
}

}  // namespace oasr

namespace oasr {

void* scratch_alloc(size_t bytes, cudaStream_t st) {
  static int pool_dev = -1;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) { set_last_error("scratch: no device"); return nullptr; }
  if (pool_dev != dev) {   // keep freed scratch in the pool instead of returning it to the driver at every sync
    cudaMemPool_t pool;
    if (cudaDeviceGetDefaultMemPool(&pool, dev) == cudaSuccess) {
      uint64_t keep = UINT64_MAX;
      cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
    }
    pool_dev = dev;
  }
  void* p = nullptr;
  const cudaError_t e = cudaMallocAsync(&p, bytes < 16 ? 16 : bytes, st);
  if (e != cudaSuccess) {
    set_last_error("scratch: cudaMallocAsync(%zu) -> %s", bytes, cudaGetErrorString(e));
    return nullptr;
  }
  return p;
}

void scratch_free(void* p, cudaStream_t st) {
  if (p) cudaFreeAsync(p, st);
}

namespace {
__global__ void add_partials_cols_kernel(const float* __restrict__ part, int n_parts, int64_t n, float* __restrict__ out) {
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    float t = 0.f;
    for (int k = 0; k < n_parts; ++k) t += part[k * n + i];
    out[i] += t;
  }
}
// one scalar from many partials: 1024 threads take fixed strided subsets, then a fixed tree
__global__ void __launch_bounds__(1024) add_partials_scalar_kernel(const float* __restrict__ part, int n_parts, float* __restrict__ out) {
  __shared__ float red[1024];
  float t = 0.f;
  for (int k = threadIdx.x; k < n_parts; k += 1024) t += part[k];
  red[threadIdx.x] = t;
  __syncthreads();
  for (int w = 512; w > 0; w >>= 1) {
    if (threadIdx.x < w) red[threadIdx.x] += red[threadIdx.x + w];
    __syncthreads();
  }
  if (threadIdx.x == 0) out[0] += red[0];
}
}  // namespace

int add_partials(const float* part, int n_parts, int64_t n, float* out, cudaStream_t st) {
  if (n == 1) {
    add_partials_scalar_kernel<<<1, 1024, 0, st>>>(part, n_parts, out);
  } else {
    int64_t blocks = ceil_div(n, 256);
    const int64_t cap = static_cast<int64_t>(num_sms()) * 8;
    add_partials_cols_kernel<<<(unsigned)(blocks < cap ? blocks : cap), 256, 0, st>>>(part, n_parts, n, out);
  }
  OASR_LAUNCH_CHECK();
  return OASR_OK;
}

}  // namespace oasr

extern "C" const char* oasr_last_error(void) { return oasr::g_err; }
extern "C" int oasr_abi_version(void) { return 1; }
extern "C" int oasr_device_sm_count(void) { return oasr::num_sms(); }

namespace oasr {
static int g_gemm_sm_budget = 0;
int gemm_sm_budget() { return (g_gemm_sm_budget > 0 && g_gemm_sm_budget < num_sms()) ? g_gemm_sm_budget : num_sms(); }
}  // namespace oasr
extern "C" int oasr_gemm_set_sm_budget(int n_sms) {
  const int prev = oasr::g_gemm_sm_budget;
  oasr::g_gemm_sm_budget = n_sms < 0 ? 0 : n_sms;
  return prev;
}
