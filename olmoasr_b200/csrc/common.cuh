// Shared host/device helpers for liboasr_b200. No torch types anywhere in csrc/.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/oasr_b200.h"

namespace oasr {

typedef __nv_bfloat16 bf16;
typedef __half f16;

#define OASR_CUDA_OK(expr)                                                                   \
  do {                                                                                       \
    cudaError_t _e = (expr);                                                                 \
    if (_e != cudaSuccess) {                                                                 \
      oasr::set_last_error("%s:%d %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
      return OASR_ERR_CUDA;                                                                  \
    }                                                                                        \
  } while (0)

#define OASR_REQUIRE(cond, ...)              \
  do {                                       \
    if (!(cond)) {                           \
      oasr::set_last_error(__VA_ARGS__);     \
      return OASR_ERR_INVALID;               \
    }                                        \
  } while (0)

#define OASR_LAUNCH_CHECK() OASR_CUDA_OK(cudaGetLastError())

void set_last_error(const char* fmt, ...);
int num_sms();

// 2-D bf16/f32 row-major tensor map: `inner` contiguous elements per row, `outer` rows,
// `row_stride_bytes` between rows, box = box_inner x box_outer, 128-byte swizzle when
// swizzle128 (box_inner * elt must then be 128 bytes).
int gemm_sm_budget();   // SMs the persistent GEMM may occupy (oasr_gemm_set_sm_budget)
// elt_bytes is 2 or 4 (f32); 2-byte maps are bf16, or IEEE fp16 when fp16.
int make_tmap_2d(CUtensorMap* out, const void* base, int elt_bytes, uint64_t inner, uint64_t outer,
                 uint64_t row_stride_bytes, uint32_t box_inner, uint32_t box_outer, bool swizzle128, bool fp16 = false);
// swizzle_bytes: 0 (none), 64 or 128
int make_tmap_2d_sw(CUtensorMap* out, const void* base, int elt_bytes, uint64_t inner, uint64_t outer,
                    uint64_t row_stride_bytes, uint32_t box_inner, uint32_t box_outer, int swizzle_bytes, bool fp16 = false);
int make_tmap_3d(CUtensorMap* out, const void* base, int elt_bytes, uint64_t d0, uint64_t d1,
                 uint64_t d2, uint64_t stride1_bytes, uint64_t stride2_bytes, uint32_t b0,
                 uint32_t b1, uint32_t b2, bool swizzle128);

__host__ __device__ inline int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }

// ---- deterministic reductions --------------------------------------------------------------------------
// Sums that several blocks contribute to are never folded with floating-point atomics (their order, and so the
// rounding of the result, would change from run to run).  Blocks write partials to stream-ordered scratch and one
// more launch adds them up in a fixed order.
// Scratch comes from the device's default memory pool on the caller's stream (cudaMallocAsync / cudaFreeAsync), so
// concurrent streams never share it; the pool keeps freed memory cached.
void* scratch_alloc(size_t bytes, cudaStream_t st);   // nullptr (and the error string set) on failure
void scratch_free(void* p, cudaStream_t st);
// out[i] += sum_{k < n_parts} part[k * n + i]   for i < n   (k ascending)
int add_partials(const float* part, int n_parts, int64_t n, float* out, cudaStream_t st);

// ---- small device helpers ---------------------------------------------------------------
__device__ __forceinline__ float bf16_round(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }

// erf via Abramowitz & Stegun 7.1.26 (|abs err| <= 1.5e-7): ~12 instructions instead of erff's ~30.  The GELU
// epilogue of the fc1 GEMM is otherwise issue-bound (128 x 256 erff per tile against 8192 cycles of MMA at K = 1024);
// the error is 4 orders of magnitude below the bf16 rounding applied to the result.
__device__ __forceinline__ float erf_fast(float x) {
  const float ax = fabsf(x);
  const float t = __frcp_rn(fmaf(0.3275911f, ax, 1.0f));
  float p = fmaf(t, 1.061405429f, -1.453152027f);
  p = fmaf(t, p, 1.421413741f);
  p = fmaf(t, p, -0.284496736f);
  p = fmaf(t, p, 0.254829592f);
  const float r = fmaf(-p * t, __expf(-ax * ax), 1.0f);
  return copysignf(r, x);
}
__device__ __forceinline__ float gelu_erf(float x) {
  // nn.GELU() / F.gelu default: 0.5 x (1 + erf(x / sqrt(2)))   (reference olmoasr/model.py:480-482,592-593)
  return 0.5f * x * (1.0f + erf_fast(x * 0.70710678118654752440f));
}
__device__ __forceinline__ float gelu_erf_grad(float x) {
  const float cdf = 0.5f * (1.0f + erf_fast(x * 0.70710678118654752440f));
  const float pdf = 0.39894228040143267794f * __expf(-0.5f * x * x);
  return cdf + x * pdf;
}

__device__ __forceinline__ float fast_rcp(float x) {
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float fast_ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// Two-lane float arithmetic, each lane rounded to nearest like the scalar operation (sm_90 has no packed fp32 pipe;
// keeping the pairs lets the callers below read as the vector maths they are).
__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) { return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y)); }
__device__ __forceinline__ float2 fadd2(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ float2 fmul2(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }

// Two-element GELU / GELU' for GEMM epilogues: same Abramowitz-Stegun erf as erf_fast, but MUFU.RCP instead of the
// IEEE reciprocal and one shared exp(-x^2/2) for cdf and pdf: ~10 instructions per element instead of ~35.
struct GeluPair { float2 ea; float2 e; };   // erf(|x|/sqrt2) (>= 0) and exp(-x^2/2)
__device__ __forceinline__ GeluPair gelu_core2(float2 x) {
  // 1 / (1 + p |x| / sqrt2)
  const float2 ax = make_float2(fabsf(x.x), fabsf(x.y));
  const float2 d = ffma2(ax, make_float2(0.23164189f, 0.23164189f), make_float2(1.0f, 1.0f));
  const float2 t = make_float2(fast_rcp(d.x), fast_rcp(d.y));
  float2 p = ffma2(t, make_float2(1.061405429f, 1.061405429f), make_float2(-1.453152027f, -1.453152027f));
  p = ffma2(p, t, make_float2(1.421413741f, 1.421413741f));
  p = ffma2(p, t, make_float2(-0.284496736f, -0.284496736f));
  p = ffma2(p, t, make_float2(0.254829592f, 0.254829592f));
  // exp(-x^2/2) = 2^(-(k x)^2), k = sqrt(log2(e) / 2)
  const float2 y = fmul2(x, make_float2(0.84932180028801907f, 0.84932180028801907f));
  const float2 a = fmul2(make_float2(-y.x, -y.y), y);
  GeluPair r;
  r.e = make_float2(fast_ex2(a.x), fast_ex2(a.y));
  const float2 pt = fmul2(p, t);
  r.ea = ffma2(make_float2(-pt.x, -pt.y), r.e, make_float2(1.0f, 1.0f));
  return r;
}
__device__ __forceinline__ float2 gelu_erf2(float2 x) {   // 0.5 x (1 + erf(x / sqrt 2)) = hx + |hx| erf(|x| / sqrt 2)
  const GeluPair g = gelu_core2(x);
  const float2 hx = fmul2(x, make_float2(0.5f, 0.5f));
  return ffma2(make_float2(fabsf(hx.x), fabsf(hx.y)), g.ea, hx);
}
__device__ __forceinline__ float2 gelu_erf_grad2(float2 x) {   // Phi(x) + x phi(x)
  const GeluPair g = gelu_core2(x);
  const float2 se = make_float2(copysignf(g.ea.x, x.x), copysignf(g.ea.y, x.y));
  const float2 cdf = ffma2(se, make_float2(0.5f, 0.5f), make_float2(0.5f, 0.5f));
  const float2 xp = fmul2(x, make_float2(0.39894228040143267794f, 0.39894228040143267794f));
  return ffma2(xp, g.e, cdf);
}

__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float2 unpack_bf16x2(uint32_t u) {   // one shift + one mask (the intrinsic costs 4-5 PRMT / IMAD)
  return make_float2(__uint_as_float(u << 16), __uint_as_float(u & 0xffff0000u));
}

// The two 16-bit activation types: bf16 (the default, and bf16 autocast) and fp16 (torch.autocast(float16)).  Kernels
// that read or write activations take one of them as a template parameter; the arithmetic is fp32 in both and only
// these conversions differ.  fp16 conversions round to nearest and give +-inf outside +-65504, as torch's casts do.
template <typename T>
struct Act16;
template <>
struct Act16<bf16> {
  static constexpr bool is_fp16 = false;   // tensor maps of this type: bf16
  static __device__ __forceinline__ uint32_t pack2(float lo, float hi) { return pack_bf16x2(lo, hi); }
  static __device__ __forceinline__ float2 unpack2(uint32_t u) { return unpack_bf16x2(u); }
  static __device__ __forceinline__ float to_f(bf16 x) { return __bfloat162float(x); }
  static __device__ __forceinline__ bf16 from_f(float x) { return __float2bfloat16_rn(x); }
  static __device__ __forceinline__ float round(float x) { return bf16_round(x); }
};
template <>
struct Act16<f16> {
  static constexpr bool is_fp16 = true;    // tensor maps of this type: FLOAT16
  static __device__ __forceinline__ uint32_t pack2(float lo, float hi) {   // cvt.rn.f16x2.f32
    __half2 v = __floats2half2_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&v);
  }
  static __device__ __forceinline__ float2 unpack2(uint32_t u) { return __half22float2(*reinterpret_cast<const __half2*>(&u)); }
  static __device__ __forceinline__ float to_f(f16 x) { return __half2float(x); }
  static __device__ __forceinline__ f16 from_f(float x) { return __float2half_rn(x); }
  static __device__ __forceinline__ float round(float x) { return __half2float(__float2half_rn(x)); }
};

// Calls fn<bf16>(args...) or fn<f16>(args...) for an OASR_DTYPE_BF16 / OASR_DTYPE_F16 code.
inline int bad_dtype16(int dtype) {
  set_last_error("16-bit activation dtype must be OASR_DTYPE_BF16 or OASR_DTYPE_F16, got %d", dtype);
  return OASR_ERR_INVALID;
}
#define OASR_BY_DTYPE16(dtype, fn, ...)                                   \
  ((dtype) == OASR_DTYPE_BF16  ? fn<oasr::bf16>(__VA_ARGS__)              \
   : (dtype) == OASR_DTYPE_F16 ? fn<oasr::f16>(__VA_ARGS__)               \
                               : oasr::bad_dtype16(dtype))

template <typename T>
__device__ __forceinline__ T warp_sum(T v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
template <typename T>
__device__ __forceinline__ T warp_max(T v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = max(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

}  // namespace oasr
