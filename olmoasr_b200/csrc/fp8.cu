// Per-row dynamic FP8 quantisation, the operand preparation of the FP8 training GEMMs (oasr_gemm_fp8):
//   amax = max |x[r, :]|,  inv = fmax / amax,  q[r, c] = fp8_rn_satfinite(x[r, c] * inv),  scale[r] = amax / fmax
// in fp32 with IEEE division and multiplication (zero row: inv = scale = 1), which is bit for bit what
// (x.float() * inv).to(torch.float8_*) gives.  fmax = 448 (e4m3) or 57344 (e5m2).
//   rows form:       one CTA per row; each thread keeps no copy, so the row is read twice (the second read hits L1/L2)
//   transposed form: the rows of x^T (a weight's input features, for the dgrad operand W^T): a CTA owns 32 columns of
//                    x, finds their amax, then transposes 32 x 32 tiles through shared memory so both the reads of x
//                    and the writes of q are row-contiguous.  It runs on weights only, once per optimizer step.
#include "common.cuh"

#include <cuda_fp8.h>

namespace oasr {
namespace {

template <int FMT>
struct Fp8Fmt;
template <>
struct Fp8Fmt<OASR_FP8_E4M3> {
  static constexpr float fmax = 448.f;
  static constexpr __nv_fp8_interpretation_t kind = __NV_E4M3;
};
template <>
struct Fp8Fmt<OASR_FP8_E5M2> {
  static constexpr float fmax = 57344.f;
  static constexpr __nv_fp8_interpretation_t kind = __NV_E5M2;
};

// (inv, scale) of a row with maximum magnitude amax
template <int FMT>
__device__ __forceinline__ float2 row_scales(float amax) {
  if (amax == 0.f) return make_float2(1.f, 1.f);
  return make_float2(__fdiv_rn(Fp8Fmt<FMT>::fmax, amax), __fdiv_rn(amax, Fp8Fmt<FMT>::fmax));
}

template <int FMT>
__device__ __forceinline__ uint8_t to_fp8(float x, float inv) {
  return static_cast<uint8_t>(__nv_cvt_float_to_fp8(__fmul_rn(x, inv), __NV_SATFINITE, Fp8Fmt<FMT>::kind));
}

constexpr int ROW_THREADS = 128;

template <typename T, int FMT>
__global__ void __launch_bounds__(ROW_THREADS) quantize_rows_kernel(const T* __restrict__ x, int64_t ldx, int64_t rows,
                                                                    int64_t cols, uint8_t* __restrict__ q, int64_t ldq,
                                                                    float* __restrict__ scale) {
  __shared__ float red[ROW_THREADS / 32];
  const int chunks = static_cast<int>(cols / 8);
  for (int64_t r = blockIdx.x; r < rows; r += gridDim.x) {
    const T* xr = x + r * ldx;
    float m = 0.f;
    for (int c = threadIdx.x; c < chunks; c += ROW_THREADS) {
      const uint4 v = __ldg(reinterpret_cast<const uint4*>(xr) + c);
      const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 f = Act16<T>::unpack2(w[e]);
        m = fmaxf(m, fmaxf(fabsf(f.x), fabsf(f.y)));
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
    __syncthreads();
    float amax = red[0];
#pragma unroll
    for (int i = 1; i < ROW_THREADS / 32; ++i) amax = fmaxf(amax, red[i]);
    const float2 is = row_scales<FMT>(amax);
    if (threadIdx.x == 0) scale[r] = is.y;
    for (int c = threadIdx.x; c < chunks; c += ROW_THREADS) {
      const uint4 v = __ldg(reinterpret_cast<const uint4*>(xr) + c);
      const uint32_t w[4] = {v.x, v.y, v.z, v.w};
      uint32_t out[2] = {0u, 0u};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 f = Act16<T>::unpack2(w[e]);
        const uint32_t pair = to_fp8<FMT>(f.x, is.x) | (uint32_t(to_fp8<FMT>(f.y, is.x)) << 8);
        out[e >> 1] |= pair << (16 * (e & 1));
      }
      *reinterpret_cast<uint2*>(q + r * ldq + 8 * c) = make_uint2(out[0], out[1]);
    }
    __syncthreads();   // red[] is reused by the next row
  }
}

// x (rows, cols) -> q (cols, rows): CTA = 32 x 8 threads over columns [32 b, 32 b + 32) of x
template <typename T, int FMT>
__global__ void __launch_bounds__(256) quantize_cols_kernel(const T* __restrict__ x, int64_t ldx, int64_t rows,
                                                            int64_t cols, uint8_t* __restrict__ q, int64_t ldq,
                                                            float* __restrict__ scale) {
  __shared__ float tile[32][33];
  __shared__ float inv_s[32];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int64_t c0 = static_cast<int64_t>(blockIdx.x) * 32;
  const bool col_ok = c0 + tx < cols;
  float m = 0.f;
  if (col_ok)
    for (int64_t r = ty; r < rows; r += 8) m = fmaxf(m, fabsf(Act16<T>::to_f(x[r * ldx + c0 + tx])));
  tile[ty][tx] = m;
  __syncthreads();
  if (ty == 0) {
    float a = tile[0][tx];
#pragma unroll
    for (int i = 1; i < 8; ++i) a = fmaxf(a, tile[i][tx]);
    const float2 is = row_scales<FMT>(a);
    inv_s[tx] = is.x;
    if (col_ok) scale[c0 + tx] = is.y;
  }
  for (int64_t r0 = 0; r0 < rows; r0 += 32) {
    __syncthreads();   // inv_s written / the previous tile consumed
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int64_t r = r0 + ty + 8 * i;
      tile[ty + 8 * i][tx] = (r < rows && col_ok) ? Act16<T>::to_f(x[r * ldx + c0 + tx]) : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int cl = ty + 8 * i;   // row c0 + cl of q, column r0 + tx
      if (c0 + cl < cols && r0 + tx < rows) q[(c0 + cl) * ldq + r0 + tx] = to_fp8<FMT>(tile[tx][cl], inv_s[cl]);
    }
  }
}

template <typename T, int FMT>
int quantize(const void* x, int64_t ldx, int64_t rows, int64_t cols, int transpose, void* q, int64_t ldq, float* scale,
             cudaStream_t st) {
  if (transpose) {
    quantize_cols_kernel<T, FMT><<<(unsigned)ceil_div(cols, 32), 256, 0, st>>>(static_cast<const T*>(x), ldx, rows, cols,
                                                                               static_cast<uint8_t*>(q), ldq, scale);
  } else {
    const int blocks = (int)std::min<int64_t>(rows, (int64_t)num_sms() * 16);
    quantize_rows_kernel<T, FMT><<<blocks, ROW_THREADS, 0, st>>>(static_cast<const T*>(x), ldx, rows, cols,
                                                                 static_cast<uint8_t*>(q), ldq, scale);
  }
  OASR_LAUNCH_CHECK();
  return OASR_OK;
}

template <typename T>
int quantize16(const void* x, int64_t ldx, int64_t rows, int64_t cols, int fmt, int transpose, void* q, int64_t ldq,
               float* scale, cudaStream_t st) {
  return fmt == OASR_FP8_E4M3 ? quantize<T, OASR_FP8_E4M3>(x, ldx, rows, cols, transpose, q, ldq, scale, st)
                              : quantize<T, OASR_FP8_E5M2>(x, ldx, rows, cols, transpose, q, ldq, scale, st);
}

}  // namespace
}  // namespace oasr

using namespace oasr;

extern "C" int oasr_quantize_fp8_rows(const void* x, int64_t ldx, int64_t rows, int64_t cols, int dtype, int fmt,
                                      int transpose, void* q, int64_t ldq, float* scale, void* stream) {
  OASR_REQUIRE(x && q && scale && rows > 0 && cols > 0, "quantize_fp8: bad arguments");
  OASR_REQUIRE(fmt == OASR_FP8_E4M3 || fmt == OASR_FP8_E5M2, "quantize_fp8: bad format %d", fmt);
  OASR_REQUIRE(ldx >= cols && ldq >= (transpose ? rows : cols), "quantize_fp8: row strides too small");
  OASR_REQUIRE((transpose ? rows : cols) % 8 == 0 && (ldx & 7) == 0 && (ldq & 7) == 0 &&
               (reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(q) & 7) == 0,
               "quantize_fp8: the quantised width must be a multiple of 8, x 16-byte and q 8-byte aligned, ldx / ldq "
               "multiples of 8");
  return OASR_BY_DTYPE16(dtype, quantize16, x, ldx, rows, cols, fmt, transpose, q, ldq, scale, (cudaStream_t)stream);
}
