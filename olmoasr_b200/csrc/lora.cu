// Low-rank adapter (LoRA) helpers: the 16-bit operands of the GEMM's low-rank tail and the merged fp32 weight.
//   cast_scaled16: dst[r][c] (row stride ld) = T(s * src[r][c])   -- adapter factors, stacked or placed in a zero block
//   lora_merge_f32: out = W + s * B A                                 -- the adapted Linear's effective weight
// The merge is one thread per output element summing over the rank in index order: the same bits on every run, and
// `out` may be W itself.
#include "common.cuh"

namespace oasr {
namespace {

template <typename T>
__global__ void cast_scaled16_kernel(const float* __restrict__ src, int64_t rows, int64_t cols, float s, T* __restrict__ dst,
                                     int64_t ld) {
  const int64_t n = rows * cols;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<int64_t>(gridDim.x) * blockDim.x)
    dst[(i / cols) * ld + i % cols] = Act16<T>::from_f(__fmul_rn(s, src[i]));
}

__global__ void lora_merge_kernel(const float* W, const float* __restrict__ B, const float* __restrict__ A, float s, float* out,
                                  int64_t N, int64_t K, int r) {
  const int64_t n_out = N * K;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n_out; i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t n = i / K, k = i % K;
    float acc = 0.f;
    for (int j = 0; j < r; ++j) acc = __fmaf_rn(__ldg(B + n * r + j), __ldg(A + j * K + k), acc);
    out[i] = __fadd_rn(W[i], __fmul_rn(s, acc));
  }
}

template <typename T>
int cast_scaled16(const float* src, int64_t rows, int64_t cols, float s, void* dst, int64_t ld, cudaStream_t st) {
  const int blocks = (int)std::min<int64_t>(ceil_div(rows * cols, 256), (int64_t)num_sms() * 16);
  cast_scaled16_kernel<T><<<blocks, 256, 0, st>>>(src, rows, cols, s, static_cast<T*>(dst), ld);
  OASR_LAUNCH_CHECK();
  return OASR_OK;
}

}  // namespace
}  // namespace oasr

using namespace oasr;

extern "C" int oasr_cast_scaled16(const float* src, int64_t rows, int64_t cols, float scale, void* dst, int64_t ld_dst, int dtype,
                                  void* stream) {
  OASR_REQUIRE(src && dst && rows > 0 && cols > 0 && ld_dst >= cols, "cast_scaled16: bad arguments");
  return OASR_BY_DTYPE16(dtype, cast_scaled16, src, rows, cols, scale, dst, ld_dst, (cudaStream_t)stream);
}

extern "C" int oasr_lora_merge_f32(const float* W, const float* B, const float* A, float scale, float* out, int64_t N, int64_t K,
                                   int64_t r, void* stream) {
  OASR_REQUIRE(W && B && A && out && N > 0 && K > 0 && r > 0 && r <= 4096, "lora_merge: bad arguments");
  const int blocks = (int)std::min<int64_t>(ceil_div(N * K, 256), (int64_t)num_sms() * 16);
  lora_merge_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(W, B, A, scale, out, N, K, (int)r);
  OASR_LAUNCH_CHECK();
  return OASR_OK;
}
