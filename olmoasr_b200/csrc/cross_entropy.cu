// Token cross-entropy over bf16 logits (fp32 math), forward and backward, one block per row.
//
// Replaces F.cross_entropy(logits.view(-1, V), y.view(-1), ignore_index=51864)
// (scripts/training/train_timestamps.py:1444-1448) and its autograd.  The reference materialises fp32
// logits (B,448,51865) = 2.97 GB at B=32 and makes three passes over them; here the logits stay bf16
// (they ARE bf16-rounded in the reference: model.py:768-770 runs the matmul in bf16 and then `.float()`),
// the forward is one online-softmax pass and the backward overwrites the logits in place with d(logits).
#include "common.cuh"

namespace oasr {
namespace {

struct MS { float m, s; };
__device__ __forceinline__ MS ms_merge(MS a, MS b) {
  const float m = fmaxf(a.m, b.m);
  if (m == -INFINITY) return {m, 0.f};
  return {m, a.s * __expf(a.m - m) + b.s * __expf(b.m - m)};
}

// lse[row] = logsumexp(logits[row, :V]);  count += 1   (rows with y == ignore skipped; the counts are exact integers)
__global__ void __launch_bounds__(256)
ce_fwd_kernel(const bf16* __restrict__ logits, const int64_t* __restrict__ targets, float* __restrict__ lse,
              float* __restrict__ loss_sum_count, int64_t ld, int V, int64_t ignore_index) {
  const int64_t row = blockIdx.x;
  const int64_t y = targets[row];
  if (y == ignore_index || y < 0 || y >= V) {  // nothing to compute for ignored rows
    if (threadIdx.x == 0) {
      lse[row] = 0.f;
      if (y != ignore_index) atomicAdd(loss_sum_count + 2, 1.0f);   // a target outside [0, V): F.cross_entropy would raise
    }
    return;
  }
  const bf16* x = logits + row * ld;
  MS acc{-INFINITY, 0.f};
  const int nvec = V >> 3;
  for (int v = threadIdx.x; v < nvec; v += blockDim.x) {
    const uint4 u = reinterpret_cast<const uint4*>(x)[v];
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
    float f[8];
#pragma unroll
    for (int j = 0; j < 4; ++j) { const float2 t = unpack_bf16x2(w[j]); f[2 * j] = t.x; f[2 * j + 1] = t.y; }
    float mx = f[0];
#pragma unroll
    for (int j = 1; j < 8; ++j) mx = fmaxf(mx, f[j]);
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) s += __expf(f[j] - mx);
    acc = ms_merge(acc, MS{mx, s});
  }
  for (int c = (nvec << 3) + threadIdx.x; c < V; c += blockDim.x) acc = ms_merge(acc, MS{__bfloat162float(x[c]), 1.f});
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    MS other{__shfl_xor_sync(0xffffffffu, acc.m, o), __shfl_xor_sync(0xffffffffu, acc.s, o)};
    acc = ms_merge(acc, other);
  }
  __shared__ MS part[8];
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    MS t = part[0];
    for (int i = 1; i < (blockDim.x >> 5); ++i) t = ms_merge(t, part[i]);
    const float l = t.m + logf(t.s);
    lse[row] = l;
    atomicAdd(loss_sum_count + 1, 1.0f);
  }
}

// loss_sum += sum over the counted rows of lse - logits[row, y], in row order: 1024 threads take fixed strided subsets
// of the rows, then a fixed tree (an atomic per row would make the rounding of the sum change from run to run)
__global__ void __launch_bounds__(1024)
ce_loss_sum_kernel(const bf16* __restrict__ logits, const int64_t* __restrict__ targets, const float* __restrict__ lse,
                   float* __restrict__ loss_sum_count, int64_t rows, int64_t ld, int V, int64_t ignore_index) {
  __shared__ float red[1024];
  float t = 0.f;
  for (int64_t row = threadIdx.x; row < rows; row += 1024) {
    const int64_t y = targets[row];
    if (y == ignore_index || y < 0 || y >= V) continue;
    t += lse[row] - __bfloat162float(logits[row * ld + y]);
  }
  red[threadIdx.x] = t;
  __syncthreads();
  for (int w = 512; w > 0; w >>= 1) {
    if (threadIdx.x < w) red[threadIdx.x] += red[threadIdx.x + w];
    __syncthreads();
  }
  if (threadIdx.x == 0) loss_sum_count[0] += red[0];
}

// in place: logits[row, v] <- bf16( g * (exp(logits - lse) - [v == y]) ),  g = grad_out / count  (0 for ignored rows)
__global__ void __launch_bounds__(256)
ce_bwd_kernel(bf16* __restrict__ logits, const int64_t* __restrict__ targets, const float* __restrict__ lse,
              const float* __restrict__ loss_sum_count, const float* __restrict__ grad_out, int64_t ld, int V,
              int64_t ignore_index) {
  const int64_t row = blockIdx.x;
  const int64_t y = targets[row];
  bf16* x = logits + row * ld;
  const bool ignored = (y == ignore_index || y < 0 || y >= V);
  const float g = ignored ? 0.f : (*grad_out) / loss_sum_count[1];
  const float l = lse[row];
  const int nvec = V >> 3;
  for (int v = threadIdx.x; v < nvec; v += blockDim.x) {
    uint4 u = make_uint4(0, 0, 0, 0);
    if (!ignored) {
      const uint4 in = reinterpret_cast<const uint4*>(x)[v];
      const uint32_t w[4] = {in.x, in.y, in.z, in.w};
      uint32_t o[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 t = unpack_bf16x2(w[j]);
        const int c = v * 8 + 2 * j;
        const float a = g * (__expf(t.x - l) - (c == y ? 1.f : 0.f));
        const float b = g * (__expf(t.y - l) - (c + 1 == y ? 1.f : 0.f));
        o[j] = pack_bf16x2(a, b);
      }
      u = make_uint4(o[0], o[1], o[2], o[3]);
    }
    reinterpret_cast<uint4*>(x)[v] = u;
  }
  for (int c = (nvec << 3) + threadIdx.x; c < V; c += blockDim.x) {
    const float a = ignored ? 0.f : g * (__expf(__bfloat162float(x[c]) - l) - (c == y ? 1.f : 0.f));
    x[c] = __float2bfloat16_rn(a);
  }
}

// loss = sum / count (mean over the non-ignored targets of this rank, train_timestamps.py:1444-1448)
__global__ void ce_finalize_kernel(const float* __restrict__ lsc, float* __restrict__ loss) { *loss = lsc[0] / lsc[1]; }

// bf16 (rows, ld) -> f32 (rows, V) contiguous: the `.float()` of model.py:770 for callers that want logits
__global__ void logits_to_f32_kernel(const bf16* __restrict__ src, float* __restrict__ dst, int64_t ld, int V) {
  const int64_t row = blockIdx.x;
  for (int c = threadIdx.x; c < V; c += blockDim.x) dst[row * V + c] = __bfloat162float(src[row * ld + c]);
}

}  // namespace
}  // namespace oasr

using namespace oasr;

extern "C" int oasr_ce_fwd(const void* logits, const int64_t* targets, float* lse, float* loss_sum_count, int64_t rows,
                           int64_t V, int64_t ld, int64_t ignore_index, void* stream) {
  OASR_REQUIRE(rows > 0 && V > 0 && ld >= V && (ld & 7) == 0, "ce_fwd: bad shape rows=%ld V=%ld ld=%ld", (long)rows, (long)V, (long)ld);
  ce_fwd_kernel<<<(unsigned)rows, 256, 0, (cudaStream_t)stream>>>((const bf16*)logits, targets, lse, loss_sum_count, ld, (int)V, ignore_index);
  OASR_LAUNCH_CHECK();
  ce_loss_sum_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>((const bf16*)logits, targets, lse, loss_sum_count, rows, ld, (int)V, ignore_index);
  OASR_LAUNCH_CHECK();
  return OASR_OK;
}

extern "C" int oasr_ce_finalize(const float* loss_sum_count, float* loss, void* stream) {
  OASR_REQUIRE(loss_sum_count != nullptr && loss != nullptr, "ce_finalize: null");
  ce_finalize_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(loss_sum_count, loss);
  OASR_LAUNCH_CHECK();
  return OASR_OK;
}

extern "C" int oasr_ce_bwd(void* logits, const int64_t* targets, const float* lse, const float* loss_sum_count,
                           const float* grad_out, int64_t rows, int64_t V, int64_t ld, int64_t ignore_index, void* stream) {
  OASR_REQUIRE(rows > 0 && V > 0 && ld >= V && (ld & 7) == 0, "ce_bwd: bad shape");
  ce_bwd_kernel<<<(unsigned)rows, 256, 0, (cudaStream_t)stream>>>((bf16*)logits, targets, lse, loss_sum_count, grad_out, ld, (int)V, ignore_index);
  OASR_LAUNCH_CHECK();
  return OASR_OK;
}

extern "C" int oasr_logits_to_f32(const void* src, float* dst, int64_t rows, int64_t V, int64_t ld, void* stream) {
  OASR_REQUIRE(rows > 0 && V > 0 && ld >= V, "logits_to_f32: bad shape");
  logits_to_f32_kernel<<<(unsigned)rows, 256, 0, (cudaStream_t)stream>>>((const bf16*)src, dst, ld, (int)V);
  OASR_LAUNCH_CHECK();
  return OASR_OK;
}
