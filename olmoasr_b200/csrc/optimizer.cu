// Fused multi-tensor optimizer step: global grad-norm, clip, (un)scale, AdamW -- two launches for the whole model.
//
// Replaces scaler.unscale_(optimizer) -> clip_grad_norm_(model.parameters(), 1.0) -> scaler.step(optimizer)
// (scripts/training/train_timestamps.py:1508-1522; AdamW lr 1.5e-3 betas (0.9, 0.98) eps 1e-6 wd 0.1, :2110-2113).
// HBM-bound: 4 B/param for the norm pass, 28 B/param for the update (read p, g, m, v; write p, m, v).
#include "common.cuh"

namespace oasr {
namespace {

constexpr int CHUNK = 16384;  // elements per block

struct TensorRec {  // one row of the device-side table (6 x int64)
  float* p;
  const float* g;
  float* m;
  float* v;
  int64_t numel;
  bf16* shadow;  // optional bf16 (or, in the fp16 kernels, fp16) copy of p, refreshed by the update itself (nullptr: none)
};

// sum over the block into this block's partial (added up in block order afterwards: add_partials).  Callers square
// UNSCALED values (g * inv_scale) so that a 65536x loss scale cannot overflow the fp32 total.
__device__ __forceinline__ void block_sum_to(float s, float* part) {
  s = warp_sum(s);
  __shared__ float part_w[8];
  if ((threadIdx.x & 31) == 0) part_w[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int i = 0; i < 8; ++i) t += part_w[i];
    part[blockIdx.x] = t;
  }
}

__global__ void __launch_bounds__(256)
grad_sqnorm_kernel(const TensorRec* __restrict__ recs, const int2* __restrict__ chunks, float* __restrict__ part,
                   float inv_scale) {
  const int2 ch = chunks[blockIdx.x];
  const TensorRec r = recs[ch.x];
  const int64_t start = static_cast<int64_t>(ch.y) * CHUNK;
  const int64_t end = min(r.numel, start + CHUNK);
  const float* g = r.g + start;
  const int n = static_cast<int>(end - start);
  float s = 0.f;
  const float k = inv_scale;
  if ((reinterpret_cast<uintptr_t>(g) & 15) == 0) {
    for (int i = threadIdx.x * 4; i + 4 <= n; i += blockDim.x * 4) {
      const float4 v = *reinterpret_cast<const float4*>(g + i);
      const float a = v.x * k, b = v.y * k, c = v.z * k, d = v.w * k;
      s += a * a + b * b + c * c + d * d;
    }
    for (int i = (n & ~3) + threadIdx.x; i < n; i += blockDim.x) { const float a = g[i] * k; s += a * a; }
  } else {
    for (int i = threadIdx.x; i < n; i += blockDim.x) { const float a = g[i] * k; s += a * a; }
  }
  block_sum_to(s, part);
}

// Same reduction over one flat gradient slab (olmoasr_b200.slab): no table, every block owns CHUNK elements.
__global__ void __launch_bounds__(256)
sqnorm_flat_kernel(const float* __restrict__ g, int64_t n, float* __restrict__ part, float inv_scale) {
  const int64_t start = static_cast<int64_t>(blockIdx.x) * CHUNK;
  const int m = static_cast<int>(min(n, start + CHUNK) - start);
  g += start;
  float s = 0.f;
  const float k = inv_scale;
  for (int i = threadIdx.x * 4; i + 4 <= m; i += blockDim.x * 4) {
    const float4 v = *reinterpret_cast<const float4*>(g + i);
    const float a = v.x * k, b = v.y * k, c = v.z * k, d = v.w * k;
    s += a * a + b * b + c * c + d * d;
  }
  for (int i = (m & ~3) + threadIdx.x; i < m; i += blockDim.x) { const float a = g[i] * k; s += a * a; }
  block_sum_to(s, part);
}

// One thread: turns the squared norm into the step's scalars.  The step counter lives on the device and advances only
// when the update is applied (GradScaler + AdamW do not count skipped steps), so no host read is needed per step.
//   st[0] step  st[1] coef (unscale x clip)  st[2] 1 - beta1^t  st[3] sqrt(1 - beta2^t)  st[4] skip  st[5] grad norm
__device__ __forceinline__ void prepare_step(float nsq, bool skip, float* __restrict__ found_inf, float* __restrict__ st,
                                             float inv_scale, float max_norm, float beta1, float beta2) {
  if (skip || !isfinite(nsq)) {
    *found_inf = 1.f;
    st[4] = 1.f;
    st[5] = sqrtf(nsq);   // the norm, as on an applied step (inf / NaN stay inf / NaN)
    return;
  }
  const float total_norm = sqrtf(nsq);
  float coef = inv_scale;
  if (max_norm > 0.f) coef *= fminf(1.f, max_norm / (total_norm + 1e-6f));  // clip_grad_norm_
  const float step = st[0] + 1.f;
  st[0] = step;
  st[1] = coef;
  st[2] = 1.f - powf(beta1, step);
  st[3] = sqrtf(1.f - powf(beta2, step));
  st[4] = 0.f;
  st[5] = total_norm;
}
__global__ void optim_prepare_kernel(const float* __restrict__ norm_sq, float* __restrict__ found_inf, float* __restrict__ st,
                                     float inv_scale, float max_norm, float beta1, float beta2) {
  // of the UNSCALED gradients (inv_scale is applied before squaring)
  prepare_step(*norm_sq, false, found_inf, st, inv_scale, max_norm, beta1, beta2);
}
// GradScaler form: the loss scale S and GradScaler's found_inf flag are read on the device, so the host never waits for
// them.  norm_sq was taken over g * inv_scale, still multiplied by S: the norm of the unscaled gradients is
// sqrt(norm_sq) / S, and every gradient is multiplied by inv_scale / S.  A set flag skips the step like a non-finite norm.
__global__ void optim_prepare_amp_kernel(const float* __restrict__ norm_sq, float* __restrict__ found_inf,
                                         float* __restrict__ st, const float* __restrict__ loss_scale,
                                         const float* __restrict__ ext_found_inf, float inv_scale, float max_norm,
                                         float beta1, float beta2) {
  float nsq = *norm_sq;
  if (loss_scale != nullptr) {
    const float r = 1.f / *loss_scale;
    nsq = nsq * r * r;
    inv_scale *= r;
  }
  const bool skip = ext_found_inf != nullptr && *ext_found_inf != 0.f;
  prepare_step(nsq, skip, found_inf, st, inv_scale, max_norm, beta1, beta2);
}

// One CHUNK of the update.  `st` is written by optim_prepare_kernel; when it flags a non-finite norm the whole update is
// skipped (GradScaler semantics).  When `sh` is given the T (bf16 / fp16) shadow the GEMMs read is refreshed from the value
// still in registers -- the reference instead re-casts every fp32 master on every forward (olmoasr/model.py:97-101).
template <typename T>
__device__ __forceinline__ void adamw_chunk(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                                            float* __restrict__ v, T* __restrict__ sh, int n, const float* __restrict__ st,
                                            float lr, float beta1, float beta2, float eps, float weight_decay) {
  if (st[4] != 0.f) return;
  const float coef = st[1], bc1 = st[2], bc2_sqrt = st[3];
  const float step_size = lr / bc1;
  const float decay = 1.f - lr * weight_decay;
  int i0 = 0;
  if (((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(m) |
        reinterpret_cast<uintptr_t>(v)) & 15) == 0 && (reinterpret_cast<uintptr_t>(sh) & 7) == 0) {
    const int n4 = n & ~3;
    for (int i = threadIdx.x * 4; i < n4; i += blockDim.x * 4) {   // 16-byte accesses: 7 vector transactions per 4 params
      float4 pv = *reinterpret_cast<float4*>(p + i);
      const float4 gv = *reinterpret_cast<const float4*>(g + i);
      float4 mv = *reinterpret_cast<float4*>(m + i);
      float4 vv = *reinterpret_cast<float4*>(v + i);
      float* pp = &pv.x; const float* gp = &gv.x; float* mp = &mv.x; float* vp = &vv.x;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float gi = gp[j] * coef;
        mp[j] = beta1 * mp[j] + (1.f - beta1) * gi;
        vp[j] = beta2 * vp[j] + (1.f - beta2) * gi * gi;
        pp[j] = pp[j] * decay - step_size * (mp[j] / (sqrtf(vp[j]) / bc2_sqrt + eps));
      }
      *reinterpret_cast<float4*>(p + i) = pv;
      *reinterpret_cast<float4*>(m + i) = mv;
      *reinterpret_cast<float4*>(v + i) = vv;
      if (sh != nullptr) *reinterpret_cast<uint2*>(sh + i) = make_uint2(Act16<T>::pack2(pv.x, pv.y), Act16<T>::pack2(pv.z, pv.w));
    }
    i0 = n4;
  }
  for (int i = i0 + threadIdx.x; i < n; i += blockDim.x) {
    const float gi = g[i] * coef;
    const float mi = beta1 * m[i] + (1.f - beta1) * gi;
    const float vi = beta2 * v[i] + (1.f - beta2) * gi * gi;
    const float denom = sqrtf(vi) / bc2_sqrt + eps;
    const float pi = p[i] * decay - step_size * (mi / denom);
    p[i] = pi;
    m[i] = mi;
    v[i] = vi;
    if (sh != nullptr) sh[i] = Act16<T>::from_f(pi);
  }
}

template <typename T>
__global__ void __launch_bounds__(256)
adamw_kernel(const TensorRec* __restrict__ recs, const int2* __restrict__ chunks, const float* __restrict__ st, float lr,
             float beta1, float beta2, float eps, float weight_decay) {
  const int2 ch = chunks[blockIdx.x];
  const TensorRec r = recs[ch.x];
  const int64_t start = static_cast<int64_t>(ch.y) * CHUNK;
  const int n = static_cast<int>(min(r.numel, start + CHUNK) - start);
  adamw_chunk(r.p + start, r.g + start, r.m + start, r.v + start, r.shadow ? reinterpret_cast<T*>(r.shadow) + start : nullptr, n, st, lr, beta1,
              beta2, eps, weight_decay);
}

template <typename T>
__global__ void __launch_bounds__(256)
adamw_flat_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                  T* __restrict__ sh, int64_t numel, const float* __restrict__ st, float lr, float beta1, float beta2,
                  float eps, float weight_decay) {
  const int64_t start = static_cast<int64_t>(blockIdx.x) * CHUNK;
  const int n = static_cast<int>(min(numel, start + CHUNK) - start);
  adamw_chunk(p + start, g + start, m + start, v + start, sh ? sh + start : nullptr, n, st, lr, beta1, beta2, eps, weight_decay);
}

}  // namespace
}  // namespace oasr

using namespace oasr;

extern "C" int oasr_optim_chunk_elems(void) { return CHUNK; }

extern "C" int oasr_grad_sqnorm(const void* recs, const void* chunks, int64_t n_chunks, float inv_scale, float* out, void* stream) {
  OASR_REQUIRE(n_chunks > 0, "grad_sqnorm: no chunks");
  cudaStream_t st = (cudaStream_t)stream;
  float* part = static_cast<float*>(scratch_alloc(sizeof(float) * n_chunks, st));
  if (!part) return OASR_ERR_CUDA;
  OASR_CUDA_OK(cudaMemsetAsync(out, 0, sizeof(float), st));
  grad_sqnorm_kernel<<<(unsigned)n_chunks, 256, 0, st>>>((const TensorRec*)recs, (const int2*)chunks, part, inv_scale);
  OASR_LAUNCH_CHECK();
  const int rc = add_partials(part, (int)n_chunks, 1, out, st);
  scratch_free(part, st);
  return rc;
}

extern "C" int oasr_grad_sqnorm_flat(const float* g, int64_t numel, float inv_scale, float* out, void* stream) {
  OASR_REQUIRE(numel > 0 && ((uintptr_t)g & 15) == 0, "grad_sqnorm_flat: empty or unaligned slab");
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t blocks = ceil_div(numel, CHUNK);
  float* part = static_cast<float*>(scratch_alloc(sizeof(float) * blocks, st));
  if (!part) return OASR_ERR_CUDA;
  OASR_CUDA_OK(cudaMemsetAsync(out, 0, sizeof(float), st));
  sqnorm_flat_kernel<<<(unsigned)blocks, 256, 0, st>>>(g, numel, part, inv_scale);
  OASR_LAUNCH_CHECK();
  const int rc = add_partials(part, (int)blocks, 1, out, st);
  scratch_free(part, st);
  return rc;
}

extern "C" int oasr_optim_prepare(const float* norm_sq, float* found_inf, float* state, float inv_scale, float max_norm,
                                  float beta1, float beta2, void* stream) {
  OASR_REQUIRE(norm_sq && found_inf && state, "optim_prepare: null pointer");
  optim_prepare_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(norm_sq, found_inf, state, inv_scale, max_norm, beta1, beta2);
  OASR_LAUNCH_CHECK();
  return OASR_OK;
}

static int adamw_step(const void* recs, const void* chunks, int64_t n_chunks, const float* state, float lr, float beta1,
                      float beta2, float eps, float weight_decay, void* stream) {
  OASR_REQUIRE(n_chunks > 0 && state, "adamw: bad arguments");
  adamw_kernel<bf16><<<(unsigned)n_chunks, 256, 0, (cudaStream_t)stream>>>((const TensorRec*)recs, (const int2*)chunks, state, lr, beta1,
                                                                    beta2, eps, weight_decay);
  OASR_LAUNCH_CHECK();
  return OASR_OK;
}

template <typename T>
static int adamw_flat(float* p, const float* g, float* m, float* v, void* shadow_bf16, int64_t numel, const float* state,
                      float lr, float beta1, float beta2, float eps, float weight_decay, void* stream) {
  OASR_REQUIRE(numel > 0 && state, "adamw_flat: bad arguments");
  OASR_REQUIRE((((uintptr_t)p | (uintptr_t)g | (uintptr_t)m | (uintptr_t)v) & 15) == 0 && ((uintptr_t)shadow_bf16 & 7) == 0,
               "adamw_flat: slabs must be 16-byte aligned");
  adamw_flat_kernel<T><<<(unsigned)ceil_div(numel, CHUNK), 256, 0, (cudaStream_t)stream>>>(p, g, m, v, (T*)shadow_bf16, numel, state, lr,
                                                                                      beta1, beta2, eps, weight_decay);
  OASR_LAUNCH_CHECK();
  return OASR_OK;
}

extern "C" int oasr_optim_prepare_amp(const float* norm_sq, float* found_inf, float* state, const float* loss_scale,
                                      const float* ext_found_inf, float inv_scale, float max_norm, float beta1, float beta2,
                                      void* stream) {
  OASR_REQUIRE(norm_sq && found_inf && state, "optim_prepare_amp: null pointer");
  optim_prepare_amp_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(norm_sq, found_inf, state, loss_scale, ext_found_inf, inv_scale,
                                                              max_norm, beta1, beta2);
  OASR_LAUNCH_CHECK();
  return OASR_OK;
}

extern "C" int oasr_adamw_step(const void* recs, const void* chunks, int64_t n_chunks, const float* state, float lr, float beta1,
                               float beta2, float eps, float weight_decay, void* stream) {
  return adamw_step(recs, chunks, n_chunks, state, lr, beta1, beta2, eps, weight_decay, stream);
}

extern "C" int oasr_adamw_flat(float* p, const float* g, float* m, float* v, void* shadow_bf16, int64_t numel, const float* state,
                               float lr, float beta1, float beta2, float eps, float weight_decay, void* stream) {
  return adamw_flat<bf16>(p, g, m, v, shadow_bf16, numel, state, lr, beta1, beta2, eps, weight_decay, stream);
}

extern "C" int oasr_adamw_flat16(float* p, const float* g, float* m, float* v, void* shadow, int64_t numel, const float* state,
                                 float lr, float beta1, float beta2, float eps, float weight_decay, int dtype, void* stream) {
  return OASR_BY_DTYPE16(dtype, adamw_flat, p, g, m, v, shadow, numel, state, lr, beta1, beta2, eps, weight_decay, stream);
}
