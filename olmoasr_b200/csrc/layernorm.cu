// LayerNorm forward / backward, bf16 or fp16 in/out with fp32 statistics (one warp per row, 16-byte loads,
// shuffle reductions).  HBM-bound: 4 B/element forward, 6-8 B/element backward.
//
// Reference: LayerNorm.forward = F.layer_norm(x.float(), eps=1e-5).type(x.dtype)  (olmoasr/model.py:25-39);
// autograd of the same.  The backward also folds in the residual-branch gradient so that
// dx_total = bf16(d_residual + bf16(dx_ln)) matches autograd's bf16 accumulation order.
#include "common.cuh"

namespace oasr {
namespace {

constexpr int LN_MAX_VEC = 5;  // d <= 5 * 32 * 8 = 1280; kernels are instantiated per ceil(d / 256) to bound registers

template <typename T, bool kWriteStats, int NV>
__global__ void __launch_bounds__(256)
layernorm_fwd_kernel(const T* __restrict__ x, const float* __restrict__ w, const float* __restrict__ b,
                     T* __restrict__ y, float* __restrict__ mean_out, float* __restrict__ rstd_out,
                     int64_t rows, int d, float eps) {
  const int warps_per_block = blockDim.x >> 5;
  const int lane = threadIdx.x & 31;
  const int nvec = d >> 3;
  for (int64_t row = static_cast<int64_t>(blockIdx.x) * warps_per_block + (threadIdx.x >> 5); row < rows;
       row += static_cast<int64_t>(gridDim.x) * warps_per_block) {
    const uint4* xr = reinterpret_cast<const uint4*>(x + row * d);
    float v[NV][8];
    float sum = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int vi = lane + 32 * i;
      if (vi < nvec) {
        const uint4 u = xr[vi];
        float2 p0 = Act16<T>::unpack2(u.x), p1 = Act16<T>::unpack2(u.y), p2 = Act16<T>::unpack2(u.z), p3 = Act16<T>::unpack2(u.w);
        v[i][0] = p0.x; v[i][1] = p0.y; v[i][2] = p1.x; v[i][3] = p1.y;
        v[i][4] = p2.x; v[i][5] = p2.y; v[i][6] = p3.x; v[i][7] = p3.y;
#pragma unroll
        for (int j = 0; j < 8; ++j) sum += v[i][j];
      }
    }
    const float mean = warp_sum(sum) / d;
    float sq = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i)
      if (lane + 32 * i < nvec) {
#pragma unroll
        for (int j = 0; j < 8; ++j) { const float c = v[i][j] - mean; sq += c * c; }
      }
    const float rstd = rsqrtf(warp_sum(sq) / d + eps);
    if (kWriteStats && lane == 0) { mean_out[row] = mean; rstd_out[row] = rstd; }
    uint4* yr = reinterpret_cast<uint4*>(y + row * d);
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int vi = lane + 32 * i;
      if (vi < nvec) {
        const float4 w0 = __ldg(reinterpret_cast<const float4*>(w) + 2 * vi), w1 = __ldg(reinterpret_cast<const float4*>(w) + 2 * vi + 1);
        const float4 b0 = __ldg(reinterpret_cast<const float4*>(b) + 2 * vi), b1 = __ldg(reinterpret_cast<const float4*>(b) + 2 * vi + 1);
        const float ww[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
        const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
        float o[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = (v[i][j] - mean) * rstd * ww[j] + bb[j];
        uint4 u;
        u.x = Act16<T>::pack2(o[0], o[1]); u.y = Act16<T>::pack2(o[2], o[3]);
        u.z = Act16<T>::pack2(o[4], o[5]); u.w = Act16<T>::pack2(o[6], o[7]);
        yr[vi] = u;
      }
    }
  }
}

// Backward.  One warp per row (grid-stride), lane l owns the same 8-column vectors l, l+32, ... of every row it visits,
// so the parameter gradients (column sums of dy*xhat and dy) accumulate in that lane's registers with no shared-memory
// traffic and no block barrier inside the row loop; the 8 warps of a block are folded through shared memory once at
// the end into this block's partial column sums, which add_partials adds up in block order.  x and dy stay packed (bf16) in registers between the statistics
// pass and the dx pass and are unpacked twice -- 32 registers instead of 64.  (History: all-fp32-in-registers needed
// 214 registers -> 23 % of the HBM roofline; staging every row through shared memory with two __syncthreads per 8
// rows -> 37 %.)
template <typename T, int NV>
__global__ void __launch_bounds__(256, 2)
layernorm_bwd_kernel(const T* __restrict__ dy, const T* __restrict__ x, const float* __restrict__ w,
                     const float* __restrict__ mean, const float* __restrict__ rstd,
                     const T* __restrict__ dres, T* __restrict__ dx, float* __restrict__ part,
                     int64_t rows, int d) {
  extern __shared__ __align__(16) float fold[];  // [8][d], used once at the end
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int nvec = d >> 3;
  float2 acc_w[NV][4], acc_b[NV][4];
#pragma unroll
  for (int i = 0; i < NV; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) { acc_w[i][j] = make_float2(0.f, 0.f); acc_b[i][j] = make_float2(0.f, 0.f); }

  for (int64_t row = static_cast<int64_t>(blockIdx.x) * 8 + warp; row < rows; row += static_cast<int64_t>(gridDim.x) * 8) {
    const uint4* xr = reinterpret_cast<const uint4*>(x + row * d);
    const uint4* gr = reinterpret_cast<const uint4*>(dy + row * d);
    const uint4* rr = dres ? reinterpret_cast<const uint4*>(dres + row * d) : nullptr;
    uint4 ux[NV], ug[NV];
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int vi = lane + 32 * i;
      if (vi < nvec) { ux[i] = xr[vi]; ug[i] = gr[vi]; }
      else { ux[i] = make_uint4(0, 0, 0, 0); ug[i] = make_uint4(0, 0, 0, 0); }
    }
    {   // pull the next row this warp will visit (and this row's residual gradient) into L2 while this one is processed:
        // one prefetch per 128-byte line (lanes 0, 8, 16, 24 of every 32-vector group)
      const int64_t nrow = row + static_cast<int64_t>(gridDim.x) * 8;
      if ((lane & 7) == 0) {
#pragma unroll
        for (int i = 0; i < NV; ++i) {
          const int vi = lane + 32 * i;
          if (vi < nvec) {
            if (rr) asm volatile("prefetch.global.L2 [%0];" ::"l"(rr + vi));
            if (nrow < rows) {
              asm volatile("prefetch.global.L2 [%0];" ::"l"(reinterpret_cast<const uint4*>(x + nrow * d) + vi));
              asm volatile("prefetch.global.L2 [%0];" ::"l"(reinterpret_cast<const uint4*>(dy + nrow * d) + vi));
            }
          }
        }
      }
    }
    const float mu = mean[row], rs = rstd[row];
    const float2 mu2 = make_float2(mu, mu), rs2 = make_float2(rs, rs);
    float2 s1 = make_float2(0.f, 0.f), s2 = make_float2(0.f, 0.f);
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int vi = lane + 32 * i;
      if (vi < nvec) {
        const float4 w0 = __ldg(reinterpret_cast<const float4*>(w) + 2 * vi), w1 = __ldg(reinterpret_cast<const float4*>(w) + 2 * vi + 1);
        const float2 ww[4] = {make_float2(w0.x, w0.y), make_float2(w0.z, w0.w), make_float2(w1.x, w1.y), make_float2(w1.z, w1.w)};
        const uint32_t xw[4] = {ux[i].x, ux[i].y, ux[i].z, ux[i].w};
        const uint32_t gw[4] = {ug[i].x, ug[i].y, ug[i].z, ug[i].w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 xh = fmul2(fadd2(Act16<T>::unpack2(xw[j]), make_float2(-mu, -mu)), rs2);
          const float2 g = Act16<T>::unpack2(gw[j]);
          const float2 gwj = fmul2(g, ww[j]);
          s1 = fadd2(s1, gwj);
          s2 = ffma2(gwj, xh, s2);
          acc_w[i][j] = ffma2(g, xh, acc_w[i][j]);
          acc_b[i][j] = fadd2(acc_b[i][j], g);
        }
      }
    }
    (void)mu2;
    const float m1 = warp_sum(s1.x + s1.y) / d;
    const float m2 = warp_sum(s2.x + s2.y) / d;
    uint4* dxr = reinterpret_cast<uint4*>(dx + row * d);
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int vi = lane + 32 * i;
      if (vi < nvec) {
        const float4 w0 = __ldg(reinterpret_cast<const float4*>(w) + 2 * vi), w1 = __ldg(reinterpret_cast<const float4*>(w) + 2 * vi + 1);
        const float2 ww[4] = {make_float2(w0.x, w0.y), make_float2(w0.z, w0.w), make_float2(w1.x, w1.y), make_float2(w1.z, w1.w)};
        const uint32_t xw[4] = {ux[i].x, ux[i].y, ux[i].z, ux[i].w};
        const uint32_t gw[4] = {ug[i].x, ug[i].y, ug[i].z, ug[i].w};
        uint4 ur = make_uint4(0, 0, 0, 0);
        if (rr) ur = rr[vi];
        const uint32_t rw[4] = {ur.x, ur.y, ur.z, ur.w};
        uint32_t ow[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 xh = fmul2(fadd2(Act16<T>::unpack2(xw[j]), make_float2(-mu, -mu)), rs2);
          const float2 gwj = fmul2(Act16<T>::unpack2(gw[j]), ww[j]);
          // rs * (g*w - mean(g*w) - xhat * mean(g*w*xhat))
          float2 o = ffma2(xh, make_float2(-m2, -m2), fadd2(gwj, make_float2(-m1, -m1)));
          o = fmul2(o, rs2);
          if (rr) {
            const float2 ob = Act16<T>::unpack2(Act16<T>::pack2(o.x, o.y));   // T(dx_ln) first, like autograd's accumulation
            o = fadd2(Act16<T>::unpack2(rw[j]), ob);
          }
          ow[j] = Act16<T>::pack2(o.x, o.y);
        }
        dxr[vi] = make_uint4(ow[0], ow[1], ow[2], ow[3]);
      }
    }
  }

  // fold the 8 warps' accumulators (two passes through one [8][d] buffer) into part[pass][block][d]
#pragma unroll
  for (int pass = 0; pass < 2; ++pass) {
    __syncthreads();
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int vi = lane + 32 * i;
      if (vi < nvec) {
        float4* dst = reinterpret_cast<float4*>(fold + warp * d + vi * 8);
        const float2* a = pass == 0 ? acc_w[i] : acc_b[i];
        dst[0] = make_float4(a[0].x, a[0].y, a[1].x, a[1].y);
        dst[1] = make_float4(a[2].x, a[2].y, a[3].x, a[3].y);
      }
    }
    __syncthreads();
    float* out = part + (static_cast<int64_t>(pass) * gridDim.x + blockIdx.x) * d;
    for (int c = threadIdx.x; c < d; c += 256) {
      float t = 0.f;
#pragma unroll
      for (int r = 0; r < 8; ++r) t += fold[r * d + c];
      out[c] = t;
    }
  }
}

template <typename T>
int layernorm_fwd(const void* x, const float* weight, const float* bias, void* y, float* mean, float* rstd, int64_t rows,
                  int64_t d, float eps, void* stream) {
  OASR_REQUIRE(rows > 0 && d > 0, "layernorm: empty input");
  OASR_REQUIRE((d & 7) == 0 && d <= LN_MAX_VEC * 256, "layernorm: d=%ld must be a multiple of 8 and <= %d", (long)d, LN_MAX_VEC * 256);
  OASR_REQUIRE((mean == nullptr) == (rstd == nullptr), "layernorm: mean and rstd go together");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int wpb = 8;
  int64_t blocks = ceil_div(rows, wpb);
  const int64_t cap = static_cast<int64_t>(num_sms()) * 16;
  if (blocks > cap) blocks = cap;
#define OASR_LN_FWD(NVv)                                                                                          \
  do {                                                                                                           \
    if (mean)                                                                                                    \
      layernorm_fwd_kernel<T, true, NVv><<<(int)blocks, wpb * 32, 0, st>>>((const T*)x, weight, bias, (T*)y, mean, rstd, rows, (int)d, eps); \
    else                                                                                                         \
      layernorm_fwd_kernel<T, false, NVv><<<(int)blocks, wpb * 32, 0, st>>>((const T*)x, weight, bias, (T*)y, nullptr, nullptr, rows, (int)d, eps); \
  } while (0)
  switch ((int)ceil_div(d, 256)) {
    case 1: case 2: OASR_LN_FWD(2); break;
    case 3: OASR_LN_FWD(3); break;
    case 4: OASR_LN_FWD(4); break;
    default: OASR_LN_FWD(5); break;
  }
#undef OASR_LN_FWD
  OASR_LAUNCH_CHECK();
  return OASR_OK;
}

template <typename T>
int layernorm_bwd(const void* dy, const void* x, const float* weight, const float* mean, const float* rstd,
                  const void* dresidual, void* dx, float* dweight, float* dbias, int64_t rows, int64_t d, void* stream) {
  OASR_REQUIRE(rows > 0 && d > 0, "layernorm_bwd: empty input");
  OASR_REQUIRE((d & 7) == 0 && d <= LN_MAX_VEC * 256, "layernorm_bwd: unsupported d=%ld", (long)d);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int wpb = 8;
  int64_t blocks = ceil_div(rows, wpb);
  const int64_t cap = static_cast<int64_t>(num_sms()) * 2;  // 2 resident blocks per SM; few blocks => few partials
  if (blocks > cap) blocks = cap;
  const size_t smem = 8 * d * sizeof(float);
  float* part = static_cast<float*>(scratch_alloc(sizeof(float) * 2 * blocks * d, st));
  if (!part) return OASR_ERR_CUDA;
#define OASR_LN_BWD(NVv)                                                                                              \
  do {                                                                                                                 \
    static bool attr_set = false;                                                                                      \
    if (!attr_set) {                                                                                                   \
      OASR_CUDA_OK(cudaFuncSetAttribute(layernorm_bwd_kernel<T, NVv>, cudaFuncAttributeMaxDynamicSharedMemorySize, NVv * 256 * 32)); \
      attr_set = true;                                                                                                 \
    }                                                                                                                  \
    layernorm_bwd_kernel<T, NVv><<<(int)blocks, wpb * 32, smem, st>>>(                                                 \
        (const T*)dy, (const T*)x, weight, mean, rstd, (const T*)dresidual, (T*)dx, part, rows, (int)d);             \
  } while (0)
  switch ((int)ceil_div(d, 256)) {
    case 1: case 2: OASR_LN_BWD(2); break;
    case 3: OASR_LN_BWD(3); break;
    case 4: OASR_LN_BWD(4); break;
    default: OASR_LN_BWD(5); break;
  }
#undef OASR_LN_BWD
  OASR_LAUNCH_CHECK();
  // a null dweight / dbias (a frozen affine) skips its reduction
  int rc = dweight ? add_partials(part, (int)blocks, d, dweight, st) : OASR_OK;
  if (rc == OASR_OK && dbias) rc = add_partials(part + blocks * d, (int)blocks, d, dbias, st);
  scratch_free(part, st);
  return rc;
}

}  // namespace
}  // namespace oasr

using namespace oasr;

extern "C" int oasr_layernorm_fwd(const void* x, const float* weight, const float* bias, void* y, float* mean,
                                  float* rstd, int64_t rows, int64_t d, float eps, void* stream) {
  return layernorm_fwd<bf16>(x, weight, bias, y, mean, rstd, rows, d, eps, stream);
}

extern "C" int oasr_layernorm_bwd(const void* dy, const void* x, const float* weight, const float* mean,
                                  const float* rstd, const void* dresidual, void* dx, float* dweight,
                                  float* dbias, int64_t rows, int64_t d, void* stream) {
  return layernorm_bwd<bf16>(dy, x, weight, mean, rstd, dresidual, dx, dweight, dbias, rows, d, stream);
}

extern "C" int oasr_layernorm_fwd16(const void* x, const float* weight, const float* bias, void* y, float* mean,
                                    float* rstd, int64_t rows, int64_t d, float eps, int dtype, void* stream) {
  return OASR_BY_DTYPE16(dtype, layernorm_fwd, x, weight, bias, y, mean, rstd, rows, d, eps, stream);
}

extern "C" int oasr_layernorm_bwd16(const void* dy, const void* x, const float* weight, const float* mean,
                                    const float* rstd, const void* dresidual, void* dx, float* dweight,
                                    float* dbias, int64_t rows, int64_t d, int dtype, void* stream) {
  return OASR_BY_DTYPE16(dtype, layernorm_bwd, dy, x, weight, mean, rstd, dresidual, dx, dweight, dbias, rows, d, stream);
}
