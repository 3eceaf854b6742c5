// Greedy kv-cache decode step (BASELINE.json config 5) as a fixed sequence of HBM-bound kernels that a CUDA graph replays:
// every piece of per-step state (current position, token ids, finished flags) lives on the device.
//
// Replaces, per step and per decoder layer, what the reference does through stock modules
// (olmoasr/inf_model.py:320-362 TextDecoder.forward, :150-196 MultiHeadAttention, :422-453 kv-cache hooks) and the
// third-party greedy loop (whisper/decoding.py: PyTorchInference.logits, SuppressBlank / SuppressTokens,
// GreedyDecoder.update) that drives it from `model.decode` (scripts/eval/eval.py:1846-1847).
//
// The reference's decode step is bound by weight and KV-cache reads (small: 277.8 MB of fp16 weights per step shared by
// all sequences, 55.3 MB of cross-attention K/V per sequence per step), plus a host-built mask, per-call fp32->fp16 weight
// casts and 2 L torch.cat reallocations.  Here:
//   * weights are cast once into the activation dtype (fp16 = upstream default `fp16=True`, or bf16);
//   * dec_linear: a skinny GEMM (<= 64 sequences) that streams each weight row exactly once with 16-byte loads and
//     feeds mma.sync.m16n8k16 (fp32 accumulate); the preceding LayerNorm, the bias, GELU, the residual add and the
//     scatter of new K/V rows into the pre-allocated cache are all fused into it -- 6 of the 10 launches per layer;
//   * dec_attn_scores / dec_attn_pv: single-query attention that reads every cached K and V element once (16-byte
//     loads, 8 lanes per key row), key ranges split over CTAs when batch x heads cannot fill the SMs;
//   * dec_sample: logit filters + argmax + log-prob + eot bookkeeping in one pass over the fp32 logits;
//   * fp8 decoding (oasr_dec_linear_fp8w / oasr_dec_attention_fp8kv): the same kernels instantiated on e4m3 weight or
//     cross K / V storage, half the bytes of the two streams that dominate the step; codes become T in registers and
//     the fp32 scales multiply outside the dot products (include/oasr_b200.h states the arithmetic).
//
// Rounding points are the reference's in the activation dtype T (inf_model.py:172-196): q*hd^-0.25 and k*hd^-0.25 rounded
// to T, q.k accumulated in fp32 and rounded to T, softmax in fp32, probabilities rounded to T, p.v accumulated in fp32 and
// rounded once; every Linear output is round_T(acc + bias_T); LayerNorm is computed in fp32 and rounded once;
// residuals are round_T(x + y); logits are float(round_T(x . E^T)).
#include "common.cuh"

#include <cuda_fp16.h>
#include <limits.h>
#include <stdlib.h>

namespace oasr {
namespace {

// ---------------------------------------------------------------------------------------------------------- dtype traits
template <typename T> struct DT;
template <> struct DT<__half> {
  static __device__ __forceinline__ float to_f(__half v) { return __half2float(v); }
  static __device__ __forceinline__ __half from_f(float v) { return __float2half_rn(v); }
  static __device__ __forceinline__ float2 unpack2(uint32_t u) {
    return __half22float2(*reinterpret_cast<const __half2*>(&u));
  }
  static __device__ __forceinline__ uint32_t pack2(float a, float b) {
    __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
  }
  static __device__ __forceinline__ void mma(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0,
                                             uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
  }
};
template <> struct DT<bf16> {
  static __device__ __forceinline__ float to_f(bf16 v) { return __bfloat162float(v); }
  static __device__ __forceinline__ bf16 from_f(float v) { return __float2bfloat16_rn(v); }
  static __device__ __forceinline__ float2 unpack2(uint32_t u) { return unpack_bf16x2(u); }
  static __device__ __forceinline__ uint32_t pack2(float a, float b) { return pack_bf16x2(a, b); }
  static __device__ __forceinline__ void mma(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0,
                                             uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
  }
};
template <typename T> __device__ __forceinline__ float rnd(float v) { return DT<T>::to_f(DT<T>::from_f(v)); }

// ---------------------------------------------------------------------------------------------------------- stored operands
// Weights and cross K / V are stored either in the activation type T or as e4m3 codes (uint8_t) with fp32 scales applied
// outside the dot product (`fp8=True`, include/oasr_b200.h).  Either way a thread reads 8 consecutive elements at a time
// -- 16 bytes of T or 8 bytes of codes, so 8 lanes on one row still cover whole 32-byte sectors -- and hands them on as
// 8 T values in the uint4 layout of an MMA fragment.  Every e4m3 value is exact in fp16 and in bf16.
__device__ __forceinline__ uint32_t e4m3x2_to_f16x2(uint32_t lo16) {
  uint32_t r;
  asm("cvt.rn.f16x2.e4m3x2 %0, %1;" : "=r"(r) : "h"(static_cast<uint16_t>(lo16)));
  return r;
}
template <typename T> __device__ __forceinline__ uint32_t e4m3x2_to(uint32_t lo16);
template <> __device__ __forceinline__ uint32_t e4m3x2_to<__half>(uint32_t lo16) { return e4m3x2_to_f16x2(lo16); }
template <> __device__ __forceinline__ uint32_t e4m3x2_to<bf16>(uint32_t lo16) {
  const uint32_t h = e4m3x2_to_f16x2(lo16);
  const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&h));
  return pack_bf16x2(f.x, f.y);
}

template <typename T, typename TS> struct Stored;
// Argument block of the skinny-GEMM kernels: 16-bit weights take the public one as it is (so those instantiations keep
// the parameter list, and the code, they had before fp8 existed); e4m3 weights add the (N,) fp32 per-row scales.
struct LinearArgsFp8 : oasr_dec_linear_args {
  const float* w_scale;
};

template <typename T> struct Stored<T, T> {       // 16-bit storage: the loaded bytes are the fragment
  using V = uint4;
  using LinearArgs = oasr_dec_linear_args;
  static constexpr bool kFp8 = false;
  static __device__ __forceinline__ V zero() { return make_uint4(0, 0, 0, 0); }
  static __device__ __forceinline__ V ldg(const T* p) { return __ldg(reinterpret_cast<const uint4*>(p)); }
  static __device__ __forceinline__ uint4 frag(V v) { return v; }
};
template <typename T> struct Stored<T, uint8_t> {  // e4m3 codes, converted in registers
  using V = uint2;
  using LinearArgs = LinearArgsFp8;
  static constexpr bool kFp8 = true;
  static __device__ __forceinline__ V zero() { return make_uint2(0, 0); }
  static __device__ __forceinline__ V ldg(const uint8_t* p) { return __ldg(reinterpret_cast<const uint2*>(p)); }
  static __device__ __forceinline__ uint4 frag(V v) {
    return make_uint4(e4m3x2_to<T>(v.x & 0xffffu), e4m3x2_to<T>(v.x >> 16), e4m3x2_to<T>(v.y & 0xffffu), e4m3x2_to<T>(v.y >> 16));
  }
};

// Per-(key, head) scales of e4m3 cross K / V: element (n, j, h) at k / v + n * seq + j * row + h.  Unused (null) when
// K / V are stored in T.
struct KvScales {
  const float* k; const float* v; int64_t seq; int64_t row;
};

__device__ __forceinline__ float gelu_exact(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f)); }

// Programmatic dependent launch (a decode step is ~120 dependent launches of tiny kernels; at 1-8 sequences their launch
// and first-byte latencies ARE the step time).  Every kernel lets its successor start launching at once
// (launch_dependents) and blocks on wait() -- which returns when the predecessor grid has completed and flushed -- before
// touching anything a predecessor writes.  What does not depend on a predecessor (the weight stream of dec_linear) is
// issued BEFORE wait(), i.e. underneath the predecessor's tail.  Without the launch attribute both are no-ops.
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// ---------------------------------------------------------------------------------------------------------- embedding
// x[n] = T(token_embedding[tokens[n, pos]] + positional_embedding[pos])   (inf_model.py:334-338; fp32 add, one rounding)
template <typename T>
__global__ void dec_embed_kernel(const int32_t* __restrict__ tokens, int64_t ld_tokens, const int32_t* __restrict__ pos_ptr,
                                 const float* __restrict__ emb, const float* __restrict__ pos_emb, T* __restrict__ x, int d,
                                 int n_vocab) {
  pdl_launch_dependents();
  pdl_wait();
  const int n = blockIdx.x;
  const int pos = *pos_ptr;
  int tok = tokens[n * ld_tokens + pos];
  if (tok < 0 || tok >= n_vocab) tok = 0;
  const float* e = emb + static_cast<int64_t>(tok) * d;
  const float* p = pos_emb + static_cast<int64_t>(pos) * d;
  for (int c = threadIdx.x; c < d; c += blockDim.x) x[static_cast<int64_t>(n) * d + c] = DT<T>::from_f(e[c] + p[c]);
}

// ---------------------------------------------------------------------------------------------------------- skinny GEMM
enum { X_PLAIN = 0, X_LAYERNORM = 1, X_PARTIAL_SUM = 2 };
enum { EPI_STORE = 0, EPI_GELU = 1, EPI_RESIDUAL = 2, EPI_LOGITS_F32 = 3, EPI_QKV_SCATTER = 4 };

template <typename T>
__device__ __forceinline__ uint4 load_x8(const oasr_dec_linear_args& a, const float (*s_stat)[2], int row, int k) {
  if (row >= a.M) return make_uint4(0, 0, 0, 0);
  if (a.x_mode == X_PARTIAL_SUM) {   // sum of S fp32 partial outputs of dec_attn_pv, rounded once (the `w @ v` output)
    float v[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    const float* p = static_cast<const float*>(a.x) + static_cast<int64_t>(row) * a.K + k;
    for (int s = 0; s < a.n_partials; ++s) {
      const float4 lo = *reinterpret_cast<const float4*>(p + static_cast<int64_t>(s) * a.partial_stride);
      const float4 hi = *reinterpret_cast<const float4*>(p + static_cast<int64_t>(s) * a.partial_stride + 4);
      v[0] += lo.x; v[1] += lo.y; v[2] += lo.z; v[3] += lo.w; v[4] += hi.x; v[5] += hi.y; v[6] += hi.z; v[7] += hi.w;
    }
    return make_uint4(DT<T>::pack2(v[0], v[1]), DT<T>::pack2(v[2], v[3]), DT<T>::pack2(v[4], v[5]), DT<T>::pack2(v[6], v[7]));
  }
  const uint4 u = *reinterpret_cast<const uint4*>(static_cast<const T*>(a.x) + static_cast<int64_t>(row) * a.ldx + k);
  if (a.x_mode == X_PLAIN) return u;
  // LayerNorm on the fly: fp32 statistics of the whole row (s_stat), affine, one rounding to T (inf_model.py LayerNorm)
  const float mean = s_stat[row][0], rstd = s_stat[row][1];
  const float4 g0 = *reinterpret_cast<const float4*>(a.ln_gamma + k), g1 = *reinterpret_cast<const float4*>(a.ln_gamma + k + 4);
  const float4 b0 = *reinterpret_cast<const float4*>(a.ln_beta + k), b1 = *reinterpret_cast<const float4*>(a.ln_beta + k + 4);
  const float2 x0 = DT<T>::unpack2(u.x), x1 = DT<T>::unpack2(u.y), x2 = DT<T>::unpack2(u.z), x3 = DT<T>::unpack2(u.w);
  return make_uint4(DT<T>::pack2((x0.x - mean) * rstd * g0.x + b0.x, (x0.y - mean) * rstd * g0.y + b0.y),
                    DT<T>::pack2((x1.x - mean) * rstd * g0.z + b0.z, (x1.y - mean) * rstd * g0.w + b0.w),
                    DT<T>::pack2((x2.x - mean) * rstd * g1.x + b1.x, (x2.y - mean) * rstd * g1.y + b1.y),
                    DT<T>::pack2((x3.x - mean) * rstd * g1.z + b1.z, (x3.y - mean) * rstd * g1.w + b1.w));
}

// Direct form for <= 32 sequences (measured faster there than the staged form below: fewer phases, 72 registers, several CTAs
// per SM): y[m, n] = epilogue( sum_k x[m, k] W[n, k] ),  M <= 16 MT rows, one CTA = 16 output columns, 8 warps split K.
// Thread (g = lane / 4, t = lane % 4) loads 16 contiguous bytes of W row n0 + 8 j + g at k0 + 8 t (a warp touches 8 rows x
// 64 B: whole sectors) and the SAME 8 k positions of x rows g, g + 8 of every 16-row tile: the two m16n8k16 MMAs per
// 32-wide k step then use a permuted k order that A and B agree on, so no shuffles and no shared-memory staging are
// needed; x (<= 64 x K, L2 / L1 resident) is re-read by every CTA, W (the HBM stream) exactly once.
// TW: the weight storage (see Stored)
template <typename T, typename TW, int MT>
__global__ void __launch_bounds__(256) dec_linear_direct_kernel(const typename Stored<T, TW>::LinearArgs a) {
  using WS = Stored<T, TW>;
  __shared__ float s_stat[16 * MT][2];
  __shared__ float s_red[8][16 * MT][17];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int n0 = blockIdx.x * 16;
  const int K = a.K;
  pdl_launch_dependents();
  // the weight stream does not depend on the previous kernel: its first round is in flight before pdl_wait()
  const TW* W = static_cast<const TW*>(a.W);
  const int r0 = n0 + g, r1 = n0 + 8 + g;
  const TW* w0 = W + static_cast<int64_t>(r0 < a.N ? r0 : 0) * K + 8 * t;
  const TW* w1 = W + static_cast<int64_t>(r1 < a.N ? r1 : 0) * K + 8 * t;
  const bool ok0 = r0 < a.N, ok1 = r1 < a.N;
  const uint4 zero = make_uint4(0, 0, 0, 0);
  int k0 = warp * 32;
  typename WS::V b0 = WS::zero(), b1 = WS::zero();
  if (k0 < K) {
    b0 = ok0 ? WS::ldg(w0 + k0) : WS::zero();
    b1 = ok1 ? WS::ldg(w1 + k0) : WS::zero();
  }
  pdl_wait();
  if (a.x_mode == X_LAYERNORM) {   // the affine parameters this thread will need: into L1 now, read as hits in the k loop
    for (int k = warp * 32 + 8 * t; k < K; k += 256) {
      asm volatile("prefetch.global.L1 [%0];" ::"l"(a.ln_gamma + k));
      asm volatile("prefetch.global.L1 [%0];" ::"l"(a.ln_beta + k));
    }
  }
  if (a.x_mode == X_LAYERNORM) {   // two-pass fp32 statistics per row (F.layer_norm(x.float()))
    for (int row = warp; row < a.M; row += 8) {
      const T* xr = static_cast<const T*>(a.x) + static_cast<int64_t>(row) * a.ldx;
      float s = 0.f;
      for (int k = lane * 8; k < K; k += 256) {
        const uint4 u = *reinterpret_cast<const uint4*>(xr + k);
        const float2 p0 = DT<T>::unpack2(u.x), p1 = DT<T>::unpack2(u.y), p2 = DT<T>::unpack2(u.z), p3 = DT<T>::unpack2(u.w);
        s += (p0.x + p0.y) + (p1.x + p1.y) + (p2.x + p2.y) + (p3.x + p3.y);
      }
      const float mean = warp_sum(s) / static_cast<float>(K);
      float q = 0.f;
      for (int k = lane * 8; k < K; k += 256) {
        const uint4 u = *reinterpret_cast<const uint4*>(xr + k);
        const float2 p0 = DT<T>::unpack2(u.x), p1 = DT<T>::unpack2(u.y), p2 = DT<T>::unpack2(u.z), p3 = DT<T>::unpack2(u.w);
        const float d0 = p0.x - mean, d1 = p0.y - mean, d2 = p1.x - mean, d3 = p1.y - mean;
        const float d4 = p2.x - mean, d5 = p2.y - mean, d6 = p3.x - mean, d7 = p3.y - mean;
        q += (d0 * d0 + d1 * d1) + (d2 * d2 + d3 * d3) + (d4 * d4 + d5 * d5) + (d6 * d6 + d7 * d7);
      }
      const float var = warp_sum(q) / static_cast<float>(K);
      if (lane == 0) { s_stat[row][0] = mean; s_stat[row][1] = rsqrtf(var + a.ln_eps); }
    }
    __syncthreads();
  }
  float acc[MT][2][4];
#pragma unroll
  for (int i = 0; i < MT; ++i)
#pragma unroll
    for (int j = 0; j < 2; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[i][j][e] = 0.f;

  // x fragments are double-buffered like W: round r + 1's loads (L2 latency each) are in flight under round r's MMAs
  // (fc2 at K = 3072 is 12 rounds per warp: serialised, the x latency alone was ~8 of its 11.5 us at one sequence)
  uint4 xa[MT], xb[MT];
  if (k0 < K) {
#pragma unroll
    for (int i = 0; i < MT; ++i) {
      xa[i] = load_x8<T>(a, s_stat, i * 16 + g, k0 + 8 * t);
      xb[i] = load_x8<T>(a, s_stat, i * 16 + 8 + g, k0 + 8 * t);
    }
  }
  for (; k0 < K; k0 += 256) {
    const int kn = k0 + 256;
    typename WS::V nb0 = WS::zero(), nb1 = WS::zero();
    uint4 nxa[MT], nxb[MT];
    if (kn < K) {   // the HBM stream and the x fragments run one round ahead of the MMAs
      nb0 = ok0 ? WS::ldg(w0 + kn) : WS::zero();
      nb1 = ok1 ? WS::ldg(w1 + kn) : WS::zero();
#pragma unroll
      for (int i = 0; i < MT; ++i) {
        nxa[i] = load_x8<T>(a, s_stat, i * 16 + g, kn + 8 * t);
        nxb[i] = load_x8<T>(a, s_stat, i * 16 + 8 + g, kn + 8 * t);
      }
    } else {
#pragma unroll
      for (int i = 0; i < MT; ++i) { nxa[i] = zero; nxb[i] = zero; }
    }
#pragma unroll
    for (int i = 0; i < MT; ++i) {
      const uint4 f0 = WS::frag(b0), f1 = WS::frag(b1);
      DT<T>::mma(acc[i][0], xa[i].x, xb[i].x, xa[i].y, xb[i].y, f0.x, f0.y);
      DT<T>::mma(acc[i][0], xa[i].z, xb[i].z, xa[i].w, xb[i].w, f0.z, f0.w);
      DT<T>::mma(acc[i][1], xa[i].x, xb[i].x, xa[i].y, xb[i].y, f1.x, f1.y);
      DT<T>::mma(acc[i][1], xa[i].z, xb[i].z, xa[i].w, xb[i].w, f1.z, f1.w);
    }
    b0 = nb0; b1 = nb1;
#pragma unroll
    for (int i = 0; i < MT; ++i) { xa[i] = nxa[i]; xb[i] = nxb[i]; }
  }
  // fixed-order reduction over the 8 K slices (deterministic), then the epilogue
#pragma unroll
  for (int i = 0; i < MT; ++i)
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      s_red[warp][i * 16 + g][j * 8 + 2 * t] = acc[i][j][0];
      s_red[warp][i * 16 + g][j * 8 + 2 * t + 1] = acc[i][j][1];
      s_red[warp][i * 16 + 8 + g][j * 8 + 2 * t] = acc[i][j][2];
      s_red[warp][i * 16 + 8 + g][j * 8 + 2 * t + 1] = acc[i][j][3];
    }
  __syncthreads();
  const int pos = (a.epi == EPI_QKV_SCATTER) ? *a.pos_ptr : 0;
  for (int idx = threadIdx.x; idx < a.M * 16; idx += 256) {
    const int row = idx >> 4, col = idx & 15, n = n0 + col;
    if (n >= a.N) continue;
    float v = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) v += s_red[w][row][col];
    if constexpr (WS::kFp8) v *= __ldg(a.w_scale + n);                // s_n sum_k x Q (include/oasr_b200.h)
    if (a.epi == EPI_LOGITS_F32) {   // (x @ E^T).float(): the matmul output is rounded to T first (inf_model.py:357-360)
      static_cast<float*>(a.out)[static_cast<int64_t>(row) * a.ldo + n] = rnd<T>(v);
      continue;
    }
    if (a.bias) v += rnd<T>(a.bias[n]);                                 // bias.to(x.dtype) (inf_model.py:56-60)
    float y = rnd<T>(v);
    if (a.epi == EPI_GELU) y = gelu_exact(y);
    if (a.epi == EPI_RESIDUAL) y = DT<T>::to_f(static_cast<const T*>(a.res)[static_cast<int64_t>(row) * a.ldres + n]) + y;
    const T o = DT<T>::from_f(y);
    if (a.epi == EPI_QKV_SCATTER) {   // [q | k | v]: q to scratch, k / v appended in place to the static self-attention cache
      const int d = a.N / 3;
      if (n < d) static_cast<T*>(a.out)[static_cast<int64_t>(row) * a.ldo + n] = o;
      else if (n < 2 * d) static_cast<T*>(a.k_cache)[(static_cast<int64_t>(row) * a.cache_len + pos) * d + (n - d)] = o;
      else static_cast<T*>(a.v_cache)[(static_cast<int64_t>(row) * a.cache_len + pos) * d + (n - 2 * d)] = o;
    } else {
      static_cast<T*>(a.out)[static_cast<int64_t>(row) * a.ldo + n] = o;
    }
  }
}

// Staged form (> 32 sequences):
// y[m, n] = epilogue( sum_k x[m, k] W[n, k] ),  M <= 16 MT rows.  One CTA = `groups` consecutive groups of 16 output columns,
// 8 warps split K.
//   * x (or LayerNorm(x), or the rounded sum of the attention partials) is staged ONCE per CTA into shared memory as T --
//     every load of the staging pass is independent, so it costs one L2 latency, and the LayerNorm arithmetic runs once per
//     CTA instead of once per k step -- in rows of K + 32 elements (the +32 makes the 16-byte A-fragment reads of rows g
//     and g + 1 fall into different bank halves);
//   * W is the HBM stream: thread (g = lane / 4, t = lane % 4) loads 16 contiguous bytes of W row n0 + 8 j + g at k0 + 8 t
//     (a warp touches 8 rows x 64 B: whole sectors), four k rounds in flight per warp; the first four are issued BEFORE
//     pdl_wait(), i.e. while the previous kernel is still draining;
//   * the SAME 8 k positions of x rows g, g + 8 feed the A operand, so the two m16n8k16 MMAs per 32-wide k step use a
//     permuted k order that A and B agree on: no shuffles, no transposes;
//   * the 8 K slices are reduced through shared memory in a fixed order (deterministic), then the fused epilogue.
constexpr int DEC_PF = 4;        // W rounds in flight per warp
constexpr int DEC_XPAD = 32;     // elements of row padding in the staged x tile

template <typename T, int R>
__device__ __forceinline__ void stage_rows_layernorm(const oasr_dec_linear_args& a, int row0, int row_step, int lane, T* x_s, int lds) {
  // one warp, R rows (row0, row0 + row_step, ...): each row lives in registers between the mean, the variance and the
  // normalisation (two-pass fp32 statistics like F.layer_norm(x.float()), one rounding to T: inf_model.py LayerNorm).
  // Every global access -- the R rows, and L1 prefetches of the affine parameters -- is issued before the first reduction.
  const int K = a.K;
  uint4 u[R][5];
#pragma unroll
  for (int r = 0; r < R; ++r) {
    const int row = row0 + r * row_step;
    const T* xr = static_cast<const T*>(a.x) + static_cast<int64_t>(row < a.M ? row : 0) * a.ldx;
#pragma unroll
    for (int i = 0; i < 5; ++i) {
      const int k = (lane + 32 * i) * 8;
      u[r][i] = (k < K && row < a.M) ? *reinterpret_cast<const uint4*>(xr + k) : make_uint4(0, 0, 0, 0);
    }
  }
#pragma unroll
  for (int i = 0; i < 5; ++i) {      // the affine parameters this lane will need: pulled into L1 now, read (as hits) below
    const int k = (lane + 32 * i) * 8;
    if (k < K) {
      asm volatile("prefetch.global.L1 [%0];" ::"l"(a.ln_gamma + k));
      asm volatile("prefetch.global.L1 [%0];" ::"l"(a.ln_beta + k));
    }
  }
#pragma unroll
  for (int r = 0; r < R; ++r) {
    const int row = row0 + r * row_step;
    T* dst = x_s + static_cast<size_t>(row) * lds;
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 5; ++i) {
      const float2 p0 = DT<T>::unpack2(u[r][i].x), p1 = DT<T>::unpack2(u[r][i].y), p2 = DT<T>::unpack2(u[r][i].z), p3 = DT<T>::unpack2(u[r][i].w);
      s += (p0.x + p0.y) + (p1.x + p1.y) + (p2.x + p2.y) + (p3.x + p3.y);      // zero-filled beyond K
    }
    const float mean = warp_sum(s) / static_cast<float>(K);
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < 5; ++i) {
      const int k = (lane + 32 * i) * 8;
      if (k < K) {
        const float2 p0 = DT<T>::unpack2(u[r][i].x), p1 = DT<T>::unpack2(u[r][i].y), p2 = DT<T>::unpack2(u[r][i].z), p3 = DT<T>::unpack2(u[r][i].w);
        const float d0 = p0.x - mean, d1 = p0.y - mean, d2 = p1.x - mean, d3 = p1.y - mean;
        const float d4 = p2.x - mean, d5 = p2.y - mean, d6 = p3.x - mean, d7 = p3.y - mean;
        q += (d0 * d0 + d1 * d1) + (d2 * d2 + d3 * d3) + (d4 * d4 + d5 * d5) + (d6 * d6 + d7 * d7);
      }
    }
    const float rstd = rsqrtf(warp_sum(q) / static_cast<float>(K) + a.ln_eps);
#pragma unroll
    for (int i = 0; i < 5; ++i) {
      const int k = (lane + 32 * i) * 8;
      if (k < K) {
        uint4 o = make_uint4(0, 0, 0, 0);
        if (row < a.M) {
          const float4 g0 = *reinterpret_cast<const float4*>(a.ln_gamma + k), g1 = *reinterpret_cast<const float4*>(a.ln_gamma + k + 4);
          const float4 b0 = *reinterpret_cast<const float4*>(a.ln_beta + k), b1 = *reinterpret_cast<const float4*>(a.ln_beta + k + 4);
          const float2 x0 = DT<T>::unpack2(u[r][i].x), x1 = DT<T>::unpack2(u[r][i].y), x2 = DT<T>::unpack2(u[r][i].z), x3 = DT<T>::unpack2(u[r][i].w);
          o = make_uint4(DT<T>::pack2((x0.x - mean) * rstd * g0.x + b0.x, (x0.y - mean) * rstd * g0.y + b0.y),
                         DT<T>::pack2((x1.x - mean) * rstd * g0.z + b0.z, (x1.y - mean) * rstd * g0.w + b0.w),
                         DT<T>::pack2((x2.x - mean) * rstd * g1.x + b1.x, (x2.y - mean) * rstd * g1.y + b1.y),
                         DT<T>::pack2((x3.x - mean) * rstd * g1.z + b1.z, (x3.y - mean) * rstd * g1.w + b1.w));
        }
        *reinterpret_cast<uint4*>(dst + k) = o;
      }
    }
  }
}

template <typename T>
__device__ __forceinline__ uint4 load_x_plain_or_partial(const oasr_dec_linear_args& a, int row, int k) {
  if (a.x_mode == X_PARTIAL_SUM) {   // sum of the fp32 partial outputs of the attention kernels, rounded once (the `w @ v` output)
    float v[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    const float* p = static_cast<const float*>(a.x) + static_cast<int64_t>(row) * a.K + k;
    for (int s = 0; s < a.n_partials; ++s) {
      const float4 lo = *reinterpret_cast<const float4*>(p + static_cast<int64_t>(s) * a.partial_stride);
      const float4 hi = *reinterpret_cast<const float4*>(p + static_cast<int64_t>(s) * a.partial_stride + 4);
      v[0] += lo.x; v[1] += lo.y; v[2] += lo.z; v[3] += lo.w; v[4] += hi.x; v[5] += hi.y; v[6] += hi.z; v[7] += hi.w;
    }
    return make_uint4(DT<T>::pack2(v[0], v[1]), DT<T>::pack2(v[2], v[3]), DT<T>::pack2(v[4], v[5]), DT<T>::pack2(v[6], v[7]));
  }
  return *reinterpret_cast<const uint4*>(static_cast<const T*>(a.x) + static_cast<int64_t>(row) * a.ldx + k);
}

template <typename T, typename TW, int MT>
__global__ void __launch_bounds__(256, (MT <= 2 ? 2 : 1)) dec_linear_kernel(const typename Stored<T, TW>::LinearArgs a, const int KC,
                                                                          const int groups) {
  using WS = Stored<T, TW>;
  constexpr int MP = 16 * MT;
  extern __shared__ __align__(16) uint8_t dec_smem[];
  const int K = a.K;
  const int lds = KC + DEC_XPAD;                                   // staged row length in elements
  T* x_s = reinterpret_cast<T*>(dec_smem);
  float (*s_red)[MP][17] = reinterpret_cast<float (*)[MP][17]>(dec_smem + static_cast<size_t>(MP) * lds * sizeof(T));
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const TW* W = static_cast<const TW*>(a.W);
  const uint4 zero = make_uint4(0, 0, 0, 0);
  const int group0 = blockIdx.x * groups;
  const int n_groups_total = (a.N + 15) / 16;
  pdl_launch_dependents();

  // W rows of a column group for this thread, and the prefetch ring (DEC_PF rounds x 2 n8 tiles)
  typename WS::V wb0[DEC_PF], wb1[DEC_PF];
  auto w_ptrs = [&](int grp, const TW*& w0, const TW*& w1, bool& ok0, bool& ok1) {
    const int r0 = grp * 16 + g, r1 = r0 + 8;
    ok0 = r0 < a.N; ok1 = r1 < a.N;
    w0 = W + static_cast<int64_t>(ok0 ? r0 : 0) * K + 8 * t;
    w1 = W + static_cast<int64_t>(ok1 ? r1 : 0) * K + 8 * t;
  };
  const TW *w0, *w1;
  bool ok0, ok1;
  w_ptrs(group0, w0, w1, ok0, ok1);
#pragma unroll
  for (int p = 0; p < DEC_PF; ++p) {
    const int k = warp * 32 + 256 * p;
    wb0[p] = (ok0 && k < K) ? WS::ldg(w0 + k) : WS::zero();
    wb1[p] = (ok1 && k < K) ? WS::ldg(w1 + k) : WS::zero();
  }
  pdl_wait();     // from here on data written by earlier kernels of the step (x, partials, pos) may be read

  const int pos = (a.epi == EPI_QKV_SCATTER) ? *a.pos_ptr : 0;
  const bool single_chunk = (KC >= K);
  auto stage = [&](int kc0) {     // x[:, kc0 : kc0 + KC) -> shared memory as T (rows >= M are zero)
    const int kc = min(KC, K - kc0);
    if (a.x_mode == X_LAYERNORM) {                       // whole rows (KC >= K is guaranteed by the host)
      // warp w owns rows w, w + 8, ...: MT of them, two at a time (all their loads in flight together)
      if constexpr (MT == 1) {
        stage_rows_layernorm<T, 2>(a, warp, 8, lane, x_s, lds);
      } else {
#pragma unroll 1
        for (int i = 0; i < 2 * MT; i += 2) stage_rows_layernorm<T, 2>(a, warp + 8 * i, 8, lane, x_s, lds);
      }
    } else {
      const int vec = kc >> 3;
      const int items = MP * vec;
      for (int idx0 = threadIdx.x; idx0 < items; idx0 += 256 * 4) {       // 4 independent loads in flight per thread
        uint4 val[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int idx = idx0 + 256 * q;
          const int row = idx / vec, v = idx - row * vec;
          val[q] = (idx < items && row < a.M) ? load_x_plain_or_partial<T>(a, row, kc0 + v * 8) : zero;
        }
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int idx = idx0 + 256 * q;
          const int row = idx / vec, v = idx - row * vec;
          if (idx < items) *reinterpret_cast<uint4*>(x_s + static_cast<size_t>(row) * lds + v * 8) = val[q];
        }
      }
    }
  };
  if (single_chunk) { stage(0); __syncthreads(); }

  for (int gi = 0; gi < groups; ++gi) {
    const int grp = group0 + gi;
    if (grp >= n_groups_total) break;
    const int n0 = grp * 16;
    float acc[MT][2][4];
#pragma unroll
    for (int i = 0; i < MT; ++i)
#pragma unroll
      for (int j = 0; j < 2; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) acc[i][j][e] = 0.f;
    // W pointers of the NEXT group: the ring is refilled from it once this group's rounds are all in flight
    const TW *nw0 = w0, *nw1 = w1;
    bool nok0 = false, nok1 = false;
    const bool has_next = (gi + 1 < groups) && (grp + 1 < n_groups_total);
    if (has_next) w_ptrs(grp + 1, nw0, nw1, nok0, nok1);

    for (int cb = 0; cb < K; cb += 256 * DEC_PF) {        // the same trip count for every warp (barriers inside)
      const int base = cb + warp * 32;
      if (!single_chunk) {                                // K-chunked staging (only the widest inputs: fc2 at 64 sequences)
        __syncthreads();                                  // previous chunk fully consumed
        stage(cb);
        __syncthreads();
      }
      const int kc0 = single_chunk ? 0 : cb;
#pragma unroll
      for (int p = 0; p < DEC_PF; ++p) {
        const int k0 = base + 256 * p;
        if (k0 < K) {
          const uint4 b0 = WS::frag(wb0[p]), b1 = WS::frag(wb1[p]);
          // refill this ring slot with the same group's round p + DEC_PF (if there is one)
          const int kn = k0 + 256 * DEC_PF;
          if (kn < K) {
            wb0[p] = ok0 ? WS::ldg(w0 + kn) : WS::zero();
            wb1[p] = ok1 ? WS::ldg(w1 + kn) : WS::zero();
          }
          const T* xrow = x_s + (k0 - kc0) + 8 * t;
#pragma unroll
          for (int i = 0; i < MT; ++i) {
            const uint4 xa = *reinterpret_cast<const uint4*>(xrow + static_cast<size_t>(i * 16 + g) * lds);
            const uint4 xb = *reinterpret_cast<const uint4*>(xrow + static_cast<size_t>(i * 16 + 8 + g) * lds);
            DT<T>::mma(acc[i][0], xa.x, xb.x, xa.y, xb.y, b0.x, b0.y);
            DT<T>::mma(acc[i][0], xa.z, xb.z, xa.w, xb.w, b0.z, b0.w);
            DT<T>::mma(acc[i][1], xa.x, xb.x, xa.y, xb.y, b1.x, b1.y);
            DT<T>::mma(acc[i][1], xa.z, xb.z, xa.w, xb.w, b1.z, b1.w);
          }
        }
      }
    }
    // next group's first DEC_PF rounds go in flight now, underneath this group's reduction and epilogue
    if (has_next) {
      w0 = nw0; w1 = nw1; ok0 = nok0; ok1 = nok1;
#pragma unroll
      for (int p = 0; p < DEC_PF; ++p) {
        const int k = warp * 32 + 256 * p;
        wb0[p] = (ok0 && k < K) ? WS::ldg(w0 + k) : WS::zero();
        wb1[p] = (ok1 && k < K) ? WS::ldg(w1 + k) : WS::zero();
      }
    }
    // fixed-order reduction over the 8 K slices (deterministic), then the epilogue
#pragma unroll
    for (int i = 0; i < MT; ++i)
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        s_red[warp][i * 16 + g][j * 8 + 2 * t] = acc[i][j][0];
        s_red[warp][i * 16 + g][j * 8 + 2 * t + 1] = acc[i][j][1];
        s_red[warp][i * 16 + 8 + g][j * 8 + 2 * t] = acc[i][j][2];
        s_red[warp][i * 16 + 8 + g][j * 8 + 2 * t + 1] = acc[i][j][3];
      }
    __syncthreads();
    for (int idx = threadIdx.x; idx < a.M * 16; idx += 256) {
      const int row = idx >> 4, col = idx & 15, n = n0 + col;
      if (n >= a.N) continue;
      float v = 0.f;
#pragma unroll
      for (int w = 0; w < 8; ++w) v += s_red[w][row][col];
      if constexpr (WS::kFp8) v *= __ldg(a.w_scale + n);              // s_n sum_k x Q (include/oasr_b200.h)
      if (a.epi == EPI_LOGITS_F32) {   // (x @ E^T).float(): the matmul output is rounded to T first (inf_model.py:357-360)
        static_cast<float*>(a.out)[static_cast<int64_t>(row) * a.ldo + n] = rnd<T>(v);
        continue;
      }
      if (a.bias) v += rnd<T>(a.bias[n]);                                 // bias.to(x.dtype) (inf_model.py:56-60)
      float y = rnd<T>(v);
      if (a.epi == EPI_GELU) y = gelu_exact(y);
      if (a.epi == EPI_RESIDUAL) y = DT<T>::to_f(static_cast<const T*>(a.res)[static_cast<int64_t>(row) * a.ldres + n]) + y;
      const T o = DT<T>::from_f(y);
      if (a.epi == EPI_QKV_SCATTER) {   // [q | k | v]: q to scratch, k / v appended in place to the static self-attention cache
        const int d = a.N / 3;
        if (n < d) static_cast<T*>(a.out)[static_cast<int64_t>(row) * a.ldo + n] = o;
        else if (n < 2 * d) static_cast<T*>(a.k_cache)[(static_cast<int64_t>(row) * a.cache_len + pos) * d + (n - d)] = o;
        else static_cast<T*>(a.v_cache)[(static_cast<int64_t>(row) * a.cache_len + pos) * d + (n - 2 * d)] = o;
      } else {
        static_cast<T*>(a.out)[static_cast<int64_t>(row) * a.ldo + n] = o;
      }
    }
    __syncthreads();     // s_red is reused by the next column group
  }
}

// ---------------------------------------------------------------------------------------------------------- attention
// scores[n, h, j] = float(round_T( sum_c round_T(q[c] * hd^-.25) * round_T(k_j[c] * hd^-.25) ))    (inf_model.py:176-181)
// grid (splits, H, N), 128 threads: 8 lanes per key row (16 bytes = 8 dims each), 16 keys per pass.
template <typename T, typename TKV>
__global__ void __launch_bounds__(128) dec_attn_scores_kernel(const oasr_dec_attn_args a, const int kv_group, const KvScales ks) {
  using KS = Stored<T, TKV>;
  pdl_launch_dependents();
  pdl_wait();
  const int s = blockIdx.x, h = blockIdx.y, n = blockIdx.z;
  const int nkeys = a.pos_ptr ? (*a.pos_ptr + 1) : a.n_keys;
  const int per = (nkeys + gridDim.x - 1) / gridDim.x;
  const int j0 = s * per, j1 = min(nkeys, j0 + per);
  const int c8 = threadIdx.x & 7, slot = threadIdx.x >> 3;
  const float scale = a.scale;
  float qs[8];
  {
    const uint4 u = *reinterpret_cast<const uint4*>(static_cast<const T*>(a.q) + static_cast<int64_t>(n) * a.ldq + h * 64 + c8 * 8);
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 p = DT<T>::unpack2(w[i]);
      qs[2 * i] = rnd<T>(p.x * scale); qs[2 * i + 1] = rnd<T>(p.y * scale);
    }
  }
  const int64_t kv_n = n / kv_group;
  const TKV* kb = static_cast<const TKV*>(a.k) + kv_n * a.kv_seq_stride + h * 64 + c8 * 8;
  float* out = a.scores + (static_cast<int64_t>(n) * gridDim.y + h) * a.scores_ld;
  for (int jb = j0; jb < j1; jb += 128) {   // 8 independent 16-byte (e4m3: 8-byte) loads in flight per thread
    typename KS::V u[8];
    float sk[8];
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      const int j = jb + r * 16 + slot;
      u[r] = (j < j1) ? KS::ldg(kb + static_cast<int64_t>(j) * a.kv_row_stride) : KS::zero();
      if constexpr (KS::kFp8) sk[r] = (j < j1) ? __ldg(ks.k + kv_n * ks.seq + static_cast<int64_t>(j) * ks.row + h) : 0.f;
    }
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      const uint4 f = KS::frag(u[r]);
      const uint32_t w[4] = {f.x, f.y, f.z, f.w};
      float acc = 0.f;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float2 p = DT<T>::unpack2(w[i]);
        if constexpr (KS::kFp8) {          // q~ . QK, scaled once below
          acc = fmaf(qs[2 * i], p.x, acc);
          acc = fmaf(qs[2 * i + 1], p.y, acc);
        } else {
          acc = fmaf(qs[2 * i], rnd<T>(p.x * scale), acc);
          acc = fmaf(qs[2 * i + 1], rnd<T>(p.y * scale), acc);
        }
      }
      acc += __shfl_xor_sync(0xffffffffu, acc, 1);
      acc += __shfl_xor_sync(0xffffffffu, acc, 2);
      acc += __shfl_xor_sync(0xffffffffu, acc, 4);
      if constexpr (KS::kFp8) acc *= sk[r] * scale;
      const int j = jb + r * 16 + slot;
      if (c8 == 0 && j < j1) out[j] = rnd<T>(acc);
    }
  }
}

// partial[s, n, h*64 + c] = sum_{j in split s} float(round_T(softmax(scores)[j])) * v_j[c]   (fp32; the consumer adds the
// splits in order and rounds once = the single rounding of `w @ v`).  Every CTA first derives the row maximum and the
// normaliser from ALL scores of its (n, h) (<= 1500 floats, L2-resident), as F.softmax(qk.float()) does.
template <typename T, typename TKV>
__global__ void __launch_bounds__(128) dec_attn_pv_kernel(const oasr_dec_attn_args a, const int kv_group, const KvScales ks) {
  using KS = Stored<T, TKV>;
  __shared__ float s_part[4];
  __shared__ float s_o[4][64];
  pdl_launch_dependents();
  pdl_wait();
  const int s = blockIdx.x, h = blockIdx.y, n = blockIdx.z;
  const int nkeys = a.pos_ptr ? (*a.pos_ptr + 1) : a.n_keys;
  const int per = (nkeys + gridDim.x - 1) / gridDim.x;
  const int j0 = s * per, j1 = min(nkeys, j0 + per);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const float* sc = a.scores + (static_cast<int64_t>(n) * gridDim.y + h) * a.scores_ld;
  float m = -INFINITY;
  for (int j = threadIdx.x; j < nkeys; j += 128) m = fmaxf(m, sc[j]);
  m = warp_max(m);
  if (lane == 0) s_part[warp] = m;
  __syncthreads();
  m = fmaxf(fmaxf(s_part[0], s_part[1]), fmaxf(s_part[2], s_part[3]));
  __syncthreads();
  float l = 0.f;
  for (int j = threadIdx.x; j < nkeys; j += 128) l += expf(sc[j] - m);
  l = warp_sum(l);
  if (lane == 0) s_part[warp] = l;
  __syncthreads();
  l = (s_part[0] + s_part[1]) + (s_part[2] + s_part[3]);
  const float inv_l = 1.0f / l;

  const int c8 = threadIdx.x & 7, slot = threadIdx.x >> 3;
  const int64_t kv_n = n / kv_group;
  const TKV* vb = static_cast<const TKV*>(a.v) + kv_n * a.kv_seq_stride + h * 64 + c8 * 8;
  float o[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  for (int jb = j0; jb < j1; jb += 128) {
    typename KS::V u[8];
    float p[8];
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      const int j = jb + r * 16 + slot;
      const bool ok = j < j1;
      u[r] = ok ? KS::ldg(vb + static_cast<int64_t>(j) * a.kv_row_stride) : KS::zero();
      p[r] = ok ? rnd<T>(expf(sc[j] - m) * inv_l) : 0.f;            // softmax(...).to(q.dtype)
      if constexpr (KS::kFp8) p[r] *= ok ? __ldg(ks.v + kv_n * ks.seq + static_cast<int64_t>(j) * ks.row + h) : 0.f;   // p_j sV_j
    }
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      const uint4 f = KS::frag(u[r]);
      const uint32_t w[4] = {f.x, f.y, f.z, f.w};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float2 vv = DT<T>::unpack2(w[i]);
        o[2 * i] = fmaf(p[r], vv.x, o[2 * i]);
        o[2 * i + 1] = fmaf(p[r], vv.y, o[2 * i + 1]);
      }
    }
  }
  // 16 key slots -> one: lanes with equal c8 inside the warp (xor 8, 16), then the 4 warps through shared memory
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    o[i] += __shfl_xor_sync(0xffffffffu, o[i], 8);
    o[i] += __shfl_xor_sync(0xffffffffu, o[i], 16);
  }
  if (lane < 8) {
#pragma unroll
    for (int i = 0; i < 8; ++i) s_o[warp][lane * 8 + i] = o[i];
  }
  __syncthreads();
  if (threadIdx.x < 64) {
    const int c = threadIdx.x;
    const float v = (s_o[0][c] + s_o[1][c]) + (s_o[2][c] + s_o[3][c]);
    a.out_partial[(static_cast<int64_t>(s) * gridDim.z + n) * a.ld_out + h * 64 + c] = v;
  }
}

// One CTA per (n, h) when the key range is not split (self-attention always; cross-attention once n x heads fills the
// machine): scores stay in shared memory, softmax and P V follow in the same kernel -- one launch and no round trip through
// global memory instead of two.  Same arithmetic and rounding points as the two-kernel form above.
template <typename T, typename TKV>
__global__ void __launch_bounds__(128) dec_attn_fused_kernel(const oasr_dec_attn_args a, const int kv_group, const KvScales ks) {
  using KS = Stored<T, TKV>;
  __shared__ float s_sc[1536];
  __shared__ float s_part[4];
  __shared__ float s_o[4][64];
  pdl_launch_dependents();
  pdl_wait();
  const int h = blockIdx.y, n = blockIdx.z;
  const int nkeys = a.pos_ptr ? (*a.pos_ptr + 1) : a.n_keys;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int c8 = threadIdx.x & 7, slot = threadIdx.x >> 3;
  const float scale = a.scale;
  float qs[8];
  {
    const uint4 u = *reinterpret_cast<const uint4*>(static_cast<const T*>(a.q) + static_cast<int64_t>(n) * a.ldq + h * 64 + c8 * 8);
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 p = DT<T>::unpack2(w[i]);
      qs[2 * i] = rnd<T>(p.x * scale); qs[2 * i + 1] = rnd<T>(p.y * scale);
    }
  }
  const int64_t kv_n = n / kv_group;
  const TKV* kb = static_cast<const TKV*>(a.k) + kv_n * a.kv_seq_stride + h * 64 + c8 * 8;
  const TKV* vb = static_cast<const TKV*>(a.v) + kv_n * a.kv_seq_stride + h * 64 + c8 * 8;
  float m = -INFINITY;
  for (int jb = 0; jb < nkeys; jb += 128) {
    typename KS::V u[8];
    float sk[8];
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      const int j = jb + r * 16 + slot;
      u[r] = (j < nkeys) ? KS::ldg(kb + static_cast<int64_t>(j) * a.kv_row_stride) : KS::zero();
      if constexpr (KS::kFp8) sk[r] = (j < nkeys) ? __ldg(ks.k + kv_n * ks.seq + static_cast<int64_t>(j) * ks.row + h) : 0.f;
    }
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      const uint4 f = KS::frag(u[r]);
      const uint32_t w[4] = {f.x, f.y, f.z, f.w};
      float acc = 0.f;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float2 p = DT<T>::unpack2(w[i]);
        if constexpr (KS::kFp8) {
          acc = fmaf(qs[2 * i], p.x, acc);
          acc = fmaf(qs[2 * i + 1], p.y, acc);
        } else {
          acc = fmaf(qs[2 * i], rnd<T>(p.x * scale), acc);
          acc = fmaf(qs[2 * i + 1], rnd<T>(p.y * scale), acc);
        }
      }
      acc += __shfl_xor_sync(0xffffffffu, acc, 1);
      acc += __shfl_xor_sync(0xffffffffu, acc, 2);
      acc += __shfl_xor_sync(0xffffffffu, acc, 4);
      if constexpr (KS::kFp8) acc *= sk[r] * scale;
      const int j = jb + r * 16 + slot;
      if (j < nkeys) {
        const float sc = rnd<T>(acc);
        if (c8 == 0) s_sc[j] = sc;
        m = fmaxf(m, sc);
      }
    }
  }
  m = warp_max(m);
  if (lane == 0) s_part[warp] = m;
  __syncthreads();
  m = fmaxf(fmaxf(s_part[0], s_part[1]), fmaxf(s_part[2], s_part[3]));
  __syncthreads();
  float l = 0.f;
  for (int j = threadIdx.x; j < nkeys; j += 128) l += expf(s_sc[j] - m);
  l = warp_sum(l);
  if (lane == 0) s_part[warp] = l;
  __syncthreads();
  l = (s_part[0] + s_part[1]) + (s_part[2] + s_part[3]);
  const float inv_l = 1.0f / l;
  float o[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  for (int jb = 0; jb < nkeys; jb += 128) {
    typename KS::V u[8];
    float p[8];
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      const int j = jb + r * 16 + slot;
      const bool ok = j < nkeys;
      u[r] = ok ? KS::ldg(vb + static_cast<int64_t>(j) * a.kv_row_stride) : KS::zero();
      p[r] = ok ? rnd<T>(expf(s_sc[j] - m) * inv_l) : 0.f;
      if constexpr (KS::kFp8) p[r] *= ok ? __ldg(ks.v + kv_n * ks.seq + static_cast<int64_t>(j) * ks.row + h) : 0.f;
    }
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      const uint4 f = KS::frag(u[r]);
      const uint32_t w[4] = {f.x, f.y, f.z, f.w};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float2 vv = DT<T>::unpack2(w[i]);
        o[2 * i] = fmaf(p[r], vv.x, o[2 * i]);
        o[2 * i + 1] = fmaf(p[r], vv.y, o[2 * i + 1]);
      }
    }
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    o[i] += __shfl_xor_sync(0xffffffffu, o[i], 8);
    o[i] += __shfl_xor_sync(0xffffffffu, o[i], 16);
  }
  if (lane < 8) {
#pragma unroll
    for (int i = 0; i < 8; ++i) s_o[warp][lane * 8 + i] = o[i];
  }
  __syncthreads();
  if (threadIdx.x < 64) {
    const int c = threadIdx.x;
    a.out_partial[static_cast<int64_t>(n) * a.ld_out + h * 64 + c] = (s_o[0][c] + s_o[1][c]) + (s_o[2][c] + s_o[3][c]);
  }
}

// ---------------------------------------------------------------------------------------------------------- sampling
constexpr int BEAM_SCR = 48;                // floats of scratch per (row, slice): rule-aware sampling and beam candidates

// Per-row logit filter of one step (every rule an index test): SuppressTokens, SuppressBlank and, with `ts_on`,
// ApplyTimestampRules.  Used by the sampling step and by beam search.
struct BeamFilter {
  const uint8_t* suppress;
  int first, blank_eot, eot, blank;
  int ts_on, no_ts, ts_begin;
  int ban_text, ban_below_eot;     // ban [0, ts_begin) / ban [0, eot)
  int ts_lo, ts_hi;                // allowed timestamps: [ts_lo, ts_hi)
  __device__ __forceinline__ bool banned(int v) const {
    if (suppress[v]) return true;
    if (blank_eot && (v == blank || v == eot)) return true;
    if (!ts_on) return false;
    if (v == no_ts) return true;
    if (v < ts_begin) return ban_text || (ban_below_eot && v < eot);
    return v < ts_lo || v >= ts_hi;
  }
};

// The filter of row `trow` at position `pos`.  With timestamps on, every thread of the block must call it (block-wide
// reduction over the row's history; s_red holds one int per warp).
__device__ BeamFilter beam_filter(const uint8_t* suppress, const int32_t* trow, int pos, int sample_begin, int suppress_blank,
                                  int blank, int eot, int timestamps, int timestamp_begin, int no_timestamps,
                                  int max_initial_timestamp, int n_vocab, int* s_red) {
  BeamFilter f;
  f.suppress = suppress;
  f.first = pos == sample_begin - 1;
  f.blank_eot = f.first && suppress_blank;
  f.eot = eot; f.blank = blank;
  f.ts_on = timestamps; f.no_ts = no_timestamps; f.ts_begin = timestamp_begin;
  f.ban_text = 0; f.ban_below_eot = 0; f.ts_lo = timestamp_begin; f.ts_hi = n_vocab;
  if (!timestamps) return f;
  // ApplyTimestampRules over seq = tokens[sample_begin .. pos]: the last timestamp (block max over positions)
  int last = -1;
  for (int p = sample_begin + threadIdx.x; p <= pos; p += blockDim.x)
    if (trow[p] >= timestamp_begin) last = p;
  last = __reduce_max_sync(0xffffffffu, last);
  if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = last;
  __syncthreads();
  last = -1;
  for (int w = 0; w < (int)(blockDim.x >> 5); ++w) last = max(last, s_red[w]);
  __syncthreads();
  const int len = pos + 1 - sample_begin;
  const bool last_ts = len >= 1 && trow[pos] >= timestamp_begin;
  const bool penult_ts = len < 2 || trow[pos - 1] >= timestamp_begin;
  if (last_ts) {
    if (penult_ts) f.ts_lo = n_vocab;          // a timestamp pair is closed: text must follow
    else f.ban_below_eot = 1;                  // an open timestamp: another timestamp or eot
  }
  if (last >= 0) {                             // timestamps never decrease (strictly increase after a closed pair)
    const int t = trow[last];
    f.ts_lo = max(f.ts_lo, (last_ts && !penult_ts) ? t : t + 1);
  }
  if (len == 0) {                              // the first sampled token is a timestamp, within the initial window
    f.ban_text = 1;
    if (max_initial_timestamp >= 0) f.ts_hi = min(f.ts_hi, timestamp_begin + max_initial_timestamp + 1);
  }
  return f;
}

// Philox4x32-10 (Salmon et al., "Parallel random numbers: as easy as 1, 2, 3", SC 2011): 4 x 32 random bits per
// (counter, key).  The sampler keys it on the row's 64-bit stream key and counts with (vocabulary id / 4, position).
__device__ __forceinline__ uint4 philox4x32_10(uint32_t c0, uint32_t c1, uint32_t k0, uint32_t k1) {
  uint32_t c2 = 0, c3 = 0;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    if (r > 0) { k0 += 0x9E3779B9u; k1 += 0xBB67AE85u; }
    const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
    c0 = hi1 ^ c1 ^ k0; c1 = lo1; c2 = hi0 ^ c3 ^ k1; c3 = lo0;
  }
  return make_uint4(c0, c1, c2, c3);
}
__device__ __forceinline__ uint32_t word_of(const uint4& r, int i) { return i == 0 ? r.x : i == 1 ? r.y : i == 2 ? r.z : r.w; }
// Gumbel(0, 1) from 23 random bits: u = (k + 1/2) / 2^23 lies in (0, 1) and is exact in fp32; g = -log(-log u)
__device__ __forceinline__ float gumbel(uint32_t bits) {
  const float u = (__uint2float_rn(bits >> 9) + 0.5f) * 0x1p-23f;
  return -logf(-logf(u));
}

// `n_slices` blocks per sequence, each over a contiguous slice of its fp32 logits row, one online pass with 16-byte loads
// (whisper/decoding.py: SuppressBlank, SuppressTokens, ApplyTimestampRules, GreedyDecoder.update); the block that arrives
// last at the sequence's counter merges the slices in slice order (deterministic) and does the bookkeeping:
//   * at pos == sot_index: no_speech_prob = softmax(raw logits)[no_speech]                       (DecodingTask._main_loop)
//   * suppress[v] != 0 -> -inf; at the first sampled position also `blank` and `eot`            (SuppressTokens / SuppressBlank)
//   * TS: every timestamp rule as an index test (BeamFilter), and "timestamp mass beats every text token": the text
//     region [0, timestamp_begin) and the timestamp region keep separate statistics, so lse(ts) > max(text) (both
//     sides share one normaliser: raw logits compare) is decided after the merge, without a second pass
//   * next = argmax (lowest index on ties), or with SAMPLING and *temperature > 0 the Gumbel-max draw
//     argmax_v x_v / T + g_v (lowest index on ties), a sample of softmax(filtered / T) (Categorical(logits / T).sample())
//   * logprob = logit[next] - logsumexp(filtered row) at temperature 1 (GreedyDecoder.update)
//   * sum_logprobs += logprob unless the previous token is eot; rows whose previous token is eot keep emitting eot
// Positions before sample_begin - 1 are teacher-forced: nothing is written there.  The draw of row n at position p is a
// function of (row_keys[n], p, vocabulary id) only: not of the slice split, the block order or the row's batch slot.
struct RegionAcc {          // one vocabulary region: online (max, sum exp) of the filtered row, its argmax, best Gumbel draw
  float m, s, g;
  int arg, gid;
};
template <int NR>
struct SampleAcc {          // raw (max, sum exp) + the regions (the whole row, or text | timestamps)
  float mraw, sraw;
  RegionAcc r[NR];
};
template <int NR>
__device__ __forceinline__ void acc_init(SampleAcc<NR>& s, int V) {
  s.mraw = -INFINITY; s.sraw = 0.f;
#pragma unroll
  for (int q = 0; q < NR; ++q) s.r[q] = RegionAcc{-INFINITY, 0.f, -INFINITY, V, V};
}
template <int NR>
__device__ __forceinline__ void acc_raw(SampleAcc<NR>& s, float x) {
  if (x > s.mraw) { s.sraw = s.sraw * expf(s.mraw - x) + 1.f; s.mraw = x; }
  else s.sraw += expf(x - s.mraw);
}
__device__ __forceinline__ void acc_filt(RegionAcc& s, float x, int v) {
  if (x > s.m) { s.s = s.s * expf(s.m - x) + 1.f; s.m = x; s.arg = v; }
  else { s.s += expf(x - s.m); if (x == s.m && v < s.arg) s.arg = v; }
}
__device__ __forceinline__ void acc_draw(RegionAcc& s, float y, int v) {
  if (y > s.g || (y == s.g && v < s.gid)) { s.g = y; s.gid = v; }
}
template <bool SAMPLING>
__device__ __forceinline__ RegionAcc region_merge(const RegionAcc& a, const RegionAcc& b) {
  RegionAcc r;
  r.m = fmaxf(a.m, b.m);
  r.s = (r.m == -INFINITY) ? 0.f : a.s * expf(a.m - r.m) + b.s * expf(b.m - r.m);
  r.arg = (a.m > b.m || (a.m == b.m && a.arg < b.arg)) ? a.arg : b.arg;
  if constexpr (SAMPLING) {
    const bool ta = a.g > b.g || (a.g == b.g && a.gid < b.gid);
    r.g = ta ? a.g : b.g; r.gid = ta ? a.gid : b.gid;
  } else {
    r.g = -INFINITY; r.gid = a.gid;
  }
  return r;
}
template <int NR, bool SAMPLING>
__device__ __forceinline__ SampleAcc<NR> acc_merge(const SampleAcc<NR>& a, const SampleAcc<NR>& b) {
  SampleAcc<NR> r;
  r.mraw = fmaxf(a.mraw, b.mraw);
  r.sraw = (r.mraw == -INFINITY) ? 0.f : a.sraw * expf(a.mraw - r.mraw) + b.sraw * expf(b.mraw - r.mraw);
#pragma unroll
  for (int q = 0; q < NR; ++q) r.r[q] = region_merge<SAMPLING>(a.r[q], b.r[q]);
  return r;
}
template <bool SAMPLING>
constexpr int region_floats() { return SAMPLING ? 5 : 3; }
template <int NR, bool SAMPLING>
__device__ __forceinline__ void acc_store(const SampleAcc<NR>& s, float* out) {   // [mraw, sraw, per region m, s, arg (, g, gid)]
  out[0] = s.mraw; out[1] = s.sraw;
#pragma unroll
  for (int q = 0; q < NR; ++q) {
    float* o = out + 2 + q * region_floats<SAMPLING>();
    o[0] = s.r[q].m; o[1] = s.r[q].s; o[2] = __int_as_float(s.r[q].arg);
    if constexpr (SAMPLING) { o[3] = s.r[q].g; o[4] = __int_as_float(s.r[q].gid); }
  }
}
template <int NR, bool SAMPLING>
__device__ __forceinline__ SampleAcc<NR> acc_load(const volatile float* in, int V) {
  SampleAcc<NR> s;
  acc_init(s, V);
  s.mraw = in[0]; s.sraw = in[1];
#pragma unroll
  for (int q = 0; q < NR; ++q) {
    const volatile float* p = in + 2 + q * region_floats<SAMPLING>();
    s.r[q].m = p[0]; s.r[q].s = p[1]; s.r[q].arg = __float_as_int(p[2]);
    if constexpr (SAMPLING) { s.r[q].g = p[3]; s.r[q].gid = __float_as_int(p[4]); }
  }
  return s;
}
template <int NR, bool SAMPLING>
__device__ __forceinline__ SampleAcc<NR> acc_shfl(const SampleAcc<NR>& s, int o) {
  SampleAcc<NR> t;
  t.mraw = __shfl_xor_sync(0xffffffffu, s.mraw, o); t.sraw = __shfl_xor_sync(0xffffffffu, s.sraw, o);
#pragma unroll
  for (int q = 0; q < NR; ++q) {
    t.r[q].m = __shfl_xor_sync(0xffffffffu, s.r[q].m, o); t.r[q].s = __shfl_xor_sync(0xffffffffu, s.r[q].s, o);
    t.r[q].arg = __shfl_xor_sync(0xffffffffu, s.r[q].arg, o);
    if constexpr (SAMPLING) {
      t.r[q].g = __shfl_xor_sync(0xffffffffu, s.r[q].g, o); t.r[q].gid = __shfl_xor_sync(0xffffffffu, s.r[q].gid, o);
    } else {
      t.r[q].g = -INFINITY; t.r[q].gid = s.r[q].gid;
    }
  }
  return t;
}

// <false, false> is greedy decoding without timestamps (oasr_dec_sample, 8 floats of scratch per slice); the other
// instantiations serve oasr_dec_sample_rules (BEAM_SCR floats per slice).
template <bool TS, bool SAMPLING>
__global__ void __launch_bounds__(256) dec_sample_kernel(const oasr_dec_sample_rules_args a) {
  constexpr int NR = TS ? 2 : 1;
  constexpr int SCR = (TS || SAMPLING) ? BEAM_SCR : 8;
  static_assert(2 + NR * region_floats<SAMPLING>() <= SCR, "sampling scratch");
  __shared__ SampleAcc<NR> s_acc[8];
  __shared__ int s_last;
  __shared__ int s_red[8];
  pdl_launch_dependents();
  pdl_wait();
  const int slice = blockIdx.x, n = blockIdx.y, S = gridDim.x;
  const int pos = *a.pos_ptr;
  const float* row = a.logits + static_cast<int64_t>(n) * a.ld_logits;
  const int32_t* trow = a.tokens + static_cast<int64_t>(n) * a.ld_tokens;
  const int V = a.n_vocab;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const bool sampling = pos >= a.sample_begin - 1;
  const bool want_raw = (pos == a.sot_index);
  if (!sampling && !want_raw) return;
  const BeamFilter f = beam_filter(a.suppress, trow, pos, a.sample_begin, a.suppress_blank, a.blank, a.eot, TS ? 1 : 0,
                                   a.timestamp_begin, a.no_timestamps, a.max_initial_timestamp, V, s_red);
  float temp = 0.f;
  uint32_t k0 = 0, k1 = 0;
  if constexpr (SAMPLING) {
    temp = *a.temperature;
    const uint64_t key = a.row_keys[n];
    k0 = static_cast<uint32_t>(key); k1 = static_cast<uint32_t>(key >> 32);
  }
  const bool draw = SAMPLING && temp > 0.f;

  const int per = ((V + S - 1) / S + 3) & ~3;                  // slice length, a multiple of 4 (16-byte loads)
  const int v0 = slice * per, v1 = min(V, v0 + per);
  SampleAcc<NR> acc;
  acc_init(acc, V);
  const bool vec_ok = ((reinterpret_cast<uintptr_t>(row) & 15) == 0);
  auto visit = [&](float x, int v, uint32_t bits) {
    if (want_raw) acc_raw(acc, x);
    if (!sampling || f.banned(v)) return;
    auto add = [&](RegionAcc& r) {
      acc_filt(r, x, v);
      if constexpr (SAMPLING) { if (draw) acc_draw(r, x / temp + gumbel(bits), v); }
    };
    if constexpr (TS) { if (v >= f.ts_begin) { add(acc.r[NR - 1]); return; } }   // compile-time indices: registers
    add(acc.r[0]);
  };
  auto bits_of = [&](int v) -> uint4 {      // the random words of the 4-id group holding v (only drawn when sampling)
    return draw ? philox4x32_10(static_cast<uint32_t>(v >> 2), static_cast<uint32_t>(pos), k0, k1) : make_uint4(0, 0, 0, 0);
  };
  if (vec_ok) {
    for (int v = v0 + threadIdx.x * 4; v < v1; v += 256 * 4) {
      if (v + 4 <= v1) {
        const float4 x = *reinterpret_cast<const float4*>(row + v);
        const uint4 b = bits_of(v);
        visit(x.x, v, b.x); visit(x.y, v + 1, b.y); visit(x.z, v + 2, b.z); visit(x.w, v + 3, b.w);
      } else {
        for (int u = v; u < v1; ++u) visit(row[u], u, word_of(bits_of(u), u & 3));
      }
    }
  } else {
    for (int v = v0 + threadIdx.x; v < v1; v += 256) visit(row[v], v, word_of(bits_of(v), v & 3));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc = acc_merge<NR, SAMPLING>(acc, acc_shfl<NR, SAMPLING>(acc, o));
  if (lane == 0) s_acc[warp] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    SampleAcc<NR> t = s_acc[0];
    for (int w = 1; w < 8; ++w) t = acc_merge<NR, SAMPLING>(t, s_acc[w]);
    acc_store<NR, SAMPLING>(t, a.scratch + (static_cast<int64_t>(n) * S + slice) * SCR);
    __threadfence();
    s_last = (atomicAdd(a.counters + n, 1) == S - 1) ? 1 : 0;
  }
  __syncthreads();
  if (!s_last || threadIdx.x != 0) return;
  __threadfence();
  SampleAcc<NR> t;
  acc_init(t, V);
  for (int sl = 0; sl < S; ++sl)         // slice order: the result does not depend on which block arrived last
    t = acc_merge<NR, SAMPLING>(t, acc_load<NR, SAMPLING>(a.scratch + (static_cast<int64_t>(n) * S + sl) * SCR, V));
  a.counters[n] = 0;                     // re-armed for the next step
  if (want_raw) a.no_speech_prob[n] = expf(row[a.no_speech] - t.mraw) / t.sraw;
  if (sampling) {
    RegionAcc c = t.r[0];
    if constexpr (TS) {                  // timestamp mass beats every text token: only timestamps remain
      const RegionAcc& ts = t.r[1];
      const float lse_ts = ts.m == -INFINITY ? -INFINITY : ts.m + logf(ts.s);
      c = (lse_ts > t.r[0].m) ? ts : region_merge<SAMPLING>(t.r[0], ts);
    }
    int pick = c.arg;
    float logprob = -logf(c.s);          // logit[arg] - (m + log sum exp(x - m)), logit[arg] == m
    if (draw && c.gid < V) {
      pick = c.gid;
      logprob = (row[pick] - c.m) - logf(c.s);
    }
    const int prev = trow[pos];
    const bool finished = (prev == a.eot);
    if (!finished) a.sum_logprobs[n] += logprob;
    const int next = finished ? a.eot : pick;
    a.tokens[static_cast<int64_t>(n) * a.ld_tokens + pos + 1] = next;
    if (next != a.eot) atomicAdd(a.n_unfinished, 1);
  }
}

// pos += 1; done = (every sequence's last token is eot) -- the stop test of DecodingTask._main_loop, kept on the device
__global__ void dec_advance_kernel(int32_t* pos_ptr, int32_t* n_unfinished, int32_t* done_flag, int sample_begin) {
  pdl_launch_dependents();
  pdl_wait();
  const int pos = *pos_ptr;
  if (pos >= sample_begin - 1) *done_flag = (*n_unfinished == 0) ? 1 : 0;
  *n_unfinished = 0;
  *pos_ptr = pos + 1;
}

// ---------------------------------------------------------------------------------------------------------- beam search
// whisper/decoding.py BeamSearchDecoder.update on the device.  Three kernels per step after the logits head:
//   * dec_beam_cand: `n_slices` blocks per row, one pass over the fp32 logits applying every filter as an index test
//     (SuppressTokens, SuppressBlank, ApplyTimestampRules).  Each slice keeps the online (max, sum exp) and the top
//     beam + 1 entries separately for the text region [0, timestamp_begin) and the timestamp region, plus the raw
//     (max, sum exp) for the no-speech probability.  Banned ids enter the top-k lists as -inf (topk includes them).
//   * dec_beam_select: one CTA per clip.  Merges the slices in slice order, applies "timestamp mass beats every text
//     token" (lse(ts) > max(text): both sides share one normaliser), ranks the clip's candidates, fills the finished
//     list and rewrites the clip's token rows, log-prob sums and source rows.  Once every clip's list is full (done flag
//     set by the previous step) it leaves all state untouched, so extra replays before the host looks are harmless.
//   * dec_beam_reorder: self-attention K / V rows [0, pos) of every layer gathered from the source beams, in place.
// Ordering: candidates by (value desc, token id asc); across a clip by (score desc, beam, rank) -- Python's stable sort
// over dict insertion order.  No float atomics: the result is the same on every run.
constexpr int BEAM_MAX = 8;
constexpr int BEAM_K = BEAM_MAX + 1;        // candidates per row: beam + 1
constexpr int BEAM_TOK_MAX = 456;           // staged token row length (n_text_ctx + 2 <= this)

__device__ __forceinline__ bool cand_better(float x, int i, float y, int j) { return x > y || (x == y && i < j); }

struct TopK {
  float v[BEAM_K];
  int i[BEAM_K];
  __device__ __forceinline__ void init() {
#pragma unroll
    for (int k = 0; k < BEAM_K; ++k) { v[k] = -INFINITY; i[k] = INT_MAX; }
  }
  __device__ __forceinline__ void push(float x, int id) {     // sorted insert, registers only (compile-time indices)
    if (!cand_better(x, id, v[BEAM_K - 1], i[BEAM_K - 1])) return;
#pragma unroll
    for (int k = 0; k < BEAM_K; ++k) {
      if (cand_better(x, id, v[k], i[k])) {
        const float tv = v[k]; const int ti = i[k];
        v[k] = x; i[k] = id; x = tv; id = ti;
      }
    }
  }
  __device__ __forceinline__ void pop() {
#pragma unroll
    for (int k = 0; k + 1 < BEAM_K; ++k) { v[k] = v[k + 1]; i[k] = i[k + 1]; }
    v[BEAM_K - 1] = -INFINITY; i[BEAM_K - 1] = INT_MAX;
  }
};

struct Lse {   // online (max, sum exp(x - max)); -inf entries add nothing
  float m, s;
  __device__ __forceinline__ void push(float x) {
    if (x == -INFINITY) return;
    if (x > m) { s = s * expf(m - x) + 1.f; m = x; }
    else s += expf(x - m);
  }
  __device__ __forceinline__ void merge(float bm, float bs) {
    const float r = fmaxf(m, bm);
    s = (r == -INFINITY) ? 0.f : s * expf(m - r) + bs * expf(bm - r);
    m = r;
  }
  __device__ __forceinline__ float lse() const { return m == -INFINITY ? -INFINITY : m + logf(s); }
};

__global__ void __launch_bounds__(256) dec_beam_cand_kernel(const oasr_dec_beam_args a) {
  __shared__ int s_red[8];
  __shared__ float s_f[8][2];
  __shared__ int s_i[8];
  pdl_launch_dependents();
  pdl_wait();
  const int slice = blockIdx.x, n = blockIdx.y, S = gridDim.x;
  const int pos = *a.pos_ptr;
  const bool sampling = pos >= a.sample_begin - 1 && *a.done_flag == 0;
  const bool want_raw = pos == a.sot_index;
  if (!sampling && !want_raw) return;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const float* row = a.logits + static_cast<int64_t>(n) * a.ld_logits;
  const int32_t* trow = a.tokens + static_cast<int64_t>(n) * a.ld_tokens;
  const int V = a.n_vocab, K = a.beam + 1;
  const BeamFilter f = beam_filter(a.suppress, trow, pos, a.sample_begin, a.suppress_blank, a.blank, a.eot, a.timestamps,
                                   a.timestamp_begin, a.no_timestamps, a.max_initial_timestamp, a.n_vocab, s_red);
  const int per = ((V + S - 1) / S + 3) & ~3;
  const int v0 = slice * per, v1 = min(V, v0 + per);
  Lse raw{-INFINITY, 0.f}, lt{-INFINITY, 0.f}, ls{-INFINITY, 0.f};
  TopK tt, ts;
  tt.init(); ts.init();
  auto visit = [&](float x, int v) {
    if (want_raw) raw.push(x);
    if (!sampling) return;
    const bool ban = f.banned(v);
    const float y = ban ? -INFINITY : x;
    if (v < f.ts_begin) { if (!ban) lt.push(y); tt.push(y, v); }
    else { if (!ban) ls.push(y); ts.push(y, v); }
  };
  for (int v = v0 + threadIdx.x * 4; v < v1; v += 256 * 4) {
    if (v + 4 <= v1) {
      const float4 x = *reinterpret_cast<const float4*>(row + v);
      visit(x.x, v); visit(x.y, v + 1); visit(x.z, v + 2); visit(x.w, v + 3);
    } else {
      for (int u = v; u < v1; ++u) visit(row[u], u);
    }
  }
  float* out = a.scratch + (static_cast<int64_t>(n) * S + slice) * BEAM_SCR;
  // (max, sum exp) of the three accumulators: warps, then warp 0 in warp order
  Lse* accs[3] = {&lt, &ls, &raw};
  for (int q = 0; q < 3; ++q) {
    Lse& l = *accs[q];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float bm = __shfl_xor_sync(0xffffffffu, l.m, o), bs = __shfl_xor_sync(0xffffffffu, l.s, o);
      l.merge(bm, bs);
    }
    if (lane == 0) { s_f[warp][0] = l.m; s_f[warp][1] = l.s; }
    __syncthreads();
    if (threadIdx.x == 0) {
      Lse t{-INFINITY, 0.f};
      for (int w = 0; w < 8; ++w) t.merge(s_f[w][0], s_f[w][1]);
      out[2 * q] = t.m; out[2 * q + 1] = t.s;
    }
    __syncthreads();
  }
  if (!sampling) return;
  // top-K of the block per region: K rounds of a block-wide best over the threads' list heads
  TopK* lists[2] = {&tt, &ts};
  for (int q = 0; q < 2; ++q) {
    TopK& t = *lists[q];
    for (int r = 0; r < K; ++r) {
      float bv = t.v[0];
      int bi = t.i[0];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (cand_better(ov, oi, bv, bi)) { bv = ov; bi = oi; }
      }
      if (lane == 0) { s_f[warp][0] = bv; s_i[warp] = bi; }
      __syncthreads();
      bv = s_f[0][0]; bi = s_i[0];
      for (int w = 1; w < 8; ++w)
        if (cand_better(s_f[w][0], s_i[w], bv, bi)) { bv = s_f[w][0]; bi = s_i[w]; }
      if (t.i[0] == bi) t.pop();                 // ids are unique (sentinels carry INT_MAX and are never consumed)
      if (threadIdx.x == 0) { out[6 + q * 2 * BEAM_K + r] = bv; out[6 + q * 2 * BEAM_K + BEAM_K + r] = __int_as_float(bi); }
      __syncthreads();
    }
  }
}

__global__ void __launch_bounds__(256) dec_beam_select_kernel(const oasr_dec_beam_args a) {
  __shared__ float s_val[BEAM_MAX][2][BEAM_K];
  __shared__ int s_id[BEAM_MAX][2][BEAM_K];
  __shared__ float s_m[BEAM_MAX][2], s_l[BEAM_MAX][2];
  __shared__ float c_lp[BEAM_MAX * BEAM_K];
  __shared__ int c_tok[BEAM_MAX * BEAM_K];
  __shared__ float c_score[BEAM_MAX * BEAM_K];
  __shared__ int c_order[BEAM_MAX * BEAM_K];
  __shared__ int s_tok[BEAM_MAX][BEAM_TOK_MAX];
  __shared__ int k_src[BEAM_MAX], k_tok[BEAM_MAX];
  __shared__ int f_slot[BEAM_MAX], f_src[BEAM_MAX];
  __shared__ int s_nfin;
  pdl_launch_dependents();
  pdl_wait();
  const int c = blockIdx.x, B = a.beam, K = B + 1, S = a.n_slices;
  const int row0 = c * B;
  const int pos = *a.pos_ptr;
  const bool sampling = pos >= a.sample_begin - 1 && *a.done_flag == 0;
  const bool first = pos == a.sample_begin - 1;
  const bool want_raw = pos == a.sot_index;
  const int tid = threadIdx.x;
  // 1. merge the slices of every (row, region) in slice order; the raw statistics give the no-speech probability
  if (tid < 2 * B) {
    const int j = tid >> 1, q = tid & 1, n = row0 + j;
    const float* in = a.scratch + static_cast<int64_t>(n) * S * BEAM_SCR;
    if (q == 0 && want_raw) {
      Lse r{-INFINITY, 0.f};
      for (int s = 0; s < S; ++s) r.merge(in[s * BEAM_SCR + 4], in[s * BEAM_SCR + 5]);
      a.no_speech_prob[n] = expf(a.logits[static_cast<int64_t>(n) * a.ld_logits + a.no_speech] - r.m) / r.s;
    }
    if (sampling) {
      Lse l{-INFINITY, 0.f};
      TopK t;
      t.init();
      for (int s = 0; s < S; ++s) {
        const float* p = in + s * BEAM_SCR;
        l.merge(p[2 * q], p[2 * q + 1]);
        for (int r = 0; r < K; ++r) t.push(p[6 + q * 2 * BEAM_K + r], __float_as_int(p[6 + q * 2 * BEAM_K + BEAM_K + r]));
      }
      s_m[j][q] = l.m;
      s_l[j][q] = l.lse();
#pragma unroll
      for (int r = 0; r < BEAM_K; ++r) { s_val[j][q][r] = t.v[r]; s_id[j][q][r] = t.i[r]; }
    }
  }
  __syncthreads();
  if (!sampling) {                           // teacher-forced step or frozen state: identity sources, nothing else
    if (tid < B) a.src_rows[row0 + tid] = row0 + tid;
    return;
  }
  // 2. per row: "timestamp mass beats every text token" bans text (then every text id is -inf, lowest ids first);
  //    the row's normaliser and its top K candidates (log-probs)
  if (tid < B) {
    const int j = tid;
    const bool ban_text = a.timestamps && s_l[j][1] > s_m[j][0];
    const float lse = ban_text ? s_l[j][1]
                               : (fmaxf(s_l[j][0], s_l[j][1]) == -INFINITY ? -INFINITY
                                  : fmaxf(s_l[j][0], s_l[j][1]) + log1pf(expf(fminf(s_l[j][0], s_l[j][1]) - fmaxf(s_l[j][0], s_l[j][1]))));
    int it = 0, is = 0;
    for (int r = 0; r < K; ++r) {
      const float vt = ban_text ? -INFINITY : s_val[j][0][it];
      const int idt = ban_text ? it : s_id[j][0][it];
      const float vs = s_val[j][1][is];
      const int ids = s_id[j][1][is];
      float v; int id;
      if (cand_better(vt, idt, vs, ids)) { v = vt; id = idt; ++it; } else { v = vs; id = ids; ++is; }
      c_lp[j * K + r] = v - lse;
      c_tok[j * K + r] = id;
    }
  }
  __syncthreads();
  // 3. scores and their rank: (score desc, candidate index asc); at the first sampled step every beam holds the same
  //    prefix, so only beam 0's candidates exist (upstream's dict keyed by sequence collapses them)
  const int n_cand = first ? K : B * K;
  if (tid < n_cand) c_score[tid] = a.sum_logprobs[row0 + tid / K] + c_lp[tid];
  for (int idx = tid; idx < B * (pos + 1); idx += blockDim.x) {
    const int j = idx / (pos + 1), p = idx - j * (pos + 1);
    s_tok[j][p] = a.tokens[static_cast<int64_t>(row0 + j) * a.ld_tokens + p];
  }
  __syncthreads();
  if (tid < n_cand) {
    const float me = c_score[tid];
    int rank = 0;
    for (int u = 0; u < n_cand; ++u) rank += (c_score[u] > me || (c_score[u] == me && u < tid)) ? 1 : 0;
    c_order[rank] = tid;
  }
  __syncthreads();
  // 4. the walk: eot -> finished (while the list has room), anything else -> the next beam, until `beam` are kept
  if (tid == 0) {
    int kept = 0, nf = 0, count = a.fin_count[c];
    float sums[BEAM_MAX];
    for (int i = 0; i < n_cand && kept < B; ++i) {
      const int t = c_order[i];
      const int tok = c_tok[t];
      if (tok == a.eot) {
        if (count < a.max_candidates) {
          const int slot = count++;
          a.fin_scores[c * a.max_candidates + slot] = c_score[t];
          a.fin_len[c * a.max_candidates + slot] = pos + 2;
          f_slot[nf] = slot; f_src[nf] = t / K; ++nf;
        }
      } else {
        k_src[kept] = t / K; k_tok[kept] = tok; sums[kept] = c_score[t]; ++kept;
      }
    }
    for (int k = 0; k < B; ++k) a.sum_logprobs[row0 + k] = sums[k];
    a.fin_count[c] = count;
    s_nfin = nf;
    if (count < a.max_candidates) atomicAdd(a.n_unfinished, 1);
    if (c == 0) *a.seq_len = pos + 2;
  }
  __syncthreads();
  // 5. new token rows (prefix of the source beam + the new token), source rows, finished sequences
  const int L = pos + 2;
  for (int idx = tid; idx < B * L; idx += blockDim.x) {
    const int k = idx / L, p = idx - k * L;
    a.tokens[static_cast<int64_t>(row0 + k) * a.ld_tokens + p] = (p <= pos) ? s_tok[k_src[k]][p] : k_tok[k];
  }
  for (int idx = tid; idx < s_nfin * L; idx += blockDim.x) {
    const int f = idx / L, p = idx - f * L;
    a.fin_tokens[(static_cast<int64_t>(c) * a.max_candidates + f_slot[f]) * a.ld_fin + p] = (p <= pos) ? s_tok[f_src[f]][p] : a.eot;
  }
  if (tid < B) a.src_rows[row0 + tid] = row0 + k_src[tid];
}

// K / V rows [0, *pos) of every layer: row r <- row src[r] (rows of one clip, in place).  One CTA iteration owns one
// (layer, K or V, clip, position) tile of all the clip's beams: every source element is in registers before the
// barrier and written after it, so cycles and forks are safe.  Rows whose source is themselves are not touched.
constexpr int REORDER_ITEMS = 5;     // 16-byte items per thread: beam 8 x d 1280 / 8 / 256 threads
__global__ void __launch_bounds__(256) dec_beam_reorder_kernel(uint16_t* k_cache, uint16_t* v_cache, int64_t layer_stride,
                                                               int64_t row_stride, const int32_t* src, const int32_t* pos_ptr,
                                                               int beam, int d) {
  __shared__ int s_src[BEAM_MAX];
  __shared__ int s_any;
  pdl_launch_dependents();
  pdl_wait();
  const int c = blockIdx.z, layer = blockIdx.y >> 1;
  uint16_t* base = ((blockIdx.y & 1) ? v_cache : k_cache) + static_cast<int64_t>(layer) * layer_stride;
  if (threadIdx.x == 0) s_any = 0;
  __syncthreads();
  if (threadIdx.x < beam) {
    s_src[threadIdx.x] = src[c * beam + threadIdx.x];
    if (s_src[threadIdx.x] != c * beam + static_cast<int>(threadIdx.x)) s_any = 1;
  }
  __syncthreads();
  if (!s_any) return;
  const int npos = *pos_ptr;
  const int vec = d >> 3, items = beam * vec;
  for (int p = blockIdx.x; p < npos; p += gridDim.x) {
    uint4 buf[REORDER_ITEMS];
#pragma unroll
    for (int q = 0; q < REORDER_ITEMS; ++q) {
      const int idx = threadIdx.x + 256 * q;
      if (idx < items) {
        const int j = idx / vec, v = idx - j * vec;
        const int s = s_src[j];
        if (s != c * beam + j) buf[q] = *reinterpret_cast<const uint4*>(base + s * row_stride + static_cast<int64_t>(p) * d + v * 8);
      }
    }
    __syncthreads();
#pragma unroll
    for (int q = 0; q < REORDER_ITEMS; ++q) {
      const int idx = threadIdx.x + 256 * q;
      if (idx < items) {
        const int j = idx / vec, v = idx - j * vec;
        const int r = c * beam + j;
        if (s_src[j] != r) *reinterpret_cast<uint4*>(base + r * row_stride + static_cast<int64_t>(p) * d + v * 8) = buf[q];
      }
    }
  }
}

template <typename TI, typename TO>
__global__ void convert_kernel(const TI* __restrict__ src, TO* __restrict__ dst, int64_t n) {
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<int64_t>(gridDim.x) * blockDim.x)
    dst[i] = static_cast<TO>(static_cast<float>(src[i]));
}

// Launch with the programmatic-dependent-launch attribute (see pdl_wait above) when OASR_DEC_PDL=1; plainly otherwise.
inline bool pdl_enabled() {
  // off by default: inside a CUDA graph the gaps between these kernels are already small, and holding several waiting
  // grids resident competes with the running one
  static const int v = [] { const char* e = getenv("OASR_DEC_PDL"); return e ? atoi(e) : 0; }();
  return v != 0;
}
template <typename... KArgs, typename... Args>
cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, cudaStream_t st, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = 0;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, args...);
}

template <typename T, typename TW, int MT>
int launch_linear(const typename Stored<T, TW>::LinearArgs& a, cudaStream_t st) {
  constexpr int MP = 16 * MT;
  // whole-K staging when it fits (always for the LayerNorm prologue, K = d <= 1280); otherwise chunks of 256 * DEC_PF
  int KC = a.K;
  const size_t red_bytes = sizeof(float) * 8 * MP * 17;
  const size_t budget = 220 * 1024;       // of the 227 KB a CTA may use
  if (static_cast<size_t>(MP) * (a.K + DEC_XPAD) * sizeof(T) + red_bytes > budget) {
    OASR_REQUIRE(a.x_mode != X_LAYERNORM, "dec_linear: LayerNorm prologue needs the whole row staged (K = %d too wide for %d rows)", a.K, MP);
    KC = 256 * DEC_PF;
  }
  const size_t smem = static_cast<size_t>(MP) * (KC + DEC_XPAD) * sizeof(T) + red_bytes;
  // column groups per CTA: enough CTAs to cover the machine about twice, but no more (each CTA stages x once)
  const int n_groups = (int)ceil_div(a.N, 16);
  int groups = (int)ceil_div(n_groups, 2 * num_sms());
  if (groups < 1) groups = 1;
  const int grid = (int)ceil_div(n_groups, groups);
  static size_t attr_smem = 0;
  if (smem > attr_smem) {
    OASR_CUDA_OK(cudaFuncSetAttribute(dec_linear_kernel<T, TW, MT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)budget));
    attr_smem = budget;
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)grid);
  cfg.blockDim = dim3(256);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  OASR_CUDA_OK(cudaLaunchKernelEx(&cfg, dec_linear_kernel<T, TW, MT>, a, KC, groups));
  return OASR_OK;
}
template <typename T, typename TW, int MT>
int launch_linear_direct(const typename Stored<T, TW>::LinearArgs& a, cudaStream_t st) {
  OASR_CUDA_OK(launch_pdl(dec_linear_direct_kernel<T, TW, MT>, dim3((unsigned)ceil_div(a.N, 16)), dim3(256), st, a));
  return OASR_OK;
}
// TW: the weight storage, T or uint8_t e4m3 codes (whose argument block carries the per-row scales)
template <typename T, typename TW>
int dispatch_linear(const typename Stored<T, TW>::LinearArgs& a, cudaStream_t st) {
  // the direct form up to 32 rows (no staging round trip for a handful of rows), the staged form from there on
  if (a.M <= 16) return launch_linear_direct<T, TW, 1>(a, st);
  if (a.M <= 32) return launch_linear_direct<T, TW, 2>(a, st);
  return launch_linear<T, TW, 4>(a, st);
}

int check_linear_args(const oasr_dec_linear_args* a) {
  OASR_REQUIRE(a != nullptr, "dec_linear: null arguments");
  OASR_REQUIRE(a->M >= 1 && a->M <= 64, "dec_linear: 1 <= M <= 64 sequences (got %d)", a->M);
  OASR_REQUIRE(a->N >= 1 && a->K >= 32 && (a->K % 32) == 0, "dec_linear: K must be a multiple of 32 (got %d)", a->K);
  OASR_REQUIRE(a->x && a->W && a->out, "dec_linear: null tensor");
  OASR_REQUIRE(((uintptr_t)a->x & 15) == 0 && ((uintptr_t)a->W & 15) == 0, "dec_linear: x and W must be 16-byte aligned");
  OASR_REQUIRE(a->x_mode >= 0 && a->x_mode <= 2 && a->epi >= 0 && a->epi <= 4, "dec_linear: bad mode");
  OASR_REQUIRE(a->x_mode != X_LAYERNORM || (a->ln_gamma && a->ln_beta), "dec_linear: LayerNorm mode needs gamma / beta");
  OASR_REQUIRE(a->x_mode != X_LAYERNORM || (a->K <= 1280 && a->K % 8 == 0), "dec_linear: LayerNorm prologue supports K <= 1280 (got %d)", a->K);
  OASR_REQUIRE(a->x_mode != X_PARTIAL_SUM || a->n_partials >= 1, "dec_linear: partial-sum mode needs n_partials >= 1");
  OASR_REQUIRE(a->x_mode == X_PARTIAL_SUM || (a->ldx % 8) == 0, "dec_linear: ldx must be a multiple of 8");
  OASR_REQUIRE(a->epi != EPI_RESIDUAL || a->res, "dec_linear: residual epilogue needs res");
  OASR_REQUIRE(a->epi != EPI_QKV_SCATTER || (a->k_cache && a->v_cache && a->pos_ptr && a->N % 3 == 0), "dec_linear: qkv scatter needs caches and pos");
  OASR_REQUIRE(a->dtype == OASR_DTYPE_F16 || a->dtype == OASR_DTYPE_BF16, "dec_linear: unknown dtype %d", a->dtype);
  return OASR_OK;
}

}  // namespace
}  // namespace oasr

using namespace oasr;

extern "C" int oasr_dec_embed(const int32_t* tokens, int64_t ld_tokens, const int32_t* pos_ptr, const float* emb, const float* pos_emb,
                              void* x, int64_t n_seq, int64_t d, int64_t n_vocab, int dtype, void* stream) {
  OASR_REQUIRE(n_seq > 0 && d > 0 && tokens && pos_ptr && emb && pos_emb && x, "dec_embed: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == OASR_DTYPE_F16)
    OASR_CUDA_OK(launch_pdl(dec_embed_kernel<__half>, dim3((unsigned)n_seq), dim3(128), st, tokens, ld_tokens, pos_ptr, emb, pos_emb,
                            (__half*)x, (int)d, (int)n_vocab));
  else
    OASR_CUDA_OK(launch_pdl(dec_embed_kernel<bf16>, dim3((unsigned)n_seq), dim3(128), st, tokens, ld_tokens, pos_ptr, emb, pos_emb,
                            (bf16*)x, (int)d, (int)n_vocab));
  return OASR_OK;
}

extern "C" int oasr_dec_linear(const oasr_dec_linear_args* a, void* stream) {
  if (int rc = check_linear_args(a)) return rc;
  if (a->dtype == OASR_DTYPE_F16) return dispatch_linear<__half, __half>(*a, (cudaStream_t)stream);
  return dispatch_linear<bf16, bf16>(*a, (cudaStream_t)stream);
}

extern "C" int oasr_dec_linear_fp8w(const oasr_dec_linear_args* a, const float* w_scale, void* stream) {
  if (int rc = check_linear_args(a)) return rc;
  OASR_REQUIRE(w_scale != nullptr, "dec_linear_fp8w: null weight scales");
  LinearArgsFp8 a8;
  static_cast<oasr_dec_linear_args&>(a8) = *a;
  a8.w_scale = w_scale;
  if (a->dtype == OASR_DTYPE_F16) return dispatch_linear<__half, uint8_t>(a8, (cudaStream_t)stream);
  return dispatch_linear<bf16, uint8_t>(a8, (cudaStream_t)stream);
}

namespace {
// TKV: the K / V storage, T (ks unused) or uint8_t e4m3 codes with per-(key, head) scales
template <typename T, typename TKV>
int launch_attention(const oasr_dec_attn_args* a, int kv_group, const KvScales& ks, cudaStream_t st) {
  dim3 grid((unsigned)a->n_splits, (unsigned)a->n_head, (unsigned)a->n_seq);
  if (a->n_splits == 1 && (a->pos_ptr != nullptr || a->n_keys <= 1536)) {   // whole key range in one CTA: fused form
    OASR_CUDA_OK(launch_pdl(dec_attn_fused_kernel<T, TKV>, grid, dim3(128), st, *a, kv_group, ks));
    return OASR_OK;
  }
  OASR_CUDA_OK(launch_pdl(dec_attn_scores_kernel<T, TKV>, grid, dim3(128), st, *a, kv_group, ks));
  OASR_CUDA_OK(launch_pdl(dec_attn_pv_kernel<T, TKV>, grid, dim3(128), st, *a, kv_group, ks));
  return OASR_OK;
}

int check_attention_args(const oasr_dec_attn_args* a, int kv_group) {
  OASR_REQUIRE(a != nullptr && a->q && a->k && a->v && a->scores && a->out_partial, "dec_attention: null tensor");
  OASR_REQUIRE(a->n_seq >= 1 && a->n_head >= 1 && a->n_splits >= 1, "dec_attention: bad sizes");
  OASR_REQUIRE(kv_group >= 1, "dec_attention: kv_group must be >= 1 (got %d)", kv_group);
  OASR_REQUIRE(a->pos_ptr != nullptr || a->n_keys >= 1, "dec_attention: key count missing");
  OASR_REQUIRE((a->ldq % 8) == 0 && (a->kv_row_stride % 8) == 0 && (a->kv_seq_stride % 8) == 0, "dec_attention: strides must be multiples of 8");
  OASR_REQUIRE(a->dtype == OASR_DTYPE_F16 || a->dtype == OASR_DTYPE_BF16, "dec_attention: unknown dtype %d", a->dtype);
  return OASR_OK;
}

int dec_attention(const oasr_dec_attn_args* a, int kv_group, cudaStream_t st) {
  if (int rc = check_attention_args(a, kv_group)) return rc;
  const KvScales none = {nullptr, nullptr, 0, 0};
  if (a->dtype == OASR_DTYPE_F16) return launch_attention<__half, __half>(a, kv_group, none, st);
  return launch_attention<bf16, bf16>(a, kv_group, none, st);
}
}  // namespace

extern "C" int oasr_dec_attention(const oasr_dec_attn_args* a, void* stream) { return dec_attention(a, 1, (cudaStream_t)stream); }

extern "C" int oasr_dec_attention_grouped(const oasr_dec_attn_args* a, int kv_group, void* stream) {
  return dec_attention(a, kv_group, (cudaStream_t)stream);
}

extern "C" int oasr_dec_attention_fp8kv(const oasr_dec_attn_args* a, const float* k_scale, const float* v_scale,
                                        int64_t scale_seq_stride, int64_t scale_row_stride, int kv_group, void* stream) {
  if (int rc = check_attention_args(a, kv_group)) return rc;
  OASR_REQUIRE(k_scale && v_scale && scale_seq_stride >= 0 && scale_row_stride >= a->n_head,
               "dec_attention_fp8kv: scales missing or row stride < n_head");
  const KvScales ks = {k_scale, v_scale, scale_seq_stride, scale_row_stride};
  if (a->dtype == OASR_DTYPE_F16) return launch_attention<__half, uint8_t>(a, kv_group, ks, (cudaStream_t)stream);
  return launch_attention<bf16, uint8_t>(a, kv_group, ks, (cudaStream_t)stream);
}

extern "C" int oasr_dec_sample(const oasr_dec_sample_args* a, void* stream) {
  OASR_REQUIRE(a != nullptr && a->logits && a->tokens && a->pos_ptr && a->suppress && a->sum_logprobs && a->no_speech_prob &&
                   a->n_unfinished && a->done_flag, "dec_sample: null tensor");
  OASR_REQUIRE(a->n_seq >= 1 && a->n_vocab >= 1, "dec_sample: bad sizes");
  OASR_REQUIRE(a->scratch && a->counters && a->n_slices >= 1 && a->n_slices <= 64, "dec_sample: scratch / counters / 1 <= n_slices <= 64");
  oasr_dec_sample_rules_args r = {};       // the rule-free, temperature-0 case of the rule-aware sampler
  r.logits = a->logits; r.ld_logits = a->ld_logits; r.tokens = a->tokens; r.ld_tokens = a->ld_tokens; r.pos_ptr = a->pos_ptr;
  r.suppress = a->suppress; r.sum_logprobs = a->sum_logprobs; r.no_speech_prob = a->no_speech_prob;
  r.n_unfinished = a->n_unfinished; r.done_flag = a->done_flag; r.scratch = a->scratch; r.counters = a->counters;
  r.n_seq = a->n_seq; r.n_vocab = a->n_vocab; r.sample_begin = a->sample_begin; r.sot_index = a->sot_index;
  r.suppress_blank = a->suppress_blank; r.blank = a->blank; r.eot = a->eot; r.no_speech = a->no_speech; r.n_slices = a->n_slices;
  OASR_CUDA_OK(launch_pdl(dec_sample_kernel<false, false>, dim3((unsigned)a->n_slices, (unsigned)a->n_seq), dim3(256),
                          (cudaStream_t)stream, r));
  OASR_CUDA_OK(launch_pdl(dec_advance_kernel, dim3(1), dim3(1), (cudaStream_t)stream, a->pos_ptr, a->n_unfinished, a->done_flag,
                          (int)a->sample_begin));
  return OASR_OK;
}

extern "C" int oasr_dec_sample_rules(const oasr_dec_sample_rules_args* a, void* stream) {
  OASR_REQUIRE(a != nullptr && a->logits && a->tokens && a->pos_ptr && a->suppress && a->sum_logprobs && a->no_speech_prob &&
                   a->n_unfinished && a->done_flag && a->scratch && a->counters, "dec_sample_rules: null tensor");
  OASR_REQUIRE(a->n_seq >= 1 && a->n_seq <= 64 && a->n_vocab >= 1, "dec_sample_rules: 1 <= n_seq <= 64 (got %d)", a->n_seq);
  OASR_REQUIRE(a->n_slices >= 1 && a->n_slices <= 64, "dec_sample_rules: 1 <= n_slices <= 64 (got %d)", a->n_slices);
  OASR_REQUIRE(((uintptr_t)a->logits & 15) == 0 && (a->ld_logits % 4) == 0, "dec_sample_rules: logits rows must be 16-byte aligned");
  OASR_REQUIRE(a->ld_tokens >= 1 && a->sample_begin >= 1, "dec_sample_rules: bad token layout");
  OASR_REQUIRE(!a->timestamps || (a->timestamp_begin > a->eot && a->timestamp_begin < a->n_vocab),
               "dec_sample_rules: bad timestamp_begin");
  OASR_REQUIRE(a->temperature == nullptr || a->row_keys != nullptr, "dec_sample_rules: sampling needs row_keys");
  const dim3 grid((unsigned)a->n_slices, (unsigned)a->n_seq);
  cudaStream_t st = (cudaStream_t)stream;
  const bool ts = a->timestamps != 0, draw = a->temperature != nullptr;
  if (ts && draw) OASR_CUDA_OK(launch_pdl(dec_sample_kernel<true, true>, grid, dim3(256), st, *a));
  else if (ts) OASR_CUDA_OK(launch_pdl(dec_sample_kernel<true, false>, grid, dim3(256), st, *a));
  else if (draw) OASR_CUDA_OK(launch_pdl(dec_sample_kernel<false, true>, grid, dim3(256), st, *a));
  else OASR_CUDA_OK(launch_pdl(dec_sample_kernel<false, false>, grid, dim3(256), st, *a));
  OASR_CUDA_OK(launch_pdl(dec_advance_kernel, dim3(1), dim3(1), st, a->pos_ptr, a->n_unfinished, a->done_flag, (int)a->sample_begin));
  return OASR_OK;
}

static int check_beam_args(const oasr_dec_beam_args* a, const char* what) {
  OASR_REQUIRE(a != nullptr && a->logits && a->tokens && a->pos_ptr && a->suppress && a->sum_logprobs && a->no_speech_prob &&
                   a->n_unfinished && a->done_flag && a->scratch && a->src_rows && a->fin_tokens && a->fin_scores && a->fin_len &&
                   a->fin_count && a->seq_len, "%s: null tensor", what);
  OASR_REQUIRE(a->beam >= 1 && a->beam <= BEAM_MAX, "%s: 1 <= beam <= %d (got %d)", what, BEAM_MAX, a->beam);
  OASR_REQUIRE(a->max_candidates >= 1 && a->max_candidates <= 32, "%s: 1 <= max_candidates <= 32 (got %d)", what, a->max_candidates);
  OASR_REQUIRE(a->n_clips >= 1 && a->n_clips * a->beam <= 64, "%s: 1 <= n_clips x beam <= 64", what);
  OASR_REQUIRE(a->n_slices >= 1 && a->n_slices <= 64 && a->n_vocab >= 1, "%s: 1 <= n_slices <= 64", what);
  OASR_REQUIRE(a->n_ctx >= 1 && a->n_ctx + 2 <= BEAM_TOK_MAX && a->ld_tokens >= a->n_ctx + 2 && a->ld_fin >= a->n_ctx + 1,
               "%s: n_ctx + 2 <= %d, ld_tokens >= n_ctx + 2, ld_fin >= n_ctx + 1", what, BEAM_TOK_MAX);
  OASR_REQUIRE(((uintptr_t)a->logits & 15) == 0 && (a->ld_logits % 4) == 0, "%s: logits rows must be 16-byte aligned", what);
  OASR_REQUIRE(!a->timestamps || (a->timestamp_begin > a->eot && a->timestamp_begin < a->n_vocab), "%s: bad timestamp_begin", what);
  return OASR_OK;
}

extern "C" int oasr_dec_beam_candidates(const oasr_dec_beam_args* a, void* stream) {
  if (int rc = check_beam_args(a, "dec_beam_candidates")) return rc;
  OASR_CUDA_OK(launch_pdl(dec_beam_cand_kernel, dim3((unsigned)a->n_slices, (unsigned)(a->n_clips * a->beam)), dim3(256),
                          (cudaStream_t)stream, *a));
  return OASR_OK;
}

extern "C" int oasr_dec_beam_select(const oasr_dec_beam_args* a, void* stream) {
  if (int rc = check_beam_args(a, "dec_beam_select")) return rc;
  OASR_CUDA_OK(launch_pdl(dec_beam_select_kernel, dim3((unsigned)a->n_clips), dim3(256), (cudaStream_t)stream, *a));
  OASR_CUDA_OK(launch_pdl(dec_advance_kernel, dim3(1), dim3(1), (cudaStream_t)stream, a->pos_ptr, a->n_unfinished, a->done_flag,
                          (int)a->sample_begin));
  return OASR_OK;
}

extern "C" int oasr_dec_beam_reorder(void* k_cache, void* v_cache, int64_t layer_stride, int64_t row_stride, int64_t n_layers,
                                     const int32_t* src_rows, const int32_t* pos_ptr, int32_t n_clips, int32_t beam, int32_t d,
                                     int32_t n_pos_blocks, int dtype, void* stream) {
  OASR_REQUIRE(k_cache && v_cache && src_rows && pos_ptr, "dec_beam_reorder: null tensor");
  OASR_REQUIRE(dtype == OASR_DTYPE_F16 || dtype == OASR_DTYPE_BF16, "dec_beam_reorder: fp16 / bf16 caches only");
  OASR_REQUIRE(beam >= 1 && beam <= BEAM_MAX && n_clips >= 1 && n_layers >= 1 && n_pos_blocks >= 1, "dec_beam_reorder: bad sizes");
  OASR_REQUIRE(d % 8 == 0 && beam * (d / 8) <= 256 * REORDER_ITEMS, "dec_beam_reorder: d must be a multiple of 8 and beam x d <= %d",
               256 * 8 * REORDER_ITEMS);
  OASR_REQUIRE((row_stride % 8) == 0 && (layer_stride % 8) == 0 && ((uintptr_t)k_cache & 15) == 0 && ((uintptr_t)v_cache & 15) == 0,
               "dec_beam_reorder: caches must be 16-byte aligned");
  OASR_CUDA_OK(launch_pdl(dec_beam_reorder_kernel, dim3((unsigned)n_pos_blocks, (unsigned)(2 * n_layers), (unsigned)n_clips), dim3(256),
                          (cudaStream_t)stream, (uint16_t*)k_cache, (uint16_t*)v_cache, layer_stride, row_stride, src_rows, pos_ptr,
                          (int)beam, (int)d));
  return OASR_OK;
}

extern "C" int oasr_convert(const void* src, int src_dtype, void* dst, int dst_dtype, int64_t n, void* stream) {
  OASR_REQUIRE(src && dst && n > 0, "convert: bad arguments");
  const int blocks = (int)std::min<int64_t>(ceil_div(n, 256), (int64_t)num_sms() * 16);
  cudaStream_t st = (cudaStream_t)stream;
  if (src_dtype == OASR_DTYPE_F32 && dst_dtype == OASR_DTYPE_F16) convert_kernel<float, __half><<<blocks, 256, 0, st>>>((const float*)src, (__half*)dst, n);
  else if (src_dtype == OASR_DTYPE_F32 && dst_dtype == OASR_DTYPE_BF16) convert_kernel<float, bf16><<<blocks, 256, 0, st>>>((const float*)src, (bf16*)dst, n);
  else if (src_dtype == OASR_DTYPE_BF16 && dst_dtype == OASR_DTYPE_F16) convert_kernel<bf16, __half><<<blocks, 256, 0, st>>>((const bf16*)src, (__half*)dst, n);
  else if (src_dtype == OASR_DTYPE_F16 && dst_dtype == OASR_DTYPE_BF16) convert_kernel<__half, bf16><<<blocks, 256, 0, st>>>((const __half*)src, (bf16*)dst, n);
  else if (src_dtype == OASR_DTYPE_BF16 && dst_dtype == OASR_DTYPE_F32) convert_kernel<bf16, float><<<blocks, 256, 0, st>>>((const bf16*)src, (float*)dst, n);
  else if (src_dtype == OASR_DTYPE_F16 && dst_dtype == OASR_DTYPE_F32) convert_kernel<__half, float><<<blocks, 256, 0, st>>>((const __half*)src, (float*)dst, n);
  else OASR_REQUIRE(false, "convert: unsupported dtype pair %d -> %d", src_dtype, dst_dtype);
  OASR_LAUNCH_CHECK();
  return OASR_OK;
}
