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
//   * dec_sample: logit filters + argmax + log-prob + eot bookkeeping in one pass over the fp32 logits.
//
// Rounding points are the reference's in the activation dtype T (inf_model.py:172-196): q*hd^-0.25 and k*hd^-0.25 rounded
// to T, q.k accumulated in fp32 and rounded to T, softmax in fp32, probabilities rounded to T, p.v accumulated in fp32 and
// rounded once; every Linear output is round_T(acc + bias_T); LayerNorm is computed in fp32 and rounded once;
// residuals are round_T(x + y); logits are float(round_T(x . E^T)).
#include "common.cuh"

#include <cuda_fp16.h>
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
template <typename T, int MT>
__global__ void __launch_bounds__(256) dec_linear_direct_kernel(const oasr_dec_linear_args a) {
  __shared__ float s_stat[16 * MT][2];
  __shared__ float s_red[8][16 * MT][17];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int n0 = blockIdx.x * 16;
  const int K = a.K;
  pdl_launch_dependents();
  // the weight stream does not depend on the previous kernel: its first round is in flight before pdl_wait()
  const T* W = static_cast<const T*>(a.W);
  const int r0 = n0 + g, r1 = n0 + 8 + g;
  const T* w0 = W + static_cast<int64_t>(r0 < a.N ? r0 : 0) * K + 8 * t;
  const T* w1 = W + static_cast<int64_t>(r1 < a.N ? r1 : 0) * K + 8 * t;
  const bool ok0 = r0 < a.N, ok1 = r1 < a.N;
  const uint4 zero = make_uint4(0, 0, 0, 0);
  int k0 = warp * 32;
  uint4 b0 = zero, b1 = zero;
  if (k0 < K) {
    b0 = ok0 ? __ldg(reinterpret_cast<const uint4*>(w0 + k0)) : zero;
    b1 = ok1 ? __ldg(reinterpret_cast<const uint4*>(w1 + k0)) : zero;
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
    uint4 nb0 = zero, nb1 = zero;
    uint4 nxa[MT], nxb[MT];
    if (kn < K) {   // the HBM stream and the x fragments run one round ahead of the MMAs
      nb0 = ok0 ? __ldg(reinterpret_cast<const uint4*>(w0 + kn)) : zero;
      nb1 = ok1 ? __ldg(reinterpret_cast<const uint4*>(w1 + kn)) : zero;
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
      DT<T>::mma(acc[i][0], xa[i].x, xb[i].x, xa[i].y, xb[i].y, b0.x, b0.y);
      DT<T>::mma(acc[i][0], xa[i].z, xb[i].z, xa[i].w, xb[i].w, b0.z, b0.w);
      DT<T>::mma(acc[i][1], xa[i].x, xb[i].x, xa[i].y, xb[i].y, b1.x, b1.y);
      DT<T>::mma(acc[i][1], xa[i].z, xb[i].z, xa[i].w, xb[i].w, b1.z, b1.w);
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

template <typename T, int MT>
__global__ void __launch_bounds__(256, (MT <= 2 ? 2 : 1)) dec_linear_kernel(const oasr_dec_linear_args a, const int KC, const int groups) {
  constexpr int MP = 16 * MT;
  extern __shared__ __align__(16) uint8_t dec_smem[];
  const int K = a.K;
  const int lds = KC + DEC_XPAD;                                   // staged row length in elements
  T* x_s = reinterpret_cast<T*>(dec_smem);
  float (*s_red)[MP][17] = reinterpret_cast<float (*)[MP][17]>(dec_smem + static_cast<size_t>(MP) * lds * sizeof(T));
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const T* W = static_cast<const T*>(a.W);
  const uint4 zero = make_uint4(0, 0, 0, 0);
  const int group0 = blockIdx.x * groups;
  const int n_groups_total = (a.N + 15) / 16;
  pdl_launch_dependents();

  // W rows of a column group for this thread, and the prefetch ring (DEC_PF rounds x 2 n8 tiles)
  uint4 wb0[DEC_PF], wb1[DEC_PF];
  auto w_ptrs = [&](int grp, const T*& w0, const T*& w1, bool& ok0, bool& ok1) {
    const int r0 = grp * 16 + g, r1 = r0 + 8;
    ok0 = r0 < a.N; ok1 = r1 < a.N;
    w0 = W + static_cast<int64_t>(ok0 ? r0 : 0) * K + 8 * t;
    w1 = W + static_cast<int64_t>(ok1 ? r1 : 0) * K + 8 * t;
  };
  const T *w0, *w1;
  bool ok0, ok1;
  w_ptrs(group0, w0, w1, ok0, ok1);
#pragma unroll
  for (int p = 0; p < DEC_PF; ++p) {
    const int k = warp * 32 + 256 * p;
    wb0[p] = (ok0 && k < K) ? __ldg(reinterpret_cast<const uint4*>(w0 + k)) : zero;
    wb1[p] = (ok1 && k < K) ? __ldg(reinterpret_cast<const uint4*>(w1 + k)) : zero;
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
    const T *nw0 = w0, *nw1 = w1;
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
          const uint4 b0 = wb0[p], b1 = wb1[p];
          // refill this ring slot with the same group's round p + DEC_PF (if there is one)
          const int kn = k0 + 256 * DEC_PF;
          if (kn < K) {
            wb0[p] = ok0 ? __ldg(reinterpret_cast<const uint4*>(w0 + kn)) : zero;
            wb1[p] = ok1 ? __ldg(reinterpret_cast<const uint4*>(w1 + kn)) : zero;
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
        wb0[p] = (ok0 && k < K) ? __ldg(reinterpret_cast<const uint4*>(w0 + k)) : zero;
        wb1[p] = (ok1 && k < K) ? __ldg(reinterpret_cast<const uint4*>(w1 + k)) : zero;
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
template <typename T>
__global__ void __launch_bounds__(128) dec_attn_scores_kernel(const oasr_dec_attn_args a) {
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
  const T* kb = static_cast<const T*>(a.k) + static_cast<int64_t>(n) * a.kv_seq_stride + h * 64 + c8 * 8;
  float* out = a.scores + (static_cast<int64_t>(n) * gridDim.y + h) * a.scores_ld;
  for (int jb = j0; jb < j1; jb += 128) {   // 8 independent 16-byte loads in flight per thread
    uint4 u[8];
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      const int j = jb + r * 16 + slot;
      u[r] = (j < j1) ? __ldg(reinterpret_cast<const uint4*>(kb + static_cast<int64_t>(j) * a.kv_row_stride)) : make_uint4(0, 0, 0, 0);
    }
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      const uint32_t w[4] = {u[r].x, u[r].y, u[r].z, u[r].w};
      float acc = 0.f;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float2 p = DT<T>::unpack2(w[i]);
        acc = fmaf(qs[2 * i], rnd<T>(p.x * scale), acc);
        acc = fmaf(qs[2 * i + 1], rnd<T>(p.y * scale), acc);
      }
      acc += __shfl_xor_sync(0xffffffffu, acc, 1);
      acc += __shfl_xor_sync(0xffffffffu, acc, 2);
      acc += __shfl_xor_sync(0xffffffffu, acc, 4);
      const int j = jb + r * 16 + slot;
      if (c8 == 0 && j < j1) out[j] = rnd<T>(acc);
    }
  }
}

// partial[s, n, h*64 + c] = sum_{j in split s} float(round_T(softmax(scores)[j])) * v_j[c]   (fp32; the consumer adds the
// splits in order and rounds once = the single rounding of `w @ v`).  Every CTA first derives the row maximum and the
// normaliser from ALL scores of its (n, h) (<= 1500 floats, L2-resident), as F.softmax(qk.float()) does.
template <typename T>
__global__ void __launch_bounds__(128) dec_attn_pv_kernel(const oasr_dec_attn_args a) {
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
  const T* vb = static_cast<const T*>(a.v) + static_cast<int64_t>(n) * a.kv_seq_stride + h * 64 + c8 * 8;
  float o[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  for (int jb = j0; jb < j1; jb += 128) {
    uint4 u[8];
    float p[8];
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      const int j = jb + r * 16 + slot;
      const bool ok = j < j1;
      u[r] = ok ? __ldg(reinterpret_cast<const uint4*>(vb + static_cast<int64_t>(j) * a.kv_row_stride)) : make_uint4(0, 0, 0, 0);
      p[r] = ok ? rnd<T>(expf(sc[j] - m) * inv_l) : 0.f;            // softmax(...).to(q.dtype)
    }
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      const uint32_t w[4] = {u[r].x, u[r].y, u[r].z, u[r].w};
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
template <typename T>
__global__ void __launch_bounds__(128) dec_attn_fused_kernel(const oasr_dec_attn_args a) {
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
  const T* kb = static_cast<const T*>(a.k) + static_cast<int64_t>(n) * a.kv_seq_stride + h * 64 + c8 * 8;
  const T* vb = static_cast<const T*>(a.v) + static_cast<int64_t>(n) * a.kv_seq_stride + h * 64 + c8 * 8;
  float m = -INFINITY;
  for (int jb = 0; jb < nkeys; jb += 128) {
    uint4 u[8];
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      const int j = jb + r * 16 + slot;
      u[r] = (j < nkeys) ? __ldg(reinterpret_cast<const uint4*>(kb + static_cast<int64_t>(j) * a.kv_row_stride)) : make_uint4(0, 0, 0, 0);
    }
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      const uint32_t w[4] = {u[r].x, u[r].y, u[r].z, u[r].w};
      float acc = 0.f;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float2 p = DT<T>::unpack2(w[i]);
        acc = fmaf(qs[2 * i], rnd<T>(p.x * scale), acc);
        acc = fmaf(qs[2 * i + 1], rnd<T>(p.y * scale), acc);
      }
      acc += __shfl_xor_sync(0xffffffffu, acc, 1);
      acc += __shfl_xor_sync(0xffffffffu, acc, 2);
      acc += __shfl_xor_sync(0xffffffffu, acc, 4);
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
    uint4 u[8];
    float p[8];
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      const int j = jb + r * 16 + slot;
      const bool ok = j < nkeys;
      u[r] = ok ? __ldg(reinterpret_cast<const uint4*>(vb + static_cast<int64_t>(j) * a.kv_row_stride)) : make_uint4(0, 0, 0, 0);
      p[r] = ok ? rnd<T>(expf(s_sc[j] - m) * inv_l) : 0.f;
    }
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      const uint32_t w[4] = {u[r].x, u[r].y, u[r].z, u[r].w};
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
// `n_slices` blocks per sequence, each over a contiguous slice of its fp32 logits row, one online pass with 16-byte loads
// (whisper/decoding.py: SuppressBlank, SuppressTokens, GreedyDecoder.update); the block that arrives last at the sequence's
// counter merges the slices in slice order (deterministic) and does the bookkeeping:
//   * at pos == sot_index: no_speech_prob = softmax(raw logits)[no_speech]                       (DecodingTask._main_loop)
//   * suppress[v] != 0 -> -inf; at the first sampled position also `blank` and `eot`            (SuppressTokens / SuppressBlank)
//   * next = argmax (lowest index on ties); logprob = logit[next] - logsumexp(filtered row)
//   * sum_logprobs += logprob unless the previous token is eot; rows whose previous token is eot keep emitting eot
// Positions before sample_begin - 1 are teacher-forced: nothing is written there.
struct SampleAcc {          // online (max, sum exp) of the raw and the filtered row + filtered argmax
  float mraw, sraw, mf, sf;
  int arg;
};
__device__ __forceinline__ void acc_raw(SampleAcc& s, float x) {
  if (x > s.mraw) { s.sraw = s.sraw * expf(s.mraw - x) + 1.f; s.mraw = x; }
  else s.sraw += expf(x - s.mraw);
}
__device__ __forceinline__ void acc_filt(SampleAcc& s, float x, int v) {
  if (x > s.mf) { s.sf = s.sf * expf(s.mf - x) + 1.f; s.mf = x; s.arg = v; }
  else { s.sf += expf(x - s.mf); if (x == s.mf && v < s.arg) s.arg = v; }
}
__device__ __forceinline__ SampleAcc acc_merge(const SampleAcc& a, const SampleAcc& b) {
  SampleAcc r;
  r.mraw = fmaxf(a.mraw, b.mraw);
  r.sraw = (r.mraw == -INFINITY) ? 0.f : a.sraw * expf(a.mraw - r.mraw) + b.sraw * expf(b.mraw - r.mraw);
  r.mf = fmaxf(a.mf, b.mf);
  r.sf = (r.mf == -INFINITY) ? 0.f : a.sf * expf(a.mf - r.mf) + b.sf * expf(b.mf - r.mf);
  r.arg = (a.mf > b.mf || (a.mf == b.mf && a.arg < b.arg)) ? a.arg : b.arg;
  return r;
}

__global__ void __launch_bounds__(256) dec_sample_kernel(const oasr_dec_sample_args a) {
  __shared__ SampleAcc s_acc[8];
  __shared__ int s_last;
  pdl_launch_dependents();
  pdl_wait();
  const int slice = blockIdx.x, n = blockIdx.y, S = gridDim.x;
  const int pos = *a.pos_ptr;
  const float* row = a.logits + static_cast<int64_t>(n) * a.ld_logits;
  const int V = a.n_vocab;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const bool first = (pos == a.sample_begin - 1);
  const bool sampling = pos >= a.sample_begin - 1;
  const bool want_raw = (pos == a.sot_index);
  if (!sampling && !want_raw) return;

  const int per = ((V + S - 1) / S + 3) & ~3;                  // slice length, a multiple of 4 (16-byte loads)
  const int v0 = slice * per, v1 = min(V, v0 + per);
  SampleAcc acc{-INFINITY, 0.f, -INFINITY, 0.f, V};
  const bool vec_ok = ((reinterpret_cast<uintptr_t>(row) & 15) == 0);
  auto visit = [&](float x, int v) {
    acc_raw(acc, x);
    const bool sup = a.suppress[v] != 0 || (first && a.suppress_blank && (v == a.blank || v == a.eot));
    if (!sup) acc_filt(acc, x, v);
  };
  if (vec_ok) {
    for (int v = v0 + threadIdx.x * 4; v < v1; v += 256 * 4) {
      if (v + 4 <= v1) {
        const float4 x = *reinterpret_cast<const float4*>(row + v);
        visit(x.x, v); visit(x.y, v + 1); visit(x.z, v + 2); visit(x.w, v + 3);
      } else {
        for (int u = v; u < v1; ++u) visit(row[u], u);
      }
    }
  } else {
    for (int v = v0 + threadIdx.x; v < v1; v += 256) visit(row[v], v);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    SampleAcc other;
    other.mraw = __shfl_xor_sync(0xffffffffu, acc.mraw, o); other.sraw = __shfl_xor_sync(0xffffffffu, acc.sraw, o);
    other.mf = __shfl_xor_sync(0xffffffffu, acc.mf, o); other.sf = __shfl_xor_sync(0xffffffffu, acc.sf, o);
    other.arg = __shfl_xor_sync(0xffffffffu, acc.arg, o);
    acc = acc_merge(acc, other);
  }
  if (lane == 0) s_acc[warp] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    SampleAcc t = s_acc[0];
    for (int w = 1; w < 8; ++w) t = acc_merge(t, s_acc[w]);
    float* out = a.scratch + (static_cast<int64_t>(n) * S + slice) * 8;
    out[0] = t.mraw; out[1] = t.sraw; out[2] = t.mf; out[3] = t.sf; out[4] = __int_as_float(t.arg);
    __threadfence();
    s_last = (atomicAdd(a.counters + n, 1) == S - 1) ? 1 : 0;
  }
  __syncthreads();
  if (!s_last || threadIdx.x != 0) return;
  __threadfence();
  SampleAcc t{-INFINITY, 0.f, -INFINITY, 0.f, V};
  for (int sl = 0; sl < S; ++sl) {       // slice order: the result does not depend on which block arrived last
    const volatile float* in = a.scratch + (static_cast<int64_t>(n) * S + sl) * 8;
    SampleAcc p;
    p.mraw = in[0]; p.sraw = in[1]; p.mf = in[2]; p.sf = in[3]; p.arg = __float_as_int(in[4]);
    t = acc_merge(t, p);
  }
  a.counters[n] = 0;                     // re-armed for the next step
  if (want_raw) a.no_speech_prob[n] = expf(row[a.no_speech] - t.mraw) / t.sraw;
  if (sampling) {
    const int prev = a.tokens[static_cast<int64_t>(n) * a.ld_tokens + pos];
    const bool finished = (prev == a.eot);
    const float logprob = -logf(t.sf);            // logit[arg] - (mf + log sum exp(x - mf)), logit[arg] == mf
    if (!finished) a.sum_logprobs[n] += logprob;
    const int next = finished ? a.eot : t.arg;
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

template <typename T, int MT>
int launch_linear(const oasr_dec_linear_args& a, cudaStream_t st) {
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
    OASR_CUDA_OK(cudaFuncSetAttribute(dec_linear_kernel<T, MT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)budget));
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
  OASR_CUDA_OK(cudaLaunchKernelEx(&cfg, dec_linear_kernel<T, MT>, a, KC, groups));
  return OASR_OK;
}
template <typename T, int MT>
int launch_linear_direct(const oasr_dec_linear_args& a, cudaStream_t st) {
  OASR_CUDA_OK(launch_pdl(dec_linear_direct_kernel<T, MT>, dim3((unsigned)ceil_div(a.N, 16)), dim3(256), st, a));
  return OASR_OK;
}
template <typename T>
int dispatch_linear(const oasr_dec_linear_args& a, cudaStream_t st) {
  // the direct form up to 32 rows (no staging round trip for a handful of rows), the staged form from there on
  if (a.M <= 16) return launch_linear_direct<T, 1>(a, st);
  if (a.M <= 32) return launch_linear_direct<T, 2>(a, st);
  return launch_linear<T, 4>(a, st);
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
  if (a->dtype == OASR_DTYPE_F16) return dispatch_linear<__half>(*a, (cudaStream_t)stream);
  if (a->dtype == OASR_DTYPE_BF16) return dispatch_linear<bf16>(*a, (cudaStream_t)stream);
  OASR_REQUIRE(false, "dec_linear: unknown dtype %d", a->dtype);
}

extern "C" int oasr_dec_attention(const oasr_dec_attn_args* a, void* stream) {
  OASR_REQUIRE(a != nullptr && a->q && a->k && a->v && a->scores && a->out_partial, "dec_attention: null tensor");
  OASR_REQUIRE(a->n_seq >= 1 && a->n_head >= 1 && a->n_splits >= 1, "dec_attention: bad sizes");
  OASR_REQUIRE(a->pos_ptr != nullptr || a->n_keys >= 1, "dec_attention: key count missing");
  OASR_REQUIRE((a->ldq % 8) == 0 && (a->kv_row_stride % 8) == 0 && (a->kv_seq_stride % 8) == 0, "dec_attention: strides must be multiples of 8");
  dim3 grid((unsigned)a->n_splits, (unsigned)a->n_head, (unsigned)a->n_seq);
  cudaStream_t st = (cudaStream_t)stream;
  OASR_REQUIRE(a->dtype == OASR_DTYPE_F16 || a->dtype == OASR_DTYPE_BF16, "dec_attention: unknown dtype %d", a->dtype);
  const bool f16 = a->dtype == OASR_DTYPE_F16;
  if (a->n_splits == 1 && (a->pos_ptr != nullptr || a->n_keys <= 1536)) {   // whole key range in one CTA: fused form
    if (f16) OASR_CUDA_OK(launch_pdl(dec_attn_fused_kernel<__half>, grid, dim3(128), st, *a));
    else OASR_CUDA_OK(launch_pdl(dec_attn_fused_kernel<bf16>, grid, dim3(128), st, *a));
    return OASR_OK;
  }
  if (f16) {
    OASR_CUDA_OK(launch_pdl(dec_attn_scores_kernel<__half>, grid, dim3(128), st, *a));
    OASR_CUDA_OK(launch_pdl(dec_attn_pv_kernel<__half>, grid, dim3(128), st, *a));
  } else {
    OASR_CUDA_OK(launch_pdl(dec_attn_scores_kernel<bf16>, grid, dim3(128), st, *a));
    OASR_CUDA_OK(launch_pdl(dec_attn_pv_kernel<bf16>, grid, dim3(128), st, *a));
  }
  return OASR_OK;
}

extern "C" int oasr_dec_sample(const oasr_dec_sample_args* a, void* stream) {
  OASR_REQUIRE(a != nullptr && a->logits && a->tokens && a->pos_ptr && a->suppress && a->sum_logprobs && a->no_speech_prob &&
                   a->n_unfinished && a->done_flag, "dec_sample: null tensor");
  OASR_REQUIRE(a->n_seq >= 1 && a->n_vocab >= 1, "dec_sample: bad sizes");
  OASR_REQUIRE(a->scratch && a->counters && a->n_slices >= 1 && a->n_slices <= 64, "dec_sample: scratch / counters / 1 <= n_slices <= 64");
  OASR_CUDA_OK(launch_pdl(dec_sample_kernel, dim3((unsigned)a->n_slices, (unsigned)a->n_seq), dim3(256), (cudaStream_t)stream, *a));
  OASR_CUDA_OK(launch_pdl(dec_advance_kernel, dim3(1), dim3(1), (cudaStream_t)stream, a->pos_ptr, a->n_unfinished, a->done_flag,
                          (int)a->sample_begin));
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
