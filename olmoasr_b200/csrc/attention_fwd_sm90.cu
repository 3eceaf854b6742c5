// Flash-style attention forward for head_dim 64 on wgmma (sm_90a).
//
//   O = softmax(Q K^T * scale + mask) V        per (batch, head); bf16 or fp16 in/out, fp32 softmax
//
// Replaces F.scaled_dot_product_attention in MultiHeadAttention.forward (olmoasr/model.py:331-340):
//   encoder self-attention (no mask), decoder self-attention (causal + per-sample key length, derived
//   from the dense additive mask the reference passes, model.py:740-743) and cross-attention (no mask).
//
// One CTA per (128-query tile, head, sample), 256 threads = two warpgroups of 64 query rows each.  K / V tiles of 128
// keys stream through a two-stage TMA ring shared by both warpgroups (the load of tile j+1 is in flight while tile j is
// computed).  Per key tile a warpgroup runs
//     S = Q K^T          4 x wgmma m64n128k16, Q and K from 128B-swizzled smem, fp32 S in registers
//     online softmax     thread owns rows lane/4 and lane/4 + 8 of its warp's 16: row max / sum over the 4-lane quad
//     O += P V           8 x wgmma m64n64k16 with P as the register A operand (the S fragment re-packed to bf16) and
//                        V MN-major from its TMA tile
// and the output leaves straight from the O fragment.
#include "common.cuh"
#include "ptx_sm90.cuh"

#include <stdlib.h>

namespace oasr {
namespace {

constexpr int HD = 64;
constexpr int BQ = 128;                      // query rows per CTA (64 per warpgroup)
constexpr int BKV = 128;
constexpr int TILE_BYTES = 128 * HD * 2;     // 16 KB: a [128 rows][64 bf16] swizzled tile
constexpr int ATT_TILES = TILE_BYTES /*Q*/ + 2 * 2 * TILE_BYTES /*K,V x 2 stages*/;   // 80 KB
constexpr int ATT_SMEM = ATT_TILES + 1024 /*barriers*/ + 1024 /*alignment slack*/;
constexpr int THREADS = 256;

struct AttnParams {
  void* o;
  int64_t ldo;
  float* lse;        // (B, H, Tq) log2-domain log-sum-exp, nullable
  const int32_t* kv_len;  // (B,) valid keys per sample, nullable
  int B, H, Tq, Tkv;
  int causal;
  float scale_log2;  // scale * log2(e)
};

__device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

template <typename T>
__global__ void __launch_bounds__(THREADS, 1)
attention_fwd_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                     const __grid_constant__ CUtensorMap tmV, const AttnParams p) {
  extern __shared__ uint8_t smem_dyn[];
  uint8_t* smem_raw = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_raw + ATT_TILES);
  uint64_t& bar_q = bars[0];
  uint64_t* bar_kv = bars + 1;   // [2]: K and V of a key tile landed in stage s (parity: (j / 2) & 1)

  const uint32_t sQ = ptx::smem_u32(smem_raw);
  const uint32_t sKV = sQ + TILE_BYTES;   // stage s: K at sKV + s*32K, V right after K
  const int qblk = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int q_base = qblk * BQ;
  int kv_valid = p.Tkv;
  if (p.kv_len) kv_valid = min(kv_valid, max(1, p.kv_len[b]));
  const int kv_end = p.causal ? min(kv_valid, q_base + BQ) : kv_valid;
  const int n_kv = (kv_end + BKV - 1) / BKV;   // >= 1: every sample has at least one visible key

  if (threadIdx.x == 0) {
    ptx::tma_prefetch_desc(&tmQ); ptx::tma_prefetch_desc(&tmK); ptx::tma_prefetch_desc(&tmV);
    ptx::mbar_init(ptx::smem_u32(&bar_q), 1);
    ptx::mbar_init(ptx::smem_u32(&bar_kv[0]), 1);
    ptx::mbar_init(ptx::smem_u32(&bar_kv[1]), 1);
    ptx::fence_barrier_init();
  }
  __syncthreads();
  auto load_kv = [&](int j) {   // thread 0 only
    const uint32_t full = ptx::smem_u32(&bar_kv[j & 1]);
    const uint32_t dst = sKV + (j & 1) * 2 * TILE_BYTES;
    ptx::mbar_arrive_expect_tx(full, 2 * TILE_BYTES);
    ptx::tma_load_2d(dst, &tmK, full, h * HD, b * p.Tkv + j * BKV);
    ptx::tma_load_2d(dst + TILE_BYTES, &tmV, full, h * HD, b * p.Tkv + j * BKV);
  };
  if (threadIdx.x == 0) {
    ptx::mbar_arrive_expect_tx(ptx::smem_u32(&bar_q), TILE_BYTES);
    ptx::tma_load_2d(sQ, &tmQ, ptx::smem_u32(&bar_q), h * HD, b * p.Tq + q_base);
    load_kv(0);
  }

  const int wg = threadIdx.x >> 7;
  const int t = threadIdx.x & 127;
  const int warp = t >> 5, lane = t & 31;
  const int r_loc = wg * 64 + warp * 16 + (lane >> 2);   // rows r_loc and r_loc + 8 of the CTA's query tile
  const float c = p.scale_log2;
  const uint64_t q_desc = ptx::desc_sw128(sQ + wg * 8192, 16, 1024);

  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};   // l: this thread's share of the row sum
  ptx::mbar_wait(ptx::smem_u32(&bar_q), 0);

  for (int j = 0; j < n_kv; ++j) {
    if (threadIdx.x == 0 && j + 1 < n_kv) load_kv(j + 1);   // its stage was released by the __syncthreads of j - 1
    ptx::mbar_wait(ptx::smem_u32(&bar_kv[j & 1]), (j >> 1) & 1);
    const uint32_t sK = sKV + (j & 1) * 2 * TILE_BYTES, sV = sK + TILE_BYTES;

    float s[64];
    const uint64_t k_desc = ptx::desc_sw128(sK, 16, 1024);
    ptx::wgmma_fence();
#pragma unroll
    for (int k = 0; k < HD / 16; ++k) ptx::wgmma_m64n128k16_ss<0, 0, T>(s, ptx::desc_add(q_desc, 32 * k), ptx::desc_add(k_desc, 32 * k), k > 0);
    ptx::wgmma_commit();
    ptx::wgmma_wait<0>();
    ptx::fence_regs(s);

    // mask: keys [0, limit) of this tile are visible to a row
    const int k0 = j * BKV;
    const int kc = 2 * (lane & 3);
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int qi = q_base + r_loc + 8 * hh;
      int limit = kv_valid - k0;
      if (p.causal) limit = min(limit, qi - k0 + 1);
      if (limit < BKV) {
#pragma unroll
        for (int i = 0; i < 16; ++i) {
          if (8 * i + kc >= limit) s[4 * i + 2 * hh] = -INFINITY;
          if (8 * i + kc + 1 >= limit) s[4 * i + 2 * hh + 1] = -INFINITY;
        }
      }
    }
    float alpha[2], neg[2];
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      float mx = -INFINITY;
#pragma unroll
      for (int i = 0; i < 16; ++i) mx = fmaxf(mx, fmaxf(s[4 * i + 2 * hh], s[4 * i + 2 * hh + 1]));
      mx = quad_max(mx);
      const float m_new = fmaxf(m[hh], mx);
      alpha[hh] = (m_new == -INFINITY) ? 1.f : fast_exp2((m[hh] - m_new) * c);
      neg[hh] = (m_new == -INFINITY) ? 0.f : -m_new * c;
      m[hh] = m_new;
      l[hh] *= alpha[hh];
    }
    // p = 2^(s c - m c); P packed to T in the A-fragment order of the P V MMA
    uint32_t pa[8][4];
#pragma unroll
    for (int i = 0; i < 16; ++i) {
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const float p0 = fast_exp2(fmaf(s[4 * i + 2 * hh], c, neg[hh]));
        const float p1 = fast_exp2(fmaf(s[4 * i + 2 * hh + 1], c, neg[hh]));
        l[hh] += p0 + p1;
        pa[i >> 1][(i & 1) * 2 + hh] = Act16<T>::pack2(p0, p1);
      }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      o[4 * i] *= alpha[0]; o[4 * i + 1] *= alpha[0];
      o[4 * i + 2] *= alpha[1]; o[4 * i + 3] *= alpha[1];
    }
    const uint64_t v_desc = ptx::desc_sw128(sV, BKV * 128, 1024);
    ptx::wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < BKV / 16; ++kk) ptx::wgmma_m64n64k16_rs<1, T>(o, pa[kk], ptx::desc_add(v_desc, 2048 * kk), 1u);
    ptx::wgmma_commit();
    ptx::wgmma_wait<0>();
    ptx::fence_regs(o);
    __syncthreads();   // both warpgroups are done with this stage: it may be refilled
  }

  // ---- output: O / l -> T, rows past Tq are not written; lse in the log2 domain
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const float lsum = quad_sum(l[hh]);
    const float inv = 1.f / lsum;
    const int qi = q_base + r_loc + 8 * hh;
    if (qi < p.Tq) {
      T* dst = static_cast<T*>(p.o) + (static_cast<int64_t>(b) * p.Tq + qi) * p.ldo + h * HD + 2 * (lane & 3);
#pragma unroll
      for (int i = 0; i < 8; ++i)
        *reinterpret_cast<uint32_t*>(dst + 8 * i) = Act16<T>::pack2(o[4 * i + 2 * hh] * inv, o[4 * i + 2 * hh + 1] * inv);
      if (p.lse && (lane & 3) == 0) p.lse[(static_cast<int64_t>(b) * p.H + h) * p.Tq + qi] = m[hh] * c + log2f(lsum);
    }
  }
}

template <typename T>
int attention_fwd(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, void* o, int64_t ldo,
                  float* lse, int64_t B, int64_t H, int64_t Tq, int64_t Tkv, int64_t head_dim, int causal,
                  const int32_t* kv_len, float scale, void* stream) {
  OASR_REQUIRE(head_dim == HD, "attention: head_dim %ld unsupported (every OLMoASR variant uses 64)", (long)head_dim);
  OASR_REQUIRE(B > 0 && H > 0 && Tq > 0 && Tkv > 0, "attention: empty problem");
  OASR_REQUIRE((ldq & 7) == 0 && (ldk & 7) == 0 && (ldv & 7) == 0 && (ldo & 7) == 0, "attention: strides must be multiples of 8");
  OASR_REQUIRE((reinterpret_cast<uintptr_t>(o) & 3) == 0, "attention: output must be 4-byte aligned");
  OASR_REQUIRE(!causal || Tq == Tkv, "attention: causal needs Tq == Tkv");
  OASR_REQUIRE(B <= 65535 && H <= 65535, "attention: B and H must fit the grid");
  CUtensorMap tmQ, tmK, tmV;
  constexpr bool f16 = Act16<T>::is_fp16;
  int rc;
  if ((rc = make_tmap_2d(&tmQ, q, 2, (uint64_t)(H * HD), (uint64_t)(B * Tq), (uint64_t)ldq * 2, HD, BQ, true, f16))) return rc;
  if ((rc = make_tmap_2d(&tmK, k, 2, (uint64_t)(H * HD), (uint64_t)(B * Tkv), (uint64_t)ldk * 2, HD, BKV, true, f16))) return rc;
  if ((rc = make_tmap_2d(&tmV, v, 2, (uint64_t)(H * HD), (uint64_t)(B * Tkv), (uint64_t)ldv * 2, HD, BKV, true, f16))) return rc;
  AttnParams p;
  p.o = o; p.ldo = ldo;
  p.lse = lse; p.kv_len = kv_len;
  p.B = (int)B; p.H = (int)H; p.Tq = (int)Tq; p.Tkv = (int)Tkv; p.causal = causal;
  p.scale_log2 = scale * 1.4426950408889634f;
  static bool attr_set = false;
  if (!attr_set) {
    OASR_CUDA_OK(cudaFuncSetAttribute(attention_fwd_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, ATT_SMEM));
    attr_set = true;
  }
  const dim3 grid((unsigned)ceil_div(Tq, BQ), (unsigned)H, (unsigned)B);
  attention_fwd_kernel<T><<<grid, THREADS, ATT_SMEM, (cudaStream_t)stream>>>(tmQ, tmK, tmV, p);
  OASR_LAUNCH_CHECK();
  return OASR_OK;
}

}  // namespace
}  // namespace oasr

using namespace oasr;

extern "C" int oasr_attention_fwd(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv,
                                  void* o, int64_t ldo, float* lse, int64_t B, int64_t H, int64_t Tq, int64_t Tkv,
                                  int64_t head_dim, int causal, const int32_t* kv_len, float scale, void* stream) {
  return attention_fwd<bf16>(q, ldq, k, ldk, v, ldv, o, ldo, lse, B, H, Tq, Tkv, head_dim, causal, kv_len, scale, stream);
}

extern "C" int oasr_attention_fwd16(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv,
                                    void* o, int64_t ldo, float* lse, int64_t B, int64_t H, int64_t Tq, int64_t Tkv,
                                    int64_t head_dim, int causal, const int32_t* kv_len, float scale, int dtype, void* stream) {
  return OASR_BY_DTYPE16(dtype, attention_fwd, q, ldq, k, ldk, v, ldv, o, ldo, lse, B, H, Tq, Tkv, head_dim, causal, kv_len,
                         scale, stream);
}
