// Flash-style attention forward for head_dim 64 on wgmma (sm_90a).
//
//   O = softmax(Q K^T * scale + mask) V        per (batch, head); bf16 or fp16 in/out, fp32 softmax
//
// Replaces F.scaled_dot_product_attention in MultiHeadAttention.forward (olmoasr/model.py:331-340):
//   encoder self-attention (no mask), decoder self-attention (causal + per-sample key length, derived
//   from the dense additive mask the reference passes, model.py:740-743) and cross-attention (no mask).
//
// One CTA per (128-query tile, head, sample), 384 threads = three warpgroups.  In warpgroup 0 one thread is the TMA
// producer: it loads Q and streams the K / V tiles of 128 keys through a three-stage ring (full / empty mbarrier per
// stage; no CTA-wide barrier in the loop).  Warpgroups 1 and 2 consume, 64 query rows each.  There is no setmaxnreg
// hand-over: ptxas allocates the whole kernel under the 168-register cap of a 384-thread launch, the consumers fit in
// it, and a producer cut below what ptxas gave it would lose live registers.  Per key tile a consumer runs
//     S = Q K^T          4 x wgmma m64n128k16, Q and K from 128B-swizzled smem, fp32 S in registers
//     online softmax     thread owns rows lane/4 and lane/4 + 8 of its warp's 16: row max / sum over the 4-lane quad
//     O += P V           8 x wgmma m64n64k16 with P as the register A operand (the S fragment re-packed to 16 bits) and
//                        V MN-major from its TMA tile
// software-pipelined one tile deep: S_{j+1} and O += P_j V_j are issued together and the exponentials of tile j + 1 run
// (in place, in fp32) while P_j V_j is still on the tensor cores; P_{j+1} is packed to 16 bits once P_j V_j retires.  The arithmetic (tile sizes, k16 order, masks, exp2) is that of the
// unpipelined loop, so the results are bit-for-bit the same.  The output leaves straight from the O fragment.
//
// Packed (varlen) batches: with q_off set, sample b's query rows are rows [q_off[b], q_off[b+1]) of Q / O, Tq is their
// total N, LSE is (1, H, N), and the grid runs one CTA per entry of `tiles` (sample, 128-row tile) instead of
// (tile, head, sample).  kv_off set: K / V are packed the same way (causal self-attention, the sample's own keys); unset:
// sample b's keys are dense rows [b Tkv, b Tkv + Tkv).  A tile's TMA box may reach into the next sample's rows; those are
// masked (keys) or never stored (queries), so every O / LSE store is guarded by the sample's own length.
#include "common.cuh"
#include "ptx_sm90.cuh"

#include <stdlib.h>

namespace oasr {
namespace {

constexpr int HD = 64;
constexpr int BQ = 128;                      // query rows per CTA (64 per consumer warpgroup)
constexpr int BKV = 128;
constexpr int STAGES = 3;                    // K/V ring: tile j + 1 is waited on while tile j - 1's stage refills
constexpr int TILE_BYTES = 128 * HD * 2;     // 16 KB: a [128 rows][64 16-bit] swizzled tile
constexpr int ATT_TILES = TILE_BYTES /*Q*/ + STAGES * 2 * TILE_BYTES /*K,V per stage*/;   // 112 KB
constexpr int ATT_SMEM = ATT_TILES + 1024 /*barriers*/ + 1024 /*alignment slack*/;
constexpr int THREADS = 384;

struct AttnParams {
  void* o;
  int64_t ldo;
  float* lse;        // (B, H, Tq) log2-domain log-sum-exp, nullable
  const int32_t* kv_len;  // (B,) valid keys per sample, nullable
  int B, H, Tq, Tkv;
  int causal;
  float scale_log2;  // scale * log2(e)
  const int32_t* q_off;   // (B+1,) packed query row offsets, nullable (dense: sample b at rows b Tq)
  const int32_t* kv_off;  // (B+1,) packed key row offsets, nullable (dense: sample b at rows b Tkv)
  const int32_t* tiles;   // (sample, query tile) int32 pairs, one per CTA when q_off is set (4-byte aligned)
};

__device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

// PACKED: the packed-batch form.  A compile-time switch, so that the dense instantiation is the dense kernel as it was.
template <typename T, bool PACKED>
__global__ void __launch_bounds__(THREADS, 1)
attention_fwd_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                     const __grid_constant__ CUtensorMap tmV, const AttnParams p) {
  extern __shared__ uint8_t smem_dyn[];
  uint8_t* smem_raw = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_raw + ATT_TILES);
  uint64_t& bar_q = bars[0];
  uint64_t* bar_full = bars + 1;             // [STAGES]: K and V of key tile j landed in stage j % STAGES
  uint64_t* bar_empty = bar_full + STAGES;   // [STAGES]: both consumers are done with the stage

  const uint32_t sQ = ptx::smem_u32(smem_raw);
  const uint32_t sKV = sQ + TILE_BYTES;   // stage s: K at sKV + s*32K, V right after K
  const int qblk = PACKED ? p.tiles[2 * blockIdx.x + 1] : blockIdx.x, h = blockIdx.y;
  const int b = PACKED ? p.tiles[2 * blockIdx.x] : blockIdx.z;
  const int q_base = qblk * BQ;
  const int q_row0 = PACKED ? p.q_off[b] : b * p.Tq;                   // first Q / O row of the sample
  const int tq = PACKED ? p.q_off[b + 1] - q_row0 : p.Tq;              // its query rows
  const bool kv_packed = PACKED && p.kv_off;
  const int kv_row0 = kv_packed ? p.kv_off[b] : b * p.Tkv;
  int kv_valid = kv_packed ? p.kv_off[b + 1] - kv_row0 : p.Tkv;
  if (p.kv_len) kv_valid = min(kv_valid, max(1, p.kv_len[b]));
  const int kv_end = p.causal ? min(kv_valid, q_base + BQ) : kv_valid;
  const int n_kv = (kv_end + BKV - 1) / BKV;   // >= 1: every sample has at least one visible key

  if (threadIdx.x == 0) {
    ptx::tma_prefetch_desc(&tmQ); ptx::tma_prefetch_desc(&tmK); ptx::tma_prefetch_desc(&tmV);
    ptx::mbar_init(ptx::smem_u32(&bar_q), 1);
    for (int s = 0; s < STAGES; ++s) {
      ptx::mbar_init(ptx::smem_u32(&bar_full[s]), 1);
      ptx::mbar_init(ptx::smem_u32(&bar_empty[s]), 2);   // one arrival per consumer warpgroup
    }
    ptx::fence_barrier_init();
  }
  __syncthreads();

  if (threadIdx.x < 128) {
    // ===================== TMA producer =====================
    if (threadIdx.x == 0) {
      ptx::mbar_arrive_expect_tx(ptx::smem_u32(&bar_q), TILE_BYTES);
      ptx::tma_load_2d(sQ, &tmQ, ptx::smem_u32(&bar_q), h * HD, PACKED ? q_row0 + q_base : b * p.Tq + q_base);
      for (int j = 0; j < n_kv; ++j) {
        const int st = j % STAGES;
        ptx::mbar_wait(ptx::smem_u32(&bar_empty[st]), ((j / STAGES) & 1) ^ 1);
        const uint32_t full = ptx::smem_u32(&bar_full[st]);
        const uint32_t dst = sKV + st * 2 * TILE_BYTES;
        ptx::mbar_arrive_expect_tx(full, 2 * TILE_BYTES);
        const int row = kv_packed ? kv_row0 + j * BKV : b * p.Tkv + j * BKV;   // dense: the expression as written before
        ptx::tma_load_2d(dst, &tmK, full, h * HD, row);
        ptx::tma_load_2d(dst + TILE_BYTES, &tmV, full, h * HD, row);
      }
    }
    return;
  }

  // ===================== consumers =====================
  const int wg = (threadIdx.x >> 7) - 1;   // query-row half of the tile
  const int t = threadIdx.x & 127;
  const int warp = t >> 5, lane = t & 31;
  const int r_loc = wg * 64 + warp * 16 + (lane >> 2);   // rows r_loc and r_loc + 8 of the CTA's query tile
  const int kc = 2 * (lane & 3);
  const float c = p.scale_log2;
  const uint64_t q_desc = ptx::desc_sw128(sQ + wg * 8192, 16, 1024);

  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};   // l: this thread's share of the row sum
  float s[64];

  // S = Q K_j^T into s (one commit group)
  auto issue_s = [&](int j) {
    const int st = j % STAGES;
    ptx::mbar_wait(ptx::smem_u32(&bar_full[st]), (j / STAGES) & 1);
    const uint64_t k_desc = ptx::desc_sw128(sKV + st * 2 * TILE_BYTES, 16, 1024);
    ptx::wgmma_fence();
#pragma unroll
    for (int k = 0; k < HD / 16; ++k) ptx::wgmma_m64n128k16_ss<0, 0, T>(s, ptx::desc_add(q_desc, 32 * k), ptx::desc_add(k_desc, 32 * k), k > 0);
    ptx::wgmma_commit();
  };
  // masks tile j of s, updates m / l and overwrites s with p = 2^(s c - m c)
  auto softmax = [&](int j, float (&alpha)[2]) {
    // mask: keys [0, limit) of this tile are visible to a row
    const int k0 = j * BKV;
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
    float neg[2];
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
#pragma unroll
    for (int i = 0; i < 16; ++i) {
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const float p0 = fast_exp2(fmaf(s[4 * i + 2 * hh], c, neg[hh]));
        const float p1 = fast_exp2(fmaf(s[4 * i + 2 * hh + 1], c, neg[hh]));
        l[hh] += p0 + p1;
        s[4 * i + 2 * hh] = p0;
        s[4 * i + 2 * hh + 1] = p1;
      }
    }
  };
  // P packed to T in the A-fragment order of the P V MMA
  uint32_t pa[8][4];
  auto pack_p = [&]() {
#pragma unroll
    for (int i = 0; i < 16; ++i)
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) pa[i >> 1][(i & 1) * 2 + hh] = Act16<T>::pack2(s[4 * i + 2 * hh], s[4 * i + 2 * hh + 1]);
  };

  float alpha[2];
  ptx::mbar_wait(ptx::smem_u32(&bar_q), 0);
  issue_s(0);
  ptx::wgmma_wait<0>();
  ptx::fence_regs(s);
  softmax(0, alpha);
  pack_p();

  // O = O alpha + P_j V_j (one commit group)
  auto issue_pv = [&](int j) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      o[4 * i] *= alpha[0]; o[4 * i + 1] *= alpha[0];
      o[4 * i + 2] *= alpha[1]; o[4 * i + 3] *= alpha[1];
    }
    const uint64_t v_desc = ptx::desc_sw128(sKV + (j % STAGES) * 2 * TILE_BYTES + TILE_BYTES, BKV * 128, 1024);
    ptx::wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < BKV / 16; ++kk) ptx::wgmma_m64n64k16_rs<1, T>(o, pa[kk], ptx::desc_add(v_desc, 2048 * kk), 1u);
    ptx::wgmma_commit();
  };
  auto retire_pv = [&](int j) {
    ptx::wgmma_wait<0>();
    ptx::fence_regs(o);
    if (t == 0) ptx::mbar_arrive(ptx::smem_u32(&bar_empty[j % STAGES]));   // K_j and V_j are no longer read
  };
  for (int j = 0; j + 1 < n_kv; ++j) {
    issue_s(j + 1);
    issue_pv(j);
    ptx::wgmma_wait<1>();   // S_{j+1} is in; P_j V_j may still be running
    ptx::fence_regs(s);
    softmax(j + 1, alpha);
    retire_pv(j);
    pack_p();
  }
  issue_pv(n_kv - 1);
  retire_pv(n_kv - 1);

  // ---- output: O / l -> T, rows past the sample's length are not written; lse in the log2 domain
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const float lsum = quad_sum(l[hh]);
    const float inv = 1.f / lsum;
    const int qi = q_base + r_loc + 8 * hh;
    if (qi < tq) {
      const int64_t row = PACKED ? static_cast<int64_t>(q_row0) + qi : static_cast<int64_t>(b) * p.Tq + qi;
      T* dst = static_cast<T*>(p.o) + row * p.ldo + h * HD + 2 * (lane & 3);
#pragma unroll
      for (int i = 0; i < 8; ++i)
        *reinterpret_cast<uint32_t*>(dst + 8 * i) = Act16<T>::pack2(o[4 * i + 2 * hh] * inv, o[4 * i + 2 * hh + 1] * inv);
      if (p.lse && (lane & 3) == 0)
        p.lse[(PACKED ? static_cast<int64_t>(h) * p.Tq + q_row0 : (static_cast<int64_t>(b) * p.H + h) * p.Tq) + qi] =
            m[hh] * c + log2f(lsum);
    }
  }
}

// Dense: B samples of Tq query and Tkv key rows.  Packed (q_off set): Tq is the total N of packed query rows, kv_off set
// makes Tkv the total of packed key rows, unset keeps B dense samples of Tkv keys; one CTA per (tiles entry, head).
template <typename T>
int attention_fwd(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, void* o, int64_t ldo,
                  float* lse, int64_t B, int64_t H, int64_t Tq, int64_t Tkv, int64_t head_dim, int causal,
                  const int32_t* kv_len, float scale, void* stream, const int32_t* q_off = nullptr,
                  const int32_t* kv_off = nullptr, const int32_t* tiles = nullptr, int64_t n_tiles = 0) {
  OASR_REQUIRE(head_dim == HD, "attention: head_dim %ld unsupported (every OLMoASR variant uses 64)", (long)head_dim);
  OASR_REQUIRE(B > 0 && H > 0 && Tq > 0 && Tkv > 0, "attention: empty problem");
  OASR_REQUIRE((ldq & 7) == 0 && (ldk & 7) == 0 && (ldv & 7) == 0 && (ldo & 7) == 0, "attention: strides must be multiples of 8");
  OASR_REQUIRE((reinterpret_cast<uintptr_t>(o) & 3) == 0, "attention: output must be 4-byte aligned");
  OASR_REQUIRE(!causal || Tq == Tkv, "attention: causal needs Tq == Tkv");
  OASR_REQUIRE(B <= 65535 && H <= 65535, "attention: B and H must fit the grid");
  OASR_REQUIRE(!q_off || (tiles && n_tiles > 0 && n_tiles <= 0x7fffffff), "attention: a packed batch needs its tile list");
  OASR_REQUIRE(!kv_off || q_off, "attention: packed keys need packed queries");
  OASR_REQUIRE(!causal || !q_off || kv_off == q_off, "attention: packed causal attention reads keys packed like the queries");
  const uint64_t q_rows = q_off ? Tq : B * Tq, kv_rows = kv_off ? Tkv : B * Tkv;
  CUtensorMap tmQ, tmK, tmV;
  constexpr bool f16 = Act16<T>::is_fp16;
  int rc;
  if ((rc = make_tmap_2d(&tmQ, q, 2, (uint64_t)(H * HD), q_rows, (uint64_t)ldq * 2, HD, BQ, true, f16))) return rc;
  if ((rc = make_tmap_2d(&tmK, k, 2, (uint64_t)(H * HD), kv_rows, (uint64_t)ldk * 2, HD, BKV, true, f16))) return rc;
  if ((rc = make_tmap_2d(&tmV, v, 2, (uint64_t)(H * HD), kv_rows, (uint64_t)ldv * 2, HD, BKV, true, f16))) return rc;
  AttnParams p;
  p.o = o; p.ldo = ldo;
  p.lse = lse; p.kv_len = kv_len;
  p.q_off = q_off; p.kv_off = kv_off; p.tiles = q_off ? tiles : nullptr;
  p.B = (int)B; p.H = (int)H; p.Tq = (int)Tq; p.Tkv = (int)Tkv; p.causal = causal;
  p.scale_log2 = scale * 1.4426950408889634f;
  static bool attr_set = false;
  if (!attr_set) {
    OASR_CUDA_OK(cudaFuncSetAttribute(attention_fwd_kernel<T, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, ATT_SMEM));
    OASR_CUDA_OK(cudaFuncSetAttribute(attention_fwd_kernel<T, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, ATT_SMEM));
    attr_set = true;
  }
  if (q_off)
    attention_fwd_kernel<T, true><<<dim3((unsigned)n_tiles, (unsigned)H, 1u), THREADS, ATT_SMEM, (cudaStream_t)stream>>>(tmQ, tmK, tmV, p);
  else
    attention_fwd_kernel<T, false><<<dim3((unsigned)ceil_div(Tq, BQ), (unsigned)H, (unsigned)B), THREADS, ATT_SMEM,
                                     (cudaStream_t)stream>>>(tmQ, tmK, tmV, p);
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

extern "C" int oasr_attention_fwd_varlen16(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v,
                                           int64_t ldv, void* o, int64_t ldo, float* lse, int64_t B, int64_t H, int64_t N,
                                           int64_t Tkv, int64_t head_dim, const int32_t* cu_seqlens,
                                           const int32_t* kv_cu_seqlens, const int32_t* tiles, int64_t n_tiles, float scale,
                                           int dtype, void* stream) {
  OASR_REQUIRE(cu_seqlens, "attention_varlen: cu_seqlens is required");
  const int causal = kv_cu_seqlens != nullptr;
  return OASR_BY_DTYPE16(dtype, attention_fwd, q, ldq, k, ldk, v, ldv, o, ldo, lse, B, H, N, causal ? N : Tkv, head_dim, causal,
                         nullptr, scale, stream, cu_seqlens, kv_cu_seqlens, tiles, n_tiles);
}
