// Flash-style attention backward for head_dim 64 on wgmma (sm_90a).
//
// Autograd of F.scaled_dot_product_attention (olmoasr/model.py:331-340) for the three training uses
// (encoder self, decoder causal+length self, cross).  Given Q, K, V, O, dO and the forward's log2-domain
// LSE it produces dQ, dK, dV without ever materialising the (Tq x Tkv) score matrix in HBM.
//
// One CTA per (128-key tile, head, sample), 256 threads = two warpgroups of 64 keys each, looping over the 64-query
// tiles that can see the keys (Q / dO tiles stream through a two-stage TMA ring shared by both warpgroups).  Everything
// is computed transposed, with the warpgroup's keys as the MMA rows, so that dK and dV stay in registers for the loop:
//     S^T  = K Q^T         dP^T = V dO^T                 wgmma m64n64k16, all operands from swizzled smem
//     P^T  = exp2(S^T c - LSE)   dS^T = P^T o (dP^T - D) thread-local: LSE / D are per query = per column
//     dV  += P^T dO        dK  += dS^T Q                 P^T / dS^T as register A operands, dO / Q MN-major
// dK / dV leave straight from the fragments.  dQ is a sum over every key tile; rather than letting the key-tile CTAs add
// into it with atomics (whose order, and so rounding, changes from run to run), a second kernel owns each 128-query tile,
// recomputes S and dP for it and accumulates dQ = sum_j dS_j K_j over the key tiles in order:
//     S = Q K^T   dP = dO V^T   (wgmma m64n128k16)   dS = P o (dP - D)   dQ += dS K   (dS as register A, K MN-major)
#include "common.cuh"
#include "ptx_sm90.cuh"

#include <stdlib.h>

namespace oasr {
namespace {

constexpr int HD = 64;
constexpr int BQ = 64;                     // queries per loop iteration
constexpr int BKV = 128;                   // keys per CTA (64 per warpgroup)
constexpr int KV_BYTES = BKV * HD * 2;     // 16 KB
constexpr int QT_BYTES = BQ * HD * 2;      // 8 KB
// K, V | (Q, dO) x 2 stages
constexpr int BWD_TILES = 2 * KV_BYTES + 2 * 2 * QT_BYTES;   // 64 KB
constexpr int BWD_SMEM = BWD_TILES + 1024 /*barriers*/ + 1024 /*alignment slack*/;
constexpr int BWD_THREADS = 256;

struct BwdParams {
  const float* lse;   // (B,H,Tq) log2 domain
  const float* delta; // (B,H,Tq) rowsum(dO o O)
  bf16* dq;
  bf16* dk;
  bf16* dv;
  int64_t lddq, lddk, lddv;
  const int32_t* kv_len;
  int B, H, Tq, Tkv;
  int causal;
  float scale, scale_log2;
};

__global__ void __launch_bounds__(BWD_THREADS, 1)
attention_bwd_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                     const __grid_constant__ CUtensorMap tmV, const __grid_constant__ CUtensorMap tmdO, const BwdParams p) {
  extern __shared__ uint8_t smem_dyn[];
  uint8_t* smem_raw = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_raw + BWD_TILES);
  uint64_t& bar_kv = bars[0];
  uint64_t* bar_q = bars + 1;   // [2]: Q and dO of a query tile landed in stage s (parity: (it / 2) & 1)

  const uint32_t sK = ptx::smem_u32(smem_raw), sV = sK + KV_BYTES;
  const uint32_t sQ0 = sV + KV_BYTES;          // stage s: Q at sQ0 + s*16K, dO right after Q
  const int kv_tile = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int kv0 = kv_tile * BKV;
  int kv_valid = p.Tkv;
  if (p.kv_len) kv_valid = min(kv_valid, max(1, p.kv_len[b]));
  const int wg = threadIdx.x >> 7;
  const int t = threadIdx.x & 127;
  const int warp = t >> 5, lane = t & 31;
  const int key_loc = wg * 64 + warp * 16 + (lane >> 2);   // keys key_loc and key_loc + 8 of the tile (fragment rows)
  const int qc = 2 * (lane & 3);                            // fragment column offset

  float dk[32], dv[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) { dk[i] = 0.f; dv[i] = 0.f; }

  const int n_q_tiles = (p.Tq + BQ - 1) / BQ;
  const int i_begin = p.causal ? kv0 / BQ : 0;                 // earlier queries cannot see these keys
  const int n_iter = (kv0 < kv_valid) ? n_q_tiles - i_begin : 0;   // fully masked key tile: zero gradients

  if (n_iter > 0) {
    if (threadIdx.x == 0) {
      ptx::tma_prefetch_desc(&tmQ); ptx::tma_prefetch_desc(&tmK); ptx::tma_prefetch_desc(&tmV); ptx::tma_prefetch_desc(&tmdO);
      ptx::mbar_init(ptx::smem_u32(&bar_kv), 1);
      ptx::mbar_init(ptx::smem_u32(&bar_q[0]), 1);
      ptx::mbar_init(ptx::smem_u32(&bar_q[1]), 1);
      ptx::fence_barrier_init();
    }
    __syncthreads();
    auto load_q = [&](int it) {   // thread 0 only
      const uint32_t full = ptx::smem_u32(&bar_q[it & 1]);
      const uint32_t dst = sQ0 + (it & 1) * 2 * QT_BYTES;
      const int qrow = b * p.Tq + (i_begin + it) * BQ;
      ptx::mbar_arrive_expect_tx(full, 2 * QT_BYTES);
      ptx::tma_load_2d(dst, &tmQ, full, h * HD, qrow);
      ptx::tma_load_2d(dst + QT_BYTES, &tmdO, full, h * HD, qrow);
    };
    if (threadIdx.x == 0) {
      ptx::mbar_arrive_expect_tx(ptx::smem_u32(&bar_kv), 2 * KV_BYTES);
      ptx::tma_load_2d(sK, &tmK, ptx::smem_u32(&bar_kv), h * HD, b * p.Tkv + kv0);
      ptx::tma_load_2d(sV, &tmV, ptx::smem_u32(&bar_kv), h * HD, b * p.Tkv + kv0);
      load_q(0);
    }
    const float c = p.scale_log2;
    const uint64_t k_desc = ptx::desc_sw128(sK + wg * 8192, 16, 1024);       // A of S^T (K-major)
    const uint64_t v_desc = ptx::desc_sw128(sV + wg * 8192, 16, 1024);       // A of dP^T (K-major)
    int key_abs[2];
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) key_abs[hh] = kv0 + key_loc + 8 * hh;   // absolute key index of the row
    ptx::mbar_wait(ptx::smem_u32(&bar_kv), 0);

    for (int it = 0; it < n_iter; ++it) {
      if (threadIdx.x == 0 && it + 1 < n_iter) load_q(it + 1);   // its stage was released by the __syncthreads of it - 1
      ptx::mbar_wait(ptx::smem_u32(&bar_q[it & 1]), (it >> 1) & 1);
      const uint32_t sQ = sQ0 + (it & 1) * 2 * QT_BYTES, sdO = sQ + QT_BYTES;
      const int q0 = (i_begin + it) * BQ;

      // lse / delta of this thread's 16 query columns (issued before the MMAs so the loads overlap them)
      float lse_c[16], dlt_c[16];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int qn = q0 + 8 * i + qc + e;
          const int64_t at = (static_cast<int64_t>(b) * p.H + h) * p.Tq + qn;
          lse_c[2 * i + e] = qn < p.Tq ? __ldg(p.lse + at) : 0.f;
          dlt_c[2 * i + e] = qn < p.Tq ? __ldg(p.delta + at) : 0.f;
        }
      }

      float s[32], dp[32];
      const uint64_t q_desc = ptx::desc_sw128(sQ, 16, 1024), do_desc = ptx::desc_sw128(sdO, 16, 1024);
      ptx::wgmma_fence();
#pragma unroll
      for (int k = 0; k < HD / 16; ++k) ptx::wgmma_m64n64k16_ss<0, 0>(s, ptx::desc_add(k_desc, 32 * k), ptx::desc_add(q_desc, 32 * k), k > 0);
#pragma unroll
      for (int k = 0; k < HD / 16; ++k) ptx::wgmma_m64n64k16_ss<0, 0>(dp, ptx::desc_add(v_desc, 32 * k), ptx::desc_add(do_desc, 32 * k), k > 0);
      ptx::wgmma_commit();
      ptx::wgmma_wait<0>();
      ptx::fence_regs(s);
      ptx::fence_regs(dp);

      // P^T, dS^T; packed to bf16 in the A-fragment order (k = queries)
      uint32_t pa[4][4], da[4][4];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          float pe[2], ds[2];
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int qn = q0 + 8 * i + qc + e;
            const int key = key_abs[hh];
            const bool vis = qn < p.Tq && key < kv_valid && (!p.causal || key <= qn);
            const int x = 4 * i + 2 * hh + e;
            pe[e] = vis ? fast_exp2(fmaf(s[x], c, -lse_c[2 * i + e])) : 0.f;
            ds[e] = pe[e] * (dp[x] - dlt_c[2 * i + e]);
          }
          pa[i >> 1][(i & 1) * 2 + hh] = pack_bf16x2(pe[0], pe[1]);
          da[i >> 1][(i & 1) * 2 + hh] = pack_bf16x2(ds[0], ds[1]);
        }
      }

      const uint64_t qB_desc = ptx::desc_sw128(sQ, 8192, 1024), doB_desc = ptx::desc_sw128(sdO, 8192, 1024);
      ptx::wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < BQ / 16; ++kk) {
        ptx::wgmma_m64n64k16_rs<1>(dv, pa[kk], ptx::desc_add(doB_desc, 2048 * kk), 1u);
        ptx::wgmma_m64n64k16_rs<1>(dk, da[kk], ptx::desc_add(qB_desc, 2048 * kk), 1u);
      }
      ptx::wgmma_commit();
      ptx::wgmma_wait<0>();
      ptx::fence_regs(dv);
      ptx::fence_regs(dk);
      __syncthreads();   // both warpgroups are done with this Q / dO stage
    }
  }

  // ---- dK (scaled), dV: key rows past Tkv are not written
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int key = kv0 + key_loc + 8 * hh;
    if (key < p.Tkv) {
      bf16* dvp = p.dv + (static_cast<int64_t>(b) * p.Tkv + key) * p.lddv + h * HD + qc;
      bf16* dkp = p.dk + (static_cast<int64_t>(b) * p.Tkv + key) * p.lddk + h * HD + qc;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        *reinterpret_cast<uint32_t*>(dvp + 8 * i) = pack_bf16x2(dv[4 * i + 2 * hh], dv[4 * i + 2 * hh + 1]);
        *reinterpret_cast<uint32_t*>(dkp + 8 * i) = pack_bf16x2(dk[4 * i + 2 * hh] * p.scale, dk[4 * i + 2 * hh + 1] * p.scale);
      }
    }
  }
}

// dQ for one (128-query tile, head, sample): two warpgroups of 64 query rows; K / V tiles of 128 keys stream through a
// two-stage TMA ring shared by both (the load of tile j+1 is in flight while tile j is computed), as in the forward.
constexpr int DQ_BQ = 128, DQ_BKV = 128;
constexpr int DQ_TILE = 128 * HD * 2;                            // 16 KB
constexpr int DQ_TILES = 2 * DQ_TILE /*Q, dO*/ + 2 * 2 * DQ_TILE /*K, V x 2 stages*/;   // 96 KB
constexpr int DQ_SMEM = DQ_TILES + 1024 /*barriers*/ + 1024 /*alignment slack*/;

__global__ void __launch_bounds__(BWD_THREADS, 1)
attention_bwd_dq_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                        const __grid_constant__ CUtensorMap tmV, const __grid_constant__ CUtensorMap tmdO, const BwdParams p) {
  extern __shared__ uint8_t smem_dyn[];
  uint8_t* smem_raw = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_raw + DQ_TILES);
  uint64_t& bar_q = bars[0];     // Q and dO landed
  uint64_t* bar_kv = bars + 1;   // [2]: K and V of key tile j landed in stage j & 1 (parity: (j / 2) & 1)

  const uint32_t sQ = ptx::smem_u32(smem_raw), sdO = sQ + DQ_TILE;
  const uint32_t sKV = sdO + DQ_TILE;   // stage s: K at sKV + s*32K, V right after K
  const int qblk = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int q_base = qblk * DQ_BQ;
  int kv_valid = p.Tkv;
  if (p.kv_len) kv_valid = min(kv_valid, max(1, p.kv_len[b]));
  const int kv_end = p.causal ? min(kv_valid, q_base + DQ_BQ) : kv_valid;
  const int n_kv = (kv_end + DQ_BKV - 1) / DQ_BKV;   // >= 1

  if (threadIdx.x == 0) {
    ptx::tma_prefetch_desc(&tmQ); ptx::tma_prefetch_desc(&tmK); ptx::tma_prefetch_desc(&tmV); ptx::tma_prefetch_desc(&tmdO);
    ptx::mbar_init(ptx::smem_u32(&bar_q), 1);
    ptx::mbar_init(ptx::smem_u32(&bar_kv[0]), 1);
    ptx::mbar_init(ptx::smem_u32(&bar_kv[1]), 1);
    ptx::fence_barrier_init();
  }
  __syncthreads();
  auto load_kv = [&](int j) {   // thread 0 only
    const uint32_t full = ptx::smem_u32(&bar_kv[j & 1]);
    const uint32_t dst = sKV + (j & 1) * 2 * DQ_TILE;
    ptx::mbar_arrive_expect_tx(full, 2 * DQ_TILE);
    ptx::tma_load_2d(dst, &tmK, full, h * HD, b * p.Tkv + j * DQ_BKV);
    ptx::tma_load_2d(dst + DQ_TILE, &tmV, full, h * HD, b * p.Tkv + j * DQ_BKV);
  };
  if (threadIdx.x == 0) {
    ptx::mbar_arrive_expect_tx(ptx::smem_u32(&bar_q), 2 * DQ_TILE);
    ptx::tma_load_2d(sQ, &tmQ, ptx::smem_u32(&bar_q), h * HD, b * p.Tq + q_base);
    ptx::tma_load_2d(sdO, &tmdO, ptx::smem_u32(&bar_q), h * HD, b * p.Tq + q_base);
    load_kv(0);
  }

  const int wg = threadIdx.x >> 7;
  const int t = threadIdx.x & 127;
  const int warp = t >> 5, lane = t & 31;
  const int r_loc = wg * 64 + warp * 16 + (lane >> 2);   // rows r_loc and r_loc + 8 of the query tile
  const int kc = 2 * (lane & 3);
  const float c = p.scale_log2;
  const uint64_t q_desc = ptx::desc_sw128(sQ + wg * 8192, 16, 1024);
  const uint64_t do_desc = ptx::desc_sw128(sdO + wg * 8192, 16, 1024);
  float lse_r[2], dlt_r[2];
  bool q_ok[2];
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int qi = q_base + r_loc + 8 * hh;
    q_ok[hh] = qi < p.Tq;
    const int64_t at = (static_cast<int64_t>(b) * p.H + h) * p.Tq + qi;
    lse_r[hh] = q_ok[hh] ? __ldg(p.lse + at) : 0.f;
    dlt_r[hh] = q_ok[hh] ? __ldg(p.delta + at) : 0.f;
  }

  float dq[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) dq[i] = 0.f;
  ptx::mbar_wait(ptx::smem_u32(&bar_q), 0);

  for (int j = 0; j < n_kv; ++j) {
    if (threadIdx.x == 0 && j + 1 < n_kv) load_kv(j + 1);   // its stage was released by the __syncthreads of j - 1
    ptx::mbar_wait(ptx::smem_u32(&bar_kv[j & 1]), (j >> 1) & 1);
    const uint32_t sK = sKV + (j & 1) * 2 * DQ_TILE, sV = sK + DQ_TILE;

    float s[64], dp[64];
    const uint64_t k_desc = ptx::desc_sw128(sK, 16, 1024), v_desc = ptx::desc_sw128(sV, 16, 1024);
    ptx::wgmma_fence();
#pragma unroll
    for (int k = 0; k < HD / 16; ++k) ptx::wgmma_m64n128k16_ss<0, 0>(s, ptx::desc_add(q_desc, 32 * k), ptx::desc_add(k_desc, 32 * k), k > 0);
#pragma unroll
    for (int k = 0; k < HD / 16; ++k) ptx::wgmma_m64n128k16_ss<0, 0>(dp, ptx::desc_add(do_desc, 32 * k), ptx::desc_add(v_desc, 32 * k), k > 0);
    ptx::wgmma_commit();
    ptx::wgmma_wait<0>();
    ptx::fence_regs(s);
    ptx::fence_regs(dp);

    // dS = P o (dP - D), P = 2^(S c - LSE) on the visible keys [0, limit); packed to bf16 in the A-fragment order (k = keys)
    const int k0 = j * DQ_BKV;
    uint32_t da[8][4];
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int qi = q_base + r_loc + 8 * hh;
      int limit = kv_valid - k0;
      if (p.causal) limit = min(limit, qi - k0 + 1);
      if (!q_ok[hh]) limit = 0;
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        float ds[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int x = 4 * i + 2 * hh + e;
          const float pe = (8 * i + kc + e < limit) ? fast_exp2(fmaf(s[x], c, -lse_r[hh])) : 0.f;
          ds[e] = pe * (dp[x] - dlt_r[hh]);
        }
        da[i >> 1][(i & 1) * 2 + hh] = pack_bf16x2(ds[0], ds[1]);
      }
    }
    const uint64_t kB_desc = ptx::desc_sw128(sK, DQ_BKV * 128, 1024);   // K as the MN-major B operand (keys are k)
    ptx::wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < DQ_BKV / 16; ++kk) ptx::wgmma_m64n64k16_rs<1>(dq, da[kk], ptx::desc_add(kB_desc, 2048 * kk), 1u);
    ptx::wgmma_commit();
    ptx::wgmma_wait<0>();
    ptx::fence_regs(dq);
    __syncthreads();   // both warpgroups are done with this stage: it may be refilled
  }

#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    if (!q_ok[hh]) continue;
    bf16* dst = p.dq + (static_cast<int64_t>(b) * p.Tq + q_base + r_loc + 8 * hh) * p.lddq + h * HD + kc;
#pragma unroll
    for (int i = 0; i < 8; ++i)
      *reinterpret_cast<uint32_t*>(dst + 8 * i) = pack_bf16x2(dq[4 * i + 2 * hh] * p.scale, dq[4 * i + 2 * hh + 1] * p.scale);
  }
}

// delta[b,h,q] = sum_d dO[b,q,h,d] * O[b,q,h,d]   (8 lanes per (row, head), 16-byte loads, 3 shuffle steps)
__global__ void attention_delta_kernel(const bf16* __restrict__ o, const bf16* __restrict__ dout, float* __restrict__ delta,
                                       int64_t ldo, int64_t lddo, int B, int H, int Tq) {
  const int64_t item = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 3;  // (row, head) pair
  const int sub = threadIdx.x & 7;
  const int64_t total = static_cast<int64_t>(B) * Tq * H;
  float s = 0.f;
  int h = 0;
  int64_t row = 0;
  if (item < total) {
    h = item % H;
    row = item / H;  // b*Tq + q
    const uint4 a = *reinterpret_cast<const uint4*>(o + row * ldo + h * HD + sub * 8);
    const uint4 g = *reinterpret_cast<const uint4*>(dout + row * lddo + h * HD + sub * 8);
    const uint32_t av[4] = {a.x, a.y, a.z, a.w}, gv[4] = {g.x, g.y, g.z, g.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 p = unpack_bf16x2(av[j]), q = unpack_bf16x2(gv[j]);
      s += p.x * q.x + p.y * q.y;
    }
  }
  s += __shfl_xor_sync(0xffffffffu, s, 1);
  s += __shfl_xor_sync(0xffffffffu, s, 2);
  s += __shfl_xor_sync(0xffffffffu, s, 4);
  if (sub == 0 && item < total) {
    const int b = row / Tq, q = row % Tq;
    delta[(static_cast<int64_t>(b) * H + h) * Tq + q] = s;
  }
}

}  // namespace
}  // namespace oasr

using namespace oasr;

extern "C" int oasr_attention_bwd(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv,
                                  const void* o, int64_t ldo, const void* dout, int64_t lddo, const float* lse,
                                  float* delta, void* dq, int64_t lddq, void* dk, int64_t lddk,
                                  void* dv, int64_t lddv, int64_t B, int64_t H, int64_t Tq, int64_t Tkv,
                                  int64_t head_dim, int causal, const int32_t* kv_len, float scale, void* stream) {
  OASR_REQUIRE(head_dim == HD, "attention_bwd: head_dim %ld unsupported", (long)head_dim);
  OASR_REQUIRE(B > 0 && H > 0 && Tq > 0 && Tkv > 0, "attention_bwd: empty problem");
  OASR_REQUIRE(((ldq | ldk | ldv | ldo | lddo | lddq | lddk | lddv) & 7) == 0, "attention_bwd: strides must be multiples of 8");
  OASR_REQUIRE((reinterpret_cast<uintptr_t>(dq) & 3) == 0 && (reinterpret_cast<uintptr_t>(dk) & 3) == 0 &&
                   (reinterpret_cast<uintptr_t>(dv) & 3) == 0,
               "attention_bwd: dQ / dK / dV must be 4-byte aligned");
  OASR_REQUIRE(!causal || Tq == Tkv, "attention_bwd: causal needs Tq == Tkv");
  OASR_REQUIRE(B <= 65535 && H <= 65535, "attention_bwd: B and H must fit the grid");
  cudaStream_t st = (cudaStream_t)stream;
  CUtensorMap tmQ, tmK, tmV, tmdO, tmQ128, tmdO128;
  int rc;
  if ((rc = make_tmap_2d(&tmQ, q, 2, (uint64_t)(H * HD), (uint64_t)(B * Tq), (uint64_t)ldq * 2, HD, BQ, true))) return rc;
  if ((rc = make_tmap_2d(&tmK, k, 2, (uint64_t)(H * HD), (uint64_t)(B * Tkv), (uint64_t)ldk * 2, HD, BKV, true))) return rc;
  if ((rc = make_tmap_2d(&tmV, v, 2, (uint64_t)(H * HD), (uint64_t)(B * Tkv), (uint64_t)ldv * 2, HD, BKV, true))) return rc;
  if ((rc = make_tmap_2d(&tmdO, dout, 2, (uint64_t)(H * HD), (uint64_t)(B * Tq), (uint64_t)lddo * 2, HD, BQ, true))) return rc;
  if ((rc = make_tmap_2d(&tmQ128, q, 2, (uint64_t)(H * HD), (uint64_t)(B * Tq), (uint64_t)ldq * 2, HD, DQ_BQ, true))) return rc;
  if ((rc = make_tmap_2d(&tmdO128, dout, 2, (uint64_t)(H * HD), (uint64_t)(B * Tq), (uint64_t)lddo * 2, HD, DQ_BQ, true))) return rc;

  const int64_t n_rows = B * Tq * H;
  attention_delta_kernel<<<(unsigned)ceil_div(n_rows * 8, 256), 256, 0, st>>>((const bf16*)o, (const bf16*)dout, delta, ldo, lddo,
                                                                              (int)B, (int)H, (int)Tq);
  OASR_LAUNCH_CHECK();

  BwdParams p;
  p.lse = lse; p.delta = delta; p.kv_len = kv_len;
  p.dq = static_cast<bf16*>(dq); p.dk = static_cast<bf16*>(dk); p.dv = static_cast<bf16*>(dv);
  p.lddq = lddq; p.lddk = lddk; p.lddv = lddv;
  p.B = (int)B; p.H = (int)H; p.Tq = (int)Tq; p.Tkv = (int)Tkv; p.causal = causal;
  p.scale = scale; p.scale_log2 = scale * 1.4426950408889634f;
  static bool attr_set = false;
  if (!attr_set) {
    OASR_CUDA_OK(cudaFuncSetAttribute(attention_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, BWD_SMEM));
    OASR_CUDA_OK(cudaFuncSetAttribute(attention_bwd_dq_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, DQ_SMEM));
    attr_set = true;
  }
  const dim3 grid((unsigned)ceil_div(Tkv, BKV), (unsigned)H, (unsigned)B);
  attention_bwd_kernel<<<grid, BWD_THREADS, BWD_SMEM, st>>>(tmQ, tmK, tmV, tmdO, p);
  OASR_LAUNCH_CHECK();
  const dim3 grid_dq((unsigned)ceil_div(Tq, DQ_BQ), (unsigned)H, (unsigned)B);
  attention_bwd_dq_kernel<<<grid_dq, BWD_THREADS, DQ_SMEM, st>>>(tmQ128, tmK, tmV, tmdO128, p);
  OASR_LAUNCH_CHECK();
  return OASR_OK;
}
