// Flash-style attention backward for head_dim 64 on wgmma (sm_90a).
//
// Autograd of F.scaled_dot_product_attention (olmoasr/model.py:331-340) for the three training uses
// (encoder self, decoder causal+length self, cross).  Given Q, K, V, O, dO and the forward's log2-domain
// LSE it produces dQ, dK, dV without ever materialising the (Tq x Tkv) score matrix in HBM.
//
// Both kernels below run two warpgroups (256 threads) and stream their operands through a three-stage TMA ring whose
// stages carry a full and an empty mbarrier: each warpgroup releases a stage by arriving on its empty barrier, and
// thread 0 refills it one step later, once both have (no CTA-wide barrier in the loop, so the two warpgroups drift
// apart and cover each other's non-MMA work).  They keep 256 threads rather than adding a producer warpgroup because
// their loops need more than the 168 registers per thread that a 384-thread launch allows (ptxas allocates the whole
// kernel under that cap; a setmaxnreg hand-over does not lift it).  Each warpgroup's loop is software-pipelined one
// step deep: the S / dP MMAs of step i + 1 are issued together with the accumulating MMAs of step i, and the exp2 / dS
// math of step i + 1 runs (in place, in fp32) while those are on the tensor cores.  Tile sizes, k16 order, masks and
// exp2 are those of an unpipelined loop, so the results are bit-for-bit the same.
//
// dK / dV: one CTA per (128-key tile, head, sample), each warpgroup owning 64 keys, looping over the 64-query
// tiles that can see the keys (Q and dO stream through a three-stage ring).  Everything is computed
// transposed, with the warpgroup's keys as the MMA rows, so that dK and dV stay in registers for the loop:
//     S^T  = K Q^T         dP^T = V dO^T                 wgmma m64n64k16, all operands from swizzled smem
//     P^T  = exp2(S^T c - LSE)   dS^T = P^T o (dP^T - D) thread-local: LSE / D are per query = per column
//     dV  += P^T dO        dK  += dS^T Q                 P^T / dS^T as register A operands, dO / Q MN-major
// dK / dV leave straight from the fragments.  dQ is a sum over every key tile; rather than letting the key-tile CTAs add
// into it with atomics (whose order, and so rounding, changes from run to run), a second kernel owns each 128-query tile,
// recomputes S and dP for it and accumulates dQ = sum_j dS_j K_j over the key tiles in order:
//     S = Q K^T   dP = dO V^T   (wgmma m64n128k16)   dS = P o (dP - D)   dQ += dS K   (dS as register A, K MN-major)
//
// Packed (varlen) batches use the row offsets of attention_fwd_sm90.cu (LSE / delta (1, H, N)).  A 64-query step of the
// dK / dV loop may then read the NEXT sample's rows, whose dO is not zero the way a padded row's is: every P^T / dS^T
// column is tested against the sample's own query count, and dQ / dK / dV stores against its own lengths.  With packed
// keys (self-attention) the dK / dV grid runs over the same (sample, 128-row tile) list as the dQ grid; with dense keys
// (cross-attention) it keeps its (key tile, head, sample) grid.
#include "common.cuh"
#include "ptx_sm90.cuh"

#include <stdlib.h>

#include <type_traits>

namespace oasr {
namespace {

constexpr int HD = 64;
constexpr int BQ = 64;                     // queries per loop iteration
constexpr int BKV = 128;                   // keys per CTA (64 per warpgroup)
constexpr int STAGES = 3;                  // both rings: step i + 1 is waited on while step i - 1's stage refills
constexpr int KV_BYTES = BKV * HD * 2;     // 16 KB
constexpr int QT_BYTES = BQ * HD * 2;      // 8 KB
// K, V | (Q, dO) per stage
constexpr int BWD_TILES = 2 * KV_BYTES + STAGES * 2 * QT_BYTES;   // 80 KB
constexpr int BWD_SMEM = BWD_TILES + 1024 /*barriers*/ + 1024 /*alignment slack*/;
constexpr int BWD_THREADS = 256;

struct BwdParams {
  const float* lse;   // (B,H,Tq) log2 domain
  const float* delta; // (B,H,Tq) rowsum(dO o O)
  void* dq;
  void* dk;
  void* dv;
  int64_t lddq, lddk, lddv;
  const int32_t* kv_len;
  const int32_t* q_off;    // (B+1,) packed query row offsets, nullable
  const int32_t* kv_off;   // (B+1,) packed key row offsets, nullable
  const int32_t* tiles;    // (sample, 128-row tile) int32 pairs of the packed grids (4-byte aligned)
  int B, H, Tq, Tkv;
  int causal;
  float scale, scale_log2;
};

template <typename T>
__global__ void __launch_bounds__(BWD_THREADS, 1)
attention_bwd_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                     const __grid_constant__ CUtensorMap tmV, const __grid_constant__ CUtensorMap tmdO, const BwdParams p) {
  extern __shared__ uint8_t smem_dyn[];
  uint8_t* smem_raw = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_raw + BWD_TILES);
  uint64_t& bar_kv = bars[0];
  uint64_t* bar_full = bars + 1;             // [STAGES]: Q and dO of query step it landed in stage it % STAGES
  uint64_t* bar_empty = bar_full + STAGES;   // [STAGES]: both warpgroups are done with the stage

  const uint32_t sK = ptx::smem_u32(smem_raw), sV = sK + KV_BYTES;
  const uint32_t sQ0 = sV + KV_BYTES;                        // stage s: Q at sQ0 + s*16K, dO right after Q
  const int h = blockIdx.y;
  int kv_tile = blockIdx.x, b = blockIdx.z;
  if (p.kv_off) { b = p.tiles[2 * blockIdx.x]; kv_tile = p.tiles[2 * blockIdx.x + 1]; }
  const int kv0 = kv_tile * BKV;
  const int q_row0 = p.q_off ? p.q_off[b] : b * p.Tq;
  const int tq = p.q_off ? p.q_off[b + 1] - q_row0 : p.Tq;     // the sample's query rows; later rows are foreign or padding
  const int kv_row0 = p.kv_off ? p.kv_off[b] : b * p.Tkv;
  const int tkv = p.kv_off ? p.kv_off[b + 1] - kv_row0 : p.Tkv;
  int kv_valid = tkv;
  if (p.kv_len) kv_valid = min(kv_valid, max(1, p.kv_len[b]));
  const int64_t lse0 = p.q_off ? static_cast<int64_t>(h) * p.Tq + q_row0 : (static_cast<int64_t>(b) * p.H + h) * p.Tq;

  const int n_q_tiles = (tq + BQ - 1) / BQ;
  const int i_begin = p.causal ? kv0 / BQ : 0;                 // earlier queries cannot see these keys
  const int n_iter = (kv0 < kv_valid) ? n_q_tiles - i_begin : 0;   // fully masked key tile: zero gradients

  if (threadIdx.x == 0) {
    ptx::tma_prefetch_desc(&tmQ); ptx::tma_prefetch_desc(&tmK); ptx::tma_prefetch_desc(&tmV); ptx::tma_prefetch_desc(&tmdO);
    ptx::mbar_init(ptx::smem_u32(&bar_kv), 1);
    for (int s = 0; s < STAGES; ++s) {
      ptx::mbar_init(ptx::smem_u32(&bar_full[s]), 1);
      ptx::mbar_init(ptx::smem_u32(&bar_empty[s]), 2);   // one arrival per consumer warpgroup
    }
    ptx::fence_barrier_init();
  }
  __syncthreads();

  // thread 0 only: Q and dO of query step it into stage it % STAGES, once both warpgroups have released it
  auto load_q = [&](int it) {
    const int st = it % STAGES;
    ptx::mbar_wait(ptx::smem_u32(&bar_empty[st]), ((it / STAGES) & 1) ^ 1);
    const uint32_t full = ptx::smem_u32(&bar_full[st]);
    const uint32_t dst = sQ0 + st * 2 * QT_BYTES;
    const int q0 = (i_begin + it) * BQ;
    ptx::mbar_arrive_expect_tx(full, 2 * QT_BYTES);
    ptx::tma_load_2d(dst, &tmQ, full, h * HD, q_row0 + q0);
    ptx::tma_load_2d(dst + QT_BYTES, &tmdO, full, h * HD, q_row0 + q0);
  };
  if (threadIdx.x == 0 && n_iter > 0) {
    ptx::mbar_arrive_expect_tx(ptx::smem_u32(&bar_kv), 2 * KV_BYTES);
    ptx::tma_load_2d(sK, &tmK, ptx::smem_u32(&bar_kv), h * HD, kv_row0 + kv0);
    ptx::tma_load_2d(sV, &tmV, ptx::smem_u32(&bar_kv), h * HD, kv_row0 + kv0);
    for (int it = 0; it < min(STAGES, n_iter); ++it) load_q(it);
  }

  const int wg = threadIdx.x >> 7;   // key half of the tile
  const int t = threadIdx.x & 127;
  const int warp = t >> 5, lane = t & 31;
  const int key_loc = wg * 64 + warp * 16 + (lane >> 2);   // keys key_loc and key_loc + 8 of the tile (fragment rows)
  const int qc = 2 * (lane & 3);                            // fragment column offset

  float dk[32], dv[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) { dk[i] = 0.f; dv[i] = 0.f; }

  if (n_iter > 0) {
    const float c = p.scale_log2;
    const uint64_t k_desc = ptx::desc_sw128(sK + wg * 8192, 16, 1024);       // A of S^T (K-major)
    const uint64_t v_desc = ptx::desc_sw128(sV + wg * 8192, 16, 1024);       // A of dP^T (K-major)
    int key_abs[2];
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) key_abs[hh] = kv0 + key_loc + 8 * hh;   // absolute key index of the row
    ptx::mbar_wait(ptx::smem_u32(&bar_kv), 0);

    float s[32], dp[32];
    // S^T, dP^T of query step it into s, dp (one commit group)
    auto issue_sdp = [&](int it) {
      const int st = it % STAGES;
      ptx::mbar_wait(ptx::smem_u32(&bar_full[st]), (it / STAGES) & 1);
      const uint32_t sQ = sQ0 + st * 2 * QT_BYTES, sdO = sQ + QT_BYTES;
      const uint64_t q_desc = ptx::desc_sw128(sQ, 16, 1024), do_desc = ptx::desc_sw128(sdO, 16, 1024);
      ptx::wgmma_fence();
#pragma unroll
      for (int k = 0; k < HD / 16; ++k) ptx::wgmma_m64n64k16_ss<0, 0, T>(s, ptx::desc_add(k_desc, 32 * k), ptx::desc_add(q_desc, 32 * k), k > 0);
#pragma unroll
      for (int k = 0; k < HD / 16; ++k) ptx::wgmma_m64n64k16_ss<0, 0, T>(dp, ptx::desc_add(v_desc, 32 * k), ptx::desc_add(do_desc, 32 * k), k > 0);
      ptx::wgmma_commit();
    };
    // s <- P^T, dp <- dS^T of query step it
    auto grads = [&](int it) {
      const int q0 = (i_begin + it) * BQ;
      // every (key, query) pair of this thread visible: no per-element test (the common case away from the edges)
      const bool all_vis = q0 + BQ <= tq && key_abs[1] < kv_valid && (!p.causal || key_abs[1] <= q0);
      auto run = [&](auto masked) {
        // lse / delta of this thread's 16 query columns
        float lse_c[16], dlt_c[16];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int qn = q0 + 8 * i + qc + e;
            const int64_t at = lse0 + qn;
            lse_c[2 * i + e] = (!masked || qn < tq) ? __ldg(p.lse + at) : 0.f;
            dlt_c[2 * i + e] = (!masked || qn < tq) ? __ldg(p.delta + at) : 0.f;
          }
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) {
#pragma unroll
          for (int hh = 0; hh < 2; ++hh) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int qn = q0 + 8 * i + qc + e;
              const int key = key_abs[hh];
              const bool vis = !masked || (qn < tq && key < kv_valid && (!p.causal || key <= qn));
              const int x = 4 * i + 2 * hh + e;
              const float pe = vis ? fast_exp2(fmaf(s[x], c, -lse_c[2 * i + e])) : 0.f;
              dp[x] = pe * (dp[x] - dlt_c[2 * i + e]);
              s[x] = pe;
            }
          }
        }
      };
      if (all_vis) run(std::false_type{});
      else run(std::true_type{});
    };
    // P^T, dS^T packed to T in the A-fragment order (k = queries)
    uint32_t pa[4][4], da[4][4];
    auto pack = [&]() {
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          const int x = 4 * i + 2 * hh;
          pa[i >> 1][(i & 1) * 2 + hh] = Act16<T>::pack2(s[x], s[x + 1]);
          da[i >> 1][(i & 1) * 2 + hh] = Act16<T>::pack2(dp[x], dp[x + 1]);
        }
    };
    // dV += P^T dO, dK += dS^T Q of query step it (one commit group)
    auto issue_dkdv = [&](int it) {
      const uint32_t sQ = sQ0 + (it % STAGES) * 2 * QT_BYTES, sdO = sQ + QT_BYTES;
      const uint64_t qB_desc = ptx::desc_sw128(sQ, 8192, 1024), doB_desc = ptx::desc_sw128(sdO, 8192, 1024);
      ptx::wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < BQ / 16; ++kk) {
        ptx::wgmma_m64n64k16_rs<1, T>(dv, pa[kk], ptx::desc_add(doB_desc, 2048 * kk), 1u);
        ptx::wgmma_m64n64k16_rs<1, T>(dk, da[kk], ptx::desc_add(qB_desc, 2048 * kk), 1u);
      }
      ptx::wgmma_commit();
    };
    auto retire_dkdv = [&](int it) {
      ptx::wgmma_wait<0>();
      ptx::fence_regs(dv);
      ptx::fence_regs(dk);
      if (t == 0) ptx::mbar_arrive(ptx::smem_u32(&bar_empty[it % STAGES]));   // this Q / dO stage is free
    };

    issue_sdp(0);
    ptx::wgmma_wait<0>();
    ptx::fence_regs(s);
    ptx::fence_regs(dp);
    grads(0);
    pack();
    for (int it = 0; it + 1 < n_iter; ++it) {
      issue_sdp(it + 1);
      issue_dkdv(it);
      if (threadIdx.x == 0 && it >= 1 && it - 1 + STAGES < n_iter) load_q(it - 1 + STAGES);   // released in step it - 1
      ptx::wgmma_wait<1>();   // S^T / dP^T of it + 1 are in; the dK / dV MMAs of it may still be running
      ptx::fence_regs(s);
      ptx::fence_regs(dp);
      grads(it + 1);
      retire_dkdv(it);
      pack();
    }
    issue_dkdv(n_iter - 1);
    retire_dkdv(n_iter - 1);
  }

  // ---- dK (scaled), dV: key rows past the sample's keys are not written
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int key = kv0 + key_loc + 8 * hh;
    if (key < tkv) {
      T* dvp = static_cast<T*>(p.dv) + (static_cast<int64_t>(kv_row0) + key) * p.lddv + h * HD + qc;
      T* dkp = static_cast<T*>(p.dk) + (static_cast<int64_t>(kv_row0) + key) * p.lddk + h * HD + qc;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        *reinterpret_cast<uint32_t*>(dvp + 8 * i) = Act16<T>::pack2(dv[4 * i + 2 * hh], dv[4 * i + 2 * hh + 1]);
        *reinterpret_cast<uint32_t*>(dkp + 8 * i) = Act16<T>::pack2(dk[4 * i + 2 * hh] * p.scale, dk[4 * i + 2 * hh + 1] * p.scale);
      }
    }
  }
}

// dQ for one (128-query tile, head, sample): each warpgroup owns 64 query rows; K / V tiles of 128 keys stream
// through a three-stage ring as in the forward.
constexpr int DQ_BQ = 128, DQ_BKV = 128;
constexpr int DQ_TILE = 128 * HD * 2;                                      // 16 KB
constexpr int DQ_TILES = 2 * DQ_TILE /*Q, dO*/ + STAGES * 2 * DQ_TILE /*K, V per stage*/;   // 128 KB
constexpr int DQ_SMEM = DQ_TILES + 1024 /*barriers*/ + 1024 /*alignment slack*/;

template <typename T>
__global__ void __launch_bounds__(BWD_THREADS, 1)
attention_bwd_dq_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                        const __grid_constant__ CUtensorMap tmV, const __grid_constant__ CUtensorMap tmdO, const BwdParams p) {
  extern __shared__ uint8_t smem_dyn[];
  uint8_t* smem_raw = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_raw + DQ_TILES);
  uint64_t& bar_q = bars[0];                 // Q and dO landed
  uint64_t* bar_full = bars + 1;             // [STAGES]: K and V of key tile j landed in stage j % STAGES
  uint64_t* bar_empty = bar_full + STAGES;   // [STAGES]: both warpgroups are done with the stage

  const uint32_t sQ = ptx::smem_u32(smem_raw), sdO = sQ + DQ_TILE;
  const uint32_t sKV = sdO + DQ_TILE;   // stage s: K at sKV + s*32K, V right after K
  const int h = blockIdx.y;
  int qblk = blockIdx.x, b = blockIdx.z;
  if (p.q_off) { b = p.tiles[2 * blockIdx.x]; qblk = p.tiles[2 * blockIdx.x + 1]; }
  const int q_base = qblk * DQ_BQ;
  const int q_row0 = p.q_off ? p.q_off[b] : b * p.Tq;
  const int tq = p.q_off ? p.q_off[b + 1] - q_row0 : p.Tq;
  const int kv_row0 = p.kv_off ? p.kv_off[b] : b * p.Tkv;
  int kv_valid = p.kv_off ? p.kv_off[b + 1] - kv_row0 : p.Tkv;
  if (p.kv_len) kv_valid = min(kv_valid, max(1, p.kv_len[b]));
  const int kv_end = p.causal ? min(kv_valid, q_base + DQ_BQ) : kv_valid;
  const int n_kv = (kv_end + DQ_BKV - 1) / DQ_BKV;   // >= 1

  if (threadIdx.x == 0) {
    ptx::tma_prefetch_desc(&tmQ); ptx::tma_prefetch_desc(&tmK); ptx::tma_prefetch_desc(&tmV); ptx::tma_prefetch_desc(&tmdO);
    ptx::mbar_init(ptx::smem_u32(&bar_q), 1);
    for (int s = 0; s < STAGES; ++s) {
      ptx::mbar_init(ptx::smem_u32(&bar_full[s]), 1);
      ptx::mbar_init(ptx::smem_u32(&bar_empty[s]), 2);   // one arrival per consumer warpgroup
    }
    ptx::fence_barrier_init();
  }
  __syncthreads();

  // thread 0 only: K and V of key tile j into stage j % STAGES, once both warpgroups have released it
  auto load_kv = [&](int j) {
    const int st = j % STAGES;
    ptx::mbar_wait(ptx::smem_u32(&bar_empty[st]), ((j / STAGES) & 1) ^ 1);
    const uint32_t full = ptx::smem_u32(&bar_full[st]);
    const uint32_t dst = sKV + st * 2 * DQ_TILE;
    ptx::mbar_arrive_expect_tx(full, 2 * DQ_TILE);
    ptx::tma_load_2d(dst, &tmK, full, h * HD, kv_row0 + j * DQ_BKV);
    ptx::tma_load_2d(dst + DQ_TILE, &tmV, full, h * HD, kv_row0 + j * DQ_BKV);
  };
  if (threadIdx.x == 0) {
    ptx::mbar_arrive_expect_tx(ptx::smem_u32(&bar_q), 2 * DQ_TILE);
    ptx::tma_load_2d(sQ, &tmQ, ptx::smem_u32(&bar_q), h * HD, q_row0 + q_base);
    ptx::tma_load_2d(sdO, &tmdO, ptx::smem_u32(&bar_q), h * HD, q_row0 + q_base);
    for (int j = 0; j < min(STAGES, n_kv); ++j) load_kv(j);
  }

  const int wg = threadIdx.x >> 7;   // query-row half of the tile
  const int t = threadIdx.x & 127;
  const int warp = t >> 5, lane = t & 31;
  const int r_loc = wg * 64 + warp * 16 + (lane >> 2);   // rows r_loc and r_loc + 8 of the query tile
  const int kc = 2 * (lane & 3);
  const float c = p.scale_log2;
  const uint64_t q_desc = ptx::desc_sw128(sQ + wg * 8192, 16, 1024);
  const uint64_t do_desc = ptx::desc_sw128(sdO + wg * 8192, 16, 1024);
  float lse_r[2], dlt_r[2];
  bool q_ok[2];
  const int64_t lse0 = p.q_off ? static_cast<int64_t>(h) * p.Tq + q_row0 : (static_cast<int64_t>(b) * p.H + h) * p.Tq;
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int qi = q_base + r_loc + 8 * hh;
    q_ok[hh] = qi < tq;
    const int64_t at = lse0 + qi;
    lse_r[hh] = q_ok[hh] ? __ldg(p.lse + at) : 0.f;
    dlt_r[hh] = q_ok[hh] ? __ldg(p.delta + at) : 0.f;
  }

  float dq[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) dq[i] = 0.f;
  float s[64], dp[64];
  // S = Q K_j^T, dP = dO V_j^T into s, dp (one commit group)
  auto issue_sdp = [&](int j) {
    const int st = j % STAGES;
    ptx::mbar_wait(ptx::smem_u32(&bar_full[st]), (j / STAGES) & 1);
    const uint32_t sK = sKV + st * 2 * DQ_TILE, sV = sK + DQ_TILE;
    const uint64_t k_desc = ptx::desc_sw128(sK, 16, 1024), v_desc = ptx::desc_sw128(sV, 16, 1024);
    ptx::wgmma_fence();
#pragma unroll
    for (int k = 0; k < HD / 16; ++k) ptx::wgmma_m64n128k16_ss<0, 0, T>(s, ptx::desc_add(q_desc, 32 * k), ptx::desc_add(k_desc, 32 * k), k > 0);
#pragma unroll
    for (int k = 0; k < HD / 16; ++k) ptx::wgmma_m64n128k16_ss<0, 0, T>(dp, ptx::desc_add(do_desc, 32 * k), ptx::desc_add(v_desc, 32 * k), k > 0);
    ptx::wgmma_commit();
  };
  // dp <- dS = P o (dP - D), P = 2^(S c - LSE) on the visible keys [0, limit) of key tile j
  auto grads = [&](int j) {
    const int k0 = j * DQ_BKV;
    int limit[2];
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int qi = q_base + r_loc + 8 * hh;
      limit[hh] = kv_valid - k0;
      if (p.causal) limit[hh] = min(limit[hh], qi - k0 + 1);
      if (!q_ok[hh]) limit[hh] = 0;
    }
    // every key of the tile visible to both of this thread's rows: no per-element test
    auto run = [&](auto masked) {
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
#pragma unroll
        for (int i = 0; i < 16; ++i) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int x = 4 * i + 2 * hh + e;
            const float pe = (!masked || 8 * i + kc + e < limit[hh]) ? fast_exp2(fmaf(s[x], c, -lse_r[hh])) : 0.f;
            dp[x] = pe * (dp[x] - dlt_r[hh]);
          }
        }
      }
    };
    if (min(limit[0], limit[1]) >= DQ_BKV) run(std::false_type{});
    else run(std::true_type{});
  };
  // dS packed to T in the A-fragment order (k = keys)
  uint32_t da[8][4];
  auto pack = [&]() {
#pragma unroll
    for (int i = 0; i < 16; ++i)
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) da[i >> 1][(i & 1) * 2 + hh] = Act16<T>::pack2(dp[4 * i + 2 * hh], dp[4 * i + 2 * hh + 1]);
  };
  // dQ += dS K_j (one commit group); K as the MN-major B operand (keys are k)
  auto issue_dq = [&](int j) {
    const uint64_t kB_desc = ptx::desc_sw128(sKV + (j % STAGES) * 2 * DQ_TILE, DQ_BKV * 128, 1024);
    ptx::wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < DQ_BKV / 16; ++kk) ptx::wgmma_m64n64k16_rs<1, T>(dq, da[kk], ptx::desc_add(kB_desc, 2048 * kk), 1u);
    ptx::wgmma_commit();
  };
  auto retire_dq = [&](int j) {
    ptx::wgmma_wait<0>();
    ptx::fence_regs(dq);
    if (t == 0) ptx::mbar_arrive(ptx::smem_u32(&bar_empty[j % STAGES]));   // K_j and V_j are no longer read
  };

  ptx::mbar_wait(ptx::smem_u32(&bar_q), 0);
  issue_sdp(0);
  ptx::wgmma_wait<0>();
  ptx::fence_regs(s);
  ptx::fence_regs(dp);
  grads(0);
  pack();
  for (int j = 0; j + 1 < n_kv; ++j) {
    issue_sdp(j + 1);
    issue_dq(j);
    if (threadIdx.x == 0 && j >= 1 && j - 1 + STAGES < n_kv) load_kv(j - 1 + STAGES);   // released in step j - 1
    ptx::wgmma_wait<1>();   // S / dP of tile j + 1 are in; dQ += dS_j K_j may still be running
    ptx::fence_regs(s);
    ptx::fence_regs(dp);
    grads(j + 1);
    retire_dq(j);
    pack();
  }
  issue_dq(n_kv - 1);
  retire_dq(n_kv - 1);

#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    if (!q_ok[hh]) continue;
    T* dst = static_cast<T*>(p.dq) + (static_cast<int64_t>(q_row0) + q_base + r_loc + 8 * hh) * p.lddq + h * HD + kc;
#pragma unroll
    for (int i = 0; i < 8; ++i)
      *reinterpret_cast<uint32_t*>(dst + 8 * i) = Act16<T>::pack2(dq[4 * i + 2 * hh] * p.scale, dq[4 * i + 2 * hh + 1] * p.scale);
  }
}

// delta[b,h,q] = sum_d dO[b,q,h,d] * O[b,q,h,d]   (8 lanes per (row, head), 16-byte loads, 3 shuffle steps)
template <typename T>
__global__ void attention_delta_kernel(const T* __restrict__ o, const T* __restrict__ dout, float* __restrict__ delta,
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
      const float2 p = Act16<T>::unpack2(av[j]), q = Act16<T>::unpack2(gv[j]);
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

// Shapes as attention_fwd (attention_fwd_sm90.cu), packed batches included.
template <typename T>
int attention_bwd(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, const void* o,
                  int64_t ldo, const void* dout, int64_t lddo, const float* lse, float* delta, void* dq, int64_t lddq,
                  void* dk, int64_t lddk, void* dv, int64_t lddv, int64_t B, int64_t H, int64_t Tq, int64_t Tkv,
                  int64_t head_dim, int causal, const int32_t* kv_len, float scale, void* stream,
                  const int32_t* q_off = nullptr, const int32_t* kv_off = nullptr, const int32_t* tiles = nullptr,
                  int64_t n_tiles = 0) {
  OASR_REQUIRE(head_dim == HD, "attention_bwd: head_dim %ld unsupported", (long)head_dim);
  OASR_REQUIRE(B > 0 && H > 0 && Tq > 0 && Tkv > 0, "attention_bwd: empty problem");
  OASR_REQUIRE(((ldq | ldk | ldv | ldo | lddo | lddq | lddk | lddv) & 7) == 0, "attention_bwd: strides must be multiples of 8");
  OASR_REQUIRE((reinterpret_cast<uintptr_t>(dq) & 3) == 0 && (reinterpret_cast<uintptr_t>(dk) & 3) == 0 &&
                   (reinterpret_cast<uintptr_t>(dv) & 3) == 0,
               "attention_bwd: dQ / dK / dV must be 4-byte aligned");
  // attention_delta_kernel reads O with 16-byte loads; dO is checked by its TMA descriptor
  OASR_REQUIRE((reinterpret_cast<uintptr_t>(o) & 15) == 0, "attention_bwd: O must be 16-byte aligned");
  OASR_REQUIRE(!causal || Tq == Tkv, "attention_bwd: causal needs Tq == Tkv");
  OASR_REQUIRE(B <= 65535 && H <= 65535, "attention_bwd: B and H must fit the grid");
  OASR_REQUIRE(!q_off || (tiles && n_tiles > 0 && n_tiles <= 0x7fffffff), "attention_bwd: a packed batch needs its tile list");
  OASR_REQUIRE(!kv_off || q_off, "attention_bwd: packed keys need packed queries");
  OASR_REQUIRE(!causal || !q_off || kv_off == q_off, "attention_bwd: packed causal attention reads keys packed like the queries");
  cudaStream_t st = (cudaStream_t)stream;
  const uint64_t q_rows = q_off ? Tq : B * Tq, kv_rows = kv_off ? Tkv : B * Tkv;
  CUtensorMap tmQ, tmK, tmV, tmdO, tmQ128, tmdO128;
  constexpr bool f16 = Act16<T>::is_fp16;
  int rc;
  if ((rc = make_tmap_2d(&tmQ, q, 2, (uint64_t)(H * HD), q_rows, (uint64_t)ldq * 2, HD, BQ, true, f16))) return rc;
  if ((rc = make_tmap_2d(&tmK, k, 2, (uint64_t)(H * HD), kv_rows, (uint64_t)ldk * 2, HD, BKV, true, f16))) return rc;
  if ((rc = make_tmap_2d(&tmV, v, 2, (uint64_t)(H * HD), kv_rows, (uint64_t)ldv * 2, HD, BKV, true, f16))) return rc;
  if ((rc = make_tmap_2d(&tmdO, dout, 2, (uint64_t)(H * HD), q_rows, (uint64_t)lddo * 2, HD, BQ, true, f16))) return rc;
  if ((rc = make_tmap_2d(&tmQ128, q, 2, (uint64_t)(H * HD), q_rows, (uint64_t)ldq * 2, HD, DQ_BQ, true, f16))) return rc;
  if ((rc = make_tmap_2d(&tmdO128, dout, 2, (uint64_t)(H * HD), q_rows, (uint64_t)lddo * 2, HD, DQ_BQ, true, f16))) return rc;

  // delta over every query row; a packed batch is one "sample" of N rows, which gives its (1, H, N) layout
  const int64_t n_rows = (int64_t)q_rows * H;
  attention_delta_kernel<T><<<(unsigned)ceil_div(n_rows * 8, 256), 256, 0, st>>>((const T*)o, (const T*)dout, delta, ldo, lddo,
                                                                              q_off ? 1 : (int)B, (int)H, (int)Tq);
  OASR_LAUNCH_CHECK();

  BwdParams p;
  p.lse = lse; p.delta = delta; p.kv_len = kv_len;
  p.q_off = q_off; p.kv_off = kv_off; p.tiles = q_off ? tiles : nullptr;
  p.dq = dq; p.dk = dk; p.dv = dv;
  p.lddq = lddq; p.lddk = lddk; p.lddv = lddv;
  p.B = (int)B; p.H = (int)H; p.Tq = (int)Tq; p.Tkv = (int)Tkv; p.causal = causal;
  p.scale = scale; p.scale_log2 = scale * 1.4426950408889634f;
  static bool attr_set = false;
  if (!attr_set) {
    OASR_CUDA_OK(cudaFuncSetAttribute(attention_bwd_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, BWD_SMEM));
    OASR_CUDA_OK(cudaFuncSetAttribute(attention_bwd_dq_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, DQ_SMEM));
    attr_set = true;
  }
  // packed keys share the query tiles' list (BKV == DQ_BQ == 128 rows); dense keys: every key tile of every sample
  static_assert(BKV == DQ_BQ, "packed self-attention runs dK / dV and dQ over one tile list");
  const dim3 grid = kv_off ? dim3((unsigned)n_tiles, (unsigned)H, 1u) : dim3((unsigned)ceil_div(Tkv, BKV), (unsigned)H, (unsigned)B);
  attention_bwd_kernel<T><<<grid, BWD_THREADS, BWD_SMEM, st>>>(tmQ, tmK, tmV, tmdO, p);
  OASR_LAUNCH_CHECK();
  const dim3 grid_dq = q_off ? dim3((unsigned)n_tiles, (unsigned)H, 1u)
                             : dim3((unsigned)ceil_div(Tq, DQ_BQ), (unsigned)H, (unsigned)B);
  attention_bwd_dq_kernel<T><<<grid_dq, BWD_THREADS, DQ_SMEM, st>>>(tmQ128, tmK, tmV, tmdO128, p);
  OASR_LAUNCH_CHECK();
  return OASR_OK;
}

}  // namespace
}  // namespace oasr

using namespace oasr;

extern "C" int oasr_attention_bwd(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv,
                                  const void* o, int64_t ldo, const void* dout, int64_t lddo, const float* lse,
                                  float* delta, void* dq, int64_t lddq, void* dk, int64_t lddk,
                                  void* dv, int64_t lddv, int64_t B, int64_t H, int64_t Tq, int64_t Tkv,
                                  int64_t head_dim, int causal, const int32_t* kv_len, float scale, void* stream) {
  return attention_bwd<bf16>(q, ldq, k, ldk, v, ldv, o, ldo, dout, lddo, lse, delta, dq, lddq, dk, lddk, dv, lddv, B, H, Tq,
                             Tkv, head_dim, causal, kv_len, scale, stream);
}

extern "C" int oasr_attention_bwd16(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv,
                                    const void* o, int64_t ldo, const void* dout, int64_t lddo, const float* lse,
                                    float* delta, void* dq, int64_t lddq, void* dk, int64_t lddk,
                                    void* dv, int64_t lddv, int64_t B, int64_t H, int64_t Tq, int64_t Tkv,
                                    int64_t head_dim, int causal, const int32_t* kv_len, float scale, int dtype, void* stream) {
  return OASR_BY_DTYPE16(dtype, attention_bwd, q, ldq, k, ldk, v, ldv, o, ldo, dout, lddo, lse, delta, dq, lddq, dk, lddk, dv,
                         lddv, B, H, Tq, Tkv, head_dim, causal, kv_len, scale, stream);
}

extern "C" int oasr_attention_bwd_varlen16(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v,
                                           int64_t ldv, const void* o, int64_t ldo, const void* dout, int64_t lddo,
                                           const float* lse, float* delta, void* dq, int64_t lddq, void* dk, int64_t lddk,
                                           void* dv, int64_t lddv, int64_t B, int64_t H, int64_t N, int64_t Tkv,
                                           int64_t head_dim, const int32_t* cu_seqlens, const int32_t* kv_cu_seqlens,
                                           const int32_t* tiles, int64_t n_tiles, float scale, int dtype, void* stream) {
  OASR_REQUIRE(cu_seqlens, "attention_bwd_varlen: cu_seqlens is required");
  const int causal = kv_cu_seqlens != nullptr;
  return OASR_BY_DTYPE16(dtype, attention_bwd, q, ldq, k, ldk, v, ldv, o, ldo, dout, lddo, lse, delta, dq, lddq, dk, lddk, dv,
                         lddv, B, H, N, causal ? N : Tkv, head_dim, causal, nullptr, scale, stream, cu_seqlens, kv_cu_seqlens,
                         tiles, n_tiles);
}
