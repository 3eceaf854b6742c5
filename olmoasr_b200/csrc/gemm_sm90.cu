// Persistent, warp-specialised bf16 GEMM for sm_90a: TMA -> 128B-swizzled smem ring -> wgmma (fp32 accumulators in
// registers) -> fused epilogue, staged through shared memory and stored by TMA for the 16-bit outputs.
//
//   D[M,N] = epi( sum_k A[m,k] B[n,k] )
//
// One CTA per SM (at most gemm_sm_budget() CTAs), walking over 128 x BN output tiles with stride gridDim.x.  384 threads:
//   warpgroup 0    producers, which give their registers up (setmaxnreg 40) ...
//                  warp 0: one thread streams A / B through the ring (the ring keeps running across tiles, so the next
//                  tile's operands arrive while this tile's epilogue runs);
//                  warp 1: the 16-bit epilogues' bias slice and aux tile (residual, GELU pre-activation), loaded into
//                  shared memory during the tile's mainloop
//   warpgroups 1-2 ... to the consumers (setmaxnreg 232): warpgroup c owns rows 64c .. 64c+63 of the tile, issues its
//                  m64 x BN x 16 wgmmas and runs the epilogue for those rows
// Tile = 128 x BN (BN = 64, 128 or 256; 256 keeps 128 fp32 accumulators per consumer thread), BK = 64 bf16 (= one
// 128-byte swizzle row).  Both operand majors are supported through the wgmma descriptors and transpose bits, so dgrad
// (B MN-major) and wgrad (A and B MN-major) need no transposes in HBM.  The epilogue is a template parameter: each
// kernel carries only its own store code.  Reference ops replaced: olmoasr/model.py:97-101 (Linear.forward) and its
// autograd, model.py:768-770 (tied logits), model.py:592-593 (Conv1d after im2col).
#include "common.cuh"
#include "ptx_sm90.cuh"

#include <stdio.h>
#include <stdlib.h>
#include <string.h>

namespace oasr {
namespace {

constexpr int BM = 128;
// FP8 accumulation: the library promotes every k-block (see gemm_body).  An A/B build with -DOASR_FP8_NO_PROMOTE
// (python -m olmoasr_b200.build --variant ... -DOASR_FP8_NO_PROMOTE) chains all k-blocks in the MMA accumulator instead,
// which is how far tools/fp8_accumulation_error.py measures the unpromoted sum from fp64; it is not a shipped form.
#ifdef OASR_FP8_NO_PROMOTE
constexpr bool FP8_PROMOTE = false;
#else
constexpr bool FP8_PROMOTE = true;
#endif
constexpr int BK = 64;               // 64 bf16 = 128 B = swizzle span
constexpr int A_STAGE_BYTES = BM * BK * 2;  // 16 KB
constexpr int THREADS = 384;
constexpr int PRODUCER_REGS = 40;    // 40 * 128 + 232 * 256 <= 64 K registers of the SM
constexpr int CONSUMER_REGS = 232;
// The 16-bit epilogues stage their results in boxes of 64 rows x 64 columns (8 KB, one consumer warpgroup's rows),
// 128-byte swizzled like the TMA boxes they are loaded and stored as: 16-byte chunk j of row r sits at
// r * 128 + (j ^ (r % 8)) * 16.
constexpr int BOX = 64;
constexpr int BOX_BYTES = BOX * BOX * 2;

struct GemmParams {
  void* C;
  void* C2;
  const float* bias;
  const void* aux;
  int64_t ldc;
  int64_t ldaux;
  int M, N, K;
  int tiles_m, tiles_n, splits;
  int num_tiles;   // tiles_m * tiles_n * splits (a parameter, so the tile loops need no register for it)
  int kblocks_total, kblocks_per_split;
  int raster_m;  // 1: consecutive tiles walk M first (B tile stays hot in L2) -- used when B is the larger operand
  int64_t split_stride;   // split-K: split s stores its fp32 partial at C + s * split_stride (0: one split)
  // 16-bit epilogues: C (and C2) / aux move by TMA (16-byte aligned base and row stride), else by plain bounded copies
  int tma_out, tma_aux;
  const float* sa;   // FP8 kernels: the per-row scales of A (M) and of B (N), applied to acc before the epilogue
  const float* sb;
};

constexpr bool is_f32_epi(int epi) { return epi == OASR_EPI_F32 || epi == OASR_EPI_F32_ATOMIC_ADD; }
constexpr bool reads_aux(int epi) { return epi == OASR_EPI_BF16_RESIDUAL || epi == OASR_EPI_BF16_GELU_BWD; }

template <int BN, int EPI, bool SCALED = false>
struct Cfg {
  static constexpr int B_STAGE_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;
  // Epilogue buffer after the ring: the aux epilogues hold the whole 128 x BN aux tile (each result is written over its
  // own aux and stored from there); BF16 and GELU cycle two output boxes per consumer warpgroup.  Then BN fp32 of bias.
  static constexpr int EPI_BYTES = is_f32_epi(EPI) ? 0 : (reads_aux(EPI) ? BM * BN * 2 : 2 * 2 * BOX_BYTES);
  static constexpr int BIAS_BYTES = is_f32_epi(EPI) ? 0 : BN * 4;
  static constexpr int SCALE_BYTES = SCALED ? BN * 4 : 0;   // FP8: B's row scales of the tile, after the bias
  static constexpr int BUDGET = 232448 - 1024 - EPI_BYTES - BIAS_BYTES - SCALE_BYTES;   // 227 KB per block, minus the barrier area
  static constexpr int STAGES = (BUDGET / STAGE_BYTES) > 8 ? 8 : (BUDGET / STAGE_BYTES);
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + EPI_BYTES + BIAS_BYTES + SCALE_BYTES + 1024;   // 1024-aligned base, barriers last
  static_assert(STAGES >= 3, "gemm: shared-memory ring too shallow");
};

// tile index -> (m block, n block, k split).  Default order walks N fastest: the CTAs running together share A row
// panels and keep the (small) weight matrix in L2; raster_m walks M fastest for wide outputs (tied logits).
__device__ __forceinline__ void decode_tile(int tile, const GemmParams& p, int& m_blk, int& n_blk, int& split) {
  if (p.raster_m) {
    m_blk = tile % p.tiles_m;
    n_blk = (tile / p.tiles_m) % p.tiles_n;
  } else {
    n_blk = tile % p.tiles_n;
    m_blk = (tile / p.tiles_n) % p.tiles_m;
  }
  split = tile / (p.tiles_n * p.tiles_m);
}

// Plain copies of one box between global (rows row0.., columns col0.., bounded by M and N; zeros past them on the way
// in) and its swizzled shared-memory image, 8 columns per step: the path for tensors TMA cannot address.
template <typename T>
__device__ __forceinline__ void box_from_global(uint8_t* box, const void* src, int64_t ld, int row0, int col0, const GemmParams& p,
                                                int tid, int nthreads) {
  for (int k = tid; k < BOX * BOX / 8; k += nthreads) {
    const int r = k >> 3, j = k & 7, row = row0 + r, col = col0 + 8 * j;
    uint16_t v[8];
    const uint16_t* s = reinterpret_cast<const uint16_t*>(src) + static_cast<int64_t>(row) * ld + col;
#pragma unroll
    for (int e = 0; e < 8; ++e) v[e] = (row < p.M && col + e < p.N) ? s[e] : uint16_t(0);
    *reinterpret_cast<uint4*>(box + r * 128 + ((j ^ (r & 7)) << 4)) =
        make_uint4(v[0] | (uint32_t(v[1]) << 16), v[2] | (uint32_t(v[3]) << 16), v[4] | (uint32_t(v[5]) << 16),
                   v[6] | (uint32_t(v[7]) << 16));
  }
}
template <typename T>
__device__ __forceinline__ void box_to_global(const uint8_t* box, void* dst, int64_t ld, int row0, int col0, const GemmParams& p,
                                              int tid) {
  for (int k = tid; k < BOX * BOX / 8; k += 128) {
    const int r = k >> 3, j = k & 7, row = row0 + r, col = col0 + 8 * j;
    if (row >= p.M || col >= p.N) continue;
    const uint16_t* s = reinterpret_cast<const uint16_t*>(box + r * 128 + ((j ^ (r & 7)) << 4));
    uint16_t* d = reinterpret_cast<uint16_t*>(dst) + static_cast<int64_t>(row) * ld + col;
#pragma unroll
    for (int e = 0; e < 8; ++e)
      if (col + e < p.N) d[e] = s[e];
  }
}

// The kernel body.  LR (a compile-time switch; the plain kernels pass false and null tail maps) adds the low-rank tail
// A2 B2^T: after a tile's k-blocks the operand producer streams kb_tail more k-blocks from tmA2 (A2 (M, K2) K-major) and
// tmB2 (B2 with B's major) into the same ring, and the consumers accumulate them into the same registers, so every
// epilogue applies to acc = A B^T + A2 B2^T unchanged.  TMA zero-fills the k columns past K2.
// F8 (a compile-time switch; 0 for the 16-bit kernels) makes A and B fp8, both K-major: 1 = e4m3 x e4m3 (forward),
// 2 = e5m2 x e4m3 (dgrad).  A k-block is then 128 elements, the same 128-byte swizzle row, so the ring, the stage bytes
// and the 32-byte descriptor k-step are those of the 16-bit kernels.  Hopper's fp8 MMA accumulates with reduced
// precision, so each k-block's four k32 MMAs go into a temporary accumulator that the consumer adds into the fp32 one
// with IEEE adds (promotion every 128 k).  Before the epilogue acc = (acc * sa[m]) * sb[n]; the output is T (bf16).
template <typename T, int BN, int A_MN, int B_MN, int EPI, bool LR, int F8 = 0>
__device__ __forceinline__ void gemm_body(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmC,
                                          const CUtensorMap& tmC2, const CUtensorMap& tmAux, const CUtensorMap* tmA2,
                                          const CUtensorMap* tmB2, const GemmParams& p, int kb_tail) {
  using C = Cfg<BN, EPI, F8 != 0>;
  static_assert(F8 == 0 || (!A_MN && !B_MN && !LR && !is_f32_epi(EPI) && BN <= 128), "gemm fp8: K-major, 16-bit epilogues, BN <= 128");
  constexpr int BKE = F8 ? 2 * BK : BK;   // elements per k-block (128 bytes either way)
  constexpr int STAGES = C::STAGES;
  constexpr int NACC = BN / 2;   // accumulator registers per thread (64 x BN fp32 over 128 threads)
  constexpr bool EPI16 = !is_f32_epi(EPI);

  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* epi_buf = smem_raw + STAGES * C::STAGE_BYTES;
  float* bias_s = reinterpret_cast<float*>(epi_buf + C::EPI_BYTES);
  float* sb_s = bias_s + BN;   // FP8 only (SCALE_BYTES)
  uint64_t* bar_full = reinterpret_cast<uint64_t*>(epi_buf + C::EPI_BYTES + C::BIAS_BYTES + C::SCALE_BYTES);
  uint64_t* bar_empty = bar_full + STAGES;
  // 16-bit epilogues: the epilogue producer fills bias (and aux) for a tile -> epi_full; both consumer warpgroups are
  // done with them -> epi_empty
  const uint32_t epi_full = ptx::smem_u32(bar_empty + STAGES);
  const uint32_t epi_empty = epi_full + 8;

  const uint32_t smem_base = ptx::smem_u32(smem_raw);
  if (smem_base & 1023u) __trap();
  const int wg = threadIdx.x >> 7;

  if (threadIdx.x == 0) {
    ptx::tma_prefetch_desc(&tmA);
    ptx::tma_prefetch_desc(&tmB);
    if (EPI16 && p.tma_out) {
      ptx::tma_prefetch_desc(&tmC);
      if (EPI == OASR_EPI_BF16_GELU) ptx::tma_prefetch_desc(&tmC2);
    }
    if (reads_aux(EPI) && p.tma_aux) ptx::tma_prefetch_desc(&tmAux);
    if (LR) {
      ptx::tma_prefetch_desc(tmA2);
      ptx::tma_prefetch_desc(tmB2);
    }
    for (int s = 0; s < STAGES; ++s) {
      ptx::mbar_init(ptx::smem_u32(&bar_full[s]), 1);
      ptx::mbar_init(ptx::smem_u32(&bar_empty[s]), 2);   // one arrival per consumer warpgroup
    }
    ptx::mbar_init(epi_full, 32);    // every lane of the epilogue producer warp
    ptx::mbar_init(epi_empty, 2);    // one arrival per consumer warpgroup
    ptx::fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    ptx::setmaxnreg_dec<PRODUCER_REGS>();
    if (threadIdx.x == 0) {
      // ===================== operand producer =====================
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
        int m_blk, n_blk, split;
        decode_tile(tile, p, m_blk, n_blk, split);
        const int kb0 = split * p.kblocks_per_split;
        const int kb1 = min(kb0 + p.kblocks_per_split, p.kblocks_total);
        for (int kb = kb0; kb < kb1 + (LR ? kb_tail : 0); ++kb) {
          ptx::mbar_wait(ptx::smem_u32(&bar_empty[stage]), phase ^ 1);
          const uint32_t sa = smem_base + stage * C::STAGE_BYTES;
          const uint32_t sb = sa + A_STAGE_BYTES;
          const uint32_t full = ptx::smem_u32(&bar_full[stage]);
          ptx::mbar_arrive_expect_tx(full, C::STAGE_BYTES);
          // a tail k-block reads A2 / B2 at k0 = (kb - kb1) * BK instead of A / B at kb * BK, nothing else
          const bool tail = LR && kb >= kb1;
          const CUtensorMap* ma = tail ? tmA2 : &tmA;
          const CUtensorMap* mb = tail ? tmB2 : &tmB;
          const int k0 = (tail ? kb - kb1 : kb) * BKE;
          if (A_MN) {
#pragma unroll
            for (int i = 0; i < BM / 64; ++i) ptx::tma_load_2d(sa + i * (BK * 128), ma, full, m_blk * BM + i * 64, k0);
          } else {
            ptx::tma_load_2d(sa, ma, full, k0, m_blk * BM);
          }
          if (B_MN) {
#pragma unroll
            for (int i = 0; i < BN / 64; ++i) ptx::tma_load_2d(sb + i * (BK * 128), mb, full, n_blk * BN + i * 64, k0);
          } else {
            ptx::tma_load_2d(sb, mb, full, k0, n_blk * BN);
          }
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    } else if (EPI16 && (threadIdx.x >> 5) == 1) {
      // ===================== epilogue producer: bias slice and aux tile of each tile =====================
      // Its own barriers: the operand producer never waits on the epilogue's buffers.
      const int lane = threadIdx.x & 31;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x, phase ^= 1) {
        int m_blk, n_blk, split;
        decode_tile(tile, p, m_blk, n_blk, split);
        const int m0 = m_blk * BM, n0 = n_blk * BN;
        ptx::mbar_wait(epi_empty, phase ^ 1);   // both consumer warpgroups are done with the previous tile's
        for (int j = lane; j < BN; j += 32)     // rounded to T like bias.to(x.dtype); 0 past N
          bias_s[j] = (p.bias != nullptr && n0 + j < p.N) ? Act16<T>::round(__ldg(p.bias + n0 + j)) : 0.f;
        if constexpr (F8 != 0)
          for (int j = lane; j < BN; j += 32) sb_s[j] = n0 + j < p.N ? __ldg(p.sb + n0 + j) : 0.f;
        if (reads_aux(EPI) && p.tma_aux) {
          if (lane == 0) {   // the boxes that hold rows < M and columns < N; TMA zero-fills past the edges
            const int halves = p.M - m0 > 64 ? 2 : 1;
            const int boxes = min(BN / BOX, (p.N - n0 + BOX - 1) / BOX);
            ptx::mbar_arrive_expect_tx(epi_full, halves * boxes * BOX_BYTES);
            for (int h = 0; h < halves; ++h)
              for (int b = 0; b < boxes; ++b)
                ptx::tma_load_2d(ptx::smem_u32(epi_buf) + (h * (BN / BOX) + b) * BOX_BYTES, &tmAux, epi_full, n0 + BOX * b,
                                 m0 + 64 * h);
          } else {
            ptx::mbar_arrive(epi_full);
          }
        } else {
          if (reads_aux(EPI)) {
            for (int h = 0; h < 2; ++h)
              for (int b = 0; b < BN / BOX; ++b)
                box_from_global<T>(epi_buf + (h * (BN / BOX) + b) * BOX_BYTES, p.aux, p.ldaux, m0 + 64 * h, n0 + BOX * b, p,
                                   lane, 32);
          }
          ptx::mbar_arrive(epi_full);
        }
      }
    }
    return;
  }

  // ===================== consumers =====================
  ptx::setmaxnreg_inc<CONSUMER_REGS>();
  const int c = wg - 1;                 // row half of the tile
  const int t = threadIdx.x & 127;
  const int warp = t >> 5, lane = t & 31;
  // K-major: 8-row groups 1024 B apart (SBO), LBO unused.  MN-major: 64-element chunks BK*128 B apart (LBO), 8-k
  // groups 1024 B apart (SBO).  This warpgroup's 64 rows of A start 8 KB into the A tile in both layouts.
  constexpr uint32_t a_kstep = A_MN ? 16 * 128 : 16 * 2;
  constexpr uint32_t b_kstep = B_MN ? 16 * 128 : 16 * 2;
  const uint64_t a_desc0 = ptx::desc_sw128(smem_base + c * 8192, A_MN ? BK * 128 : 16, 1024);
  const uint64_t b_desc0 = ptx::desc_sw128(smem_base + A_STAGE_BYTES, B_MN ? BK * 128 : 16, 1024);
  const bool vec_c = is_f32_epi(EPI) && (p.ldc & 1) == 0 && (reinterpret_cast<uintptr_t>(p.C) & 7) == 0;
  // this warpgroup's half of the epilogue buffer
  const uint32_t epi_wg = ptx::smem_u32(epi_buf) + c * (C::EPI_BYTES / 2);

  int stage = 0;
  uint32_t phase = 0, epi_phase = 0;
  float acc[NACC];
  for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
    int m_blk, n_blk, split;
    decode_tile(tile, p, m_blk, n_blk, split);
    const int kb0 = split * p.kblocks_per_split;
    const int kb1 = min(kb0 + p.kblocks_per_split, p.kblocks_total);
    if constexpr (F8 != 0) {
      // one k-block at a time: its MMAs into tmp, retired, the slot handed back, then tmp promoted into acc
      float tmp[NACC];
      for (int kb = kb0; kb < kb1; ++kb) {
        ptx::mbar_wait(ptx::smem_u32(&bar_full[stage]), phase);
        const uint64_t ad = ptx::desc_add(a_desc0, stage * C::STAGE_BYTES);
        const uint64_t bd = ptx::desc_add(b_desc0, stage * C::STAGE_BYTES);
        ptx::wgmma_fence();
#pragma unroll
        for (int k = 0; k < BKE / 32; ++k) {
          const uint64_t da = ptx::desc_add(ad, k * 32), db = ptx::desc_add(bd, k * 32);
          float (&d)[NACC] = FP8_PROMOTE ? tmp : acc;
          const uint32_t accumulate = (k > 0 || (!FP8_PROMOTE && kb > kb0)) ? 1u : 0u;
          if constexpr (BN == 128) ptx::wgmma_m64n128k32_f8<F8>(d, da, db, accumulate);
          else ptx::wgmma_m64n64k32_f8<F8>(d, da, db, accumulate);
        }
        ptx::wgmma_commit();
        if (kb == kb0 && tile != static_cast<int>(blockIdx.x) && t == 0) {   // as in the 16-bit loop below
          if (reads_aux(EPI) && p.tma_out) ptx::bulk_wait_group_read<0>();
          ptx::mbar_arrive(epi_empty);
        }
        ptx::wgmma_wait<0>();
        ptx::fence_regs(FP8_PROMOTE ? tmp : acc);
        if (t == 0) ptx::mbar_arrive(ptx::smem_u32(&bar_empty[stage]));
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
        if constexpr (FP8_PROMOTE) {
#pragma unroll
          for (int i = 0; i < NACC; ++i) acc[i] = kb == kb0 ? tmp[i] : __fadd_rn(acc[i], tmp[i]);
        }
      }
    } else {   // 16-bit: one k-block of MMAs kept in flight behind the next one
      int prev = -1;
      for (int kb = kb0; kb < kb1 + (LR ? kb_tail : 0); ++kb) {
        ptx::mbar_wait(ptx::smem_u32(&bar_full[stage]), phase);
        const uint64_t ad = ptx::desc_add(a_desc0, stage * C::STAGE_BYTES);
        const uint64_t bd = ptx::desc_add(b_desc0, stage * C::STAGE_BYTES);
        ptx::wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k) {
          const uint32_t accumulate = (kb > kb0 || k > 0) ? 1u : 0u;
          const uint64_t da = ptx::desc_add(ad, k * a_kstep), db = ptx::desc_add(bd, k * b_kstep);
          if constexpr (BN == 256) ptx::wgmma_m64n256k16_ss<A_MN, B_MN, T>(acc, da, db, accumulate);
          else if constexpr (BN == 128) ptx::wgmma_m64n128k16_ss<A_MN, B_MN, T>(acc, da, db, accumulate);
          else ptx::wgmma_m64n64k16_ss<A_MN, B_MN, T>(acc, da, db, accumulate);
        }
        ptx::wgmma_commit();
        if (EPI16 && kb == kb0 && tile != static_cast<int>(blockIdx.x) && t == 0) {
          // The previous tile's epilogue is over (its last box barrier came after every read of bias and aux); with the
          // MMAs of this tile under way, hand its buffers back once the TMA engine has read the stores' sources.
          if (reads_aux(EPI) && p.tma_out) ptx::bulk_wait_group_read<0>();
          ptx::mbar_arrive(epi_empty);
        }
        ptx::wgmma_wait<1>();   // the previous k-block's MMAs have retired: its slot may be refilled
        if (prev >= 0 && t == 0) ptx::mbar_arrive(ptx::smem_u32(&bar_empty[prev]));
        prev = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      ptx::wgmma_wait<0>();
      ptx::fence_regs(acc);
      if (t == 0) ptx::mbar_arrive(ptx::smem_u32(&bar_empty[prev]));
    }

    if constexpr (is_f32_epi(EPI)) {
      // ---- straight from the fragments: row 16*warp + lane/4 (+8), columns 8i + 2*(lane%4) (+1)
      const int row0 = m_blk * BM + c * 64 + warp * 16 + (lane >> 2);
      const int col0 = n_blk * BN + 2 * (lane & 3);
#pragma unroll
      for (int i = 0; i < BN / 8; ++i) {
        const int col = col0 + 8 * i;
        if (col >= p.N) continue;
        const bool two = col + 1 < p.N;
        float b0 = 0.f, b1 = 0.f;
        if (p.bias != nullptr) {
          b0 = __ldg(p.bias + col);
          b1 = two ? __ldg(p.bias + col + 1) : 0.f;
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = row0 + 8 * h;
          if (row >= p.M) continue;
          const float x0 = __fadd_rn(acc[4 * i + 2 * h], b0), x1 = __fadd_rn(acc[4 * i + 2 * h + 1], b1);
          float* dst = reinterpret_cast<float*>(p.C) + static_cast<int64_t>(row) * p.ldc + col + split * p.split_stride;
          if constexpr (EPI == OASR_EPI_F32_ATOMIC_ADD) {
            atomicAdd(dst, x0);
            if (two) atomicAdd(dst + 1, x1);
          } else if (two && vec_c) {
            *reinterpret_cast<float2*>(dst) = make_float2(x0, x1);
          } else {
            dst[0] = x0;
            if (two) dst[1] = x1;
          }
        }
      }
    } else {
      // ---- 16-bit: T(acc + T(bias)) per column pair (then GELU / residual / GELU backward) into 64 x 64 boxes in shared
      // memory, each stored by one TMA while the warpgroup goes on.  Fragment rows r = 16*warp + lane/4 and r + 8
      // (r % 8 = lane / 4), columns 8i + 2*(lane%4) (+1): one 4-byte word per row of 16-byte chunk i % 8 of box i / 8,
      // and the 8 rows a warp writes at once fall in 8 different chunks, i.e. all 32 banks.
      ptx::mbar_wait(epi_full, epi_phase);
      epi_phase ^= 1;
      const int row0 = m_blk * BM + c * 64;   // first row of this warpgroup's boxes
      if (row0 < p.M) {
        const uint32_t word = (16 * warp + (lane >> 2)) * 128 + 4 * (lane & 3);
        const uint32_t bias_q = ptx::smem_u32(bias_s) + 8 * (lane & 3);
        float sa[2] = {0.f, 0.f};   // FP8: A's scales of this thread's rows r and r + 8
        if constexpr (F8 != 0) {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int row = row0 + 16 * warp + (lane >> 2) + 8 * h;
            sa[h] = row < p.M ? __ldg(p.sa + row) : 0.f;
          }
        }
#pragma unroll
        for (int b = 0; b < BN / BOX; ++b) {
          const int col0 = n_blk * BN + BOX * b;
          if (col0 >= p.N) break;   // warpgroup-uniform
          // TMA stores whole 16-byte chunks: with N % 8 != 0 the box that holds column N - 1 would also write zeros to
          // columns N .. round8(N) - 1, outside the output, so that box goes out by plain bounded copies
          const bool tma_box = p.tma_out && (col0 + BOX <= p.N || (p.N & 7) == 0);
#pragma unroll
          for (int out = 0; out < (EPI == OASR_EPI_BF16_GELU ? 2 : 1); ++out) {
            uint32_t box;
            if constexpr (reads_aux(EPI)) {
              box = epi_wg + b * BOX_BYTES;   // the aux box: each result goes over its own aux
            } else {   // two slots in turn; the store that last read this one is done with it
              constexpr int NOUT = EPI == OASR_EPI_BF16_GELU ? 2 : 1;
              box = epi_wg + ((b * NOUT + out) & 1) * BOX_BYTES;
              if (t == 0) {   // (a tile's first box: the previous tile's stores went out a whole mainloop ago)
                // (a plain-copy box commits no store group, so the latest group may be reading this slot)
                if ((b == 0 && out == 0) || !tma_box) ptx::bulk_wait_group_read<0>();
                else ptx::bulk_wait_group_read<1>();
              }
              ptx::named_bar_sync(1 + c, 128);
            }
#pragma unroll
            for (int j = 0; j < BOX / 8; ++j) {
              const int i = (BOX / 8) * b + j;
              const float2 bb = ptx::ld_shared_f32x2(bias_q + 32 * i);
              float2 sbv = make_float2(0.f, 0.f);
              if constexpr (F8 != 0) sbv = ptx::ld_shared_f32x2(bias_q + BN * 4 + 32 * i);
              const uint32_t wa = box + word + ((j ^ (lane >> 2)) << 4);
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                using A = Act16<T>;
                float a0 = acc[4 * i + 2 * h], a1 = acc[4 * i + 2 * h + 1];
                if constexpr (F8 != 0) {
                  a0 = __fmul_rn(__fmul_rn(a0, sa[h]), sbv.x);
                  a1 = __fmul_rn(__fmul_rn(a1, sa[h]), sbv.y);
                }
                const uint32_t v = A::pack2(__fadd_rn(a0, bb.x), __fadd_rn(a1, bb.y));
                uint32_t o = v;
                if constexpr (EPI == OASR_EPI_BF16_GELU) {   // h = T(acc + b), g = T(gelu(h))
                  if (out) {
                    const float2 x = gelu_erf2(A::unpack2(v));
                    o = A::pack2(x.x, x.y);
                  }
                } else if constexpr (EPI == OASR_EPI_BF16_RESIDUAL) {   // C = T(aux + T(acc + b))
                  const float2 x = fadd2(A::unpack2(ptx::ld_shared_u32(wa + 1024 * h)), A::unpack2(v));
                  o = A::pack2(x.x, x.y);
                } else if constexpr (EPI == OASR_EPI_BF16_GELU_BWD) {   // C = T(T(acc) * gelu'(aux))
                  const float2 x = fmul2(A::unpack2(v), gelu_erf_grad2(A::unpack2(ptx::ld_shared_u32(wa + 1024 * h))));
                  o = A::pack2(x.x, x.y);
                }
                ptx::st_shared_u32(wa + 1024 * h, o);   // row r + 8h: 1024 bytes on, same swizzle
              }
            }
            if (tma_box) {
              ptx::fence_proxy_async_smem();
              ptx::named_bar_sync(1 + c, 128);
              if (t == 0) {
                ptx::tma_store_2d(out ? &tmC2 : &tmC, box, col0, row0);
                ptx::bulk_commit_group();
              }
            } else {
              ptx::named_bar_sync(1 + c, 128);
              box_to_global<T>(smem_raw + (box - smem_base), out ? p.C2 : p.C, p.ldc, row0, col0, p, t);
              ptx::named_bar_sync(1 + c, 128);
            }
          }
        }
      }
    }
  }
  if (EPI16 && t == 0) ptx::bulk_wait_group<0>();   // the stores read shared memory until they complete
}

template <typename T, int BN, int A_MN, int B_MN, int EPI>
__global__ void __launch_bounds__(THREADS, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                  const __grid_constant__ CUtensorMap tmC, const __grid_constant__ CUtensorMap tmC2,
                  const __grid_constant__ CUtensorMap tmAux, const GemmParams p) {
  gemm_body<T, BN, A_MN, B_MN, EPI, false>(tmA, tmB, tmC, tmC2, tmAux, nullptr, nullptr, p, 0);
}

// D = epi(A B^T + A2 B2^T), A and A2 K-major, B2 with B's major
template <typename T, int BN, int B_MN, int EPI>
__global__ void __launch_bounds__(THREADS, 1)
gemm_lowrank_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                    const __grid_constant__ CUtensorMap tmC, const __grid_constant__ CUtensorMap tmC2,
                    const __grid_constant__ CUtensorMap tmAux, const __grid_constant__ CUtensorMap tmA2,
                    const __grid_constant__ CUtensorMap tmB2, const GemmParams p, const int kb_tail) {
  gemm_body<T, BN, 0, B_MN, EPI, true>(tmA, tmB, tmC, tmC2, tmAux, &tmA2, &tmB2, p, kb_tail);
}

// D = epi((sa[m] sb[n]) sum_k A[m,k] B[n,k]), A (M, K) and B (N, K) fp8, K-major, bf16 output
template <int BN, int F8, int EPI>
__global__ void __launch_bounds__(THREADS, 1)
gemm_fp8_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                const __grid_constant__ CUtensorMap tmC, const __grid_constant__ CUtensorMap tmC2,
                const __grid_constant__ CUtensorMap tmAux, const GemmParams p) {
  gemm_body<bf16, BN, 0, 0, EPI, false, F8>(tmA, tmB, tmC, tmC2, tmAux, nullptr, nullptr, p, 0);
}

// split-K: out[m, n] += sum_s ws[s][m][n], splits in order (fp32 atomics would round differently from run to run)
__global__ void splitk_reduce_kernel(const float* __restrict__ ws, int splits, int M, int N, float* __restrict__ out, int64_t ldc) {
  const int64_t mn = static_cast<int64_t>(M) * N;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < mn; i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    float t = 0.f;
    for (int s = 0; s < splits; ++s) t += ws[s * mn + i];
    out[(i / N) * ldc + i % N] += t;
  }
}

// operand maps (A, B), the 16-bit epilogues' maps (C, C2, aux) and the low-rank tail's (A2, B2); zero when unused
struct Maps {
  CUtensorMap a, b, c, c2, aux, a2, b2;
};

template <typename T, int BN, int A_MN, int B_MN, int EPI>
int launch(const Maps& m, const GemmParams& p, cudaStream_t st) {
  using C = Cfg<BN, EPI>;
  auto kern = gemm_wgmma_kernel<T, BN, A_MN, B_MN, EPI>;
  static bool attr_set = false;  // per instantiation
  if (!attr_set) {
    OASR_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES));
    attr_set = true;
  }
  const int grid = p.num_tiles < gemm_sm_budget() ? p.num_tiles : gemm_sm_budget();
  kern<<<grid, THREADS, C::SMEM_BYTES, st>>>(m.a, m.b, m.c, m.c2, m.aux, p);
  OASR_LAUNCH_CHECK();
  return OASR_OK;
}

template <typename T, int BN, int B_MN, int EPI>
int launch_lowrank(const Maps& m, const GemmParams& p, int kb_tail, cudaStream_t st) {
  using C = Cfg<BN, EPI>;
  auto kern = gemm_lowrank_kernel<T, BN, B_MN, EPI>;
  static bool attr_set = false;  // per instantiation
  if (!attr_set) {
    OASR_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES));
    attr_set = true;
  }
  const int grid = p.num_tiles < gemm_sm_budget() ? p.num_tiles : gemm_sm_budget();
  kern<<<grid, THREADS, C::SMEM_BYTES, st>>>(m.a, m.b, m.c, m.c2, m.aux, m.a2, m.b2, p, kb_tail);
  OASR_LAUNCH_CHECK();
  return OASR_OK;
}

template <int BN, int F8, int EPI>
int launch_fp8(const Maps& m, const GemmParams& p, cudaStream_t st) {
  using C = Cfg<BN, EPI, true>;
  auto kern = gemm_fp8_kernel<BN, F8, EPI>;
  static bool attr_set = false;  // per instantiation
  if (!attr_set) {
    OASR_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES));
    attr_set = true;
  }
  const int grid = p.num_tiles < gemm_sm_budget() ? p.num_tiles : gemm_sm_budget();
  kern<<<grid, THREADS, C::SMEM_BYTES, st>>>(m.a, m.b, m.c, m.c2, m.aux, p);
  OASR_LAUNCH_CHECK();
  return OASR_OK;
}

// The FP8 forms of a block projection: forward (e4m3 x e4m3) BF16, BF16_GELU and BF16_RESIDUAL; dgrad (e5m2 x e4m3)
// BF16, BF16_RESIDUAL and BF16_GELU_BWD.
template <int BN>
int dispatch_fp8(int f8, int epi, const Maps& m, const GemmParams& p, cudaStream_t st) {
  if (f8 == 1) {
    switch (epi) {
      case OASR_EPI_BF16: return launch_fp8<BN, 1, OASR_EPI_BF16>(m, p, st);
      case OASR_EPI_BF16_GELU: return launch_fp8<BN, 1, OASR_EPI_BF16_GELU>(m, p, st);
      case OASR_EPI_BF16_RESIDUAL: return launch_fp8<BN, 1, OASR_EPI_BF16_RESIDUAL>(m, p, st);
    }
  } else {
    switch (epi) {
      case OASR_EPI_BF16: return launch_fp8<BN, 2, OASR_EPI_BF16>(m, p, st);
      case OASR_EPI_BF16_RESIDUAL: return launch_fp8<BN, 2, OASR_EPI_BF16_RESIDUAL>(m, p, st);
      case OASR_EPI_BF16_GELU_BWD: return launch_fp8<BN, 2, OASR_EPI_BF16_GELU_BWD>(m, p, st);
    }
  }
  set_last_error("gemm_fp8: no kernel for %s with epilogue %d", f8 == 1 ? "e4m3 x e4m3" : "e5m2 x e4m3", epi);
  return OASR_ERR_UNSUPPORTED;
}

// The pairs a Linear with a low-rank adapter needs, for every tile width: forward (B K-major) BF16, BF16_GELU and
// BF16_RESIDUAL; dgrad (B MN-major) BF16, BF16_RESIDUAL and BF16_GELU_BWD.
template <typename T, int BN>
int dispatch_lowrank(int b_mn, int epi, const Maps& m, const GemmParams& p, int kb_tail, cudaStream_t st) {
  if (!b_mn) {
    switch (epi) {
      case OASR_EPI_BF16: return launch_lowrank<T, BN, 0, OASR_EPI_BF16>(m, p, kb_tail, st);
      case OASR_EPI_BF16_GELU: return launch_lowrank<T, BN, 0, OASR_EPI_BF16_GELU>(m, p, kb_tail, st);
      case OASR_EPI_BF16_RESIDUAL: return launch_lowrank<T, BN, 0, OASR_EPI_BF16_RESIDUAL>(m, p, kb_tail, st);
    }
  } else {
    switch (epi) {
      case OASR_EPI_BF16: return launch_lowrank<T, BN, 1, OASR_EPI_BF16>(m, p, kb_tail, st);
      case OASR_EPI_BF16_RESIDUAL: return launch_lowrank<T, BN, 1, OASR_EPI_BF16_RESIDUAL>(m, p, kb_tail, st);
      case OASR_EPI_BF16_GELU_BWD: return launch_lowrank<T, BN, 1, OASR_EPI_BF16_GELU_BWD>(m, p, kb_tail, st);
    }
  }
  set_last_error("gemm_lowrank: no kernel for b_layout=%d epilogue=%d", b_mn, epi);
  return OASR_ERR_UNSUPPORTED;
}

// The (operand majors, epilogue) pairs the library calls; each is compiled for every tile width:
//   A K-major,  B K-major  (forward Linear / Conv1d, tied logits): BF16, BF16_GELU, BF16_RESIDUAL, BF16_GELU_BWD, F32
//   A K-major,  B MN-major (dgrad, logits dx):                     BF16, BF16_RESIDUAL, BF16_GELU_BWD, F32
//   A MN-major, B MN-major (wgrad):                                F32, F32_ATOMIC_ADD
// (split-K launches store fp32 partials: they run the F32 kernel).  Any other pair is rejected.
template <typename T, int BN>
int dispatch(int a_mn, int b_mn, int epi, const Maps& m, const GemmParams& p, cudaStream_t st) {
  if (!a_mn && !b_mn) {
    switch (epi) {
      case OASR_EPI_BF16: return launch<T, BN, 0, 0, OASR_EPI_BF16>(m, p, st);
      case OASR_EPI_BF16_GELU: return launch<T, BN, 0, 0, OASR_EPI_BF16_GELU>(m, p, st);
      case OASR_EPI_BF16_RESIDUAL: return launch<T, BN, 0, 0, OASR_EPI_BF16_RESIDUAL>(m, p, st);
      case OASR_EPI_BF16_GELU_BWD: return launch<T, BN, 0, 0, OASR_EPI_BF16_GELU_BWD>(m, p, st);
      case OASR_EPI_F32: return launch<T, BN, 0, 0, OASR_EPI_F32>(m, p, st);
    }
  } else if (!a_mn && b_mn) {
    switch (epi) {
      case OASR_EPI_BF16: return launch<T, BN, 0, 1, OASR_EPI_BF16>(m, p, st);
      case OASR_EPI_BF16_RESIDUAL: return launch<T, BN, 0, 1, OASR_EPI_BF16_RESIDUAL>(m, p, st);
      case OASR_EPI_BF16_GELU_BWD: return launch<T, BN, 0, 1, OASR_EPI_BF16_GELU_BWD>(m, p, st);
      case OASR_EPI_F32: return launch<T, BN, 0, 1, OASR_EPI_F32>(m, p, st);
    }
  } else if (a_mn && b_mn) {
    switch (epi) {
      case OASR_EPI_F32: return launch<T, BN, 1, 1, OASR_EPI_F32>(m, p, st);
      case OASR_EPI_F32_ATOMIC_ADD: return launch<T, BN, 1, 1, OASR_EPI_F32_ATOMIC_ADD>(m, p, st);
    }
  }
  set_last_error("gemm: no kernel for a_layout=%d b_layout=%d epilogue=%d", a_mn, b_mn, epi);
  return OASR_ERR_UNSUPPORTED;
}

// TMA addresses a 16-bit matrix whose base and row stride are multiples of 16 bytes
bool tma_addressable(const void* base, int64_t ld) {
  return (reinterpret_cast<uintptr_t>(base) & 15) == 0 && (ld & 7) == 0;
}

template <typename T>
int gemm(const void* A, int64_t lda, int a_layout, const void* B, int64_t ldb, int b_layout, void* Cout, int64_t ldc,
         void* C2, const float* bias, const void* aux, int64_t ldaux, int64_t M, int64_t N, int64_t K, int epilogue,
         int split_k, int block_n, void* stream, const void* A2 = nullptr, int64_t lda2 = 0, const void* B2 = nullptr,
         int64_t ldb2 = 0, int64_t K2 = 0) {
  OASR_REQUIRE(M > 0 && N > 0 && K > 0, "gemm: empty problem M=%ld N=%ld K=%ld", (long)M, (long)N, (long)K);
  OASR_REQUIRE(A && B && Cout, "gemm: null operand");
  OASR_REQUIRE((reinterpret_cast<uintptr_t>(A) & 15) == 0 && (reinterpret_cast<uintptr_t>(B) & 15) == 0,
               "gemm: A/B must be 16-byte aligned");
  OASR_REQUIRE((lda & 7) == 0 && (ldb & 7) == 0, "gemm: lda/ldb must be multiples of 8 elements (TMA)");
  OASR_REQUIRE(epilogue >= OASR_EPI_BF16 && epilogue <= OASR_EPI_F32_ATOMIC_ADD, "gemm: bad epilogue %d", epilogue);
  OASR_REQUIRE(a_layout == OASR_K_MAJOR || a_layout == OASR_MN_MAJOR, "gemm: bad a_layout");
  OASR_REQUIRE(b_layout == OASR_K_MAJOR || b_layout == OASR_MN_MAJOR, "gemm: bad b_layout");
  if (epilogue == OASR_EPI_BF16_GELU) OASR_REQUIRE(C2 != nullptr, "gemm: GELU epilogue needs C2");
  if (epilogue == OASR_EPI_BF16_RESIDUAL || epilogue == OASR_EPI_BF16_GELU_BWD)
    OASR_REQUIRE(aux != nullptr, "gemm: epilogue %d needs aux", epilogue);
  if (split_k < 1) split_k = 1;
  OASR_REQUIRE(split_k == 1 || epilogue == OASR_EPI_F32_ATOMIC_ADD, "gemm: split_k needs the accumulating fp32 epilogue");
  // C += acc: a bias would be added once per split (each split's partial runs the F32 epilogue)
  OASR_REQUIRE(bias == nullptr || epilogue != OASR_EPI_F32_ATOMIC_ADD, "gemm: the accumulating fp32 epilogue takes no bias");
  if (A2 != nullptr) {   // low-rank tail: the 16-bit epilogues of a Linear's forward or dgrad, one split
    OASR_REQUIRE(B2 != nullptr && K2 > 0 && K2 <= 192 && (K2 & 7) == 0,
                 "gemm_lowrank: K2=%ld must be a multiple of 8 in [8, 192] with both tail operands given", (long)K2);
    OASR_REQUIRE(a_layout == OASR_K_MAJOR, "gemm_lowrank: A must be K-major");
    OASR_REQUIRE(!is_f32_epi(epilogue) && split_k == 1, "gemm_lowrank: 16-bit epilogues only, without split-K");
    OASR_REQUIRE((reinterpret_cast<uintptr_t>(A2) & 15) == 0 && (reinterpret_cast<uintptr_t>(B2) & 15) == 0 &&
                 (lda2 & 7) == 0 && (ldb2 & 7) == 0, "gemm_lowrank: A2/B2 must be 16-byte aligned with lda2/ldb2 multiples of 8");
  }
  if (block_n == 0) block_n = (N > 128) ? 256 : (N > 64 ? 128 : 64);
  OASR_REQUIRE(block_n == 64 || block_n == 128 || block_n == 256, "gemm: block_n must be 64/128/256");

  GemmParams p;
  p.C = Cout; p.C2 = C2; p.bias = bias; p.aux = aux; p.ldc = ldc; p.ldaux = ldaux;
  p.M = (int)M; p.N = (int)N; p.K = (int)K;
  p.tiles_m = (int)ceil_div(M, BM);
  p.tiles_n = (int)ceil_div(N, block_n);
  p.kblocks_total = (int)ceil_div(K, BK);
  if (split_k > p.kblocks_total) split_k = p.kblocks_total;
  p.kblocks_per_split = (int)ceil_div(p.kblocks_total, split_k);
  p.splits = (int)ceil_div(p.kblocks_total, p.kblocks_per_split);
  p.raster_m = (N > M) ? 1 : 0;
  p.num_tiles = p.tiles_m * p.tiles_n * p.splits;
  p.split_stride = 0;
  p.sa = p.sb = nullptr;

  Maps m;
  memset(&m, 0, sizeof(m));
  constexpr bool f16 = Act16<T>::is_fp16;
  int rc;
  if (a_layout == OASR_K_MAJOR)
    rc = make_tmap_2d(&m.a, A, 2, (uint64_t)K, (uint64_t)M, (uint64_t)lda * 2, BK, BM, true, f16);
  else
    rc = make_tmap_2d(&m.a, A, 2, (uint64_t)M, (uint64_t)K, (uint64_t)lda * 2, 64, BK, true, f16);
  if (rc) return rc;
  if (b_layout == OASR_K_MAJOR)
    rc = make_tmap_2d(&m.b, B, 2, (uint64_t)K, (uint64_t)N, (uint64_t)ldb * 2, BK, block_n, true, f16);
  else
    rc = make_tmap_2d(&m.b, B, 2, (uint64_t)N, (uint64_t)K, (uint64_t)ldb * 2, 64, BK, true, f16);
  if (rc) return rc;
  if (A2 != nullptr) {
    if ((rc = make_tmap_2d(&m.a2, A2, 2, (uint64_t)K2, (uint64_t)M, (uint64_t)lda2 * 2, BK, BM, true, f16))) return rc;
    if (b_layout == OASR_K_MAJOR)
      rc = make_tmap_2d(&m.b2, B2, 2, (uint64_t)K2, (uint64_t)N, (uint64_t)ldb2 * 2, BK, block_n, true, f16);
    else
      rc = make_tmap_2d(&m.b2, B2, 2, (uint64_t)N, (uint64_t)K2, (uint64_t)ldb2 * 2, 64, BK, true, f16);
    if (rc) return rc;
  }

  // 16-bit epilogues: outputs and aux move by TMA in 64 x 64 boxes where TMA can address them (clipped at M and N by
  // the maps; an output box past N with N % 8 != 0 is stored by plain copies, see the consumer), by plain bounded
  // copies otherwise
  const bool epi16 = !is_f32_epi(epilogue);
  p.tma_out = epi16 && tma_addressable(Cout, ldc) && (epilogue != OASR_EPI_BF16_GELU || tma_addressable(C2, ldc));
  p.tma_aux = reads_aux(epilogue) && tma_addressable(aux, ldaux);
  if (p.tma_out) {
    if ((rc = make_tmap_2d(&m.c, Cout, 2, (uint64_t)N, (uint64_t)M, (uint64_t)ldc * 2, BOX, BOX, true, f16))) return rc;
    if (epilogue == OASR_EPI_BF16_GELU &&
        (rc = make_tmap_2d(&m.c2, C2, 2, (uint64_t)N, (uint64_t)M, (uint64_t)ldc * 2, BOX, BOX, true, f16)))
      return rc;
  }
  if (p.tma_aux &&
      (rc = make_tmap_2d(&m.aux, aux, 2, (uint64_t)N, (uint64_t)M, (uint64_t)ldaux * 2, BOX, BOX, true, f16)))
    return rc;

  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  float* ws = nullptr;
  if (p.splits > 1) {   // every split stores its partial product; one more launch adds them to C in split order
    ws = static_cast<float*>(scratch_alloc(sizeof(float) * p.splits * M * N, st));
    if (!ws) return OASR_ERR_CUDA;
    p.C = ws; p.ldc = N; epilogue = OASR_EPI_F32; p.split_stride = M * N;
  }
  if (A2 != nullptr) {
    const int kb_tail = (int)ceil_div(K2, BK);
    return block_n == 256 ? dispatch_lowrank<T, 256>(b_layout, epilogue, m, p, kb_tail, st)
         : block_n == 128 ? dispatch_lowrank<T, 128>(b_layout, epilogue, m, p, kb_tail, st)
                          : dispatch_lowrank<T, 64>(b_layout, epilogue, m, p, kb_tail, st);
  }
  rc = block_n == 256 ? dispatch<T, 256>(a_layout, b_layout, epilogue, m, p, st)
     : block_n == 128 ? dispatch<T, 128>(a_layout, b_layout, epilogue, m, p, st)
                      : dispatch<T, 64>(a_layout, b_layout, epilogue, m, p, st);
  if (ws) {
    if (rc == OASR_OK) {
      int64_t blocks = ceil_div(M * N, 256);
      const int64_t cap = static_cast<int64_t>(num_sms()) * 8;
      splitk_reduce_kernel<<<(unsigned)(blocks < cap ? blocks : cap), 256, 0, st>>>(ws, p.splits, (int)M, (int)N, static_cast<float*>(Cout), ldc);
      const cudaError_t e = cudaGetLastError();
      if (e != cudaSuccess) { set_last_error("gemm split-K reduce: %s", cudaGetErrorString(e)); rc = OASR_ERR_CUDA; }
    }
    scratch_free(ws, st);
  }
  return rc;
}

int gemm_fp8(const void* A, int64_t lda, int a_fmt, const float* a_scale, const void* B, int64_t ldb, int b_fmt,
             const float* b_scale, void* Cout, int64_t ldc, void* C2, const float* bias, const void* aux, int64_t ldaux,
             int64_t M, int64_t N, int64_t K, int epilogue, int block_n, void* stream) {
  OASR_REQUIRE(M > 0 && N > 0 && K > 0, "gemm_fp8: empty problem M=%ld N=%ld K=%ld", (long)M, (long)N, (long)K);
  OASR_REQUIRE(A && B && Cout && a_scale && b_scale, "gemm_fp8: null operand or scale");
  OASR_REQUIRE(b_fmt == OASR_FP8_E4M3 && (a_fmt == OASR_FP8_E4M3 || a_fmt == OASR_FP8_E5M2),
               "gemm_fp8: formats A=%d B=%d; supported are e4m3 x e4m3 and e5m2 x e4m3", a_fmt, b_fmt);
  // TMA: 16-byte aligned bases and row strides, i.e. multiples of 16 one-byte elements
  OASR_REQUIRE((K & 15) == 0, "gemm_fp8: K=%ld must be a multiple of 16", (long)K);
  OASR_REQUIRE((reinterpret_cast<uintptr_t>(A) & 15) == 0 && (reinterpret_cast<uintptr_t>(B) & 15) == 0 && (lda & 15) == 0 &&
               (ldb & 15) == 0, "gemm_fp8: A/B must be 16-byte aligned with lda/ldb multiples of 16");
  OASR_REQUIRE(epilogue >= OASR_EPI_BF16 && epilogue <= OASR_EPI_BF16_GELU_BWD, "gemm_fp8: 16-bit epilogues only, got %d",
               epilogue);
  if (epilogue == OASR_EPI_BF16_GELU) OASR_REQUIRE(C2 != nullptr, "gemm_fp8: GELU epilogue needs C2");
  if (reads_aux(epilogue)) OASR_REQUIRE(aux != nullptr, "gemm_fp8: epilogue %d needs aux", epilogue);
  if (block_n == 0) block_n = N > 64 ? 128 : 64;
  OASR_REQUIRE(block_n == 64 || block_n == 128, "gemm_fp8: block_n must be 64 or 128");

  GemmParams p;
  memset(&p, 0, sizeof(p));
  p.C = Cout; p.C2 = C2; p.bias = bias; p.aux = aux; p.ldc = ldc; p.ldaux = ldaux;
  p.M = (int)M; p.N = (int)N; p.K = (int)K;
  p.tiles_m = (int)ceil_div(M, BM);
  p.tiles_n = (int)ceil_div(N, block_n);
  p.kblocks_total = p.kblocks_per_split = (int)ceil_div(K, 2 * BK);
  p.splits = 1;
  p.raster_m = (N > M) ? 1 : 0;
  p.num_tiles = p.tiles_m * p.tiles_n;
  p.sa = a_scale; p.sb = b_scale;

  Maps m;
  memset(&m, 0, sizeof(m));
  int rc;
  if ((rc = make_tmap_2d(&m.a, A, 1, (uint64_t)K, (uint64_t)M, (uint64_t)lda, 2 * BK, BM, true))) return rc;
  if ((rc = make_tmap_2d(&m.b, B, 1, (uint64_t)K, (uint64_t)N, (uint64_t)ldb, 2 * BK, block_n, true))) return rc;
  p.tma_out = tma_addressable(Cout, ldc) && (epilogue != OASR_EPI_BF16_GELU || tma_addressable(C2, ldc));
  p.tma_aux = reads_aux(epilogue) && tma_addressable(aux, ldaux);
  if (p.tma_out) {
    if ((rc = make_tmap_2d(&m.c, Cout, 2, (uint64_t)N, (uint64_t)M, (uint64_t)ldc * 2, BOX, BOX, true))) return rc;
    if (epilogue == OASR_EPI_BF16_GELU &&
        (rc = make_tmap_2d(&m.c2, C2, 2, (uint64_t)N, (uint64_t)M, (uint64_t)ldc * 2, BOX, BOX, true)))
      return rc;
  }
  if (p.tma_aux && (rc = make_tmap_2d(&m.aux, aux, 2, (uint64_t)N, (uint64_t)M, (uint64_t)ldaux * 2, BOX, BOX, true)))
    return rc;
  const int f8 = a_fmt == OASR_FP8_E4M3 ? 1 : 2;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  return block_n == 128 ? dispatch_fp8<128>(f8, epilogue, m, p, st) : dispatch_fp8<64>(f8, epilogue, m, p, st);
}

}  // namespace
}  // namespace oasr

using namespace oasr;

extern "C" int oasr_gemm_fp8(const void* A, int64_t lda, int a_fmt, const float* a_scale, const void* B, int64_t ldb,
                             int b_fmt, const float* b_scale, void* Cout, int64_t ldc, void* C2, const float* bias,
                             const void* aux, int64_t ldaux, int64_t M, int64_t N, int64_t K, int epilogue, int block_n,
                             void* stream) {
  return gemm_fp8(A, lda, a_fmt, a_scale, B, ldb, b_fmt, b_scale, Cout, ldc, C2, bias, aux, ldaux, M, N, K, epilogue,
                  block_n, stream);
}

extern "C" int oasr_gemm_bf16(const void* A, int64_t lda, int a_layout, const void* B, int64_t ldb,
                              int b_layout, void* Cout, int64_t ldc, void* C2, const float* bias,
                              const void* aux, int64_t ldaux, int64_t M, int64_t N, int64_t K,
                              int epilogue, int split_k, int block_n, void* stream) {
  return gemm<bf16>(A, lda, a_layout, B, ldb, b_layout, Cout, ldc, C2, bias, aux, ldaux, M, N, K, epilogue, split_k, block_n,
                    stream);
}

extern "C" int oasr_gemm16(const void* A, int64_t lda, int a_layout, const void* B, int64_t ldb, int b_layout, void* Cout,
                           int64_t ldc, void* C2, const float* bias, const void* aux, int64_t ldaux, int64_t M, int64_t N,
                           int64_t K, int epilogue, int split_k, int block_n, int dtype, void* stream) {
  return OASR_BY_DTYPE16(dtype, gemm, A, lda, a_layout, B, ldb, b_layout, Cout, ldc, C2, bias, aux, ldaux, M, N, K, epilogue,
                         split_k, block_n, stream);
}

extern "C" int oasr_gemm_lowrank16(const void* A, int64_t lda, const void* B, int64_t ldb, int b_layout, const void* A2,
                                   int64_t lda2, const void* B2, int64_t ldb2, void* Cout, int64_t ldc, void* C2,
                                   const float* bias, const void* aux, int64_t ldaux, int64_t M, int64_t N, int64_t K,
                                   int64_t K2, int epilogue, int block_n, int dtype, void* stream) {
  OASR_REQUIRE(A2 != nullptr, "gemm_lowrank: null tail operand A2");
  return OASR_BY_DTYPE16(dtype, gemm, A, lda, OASR_K_MAJOR, B, ldb, b_layout, Cout, ldc, C2, bias, aux, ldaux, M, N, K,
                         epilogue, 1, block_n, stream, A2, lda2, B2, ldb2, K2);
}
