// Persistent, warp-specialised bf16 GEMM for sm_90a: TMA -> 128B-swizzled smem ring -> wgmma (fp32 accumulators in
// registers) -> fused epilogue stored straight from the accumulator fragments.
//
//   D[M,N] = epi( sum_k A[m,k] B[n,k] )
//
// One CTA per SM (at most gemm_sm_budget() CTAs), walking over 128 x BN output tiles with stride gridDim.x.  384 threads:
//   warpgroup 0    TMA producer (one thread issues; the ring keeps running across tiles, so the next tile's operands
//                  arrive while this tile's epilogue runs)
//   warpgroups 1-2 consumers: warpgroup c owns rows 64c .. 64c+63 of the tile, issues its m64 x BN x 16 wgmmas and runs
//                  the epilogue for those rows
// Tile = 128 x BN (BN = 64 or 128), BK = 64 bf16 (= one 128-byte swizzle row).  Both operand majors are supported
// through the wgmma descriptors and transpose bits, so dgrad (B MN-major) and wgrad (A and B MN-major) need no
// transposes in HBM.  Reference ops replaced: olmoasr/model.py:97-101 (Linear.forward) and its
// autograd, model.py:768-770 (tied logits), model.py:592-593 (Conv1d after im2col).
#include "common.cuh"
#include "ptx_sm90.cuh"

#include <stdio.h>
#include <stdlib.h>

namespace oasr {
namespace {

constexpr int BM = 128;
constexpr int BK = 64;               // 64 bf16 = 128 B = swizzle span
constexpr int A_STAGE_BYTES = BM * BK * 2;  // 16 KB
constexpr int THREADS = 384;

struct GemmParams {
  void* C;
  void* C2;
  const float* bias;
  const void* aux;
  int64_t ldc;
  int64_t ldaux;
  int M, N, K;
  int tiles_m, tiles_n, splits;
  int kblocks_total, kblocks_per_split;
  int epi;
  int raster_m;  // 1: consecutive tiles walk M first (B tile stays hot in L2) -- used when B is the larger operand
  int64_t split_stride;   // split-K: split s stores its fp32 partial at C + s * split_stride (0: one split)
};

template <int BN>
struct Cfg {
  static constexpr int B_STAGE_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;
  static constexpr int BUDGET = 232448 - 1024;   // 227 KB of dynamic smem per block, minus the barrier area
  static constexpr int STAGES = (BUDGET / STAGE_BYTES) > 8 ? 8 : (BUDGET / STAGE_BYTES);
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024;   // 1024-aligned base: tiles first, barriers last
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

// two adjacent output columns of one row
__device__ __forceinline__ void store_pair(const GemmParams& p, int row, int col, int split, float x0, float x1, bool vec_c,
                                           bool vec_aux) {
  const bool two = col + 1 < p.N;
  const int64_t off = static_cast<int64_t>(row) * p.ldc + col + split * p.split_stride;
  if (p.epi == OASR_EPI_F32) {
    float* dst = reinterpret_cast<float*>(p.C) + off;
    if (two && vec_c) *reinterpret_cast<float2*>(dst) = make_float2(x0, x1);
    else { dst[0] = x0; if (two) dst[1] = x1; }
    return;
  }
  if (p.epi == OASR_EPI_F32_ATOMIC_ADD) {
    float* dst = reinterpret_cast<float*>(p.C) + off;
    atomicAdd(dst, x0);
    if (two) atomicAdd(dst + 1, x1);
    return;
  }
  uint32_t o1 = pack_bf16x2(x0, x1), o2 = 0;
  if (p.epi == OASR_EPI_BF16_GELU) {   // h = bf16(acc + b), g = bf16(gelu(h))
    const float2 g = gelu_erf2(unpack_bf16x2(o1));
    o2 = pack_bf16x2(g.x, g.y);
  } else if (p.epi == OASR_EPI_BF16_RESIDUAL || p.epi == OASR_EPI_BF16_GELU_BWD) {
    const bf16* ap = reinterpret_cast<const bf16*>(p.aux) + static_cast<int64_t>(row) * p.ldaux + col;
    uint32_t aw;
    if (two && vec_aux) aw = *reinterpret_cast<const uint32_t*>(ap);
    else aw = pack_bf16x2(__bfloat162float(ap[0]), two ? __bfloat162float(ap[1]) : 0.f);
    const float2 a = unpack_bf16x2(aw);
    const float2 y = unpack_bf16x2(o1);   // bf16(acc + b): the matmul output as the reference rounds it
    if (p.epi == OASR_EPI_BF16_RESIDUAL) {   // C = bf16(aux + bf16(acc + b))
      const float2 o = fadd2(a, y);
      o1 = pack_bf16x2(o.x, o.y);
    } else {                                 // C = bf16(bf16(acc) * gelu'(aux))
      const float2 o = fmul2(y, gelu_erf_grad2(a));
      o1 = pack_bf16x2(o.x, o.y);
    }
  }
  bf16* dst = reinterpret_cast<bf16*>(p.C) + off;
  if (two && vec_c) *reinterpret_cast<uint32_t*>(dst) = o1;
  else { reinterpret_cast<uint16_t*>(dst)[0] = static_cast<uint16_t>(o1); if (two) reinterpret_cast<uint16_t*>(dst)[1] = static_cast<uint16_t>(o1 >> 16); }
  if (p.epi == OASR_EPI_BF16_GELU) {
    bf16* dst2 = reinterpret_cast<bf16*>(p.C2) + off;
    if (two && vec_c) *reinterpret_cast<uint32_t*>(dst2) = o2;
    else { reinterpret_cast<uint16_t*>(dst2)[0] = static_cast<uint16_t>(o2); if (two) reinterpret_cast<uint16_t*>(dst2)[1] = static_cast<uint16_t>(o2 >> 16); }
  }
}

template <int BN, int A_MN, int B_MN>
__global__ void __launch_bounds__(THREADS, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GemmParams p) {
  using C = Cfg<BN>;
  constexpr int STAGES = C::STAGES;
  constexpr int NACC = BN / 2;   // accumulator registers per thread (64 x BN fp32 over 128 threads)

  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint64_t* bar_full = reinterpret_cast<uint64_t*>(smem_raw + STAGES * C::STAGE_BYTES);
  uint64_t* bar_empty = bar_full + STAGES;

  const uint32_t smem_base = ptx::smem_u32(smem_raw);
  if (smem_base & 1023u) __trap();
  const int wg = threadIdx.x >> 7;

  if (threadIdx.x == 0) {
    ptx::tma_prefetch_desc(&tmA);
    ptx::tma_prefetch_desc(&tmB);
    for (int s = 0; s < STAGES; ++s) {
      ptx::mbar_init(ptx::smem_u32(&bar_full[s]), 1);
      ptx::mbar_init(ptx::smem_u32(&bar_empty[s]), 2);   // one arrival per consumer warpgroup
    }
    ptx::fence_barrier_init();
  }
  __syncthreads();

  const int num_tiles = p.tiles_m * p.tiles_n * p.splits;

  if (wg == 0) {
    // ===================== TMA producer =====================
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        int m_blk, n_blk, split;
        decode_tile(tile, p, m_blk, n_blk, split);
        const int kb0 = split * p.kblocks_per_split;
        const int kb1 = min(kb0 + p.kblocks_per_split, p.kblocks_total);
        for (int kb = kb0; kb < kb1; ++kb) {
          ptx::mbar_wait(ptx::smem_u32(&bar_empty[stage]), phase ^ 1);
          const uint32_t sa = smem_base + stage * C::STAGE_BYTES;
          const uint32_t sb = sa + A_STAGE_BYTES;
          const uint32_t full = ptx::smem_u32(&bar_full[stage]);
          ptx::mbar_arrive_expect_tx(full, C::STAGE_BYTES);
          if (A_MN) {
#pragma unroll
            for (int i = 0; i < BM / 64; ++i) ptx::tma_load_2d(sa + i * (BK * 128), &tmA, full, m_blk * BM + i * 64, kb * BK);
          } else {
            ptx::tma_load_2d(sa, &tmA, full, kb * BK, m_blk * BM);
          }
          if (B_MN) {
#pragma unroll
            for (int i = 0; i < BN / 64; ++i) ptx::tma_load_2d(sb + i * (BK * 128), &tmB, full, n_blk * BN + i * 64, kb * BK);
          } else {
            ptx::tma_load_2d(sb, &tmB, full, kb * BK, n_blk * BN);
          }
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }

  // ===================== consumers =====================
  const int c = wg - 1;                 // row half of the tile
  const int t = threadIdx.x & 127;
  const int warp = t >> 5, lane = t & 31;
  // K-major: 8-row groups 1024 B apart (SBO), LBO unused.  MN-major: 64-element chunks BK*128 B apart (LBO), 8-k
  // groups 1024 B apart (SBO).  This warpgroup's 64 rows of A start 8 KB into the A tile in both layouts.
  constexpr uint32_t a_kstep = A_MN ? 16 * 128 : 16 * 2;
  constexpr uint32_t b_kstep = B_MN ? 16 * 128 : 16 * 2;
  const uint64_t a_desc0 = ptx::desc_sw128(smem_base + c * 8192, A_MN ? BK * 128 : 16, 1024);
  const uint64_t b_desc0 = ptx::desc_sw128(smem_base + A_STAGE_BYTES, B_MN ? BK * 128 : 16, 1024);
  const bool c_is_f32 = (p.epi == OASR_EPI_F32 || p.epi == OASR_EPI_F32_ATOMIC_ADD);
  const bool vec_c = c_is_f32 ? ((p.ldc & 1) == 0 && (reinterpret_cast<uintptr_t>(p.C) & 7) == 0)
                              : ((p.ldc & 1) == 0 && (reinterpret_cast<uintptr_t>(p.C) & 3) == 0 &&
                                 (p.C2 == nullptr || (reinterpret_cast<uintptr_t>(p.C2) & 3) == 0));
  const bool vec_aux = (p.ldaux & 1) == 0 && (reinterpret_cast<uintptr_t>(p.aux) & 3) == 0;

  int stage = 0;
  uint32_t phase = 0;
  float acc[NACC];
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    int m_blk, n_blk, split;
    decode_tile(tile, p, m_blk, n_blk, split);
    const int kb0 = split * p.kblocks_per_split;
    const int kb1 = min(kb0 + p.kblocks_per_split, p.kblocks_total);
    int prev = -1;
    for (int kb = kb0; kb < kb1; ++kb) {
      ptx::mbar_wait(ptx::smem_u32(&bar_full[stage]), phase);
      const uint64_t ad = ptx::desc_add(a_desc0, stage * C::STAGE_BYTES);
      const uint64_t bd = ptx::desc_add(b_desc0, stage * C::STAGE_BYTES);
      ptx::wgmma_fence();
#pragma unroll
      for (int k = 0; k < BK / 16; ++k) {
        const uint32_t accumulate = (kb > kb0 || k > 0) ? 1u : 0u;
        if constexpr (BN == 128) ptx::wgmma_m64n128k16_ss<A_MN, B_MN>(acc, ptx::desc_add(ad, k * a_kstep), ptx::desc_add(bd, k * b_kstep), accumulate);
        else ptx::wgmma_m64n64k16_ss<A_MN, B_MN>(acc, ptx::desc_add(ad, k * a_kstep), ptx::desc_add(bd, k * b_kstep), accumulate);
      }
      ptx::wgmma_commit();
      ptx::wgmma_wait<1>();   // the previous k-block's MMAs have retired: its slot may be refilled
      if (prev >= 0 && t == 0) ptx::mbar_arrive(ptx::smem_u32(&bar_empty[prev]));
      prev = stage;
      if (++stage == STAGES) { stage = 0; phase ^= 1; }
    }
    ptx::wgmma_wait<0>();
    ptx::fence_regs(acc);
    if (t == 0) ptx::mbar_arrive(ptx::smem_u32(&bar_empty[prev]));

    // ---- epilogue straight from the fragments: row 16*warp + lane/4 (+8), columns 8i + 2*(lane%4) (+1)
    const int row0 = m_blk * BM + c * 64 + warp * 16 + (lane >> 2);
    const int col0 = n_blk * BN + 2 * (lane & 3);
#pragma unroll
    for (int i = 0; i < BN / 8; ++i) {
      const int col = col0 + 8 * i;
      if (col >= p.N) continue;
      float b0 = 0.f, b1 = 0.f;
      if (p.bias != nullptr) {   // rounded to bf16 like bias.to(x.dtype) unless the output is fp32
        b0 = __ldg(p.bias + col);
        b1 = col + 1 < p.N ? __ldg(p.bias + col + 1) : 0.f;
        if (!c_is_f32) { b0 = bf16_round(b0); b1 = bf16_round(b1); }
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = row0 + 8 * h;
        if (row < p.M)
          store_pair(p, row, col, split, __fadd_rn(acc[4 * i + 2 * h], b0), __fadd_rn(acc[4 * i + 2 * h + 1], b1), vec_c, vec_aux);
      }
    }
  }
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

template <int BN, int A_MN, int B_MN>
int launch(const CUtensorMap& tmA, const CUtensorMap& tmB, const GemmParams& p, cudaStream_t st) {
  using C = Cfg<BN>;
  auto kern = gemm_wgmma_kernel<BN, A_MN, B_MN>;
  static bool attr_set = false;  // per instantiation
  if (!attr_set) {
    OASR_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES));
    attr_set = true;
  }
  const int tiles = p.tiles_m * p.tiles_n * p.splits;
  const int grid = tiles < gemm_sm_budget() ? tiles : gemm_sm_budget();
  kern<<<grid, THREADS, C::SMEM_BYTES, st>>>(tmA, tmB, p);
  OASR_LAUNCH_CHECK();
  return OASR_OK;
}

template <int BN>
int dispatch_major(int a_mn, int b_mn, const CUtensorMap& tmA, const CUtensorMap& tmB, const GemmParams& p, cudaStream_t st) {
  if (!a_mn && !b_mn) return launch<BN, 0, 0>(tmA, tmB, p, st);
  if (!a_mn && b_mn) return launch<BN, 0, 1>(tmA, tmB, p, st);
  if (a_mn && b_mn) return launch<BN, 1, 1>(tmA, tmB, p, st);
  return launch<BN, 1, 0>(tmA, tmB, p, st);
}

}  // namespace
}  // namespace oasr

using namespace oasr;

extern "C" int oasr_gemm_bf16(const void* A, int64_t lda, int a_layout, const void* B, int64_t ldb,
                              int b_layout, void* Cout, int64_t ldc, void* C2, const float* bias,
                              const void* aux, int64_t ldaux, int64_t M, int64_t N, int64_t K,
                              int epilogue, int split_k, int block_n, void* stream) {
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
  if (block_n == 0) block_n = (N > 64) ? 128 : 64;
  OASR_REQUIRE(block_n == 64 || block_n == 128 || block_n == 256, "gemm: block_n must be 64/128/256");
  // 128 is the widest tile on sm_90a: two consumer warpgroups of 64 x 128 fp32 accumulators each; a 256-wide request
  // is served by 128-wide tiles (same result, the registers of a 64 x 256 accumulator would spill)
  if (block_n == 256) block_n = 128;

  GemmParams p;
  p.C = Cout; p.C2 = C2; p.bias = bias; p.aux = aux; p.ldc = ldc; p.ldaux = ldaux;
  p.M = (int)M; p.N = (int)N; p.K = (int)K;
  p.tiles_m = (int)ceil_div(M, BM);
  p.tiles_n = (int)ceil_div(N, block_n);
  p.kblocks_total = (int)ceil_div(K, BK);
  if (split_k > p.kblocks_total) split_k = p.kblocks_total;
  p.kblocks_per_split = (int)ceil_div(p.kblocks_total, split_k);
  p.splits = (int)ceil_div(p.kblocks_total, p.kblocks_per_split);
  p.epi = epilogue;
  p.raster_m = (N > M) ? 1 : 0;
  p.split_stride = 0;

  CUtensorMap tmA, tmB;
  int rc;
  if (a_layout == OASR_K_MAJOR)
    rc = make_tmap_2d(&tmA, A, 2, (uint64_t)K, (uint64_t)M, (uint64_t)lda * 2, BK, BM, true);
  else
    rc = make_tmap_2d(&tmA, A, 2, (uint64_t)M, (uint64_t)K, (uint64_t)lda * 2, 64, BK, true);
  if (rc) return rc;
  if (b_layout == OASR_K_MAJOR)
    rc = make_tmap_2d(&tmB, B, 2, (uint64_t)K, (uint64_t)N, (uint64_t)ldb * 2, BK, block_n, true);
  else
    rc = make_tmap_2d(&tmB, B, 2, (uint64_t)N, (uint64_t)K, (uint64_t)ldb * 2, 64, BK, true);
  if (rc) return rc;

  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  float* ws = nullptr;
  if (p.splits > 1) {   // every split stores its partial product; one more launch adds them to C in split order
    ws = static_cast<float*>(scratch_alloc(sizeof(float) * p.splits * M * N, st));
    if (!ws) return OASR_ERR_CUDA;
    p.C = ws; p.ldc = N; p.epi = OASR_EPI_F32; p.split_stride = M * N;
  }
  rc = (block_n == 128) ? dispatch_major<128>(a_layout, b_layout, tmA, tmB, p, st) : dispatch_major<64>(a_layout, b_layout, tmA, tmB, p, st);
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
