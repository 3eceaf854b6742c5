// Persistent, warp-specialised bf16 GEMM for sm_90a: TMA -> 128B-swizzled smem ring -> wgmma (fp32 accumulators in
// registers) -> fused epilogue stored straight from the accumulator fragments.
//
//   D[M,N] = epi( sum_k A[m,k] B[n,k] )
//
// One CTA per SM (at most gemm_sm_budget() CTAs), walking over 128 x BN output tiles with stride gridDim.x.  384 threads:
//   warpgroup 0    TMA producer (one thread issues; the ring keeps running across tiles, so the next tile's operands
//                  arrive while this tile's epilogue runs).  It gives its registers up (setmaxnreg 40) ...
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

namespace oasr {
namespace {

constexpr int BM = 128;
constexpr int BK = 64;               // 64 bf16 = 128 B = swizzle span
constexpr int A_STAGE_BYTES = BM * BK * 2;  // 16 KB
constexpr int THREADS = 384;
constexpr int PRODUCER_REGS = 40;    // 40 * 128 + 232 * 256 <= 64 K registers of the SM
constexpr int CONSUMER_REGS = 232;

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

constexpr bool is_f32_epi(int epi) { return epi == OASR_EPI_F32 || epi == OASR_EPI_F32_ATOMIC_ADD; }
constexpr bool reads_aux(int epi) { return epi == OASR_EPI_BF16_RESIDUAL || epi == OASR_EPI_BF16_GELU_BWD; }

__device__ __forceinline__ uint32_t pick4(const uint32_t (&w)[4], int i) {
  return i == 0 ? w[0] : (i == 1 ? w[1] : (i == 2 ? w[2] : w[3]));
}

// 4 x 4 word transpose inside each quad of lanes: lane q holds w[k] = bf16 columns 8k + 2q, 8k + 2q + 1 (k = 0..3) of
// one row; afterwards it holds v[k] = columns 8q + 2k, 8q + 2k + 1, i.e. 8 consecutive columns (one 16-byte store).
__device__ __forceinline__ void quad_transpose(const uint32_t (&w)[4], uint32_t (&v)[4], int lane) {
  const int q = lane & 3;
#pragma unroll
  for (int r = 0; r < 4; ++r) {   // round r: lane p sends its w[(p + r) % 4], lane q receives from lane (q - r) % 4
    const int src = (q - r) & 3;
    const uint32_t x = __shfl_sync(0xffffffffu, pick4(w, (q + r) & 3), (lane & ~3) | src);
#pragma unroll
    for (int k = 0; k < 4; ++k)
      if (src == k) v[k] = x;
  }
}

// aux of 8 consecutive columns col .. col+7 of one row, a[k] = columns col+2k, col+2k+1 (0 past N).  Plain loads: aux
// may be the output itself (in-place residual).
template <typename T>
__device__ __forceinline__ void load_aux_16x8(const GemmParams& p, int row, int col, uint32_t (&a)[4], bool vec_aux) {
  const T* ap = reinterpret_cast<const T*>(p.aux) + static_cast<int64_t>(row) * p.ldaux + col;
  if (col + 8 <= p.N && vec_aux) {
    const uint4 t = *reinterpret_cast<const uint4*>(ap);
    a[0] = t.x; a[1] = t.y; a[2] = t.z; a[3] = t.w;
  } else {
    const uint16_t* ah = reinterpret_cast<const uint16_t*>(ap);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const uint32_t lo = col + 2 * k < p.N ? ah[2 * k] : 0u;
      const uint32_t hi = col + 2 * k + 1 < p.N ? ah[2 * k + 1] : 0u;
      a[k] = lo | (hi << 16);
    }
  }
}

// 16-bit epilogues: 8 consecutive columns col .. col+7 of one row, v[k] = T(acc + bias) of columns col+2k, col+2k+1,
// a = their aux (load_aux_16x8) for the epilogues that read it
template <typename T, int EPI>
__device__ __forceinline__ void store_16x8(const GemmParams& p, int row, int col, const uint32_t (&v)[4],
                                           const uint32_t (&a)[4], bool vec_c) {
  const bool full = col + 8 <= p.N;
  using A = Act16<T>;
  uint32_t o[4], g[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    o[k] = v[k];
    if constexpr (EPI == OASR_EPI_BF16_GELU) {   // h = bf16(acc + b), g = bf16(gelu(h))
      const float2 x = gelu_erf2(A::unpack2(v[k]));
      g[k] = A::pack2(x.x, x.y);
    } else if constexpr (EPI == OASR_EPI_BF16_RESIDUAL) {   // C = bf16(aux + bf16(acc + b))
      const float2 x = fadd2(A::unpack2(a[k]), A::unpack2(v[k]));
      o[k] = A::pack2(x.x, x.y);
    } else if constexpr (EPI == OASR_EPI_BF16_GELU_BWD) {   // C = bf16(bf16(acc) * gelu'(aux))
      const float2 x = fmul2(A::unpack2(v[k]), gelu_erf_grad2(A::unpack2(a[k])));
      o[k] = A::pack2(x.x, x.y);
    }
  }
  const int64_t off = static_cast<int64_t>(row) * p.ldc + col;
#pragma unroll
  for (int out = 0; out < (EPI == OASR_EPI_BF16_GELU ? 2 : 1); ++out) {
    const uint32_t* src = out ? g : o;
    T* dst = reinterpret_cast<T*>(out ? p.C2 : p.C) + off;
    if (full && vec_c) {
      *reinterpret_cast<uint4*>(dst) = make_uint4(src[0], src[1], src[2], src[3]);
    } else {
      uint16_t* dh = reinterpret_cast<uint16_t*>(dst);
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        if (col + 2 * k < p.N) dh[2 * k] = static_cast<uint16_t>(src[k]);
        if (col + 2 * k + 1 < p.N) dh[2 * k + 1] = static_cast<uint16_t>(src[k] >> 16);
      }
    }
  }
}

template <typename T, int BN, int A_MN, int B_MN, int EPI>
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
    ptx::setmaxnreg_dec<PRODUCER_REGS>();
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
  const bool vec_c = is_f32_epi(EPI) ? ((p.ldc & 1) == 0 && (reinterpret_cast<uintptr_t>(p.C) & 7) == 0)
                                     : ((p.ldc & 7) == 0 && (reinterpret_cast<uintptr_t>(p.C) & 15) == 0 &&
                                        (p.C2 == nullptr || (reinterpret_cast<uintptr_t>(p.C2) & 15) == 0));
  const bool vec_aux = (p.ldaux & 7) == 0 && (reinterpret_cast<uintptr_t>(p.aux) & 15) == 0;

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
        const uint64_t da = ptx::desc_add(ad, k * a_kstep), db = ptx::desc_add(bd, k * b_kstep);
        if constexpr (BN == 256) ptx::wgmma_m64n256k16_ss<A_MN, B_MN, T>(acc, da, db, accumulate);
        else if constexpr (BN == 128) ptx::wgmma_m64n128k16_ss<A_MN, B_MN, T>(acc, da, db, accumulate);
        else ptx::wgmma_m64n64k16_ss<A_MN, B_MN, T>(acc, da, db, accumulate);
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
    const int ncol0 = n_blk * BN;
    if constexpr (is_f32_epi(EPI)) {
      const int col0 = ncol0 + 2 * (lane & 3);
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
      // T(acc + T(bias)) per column pair, then a quad transpose so that each lane stores 8 consecutive columns.  The
      // bias and aux loads of 128 columns are issued together before any of their arithmetic and stores: one round trip
      // to memory per 128 columns instead of one per 32 (a store may alias a later aux load, so the compiler cannot
      // hoist those loads itself).  Loading before storing keeps the in-place residual right: every element is read and
      // written by the same thread.  (Whole 256-column rows at once measured no faster, and slower on the tied logits.)
      constexpr int JC = BN / 32 < 4 ? BN / 32 : 4;   // 32-column steps per chunk
#pragma unroll
      for (int j0 = 0; j0 < BN / 32; j0 += JC) {
        if (ncol0 + 32 * j0 >= p.N) break;
        float b[JC][4][2];
        uint32_t a[JC][2][4];
#pragma unroll
        for (int jj = 0; jj < JC; ++jj) {
          const int j = j0 + jj;
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const int col = ncol0 + 8 * (4 * j + k) + 2 * (lane & 3);
            b[jj][k][0] = b[jj][k][1] = 0.f;
            if (p.bias != nullptr) {   // rounded to T like bias.to(x.dtype)
              if (col < p.N) b[jj][k][0] = Act16<T>::round(__ldg(p.bias + col));
              if (col + 1 < p.N) b[jj][k][1] = Act16<T>::round(__ldg(p.bias + col + 1));
            }
          }
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            a[jj][h][0] = a[jj][h][1] = a[jj][h][2] = a[jj][h][3] = 0u;
            if constexpr (reads_aux(EPI)) {
              const int row = row0 + 8 * h, col = ncol0 + 32 * j + 8 * (lane & 3);
              if (row < p.M && col < p.N) load_aux_16x8<T>(p, row, col, a[jj][h], vec_aux);
            }
          }
        }
#pragma unroll
        for (int jj = 0; jj < JC; ++jj) {
          const int j = j0 + jj;
          if (ncol0 + 32 * j >= p.N) break;   // warp-uniform: the quad shuffles below need every lane
          uint32_t w[2][4];
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const int i = 4 * j + k;
#pragma unroll
            for (int h = 0; h < 2; ++h)
              w[h][k] = Act16<T>::pack2(__fadd_rn(acc[4 * i + 2 * h], b[jj][k][0]),
                                        __fadd_rn(acc[4 * i + 2 * h + 1], b[jj][k][1]));
          }
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            uint32_t v[4];
            quad_transpose(w[h], v, lane);
            const int row = row0 + 8 * h;
            if (row < p.M) store_16x8<T, EPI>(p, row, ncol0 + 32 * j + 8 * (lane & 3), v, a[jj][h], vec_c);
          }
        }
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

template <typename T, int BN, int A_MN, int B_MN, int EPI>
int launch(const CUtensorMap& tmA, const CUtensorMap& tmB, const GemmParams& p, cudaStream_t st) {
  using C = Cfg<BN>;
  auto kern = gemm_wgmma_kernel<T, BN, A_MN, B_MN, EPI>;
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

// The (operand majors, epilogue) pairs the library calls; each is compiled for every tile width:
//   A K-major,  B K-major  (forward Linear / Conv1d, tied logits): BF16, BF16_GELU, BF16_RESIDUAL, BF16_GELU_BWD, F32
//   A K-major,  B MN-major (dgrad, logits dx):                     BF16, BF16_RESIDUAL, BF16_GELU_BWD, F32
//   A MN-major, B MN-major (wgrad):                                F32, F32_ATOMIC_ADD
// (split-K launches store fp32 partials: they run the F32 kernel).  Any other pair is rejected.
template <typename T, int BN>
int dispatch(int a_mn, int b_mn, int epi, const CUtensorMap& tmA, const CUtensorMap& tmB, const GemmParams& p, cudaStream_t st) {
  if (!a_mn && !b_mn) {
    switch (epi) {
      case OASR_EPI_BF16: return launch<T, BN, 0, 0, OASR_EPI_BF16>(tmA, tmB, p, st);
      case OASR_EPI_BF16_GELU: return launch<T, BN, 0, 0, OASR_EPI_BF16_GELU>(tmA, tmB, p, st);
      case OASR_EPI_BF16_RESIDUAL: return launch<T, BN, 0, 0, OASR_EPI_BF16_RESIDUAL>(tmA, tmB, p, st);
      case OASR_EPI_BF16_GELU_BWD: return launch<T, BN, 0, 0, OASR_EPI_BF16_GELU_BWD>(tmA, tmB, p, st);
      case OASR_EPI_F32: return launch<T, BN, 0, 0, OASR_EPI_F32>(tmA, tmB, p, st);
    }
  } else if (!a_mn && b_mn) {
    switch (epi) {
      case OASR_EPI_BF16: return launch<T, BN, 0, 1, OASR_EPI_BF16>(tmA, tmB, p, st);
      case OASR_EPI_BF16_RESIDUAL: return launch<T, BN, 0, 1, OASR_EPI_BF16_RESIDUAL>(tmA, tmB, p, st);
      case OASR_EPI_BF16_GELU_BWD: return launch<T, BN, 0, 1, OASR_EPI_BF16_GELU_BWD>(tmA, tmB, p, st);
      case OASR_EPI_F32: return launch<T, BN, 0, 1, OASR_EPI_F32>(tmA, tmB, p, st);
    }
  } else if (a_mn && b_mn) {
    switch (epi) {
      case OASR_EPI_F32: return launch<T, BN, 1, 1, OASR_EPI_F32>(tmA, tmB, p, st);
      case OASR_EPI_F32_ATOMIC_ADD: return launch<T, BN, 1, 1, OASR_EPI_F32_ATOMIC_ADD>(tmA, tmB, p, st);
    }
  }
  set_last_error("gemm: no kernel for a_layout=%d b_layout=%d epilogue=%d", a_mn, b_mn, epi);
  return OASR_ERR_UNSUPPORTED;
}

template <typename T>
int gemm(const void* A, int64_t lda, int a_layout, const void* B, int64_t ldb, int b_layout, void* Cout, int64_t ldc,
         void* C2, const float* bias, const void* aux, int64_t ldaux, int64_t M, int64_t N, int64_t K, int epilogue,
         int split_k, int block_n, void* stream) {
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
  p.split_stride = 0;

  CUtensorMap tmA, tmB;
  constexpr bool f16 = Act16<T>::is_fp16;
  int rc;
  if (a_layout == OASR_K_MAJOR)
    rc = make_tmap_2d(&tmA, A, 2, (uint64_t)K, (uint64_t)M, (uint64_t)lda * 2, BK, BM, true, f16);
  else
    rc = make_tmap_2d(&tmA, A, 2, (uint64_t)M, (uint64_t)K, (uint64_t)lda * 2, 64, BK, true, f16);
  if (rc) return rc;
  if (b_layout == OASR_K_MAJOR)
    rc = make_tmap_2d(&tmB, B, 2, (uint64_t)K, (uint64_t)N, (uint64_t)ldb * 2, BK, block_n, true, f16);
  else
    rc = make_tmap_2d(&tmB, B, 2, (uint64_t)N, (uint64_t)K, (uint64_t)ldb * 2, 64, BK, true, f16);
  if (rc) return rc;

  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  float* ws = nullptr;
  if (p.splits > 1) {   // every split stores its partial product; one more launch adds them to C in split order
    ws = static_cast<float*>(scratch_alloc(sizeof(float) * p.splits * M * N, st));
    if (!ws) return OASR_ERR_CUDA;
    p.C = ws; p.ldc = N; epilogue = OASR_EPI_F32; p.split_stride = M * N;
  }
  rc = block_n == 256 ? dispatch<T, 256>(a_layout, b_layout, epilogue, tmA, tmB, p, st)
     : block_n == 128 ? dispatch<T, 128>(a_layout, b_layout, epilogue, tmA, tmB, p, st)
                      : dispatch<T, 64>(a_layout, b_layout, epilogue, tmA, tmB, p, st);
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

}  // namespace
}  // namespace oasr

using namespace oasr;

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
