// Thin inline-PTX wrappers for the sm_90a features this library uses:
// mbarrier, TMA (cp.async.bulk.tensor) and warpgroup MMA (wgmma.mma_async) with its shared-memory descriptors.
//
// Descriptor bit layouts follow the PTX ISA "Matrix Descriptor Format" table for wgmma
// (the same layout CUTLASS documents in cute/arch/mma_sm90_desc.hpp).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>

#include <type_traits>

namespace oasr {
namespace ptx {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// shared-memory accesses by 32-bit address (a generic pointer costs two registers)
__device__ __forceinline__ uint32_t ld_shared_u32(uint32_t a) {
  uint32_t v;
  asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(a) : "memory");
  return v;
}
__device__ __forceinline__ float2 ld_shared_f32x2(uint32_t a) {
  float2 v;
  asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(a) : "memory");
  return v;
}
__device__ __forceinline__ void st_shared_u32(uint32_t a, uint32_t v) {
  asm volatile("st.shared.b32 [%0], %1;" ::"r"(a), "r"(v) : "memory");
}

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
// generic-proxy writes (st.shared) -> visible to the async proxy (TMA stores / wgmma operand reads)
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug must surface as a CUDA error, never as a hung GPU.
// ~4 s at 2 GHz before the trap.  (No printf here: a call inside a wgmma loop makes ptxas serialise the MMAs.)
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > 8000000000LL) __trap();
  }
}

// Warpgroup-wide register reallocation (counts are multiples of 8 in 24..256; every warp of the warpgroup executes it)
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }

// ---------------------------------------------------------------- TMA
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t smem_dst, const CUtensorMap* m, uint32_t bar,
                                            int32_t c0, int32_t c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_dst), "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}
// TMA store of one box (the source must be published to the async proxy first: fence_proxy_async_smem).  Stores
// issued by a thread join its current bulk group; commit closes the group.  Boxes are clipped at the map's bounds.
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* m, uint32_t smem_src, int32_t c0, int32_t c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(m)), "r"(smem_src), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void bulk_commit_group() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// at most N of this thread's bulk groups still read their shared-memory source
template <int N>
__device__ __forceinline__ void bulk_wait_group_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
// at most N of this thread's bulk groups are still incomplete (writes visible in global memory)
template <int N>
__device__ __forceinline__ void bulk_wait_group() {
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}
// barrier over `count` threads (a multiple of 32) with id 1..15 (0 is __syncthreads)
__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t count) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}

// ---------------------------------------------------------------- wgmma
// A warpgroup (4 consecutive, 4-aligned warps) issues one 64 x N x 16 MMA.  Accumulator fragment of thread t
// (warp w = t / 32, lane l): d[4i + {0,1}] = row 16w + l/4, columns 8i + 2(l%4) + {0,1}; d[4i + {2,3}] = row + 8.
// A register fragment (bf16x2 words) for k-step kk is the accumulator layout of columns 16kk .. 16kk+15:
// {d[8kk], d[8kk+1]}, {d[8kk+2], d[8kk+3]}, {d[8kk+4], d[8kk+5]}, {d[8kk+6], d[8kk+7]}.
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from touching accumulator registers across the asynchronous MMA window
template <int N>
__device__ __forceinline__ void fence_regs(float (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// Shared-memory matrix descriptor (64 bit), 128-byte swizzle (tiles 1024-byte aligned):
//   [0,14)  start address >> 4      [16,30) leading byte offset >> 4
//   [32,46) stride byte offset >> 4 [62,64) layout (1 = 128 B swizzle)
// K-major operand: rows of 64 bf16 (128 B), 8-row groups SBO = 1024 B apart, LBO unused; a 16-wide k-step adds 32 B.
// MN-major operand: rows of 64 MN-elements per k, 64-element MN chunks LBO apart, 8-k groups SBO = 1024 B apart;
// a 16-deep k-step adds 2048 B.
__device__ __forceinline__ uint64_t desc_sw128(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((saddr & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}
// the start address field is the low 14 bits: adding (bytes >> 4) advances the operand by `bytes`
__device__ __forceinline__ uint64_t desc_add(uint64_t d, uint32_t bytes) { return d + (bytes >> 4); }

// D (+)= A * B, A and B from shared memory; TA / TB = 1: operand is MN-major.  T (bf16 or fp16) is the type of both
// operands; the descriptors, swizzles and transpose bits are the same for the two 16-bit types.
#define OASR_WGMMA_SS(N, TY, REGS, DOUT, P, A, B, TA, TB)                                                   \
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %" P ", 0;\n\t"                                    \
               "wgmma.mma_async.sync.aligned.m64n" #N "k16.f32." TY "." TY " " REGS ", %" A ", %" B           \
               ", p, 1, 1, %" TA ", %" TB ";\n\t}"                                                            \
               : DOUT : "l"(da), "l"(db), "r"(acc), "n"(TA_), "n"(TB_))
#define OASR_R32 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}"
#define OASR_D32 "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
#define OASR_R64 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}"
#define OASR_D64 "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
#define OASR_R128 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}"
#define OASR_D128 "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
template <int TA_, int TB_, typename T = __nv_bfloat16>
__device__ __forceinline__ void wgmma_m64n64k16_ss(float (&d)[32], uint64_t da, uint64_t db, uint32_t acc) {
  if constexpr (std::is_same<T, __half>::value)
    OASR_WGMMA_SS(64, "f16", OASR_R32, OASR_D32, "34", "32", "33", "35", "36");
  else
    OASR_WGMMA_SS(64, "bf16", OASR_R32, OASR_D32, "34", "32", "33", "35", "36");
}
template <int TA_, int TB_, typename T = __nv_bfloat16>
__device__ __forceinline__ void wgmma_m64n128k16_ss(float (&d)[64], uint64_t da, uint64_t db, uint32_t acc) {
  if constexpr (std::is_same<T, __half>::value)
    OASR_WGMMA_SS(128, "f16", OASR_R64, OASR_D64, "66", "64", "65", "67", "68");
  else
    OASR_WGMMA_SS(128, "bf16", OASR_R64, OASR_D64, "66", "64", "65", "67", "68");
}
template <int TA_, int TB_, typename T = __nv_bfloat16>
__device__ __forceinline__ void wgmma_m64n256k16_ss(float (&d)[128], uint64_t da, uint64_t db, uint32_t acc) {
  if constexpr (std::is_same<T, __half>::value)
    OASR_WGMMA_SS(256, "f16", OASR_R128, OASR_D128, "130", "128", "129", "131", "132");
  else
    OASR_WGMMA_SS(256, "bf16", OASR_R128, OASR_D128, "130", "128", "129", "131", "132");
}
// D (+)= A * B, A from registers (the fragment layout above, T x 2 words), B from shared memory
#define OASR_WGMMA_RS64(TY)                                                                                  \
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"                                        \
               "wgmma.mma_async.sync.aligned.m64n64k16.f32." TY "." TY " " OASR_R32 ", "                     \
               "{%32, %33, %34, %35}, %36, p, 1, 1, %38;\n\t}"                                               \
               : OASR_D32 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(acc), "n"(TB))
template <int TB, typename T = __nv_bfloat16>
__device__ __forceinline__ void wgmma_m64n64k16_rs(float (&d)[32], const uint32_t (&a)[4], uint64_t db, uint32_t acc) {
  if constexpr (std::is_same<T, __half>::value)
    OASR_WGMMA_RS64("f16");
  else
    OASR_WGMMA_RS64("bf16");
}
#undef OASR_WGMMA_RS64
// FP8: D (+)= A * B over k = 32, both operands K-major from shared memory (wgmma has no transpose for 8-bit types).
// F8 = 1: e4m3 x e4m3, F8 = 2: e5m2 (A) x e4m3 (B).  A 32-deep k-step is 32 bytes, like a 16-deep 16-bit one.
#define OASR_WGMMA_F8(N, TA, TB, REGS, DOUT, P, A, B)                                                        \
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %" P ", 0;\n\t"                                    \
               "wgmma.mma_async.sync.aligned.m64n" #N "k32.f32." TA "." TB " " REGS ", %" A ", %" B ", p, 1, 1;\n\t}" \
               : DOUT : "l"(da), "l"(db), "r"(acc))
template <int F8>
__device__ __forceinline__ void wgmma_m64n64k32_f8(float (&d)[32], uint64_t da, uint64_t db, uint32_t acc) {
  static_assert(F8 == 1 || F8 == 2, "wgmma fp8: F8 is 1 (e4m3.e4m3) or 2 (e5m2.e4m3)");
  if constexpr (F8 == 1)
    OASR_WGMMA_F8(64, "e4m3", "e4m3", OASR_R32, OASR_D32, "34", "32", "33");
  else
    OASR_WGMMA_F8(64, "e5m2", "e4m3", OASR_R32, OASR_D32, "34", "32", "33");
}
template <int F8>
__device__ __forceinline__ void wgmma_m64n128k32_f8(float (&d)[64], uint64_t da, uint64_t db, uint32_t acc) {
  static_assert(F8 == 1 || F8 == 2, "wgmma fp8: F8 is 1 (e4m3.e4m3) or 2 (e5m2.e4m3)");
  if constexpr (F8 == 1)
    OASR_WGMMA_F8(128, "e4m3", "e4m3", OASR_R64, OASR_D64, "66", "64", "65");
  else
    OASR_WGMMA_F8(128, "e5m2", "e4m3", OASR_R64, OASR_D64, "66", "64", "65");
}
#undef OASR_WGMMA_F8
#undef OASR_WGMMA_SS
#undef OASR_R32
#undef OASR_R64
#undef OASR_R128
#undef OASR_D32
#undef OASR_D64
#undef OASR_D128
}  // namespace ptx
}  // namespace oasr
