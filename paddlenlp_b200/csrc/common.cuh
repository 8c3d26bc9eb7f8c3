// Device-side primitives for sm_90a: mbarrier, TMA (cp.async.bulk.tensor), wgmma, mma.sync / ldmatrix, cp.async,
// plus small vector / bf16 helpers shared by every kernel in this directory.
//
// Everything here is inline PTX; there is no CUTLASS/CuTe dependency.  The wgmma descriptor layout follows the
// PTX ISA "matrix descriptor" table for sm_90.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

namespace b200 {

typedef __nv_bfloat16 bf16;

// ------------------------------------------------------------------------------------------------
// misc
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// Programmatic dependent launch (PDL).  A kernel launched with the programmatic-stream-serialization attribute may start
// while its predecessor is still running: it must execute pdl_wait() before its first access to data the predecessor
// produces (or overwrites).  pdl_launch_dependents() lets the NEXT kernel in the stream begin launching early; it is
// harmless when that kernel was launched without the attribute.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// ------------------------------------------------------------------------------------------------
// mbarrier
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a barrier that never flips (a protocol bug) traps after ~4 s instead of hanging the GPU.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  long long t0 = clock64();
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if ((++spins & 0x3FFu) == 0 && (clock64() - t0) > 8000000000LL) {
      printf("[b200 watchdog] mbarrier wait timed out: block %d thread %d bar 0x%x parity %u\n", (int)blockIdx.x,
             (int)threadIdx.x, smem_u32(bar), parity);
      __trap();
    }
  }
}
// The same bounded wait without the printf.  For kernels that issue wgmma: a function call in a loop that keeps accumulators
// live makes ptxas save them around it (local-memory spills), and a call anywhere in the kernel, the producer branch included,
// makes it wait for each wgmma before it issues the next (ptxas info C7510).
__device__ __forceinline__ void mbar_wait_nocall(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  long long t0 = clock64();
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if ((++spins & 0x3FFu) == 0 && (clock64() - t0) > 8000000000LL) __trap();
  }
}

// ------------------------------------------------------------------------------------------------
// TMA
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* tm) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tm)) : "memory");
}
// global -> shared, 2D tile, completion on an mbarrier in this CTA.
__device__ __forceinline__ void tma_load_2d(const CUtensorMap* tm, uint64_t* bar, void* smem_dst, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(tm)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
// Contiguous global -> shared copy by the bulk-copy (TMA) engine, completion on an mbarrier in this CTA; 16-byte aligned,
// `bytes` a multiple of 16.
__device__ __forceinline__ void bulk_load(void* smem_dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_dst)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
// global -> shared, 3D tile, completion on an mbarrier in this CTA.
__device__ __forceinline__ void tma_load_3d(const CUtensorMap* tm, uint64_t* bar, void* smem_dst, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(tm)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(const CUtensorMap* tm, uint64_t* bar, void* smem_dst, int c0, int c1,
                                            int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(tm)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2),
      "r"(c3)
      : "memory");
}
// shared -> global element-wise ADD (fp32 tensor map), 4D tile: the TMA unit performs the reduction in L2.
__device__ __forceinline__ void tma_reduce_add_4d(const CUtensorMap* tm, const void* smem_src, int c0, int c1, int c2,
                                                  int c3) {
  asm volatile("cp.reduce.async.bulk.tensor.4d.global.shared::cta.add.tile.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(tm)),
               "r"(smem_u32(smem_src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
// shared -> global element-wise ADD (fp32 tensor map), 2D tile (bulk-group completion); elements outside the tensor are not
// touched.  The reduction runs in L2 and flushes subnormal results to zero.
__device__ __forceinline__ void tma_reduce_add_2d(const CUtensorMap* tm, uint32_t smem_src, int c0, int c1) {
  asm volatile("cp.reduce.async.bulk.tensor.2d.global.shared::cta.add.tile.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(tm)),
               "r"(smem_src), "r"(c0), "r"(c1)
               : "memory");
}
// shared -> global, 2D tile (bulk-group completion); elements outside the tensor are not written.
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* tm, uint32_t smem_src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(reinterpret_cast<uint64_t>(tm)),
               "r"(smem_src), "r"(c0), "r"(c1)
               : "memory");
}
// Pull a 2D tile of a tensor map into L2 (no shared memory, no completion to wait for).
__device__ __forceinline__ void tma_prefetch_l2_2d(const CUtensorMap* tm, int c0, int c1) {
  asm volatile("cp.async.bulk.prefetch.tensor.2d.L2.global.tile [%0, {%1, %2}];" ::"l"(reinterpret_cast<uint64_t>(tm)), "r"(c0),
               "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void tma_store_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void tma_store_wait() {
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}

// Persistent-GEMM tile order: GM consecutive m-tiles share each n-tile column, so that concurrently running CTAs reuse
// A and B tiles out of L2.
__device__ __forceinline__ void tile_coords(int t, int num_m, int num_n, int& m_blk, int& n_blk, int GM) {
  const int per_group = GM * num_n;
  const int g = t / per_group;
  const int first_m = g * GM;
  const int gsize = min(GM, num_m - first_m);
  const int r = t - g * per_group;
  m_blk = first_m + (r % gsize);
  n_blk = r / gsize;
}

// ------------------------------------------------------------------------------------------------
// Hopper warpgroup MMA (wgmma.mma_async): operands in shared memory, fp32 accumulators in registers
// ------------------------------------------------------------------------------------------------
// 64-bit shared-memory matrix descriptor (sm_90), 128-byte swizzle.
//   start address  bits [0,14)   (>>4)
//   LBO            bits [16,30)  (>>4)   MN-major: byte distance between 64-element swizzle atoms along M/N
//   SBO            bits [32,46)  (>>4)   byte distance between groups of 8 rows (K-major) / 8 k (MN-major)
//   layout type    bits [62,64)  = 1 (SWIZZLE_128B)
__device__ __forceinline__ uint64_t wgmma_desc_sw128(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((saddr & 0x3FFFFu) >> 4);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFFu) << 16;
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFFu) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// Register budget of a warpgroup (warp-specialised kernels: the TMA producer gives registers to the MMA warpgroups).
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }

// d[64 x 256] (+)= A[64 x 16] * B[16 x 256], bf16 in, fp32 accumulate.  TA / TB: operand is MN-major (transposed).
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n256k16(float (&d)[128], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p, 1, 1, %131, %132;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(desc_a), "l"(desc_b), "r"(accumulate), "n"(TA), "n"(TB));
}
// d[64 x 64] (+)= A[64 x 16] * B[16 x 64], both operands in shared memory.
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n64k16(float (&d)[32], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, %35, %36;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(desc_a), "l"(desc_b), "r"(accumulate), "n"(TA), "n"(TB));
}
// d[64 x 128] (+)= A[64 x 16] * B[16 x 128], both operands in shared memory.
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n128k16(float (&d)[64], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, %67, %68;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(desc_a), "l"(desc_b), "r"(accumulate), "n"(TA), "n"(TB));
}
// d[64 x 128] (+)= A[64 x 16] * B[16 x 128]; A from registers: each warp holds its 16 rows as the mma.sync m16n8k16 A
// fragment (a[0..3], pack_bf16x2 pairs), B in shared memory (TB: MN-major).
template <int TB>
__device__ __forceinline__ void wgmma_m64n128k16_rs(float (&d)[64], const uint32_t* a, uint64_t desc_b, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %69, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, {%64, %65, %66, %67}, %68, p, 1, 1, %70;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b), "r"(accumulate), "n"(TB));
}
// d[64 x 64] (+)= A[64 x 16] * B[16 x 64]; A from registers as in wgmma_m64n128k16_rs.
template <int TB>
__device__ __forceinline__ void wgmma_m64n64k16_rs(float (&d)[32], const uint32_t* a, uint64_t desc_b, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1, %38;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b), "r"(accumulate), "n"(TB));
}

// ------------------------------------------------------------------------------------------------
// warp-level MMA (mma.sync m16n8k16, bf16 in, fp32 accumulate) and ldmatrix, for the attention kernels
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void mma_bf16_16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
      "{%0, %1, %2, %3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void ldsm_x4(uint32_t saddr, uint32_t (&r)[4]) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(saddr));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t saddr, uint32_t (&r)[4]) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(saddr));
}
// 16-byte global -> shared copy (cp.async, L2 only); src_bytes = 0 fills the destination with zeros.
__device__ __forceinline__ void cp_async_16(uint32_t saddr, const void* gptr, uint32_t src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(saddr), "l"(gptr), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// ------------------------------------------------------------------------------------------------
// bf16 / vector helpers
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float2 unpack_bf16x2(uint32_t u) {
  __nv_bfloat162 v = *reinterpret_cast<__nv_bfloat162*>(&u);
  return __bfloat1622float2(v);
}
__device__ __forceinline__ float bf16_round(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }

// NOT volatile: a read-only load has no side effects, and `asm volatile` statements are never reordered relative to
// each other, which serialises "load, compute, store" loops into one memory round trip per iteration.  Only use on data that
// no thread writes during the kernel.
__device__ __forceinline__ uint4 ld_nc_v4(const void* p) {
  uint4 r;
  asm("ld.global.nc.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}
// No "memory" clobber on purpose: a clobber pins every other load/store of the loop body around this store, which turns
// unrolled "load row i, compute, store row i" loops into one DRAM round trip per iteration (measured 24 us for a 64-row
// add_rmsnorm).  Only use for write-only outputs that the same kernel never reads back.
__device__ __forceinline__ void st_na_v4(void* p, const uint4& v) {
  asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1, %2, %3, %4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z),
               "r"(v.w));
}
// Ordered against other asm volatile statements (e.g. fence.proxy.async), but no "memory" clobber: global loads of the same
// loop may still be scheduled ahead of it.
__device__ __forceinline__ void st_shared_u32(uint32_t saddr, uint32_t v) {
  asm volatile("st.shared.u32 [%0], %1;" ::"r"(saddr), "r"(v));
}
__device__ __forceinline__ void st_shared_f32x2(uint32_t saddr, float a, float b) {
  asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(saddr), "f"(a), "f"(b));
}
__device__ __forceinline__ uint4 ld_shared_v4(uint32_t saddr) {
  uint4 r;
  asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "r"(saddr));
  return r;
}

// 2^x on the SFU (MUFU.EX2), flush-to-zero, no denormal fix-up code around it (exp2f() without fast-math expands to
// several instructions per call, which matters in the attention inner loops: 128x128 of them per tile).
__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float fast_rcp(float x) {
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// Pairs of fp32 operations with explicit round-to-nearest intrinsics: never re-associated or contracted by the compiler, so
// every kernel that uses them (and the fused GEMM epilogues) produces the same bits.
struct f32x2 { float x, y; };
__device__ __forceinline__ f32x2 f2_mul(f32x2 a, f32x2 b) { return f32x2{__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)}; }
__device__ __forceinline__ f32x2 f2_add(f32x2 a, f32x2 b) { return f32x2{__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)}; }
__device__ __forceinline__ f32x2 f2_fma(f32x2 a, f32x2 b, f32x2 c) {
  return f32x2{__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y)};
}

// SwiGLU forward for two adjacent channels (llama/modeling.py:38-45, 648-650): m = bf16(silu(g) * u) from the bf16-rounded gate and
// up projections.  sigmoid = rcp.approx(1 + ex2.approx(-g log2 e)) like the backward below (two SFU operations; an IEEE division
// plus expf costs ~35 instructions per element, which made the fused ffn1 epilogue of the decode step 6 us long).  The ONE
// definition used by b200_swiglu_fwd / _f32 and by the GEMM epilogue that fuses it (gemm_wgmma.cu mode 4): the operation order
// is pinned by the round-to-nearest intrinsics, so all of them produce the same bits.
__device__ __forceinline__ uint32_t swiglu_fwd_pair(uint32_t g2, uint32_t u2) {
  const float2 gf = unpack_bf16x2(g2), uf = unpack_bf16x2(u2);
  const f32x2 g{gf.x, gf.y}, u{uf.x, uf.y}, one{1.f, 1.f};
  const f32x2 t = f2_mul(g, f32x2{-1.4426950408889634f, -1.4426950408889634f});
  const f32x2 a = f2_add(f32x2{fast_exp2(t.x), fast_exp2(t.y)}, one);
  const f32x2 sg{fast_rcp(a.x), fast_rcp(a.y)};
  const f32x2 m = f2_mul(f2_mul(g, sg), u);
  return pack_bf16x2(m.x, m.y);
}

// SwiGLU backward for two adjacent channels (llama/modeling.py:632-652 swiglu, backward of silu(g) * u):
//   sg = sigmoid(g) ; d(gate) = d * u * sg * (1 + g (1 - sg)) ; d(up) = d * g * sg          (fp32, results rounded once to bf16)
// sigmoid = rcp.approx(1 + ex2.approx(-g log2 e)): two SFU operations (a few fp32 ulp, far inside the bf16 rounding of the
// outputs) instead of an IEEE division.  The ONE definition used by b200_swiglu_bwd and by the GEMM epilogue that fuses it
// (gemm_wgmma.cu mode 5): the operation order is pinned by the round-to-nearest intrinsics, so both produce the same bits.
__device__ __forceinline__ void swiglu_bwd_pair(uint32_t g2, uint32_t u2, float d0, float d1, uint32_t& dg2, uint32_t& du2) {
  const float2 gf = unpack_bf16x2(g2), uf = unpack_bf16x2(u2);
  const f32x2 g{gf.x, gf.y}, u{uf.x, uf.y}, d{d0, d1}, one{1.f, 1.f};
  const f32x2 t = f2_mul(g, f32x2{-1.4426950408889634f, -1.4426950408889634f});
  const f32x2 a = f2_add(f32x2{fast_exp2(t.x), fast_exp2(t.y)}, one);
  const f32x2 sg{fast_rcp(a.x), fast_rcp(a.y)};
  const f32x2 silu = f2_mul(g, sg);
  const f32x2 om = f2_fma(sg, f32x2{-1.f, -1.f}, one);           // 1 - sg
  const f32x2 ds = f2_mul(sg, f2_fma(g, om, one));               // sg (1 + g (1 - sg))
  const f32x2 dgv = f2_mul(f2_mul(d, u), ds);
  const f32x2 duv = f2_mul(d, silu);
  dg2 = pack_bf16x2(dgv.x, dgv.y);
  du2 = pack_bf16x2(duv.x, duv.y);
}

// RoPE (rotate-half, fp32 math, one rounding) of one 8-column chunk pair of a head at position pos: a holds columns j8 .. j8 + 7
// of the first half, b the same columns of the second half; cos / sin tables are fp32 [positions, half].
//   first half: x1 cos - x2 sin ; second half: x2 cos + x1 sin.  sign = -1 is the backward (sin -> -sin).
// The round-to-nearest intrinsics pin which product is fused into each FMA.  The training RoPE (rope_kernel) fuses x1 sin into
// the second half and the decode kernels fuse x2 cos; the two forms round differently, and FUSE_SIN keeps each caller's
// results bit for bit.
template <bool FUSE_SIN = false>
__device__ __forceinline__ void rope_rotate_chunk(uint4& a, uint4& b, const float* cos_t, const float* sin_t, int pos, int half,
                                                  int j8, float sign = 1.f) {
  const float4* c4 = reinterpret_cast<const float4*>(cos_t + static_cast<size_t>(pos) * half + j8);
  const float4* s4 = reinterpret_cast<const float4*>(sin_t + static_cast<size_t>(pos) * half + j8);
  const float4 c0 = __ldg(c4), c1 = __ldg(c4 + 1), s0 = __ldg(s4), s1 = __ldg(s4 + 1);
  const float cs[8] = {c0.x, c0.y, c0.z, c0.w, c1.x, c1.y, c1.z, c1.w};
  const float sn[8] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w};
  uint32_t* ai = reinterpret_cast<uint32_t*>(&a);
  uint32_t* bi = reinterpret_cast<uint32_t*>(&b);
  auto first = [](float x1, float x2, float c, float s) { return __fmaf_rn(x1, c, -__fmul_rn(x2, s)); };
  auto second = [](float x1, float x2, float c, float s) {
    return FUSE_SIN ? __fmaf_rn(x1, s, __fmul_rn(x2, c)) : __fmaf_rn(x2, c, __fmul_rn(x1, s));
  };
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float2 x1 = unpack_bf16x2(ai[j]), x2 = unpack_bf16x2(bi[j]);
    const float s_lo = sign * sn[2 * j], s_hi = sign * sn[2 * j + 1];
    ai[j] = pack_bf16x2(first(x1.x, x2.x, cs[2 * j], s_lo), first(x1.y, x2.y, cs[2 * j + 1], s_hi));
    bi[j] = pack_bf16x2(second(x1.x, x2.x, cs[2 * j], s_lo), second(x1.y, x2.y, cs[2 * j + 1], s_hi));
  }
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Split-KV partials of the decode-attention kernels (decode_attn_tc.cu), merged by
// decode_attention_merge_kernel: one row of DECODE_PART_ROW floats per (sequence, head, split) at every head_dim
// (b200_decode_attention_workspace_bytes takes no head_dim), the unnormalised o in the first d columns, the running max
// (log2 units) at column DECODE_PART_M and the sum at DECODE_PART_M + 1.  The 132-float stride keeps the merge kernel's
// vector reads 16-byte aligned.
constexpr int DECODE_PART_ROW = 132;
constexpr int DECODE_PART_M = 128;

}  // namespace b200
