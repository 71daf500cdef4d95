// pyg_lib_b200/csrc/hopper_ptx.cuh — the hand-written PTX the tensor-core kernels of this library are built from on
// sm_90a (mbarrier, TMA tiled loads, wgmma.mma_async and its shared-memory matrix descriptors).  Include inside
// namespace pygb200 { namespace { ... } } of a .cu file that has already included <cuda.h>, <cuda_bf16.h>, <cuda_fp16.h>
// and "common.cuh" (no system header is pulled in from here, so the include is safe inside a namespace).
#pragma once

// ---------------------------------------------------------------------------------- PTX helpers
__device__ __forceinline__ u32 smem_u32(const void* p) { return (u32)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(u32 bar, u32 count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(u32 bar, u32 bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(u32 bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(u32 bar, u32 parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_LOOP:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE;\n"
      "bra WAIT_LOOP;\n"
      "DONE:\n"
      "}\n" ::"r"(bar), "r"(parity)
      : "memory");
}
__device__ __forceinline__ void tma_load_2d(u32 dst, const CUtensorMap* map, int c0, int c1, u32 bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(dst),
      "l"(map), "r"(c0), "r"(c1), "r"(bar)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(u32 dst, const CUtensorMap* map, int c0, int c1, int c2, u32 bar) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];" ::"r"(dst),
      "l"(map), "r"(c0), "r"(c1), "r"(c2), "r"(bar)
      : "memory");
}
// generic-proxy stores to shared memory (zeroed tails) must be fenced before wgmma reads them through the async proxy
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// a tensor map that was written to global memory through the generic proxy (the host's copy) must be fenced into the
// tensormap proxy before the TMA unit reads it
__device__ __forceinline__ void fence_tensormap(const CUtensorMap* map) {
  asm volatile("fence.proxy.tensormap::generic.acquire.sys [%0], 128;" ::"l"(map) : "memory");
}
__device__ __forceinline__ void named_bar(int id, int threads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory"); }

// ---------------------------------------------------------------------------------- wgmma
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

#define PYGB_WG_D64                                                                       \
  "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "              \
  "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "     \
  "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "     \
  "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}"
#define PYGB_WG_D64_OPS(d)                                                                                       \
  "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),               \
  "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),         \
  "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),       \
  "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),       \
  "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),       \
  "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),       \
  "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),       \
  "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])

// D[64 x 128] (fp32 m64n128 register fragment of one warpgroup) += A[64 x 16] * B[16 x 128].  TA / TB = 1: that
// operand is stored MN-major (transposed); only the 16-bit kinds can transpose.
template <bool BF16, int TA, int TB>
__device__ __forceinline__ void wgmma_16(float (&d)[64], u64 da, u64 db) {
  if (BF16)
    asm volatile("wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 " PYGB_WG_D64 ", %64, %65, 1, 1, 1, %66, %67;"
                 : PYGB_WG_D64_OPS(d)
                 : "l"(da), "l"(db), "n"(TA), "n"(TB));
  else
    asm volatile("wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 " PYGB_WG_D64 ", %64, %65, 1, 1, 1, %66, %67;"
                 : PYGB_WG_D64_OPS(d)
                 : "l"(da), "l"(db), "n"(TA), "n"(TB));
}
// D[64 x 128] += A[64 x 8] * B[8 x 128] with TF32 inputs (both operands K-major)
__device__ __forceinline__ void wgmma_tf32(float (&d)[64], u64 da, u64 db) {
  asm volatile("wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 " PYGB_WG_D64 ", %64, %65, 1, 1, 1;"
               : PYGB_WG_D64_OPS(d)
               : "l"(da), "l"(db));
}

// sm_90 shared-memory matrix descriptor (cute/arch/mma_sm90_desc.hpp GmmaDescriptor bit layout):
// [0,14) start>>4 | [16,30) LBO>>4 | [32,46) SBO>>4 | [49,52) base offset (0: swizzle atoms are 1024-byte aligned) |
// [62,64) layout (1 = SWIZZLE_128B).  K-major: SBO = stride of 8-row groups (LBO unused).  MN-major: LBO = stride of
// 64-element groups along M / N, SBO = stride of 8-row groups along K.
__device__ __forceinline__ u64 make_desc(u32 saddr, u32 lbo_bytes, u32 sbo_bytes) {
  u64 d = 0;
  d |= (u64)((saddr & 0x3ffffu) >> 4);
  d |= (u64)((lbo_bytes >> 4) & 0x3fffu) << 16;
  d |= (u64)((sbo_bytes >> 4) & 0x3fffu) << 32;
  d |= (u64)1 << 62;
  return d;
}

template <bool BF16>
__device__ __forceinline__ u32 pack2(float a, float b) {
  if (BF16) {
    __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<u32*>(&h);
  } else {
    __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<u32*>(&h);
  }
}
template <bool BF16>
__device__ __forceinline__ float ld_bias(const void* bias, i64 idx) {
  if (BF16) return __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(bias)[idx]);
  return __half2float(reinterpret_cast<const __half*>(bias)[idx]);
}
