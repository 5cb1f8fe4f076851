// sm_90a PTX wrappers shared by the SAM-Audio kernels:
// mbarrier, TMA (cp.async.bulk.tensor), wgmma fences and shared-memory descriptors, small math helpers.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda.h>
#include <stdint.h>

namespace sab {

#define SAB_DEVICE __device__ __forceinline__

SAB_DEVICE uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ----------------------------------------------------------------------------- mbarrier
SAB_DEVICE void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
SAB_DEVICE void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

SAB_DEVICE void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
SAB_DEVICE void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
SAB_DEVICE bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.b32 %0, 1, 0, p;\n\t}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
SAB_DEVICE void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}

// ----------------------------------------------------------------------------- TMA
SAB_DEVICE void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
SAB_DEVICE void tma_load_2d(void* smem, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(smem)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
SAB_DEVICE void tma_load_3d(void* smem, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(smem)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}

// ----------------------------------------------------------------------------- wgmma
// Order this thread's register / shared-memory writes before the warpgroup's next wgmma.mma_async.
SAB_DEVICE void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
SAB_DEVICE void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int kPending>
SAB_DEVICE void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(kPending) : "memory"); }
// keep registers an asynchronous wgmma reads or writes where they are until the wgmma has retired
template <int N>
SAB_DEVICE void reg_fence(float (&r)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(r[i])::"memory");
}
template <int N>
SAB_DEVICE void reg_fence(uint32_t (&r)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+r"(r[i])::"memory");
}

// generic-proxy shared-memory writes -> reads by the async proxy (wgmma operands, TMA stores)
SAB_DEVICE void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// barrier over a subset of the CTA's warps (ids 1..15; 0 is __syncthreads)
SAB_DEVICE void named_bar_sync(int id, int threads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory"); }

// Shared-memory matrix descriptor (sm_90 GMMA) for a K-major bf16 tile whose rows are kRowBytes wide
// (kRowBytes = 128 -> SWIZZLE_128B, 64 -> SWIZZLE_64B) as written by a TMA box of that inner extent;
// 8-row core-matrix groups are kRowBytes*8 apart (SBO).  Fields: start[0,14) lbo[16,30) sbo[32,46)
// layout_type[62,64) (1 = 128B, 2 = 64B, 3 = 32B swizzle).  Advancing 16 bf16 along K inside the swizzle row
// adds 2 to the start field.
template <int kRowBytes>
SAB_DEVICE uint64_t make_kmajor_desc(uint32_t smem_addr) {
  constexpr uint64_t layout = (kRowBytes == 128) ? 1ull : (kRowBytes == 64 ? 2ull : 3ull);
  constexpr uint64_t sbo = (uint64_t)(kRowBytes * 8) >> 4;
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);
  d |= (uint64_t)1 << 16;   // LBO: unused for swizzled K-major (one swizzle atom along K); canonical value 1
  d |= sbo << 32;
  d |= layout << 62;
  return d;
}
// MN-major SWIZZLE_128B descriptor: 64-element (128 B) chunks along MN are `lbo` bytes apart, 8-row groups along K
// are `sbo` bytes apart.
SAB_DEVICE uint64_t make_mnmajor_desc(uint32_t smem_addr, uint32_t lbo, uint32_t sbo) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);
  d |= (uint64_t)((lbo >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo >> 4) & 0x3FFF) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}

// explicit shared-window accesses (a pointer carved out of `extern __shared__` by byte arithmetic is a generic
// pointer to the compiler: it would emit LD.E/ST.E with an address-space check instead of LDS/STS)
SAB_DEVICE void sts128(uint32_t addr, float4 v) {
  asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
SAB_DEVICE void sts128u(uint32_t addr, uint4 v) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
SAB_DEVICE float4 lds128(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr) : "memory");
  return v;
}

// ----------------------------------------------------------------------------- math / packing
// 16-byte global load that does not allocate in L1 (streamed once; plain ld.global, so in-place updates stay coherent)
SAB_DEVICE float4 ldg_stream128(const float* p) {
  float4 v;
  asm volatile("ld.global.L1::no_allocate.v4.f32 {%0, %1, %2, %3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
  return v;
}
SAB_DEVICE float rcp_approx(float x) {   // one MUFU.RCP (<= 1 ulp), no IEEE-division slow path
  float r;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}
// x * sigmoid(x), branch-free (6 instructions; the IEEE division was ~20 with a slow-path branch per element and made up
// about half of the instructions the ffn.w13 kernel issued); exp(-x) = inf gives rcp = +0 and the exact limit -0
SAB_DEVICE float silu_f(float x) { return x * rcp_approx(1.f + __expf(-x)); }
SAB_DEVICE uint32_t pack_bf16(float a, float b) {
  __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}
SAB_DEVICE float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
SAB_DEVICE float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

}  // namespace sab
