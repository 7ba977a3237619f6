// Thin wrappers over the sm_90 PTX used by the scan pipeline:
// mbarrier (init / expect_tx / try_wait.parity / arrive) and 1-D bulk async copy
// (cp.async.bulk global -> shared, SASS UBLKCP) completing on an mbarrier.
// On the host: set_attribute_once, e.g. to let a kernel use more than 48 KB of dynamic shared memory.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>

namespace kge {

// cudaFuncSetAttribute(KERNEL, attr, value) on the current device, once per (attribute, device
// ordinal): a function attribute is a per-device property, and each caller always passes the same
// value for a given kernel and attribute.  Ordinals of 64 and above set it on every call.  Launchers
// run from several host threads at once, hence the atomic record.
template <auto KERNEL>
inline cudaError_t set_attribute_once(cudaFuncAttribute attr, int value) {
  static std::atomic<uint64_t> done[cudaFuncAttributeMax] = {};   // [attr]: bit d set on device d
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  const bool known = attr >= 0 && attr < cudaFuncAttributeMax && dev >= 0 && dev < 64;
  if (known && ((done[attr].load(std::memory_order_acquire) >> dev) & 1u)) return cudaSuccess;
  e = cudaFuncSetAttribute(KERNEL, attr, value);
  if (e == cudaSuccess && known) done[attr].fetch_or(1ull << dev, std::memory_order_release);
  return e;
}

namespace ptx {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}

__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}

__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}

__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}

__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t"
      "}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}

__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}

// global -> shared bulk copy of `bytes` (multiple of 16, both sides 16-B aligned); the
// mbarrier receives complete_tx(bytes) when the data has landed.
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes,
                                         uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
      ::"r"(smem_u32(smem_dst)),
      "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}

}  // namespace ptx
}  // namespace kge
