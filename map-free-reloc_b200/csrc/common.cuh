// Shared device/host helpers for the mfr_b200 CUDA library (sm_90a).
//
// PTX wrappers for the Hopper async machinery used by the tensor-core kernels: mbarrier and TMA
// (cp.async.bulk.tensor); the warpgroup MMA wrappers are in wgmma.cuh.
// Everything here is hand-written inline PTX; no CUTLASS/CuTe types are used.
#pragma once

#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#define MFR_OK 0
#define MFR_ERR_CUDA 1
#define MFR_ERR_ARG 2
#define MFR_ERR_UNSUPPORTED 3

#define MFR_CUDA_CHECK(expr)                                                         \
  do {                                                                               \
    cudaError_t _e = (expr);                                                         \
    if (_e != cudaSuccess) {                                                         \
      fprintf(stderr, "[mfr_b200] CUDA error %s at %s:%d: %s\n", cudaGetErrorName(_e), \
              __FILE__, __LINE__, cudaGetErrorString(_e));                           \
      return MFR_ERR_CUDA;                                                           \
    }                                                                                \
  } while (0)

// Kernel attributes (dynamic shared-memory opt-in) are per device: true the first time a call site runs on the
// current device. `seen` is the call site's own static table.
inline bool first_call_on_device(bool (&seen)[64]) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return true;
  if (seen[dev]) return false;
  seen[dev] = true;
  return true;
}

namespace mfr {

// SMs of the current device (launch-size heuristics); 132 (H100 SXM) when no device can be queried
inline int sm_count() {
  static int sms = 0;
  if (sms == 0) {
    int dev = 0, n = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return 132;
    sms = n;
  }
  return sms;
}

// ---------------------------------------------------------------------------------------------
// generic
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31u; }

// A kernel that hangs on a barrier would burn the whole GPU lease; every spin loop is bounded
// (~2 s of SM clocks) and traps with a message instead.
#ifndef MFR_SPIN_TIMEOUT_CYCLES
#define MFR_SPIN_TIMEOUT_CYCLES (4000000000LL)
#endif

// ---------------------------------------------------------------------------------------------
// mbarrier
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred P1;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%1], %2;\n"
      "selp.u32 %0, 1, 0, P1;\n"
      "}\n"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
// Slow path kept out of line so that the waits inside the single-thread TMA / MMA issue loops stay a
// handful of instructions (those loops are instruction-issue bound).
static __device__ __noinline__ void mbar_wait_slow(uint32_t bar, uint32_t parity, int tag) {
  long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > MFR_SPIN_TIMEOUT_CYCLES) {
      printf("[mfr_b200] mbarrier timeout: block %d thread %d tag %d parity %u\n", blockIdx.x,
             threadIdx.x, tag, parity);
      __trap();
    }
  }
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity, int tag = 0) {
  if (mbar_try_wait(bar, parity)) return;
  mbar_wait_slow(bar, parity, tag);
}
// Barrier wait for kernels that issue wgmma: spin loop inlined and without printf. Any function call (mbar_wait's
// out-of-line slow path, vprintf) in such a kernel makes ptxas serialise the wgmma pipeline. A wait that exceeds the
// bound traps (`tag` names the wait site for a debugger).
__device__ __forceinline__ void mbar_wait_inl(uint32_t bar, uint32_t parity, int tag) {
  (void)tag;
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity))
    if (clock64() - t0 > MFR_SPIN_TIMEOUT_CYCLES) __trap();
}

// One lane of a converged warp (elect.sync): lets ptxas emit a single UTMALDG instead of the
// per-active-thread loop it wraps around uniform-datapath instructions in divergent code.
__device__ __forceinline__ bool elect_one_sync() {
  uint32_t pred;
  asm volatile(
      "{\n"
      ".reg .pred P1;\n"
      "elect.sync _|P1, 0xffffffff;\n"
      "selp.u32 %0, 1, 0, P1;\n"
      "}\n"
      : "=r"(pred));
  return pred != 0;
}

// ---------------------------------------------------------------------------------------------
// TMA (tiled mode) : global -> shared, completion on an mbarrier
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* tm) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tm)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* tm, uint32_t bar,
                                            int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4}], [%2];" ::"r"(dst),
      "l"(reinterpret_cast<uint64_t>(tm)), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* tm, uint32_t bar,
                                            int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(dst),
      "l"(reinterpret_cast<uint64_t>(tm)), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* tm, uint32_t bar,
                                            int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(dst),
      "l"(reinterpret_cast<uint64_t>(tm)), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

}  // namespace mfr
