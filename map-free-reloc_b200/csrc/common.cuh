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

#include "../../include/mfr_b200.h"   // MFR_OK, MFR_ERR_*

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
// mbar_wait_inl with the trap after the spin loop rather than inside it, for warp-specialised kernels: a trap inside the
// loop makes ptxas allocate the whole kernel at the launch-bounds register count (168 at 384 threads), ignoring the
// consumers' setmaxnreg.inc
__device__ __forceinline__ void wait_bounded(uint32_t bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  bool ok;
  while (!(ok = mbar_try_wait(bar, parity)) && clock64() - t0 <= MFR_SPIN_TIMEOUT_CYCLES) {
  }
  if (!ok) __trap();
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

// ---------------------------------------------------------------------------------------------
// TMA (tiled mode) : shared -> global, bulk async-group completion
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* tm, uint32_t src, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(tm)),
               "r"(src), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// the shared-memory sources of every committed store have been read (the buffer may be refilled)
__device__ __forceinline__ void tma_store_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
// every committed store has completed
__device__ __forceinline__ void tma_store_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// named barrier over `count` threads (a multiple of 32); id 0 is __syncthreads
__device__ __forceinline__ void named_bar_sync(int id, int count) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}

// byte address of the 2-byte element (row, col) in a 128B-swizzled stack of 64-column k-blocks, kb_bytes apart (the
// TMA / wgmma layout: 128-byte rows whose 16-byte chunks are permuted by row % 8; base 1 KB aligned)
__device__ __forceinline__ uint32_t sw_addr(uint32_t base, int row, int col, uint32_t kb_bytes) {
  const int c64 = col & 63;
  return base + static_cast<uint32_t>((col >> 6) * kb_bytes + row * 128 + (((c64 >> 3) ^ (row & 7)) << 4) + (c64 & 7) * 2);
}

// 8x8 b16 matrices between registers and shared memory in the mma fragment layout (lane l: row l / 4, columns
// 2 (l % 4) + {0, 1} of matrix i in register i); lanes 8i .. 8i + 7 give the row addresses of matrix i
__device__ __forceinline__ void stsm_x4(uint32_t addr, uint32_t r0, uint32_t r1, uint32_t r2, uint32_t r3) {
  asm volatile("stmatrix.sync.aligned.m8n8.x4.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(r0), "r"(r1), "r"(r2),
               "r"(r3)
               : "memory");
}
__device__ __forceinline__ void stsm_x2(uint32_t addr, uint32_t r0, uint32_t r1) {
  asm volatile("stmatrix.sync.aligned.m8n8.x2.shared.b16 [%0], {%1, %2};" ::"r"(addr), "r"(r0), "r"(r1) : "memory");
}
__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(addr)
               : "memory");
}
__device__ __forceinline__ void ldsm_x2(uint32_t addr, uint32_t& r0, uint32_t& r1) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x2.shared.b16 {%0, %1}, [%2];" : "=r"(r0), "=r"(r1) : "r"(addr) : "memory");
}

}  // namespace mfr
