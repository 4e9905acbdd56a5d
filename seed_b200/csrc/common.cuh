// common.cuh -- shared host/device helpers for libseedb200 (sm_90a, H100).
//
// Device side: thin inline-PTX wrappers for the Hopper primitives the kernels
// use (mbarrier, TMA bulk-tensor loads, programmatic dependent launch).
// Host side: error plumbing for the C ABI (no exceptions cross it).
#pragma once

#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/seedb200.h"

namespace sb {

// ----------------------------------------------------------------------------
// host-side error handling
// ----------------------------------------------------------------------------
void set_error(const char* fmt, ...);
void count_launch(int n = 1);

#define SB_CHECK_CUDA(expr)                                                              \
  do {                                                                                   \
    cudaError_t _e = (expr);                                                             \
    if (_e != cudaSuccess) {                                                             \
      sb::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__,    \
                    __LINE__);                                                           \
      (void)cudaGetLastError(); /* reported: do not leave it for an unrelated later launch check */ \
      return SEEDB200_ERR_CUDA;                                                          \
    }                                                                                    \
  } while (0)

#define SB_REQUIRE(cond, ...)                                                            \
  do {                                                                                   \
    if (!(cond)) {                                                                       \
      sb::set_error(__VA_ARGS__);                                                        \
      return SEEDB200_ERR_INVALID;                                                       \
    }                                                                                    \
  } while (0)

#define SB_LAUNCH_CHECK()                                                                \
  do {                                                                                   \
    sb::count_launch();                                                                  \
    SB_CHECK_CUDA(cudaGetLastError());                                                   \
  } while (0)

#define SB_PROPAGATE(expr)                                                               \
  do {                                                                                   \
    int _s = (expr);                                                                     \
    if (_s != 0) return _s;                                                              \
  } while (0)

constexpr int SB_MAX_DEVICES = 64;
int cur_device();     // cudaGetDevice(), clamped to [0, SB_MAX_DEVICES)
int num_sms();        // of the current device
// A handle lives on the device that was current at *_create; every handle-level entry point runs under this guard,
// so a caller whose current device differs (reference pattern: tokenizer_device != llm_device in one process,
// gradio_demo/seed_llama_flask.py:51-52,69,78) still launches next to the handle's weights and workspace.
struct DeviceGuard {
  int prev; bool switched;
  explicit DeviceGuard(int dev) : prev(0), switched(false) {
    if (cudaGetDevice(&prev) == cudaSuccess && prev != dev) switched = cudaSetDevice(dev) == cudaSuccess;
  }
  ~DeviceGuard() { if (switched) cudaSetDevice(prev); }
};

// Programmatic dependent launch (decode chain): a kernel launched through launch_chain() while a PdlScope is active
// may start while its predecessor is still running; it must execute pdl_wait() before touching anything the
// predecessor writes, and everything it does earlier (weight prefetch) overlaps the predecessor's tail and the
// launch gap.  Outside a PdlScope launch_chain() is a plain launch and pdl_wait()/pdl_trigger() are no-ops.
bool pdl_scope_active();
void pdl_scope_set(bool on);
struct PdlScope {
  bool prev;
  explicit PdlScope(bool on) : prev(pdl_scope_active()) { pdl_scope_set(on); }
  ~PdlScope() { pdl_scope_set(prev); }
};

// per-kernel event timing (seedb200_profile_begin/end); no-ops unless enabled on this thread
bool profile_enabled();
void profile_mark_begin(int kind, cudaStream_t stream);
void profile_mark_end(int kind, cudaStream_t stream, double flops);

#ifdef __CUDACC__
template <typename... KArgs, typename... Args>
inline cudaError_t launch_chain(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                                Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  if (pdl_scope_active()) {
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr; cfg.numAttrs = 1;
  }
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

// ----------------------------------------------------------------------------
// device helpers
// ----------------------------------------------------------------------------
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---- mbarrier ---------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
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
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded waits: a protocol bug traps (kernel error) instead of hanging the GPU.  The deadline is checked once every
// 4096 polls only, so that the wait loops do not take issue slots from the warps doing work.
#ifndef SB_MBAR_TIMEOUT_CYCLES
#define SB_MBAR_TIMEOUT_CYCLES (8000000000LL)
#endif
// try_wait that lets the hardware park the thread for up to `ns` nanoseconds before it reports "not yet"
__device__ __forceinline__ bool mbar_try_wait_hint(uint32_t bar, uint32_t parity, uint32_t ns) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(ok)
      : "r"(bar), "r"(parity), "r"(ns)
      : "memory");
  return ok != 0;
}
static __device__ __noinline__ void mbar_timeout_trap(uint32_t bar, uint32_t parity) {
  printf("seedb200: mbarrier timeout block %d thread %d bar 0x%x parity %u\n", blockIdx.x, threadIdx.x, bar, parity);
  __trap();
}
// latency-critical waits: plain polling, deadline check amortised
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  uint32_t polls = 0;
  while (!mbar_try_wait(bar, parity)) {
    if ((++polls & 4095u) == 0 && clock64() - t0 > SB_MBAR_TIMEOUT_CYCLES) mbar_timeout_trap(bar, parity);
  }
}

// waits that are expected to be long (the TMA producer waiting for a free buffer):
// the thread is parked by the hardware (suspend-time hint) instead of spinning, so it neither steals issue slots from
// the warps doing work nor burns power polling.
__device__ __forceinline__ void mbar_wait_relaxed(uint32_t bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  uint32_t polls = 0;
  while (!mbar_try_wait_hint(bar, parity, 2000u)) {
    if ((++polls & 255u) == 0 && clock64() - t0 > SB_MBAR_TIMEOUT_CYCLES) mbar_timeout_trap(bar, parity);
  }
}

// ---- TMA --------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const void* tmap) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tmap)) : "memory");
}
// 2-D tiled load global -> local smem, completion on a local mbarrier
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const void* tmap, uint32_t bar, int32_t c0,
                                            int32_t c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, "
      "%4}], [%2];" ::"r"(dst),
      "l"(reinterpret_cast<uint64_t>(tmap)), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
#endif  // __CUDACC__

}  // namespace sb
