// distrifuser_b200 -- shared device/host helpers (sm_90a only).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/distrifuser_b200.h"

namespace df {

// SMs of the H100 SXM the grid-size heuristics are tuned for (kernels that size a persistent grid query the device)
constexpr int kSmCount = 132;

void set_error(const char* fmt, ...);

#define DF_CHECK_CUDA(expr)                                                              \
  do {                                                                                   \
    cudaError_t _e = (expr);                                                             \
    if (_e != cudaSuccess) {                                                             \
      df::set_error("%s:%d %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
      return 1;                                                                          \
    }                                                                                    \
  } while (0)

#define DF_REQUIRE(cond, ...)        \
  do {                               \
    if (!(cond)) {                   \
      df::set_error(__VA_ARGS__);    \
      return 2;                      \
    }                                \
  } while (0)

#define DF_CHECK_LAUNCH() DF_CHECK_CUDA(cudaGetLastError())

// ------------------------------------------------------------------ system-scope flag primitives
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_volatile_u32(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.volatile.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
// epoch compare that survives wrap-around of the 32-bit clock
__device__ __forceinline__ bool epoch_reached(uint32_t flag, uint32_t want) { return (int32_t)(flag - want) >= 0; }

__device__ __forceinline__ uint64_t globaltimer_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}
#ifndef DF_SPIN_TIMEOUT_NS
#define DF_SPIN_TIMEOUT_NS 30000000000ull  // a peer that never arrives becomes a CUDA error, not a hung GPU
#endif
__device__ __forceinline__ void spin_until(const uint32_t* flag, uint32_t want, uint64_t timeout_ns = 0) {
  if (epoch_reached(ld_acquire_sys(flag), want)) return;
  if (timeout_ns == 0) timeout_ns = DF_SPIN_TIMEOUT_NS;
  const uint64_t t0 = globaltimer_ns();
  uint32_t polls = 0;
  while (!epoch_reached(ld_acquire_sys(flag), want)) {
    __nanosleep(64);
    if ((++polls & 1023u) == 0 && globaltimer_ns() - t0 > timeout_ns) {
      printf("distrifuser_b200: timeout waiting for flag %p (have %u, want %u)\n", (const void*)flag, ld_volatile_u32(flag), want);
      __trap();
    }
  }
}

// 16-byte streaming accesses (activations are touched once per kernel)
__device__ __forceinline__ int4 ld_nc_v4(const void* p) {
  int4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.s32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}
__device__ __forceinline__ int4 ld_v4(const void* p) {
  int4 r;
  asm volatile("ld.global.v4.s32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  return r;
}
__device__ __forceinline__ void st_v4(void* p, const int4& v) {
  asm volatile("st.global.v4.s32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

// ------------------------------------------------------------------ programmatic dependent launch (PDL)
// A denoise step is a chain of ~1 400 short kernels; with the launch attribute below a kernel of this library may be scheduled
// while its predecessor in the stream is still draining, run its prologue (barrier set-up, tensor-map prefetch, index
// arithmetic) and then block in pdl_wait() until the predecessor has completed and flushed its writes.  No global memory is
// read or written before pdl_wait().  Opt-in per kernel family with the DF_PDL bit mask (without the attribute the device-side wait
// is a no-op).
unsigned pdl_mask();   // DF_PDL bit mask: 1 attention, 2 add+LayerNorm / GEGLU, 4 GroupNorm, 8 GEMM (0 = off, default)
enum { PDL_ATTN = 1, PDL_ELEM = 2, PDL_GN = 4, PDL_GEMM = 8 };

__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(unsigned family, void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = (pdl_mask() & family) ? 1 : 0;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

__device__ __forceinline__ char* slot_ptr(const df_comm_t& c, int rank, uint32_t epoch, uint64_t tensor_off,
                                          uint64_t slot_bytes, int src) {
  return (char*)c.base[rank] + (uint64_t)(epoch % DF_NBANKS) * c.bank_stride + tensor_off + (uint64_t)src * slot_bytes;
}

}  // namespace df
