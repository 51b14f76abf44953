// distrifuser_b200 -- shared device/host helpers (sm_90a only).
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/distrifuser_b200.h"

namespace df {

// SMs of the H100 SXM the grid-size heuristics are tuned for (kernels that size a persistent grid query the device)
constexpr int kSmCount = 132;
// SMs of the current device, queried once (kSmCount if the query fails)
int sm_count();

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
// cuTensorMapEncodeTiled of the driver, looked up once (nullptr if the driver does not provide it)
EncodeTiledFn tensor_map_encoder();

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
constexpr uint64_t kSpinTimeoutNs = 30000000000ull;  // a peer that never arrives becomes a CUDA error, not a hung GPU
// kReport = false drops the printf before the trap: a kernel that issues wgmma must contain no function call (printf is one),
// or ptxas serialises every wgmma of the kernel (warning C7510).
template <bool kReport = true>
__device__ __forceinline__ void spin_until(const uint32_t* flag, uint32_t want, uint64_t timeout_ns = 0) {
  if (epoch_reached(ld_acquire_sys(flag), want)) return;
  if (timeout_ns == 0) timeout_ns = kSpinTimeoutNs;
  const uint64_t t0 = globaltimer_ns();
  uint32_t polls = 0;
  while (!epoch_reached(ld_acquire_sys(flag), want)) {
    __nanosleep(64);
    if ((++polls & 1023u) == 0 && globaltimer_ns() - t0 > timeout_ns) {
      if constexpr (kReport)
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

// ------------------------------------------------------------------ cross-rank protocol (include/distrifuser_b200.h: arena layout)
// A writer stores into slot(epoch, idx, src = its rank) of the readers' arenas, then stamps flags[idx*world + src] = epoch on
// each reader (release, system scope); a reader acquires that flag before it reads the slot.

// byte offset of slot(epoch, tensor, src) in every member's arena
__host__ __device__ __forceinline__ uint64_t slot_offset(const df_comm_t& c, uint32_t epoch, uint64_t tensor_off,
                                                         uint64_t slot_bytes, int src) {
  return (uint64_t)(epoch % DF_NBANKS) * c.bank_stride + tensor_off + (uint64_t)src * slot_bytes;
}
__host__ __device__ __forceinline__ char* slot_ptr(const df_comm_t& c, int rank, uint32_t epoch, uint64_t tensor_off,
                                                   uint64_t slot_bytes, int src) {
  return (char*)c.base[rank] + slot_offset(c, epoch, tensor_off, slot_bytes, src);
}

// flag word of tensor `idx` and source `src` in the flag array of `member`
__device__ __forceinline__ uint32_t* flag_ptr(const df_comm_t& c, int member, int idx, int src) {
  return c.flags[member] + (size_t)idx * c.world + src;
}

// stamps this rank's flag of tensor `idx` with `epoch` at the members in `mask` (the caller has fenced its slot stores); a CTA
// may share the members out: the calling thread takes members first, first + step, ...
__device__ __forceinline__ void stamp_flags(const df_comm_t& c, int idx, uint32_t mask, uint32_t epoch, int first = 0, int step = 1) {
  for (int p = first; p < c.world; p += step)
    if (mask >> p & 1) st_release_sys(flag_ptr(c, p, idx, c.rank), epoch);
}

// the CTA waits until this rank's flags of tensor `idx` from every source in `mask` reached `epoch` (thread s waits on source s)
__device__ __forceinline__ void wait_sources(const df_comm_t& c, int idx, uint32_t mask, uint32_t epoch) {
  const int s = threadIdx.x;
  if (s < c.world && (mask >> s & 1)) spin_until(flag_ptr(c, c.rank, idx, s), epoch, c.spin_timeout_ns);
  __syncthreads();
}

// member mask of the patch neighbours of a halo exchange (-1: image border)
__device__ __forceinline__ uint32_t neighbour_mask(int up, int down) {
  return (up >= 0 ? 1u << up : 0u) | (down >= 0 ? 1u << down : 0u);
}

// Called by every thread of each of the `nctas` CTAs of a grid after its slot stores: the last CTA to take a ticket resets the
// counter (the next launch that uses it is stream-ordered after this one) and stamps the flags of `mask`.
__device__ __forceinline__ void signal_when_last(const df_comm_t& c, unsigned int* ticket, unsigned int nctas, int idx,
                                                 uint32_t mask, uint32_t epoch) {
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0) {
    if (atomicAdd(ticket, 1u) == nctas - 1) {
      __threadfence();
      *ticket = 0;
      stamp_flags(c, idx, mask, epoch);
    }
  }
}

}  // namespace df
