// distrifuser_b200 -- symmetric arena, epoch clock, activation publication over NVLink peer memory,
// final epsilon gather.  Replaces PatchParallelismCommManager (distrifuser/utils.py:112-199) and the
// blocking collectives of the pp modules (attn.py:133, conv2d.py:93, distri_sdxl_unet_pp.py:166,191).
#include <stdarg.h>
#include <string.h>

#include "common.cuh"

namespace df {
static thread_local char g_err[1024] = "";
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
}  // namespace df

using namespace df;

extern "C" const char* df_last_error(void) { return df::g_err; }
extern "C" int df_version(void) { return 2; }
extern "C" int df_device_sm_count(int* out) {
  int dev = 0;
  DF_CHECK_CUDA(cudaGetDevice(&dev));
  DF_CHECK_CUDA(cudaDeviceGetAttribute(out, cudaDevAttrMultiProcessorCount, dev));
  return 0;
}

int df::sm_count() {
  static int sms = 0;
  if (!sms && (df_device_sm_count(&sms) != 0 || sms <= 0)) sms = kSmCount;
  return sms;
}

EncodeTiledFn df::tensor_map_encoder() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = (EncodeTiledFn)p;
  }
  return fn;
}

// ------------------------------------------------------------------------------------ symmetric memory
extern "C" int df_symm_alloc(size_t bytes, void** dptr, void* ipc_handle_out_host) {
  DF_REQUIRE(dptr != nullptr && bytes > 0, "df_symm_alloc: bad arguments");
  static_assert(sizeof(cudaIpcMemHandle_t) == DF_IPC_HANDLE_BYTES, "ipc handle size");
  // >= 4 MiB and a multiple of 2 MiB: the allocation then owns its VA block, so the pointer a peer gets from
  // cudaIpcOpenMemHandle is this base and not the base of a shared small-allocation block.
  const size_t gran = 2u << 20;
  size_t rounded = ((bytes + gran - 1) / gran) * gran;
  if (rounded < 2 * gran) rounded = 2 * gran;
  void* p = nullptr;
  DF_CHECK_CUDA(cudaMalloc(&p, rounded));
  DF_CHECK_CUDA(cudaMemset(p, 0, rounded));
  DF_CHECK_CUDA(cudaDeviceSynchronize());
  if (ipc_handle_out_host) {
    cudaIpcMemHandle_t h;
    DF_CHECK_CUDA(cudaIpcGetMemHandle(&h, p));
    memcpy(ipc_handle_out_host, &h, sizeof(h));
  }
  *dptr = p;
  return 0;
}

extern "C" int df_symm_open(const void* ipc_handle_host, void** peer_dptr) {
  DF_REQUIRE(ipc_handle_host && peer_dptr, "df_symm_open: bad arguments");
  cudaIpcMemHandle_t h;
  memcpy(&h, ipc_handle_host, sizeof(h));
  DF_CHECK_CUDA(cudaIpcOpenMemHandle(peer_dptr, h, cudaIpcMemLazyEnablePeerAccess));
  return 0;
}
extern "C" int df_symm_close(void* peer_dptr) {
  DF_CHECK_CUDA(cudaIpcCloseMemHandle(peer_dptr));
  return 0;
}
extern "C" int df_symm_free(void* dptr) {
  DF_CHECK_CUDA(cudaFree(dptr));
  return 0;
}

// ------------------------------------------------------------------------------------ epoch clock
__global__ void step_begin_kernel(uint32_t* clock, int kind) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    uint32_t pub = clock[0];
    if (kind == 0) { pub += 1; clock[0] = pub; clock[1] = pub; }
    else if (kind == 1) { clock[1] = pub; clock[0] = pub + 1; }
    clock[2] += 1;  // output-gather epoch: advances on every UNet call
  }
}
extern "C" int df_step_begin(uint32_t* clock, int kind, void* stream) {
  DF_REQUIRE(clock && kind >= 0 && kind <= 2, "df_step_begin: bad arguments");
  step_begin_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(clock, kind);
  DF_CHECK_LAUNCH();
  return 0;
}

// ------------------------------------------------------------------------------------ publication
// One load, `npeer` stores per 16-byte vector; the last CTA to finish stamps the peers' flags.
// 128 threads, kPubUnroll 16-byte loads in flight per thread: the transfer is bound by how many loads are outstanding (local
// read latency ~1 us; the peer stores are posted).  What is exposed is the tail of the step's last publications, so a faster
// transfer wins over taking fewer SM slots.
constexpr int kPubUnroll = 8;
__global__ void __launch_bounds__(128, 8) publish_kernel(df_comm_t c, const char* __restrict__ src, uint64_t rows,
                                                          uint64_t vec_per_row, uint64_t src_pitch, uint64_t tensor_off,
                                                          uint64_t slot_bytes, int idx, uint32_t peer_mask) {
  const uint32_t epoch = c.clock[0];
  const uint64_t total = rows * vec_per_row;
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  const uint64_t slot_off = slot_offset(c, epoch, tensor_off, slot_bytes, c.rank);
  constexpr int U = kPubUnroll;
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  for (; i + (U - 1) * stride < total; i += U * stride) {
    int4 v[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const uint64_t j = i + u * stride;
      uint64_t soff = j * 16;                                      // contiguous source (rows == 1)
      if (rows > 1) { const uint32_t r = (uint32_t)j / (uint32_t)vec_per_row; soff = (uint64_t)r * src_pitch + (uint64_t)((uint32_t)j - r * (uint32_t)vec_per_row) * 16; }
      v[u] = ld_nc_v4(src + soff);
    }
    for (int p = 0; p < c.world; ++p) {
      if (!(peer_mask >> p & 1)) continue;
      char* dst = (char*)c.base[p] + slot_off;
#pragma unroll
      for (int u = 0; u < U; ++u) st_v4(dst + (i + u * stride) * 16, v[u]);
    }
  }
  for (; i < total; i += stride) {
    uint64_t soff = i * 16;
    if (rows > 1) { const uint32_t r = (uint32_t)i / (uint32_t)vec_per_row; soff = (uint64_t)r * src_pitch + (uint64_t)((uint32_t)i - r * (uint32_t)vec_per_row) * 16; }
    int4 v = ld_nc_v4(src + soff);
    for (int p = 0; p < c.world; ++p)
      if (peer_mask >> p & 1) st_v4((char*)c.base[p] + slot_off + i * 16, v);
  }
  signal_when_last(c, &c.tickets[idx], gridDim.x, idx, peer_mask, epoch);
}

extern "C" int df_slot_publish(df_comm_t comm, const void* src, uint64_t rows, uint64_t row_bytes, uint64_t src_pitch,
                               uint64_t tensor_off, uint64_t slot_bytes, int idx, uint32_t peer_mask, int num_ctas,
                               void* stream) {
  DF_REQUIRE(row_bytes % 16 == 0 && ((uintptr_t)src % 16) == 0 && src_pitch % 16 == 0,
             "df_slot_publish: rows must be 16-byte aligned (row_bytes=%llu)", (unsigned long long)row_bytes);
  DF_REQUIRE(rows * row_bytes <= slot_bytes, "df_slot_publish: payload larger than the slot");
  DF_REQUIRE(rows * (row_bytes / 16) < (1ull << 31), "df_slot_publish: payload too large for 32-bit row arithmetic");
  if (peer_mask == 0) return 0;
  uint64_t total = rows * (row_bytes / 16);
  int grid = num_ctas > 0 ? num_ctas : 64;
  uint64_t need = (total + 127) / 128;
  if ((uint64_t)grid > need) grid = (int)(need ? need : 1);
  publish_kernel<<<grid, 128, 0, (cudaStream_t)stream>>>(comm, (const char*)src, rows, row_bytes / 16, src_pitch,
                                                         tensor_off, slot_bytes, idx, peer_mask);
  DF_CHECK_LAUNCH();
  return 0;
}

__global__ void wait_kernel(df_comm_t c, int idx, uint32_t src_mask) { wait_sources(c, idx, src_mask, c.clock[1]); }
extern "C" int df_slot_wait(df_comm_t comm, int idx, uint32_t src_mask, void* stream) {
  if (src_mask == 0) return 0;
  wait_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(comm, idx, src_mask);
  DF_CHECK_LAUNCH();
  return 0;
}

// ------------------------------------------------------------------------------------ final epsilon gather
// Each (batch, channel) plane of the strip is `rows` runs of `vpr` vectors; run r lands at row row0 + r, column col0 of the
// image plane.  A full-width strip is one run of hs*W elements (rows = 1), so it vectorises whenever hs*W does.  V: the access
// (a 16-byte vector or one element), ES: the element size in bytes.
template <typename V, int ES>
__global__ void __launch_bounds__(256) out_scatter_kernel(df_comm_t c, const V* __restrict__ strip, int C, int H, int W,
                                                          int bs, int rows, int vpr, int batch0, int row0, int col0, int idx,
                                                          uint64_t tensor_off, uint32_t world_mask) {
  const uint32_t epoch = c.clock[2];
  constexpr int E = sizeof(V) / ES;
  const int plane = rows * vpr;                    // vectors per (batch, channel) plane of the strip
  const int64_t total = (int64_t)bs * C * plane;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t bc = i / plane;
    int q = (int)(i - bc * plane);
    int r = q / vpr;
    q -= r * vpr;
    int bb = (int)(bc / C), ch = (int)(bc - (int64_t)bb * C);
    V v = strip[i];
    int64_t dst_el = (((int64_t)(batch0 + bb) * C + ch) * H + row0 + r) * W + col0 + (int64_t)q * E;
    for (int p = 0; p < c.world; ++p) {
      V* d = (V*)(slot_ptr(c, p, epoch, tensor_off, 0, 0) + dst_el * ES);
      *d = v;
    }
  }
  signal_when_last(c, &c.tickets[idx], gridDim.x, idx, world_mask, epoch);
}

template <typename V>
__global__ void __launch_bounds__(256) out_collect_kernel(df_comm_t c, V* __restrict__ out, int64_t total_vec, int idx,
                                                          uint64_t tensor_off) {
  const uint32_t epoch = c.clock[2];
  wait_sources(c, idx, 0xffffffffu, epoch);
  const V* src = (const V*)slot_ptr(c, c.rank, epoch, tensor_off, 0, 0);
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total_vec; i += (int64_t)gridDim.x * blockDim.x)
    out[i] = src[i];
}

// Scatter of a strip made of bs*C planes of `rows` runs of `run` elements of T, then the collect of the whole image.
// `vec_shape`: the runs and their destinations are whole 16-byte vectors.
template <typename T>
static int output_gather(df_comm_t comm, const void* strip, void* out, int B, int C, int H, int W, int bs, int rows, int run,
                         int batch0, int row0, int col0, bool vec_shape, int idx, uint64_t tensor_off, void* stream) {
  constexpr int ES = sizeof(T), E = 16 / ES;
  uint32_t mask = comm.world >= 32 ? 0xffffffffu : ((1u << comm.world) - 1u);
  int64_t strip_el = (int64_t)bs * C * rows * run, total_el = (int64_t)B * C * H * W;
  bool vec = vec_shape && ((uintptr_t)strip % 16) == 0 && ((uintptr_t)out % 16) == 0 && tensor_off % 16 == 0;
  cudaStream_t st = (cudaStream_t)stream;
  if (vec) {
    int g1 = (int)((strip_el / E + 255) / 256); g1 = g1 < 1 ? 1 : (g1 > 64 ? 64 : g1);
    out_scatter_kernel<int4, ES><<<g1, 256, 0, st>>>(comm, (const int4*)strip, C, H, W, bs, rows, run / E, batch0, row0, col0,
                                                     idx, tensor_off, mask);
    DF_CHECK_LAUNCH();
    int g2 = (int)((total_el / E + 255) / 256); g2 = g2 < 1 ? 1 : (g2 > 64 ? 64 : g2);
    out_collect_kernel<int4><<<g2, 256, 0, st>>>(comm, (int4*)out, total_el / E, idx, tensor_off);
    DF_CHECK_LAUNCH();
  } else {
    int g1 = (int)((strip_el + 255) / 256); g1 = g1 < 1 ? 1 : (g1 > 64 ? 64 : g1);
    out_scatter_kernel<T, ES><<<g1, 256, 0, st>>>(comm, (const T*)strip, C, H, W, bs, rows, run, batch0, row0, col0, idx,
                                                  tensor_off, mask);
    DF_CHECK_LAUNCH();
    int g2 = (int)((total_el + 255) / 256); g2 = g2 < 1 ? 1 : (g2 > 64 ? 64 : g2);
    out_collect_kernel<T><<<g2, 256, 0, st>>>(comm, (T*)out, total_el, idx, tensor_off);
    DF_CHECK_LAUNCH();
  }
  return 0;
}

// A full-width strip is one run per plane; it takes the 16-byte path only when every plane's run starts on a vector (the image
// plane H*W and the strip's offset row0*W are whole vectors) and is whole vectors long.
static bool full_width_vec(int H, int W, int hs, int row0, int E) {
  return (int64_t)hs * W % E == 0 && (int64_t)row0 * W % E == 0 && (int64_t)H * W % E == 0;
}

extern "C" int df_output_gather(df_comm_t comm, const void* strip, void* out, int B, int C, int H, int W, int bs, int hs,
                                int batch0, int row0, int idx, uint64_t tensor_off, void* stream) {
  DF_REQUIRE(batch0 + bs <= B && row0 + hs <= H, "df_output_gather: strip outside the image");
  return output_gather<__half>(comm, strip, out, B, C, H, W, bs, 1, hs * W, batch0, row0, 0, full_width_vec(H, W, hs, row0, 8), idx,
                               tensor_off, stream);
}

template <typename T>
static int output_gather_2d(df_comm_t comm, const void* strip, void* out, int B, int C, int H, int W, int bs, int hs, int ws,
                            int batch0, int row0, int col0, int idx, uint64_t tensor_off, void* stream) {
  constexpr int E = 16 / sizeof(T);
  DF_REQUIRE(bs > 0 && hs > 0 && ws > 0 && batch0 >= 0 && row0 >= 0 && col0 >= 0,
             "df_output_gather_2d: bad strip (bs=%d hs=%d ws=%d at %d,%d,%d)", bs, hs, ws, batch0, row0, col0);
  DF_REQUIRE(batch0 + bs <= B && row0 + hs <= H && col0 + ws <= W, "df_output_gather_2d: strip outside the image");
  if (ws == W)                                      // full-width strip: one contiguous run per plane, as df_output_gather
    return output_gather<T>(comm, strip, out, B, C, H, W, bs, 1, hs * W, batch0, row0, 0, full_width_vec(H, W, hs, row0, E), idx,
                            tensor_off, stream);
  return output_gather<T>(comm, strip, out, B, C, H, W, bs, hs, ws, batch0, row0, col0, ws % E == 0 && col0 % E == 0 && W % E == 0,
                          idx, tensor_off, stream);
}

extern "C" int df_output_gather_2d_dtype(df_comm_t comm, const void* strip, void* out, int B, int C, int H, int W, int bs, int hs,
                                         int ws, int batch0, int row0, int col0, int idx, uint64_t tensor_off, int dtype,
                                         void* stream) {
  DF_REQUIRE(dtype == DF_F16 || dtype == DF_F32, "df_output_gather_2d: unknown element type %d", dtype);
  return (dtype == DF_F32 ? output_gather_2d<float> : output_gather_2d<__half>)(comm, strip, out, B, C, H, W, bs, hs, ws, batch0,
                                                                                row0, col0, idx, tensor_off, stream);
}

extern "C" int df_output_gather_2d(df_comm_t comm, const void* strip, void* out, int B, int C, int H, int W, int bs, int hs,
                                   int ws, int batch0, int row0, int col0, int idx, uint64_t tensor_off, void* stream) {
  return df_output_gather_2d_dtype(comm, strip, out, B, C, H, W, bs, hs, ws, batch0, row0, col0, idx, tensor_off, DF_F16, stream);
}
