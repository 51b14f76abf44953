// distrifuser_b200 -- 3x3-conv halo exchange (NHWC fp16 or fp32, one halo row).
// Replaces the boundary torch.stack + all_gather over ALL ranks + cat/F.pad of DistriConv2dPP.forward
// (distrifuser/modules/pp/conv2d.py:72-93): rows travel to the two patch neighbours only, written straight
// into their arena slots with 16-byte peer stores, and the padded conv input is assembled by one coalesced
// vectorised kernel.
//
// Slot layout of tensor idx, source s:  [2][b][w*C] elements  -- part 0 = s's first row, part 1 = s's last row
// (the reference's buffer_list[s][0] / [s][1], conv2d.py:61-65,90).
#include "common.cuh"

using namespace df;

namespace {

__global__ void __launch_bounds__(256) halo_push_kernel(df_comm_t c, const char* __restrict__ x, int b, int h,
                                                        uint64_t row_vec, int idx, uint64_t tensor_off, uint64_t slot_bytes,
                                                        int up_rank, int down_rank) {
  const uint32_t epoch = c.clock[0];
  const uint64_t row_bytes = row_vec * 16;
  // part 0: my first row -> up neighbour (it is that rank's bottom halo); part 1: my last row -> down neighbour
  char* dst_up = up_rank >= 0 ? slot_ptr(c, up_rank, epoch, tensor_off, slot_bytes, c.rank) : nullptr;
  char* dst_dn = down_rank >= 0 ? slot_ptr(c, down_rank, epoch, tensor_off, slot_bytes, c.rank) + (uint64_t)b * row_bytes : nullptr;
  const uint64_t total = 2ull * b * row_vec;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (uint64_t)gridDim.x * blockDim.x) {
    uint64_t part = i / ((uint64_t)b * row_vec), r = i - part * b * row_vec;
    uint64_t bb = r / row_vec, q = r - bb * row_vec;
    char* dst = part == 0 ? dst_up : dst_dn;
    if (dst == nullptr) continue;
    uint64_t src_row = bb * h + (part == 0 ? 0 : h - 1);
    st_v4(dst + (bb * row_vec + q) * 16, ld_nc_v4(x + (src_row * row_vec + q) * 16));
  }
  signal_when_last(c, &c.tickets[idx], gridDim.x, idx, neighbour_mask(up_rank, down_rank), epoch);
}

__global__ void __launch_bounds__(256) halo_assemble_kernel(df_comm_t c, const char* __restrict__ x, char* __restrict__ xp,
                                                            int b, int h, uint64_t row_vec, int idx, uint64_t tensor_off,
                                                            uint64_t slot_bytes, int up_rank, int down_rank, int wait_flags) {
  const uint32_t rd = (up_rank >= 0 || down_rank >= 0) ? c.clock[1] : 0u;
  if (wait_flags) wait_sources(c, idx, neighbour_mask(up_rank, down_rank), rd);
  const uint64_t row_bytes = row_vec * 16;
  // top halo = up neighbour's LAST row (its part 1); bottom halo = down neighbour's FIRST row (its part 0)
  const char* top = up_rank >= 0 ? slot_ptr(c, c.rank, rd, tensor_off, slot_bytes, up_rank) + (uint64_t)b * row_bytes : nullptr;
  const char* bot = down_rank >= 0 ? slot_ptr(c, c.rank, rd, tensor_off, slot_bytes, down_rank) : nullptr;
  const uint64_t hp = h + 2;
  const uint64_t total = (uint64_t)b * hp * row_vec;
  const int4 zero = make_int4(0, 0, 0, 0);
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (uint64_t)gridDim.x * blockDim.x) {
    uint64_t row = i / row_vec, q = i - row * row_vec;
    uint64_t bb = row / hp, yy = row - bb * hp;
    int4 v;
    if (yy == 0) v = top ? ld_v4(top + (bb * row_vec + q) * 16) : zero;
    else if (yy == hp - 1) v = bot ? ld_v4(bot + (bb * row_vec + q) * 16) : zero;
    else v = ld_nc_v4(x + ((bb * h + (yy - 1)) * row_vec + q) * 16);
    st_v4(xp + i * 16, v);
  }
}

}  // namespace

// the kernels copy bytes: the element type only sets the row size
static uint64_t halo_row_bytes(int w, int C, int dtype) { return (uint64_t)w * C * (dtype == DF_F32 ? 4 : 2); }

extern "C" int df_halo_push_dtype(df_comm_t comm, const void* x, int b, int h, int w, int C, int idx, uint64_t tensor_off,
                                  uint64_t slot_bytes, int up_rank, int down_rank, int dtype, void* stream) {
  DF_REQUIRE(dtype == DF_F16 || dtype == DF_F32, "df_halo_push: unknown element type %d", dtype);
  uint64_t row_bytes = halo_row_bytes(w, C, dtype);
  DF_REQUIRE(row_bytes % 16 == 0 && ((uintptr_t)x % 16) == 0, "df_halo_push: rows must be 16-byte multiples");
  DF_REQUIRE(slot_bytes >= 2ull * b * row_bytes, "df_halo_push: slot too small");
  if (up_rank < 0 && down_rank < 0) return 0;
  uint64_t total = 2ull * b * (row_bytes / 16);
  int grid = (int)((total + 255) / 256);
  grid = grid < 1 ? 1 : (grid > 32 ? 32 : grid);
  halo_push_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(comm, (const char*)x, b, h, row_bytes / 16, idx, tensor_off,
                                                          slot_bytes, up_rank, down_rank);
  DF_CHECK_LAUNCH();
  return 0;
}

extern "C" int df_halo_assemble_dtype(df_comm_t comm, const void* x, void* xp, int b, int h, int w, int C, int idx,
                                      uint64_t tensor_off, uint64_t slot_bytes, int up_rank, int down_rank, int wait_flags,
                                      int dtype, void* stream) {
  DF_REQUIRE(dtype == DF_F16 || dtype == DF_F32, "df_halo_assemble: unknown element type %d", dtype);
  uint64_t row_bytes = halo_row_bytes(w, C, dtype);
  DF_REQUIRE(row_bytes % 16 == 0 && ((uintptr_t)x % 16) == 0 && ((uintptr_t)xp % 16) == 0,
             "df_halo_assemble: rows must be 16-byte multiples");
  uint64_t total = (uint64_t)b * (h + 2) * (row_bytes / 16);
  uint64_t g = (total + 256 * 8 - 1) / (256 * 8);
  int grid = (int)(g < 1 ? 1 : (g > kSmCount * 8 ? kSmCount * 8 : g));
  halo_assemble_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(comm, (const char*)x, (char*)xp, b, h, row_bytes / 16, idx,
                                                              tensor_off, slot_bytes, up_rank, down_rank, wait_flags);
  DF_CHECK_LAUNCH();
  return 0;
}

extern "C" int df_halo_push(df_comm_t comm, const void* x, int b, int h, int w, int C, int idx, uint64_t tensor_off,
                            uint64_t slot_bytes, int up_rank, int down_rank, void* stream) {
  return df_halo_push_dtype(comm, x, b, h, w, C, idx, tensor_off, slot_bytes, up_rank, down_rank, DF_F16, stream);
}

extern "C" int df_halo_assemble(df_comm_t comm, const void* x, void* xp, int b, int h, int w, int C, int idx,
                                uint64_t tensor_off, uint64_t slot_bytes, int up_rank, int down_rank, int wait_flags,
                                void* stream) {
  return df_halo_assemble_dtype(comm, x, xp, b, h, w, C, idx, tensor_off, slot_bytes, up_rank, down_rank, wait_flags, DF_F16,
                                stream);
}
