// distrifuser_b200 -- attention for ONE head of width 512 over per-rank K/V segments (sm_90a: wgmma + TMA + mbarrier): the
// mid-block self-attention of the VAE decoder (diffusers Attention with heads = 1, dim_head = 512), which df_attn_fwd (d <= 192)
// does not cover.
//
// One CTA per 64 Q rows of one batch item, 256 threads = two warpgroups, one CTA per SM (193 KiB of shared memory):
//   Both warpgroups compute the same S = Q K^T of a 64-row K/V tile (m64n64k16 wgmmas over the 512 columns, both operands in
//   shared memory) and the same online softmax; warpgroup w keeps O's columns [256 w, 256 w + 256) in 128 fp32 registers per
//   thread and adds P V[:, its half] with P packed to fp16 in registers as the A operand (m64n64k16, V MN-major from shared
//   memory).  One warpgroup holding all 512 columns of O would need 256 accumulator registers per thread.
//   Thread 0 also drives the TMA: Q once, then the K and the V tile of every 64 K/V rows (64 KiB each, one stage each) through
//   mbarrier pairs.  K of tile j + 1 is issued once both warpgroups have finished S_j (under P V_j), V of tile j + 1 once both
//   have finished P V_j (under S_{j+1} and its softmax).  Before the first tile of a peer's segment it acquires that peer's flag.
//   A separate producer warp would cost registers: with 9 or 12 warps ptxas caps every thread at 168 registers (the O fragment,
//   S and packed P alone take 176), with 8 warps it allows 255 (ptxas -v: 190, no spills).
// Recomputing S in both warpgroups costs 1.5x the tensor-core work of one S and one P V; sharing P through shared memory would
// cost an 8 KiB store + a barrier between the warpgroups on every tile.  At 64 Q rows per CTA each 2 KiB K/V row read from L2
// feeds only 64 x 512 x 4 FLOP, so the loads rather than the tensor cores are the expected limit (DESIGN §3.6).
// No printf anywhere in this kernel (DESIGN §3.1): spin_until<false>.

#include "tc_ptx.cuh"

using namespace df;
using namespace df::tc;

namespace {

constexpr int WD = 512;                 // head width
constexpr int WBM = 64;                 // Q rows per CTA
constexpr int WBN = 64;                 // K/V rows per tile
constexpr int WHB = 64;                 // columns per swizzled block (one 128-byte row)
constexpr int WSN = 64;                 // K/V rows per S slice (the m64n64k16 wgmmas of S below)
constexpr int WNB = WD / WHB;           // 8 column blocks
constexpr int WNTHREADS = 256;          // two warpgroups
constexpr uint32_t W_BLK_BYTES = WBN * WHB * 2;              // one 64 x 64 fp16 block = 8 KiB
constexpr uint32_t W_TILE_BYTES = WNB * W_BLK_BYTES;         // 64 KiB
static_assert(WBM == WBN, "Q and K/V blocks share the tensor-map box");

struct __align__(1024) WideSmem {
  __half q[WNB][WBM * WHB];
  __half k[WNB][WBN * WHB];
  __half v[WNB][WBN * WHB];
  uint64_t q_full, k_full, k_empty, v_full, v_empty;
};

// K/V segments in walk order o = 0 .. nseg - 1 (segment (own_seg + o) mod nseg: the own fresh segment first)
struct WideSegs {
  int32_t rank[DF_MAX_WORLD];      // communicator member holding segment s
  int32_t len[DF_MAX_WORLD];       // K/V rows of walk order o
  int32_t tile0[DF_MAX_WORLD + 1]; // first tile of walk order o; tile0[nseg] = all tiles
};

__global__ void __launch_bounds__(WNTHREADS, 1)
fmha_wide_kernel(const __grid_constant__ CUtensorMap tm_q, const __grid_constant__ CUtensorMap tm_kv_own,
                 const CUtensorMap* __restrict__ kvmaps, df_comm_t comm, const __grid_constant__ WideSegs segs,
                 __half* __restrict__ out, int lq, int64_t o_pitch, int nseg, int own_seg, int idx, int wait_flags,
                 float scale_log2) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  WideSmem& sm = *reinterpret_cast<WideSmem*>(smem_raw);
  if ((smem_u32(smem_raw) & 1023u) != 0) __trap();  // SWIZZLE_128B tiles need a 1 KiB aligned base

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * WBM, bat = blockIdx.y;
  const int T = segs.tile0[nseg];

  if (threadIdx.x == 0) {
    mbar_init(&sm.q_full, 1);
    mbar_init(&sm.k_full, 1);
    mbar_init(&sm.k_empty, 8);
    mbar_init(&sm.v_full, 1);
    mbar_init(&sm.v_empty, 8);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  // Thread 0 also issues the loads (a producer warp would cap every thread at 168 registers: ptxas sizes the register file share
  // of one SM sub-partition for 3 warps).  Tile j of the concatenated segments -> its tensor map and first row; before the first
  // tile of a peer's segment the peer's flag is acquired.
  auto issue = [&](int j, bool is_k) {
    int so = 0;
    while (so + 1 < nseg && segs.tile0[so + 1] <= j) ++so;
    const int t = j - segs.tile0[so];
    int seg = own_seg + so;
    if (seg >= nseg) seg -= nseg;
    const void* map = &tm_kv_own;
    if (seg != own_seg) {
      const uint32_t rd = comm.clock[1];
      const int r = segs.rank[seg];
      if (is_k && t == 0 && wait_flags) {
        spin_until<false>(flag_ptr(comm, comm.rank, idx, r), rd, comm.spin_timeout_ns);
        // the acquire above is a generic-proxy read; the peer's rows are fetched next through the async proxy (TMA)
        asm volatile("fence.proxy.async.global;" ::: "memory");
      }
      map = kvmaps + (size_t)(rd % DF_NBANKS) * comm.world + r;
    }
    uint64_t* bar = is_k ? &sm.k_full : &sm.v_full;
    mbar_expect_tx(bar, W_TILE_BYTES);
#pragma unroll
    for (int blk = 0; blk < WNB; ++blk) tma_load_4d(is_k ? sm.k[blk] : sm.v[blk], map, bar, blk * WHB, is_k ? 0 : 1, t * WBN, bat);
  };
  if (threadIdx.x == 0) {
    prefetch_tmap(&tm_q);
    prefetch_tmap(&tm_kv_own);
    mbar_expect_tx(&sm.q_full, W_TILE_BYTES);
#pragma unroll
    for (int blk = 0; blk < WNB; ++blk) tma_load_4d(sm.q[blk], &tm_q, &sm.q_full, blk * WHB, 0, q0, bat);
    issue(0, true);
    issue(0, false);
  }
  __syncwarp();
  {
    // =============================================================== consumers: S, softmax, P V (warpgroup wg: O columns 256 wg ..)
    // Accumulator fragment: thread t of warp w (in its warpgroup) holds rows rA = 16 (w & 3) + t/4 and rA + 8, columns
    // 8i + 2(t%4) + {0,1} of each 64-column block: s[4i + {0,1}] (row rA), s[4i + {2,3}] (row rA + 8).
    const int wg = warp >> 2;
    const int c4 = lane & 3;
    const int rowA = (warp & 3) * 16 + (lane >> 2);
    // descriptor start-address fields (14 bits of address / 16) do not carry: every offset stays inside the 227 KiB window
    const uint64_t q_desc = smem_desc(smem_u32(sm.q), 16, 1024), k_desc = smem_desc(smem_u32(sm.k), 16, 1024);
    const uint64_t v_desc = smem_desc(smem_u32(sm.v) + wg * (WNB / 2) * W_BLK_BYTES, W_BLK_BYTES, 1024);
    float o[4 * 32];
#pragma unroll
    for (int i = 0; i < 4 * 32; ++i) o[i] = 0.f;
    float s[WSN / 2];                            // S of the current slice, then its P in fp32
    uint32_t pk[WSN / 4];                        // P of the slice packed to fp16: the A operand of its P V
    float mA = -INFINITY, mB = -INFINITY;        // running row maxima of S * scale_log2
    float lA = 0.f, lB = 0.f;                    // partial row sums over this thread's columns
    mbar_wait(&sm.q_full, 0);
    int so = 0, t = 0, lseg = segs.len[0];
    for (int j = 0; j < T; ++j, ++t) {
      if (j == segs.tile0[so + 1]) { ++so; t = 0; lseg = segs.len[so]; }
      const int valid = min(WBN, lseg - t * WBN);
      const uint32_t ph = (uint32_t)j & 1u;
#pragma unroll
      for (int sub = 0; sub < WBN / WSN; ++sub) {
        // ---- S = Q K^T of the slice's WSN K/V rows
        if (sub == 0) mbar_wait(&sm.k_full, ph);
        // The descriptors are base descriptors plus constants; the empty asm keeps ptxas from hoisting all of them out of the
        // tile loop (registers the O fragment needs), so each is one add before its MMA.
        uint64_t qd = q_desc, kd = k_desc + ((sub * WSN * 128) >> 4);
        asm volatile("" : "+l"(qd), "+l"(kd));
        wgmma_fence();
#pragma unroll
        for (int blk = 0; blk < WNB; ++blk)
#pragma unroll
          for (int kk = 0; kk < WHB / 16; ++kk)
            wgmma_ss_n64(s, qd + ((blk * W_BLK_BYTES + kk * 32) >> 4), kd + ((blk * W_BLK_BYTES + kk * 32) >> 4), (blk | kk) > 0);
        wgmma_commit();
        if (sub == 0 && j > 0) {                         // V of this tile, once both warpgroups are done with the last one
          if (threadIdx.x == 0) {
            mbar_wait(&sm.v_empty, (uint32_t)(j - 1) & 1u);
            issue(j, false);
          }
          __syncwarp();
        }
        wgmma_wait<0>();
        fence_regs<WSN / 2>(s);
        if (sub == WBN / WSN - 1) {
          __syncwarp();
          if (lane == 0) mbar_arrive(&sm.k_empty);
        }
        const int vcols = valid - sub * WSN;             // valid columns of this slice
        if (vcols < WSN) {                               // ragged last tile of a segment (warp-uniform branch)
#pragma unroll
          for (int i = 0; i < WSN / 8; ++i)
#pragma unroll
            for (int k = 0; k < 2; ++k)
              if (8 * i + 2 * c4 + k >= vcols) { s[4 * i + k] = -INFINITY; s[4 * i + 2 + k] = -INFINITY; }
        }
        // ---- online softmax.  The first slice of every tile has >= 1 valid column, so the maxima are finite from the first
        //      slice on; a fully masked later slice leaves them unchanged and contributes P = 0.
        float xA = -INFINITY, xB = -INFINITY;
#pragma unroll
        for (int i = 0; i < WSN / 8; ++i) {
          xA = fmaxf(xA, fmaxf(s[4 * i], s[4 * i + 1]));
          xB = fmaxf(xB, fmaxf(s[4 * i + 2], s[4 * i + 3]));
        }
        xA = fmaxf(xA, __shfl_xor_sync(0xffffffffu, xA, 1));
        xB = fmaxf(xB, __shfl_xor_sync(0xffffffffu, xB, 1));
        xA = fmaxf(xA, __shfl_xor_sync(0xffffffffu, xA, 2));
        xB = fmaxf(xB, __shfl_xor_sync(0xffffffffu, xB, 2));
        const float nA = fmaxf(mA, xA * scale_log2), nB = fmaxf(mB, xB * scale_log2);
        const float alphaA = ex2(mA - nA), alphaB = ex2(mB - nB);      // 0 on the first slice (m = -inf)
        mA = nA;
        mB = nB;
        float sA = 0.f, sB = 0.f;
#pragma unroll
        for (int i = 0; i < WSN / 8; ++i) {
          s[4 * i] = ex2(fmaf(s[4 * i], scale_log2, -mA));
          s[4 * i + 1] = ex2(fmaf(s[4 * i + 1], scale_log2, -mA));
          s[4 * i + 2] = ex2(fmaf(s[4 * i + 2], scale_log2, -mB));
          s[4 * i + 3] = ex2(fmaf(s[4 * i + 3], scale_log2, -mB));
          sA += s[4 * i] + s[4 * i + 1];
          sB += s[4 * i + 2] + s[4 * i + 3];
          pk[2 * i] = pack_h2(s[4 * i], s[4 * i + 1]);
          pk[2 * i + 1] = pack_h2(s[4 * i + 2], s[4 * i + 3]);
        }
        lA = fmaf(lA, alphaA, sA);
        lB = fmaf(lB, alphaB, sB);
#pragma unroll
        for (int i = 0; i < 32; ++i) {
          o[4 * i] *= alphaA; o[4 * i + 1] *= alphaA;
          o[4 * i + 2] *= alphaB; o[4 * i + 3] *= alphaB;
        }
        // ---- O[:, 256 wg ..] += P V[slice rows, 256 wg ..]
        if (sub == 0) mbar_wait(&sm.v_full, ph);
        uint64_t vd = v_desc + ((sub * WSN * 128) >> 4);
        asm volatile("" : "+l"(vd));
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < WSN / 16; ++kk)
#pragma unroll
          for (int blk = 0; blk < WNB / 2; ++blk)
            wgmma_rs_n64(o + 32 * blk, pk + 4 * kk, vd + ((blk * W_BLK_BYTES + kk * 2048) >> 4), 1u);
        wgmma_commit();
        if (sub == WBN / WSN - 1 && j + 1 < T) {         // K of the next tile, once both warpgroups are done with this one
          if (threadIdx.x == 0) {
            mbar_wait(&sm.k_empty, ph);
            issue(j + 1, true);
          }
          __syncwarp();
        }
        wgmma_wait<0>();
        fence_regs<4 * 32>(o);
        if (sub == WBN / WSN - 1) {
          __syncwarp();
          if (lane == 0) mbar_arrive(&sm.v_empty);
        }
      }
    }
    // ---- epilogue: quad-reduce the row sums, O / l -> fp16 -> HBM
    lA += __shfl_xor_sync(0xffffffffu, lA, 1); lB += __shfl_xor_sync(0xffffffffu, lB, 1);
    lA += __shfl_xor_sync(0xffffffffu, lA, 2); lB += __shfl_xor_sync(0xffffffffu, lB, 2);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = rowA + 8 * h;
      if (q0 + row >= lq) continue;
      const float inv = 1.f / (h == 0 ? lA : lB);
      __half* dst = out + ((int64_t)bat * lq + q0 + row) * o_pitch + wg * (WD / 2);
#pragma unroll
      for (int blk = 0; blk < WNB / 2; ++blk)
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int col = blk * WHB + 8 * i + 2 * c4;
          *reinterpret_cast<uint32_t*>(dst + col) = pack_h2(o[32 * blk + 4 * i + 2 * h] * inv, o[32 * blk + 4 * i + 2 * h + 1] * inv);
        }
    }
  }
}

// 4-D view [512, nheads, rows, batch] of a row-major [batch, rows, pitch] fp16 matrix; box = [64, 1, 64, 1], 128B swizzle.
int make_wide_map(CUtensorMap* m, const void* base, int nheads, int rows, int batch, int64_t pitch) {
  EncodeTiledFn enc = tensor_map_encoder();
  DF_REQUIRE(enc != nullptr, "cuTensorMapEncodeTiled is not available from this driver");
  cuuint64_t dims[4] = {(cuuint64_t)WD, (cuuint64_t)nheads, (cuuint64_t)rows, (cuuint64_t)batch};
  cuuint64_t strides[3] = {(cuuint64_t)WD * 2, (cuuint64_t)pitch * 2, (cuuint64_t)rows * pitch * 2};
  cuuint32_t box[4] = {WHB, 1, WBN, 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  DF_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed (%d): base=%p heads=%d rows=%d batch=%d pitch=%lld", (int)r, base,
             nheads, rows, batch, (long long)pitch);
  return 0;
}

}  // namespace

extern "C" int df_attn_wide_make_kvmaps(df_comm_t comm, uint64_t tensor_off, uint64_t slot_bytes, int b,
                                        const int32_t* seg_len_host, int d, void* maps_out, void* stream) {
  static_assert(sizeof(CUtensorMap) == DF_TENSORMAP_BYTES, "tensor map size");
  DF_REQUIRE(d == WD, "df_attn_wide: head width %d not supported (512 only)", d);
  DF_REQUIRE(seg_len_host != nullptr && comm.world >= 1 && comm.world <= DF_MAX_WORLD && b >= 1,
             "df_attn_wide_make_kvmaps: bad arguments");
  for (int s = 0; s < comm.world; ++s) {
    DF_REQUIRE(seg_len_host[s] >= 1, "df_attn_wide_make_kvmaps: member %d has %d K/V rows", s, seg_len_host[s]);
    DF_REQUIRE(slot_bytes >= (uint64_t)b * seg_len_host[s] * 2 * WD * 2, "df_attn_wide_make_kvmaps: slot too small");
  }
  CUtensorMap host[DF_NBANKS * DF_MAX_WORLD];
  memset(host, 0, sizeof(host));
  for (int k = 0; k < DF_NBANKS; ++k)
    for (int s = 0; s < comm.world; ++s) {
      const char* base = slot_ptr(comm, comm.rank, (uint32_t)k, tensor_off, slot_bytes, s);
      if (int rc = make_wide_map(&host[k * comm.world + s], base, 2, seg_len_host[s], b, 2 * WD)) return rc;
    }
  DF_CHECK_CUDA(cudaMemcpyAsync(maps_out, host, sizeof(CUtensorMap) * DF_NBANKS * comm.world, cudaMemcpyHostToDevice,
                                (cudaStream_t)stream));
  DF_CHECK_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
  return 0;
}

extern "C" int df_attn_wide_fwd(df_comm_t comm, const void* q, const void* kv_own, void* out, const void* kvmaps, int b, int lq,
                                const int32_t* seg_len_host, int d, int64_t q_pitch, int64_t kv_pitch, int64_t o_pitch, int nseg,
                                int own_seg, const int32_t* seg_rank_host, int idx, int wait_flags, float scale, void* stream) {
  DF_REQUIRE(d == WD, "df_attn_wide_fwd: head width %d not supported (512 only)", d);
  DF_REQUIRE(seg_len_host != nullptr && nseg >= 1 && nseg <= DF_MAX_WORLD && own_seg >= 0 && own_seg < nseg,
             "df_attn_wide_fwd: bad segment layout");
  DF_REQUIRE(nseg == 1 || kvmaps != nullptr, "df_attn_wide_fwd: peer segments need tensor maps (df_attn_wide_make_kvmaps)");
  DF_REQUIRE(q_pitch % 8 == 0 && kv_pitch % 8 == 0 && o_pitch % 8 == 0 && q_pitch >= WD && kv_pitch >= 2 * WD && o_pitch >= WD &&
                 ((uintptr_t)q % 16) == 0 && ((uintptr_t)kv_own % 16) == 0 && ((uintptr_t)out % 16) == 0,
             "df_attn_wide_fwd: q/kv/out must be 16-byte aligned with pitches multiple of 8");
  DF_REQUIRE(b >= 1 && b <= 65535 && lq >= 1, "df_attn_wide_fwd: bad shape");
  for (int s = 0; s < nseg; ++s) DF_REQUIRE(seg_len_host[s] >= 1, "df_attn_wide_fwd: segment %d has %d K/V rows", s, seg_len_host[s]);
  CUtensorMap tq, tkv;
  if (int rc = make_wide_map(&tq, q, 1, lq, b, q_pitch)) return rc;
  if (int rc = make_wide_map(&tkv, kv_own, 2, seg_len_host[own_seg], b, kv_pitch)) return rc;
  WideSegs segs;
  memset(&segs, 0, sizeof(segs));
  for (int s = 0; s < nseg; ++s) segs.rank[s] = seg_rank_host ? seg_rank_host[s] : s;
  for (int o = 0; o < nseg; ++o) {                       // walk order: the own segment first, then the next ones cyclically
    const int s = (own_seg + o) % nseg;
    segs.len[o] = seg_len_host[s];
    segs.tile0[o + 1] = segs.tile0[o] + (seg_len_host[s] + WBN - 1) / WBN;
  }
  const float sl2 = (scale > 0.f ? scale : 1.f / sqrtf((float)WD)) * 1.4426950408889634f;
  static bool attr_set = false;
  const size_t smem_bytes = sizeof(WideSmem);
  if (!attr_set) {
    DF_CHECK_CUDA(cudaFuncSetAttribute(fmha_wide_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes));
    attr_set = true;
  }
  dim3 grid((unsigned)((lq + WBM - 1) / WBM), (unsigned)b, 1);
  fmha_wide_kernel<<<grid, WNTHREADS, smem_bytes, (cudaStream_t)stream>>>(tq, tkv, (const CUtensorMap*)kvmaps, comm, segs,
                                                                          (__half*)out, lq, o_pitch, nseg, own_seg, idx,
                                                                          wait_flags, sl2);
  DF_CHECK_LAUNCH();
  return 0;
}
