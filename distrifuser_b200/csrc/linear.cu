// distrifuser_b200 -- Linear layers of the transformer blocks as a hand-written wgmma GEMM with fused epilogues
// (SURVEY 8f N1: "fused Linear epilogues (to_kv -> comm slot, GEGLU)"; reference call sites distrifuser/modules/pp/attn.py:121-125,159
// and the diffusers FeedForward the wrappers live in).
//
//   out[M, N] = A[M, K] . W[N, K]^T  (+ bias[N]) (+ residual[M, N])          fp16 in, fp32 accumulate in registers, fp16 out
//   GEGLU:  out[M, N/2] = (A.Wh^T + bh) * gelu_erf(A.Wg^T + bg)  with the rows of W interleaved in blocks of BN/2
//           (hidden block t | gate block t), so that one BN-column accumulator tile holds both halves of BN/2 outputs:
//           the [M, 8C] projection of diffusers' GEGLU is never written to HBM (saves 3 * M * 4C * 2 B of traffic per layer
//           and the separate geglu kernel)
//   publish: columns >= pub_col0 of the result are ALSO stored into slot(pub, idx, me) of every peer in `peer_mask`
//           (fused q|k|v projection: the k|v columns go straight into the peers' arenas over NVLink -- replaces the
//           enqueue copy, utils.py:187, and the separate publication kernel); the last CTA stamps the peers' flags.
//
// Kernel: persistent CTAs, one per SM, each owning 128 x BN output tiles (BN = 256, or 160 where that fills the SMs better).
// Per 64-wide K block the producer TMA-loads 128 rows of A and BN rows of W into a SWIZZLE_128B ring; two consumer warpgroups
// each issue m64nBNk16 wgmmas for their 64 rows with the fp32 accumulators in registers and release the stage once the wgmma
// that read it has retired.  At the end of a tile the consumers add the bias, round to fp16 and stmatrix the tile into a
// staging buffer, then start the next tile's mainloop at once.  The epilogue warps read the staged tile in 16-byte vectors and
// finish it while the tensor cores run the next tile: GEGLU gate, residual add, coalesced 16-byte stores of the output and of
// the published columns.
//   warps 0-7  two consumer warpgroups (rows 0-63, 64-127 of the tile)
//   warp 8     TMA producer (one lane)                 warps 9-11  epilogue
#include <math.h>
#include <string.h>

#include "tc_ptx.cuh"

using namespace df;
using namespace df::tc;

namespace {

constexpr int BM = 128;            // rows of A per tile (64 per consumer warpgroup)
constexpr int BK = 64;             // one 128-byte swizzled row of fp16
constexpr int NCONSUMER_WARPS = 8;
constexpr int NCONSUMERS = 32 * NCONSUMER_WARPS;
constexpr int NTHREADS = NCONSUMERS + 128;   // GEMM: warps 0-7 consumers, warp 8 TMA producer, warps 9-11 epilogue
constexpr int NEPILOGUE = 96;
constexpr int NTHREADS_ZC = NCONSUMERS + 32; // zero convs: warps 0-7 consumers (own epilogue), warp 8 TMA producer
// registers per thread after setmaxnreg: 256 x CONSUMER_REGS + 128 x WG2_REGS = 384 x 168, what the block launches with
constexpr int CONSUMER_REGS = 208, WG2_REGS = 88;
constexpr uint32_t A_BYTES = BM * BK * 2;

// BN = output-tile columns (W rows): 256 for large N and the GEGLU epilogue, 160 where 256 would leave SMs idle.  Stages: as
// many as fit in the 227 KiB a block may use next to the GEMM's staging buffer (LinearSmem).
template <int BN> struct Stages { static constexpr int value = BN == 256 ? 3 : 5; };

template <int BN>
struct __align__(1024) SmemT {
  __half a[Stages<BN>::value][BM * BK];
  __half b[Stages<BN>::value][BN * BK];      // BN * 128 B per stage: a multiple of 1 KiB for BN in {160, 256}
  uint64_t full[Stages<BN>::value], empty[Stages<BN>::value];
};

// Staged fp16 tile: rows of BN + 8 halves.  The 16-byte pad moves row r by r 16-byte units (BN = 256) or 5r (BN = 160) modulo
// the 8 units of a 128-byte bank line, so the 8 row addresses of one stmatrix phase hit 8 different units: no bank conflicts.
template <int BN> __host__ __device__ constexpr int stage_pitch() { return BN + 8; }

template <int BN>
struct __align__(1024) LinearSmem {
  SmemT<BN> ring;
  __half stg[BM * stage_pitch<BN>()];
  uint64_t stg_full, stg_empty;              // staged tile written by the consumers / read by the epilogue warps
};

enum { EPI_PLAIN = 0, EPI_GEGLU = 1 };

struct LinearArgs {
  const __half* bias;       // [N] or null
  const __half* residual;   // [M, N] (pitch ldr) or null
  __half* out;              // [M, N] (GEGLU: [M, N/2]), pitch ldo
  int64_t M;
  int N, K;
  int64_t ldr, ldo;
  int tiles_m, tiles_n;
  // publication of the columns >= pub_col0 (fused q|k|v projection)
  int publish;              // 0 / 1
  int pub_col0, pub_cols;   // first published column, number of published columns (slot row = pub_cols halves)
  int idx;
  uint32_t peer_mask;
  uint64_t tensor_off, slot_bytes;
  df_comm_t comm;
};

__device__ __forceinline__ float gelu_erf(float x) {      // same approximation as csrc/elementwise.cu (A&S 7.1.26, |err| < 1.5e-7)
  const float z = fabsf(x) * 0.70710678118654752f;
  const float t = __fdividef(1.f, fmaf(0.3275911f, z, 1.f));
  float p = fmaf(1.061405429f, t, -1.453152027f);
  p = fmaf(p, t, 1.421413741f);
  p = fmaf(p, t, -0.284496736f);
  p = fmaf(p, t, 0.254829592f);
  const float e = p * t * __expf(-z * z);
  const float phi = x >= 0.f ? 1.f - 0.5f * e : 0.5f * e;
  return x * phi;
}

__device__ __forceinline__ float2 ld_h2f(const __half* p) { return __half22float2(*reinterpret_cast<const __half2*>(p)); }

// four 8 x 8 fp16 matrices from the accumulator fragment layout into shared memory; lane l gives the address of row l % 8 of
// matrix l / 8
__device__ __forceinline__ void stmatrix_x4(uint32_t addr, uint32_t r0, uint32_t r1, uint32_t r2, uint32_t r3) {
  asm volatile("stmatrix.sync.aligned.m8n8.x4.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(r0), "r"(r1), "r"(r2), "r"(r3)
               : "memory");
}

union H8 {                                  // one 16-byte vector of 8 fp16
  uint4 u;
  __half2 h[4];
};

template <int BN>
__device__ __forceinline__ void wgmma_tile(float* acc, uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
  if constexpr (BN == 256) wgmma_ss_n256(acc, a_desc, b_desc, accumulate);
  else wgmma_ss_n160(acc, a_desc, b_desc, accumulate);
}

// The mainloop, shared by every GEMM kernel of this file.  Producer (one lane): TMA-loads the K blocks of the 128 x BN tile
// (tm, tn) into the stage ring.  Consumers (both warpgroups): acc = A tile . W tile^T over those K blocks, each stage released
// once the wgmmas that read it have retired.  Producer and consumers walk the same tile sequence, so the ring stays in step.
template <int BN>
__device__ __forceinline__ void load_tile(SmemT<BN>& sm, const void* tm_a, const void* tm_w, int tm, int tn, int kblocks,
                                          uint32_t& stage, uint32_t& phase) {
  constexpr int STAGES = Stages<BN>::value;
  constexpr uint32_t B_BYTES = BN * BK * 2;
  for (int kb = 0; kb < kblocks; ++kb) {
    mbar_wait(&sm.empty[stage], phase ^ 1u);
    mbar_expect_tx(&sm.full[stage], A_BYTES + B_BYTES);
    tma_load_2d(sm.a[stage], tm_a, &sm.full[stage], kb * BK, tm * BM);
    tma_load_2d(sm.b[stage], tm_w, &sm.full[stage], kb * BK, tn * BN);
    if (++stage == STAGES) { stage = 0; phase ^= 1u; }
  }
}

template <int BN>
__device__ __forceinline__ void mma_tile(SmemT<BN>& sm, float* acc, int wg, int lane, int kblocks, uint32_t& stage,
                                         uint32_t& phase) {
  constexpr int STAGES = Stages<BN>::value;
  fence_regs<BN / 2>(acc);
  uint32_t prev = 0;
  for (int kb = 0; kb < kblocks; ++kb) {
    mbar_wait(&sm.full[stage], phase);
    const uint32_t a_addr = smem_u32(sm.a[stage]) + wg * 64 * 128, b_addr = smem_u32(sm.b[stage]);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < BK / 16; ++kk)
      wgmma_tile<BN>(acc, smem_desc(a_addr + kk * 32, 16, 1024), smem_desc(b_addr + kk * 32, 16, 1024), (kb | kk) > 0);
    wgmma_commit();
    wgmma_wait<1>();                                   // the previous K block's wgmmas have retired: its stage is free
    if (kb > 0 && lane == 0) mbar_arrive(&sm.empty[prev]);
    prev = stage;
    if (++stage == STAGES) { stage = 0; phase ^= 1u; }
  }
  wgmma_wait<0>();
  fence_regs<BN / 2>(acc);
  if (lane == 0) mbar_arrive(&sm.empty[prev]);
}

template <int EPI, int BN>
__global__ void __launch_bounds__(NTHREADS, 1)
linear_kernel(const __grid_constant__ CUtensorMap tm_a, const __grid_constant__ CUtensorMap tm_w, LinearArgs p) {
  static_assert(BN % 32 == 0 && BN <= 256 && (BN * BK * 2) % 1024 == 0, "tile shape");
  constexpr int STAGES = Stages<BN>::value;
  constexpr int SP = stage_pitch<BN>();
  using Smem = LinearSmem<BN>;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  Smem& sm = *reinterpret_cast<Smem*>(smem_raw);
  if ((smem_u32(smem_raw) & 1023u) != 0) __trap();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int ntiles = p.tiles_m * p.tiles_n;
  const int kblocks = p.K / BK;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) { mbar_init(&sm.ring.full[s], 1); mbar_init(&sm.ring.empty[s], NCONSUMER_WARPS); }
    mbar_init(&sm.stg_full, NCONSUMERS);
    mbar_init(&sm.stg_empty, NEPILOGUE);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp < NCONSUMER_WARPS) {
    // =============================================================== consumers (warps 0-7): mainloop, bias, stage the tile
    setmaxnreg_inc<CONSUMER_REGS>();
    const int wg = warp >> 2;
    const int c4 = lane & 3;
    // stmatrix row address of this lane: matrix lane / 8 of an x4 holds rows 8 * (lane / 8 % 2) + lane % 8 of the warp's 16
    // rows, columns 8 * (lane / 16) + [0, 8) of the pair of 8-column blocks the x4 stores
    const int mrow = wg * 64 + (warp & 3) * 16 + ((lane >> 3) & 1) * 8 + (lane & 7);
    const uint32_t st_addr = smem_u32(sm.stg) + (uint32_t)(mrow * SP + (lane >> 4) * 8) * 2u;
    uint32_t stage = 0, phase = 0, sphase = 0;
    float acc[BN / 2];
    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
      const int tn = tile / p.tiles_m;
      // the bias pairs of this thread's columns, loaded before the mainloop so that their latency hides behind it
      __half2 bias2[BN / 8];
#pragma unroll
      for (int i = 0; i < BN / 8; ++i) {
        const int col = tn * BN + 8 * i + 2 * c4;         // GEGLU: the interleaved bias has the tile's column order
        bias2[i] = p.bias && col < p.N ? *reinterpret_cast<const __half2*>(p.bias + col) : __float2half2_rn(0.f);
      }
      mma_tile<BN>(sm.ring, acc, wg, lane, kblocks, stage, phase);
      mbar_wait(&sm.stg_empty, sphase ^ 1u);             // the epilogue warps have read the previous tile
#pragma unroll
      for (int j = 0; j < BN / 16; ++j) {
        uint32_t r[4];
#pragma unroll
        for (int q = 0; q < 2; ++q) {
          const int i = 2 * j + q;
          const float2 bb = __half22float2(bias2[i]);
          // fp32 + bias rounded to fp16: torch's Linear output (GEGLU: diffusers rounds the projection before the gate)
          r[2 * q] = pack_h2(acc[4 * i] + bb.x, acc[4 * i + 1] + bb.y);
          r[2 * q + 1] = pack_h2(acc[4 * i + 2] + bb.x, acc[4 * i + 3] + bb.y);
        }
        stmatrix_x4(st_addr + j * 32, r[0], r[1], r[2], r[3]);
      }
      mbar_arrive(&sm.stg_full);
      sphase ^= 1u;
    }
  } else {
    setmaxnreg_dec<WG2_REGS>();
    if (warp == NCONSUMER_WARPS) {
      // ============================================================= TMA producer
      if (lane == 0) {
        prefetch_tmap(&tm_a);
        prefetch_tmap(&tm_w);
        uint32_t stage = 0, phase = 0;
        for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x)
          load_tile<BN>(sm.ring, &tm_a, &tm_w, tile % p.tiles_m, tile / p.tiles_m, kblocks, stage, phase);
      }
    } else {
      // ============================================================= epilogue (warps 9-11): staged tile -> global memory
      const int et = threadIdx.x - (NCONSUMERS + 32);
      uint32_t pub_epoch = 0;
      if (p.publish) pub_epoch = p.comm.clock[0];
      uint32_t sphase = 0;
      for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const int tm = tile % p.tiles_m, tn = tile / p.tiles_m;
        mbar_wait(&sm.stg_full, sphase);
        if (EPI == EPI_GEGLU) {
          // staged columns [0, BN/2) = hidden, [BN/2, BN) = gate of output columns [tn*BN/2, (tn+1)*BN/2); N % BN == 0
          constexpr int CH = BN / 16;                     // 16-byte output vectors per row
          for (int v = et; v < BM * CH; v += NEPILOGUE) {
            const int r = v / CH, c = v % CH;
            const int64_t grow = (int64_t)tm * BM + r;
            if (grow >= p.M) continue;
            H8 hv, gv, o;
            hv.u = *reinterpret_cast<const uint4*>(sm.stg + r * SP + 8 * c);
            gv.u = *reinterpret_cast<const uint4*>(sm.stg + r * SP + 8 * (c + CH));
#pragma unroll
            for (int k = 0; k < 4; ++k) {
              const float2 hf = __half22float2(hv.h[k]), gf = __half22float2(gv.h[k]);
              o.h[k] = __floats2half2_rn(hf.x * gelu_erf(gf.x), hf.y * gelu_erf(gf.y));
            }
            *reinterpret_cast<uint4*>(p.out + grow * p.ldo + tn * (BN / 2) + 8 * c) = o.u;
          }
        } else {
          constexpr int CH = BN / 8;
          // unrolled, with the residual read through the read-only path, so that the residual loads of several vectors are
          // in flight at once
#pragma unroll 4
          for (int v = et; v < BM * CH; v += NEPILOGUE) {
            const int r = v / CH, c = v % CH;
            const int64_t grow = (int64_t)tm * BM + r;
            const int col = tn * BN + 8 * c;
            if (grow >= p.M || col >= p.N) continue;     // N % 8 == 0: a vector is entirely inside or outside
            H8 o;
            o.u = *reinterpret_cast<const uint4*>(sm.stg + r * SP + 8 * c);
            if (p.residual) {                             // torch: fp16 linear output, then fp16 add
              H8 rv;
              rv.u = __ldg(reinterpret_cast<const uint4*>(p.residual + grow * p.ldr + col));
#pragma unroll
              for (int k = 0; k < 4; ++k) o.h[k] = __hadd2(o.h[k], rv.h[k]);
            }
            *reinterpret_cast<uint4*>(p.out + grow * p.ldo + col) = o.u;
            if (p.publish && col >= p.pub_col0) {         // k|v columns: also into every peer's slot of the publish epoch
              const uint64_t off = slot_offset(p.comm, pub_epoch, p.tensor_off, p.slot_bytes, p.comm.rank) +
                                   ((uint64_t)grow * p.pub_cols + (col - p.pub_col0)) * 2;
              for (int q = 0; q < p.comm.world; ++q)
                if (p.peer_mask >> q & 1) *reinterpret_cast<uint4*>((char*)p.comm.base[q] + off) = o.u;
            }
          }
        }
        mbar_arrive(&sm.stg_empty);
        sphase ^= 1u;
      }
    }
  }
  // every thread fences its own peer stores before the CTA's ticket is taken
  if (p.publish) signal_when_last(p.comm, &p.comm.tickets[p.idx], gridDim.x, p.idx, p.peer_mask, p.comm.clock[0]);
}

// 2-D view [K (contiguous), rows] of a row-major [rows, pitch] fp16 matrix; box = [64, box_rows], 128B swizzle, zero fill
int make_map2d(CUtensorMap* m, const void* base, int64_t rows, int K, int64_t pitch, int box_rows) {
  EncodeTiledFn enc = tensor_map_encoder();
  DF_REQUIRE(enc != nullptr, "cuTensorMapEncodeTiled is not available from this driver");
  cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)pitch * 2};
  cuuint32_t box[2] = {BK, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  DF_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed (%d): base=%p rows=%lld K=%d pitch=%lld", (int)r, base,
             (long long)rows, K, (long long)pitch);
  return 0;
}

template <int EPI, int BN>
int launch_linear(const CUtensorMap& ta, const CUtensorMap& tw, const LinearArgs& args, int ctas, cudaStream_t st) {
  static bool attr_set = false;
  if (!attr_set) {
    DF_CHECK_CUDA(cudaFuncSetAttribute(linear_kernel<EPI, BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(LinearSmem<BN>)));
    attr_set = true;
  }
  linear_kernel<EPI, BN><<<ctas, NTHREADS, sizeof(LinearSmem<BN>), st>>>(ta, tw, args);
  DF_CHECK_LAUNCH();
  return 0;
}

// Relative cost of a problem with 128 x bn tiles: rounds x cycles per 64-wide K block of one tile.  The wgmmas of a K block take
// time proportional to bn, while the A half of the operand traffic (16 KiB per K block) is paid whatever bn is: a 160-wide tile
// moves 36 KiB for 160 columns, a 256-wide one 48 KiB for 256, so narrow tiles only pay off when they fill clearly more SMs.
double tile_cost(int64_t M, int N, int bn, int ctas_avail) {
  const long long tm = (M + BM - 1) / BM, tn = (N + bn - 1) / bn, tiles = tm * tn;
  const long long rounds = (tiles + ctas_avail - 1) / ctas_avail;
  return (double)rounds * (bn + 64);
}

}  // namespace

namespace {
// tile width for a problem: 256, or 160 where that fills the SMs better (GEGLU: only widths that tile N exactly)
int pick_bn(int64_t M, int N, int epilogue, int cap) {
  const bool ok160 = epilogue == EPI_PLAIN || N % 160 == 0, ok256 = epilogue == EPI_PLAIN || N % 256 == 0;
  if (!ok256) return ok160 ? 160 : 0;
  if (ok160 && tile_cost(M, N, 160, cap) < 0.97 * tile_cost(M, N, 256, cap)) return 160;
  return 256;
}
}  // namespace

extern "C" int df_linear_supported(int64_t M, int N, int K, int epilogue) {
  if (M < 1 || N < 8 || N % 8 != 0 || K < BK || K % BK != 0) return 0;
  if (epilogue == EPI_GEGLU && pick_bn(M, N, epilogue, sm_count()) == 0) return 0;   // blocks of 80 / 128 must tile N / 2
  return 1;
}

// GEGLU epilogue: rows of the interleaved weight per hidden / gate block (= half the tile width chosen for this problem)
extern "C" int df_linear_geglu_block(int64_t M, int N, int K) {
  (void)K;
  const int bn = pick_bn(M, N, EPI_GEGLU, sm_count());
  return bn / 2;
}

extern "C" int df_linear_fwd(df_comm_t comm, const void* a, const void* w, const void* bias, const void* residual, void* out,
                             int64_t M, int N, int K, int64_t lda, int64_t ldw, int64_t ldr, int64_t ldo, int epilogue,
                             int geglu_block, int publish, int pub_col0, int idx, uint32_t peer_mask, uint64_t tensor_off,
                             uint64_t slot_bytes, int max_ctas, void* stream) {
  DF_REQUIRE(epilogue == EPI_PLAIN || epilogue == EPI_GEGLU, "df_linear_fwd: unknown epilogue %d", epilogue);
  DF_REQUIRE(df_linear_supported(M, N, K, epilogue), "df_linear_fwd: unsupported shape M=%lld N=%d K=%d (N %% 8, K %% 64%s)",
             (long long)M, N, K, epilogue == EPI_GEGLU ? ", GEGLU: N % 256" : "");
  DF_REQUIRE(((uintptr_t)a % 16) == 0 && ((uintptr_t)w % 16) == 0 && ((uintptr_t)out % 16) == 0 && ((uintptr_t)bias % 16) == 0 &&
                 ((uintptr_t)residual % 16) == 0 && lda % 8 == 0 && ldw % 8 == 0 && ldo % 8 == 0 && ldr % 8 == 0,
             "df_linear_fwd: operands must be 16-byte aligned with pitches multiple of 8");
  DF_REQUIRE(!(publish && epilogue != EPI_PLAIN), "df_linear_fwd: publication is a plain-epilogue feature");
  LinearArgs args;
  memset(&args, 0, sizeof(args));
  args.bias = (const __half*)bias; args.residual = (const __half*)residual; args.out = (__half*)out;
  args.M = M; args.N = N; args.K = K; args.ldr = ldr; args.ldo = ldo;
  const int sms = sm_count();
  const int cap = max_ctas > 0 ? max_ctas : sms;
  int bn = pick_bn(M, N, epilogue, epilogue == EPI_GEGLU ? sms : cap);   // GEGLU: must agree with df_linear_geglu_block()
  if (epilogue == EPI_GEGLU && geglu_block > 0) {
    DF_REQUIRE(geglu_block == 80 || geglu_block == 128, "df_linear_fwd: geglu_block must be 80 or 128");
    bn = 2 * geglu_block;
    DF_REQUIRE(N % bn == 0, "df_linear_fwd: interleave block %d does not tile N=%d", geglu_block, N);
  }
  args.tiles_m = (int)((M + BM - 1) / BM);
  args.tiles_n = (N + bn - 1) / bn;
  args.publish = publish && peer_mask != 0;
  args.comm = comm;
  if (args.publish) {
    DF_REQUIRE(pub_col0 >= 0 && pub_col0 < N && pub_col0 % 8 == 0, "df_linear_fwd: bad pub_col0");
    DF_REQUIRE(tensor_off % 16 == 0 && slot_bytes % 16 == 0, "df_linear_fwd: slots must be 16-byte aligned");
    args.pub_col0 = pub_col0; args.pub_cols = N - pub_col0; args.idx = idx; args.peer_mask = peer_mask;
    args.tensor_off = tensor_off; args.slot_bytes = slot_bytes;
    DF_REQUIRE((uint64_t)M * args.pub_cols * 2 <= slot_bytes, "df_linear_fwd: published columns larger than the slot");
  }
  int ctas = args.tiles_m * args.tiles_n;
  if (ctas > cap) ctas = cap;
  if (ctas < 1) ctas = 1;
  CUtensorMap ta, tw;
  if (int rc = make_map2d(&ta, a, M, K, lda, BM)) return rc;
  if (int rc = make_map2d(&tw, w, N, K, ldw, bn)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  if (epilogue == EPI_GEGLU) {
    if (bn == 160) return launch_linear<EPI_GEGLU, 160>(ta, tw, args, ctas, st);
    return launch_linear<EPI_GEGLU, 256>(ta, tw, args, ctas, st);
  }
  if (bn == 160) return launch_linear<EPI_PLAIN, 160>(ta, tw, args, ctas, st);
  return launch_linear<EPI_PLAIN, 256>(ta, tw, args, ctas, st);
}

// ----------------------------------------------------------------------------------------- ControlNet zero convolutions
// out_i[M_i, N_i] = scale * (x_i[M_i, K_i] . W_i[N_i, K_i]^T + b_i) for every 1x1 "zero" conv of one ControlNet call, in ONE
// persistent launch of the mainloop above.  The problem list (tensor maps, bias / output pointers, tile offsets) is a
// __grid_constant__ parameter: it lives in the kernel's parameter space on the device, so a captured CUDA graph carries it and
// no host-to-device upload of a list is needed per call or per graph.  `scale` is read from device memory, so a replay of a
// captured graph honours a new conditioning scale.  Tiles are 128 x 160: 160 divides every ControlNet width (320, 640, 1280).
// K need only be a multiple of 8 (16-byte rows for TMA): the last K block's columns past K arrive as zeros in both operands.
namespace {
constexpr int ZC_BN = 160;

struct ZeroConvProblem {
  const __half* bias;       // [N] or null
  __half* out;              // [M, N] contiguous
  int M, N, tiles_m, tile0, kblocks;
};

struct ZeroConvArgs {
  CUtensorMap a[DF_ZERO_CONV_MAX_PROBLEMS], w[DF_ZERO_CONV_MAX_PROBLEMS];
  ZeroConvProblem p[DF_ZERO_CONV_MAX_PROBLEMS];
  const float* scale;
  int nproblems, ntiles;
};
static_assert(sizeof(ZeroConvArgs) <= 4096, "the problem list must fit the 4 KiB kernel parameter space");

__device__ __forceinline__ int zc_problem(const ZeroConvArgs& z, int tile) {
  int q = 0;
  while (q + 1 < z.nproblems && tile >= z.p[q + 1].tile0) ++q;
  return q;
}

__global__ void __launch_bounds__(NTHREADS_ZC, 1) zero_conv_kernel(const __grid_constant__ ZeroConvArgs z) {
  constexpr int BN = ZC_BN;
  constexpr int STAGES = Stages<BN>::value;
  using Smem = SmemT<BN>;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  Smem& sm = *reinterpret_cast<Smem*>(smem_raw);
  if ((smem_u32(smem_raw) & 1023u) != 0) __trap();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) { mbar_init(&sm.full[s], 1); mbar_init(&sm.empty[s], NCONSUMER_WARPS); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == NCONSUMER_WARPS) {
    if (lane == 0) {
      uint32_t stage = 0, phase = 0;
      for (int tile = blockIdx.x; tile < z.ntiles; tile += gridDim.x) {
        const int q = zc_problem(z, tile);
        const ZeroConvProblem& p = z.p[q];
        const int t = tile - p.tile0;
        load_tile<BN>(sm, &z.a[q], &z.w[q], t % p.tiles_m, t / p.tiles_m, p.kblocks, stage, phase);
      }
    }
  } else {
    const int wg = warp >> 2;
    const int c4 = lane & 3;
    const int rloc = wg * 64 + (warp & 3) * 16 + (lane >> 2);
    const float scale = *z.scale;
    uint32_t stage = 0, phase = 0;
    float acc[BN / 2];
    for (int tile = blockIdx.x; tile < z.ntiles; tile += gridDim.x) {
      const ZeroConvProblem& p = z.p[zc_problem(z, tile)];
      const int t = tile - p.tile0;
      const int tm = t % p.tiles_m, tn = t / p.tiles_m;
      mma_tile<BN>(sm, acc, wg, lane, p.kblocks, stage, phase);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int64_t grow = (int64_t)tm * BM + rloc + 8 * h;
        if (grow >= p.M) continue;
        const int col0 = tn * BN;
        __half* dst = p.out + grow * p.N + col0;
#pragma unroll
        for (int i = 0; i < BN / 8; ++i) {
          const int c = 8 * i + 2 * c4;
          const int col = col0 + c;
          if (col >= p.N) continue;                        // N % 8 == 0: a column pair is entirely inside or outside
          float2 f = make_float2(acc[4 * i + 2 * h], acc[4 * i + 2 * h + 1]);
          if (p.bias) { const float2 bb = ld_h2f(p.bias + col); f.x += bb.x; f.y += bb.y; }
          // torch: the fp16 conv output, then the scale multiply in fp32 rounded to fp16
          const float2 r = __half22float2(__floats2half2_rn(f.x, f.y));
          *reinterpret_cast<__half2*>(dst + c) = __floats2half2_rn(r.x * scale, r.y * scale);
        }
      }
    }
  }
}
}  // namespace

extern "C" int df_controlnet_zero_convs(int nproblems, const void* const* x_host, const void* const* w_host,
                                        const void* const* bias_host, void* const* out_host, const int64_t* m_host,
                                        const int32_t* n_host, const int32_t* k_host, const float* scale, int max_ctas,
                                        void* stream) {
  DF_REQUIRE(nproblems >= 1 && nproblems <= DF_ZERO_CONV_MAX_PROBLEMS, "df_controlnet_zero_convs: %d problems (1..%d)",
             nproblems, DF_ZERO_CONV_MAX_PROBLEMS);
  DF_REQUIRE(x_host && w_host && out_host && m_host && n_host && k_host && scale, "df_controlnet_zero_convs: null argument");
  DF_REQUIRE(((uintptr_t)scale % 4) == 0, "df_controlnet_zero_convs: scale must be a 4-byte aligned fp32");
  ZeroConvArgs z;
  memset(&z, 0, sizeof(z));
  int ntiles = 0;
  for (int i = 0; i < nproblems; ++i) {
    const int64_t M = m_host[i];
    const int N = n_host[i], K = k_host[i];
    const void* bias = bias_host ? bias_host[i] : nullptr;
    DF_REQUIRE(M >= 1 && M <= INT32_MAX && N >= 8 && N % 8 == 0 && K >= 8 && K % 8 == 0,
               "df_controlnet_zero_convs: problem %d has unsupported shape M=%lld N=%d K=%d (N %% 8, K %% 8)", i,
               (long long)M, N, K);
    DF_REQUIRE(x_host[i] && w_host[i] && out_host[i] && ((uintptr_t)x_host[i] % 16) == 0 &&
                   ((uintptr_t)w_host[i] % 16) == 0 && ((uintptr_t)out_host[i] % 16) == 0 && ((uintptr_t)bias % 16) == 0,
               "df_controlnet_zero_convs: problem %d: operands must be non-null and 16-byte aligned", i);
    if (int rc = make_map2d(&z.a[i], x_host[i], M, K, K, BM)) return rc;
    if (int rc = make_map2d(&z.w[i], w_host[i], N, K, K, ZC_BN)) return rc;
    ZeroConvProblem& p = z.p[i];
    p.bias = (const __half*)bias; p.out = (__half*)out_host[i];
    p.M = (int)M; p.N = N; p.kblocks = (K + BK - 1) / BK;        // TMA zero-fills the columns past K of the last block
    p.tiles_m = (int)((M + BM - 1) / BM);
    p.tile0 = ntiles;
    const int64_t t = (int64_t)p.tiles_m * ((N + ZC_BN - 1) / ZC_BN);
    DF_REQUIRE(ntiles + t <= INT32_MAX, "df_controlnet_zero_convs: too many tiles");
    ntiles += (int)t;
  }
  z.scale = scale; z.nproblems = nproblems; z.ntiles = ntiles;
  const int cap = max_ctas > 0 ? max_ctas : sm_count();
  const int ctas = ntiles < cap ? ntiles : cap;
  static bool attr_set = false;
  if (!attr_set) {
    DF_CHECK_CUDA(cudaFuncSetAttribute(zero_conv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(SmemT<ZC_BN>)));
    attr_set = true;
  }
  zero_conv_kernel<<<ctas, NTHREADS_ZC, sizeof(SmemT<ZC_BN>), (cudaStream_t)stream>>>(z);
  DF_CHECK_LAUNCH();
  return 0;
}
