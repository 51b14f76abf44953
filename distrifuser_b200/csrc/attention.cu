// distrifuser_b200 -- fused multi-head attention over per-rank K/V segments (sm_90a: wgmma + TMA + mbarrier).
//
// Replaces, for DistriSelfAttentionPP._forward (distrifuser/modules/pp/attn.py:127-153):
//     torch.cat(full_kv) over ranks  -> the K/V tiles are TMA-loaded straight from the n per-rank segments
//                                       (own fresh projection + peers' 1-step-stale arena slots)
//     torch.split + view/transpose   -> tensor-map coordinates (head, row) select K at column h*d, V at C + h*d
//     F.scaled_dot_product_attention -> S = Q K^T and O += P V as wgmma tiles, accumulators in registers
// and the SDPA of DistriCrossAttentionPP.forward (attn.py:79-87) with nseg = 1, lseg = 77.
//
// Persistent CTAs (384 threads: two consumer warpgroups + one producer warpgroup; one CTA per SM)
// walk work items = one 128-row Q tile of one (batch, head), or a K/V range of one:
//   warps 0-7  two consumer warpgroups, 64 Q rows each.  Per S slice (SN K/V rows): S = Q K^T (m64nSNk16 wgmmas, both operands
//              in shared memory) into SN/2 fp32 registers per thread, online softmax on that fragment (a row lives in one quad:
//              row maxima and sums are two shuffles; exp2 on MUFU with 3 of 16 column groups on a polynomial on the FMA pipe; the
//              exponent reference only moves when the row maximum grew by more than 2^8), P packed to fp16 IN REGISTERS as the A
//              operand of O += P V (m64n64k16 wgmmas, V MN-major from shared memory), O in registers; epilogue O / l -> HBM (or
//              fp32 partials merged by the last part of a split unit).  At d <= 80 the MMAs of slice i + 1's S and slice i's
//              P V are issued together, so the softmax of slice i + 1 runs while the tensor cores compute P_i V_i, and the two
//              warpgroups take turns on the tensor cores (Cfg::OVERLAP / PINGPONG).
//   warps 8-11 producer warpgroup (gives its registers to the consumers); lane 0 of warp 8 is the scheduler + TMA producer: hands
//              out work items through a two-entry ring (whole units drawn from an atomic ticket counter when the grid fills the
//              SMs, a static one-item list otherwise), then Q per item and K (KST stages) / V (VST stages) tiles through mbarrier
//              rings; waits the peers' flags

#include "tc_ptx.cuh"

using namespace df;
using namespace df::tc;

namespace {

constexpr int BM = 128;      // Q rows per CTA (64 per consumer warpgroup)
constexpr int BN = 128;      // K/V rows per tile
constexpr int HB = 64;       // head-dim block: one 128-byte swizzled row; d is padded to NBLK * 64 columns (TMA zero-fills)
constexpr int NCONSUMER_WARPS = 8;
constexpr int NTHREADS = 32 * (NCONSUMER_WARPS + 4);
constexpr int WARP_TMA = NCONSUMER_WARPS;
// registers per thread after setmaxnreg: 128 x PRODUCER_REGS + 256 x CONSUMER_REGS <= 65536
constexpr int PRODUCER_REGS = 56, CONSUMER_REGS = 224;    // the producer lane spills below 56
constexpr uint32_t BLK_BYTES = BN * HB * 2;                // one 128 x 64 fp16 block = 16 KiB

// NBLK = ceil(d / 64): 1 for d in {40, 64} (SDXL, SD1.x level 0), 2 for d = 80, 3 for d = 160 (SD1.x)
template <int NBLK, int KSTAGES, int VSTAGES>
struct __align__(1024) SmemT {
  __half q[NBLK][BM * HB];
  __half k[KSTAGES][NBLK][BN * HB];
  __half v[VSTAGES][NBLK][BN * HB];
  uint64_t q_full, q_empty;   // Q tile of the current work item loaded / no longer read by the tensor cores
  uint64_t k_full[KSTAGES], k_empty[KSTAGES], v_full[VSTAGES], v_empty[VSTAGES];
  uint64_t sched_full[2];     // work-item ring: the TMA lane (scheduler) publishes the next item code, the consumers read it
  int sched_code[2];
  uint32_t ticket;            // arrival ticket of this part among the parts of its left-over unit
};
// One CTA per SM.  A consumer thread holds the S slice (SN / 2), the O fragment (32 per head block) and the packed P (SN / 4) in
// at most CONSUMER_REGS registers: 128-wide S slices at d <= 64, 64-wide ones for the wider heads.  Shared memory (227 KiB)
// sets the stage counts.  OVERLAP picks the order inside a warpgroup (see the consumer loop): serial (S, softmax, P V, wait)
// or S of slice i + 1 issued with P V of slice i; PINGPONG (overlapped order only) hands the tensor cores to the two
// warpgroups in turns.  The overlapped order frees a V stage one slice later, so it needs a spare V stage: d = 160 has room
// for one only and keeps the serial order.  Without the turns the overlapped order was slower than the serial one at d <= 64
// (both warpgroups wait on the same K tile and then run their softmax at the same time); with them it is faster (DESIGN §3.1).
template <int NBLK> struct Cfg;
template <> struct Cfg<1> { static constexpr int KST = 4, VST = 4, SN = 128; static constexpr bool OVERLAP = true, PINGPONG = true; };
template <> struct Cfg<2> { static constexpr int KST = 3, VST = 3, SN = 64; static constexpr bool OVERLAP = true, PINGPONG = true; };
template <> struct Cfg<3> { static constexpr int KST = 2, VST = 1, SN = 64; static constexpr bool OVERLAP = false, PINGPONG = false; };
constexpr int TURN_BAR = 2;   // named barriers TURN_BAR + wg: the tensor-core turns of the two warpgroups (1: split merge)

// work schedule of one launch (host: plan_schedule): every CTA takes `a` whole units; the R left-over units are cut into P parts
struct Sched {
  int a, R, P;
  int dyn;      // 1: whole units are handed out by an atomic ticket counter (grids that fill the SMs); 0: static list per CTA
  int units;
};
constexpr int ITEM_END = -1;

__device__ __forceinline__ float2 ld_f2(const float2* p) {          // coherent load (partials were written during this launch)
  float2 r;
  asm volatile("ld.global.v2.f32 {%0, %1}, [%2];" : "=f"(r.x), "=f"(r.y) : "l"(p) : "memory");
  return r;
}

// K/V segment layout of a launch.  Segments may have different lengths (uneven row strips of patch parallelism); the
// kernel walks them in ORDER o = 0 .. nseg - 1, segment (own_seg + o) mod nseg, so that the own fresh segment comes first.
struct SegInfo {
  int32_t rank[DF_MAX_WORLD];      // world rank holding segment s
  int32_t len[DF_MAX_WORLD];       // K/V rows of the segment at walk order o
  int32_t tile0[DF_MAX_WORLD + 1]; // first tile of walk order o in the concatenated tile range; tile0[nseg] = all tiles
};

// of the 16 column groups of a tile row, this many (evenly spread) take the polynomial exp2 (FMA/ALU pipes) instead of MUFU
constexpr int kEmuGroups = 3;

template <int N>
__device__ __forceinline__ void wgmma_ss(float* d, uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
  if constexpr (N == 64) wgmma_ss_n64(d, a_desc, b_desc, accumulate);
  else wgmma_ss_n128(d, a_desc, b_desc, accumulate);
}

// ----------------------------------------------------------------------------------------- kernel
template <int NBLK>
__global__ void __launch_bounds__(NTHREADS, 1)
fmha_fwd_kernel(const __grid_constant__ CUtensorMap tm_q, const __grid_constant__ CUtensorMap tm_kv_own,
                const CUtensorMap* __restrict__ kvmaps, df_comm_t comm, const __grid_constant__ SegInfo segs, __half* __restrict__ out, int lq,
                int heads, int d, int64_t o_pitch, int nseg, int own_seg, int idx, int wait_flags,
                float scale_log2, Sched sched, float* part_o, float2* part_ml, unsigned int* part_cnt, unsigned int* sched_ctr) {
  constexpr int KSTAGES = Cfg<NBLK>::KST, VSTAGES = Cfg<NBLK>::VST;
  constexpr uint32_t TILE_BYTES = NBLK * BLK_BYTES;
  constexpr int SN = Cfg<NBLK>::SN, NSUB = BN / SN;
  constexpr bool OVERLAP = Cfg<NBLK>::OVERLAP, PINGPONG = Cfg<NBLK>::PINGPONG;
  using Smem = SmemT<NBLK, KSTAGES, VSTAGES>;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  Smem& sm = *reinterpret_cast<Smem*>(smem_raw);
  if ((smem_u32(smem_raw) & 1023u) != 0) __trap();  // SWIZZLE_128B tiles need a 1 KiB aligned base

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // PERSISTENT CTAs.  A work unit is one 128-row Q tile of one (batch, head).  CTA c walks the whole units c, c + G, ...
  // (G = gridDim.x resident CTAs) and then, if c < R*P, one more item: part (c mod P) of left-over unit (c div P).  With P = 1
  // the left-over units are simply whole units of the last round.  With P > 1 (grids that leave most SMs idle: short per-rank Q
  // at n >= 4 with long K/V) a unit's K/V range is cut into P parts that run on otherwise idle SMs; the parts leave
  // un-normalised fp32 partials in the workspace and the LAST part to finish (a ticket per unit) merges them and writes the rows
  // -- no second kernel.  The roles keep their rings / barrier phases running across items (tile counter g): barrier set-up,
  // tensor-map fetch and pipeline fill are paid once per CTA, and the K/V loads of the next item run under the epilogue of the
  // current one.
  const int nqt = (lq + BM - 1) / BM;
  const int T_all = segs.tile0[nseg];    // K/V tiles of all segments (each segment's last tile may be ragged)
  const int tiles_own = segs.tile0[1], len_own = segs.len[0];     // the own segment (walk order 0), kept in registers
  // walk order, tile inside that segment, its tile count and length for concatenated tile j (once per item, outside the tile
  // loops).  Whole units start in the own segment and need no parameter loads; only split parts may start further on.
  auto locate = [&](int j, int& so, int& t, int& tseg, int& lseg) {
    so = 0; t = j; tseg = tiles_own; lseg = len_own;
    if (j >= tiles_own) {
      while (so + 1 < nseg && segs.tile0[so + 1] <= j) ++so;
      t = j - segs.tile0[so]; tseg = segs.tile0[so + 1] - segs.tile0[so]; lseg = segs.len[so];
    }
  };
  const int n_items = sched.a + ((int)blockIdx.x < sched.R * sched.P ? 1 : 0);     // static schedule only
  // item code (from the ring, see the scheduler in the TMA lane) -> Q tile origin, head, batch, first K/V tile, tile count,
  // partial slot (-1: whole unit), left-over index.  Dynamic schedule: the code is the unit; static: the index into this
  // CTA's list (`a` whole units, then at most one part of a left-over unit).
  auto decode = [&](int it, int& q0, int& head, int& bat, int& j_begin, int& T, int& slot, int& lo) {
    int u;
    if (sched.dyn) {
      u = it; j_begin = 0; T = T_all; slot = -1; lo = -1;
    } else if (it < sched.a) {
      u = it * (int)gridDim.x + (int)blockIdx.x; j_begin = 0; T = T_all; slot = -1; lo = -1;
    } else {
      lo = (int)blockIdx.x / sched.P;
      const int part = (int)blockIdx.x - lo * sched.P;
      u = sched.a * (int)gridDim.x + lo;
      j_begin = (int)((long long)part * T_all / sched.P);
      T = (int)((long long)(part + 1) * T_all / sched.P) - j_begin;     // >= 1: P <= T_all
      slot = sched.P > 1 ? (int)blockIdx.x : -1;
    }
    const int qt = u % nqt, rest = u / nqt;
    head = rest % heads;
    bat = rest / heads;
    q0 = qt * BM;
  };

  if (threadIdx.x == 0) {
    mbar_init(&sm.q_full, 1);
    mbar_init(&sm.q_empty, NCONSUMER_WARPS);
    for (int s = 0; s < KSTAGES; ++s) { mbar_init(&sm.k_full[s], 1); mbar_init(&sm.k_empty[s], NCONSUMER_WARPS); }
    for (int s = 0; s < VSTAGES; ++s) { mbar_init(&sm.v_full[s], 1); mbar_init(&sm.v_empty[s], NCONSUMER_WARPS); }
    mbar_init(&sm.sched_full[0], 1);
    mbar_init(&sm.sched_full[1], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp >= WARP_TMA) {
    // =============================================================== scheduler + TMA producer
    setmaxnreg_dec<PRODUCER_REGS>();
    if (warp == WARP_TMA && lane == 0) {
      prefetch_tmap(&tm_q);
      prefetch_tmap(&tm_kv_own);
      uint32_t rd = 0;
      if (nseg > 1) rd = comm.clock[1];
      // This lane decides what the CTA works on next and tells the consumers through a two-entry ring (sched_code /
      // sched_full).  Grids that fill the SMs draw whole units from an atomic ticket counter: a CTA that starts late -- its SM
      // slot was held by a publication kernel of the communication stream -- or runs slower simply takes fewer units.  Small
      // grids keep their static one-item list (a part of a split unit).  The raw ticket of the next item is drawn one item
      // ahead: the atomic's latency hides under this item's loads.
      int it_static = 0;
      auto draw = [&]() -> unsigned int {
        if (sched.dyn) return atomicAdd(sched_ctr, 1u);
        return (unsigned int)it_static++;
      };
      const unsigned int n_fresh = sched.dyn ? (unsigned int)sched.units : (unsigned int)n_items;
      unsigned int next_t = draw();
      uint32_t g = 0;                                      // K/V tiles issued so far by this CTA
      for (uint32_t ui = 0;; ++ui) {
        int code = ITEM_END;
        if (next_t < n_fresh) {
          code = (int)next_t;
          next_t = draw();
        } else if (sched.dyn && next_t == n_fresh + gridDim.x - 1u) {
          *sched_ctr = 0u;                                 // every CTA fails exactly one draw; the last one resets the counter
        }
        mbar_wait(&sm.q_empty, (ui & 1u) ^ 1u);            // every Q K^T of the previous item has completed: its ring
        *(volatile int*)&sm.sched_code[ui & 1u] = code;    // entry (item ui - 2's slot) has been read by every consumer
        mbar_arrive(&sm.sched_full[ui & 1u]);
        if (code == ITEM_END) break;
        int q0, head, bat, j_begin, T, slot, lo;
        decode(code, q0, head, bat, j_begin, T, slot, lo);
        mbar_expect_tx(&sm.q_full, TILE_BYTES);
#pragma unroll
        for (int blk = 0; blk < NBLK; ++blk) tma_load_4d(sm.q[blk], &tm_q, &sm.q_full, blk * HB, head, q0, bat);
        int so, t, tseg, lseg;                            // segment walk order, tile inside it, its tiles and rows
        locate(j_begin, so, t, tseg, lseg);
        for (int j = 0; j < T; ++j, ++t, ++g) {
          if (t == tseg) { t = 0; ++so; tseg = segs.tile0[so + 1] - segs.tile0[so]; }
          int seg = own_seg + so;
          if (seg >= nseg) seg -= nseg;
          const void* map = &tm_kv_own;
          if (seg != own_seg) {
            const int r = segs.rank[seg];
            if ((t == 0 || j == 0) && wait_flags) {
              spin_until<false>(flag_ptr(comm, comm.rank, idx, r), rd, comm.spin_timeout_ns);
              // the acquire above is a generic-proxy read; the peers' rows are fetched next through the async proxy (TMA)
              asm volatile("fence.proxy.async.global;" ::: "memory");
            }
            map = kvmaps + (size_t)(rd % DF_NBANKS) * comm.world + r;
          }
          const uint32_t ks = g % KSTAGES, vs = g % VSTAGES;
          mbar_wait(&sm.k_empty[ks], ((g / KSTAGES) & 1u) ^ 1u);
          mbar_expect_tx(&sm.k_full[ks], TILE_BYTES);
#pragma unroll
          for (int blk = 0; blk < NBLK; ++blk) tma_load_4d(sm.k[ks][blk], map, &sm.k_full[ks], blk * HB, head, t * BN, bat);
          mbar_wait(&sm.v_empty[vs], ((g / VSTAGES) & 1u) ^ 1u);
          mbar_expect_tx(&sm.v_full[vs], TILE_BYTES);
#pragma unroll
          for (int blk = 0; blk < NBLK; ++blk) tma_load_4d(sm.v[vs][blk], map, &sm.v_full[vs], blk * HB, heads + head, t * BN, bat);
        }
      }
    }
  } else {
    // =============================================================== consumers (warps 0-7): S, softmax, P V, epilogue
    // Warpgroup wg owns Q rows [64 wg, 64 wg + 64).  In the wgmma accumulator fragment thread t of warp w holds rows
    // rA = 64 wg + 16 (w & 3) + t/4 and rB = rA + 8, columns 8i + 2(t%4) + {0,1}: s[4i + {0,1}] (row rA), s[4i + {2,3}] (row rB).
    setmaxnreg_inc<CONSUMER_REGS>();
    const int wg = warp >> 2;
    const int c4 = lane & 3;
    const int rowA = wg * 64 + (warp & 3) * 16 + (lane >> 2);
    const uint32_t q_base = smem_u32(sm.q) + wg * 64 * 128;
    uint32_t g = 0;                                                // K/V tiles processed so far by this CTA (barrier phases)
    // Ping-pong: a warpgroup issues its MMAs of a slice only in its turn (named barrier TURN_BAR + wg) and then hands the turn
    // to the other one, so one warpgroup's softmax runs under the other's MMAs instead of both waiting on the same tiles in
    // step.  Both warpgroups take the same number of turns (they walk the same items and slices); warpgroup 0 takes the first
    // turn, and its final sync below consumes warpgroup 1's last hand-over.
    auto turn_begin = [&]() {
      if constexpr (PINGPONG) {
        if (wg == 0) named_bar_sync<TURN_BAR, 256>(); else named_bar_sync<TURN_BAR + 1, 256>();
      }
    };
    auto turn_end = [&]() {
      if constexpr (PINGPONG) {
        if (wg == 0) named_bar_arrive<TURN_BAR + 1, 256>(); else named_bar_arrive<TURN_BAR, 256>();
      }
    };
    if (PINGPONG && wg == 1) named_bar_arrive<TURN_BAR, 256>();
    for (uint32_t ui = 0;; ++ui) {
      mbar_wait(&sm.sched_full[ui & 1u], (ui >> 1) & 1u);
      const int code = *(volatile int*)&sm.sched_code[ui & 1u];
      if (code == ITEM_END) {
        if (PINGPONG && wg == 0) named_bar_sync<TURN_BAR, 256>();
        break;
      }
      int q0, head, bat, j_begin, T, slot, lo;
      decode(code, q0, head, bat, j_begin, T, slot, lo);
      // exponent references of rows rA / rB, kept NEGATED and in log2 units: P = 2^(S * scale_log2 + n)
      float nA = INFINITY, nB = INFINITY;
      float lA = 0.f, lB = 0.f;                                    // partial row sums over this thread's columns
      float o[NBLK * 32];
#pragma unroll
      for (int i = 0; i < NBLK * 32; ++i) o[i] = 0.f;
      float s[SN / 2];                                             // S of the current slice, then its P in fp32
      uint32_t pk[SN / 4];                                         // P of a slice packed to fp16: the A operand of its P V
      auto issue_s = [&](uint32_t ks, int sub) {                   // S = Q K^T of slice `sub` of K stage ks
        const uint32_t k_addr = smem_u32(sm.k[ks]) + sub * SN * 128;
        wgmma_fence();
#pragma unroll
        for (int blk = 0; blk < NBLK; ++blk)
#pragma unroll
          for (int kk = 0; kk < HB / 16; ++kk)
            wgmma_ss<SN>(s, smem_desc(q_base + blk * BLK_BYTES + kk * 32, 16, 1024), smem_desc(k_addr + blk * BLK_BYTES + kk * 32, 16, 1024),
                         (blk | kk) > 0);
        wgmma_commit();
      };
      auto issue_pv = [&](uint32_t vs, int sub) {                  // O += P V of slice `sub` of V stage vs
        const uint32_t v_addr = smem_u32(sm.v[vs]) + sub * SN * 128;
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < SN / 16; ++kk)
#pragma unroll
          for (int blk = 0; blk < NBLK; ++blk)
            wgmma_rs_n64(o + 32 * blk, pk + 4 * kk, smem_desc(v_addr + blk * BLK_BYTES + kk * 2048, 16384, 1024), 1u);
        wgmma_commit();
      };
      mbar_wait(&sm.q_full, ui & 1u);
      // The item's K/V tiles are processed in NSUB column slices of SN K/V rows (online softmax per slice): for the wider heads
      // two slices of 64 keep the S fragment at 32 registers next to the larger O fragment.  Overlapped order, per slice i:
      //   issue S_i = Q K_i^T and O += P_{i-1} V_{i-1} (two commit groups) -> wait<1> (S_i retired) -> row maxima, exp2, sums
      //   of S_i in place -> wait<0> (P V retired) -> rescale O if slice i moved the reference -> pack P_i
      // and the last slice's P V after the loop.  P_{i-1} stays in `pk` until its P V retires; the tensor cores run P V while
      // this warpgroup runs the softmax.
      int so, t, tseg, lseg;                                       // segment walk order, tile inside it, its tiles and rows
      locate(j_begin, so, t, tseg, lseg);
      for (int j = 0; j < T; ++j, ++t, ++g) {
        if (t == tseg) { t = 0; ++so; tseg = segs.tile0[so + 1] - segs.tile0[so]; lseg = segs.len[so]; }
        const int valid = min(BN, lseg - t * BN);
        const uint32_t ks = g % KSTAGES, vs = g % VSTAGES;
#pragma unroll
        for (int sub = 0; sub < NSUB; ++sub) {
          // ---- S = Q K_j^T (this slice), and the previous slice's P V
          if (sub == 0) mbar_wait(&sm.k_full[ks], (g / KSTAGES) & 1u);
          const bool pv = OVERLAP && (j > 0 || sub > 0);
          const int subp = sub > 0 ? sub - 1 : NSUB - 1;             // the previous slice: tile gp, slice subp
          const uint32_t gp = sub > 0 ? g : g - 1u, vsp = gp % VSTAGES;
          if (pv && subp == 0) mbar_wait(&sm.v_full[vsp], (gp / VSTAGES) & 1u);
          turn_begin();
          issue_s(ks, sub);
          // Always two commit groups in the overlapped order (an empty one when there is no previous slice): with the same
          // wait counts on every path ptxas keeps the wgmmas asynchronous instead of serialising them (C7514 / C7515).
          if (pv) issue_pv(vsp, subp);
          else if (OVERLAP) wgmma_commit();
          turn_end();
          wgmma_wait<OVERLAP ? 1 : 0>();
          fence_regs<SN / 2>(s);
          if (sub == NSUB - 1) {
            __syncwarp();
            if (lane == 0) {
              mbar_arrive(&sm.k_empty[ks]);
              if (j + 1 == T) mbar_arrive(&sm.q_empty);    // last Q K^T of this item: the Q tile may be overwritten
            }
          }
          const int vcols = valid - sub * SN;              // valid columns of this slice
          if (vcols < SN) {                                // ragged last tile of a segment only (warp-uniform branch)
#pragma unroll
            for (int i = 0; i < SN / 8; ++i)
#pragma unroll
              for (int k = 0; k < 2; ++k)
                if (8 * i + 2 * c4 + k >= vcols) { s[4 * i + k] = -INFINITY; s[4 * i + 2 + k] = -INFINITY; }
          }
          // ---- row maxima; lazy rescale: keep the old reference while the maximum moved by < 2^8 (P stays below 2^8 in fp16)
          float mA0 = -INFINITY, mA1 = -INFINITY, mB0 = -INFINITY, mB1 = -INFINITY;   // two chains per row
#pragma unroll
          for (int i = 0; i < SN / 8; i += 2) {
            mA0 = fmaxf(mA0, fmaxf(s[4 * i], s[4 * i + 1]));
            mB0 = fmaxf(mB0, fmaxf(s[4 * i + 2], s[4 * i + 3]));
            mA1 = fmaxf(mA1, fmaxf(s[4 * i + 4], s[4 * i + 5]));
            mB1 = fmaxf(mB1, fmaxf(s[4 * i + 6], s[4 * i + 7]));
          }
          float mA = fmaxf(mA0, mA1), mB = fmaxf(mB0, mB1);
          mA = fmaxf(mA, __shfl_xor_sync(0xffffffffu, mA, 1));
          mB = fmaxf(mB, __shfl_xor_sync(0xffffffffu, mB, 1));
          mA = fmaxf(mA, __shfl_xor_sync(0xffffffffu, mA, 2));
          mB = fmaxf(mB, __shfl_xor_sync(0xffffffffu, mB, 2));
          const float dA = fmaf(mA, scale_log2, nA), dB = fmaf(mB, scale_log2, nB);    // log2 of the largest P of the slice
          const bool moveA = dA > 8.f, moveB = dB > 8.f;
          float alphaA = 1.f, alphaB = 1.f;                // O's rescale waits for the P V in flight (it accumulates into O)
          if (moveA) { alphaA = ex2(-dA); nA = -mA * scale_log2; lA *= alphaA; }
          if (moveB) { alphaB = ex2(-dB); nB = -mB * scale_log2; lB *= alphaB; }
          // ---- P = 2^(S * scale_log2 + n) in place, row sums
#pragma unroll
          for (int i = 0; i < SN / 8; ++i) {
            const int grp = sub * (SN / 8) + i;            // column group of the 128-wide tile row
#pragma unroll
            for (int k = 0; k < 4; ++k) {
              const float x = fmaf(s[4 * i + k], scale_log2, k < 2 ? nA : nB);
              s[4 * i + k] = ((grp * kEmuGroups) / 16 != ((grp + 1) * kEmuGroups) / 16) ? ex2_poly(x) : ex2(x);
            }
            lA += s[4 * i] + s[4 * i + 1];
            lB += s[4 * i + 2] + s[4 * i + 3];
          }
          if (OVERLAP) {
            wgmma_wait<0>();
            fence_regs<NBLK * 32>(o);
          }
          if (pv) {                                        // the previous slice's P V has retired: its V stage and `pk` are free
            if (subp == NSUB - 1) {
              __syncwarp();
              if (lane == 0) mbar_arrive(&sm.v_empty[vsp]);
            }
          }
          if (moveA) {
#pragma unroll
            for (int i = 0; i < NBLK * 8; ++i) { o[4 * i] *= alphaA; o[4 * i + 1] *= alphaA; }
          }
          if (moveB) {
#pragma unroll
            for (int i = 0; i < NBLK * 8; ++i) { o[4 * i + 2] *= alphaB; o[4 * i + 3] *= alphaB; }
          }
          // ---- P packed to fp16 as the A fragment of the P V wgmmas
#pragma unroll
          for (int i = 0; i < SN / 8; ++i) {
            pk[2 * i] = pack_h2(s[4 * i], s[4 * i + 1]);
            pk[2 * i + 1] = pack_h2(s[4 * i + 2], s[4 * i + 3]);
          }
          if constexpr (!OVERLAP) {                        // serial order: O += P V_j (this slice) right away
            if (sub == 0) mbar_wait(&sm.v_full[vs], (g / VSTAGES) & 1u);
            issue_pv(vs, sub);
            wgmma_wait<0>();
            fence_regs<NBLK * 32>(o);
            if (sub == NSUB - 1) {
              __syncwarp();
              if (lane == 0) mbar_arrive(&sm.v_empty[vs]);
            }
          }
        }
      }
      if constexpr (OVERLAP) {                             // P V of the item's last slice (tile g - 1, slice NSUB - 1)
        const uint32_t vsp = (g - 1u) % VSTAGES;
        if (NSUB == 1) mbar_wait(&sm.v_full[vsp], ((g - 1u) / VSTAGES) & 1u);
        turn_begin();
        issue_pv(vsp, NSUB - 1);
        turn_end();
        wgmma_wait<0>();
        fence_regs<NBLK * 32>(o);
        __syncwarp();
        if (lane == 0) mbar_arrive(&sm.v_empty[vsp]);
      }
      // ---- epilogue: quad-reduce the row sums, then O / l -> fp16 -> HBM (or an fp32 partial of a split unit)
      lA += __shfl_xor_sync(0xffffffffu, lA, 1); lB += __shfl_xor_sync(0xffffffffu, lB, 1);
      lA += __shfl_xor_sync(0xffffffffu, lA, 2); lB += __shfl_xor_sync(0xffffffffu, lB, 2);
      const bool partial = slot >= 0;
      bool finish = !partial;                            // this CTA writes the output rows
      float denA = lA, denB = lB;
      if (partial) {
        // ---- un-normalised fp32 partial (reference -n) -> workspace; the last part of this unit to arrive merges
        const int64_t prow = (int64_t)slot * BM + rowA;                  // row of this part's partial in the workspace
        if (c4 == 0) { part_ml[prow] = make_float2(-nA, lA); part_ml[prow + 8] = make_float2(-nB, lB); }
#pragma unroll
        for (int i = 0; i < NBLK * 8; ++i) {
          const int col = 8 * i + 2 * c4;
          *reinterpret_cast<float2*>(part_o + prow * (NBLK * HB) + col) = make_float2(o[4 * i], o[4 * i + 1]);
          *reinterpret_cast<float2*>(part_o + (prow + 8) * (NBLK * HB) + col) = make_float2(o[4 * i + 2], o[4 * i + 3]);
        }
        __threadfence();
        asm volatile("bar.sync 1, 256;" ::: "memory");
        if (threadIdx.x == 0) {
          const unsigned int tk = atomicAdd(part_cnt + lo, 1u);
          sm.ticket = tk;
          if (tk == (unsigned int)sched.P - 1) part_cnt[lo] = 0;        // self-resetting: the next launch is stream-ordered
        }
        asm volatile("bar.sync 1, 256;" ::: "memory");
        finish = sm.ticket == (unsigned int)sched.P - 1;
        if (finish) {
          __threadfence();
          // merge: out = sum_p w_p O_p / sum_p w_p l_p,  w_p = 2^(m_p - max_p m_p)   (parts of unit `lo`: slots lo*P ..)
          const int s0 = lo * sched.P;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int64_t r = rowA + 8 * h;
            float m_max = -INFINITY;
            for (int pp = 0; pp < sched.P; ++pp) m_max = fmaxf(m_max, ld_f2(part_ml + (int64_t)(s0 + pp) * BM + r).x);
            float den = 0.f;
#pragma unroll
            for (int i = 0; i < NBLK * 8; ++i) { o[4 * i + 2 * h] = 0.f; o[4 * i + 2 * h + 1] = 0.f; }
            for (int pp = 0; pp < sched.P; ++pp) {
              const float2 ml = ld_f2(part_ml + (int64_t)(s0 + pp) * BM + r);
              const float w = ex2(ml.x - m_max);        // references are kept in log2 units
              den = fmaf(w, ml.y, den);
              const float2* src = reinterpret_cast<const float2*>(part_o + ((int64_t)(s0 + pp) * BM + r) * (NBLK * HB));
#pragma unroll
              for (int i = 0; i < NBLK * 8; ++i) {
                const float2 v = ld_f2(src + 4 * i + c4);
                o[4 * i + 2 * h] = fmaf(w, v.x, o[4 * i + 2 * h]);
                o[4 * i + 2 * h + 1] = fmaf(w, v.y, o[4 * i + 2 * h + 1]);
              }
            }
            if (h == 0) denA = den; else denB = den;
          }
        }
      }
      if (finish) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = rowA + 8 * h;
          if (q0 + row >= lq) continue;
          const float inv = 1.f / (h == 0 ? denA : denB);
          __half* dst = out + ((int64_t)bat * lq + q0 + row) * o_pitch + (int64_t)head * d;
#pragma unroll
          for (int i = 0; i < NBLK * 8; ++i) {
            const int col = 8 * i + 2 * c4;
            if (col < d)                                 // d % 8 == 0: a column pair is entirely inside or outside the head
              *reinterpret_cast<uint32_t*>(dst + col) = pack_h2(o[4 * i + 2 * h] * inv, o[4 * i + 2 * h + 1] * inv);
          }
        }
      }
    }   // work items
  }
}


// ----------------------------------------------------------------------------------------- host side
// 4-D view [d, nheads, rows, batch] of a row-major [batch, rows, pitch] fp16 matrix; box = [64, 1, 128, 1], 128B swizzle.
int make_map(CUtensorMap* m, const void* base, int d, int nheads, int rows, int batch, int64_t pitch) {
  EncodeTiledFn enc = tensor_map_encoder();
  DF_REQUIRE(enc != nullptr, "cuTensorMapEncodeTiled is not available from this driver");
  cuuint64_t dims[4] = {(cuuint64_t)d, (cuuint64_t)nheads, (cuuint64_t)rows, (cuuint64_t)batch};
  cuuint64_t strides[3] = {(cuuint64_t)d * 2, (cuuint64_t)pitch * 2, (cuuint64_t)rows * pitch * 2};
  cuuint32_t box[4] = {HB, 1, BN, 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  DF_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed (%d): base=%p d=%d heads=%d rows=%d batch=%d pitch=%lld", (int)r,
             base, d, nheads, rows, batch, (long long)pitch);
  return 0;
}

}  // namespace

// Tensor maps of every (bank, member) slot of a K/V tensor; member s holds seg_len_host[s] rows (its own strip's tokens).
extern "C" int df_attn_make_kvmaps_ragged(df_comm_t comm, uint64_t tensor_off, uint64_t slot_bytes, int b,
                                          const int32_t* seg_len_host, int heads, int d, void* maps_out, void* stream) {
  static_assert(sizeof(CUtensorMap) == DF_TENSORMAP_BYTES, "tensor map size");
  DF_REQUIRE(d % 8 == 0 && d >= 8 && d <= 192, "df_attn: head dim %d not supported (multiple of 8, <= 192)", d);
  DF_REQUIRE(seg_len_host != nullptr && comm.world >= 1 && comm.world <= DF_MAX_WORLD, "df_attn_make_kvmaps: bad lengths");
  for (int s = 0; s < comm.world; ++s) {
    DF_REQUIRE(seg_len_host[s] >= 1, "df_attn_make_kvmaps: member %d has %d K/V rows", s, seg_len_host[s]);
    DF_REQUIRE(slot_bytes >= (uint64_t)b * seg_len_host[s] * 2 * heads * d * 2, "df_attn_make_kvmaps: slot too small");
  }
  CUtensorMap host[DF_NBANKS * DF_MAX_WORLD];
  memset(host, 0, sizeof(host));
  const int64_t pitch = 2 * (int64_t)heads * d;
  for (int k = 0; k < DF_NBANKS; ++k)
    for (int s = 0; s < comm.world; ++s) {
      const char* base = slot_ptr(comm, comm.rank, (uint32_t)k, tensor_off, slot_bytes, s);
      if (int rc = make_map(&host[k * comm.world + s], base, d, 2 * heads, seg_len_host[s], b, pitch)) return rc;
    }
  DF_CHECK_CUDA(cudaMemcpyAsync(maps_out, host, sizeof(CUtensorMap) * DF_NBANKS * comm.world, cudaMemcpyHostToDevice,
                                (cudaStream_t)stream));
  DF_CHECK_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
  return 0;
}

extern "C" int df_attn_make_kvmaps(df_comm_t comm, uint64_t tensor_off, uint64_t slot_bytes, int b, int lseg, int heads,
                                   int d, void* maps_out, void* stream) {
  int32_t len[DF_MAX_WORLD];
  for (int s = 0; s < DF_MAX_WORLD; ++s) len[s] = lseg;
  return df_attn_make_kvmaps_ragged(comm, tensor_off, slot_bytes, b, len, heads, d, maps_out, stream);
}

namespace {
constexpr int kMinPartTiles = 8;    // a part of a split unit keeps at least this many K/V tiles (Q load + partial write + merge per part)
// Grid and work schedule of a launch (see the kernel): G resident CTAs, `a` whole units per CTA, R left-over units in P parts.
// Policy: the left-over units of a grid that already fills the SMs are not cut -- the R CTAs of the last round have the memory
// system to themselves, which a balanced tail would trade for partial writes and a merge -- so P > 1 only when the units leave
// at least half of the SMs idle AND every part keeps >= 8 K/V tiles.  t_all: the K/V tiles of all segments together.
void plan_schedule(int b, int lq, int t_all, int heads, bool have_ws, int& grid, Sched& sc) {
  const long long slots = sm_count();
  const long long units = (long long)((lq + BM - 1) / BM) * heads * b;
  sc.units = (int)units;
  if (units >= slots) {
    grid = (int)slots;
    sc.a = (int)(units / slots);
    sc.R = (int)(units % slots);
    sc.P = 1;
    sc.dyn = have_ws ? 1 : 0;                          // the ticket counter lives in the workspace
  } else {
    long long p = have_ws ? slots / units : 1;
    if (p > t_all / kMinPartTiles) p = t_all / kMinPartTiles;
    if (p < 1) p = 1;
    sc.a = 0; sc.R = (int)units; sc.P = (int)p; sc.dyn = 0;
    grid = (int)(units * p);
  }
}
// workspace: [1 KiB header: ticket counter of the dynamic schedule] [arrival tickets of split units] [partials (m, l)] [partials O]
constexpr size_t WS_HEADER = 1024;
size_t workspace_need(const Sched& sc, int d) {
  if (sc.P <= 1) return WS_HEADER;
  const size_t hd_pad = (size_t)((d + HB - 1) / HB) * HB;
  const size_t parts = (size_t)sc.R * sc.P;
  return WS_HEADER + 1024 + ((size_t)sc.R * sizeof(unsigned int) + 255) / 256 * 256 + parts * BM * sizeof(float2) + parts * BM * hd_pad * sizeof(float);
}
// K/V tiles of all nseg segments; seg_len_host == nullptr: every segment has lseg rows
int total_tiles(int nseg, int lseg, const int32_t* seg_len_host) {
  int t = 0;
  for (int s = 0; s < nseg; ++s) t += ((seg_len_host ? seg_len_host[s] : lseg) + BN - 1) / BN;
  return t;
}

int attn_fwd_impl(df_comm_t comm, const void* q, const void* kv_own, void* out, const void* kvmaps, int b, int lq,
                  const int32_t* seg_len, int heads, int d, int64_t q_pitch, int64_t kv_pitch, int64_t o_pitch, int nseg,
                  int own_seg, const int32_t* seg_rank_host, int idx, int wait_flags, float scale, void* workspace,
                  size_t workspace_bytes, void* stream) {
  DF_REQUIRE(d % 8 == 0 && d >= 8 && d <= 192, "df_attn_fwd: head dim %d not supported (multiple of 8, <= 192)", d);
  DF_REQUIRE(nseg >= 1 && nseg <= DF_MAX_WORLD && own_seg >= 0 && own_seg < nseg, "df_attn_fwd: bad segment layout");
  DF_REQUIRE(nseg == 1 || kvmaps != nullptr, "df_attn_fwd: peer segments need tensor maps (df_attn_make_kvmaps)");
  DF_REQUIRE(q_pitch % 8 == 0 && kv_pitch % 8 == 0 && o_pitch % 8 == 0 && ((uintptr_t)q % 16) == 0 &&
                 ((uintptr_t)kv_own % 16) == 0 && ((uintptr_t)out % 16) == 0,
             "df_attn_fwd: q/kv/out must be 16-byte aligned with pitches multiple of 8");
  DF_REQUIRE(b >= 1 && lq >= 1 && heads >= 1 && heads <= 65535 && b <= 65535, "df_attn_fwd: bad shape");
  for (int s = 0; s < nseg; ++s) DF_REQUIRE(seg_len[s] >= 1, "df_attn_fwd: segment %d has %d K/V rows", s, seg_len[s]);
  CUtensorMap tq, tkv;
  if (int rc = make_map(&tq, q, d, heads, lq, b, q_pitch)) return rc;
  if (int rc = make_map(&tkv, kv_own, d, 2 * heads, seg_len[own_seg], b, kv_pitch)) return rc;
  SegInfo segs;
  memset(&segs, 0, sizeof(segs));
  for (int s = 0; s < DF_MAX_WORLD; ++s) segs.rank[s] = (s < nseg && seg_rank_host) ? seg_rank_host[s] : 0;
  for (int o = 0; o < nseg; ++o) {                     // walk order: the own segment first, then the next ones cyclically
    const int s = (own_seg + o) % nseg;
    segs.len[o] = seg_len[s];
    segs.tile0[o + 1] = segs.tile0[o] + (seg_len[s] + BN - 1) / BN;
  }
  const int t_all = segs.tile0[nseg];
  const float sc = (scale > 0.f ? scale : 1.f / sqrtf((float)d)) * 1.4426950408889634f;
  const int nblk = (d + HB - 1) / HB;
  // work schedule; the dynamic ticket counter and the K/V split of small grids need a ZERO-INITIALISED workspace of
  // df_attn_workspace_bytes() (self-resetting counters); without one every CTA walks a static list of whole units
  int grid_x;
  Sched sched;
  plan_schedule(b, lq, t_all, heads, true, grid_x, sched);
  if (workspace == nullptr || workspace_bytes < workspace_need(sched, d))
    plan_schedule(b, lq, t_all, heads, false, grid_x, sched);
  unsigned int* sched_ctr = sched.dyn ? (unsigned int*)workspace : nullptr;
  unsigned int* part_cnt = nullptr;
  float2* part_ml = nullptr;
  float* part_o = nullptr;
  if (sched.P > 1) {
    char* w = (char*)workspace + WS_HEADER;
    part_cnt = (unsigned int*)w;
    w += ((size_t)sched.R * sizeof(unsigned int) + 255) / 256 * 256;
    part_ml = (float2*)w;
    w += (size_t)sched.R * sched.P * BM * sizeof(float2);
    part_o = (float*)(((uintptr_t)w + 255) / 256 * 256);
  }
  dim3 grid((unsigned)grid_x, 1, 1);
#define DF_LAUNCH_FMHA(NB)                                                                                                  \
  {                                                                                                                          \
    static bool attr_set = false;                                                                                            \
    const size_t smem_bytes = sizeof(SmemT<NB, Cfg<NB>::KST, Cfg<NB>::VST>);                                                 \
    if (!attr_set) {                                                                                                         \
      DF_CHECK_CUDA(cudaFuncSetAttribute(fmha_fwd_kernel<NB>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes)); \
      attr_set = true;                                                                                                       \
    }                                                                                                                        \
    fmha_fwd_kernel<NB><<<grid, NTHREADS, smem_bytes, (cudaStream_t)stream>>>(                                             \
        tq, tkv, (const CUtensorMap*)kvmaps, comm, segs, (__half*)out, lq, heads, d, o_pitch, nseg, own_seg, idx, wait_flags,  \
        sc, sched, part_o, part_ml, part_cnt, sched_ctr);                                                                    \
  }
  if (nblk == 1) DF_LAUNCH_FMHA(1) else if (nblk == 2) DF_LAUNCH_FMHA(2) else DF_LAUNCH_FMHA(3)
#undef DF_LAUNCH_FMHA
  DF_CHECK_LAUNCH();
  return 0;
}
}  // namespace

extern "C" size_t df_attn_workspace_bytes_ragged(int b, int lq, const int32_t* seg_len_host, int nseg, int heads, int d) {
  if (seg_len_host == nullptr || nseg < 1 || nseg > DF_MAX_WORLD) return 0;
  int grid;
  Sched sc;
  plan_schedule(b, lq, total_tiles(nseg, 0, seg_len_host), heads, true, grid, sc);
  return workspace_need(sc, d);
}

extern "C" size_t df_attn_workspace_bytes(int b, int lq, int lseg, int nseg, int heads, int d) {
  int grid;
  Sched sc;
  plan_schedule(b, lq, total_tiles(nseg, lseg, nullptr), heads, true, grid, sc);
  return workspace_need(sc, d);
}

extern "C" int df_attn_fwd_ragged(df_comm_t comm, const void* q, const void* kv_own, void* out, const void* kvmaps, int b,
                                  int lq, const int32_t* seg_len_host, int heads, int d, int64_t q_pitch, int64_t kv_pitch,
                                  int64_t o_pitch, int nseg, int own_seg, const int32_t* seg_rank_host, int idx, int wait_flags,
                                  float scale, void* workspace, size_t workspace_bytes, void* stream) {
  DF_REQUIRE(seg_len_host != nullptr, "df_attn_fwd_ragged: segment lengths missing");
  DF_REQUIRE(nseg >= 1 && nseg <= DF_MAX_WORLD, "df_attn_fwd: bad segment layout");
  return attn_fwd_impl(comm, q, kv_own, out, kvmaps, b, lq, seg_len_host, heads, d, q_pitch, kv_pitch, o_pitch, nseg, own_seg,
                       seg_rank_host, idx, wait_flags, scale, workspace, workspace_bytes, stream);
}

extern "C" int df_attn_fwd(df_comm_t comm, const void* q, const void* kv_own, void* out, const void* kvmaps, int b, int lq,
                           int lseg, int heads, int d, int64_t q_pitch, int64_t kv_pitch, int64_t o_pitch, int nseg,
                           int own_seg, const int32_t* seg_rank_host, int idx, int wait_flags, float scale, void* workspace,
                           size_t workspace_bytes, void* stream) {
  int32_t len[DF_MAX_WORLD];
  for (int s = 0; s < DF_MAX_WORLD; ++s) len[s] = lseg;
  return attn_fwd_impl(comm, q, kv_own, out, kvmaps, b, lq, len, heads, d, q_pitch, kv_pitch, o_pitch, nseg, own_seg,
                       seg_rank_host, idx, wait_flags, scale, workspace, workspace_bytes, stream);
}
