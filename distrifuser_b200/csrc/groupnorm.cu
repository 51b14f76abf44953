// distrifuser_b200 -- GroupNorm with cross-rank sufficient statistics (NHWC fp16, or fp32 for the VAE decoder's upcast part).
// Replaces DistriGroupNorm.forward (distrifuser/modules/pp/groupnorm.py:14-97): the ~10 eager reduction /
// elementwise kernels and the 256-byte NCCL all_gather / all_reduce per layer become ONE launch (gn_fused_kernel): one HBM
// read with fp32 per-channel register accumulation, a grid barrier, the exchange of (E[x], E[x^2]) with the patch group through
// peer stores + release/acquire flags over NVLink, and the normalisation with optional fused SiLU.  It accepts a
// per-(sample, channel) addend so that ResnetBlock2D's `conv1(x) + time_emb` never materialises.
//
// One kernel for both element types (gn_fused_kernel<T>): 16-byte accesses carry 8 halves or 4 floats, statistics are fp32
// either way.  The fp32 instantiation serves activations that overflow fp16 (the SDXL VAE's up blocks reach 1e5), where the
// one-pass E[x^2] - E[x]^2 in fp32 cancels catastrophically once |mean| >> std.  So it accumulates around a shift K per
// (sample, group) -- the first element of the group in pixel 0 of the sample, the same value in every CTA -- and a rank's
// statistics are (mean, biased variance) instead of (mean, mean of squares); ranks combine them with the exact pooled
// formula var = sum_p w_p (var_p + (mean_p - mean)^2).  That form is not linear in the moments, so the fp32 kernel has the
// local and synchronous modes only (the ones the decoder uses).
#include <string.h>
#include <type_traits>

#include "common.cuh"

using namespace df;

namespace {

#ifdef DF_GN_TRACE
// %globaltimer stamps of one launch for kernel tuning (tools/trace_gn.py); compiled out by default
__device__ unsigned long long df_gn_trace[16];
#define GN_TR(slot, cond) do { if (cond) df_gn_trace[slot] = globaltimer_ns(); } while (0)
#else
#define GN_TR(slot, cond) do {} while (0)
#endif

struct GnPlan {
  int V;        // 16-byte channel vectors per pixel (C/8 halves, C/4 floats)
  int lanes;    // pixels processed concurrently by one CTA
  int threads;  // blockDim
  int nchunk;   // CTAs per sample
  int ppc;      // pixels per CTA
};

constexpr int kGnMaxSmem = 32 * 1024;   // dynamic shared memory of gn_fused_kernel: lanes * C <= 4096 moments

// 16-byte vector of the element type: E elements, unpacked to / packed from fp32
template <typename T> struct GnVec;
template <> struct GnVec<__half> {
  static constexpr int E = 8;
  __device__ __forceinline__ static void unpack(const int4& v, float* f) {
    const __half2* h = reinterpret_cast<const __half2*>(&v);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float2 t = __half22float2(h[i]);
      f[2 * i] = t.x;
      f[2 * i + 1] = t.y;
    }
  }
  __device__ __forceinline__ static int4 pack(const float* f) {
    int4 o;
    __half2* oh = reinterpret_cast<__half2*>(&o);
#pragma unroll
    for (int j = 0; j < 4; ++j) oh[j] = __floats2half2_rn(f[2 * j], f[2 * j + 1]);
    return o;
  }
  __device__ __forceinline__ static float to_float(__half v) { return __half2float(v); }
};
template <> struct GnVec<float> {
  static constexpr int E = 4;
  __device__ __forceinline__ static void unpack(const int4& v, float* f) {
    f[0] = __int_as_float(v.x); f[1] = __int_as_float(v.y); f[2] = __int_as_float(v.z); f[3] = __int_as_float(v.w);
  }
  __device__ __forceinline__ static int4 pack(const float* f) {
    return make_int4(__float_as_int(f[0]), __float_as_int(f[1]), __float_as_int(f[2]), __float_as_int(f[3]));
  }
  __device__ __forceinline__ static float to_float(float v) { return v; }
};
// fp32: shifted statistics, exchanged as (mean, variance) (see the file comment)
template <typename T> constexpr bool kGnShift = std::is_same<T, float>::value;

template <typename T> int gn_resident_ctas();

template <typename T>
inline GnPlan gn_plan(int b, int h, int w, int C) {
  GnPlan p;
  p.V = C / GnVec<T>::E;
  p.lanes = 512 / p.V;
  if (p.lanes < 1) p.lanes = 1;
  int active = p.lanes * p.V;
  p.threads = (active + 31) / 32 * 32;
  int hw = h * w;
  int want = (2 * kSmCount + b - 1) / b;                  // ~2 CTAs per SM over the batch
  int cap = hw / (p.lanes * 8);                      // >= 8 pixels per thread
  if (cap < 1) cap = 1;
  auto split = [&](int n) { p.ppc = (hw + n - 1) / n; p.nchunk = (hw + p.ppc - 1) / p.ppc; };
  split(want < cap ? want : cap);
  // the grid barrier needs every CTA resident at once: fewer, longer chunks where the batch would not fit
  const int resident = gn_resident_ctas<T>();
  if (p.nchunk * b > resident && resident >= b) split(resident / b);
  return p;
}

// The shift K of group g of sample b (fp32 only): x + addend at pixel 0, channel g * C / G
template <typename T>
__device__ __forceinline__ float gn_shift(const T* __restrict__ x, const T* __restrict__ addend, int64_t addend_pitch, int b,
                                          int hw, int C, int cpg, int g) {
  const int ch = g * cpg;
  float k = GnVec<T>::to_float(x[(size_t)b * hw * C + ch]);
  if (addend) k += GnVec<T>::to_float(addend[(size_t)b * addend_pitch + ch]);
  return k;
}

struct GnExchange {   // grid barrier and cross-rank exchange of the statistics
  df_comm_t c;
  unsigned int* ticket;
  int bG, nchunk_total;
  float inv_ne, bessel, eps;
  int mode, neg_fb, idx;
  uint64_t tensor_off, slot_bytes;
  uint32_t group_mask;
  // statistics of source p weigh wgt[p] / sum(wgt) (its share of the patch group's rows, reduced by the gcd: equal strips give
  // wgt = 1 and inv_w = 1/n)
  int32_t wgt[DF_MAX_WORLD];
  float inv_w;
};

// Fused conv-halo handling of the normalise pass (GroupNorm -> SiLU -> 3x3 conv, the ResnetBlock2D pattern): the output goes
// into the interior rows of a [b, h+2, w, C] buffer, this rank's first / last output rows are ALSO stored into the patch
// neighbours' arena slots of the conv (replaces df_halo_push), and the two margin rows are filled from the neighbours' slots
// of the read epoch (replaces df_halo_assemble and its full-activation copy; distrifuser/modules/pp/conv2d.py:72-93).
struct GnHalo {
  int enabled;
  int h, w;                 // local rows, width
  int up, down;             // patch neighbours (communicator indices) or -1 at the image border
  int push;                 // ship this call's boundary rows (synchronous step: for this step; asynchronous: for the next one)
  int wait_flags;
  int idx;                  // comm tensor index of the CONV
  uint64_t off, slot_bytes;
  unsigned int* ticket2;    // CTA ticket of the normalise pass (self-resetting)
  df_comm_t c;
};

// Statistics pass of one CTA: the group moments of its pixels -> partial[] (fp32: of x - K, the group's shift).  Loads use the
// default caching, so that the normalise pass finds this CTA's pixels in L1 / L2.
template <typename T>
__device__ __forceinline__ void gn_moments(const T* __restrict__ x, const T* __restrict__ addend, int64_t addend_pitch,
                                           float2* __restrict__ partial, int hw, int C, int G, int V, int lanes,
                                           int ppc, float2* ch) {
  using Vec = GnVec<T>;
  constexpr int E = Vec::E;
  const int b = blockIdx.y, chunk = blockIdx.x, nchunk = gridDim.x;
  const int tid = threadIdx.x;
  const int v = tid % V, pl = tid / V;
  if (pl < lanes) {
    const int p0 = chunk * ppc, p1 = min(hw, p0 + ppc);
    const T* base = x + ((size_t)b * hw) * C + (size_t)v * E;
    float s[E], ss[E], ad[E];
#pragma unroll
    for (int j = 0; j < E; ++j) s[j] = ss[j] = ad[j] = 0.f;
    if (addend) Vec::unpack(ld_v4(addend + (size_t)b * addend_pitch + (size_t)v * E), ad);   // per-(sample, channel) bias, e.g. the time embedding
    if constexpr (kGnShift<T>) {                 // moments of x - K: ad[j] - K keeps one add per element
      const int cpg = C / G;
#pragma unroll
      for (int j = 0; j < E; ++j) ad[j] -= gn_shift(x, addend, addend_pitch, b, hw, C, cpg, (v * E + j) / cpg);
    }
    int p = p0 + pl;
    constexpr int U = 8;                          // loads in flight per thread (one DRAM latency round per 8 pixels)
    for (; p + (U - 1) * lanes < p1; p += U * lanes) {
      int4 r[U];
#pragma unroll
      for (int u = 0; u < U; ++u) r[u] = ld_v4(base + (size_t)(p + u * lanes) * C);
#pragma unroll
      for (int u = 0; u < U; ++u) {
        float f[E];
        Vec::unpack(r[u], f);
#pragma unroll
        for (int j = 0; j < E; ++j) { float t = f[j] + ad[j]; s[j] += t; ss[j] = fmaf(t, t, ss[j]); }
      }
    }
    for (; p < p1; p += lanes) {
      float f[E];
      Vec::unpack(ld_v4(base + (size_t)p * C), f);
#pragma unroll
      for (int j = 0; j < E; ++j) { float t = f[j] + ad[j]; s[j] += t; ss[j] = fmaf(t, t, ss[j]); }
    }
#pragma unroll
    for (int j = 0; j < E; ++j) ch[(size_t)pl * C + v * E + j] = make_float2(s[j], ss[j]);
  }
  GN_TR(1, blockIdx.x == 0 && blockIdx.y == 0 && tid == 0);
  __syncthreads();
  // fold channels x pixel-lanes into the G groups in a FIXED order (no atomics: results are bit-reproducible run to run)
  __shared__ float2 fold[256];
  const int cpg = C / G;
  const int parts = min(256 / G, 32);
  if (tid < parts * G) {
    const int g = tid % G, part = tid / G;
    const int per_group = cpg * lanes;
    float a = 0.f, q = 0.f;
    for (int e = part; e < per_group; e += parts) {
      const int pl2 = e / cpg, cc = e - pl2 * cpg;
      const float2 t = ch[(size_t)pl2 * C + g * cpg + cc];
      a += t.x; q += t.y;
    }
    fold[part * G + g] = make_float2(a, q);
  }
  __syncthreads();
  for (int g = tid; g < G; g += blockDim.x) {
    float a = 0.f, q = 0.f;
    for (int part = 0; part < parts; ++part) { a += fold[part * G + g].x; q += fold[part * G + g].y; }
    partial[((size_t)b * nchunk + chunk) * G + g] = make_float2(a, q);
  }
}

// ---- after the grid barrier EVERY CTA finishes the statistics of its own sample
__device__ __forceinline__ float2 ld_cg_f2(const float2* p) {      // L2 load: the partials were written during this launch
  float2 r;
  asm volatile("ld.global.cg.v2.f32 {%0, %1}, [%2];" : "=f"(r.x), "=f"(r.y) : "l"(p) : "memory");
  return r;
}
// (mean, mean of squares) of the G groups of sample b over the per-CTA partials, in a FIXED order (bit-reproducible):
// thread (g, r) sums the partials r, r + tpp, ... of group g (a warp reads 32 consecutive groups of one partial row: coalesced),
// then G threads fold the tpp pieces.  `red` holds G * tpp entries, `mine` G entries.  fp32: `mine` is (mean, biased variance),
// from the moments of x - K.
template <typename T>
__device__ __forceinline__ void gn_reduce_sample(const float2* __restrict__ partial, int b, int G, int nchunk, float inv_ne,
                                                 float2* red, float2* mine, const T* __restrict__ x, const T* __restrict__ addend,
                                                 int64_t addend_pitch, int hw, int C) {
  const int tid = threadIdx.x, nthr = blockDim.x;
  const int tpp = max(1, min(nthr / G, 16));
  const float2* src = partial + (size_t)b * nchunk * G;
  for (int e = tid; e < G * tpp; e += nthr) {
    const int g = e % G, r = e / G;
    float s0 = 0.f, q0 = 0.f, s1 = 0.f, q1 = 0.f;
    int k = r;
    for (; k + tpp < nchunk; k += 2 * tpp) {              // two loads in flight per thread and iteration
      const float2 u = ld_cg_f2(src + (size_t)k * G + g), w = ld_cg_f2(src + (size_t)(k + tpp) * G + g);
      s0 += u.x; q0 += u.y; s1 += w.x; q1 += w.y;
    }
    if (k < nchunk) { const float2 u = ld_cg_f2(src + (size_t)k * G + g); s0 += u.x; q0 += u.y; }
    red[r * G + g] = make_float2(s0 + s1, q0 + q1);
  }
  __syncthreads();
  for (int g = tid; g < G; g += nthr) {
    float s = 0.f, ss = 0.f;
    for (int r = 0; r < tpp; ++r) { s += red[r * G + g].x; ss += red[r * G + g].y; }
    if constexpr (kGnShift<T>) {
      const float m1 = s * inv_ne;
      mine[g] = make_float2(gn_shift(x, addend, addend_pitch, b, hw, C, C / G, g) + m1, fmaxf(fmaf(-m1, m1, ss * inv_ne), 0.f));
    } else {
      mine[g] = make_float2(s * inv_ne, ss * inv_ne);
    }
  }
  __syncthreads();
}

// This rank's statistics of ALL samples go to the patch group's slots of the publish epoch (one CTA of the grid does this:
// synchronous exchange -> at once, the peers are waiting; asynchronous modes -> for the next step, off the critical path).
template <typename T>
__device__ void gn_publish_all(const GnExchange& e, const float2* __restrict__ partial, int G, int nchunk, float2* red, float2* mine_b,
                               const T* __restrict__ x, const T* __restrict__ addend, int64_t addend_pitch, int hw, int C) {
  const df_comm_t& c = e.c;
  const int tid = threadIdx.x, nthr = blockDim.x;
  const uint32_t pub = c.clock[0];
  const int nb = e.bG / G;
  for (int b = 0; b < nb; ++b) {
    gn_reduce_sample(partial, b, G, nchunk, e.inv_ne, red, mine_b, x, addend, addend_pitch, hw, C);
    for (int p = 0; p < c.world; ++p) {
      if (!(e.group_mask >> p & 1)) continue;
      float2* dst = (float2*)slot_ptr(c, p, pub, e.tensor_off, e.slot_bytes, c.rank) + (size_t)b * G;
      for (int g = tid; g < G; g += nthr) dst[g] = mine_b[g];
    }
    __syncthreads();
  }
  __threadfence_system();
  __syncthreads();
  stamp_flags(c, e.idx, e.group_mask, pub, tid, nthr);
}

// (mean, rstd) of the G groups of sample b from this rank's statistics `mine` and, in the exchange modes, the patch group's
// slots of the read epoch (groupnorm.py:40-66).  shift: statistics are (mean, variance), modes 0 and 1 only.
template <bool shift>
__device__ __forceinline__ void gn_coef_sample(const GnExchange& e, int b, int G, const float2* mine, float2* coef_s) {
  const df_comm_t& c = e.c;
  const int tid = threadIdx.x, nthr = blockDim.x, mode = e.mode;
  uint32_t rd = 0;
  if (mode != 0) {
    rd = mode == 1 ? c.clock[0] : c.clock[1];   // a synchronous exchange reads THIS epoch even inside an asynchronous step
    wait_sources(c, e.idx, e.group_mask, rd);
  }
  for (int g = tid; g < G; g += nthr) {
    const float2 m = mine[g];
    float mean = m.x, msq = m.y;
    if constexpr (shift) {
      float var = m.y;
      if (mode != 0) {                              // the pooled variance of the members' strips, weights w_p
        float sx = 0.f;
        for (int p = 0; p < c.world; ++p) {
          if (!(e.group_mask >> p & 1)) continue;
          sx = fmaf((float)e.wgt[p], ((const float2*)slot_ptr(c, c.rank, rd, e.tensor_off, e.slot_bytes, p))[(size_t)b * G + g].x, sx);
        }
        mean = sx * e.inv_w;
        float sv = 0.f;
        for (int p = 0; p < c.world; ++p) {
          if (!(e.group_mask >> p & 1)) continue;
          const float2 v = ((const float2*)slot_ptr(c, c.rank, rd, e.tensor_off, e.slot_bytes, p))[(size_t)b * G + g];
          const float d = v.x - mean;
          sv = fmaf((float)e.wgt[p], fmaf(d, d, v.y), sv);
        }
        var = sv * e.inv_w;
      }
      coef_s[g] = make_float2(mean, rsqrtf(var * e.bessel + e.eps));
      continue;
    }
    if (mode != 0) {
      // weighted sums sum_p w_p v_p (w_p = 1 on equal strips: fmaf(1, v, s) rounds exactly like s + v)
      float sx = 0.f, sy = 0.f;
      float2 own_stale = make_float2(0.f, 0.f);
      for (int p = 0; p < c.world; ++p) {
        if (!(e.group_mask >> p & 1)) continue;
        const float2 v = ((const float2*)slot_ptr(c, c.rank, rd, e.tensor_off, e.slot_bytes, p))[(size_t)b * G + g];
        const float w = (float)e.wgt[p];
        if (p == c.rank) own_stale = v;
        sx = fmaf(w, v.x, sx); sy = fmaf(w, v.y, sy);
      }
      const float invw = e.inv_w, wown = (float)e.wgt[c.rank];
      if (mode == 1) { mean = sx * invw; msq = sy * invw; }
      else if (mode == 2) { mean = sx * invw + (m.x - own_stale.x); msq = sy * invw + (m.y - own_stale.y); }
      else { mean = fmaf(wown, m.x, fmaf(-wown, own_stale.x, sx)) * invw; msq = fmaf(wown, m.y, fmaf(-wown, own_stale.y, sy)) * invw; }
    }
    float var = msq - mean * mean;
    if (e.neg_fb && var < 0.f) var = m.y - m.x * m.x;
    var *= e.bessel;
    coef_s[g] = make_float2(mean, rsqrtf(var + e.eps));
  }
  __syncthreads();
}

template <typename T>
__device__ __forceinline__ void gn_normalise(const T* __restrict__ x, const T* __restrict__ addend, int64_t addend_pitch,
                                             T* __restrict__ y, const T* __restrict__ gamma, const T* __restrict__ beta,
                                             const float2* coef, int hw, int C, int G, int V, int lanes,
                                             int ppc, int silu, const GnHalo& halo) {
  using Vec = GnVec<T>;
  constexpr int E = Vec::E;
  const int b = blockIdx.y, chunk = blockIdx.x;
  const int tid = threadIdx.x;
  const int v = tid % V, pl = tid / V;
  const size_t row_el = halo.enabled ? (size_t)halo.w * C : 0;          // elements of one image row
  uint32_t pub = 0;
  if (halo.enabled && halo.push) pub = halo.c.clock[0];
  if (pl < lanes) {
    const int cpg = C / G;
    float sc[E], sh[E];
#pragma unroll
    for (int j = 0; j < E; ++j) {
      int ch = v * E + j;
      const float2 mr = coef[ch / cpg];
      float ga = gamma ? Vec::to_float(gamma[ch]) : 1.f, be = beta ? Vec::to_float(beta[ch]) : 0.f;
      sc[j] = mr.y * ga;
      sh[j] = be - mr.x * sc[j];
    }
    if (addend) {                     // y = ((x + a) - mean) * rstd * gamma + beta  ==  x * sc + (sh + a * sc)
      float ad[E];
      Vec::unpack(ld_v4(addend + (size_t)b * addend_pitch + (size_t)v * E), ad);
#pragma unroll
      for (int j = 0; j < E; ++j) sh[j] = fmaf(ad[j], sc[j], sh[j]);
    }
    const int p0 = chunk * ppc, p1 = min(hw, p0 + ppc);
    const size_t base = ((size_t)b * hw) * C + (size_t)v * E;
    // padded output: sample b starts at row b*(h+2), the interior at row 1
    const size_t ybase = halo.enabled ? ((size_t)b * (hw + 2 * halo.w) + halo.w) * C + (size_t)v * E : base;
    // neighbours' slots [2][batch][w*C]: part 0 = the sender's first row, part 1 = its last row (conv2d.py:61-65,90)
    T* dst_up = nullptr;
    T* dst_dn = nullptr;
    if (halo.enabled && halo.push) {
      const size_t nb = gridDim.y;
      if (halo.up >= 0) dst_up = (T*)slot_ptr(halo.c, halo.up, pub, halo.off, halo.slot_bytes, halo.c.rank) + ((size_t)b) * row_el + (size_t)v * E;
      if (halo.down >= 0) dst_dn = (T*)slot_ptr(halo.c, halo.down, pub, halo.off, halo.slot_bytes, halo.c.rank) + (nb + b) * row_el + (size_t)v * E;
    }
    const int last_row0 = hw - halo.w;                                  // first pixel of the last row (halo.enabled only)
    auto xform = [&](const int4& in) {
      float f[E];
      Vec::unpack(in, f);
#pragma unroll
      for (int j = 0; j < E; ++j) {
        float t = fmaf(f[j], sc[j], sh[j]);
        if (silu) t = __fdividef(t, 1.f + __expf(-t));
        f[j] = t;
      }
      return Vec::pack(f);
    };
    auto emit = [&](int p, const int4& o) {
      st_v4(y + ybase + (size_t)p * C, o);
      if (dst_up && p < halo.w) st_v4(dst_up + (size_t)p * C, o);
      if (dst_dn && p >= last_row0) st_v4(dst_dn + (size_t)(p - last_row0) * C, o);
    };
    int p = p0 + pl;
    for (; p + 3 * lanes < p1; p += 4 * lanes) {
      int4 r[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) r[u] = ld_v4(x + base + (size_t)(p + u * lanes) * C);
#pragma unroll
      for (int u = 0; u < 4; ++u) emit(p + u * lanes, xform(r[u]));
    }
    for (; p < p1; p += lanes) emit(p, xform(ld_v4(x + base + (size_t)p * C)));
  }
  if (!halo.enabled) return;
  // ---- boundary rows shipped: the last CTA of the grid stamps the neighbours' flags
  if (halo.push) signal_when_last(halo.c, halo.ticket2, gridDim.x * gridDim.y, halo.idx, neighbour_mask(halo.up, halo.down), pub);
  // ---- margin rows of sample b: first chunk fills the top one, last chunk the bottom one (zeros at the image border)
  const bool top = chunk == 0, bottom = chunk == (int)gridDim.x - 1;
  if (!top && !bottom) return;
  const uint32_t rd = (halo.up >= 0 || halo.down >= 0) ? halo.c.clock[1] : 0u;
  const size_t nb = gridDim.y;
  const int row_vec = (int)(row_el / E);
#pragma unroll 1
  for (int side = 0; side < 2; ++side) {
    if (side == 0 ? !top : !bottom) continue;
    const int src = side == 0 ? halo.up : halo.down;
    T* dst = y + ((size_t)b * (halo.h + 2) + (side == 0 ? 0 : halo.h + 1)) * row_el;
    if (src >= 0) {
      if (halo.wait_flags) wait_sources(halo.c, halo.idx, 1u << src, rd);
      // top margin = the up neighbour's LAST row (its part 1); bottom margin = the down neighbour's FIRST row (part 0)
      const T* from = (const T*)slot_ptr(halo.c, halo.c.rank, rd, halo.off, halo.slot_bytes, src) +
                      ((side == 0 ? nb : 0) + b) * row_el;
      for (int i = tid; i < row_vec; i += blockDim.x) st_v4(dst + (size_t)i * E, ld_v4(from + (size_t)i * E));
    } else {
      const int4 zero = make_int4(0, 0, 0, 0);
      for (int i = tid; i < row_vec; i += blockDim.x) st_v4(dst + (size_t)i * E, zero);
    }
  }
}

// ONE launch: partial moments -> grid barrier -> every CTA finishes the statistics of ITS sample -> normalise.  Every CTA of the
// grid is resident at once (the host caps the grid at the occupancy of this kernel), so a CTA may wait on the generation word
// that the last arriver bumps.  After the barrier each CTA folds the per-CTA partials of its own sample itself (G x nchunk
// values from L2, a coalesced microsecond) and keeps (mean, rstd) in shared memory; the first design let the last CTA reduce
// everything, write coef[] and only then release the grid -- 6 us of serial work plus a global round trip in front of the
// normalise pass of the whole grid.  Then each CTA normalises the pixels it has just read (L1 / L2
// hits: one HBM read and one write per element, one launch instead of two).  Exchange modes: the last arriver also publishes
// this rank's statistics to the patch group (synchronous mode: before anything else -- the peers wait for them).
template <typename T>
__global__ void __launch_bounds__(512, 2) gn_fused_kernel(const T* __restrict__ x, const T* __restrict__ addend, int64_t addend_pitch,
                                                          T* __restrict__ y, const T* __restrict__ gamma,
                                                          const T* __restrict__ beta, float2* __restrict__ partial,
                                                          int hw, int C, int G, int V,
                                                          int lanes, int ppc, int silu, GnExchange ex, unsigned int* gen,
                                                          GnHalo halo) {
  extern __shared__ float2 ch[];                         // [lanes][C] moments; after the fold: red[G*tpp] | mine[G] | coef[G]
  __shared__ unsigned int my_gen;
  __shared__ bool is_last;
  GN_TR(0, blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0);
  if (threadIdx.x == 0) my_gen = ld_volatile_u32(gen);   // read before this CTA's ticket: the bump needs every CTA's ticket
  __syncthreads();
  gn_moments(x, addend, addend_pitch, partial, hw, C, G, V, lanes, ppc, ch);
  // ---- grid barrier: ticket, the last arriver resets it and bumps the generation
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned int t = atomicAdd(ex.ticket, 1u);
    is_last = (t == (unsigned int)ex.nchunk_total - 1);
    if (is_last) {
      *ex.ticket = 0;
      __threadfence();
      asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(gen), "r"(my_gen + 1u) : "memory");
    } else {
      unsigned int v;
      do {
        asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(gen) : "memory");
        if (v == my_gen) __nanosleep(20);
      } while (v == my_gen);
    }
  }
  __syncthreads();
  GN_TR(2, blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0);
  const int tpp = max(1, min((int)blockDim.x / G, 16));
  float2* red = ch;
  float2* mine = ch + G * tpp;
  float2* coef_s = mine + G;
  const int nchunk = gridDim.x, b = blockIdx.y;
  if (is_last && ex.mode == 1)                           // the peers (and this rank's CTAs) wait for it
    gn_publish_all(ex, partial, G, nchunk, red, mine, x, addend, addend_pitch, hw, C);
  gn_reduce_sample(partial, b, G, nchunk, ex.inv_ne, red, mine, x, addend, addend_pitch, hw, C);
  GN_TR(3, blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0);
  gn_coef_sample<kGnShift<T>>(ex, b, G, mine, coef_s);
  GN_TR(4, blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0);
  if (is_last && ex.mode >= 2) {                         // next step's statistics: only this CTA is late for its normalise pass
    float2* red2 = coef_s + G;                           // keep coef_s: scratch behind it (host sizes smem for both)
    gn_publish_all(ex, partial, G, nchunk, red2, red2 + G * tpp, x, addend, addend_pitch, hw, C);
  }
  GN_TR(5, blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0);
  gn_normalise(x, addend, addend_pitch, y, gamma, beta, coef_s, hw, C, G, V, lanes, ppc, silu, halo);
  GN_TR(6, blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0);
  GN_TR(7, is_last && threadIdx.x == 0);
}

// CTAs of gn_fused_kernel<T> the device holds at once (at its largest block and shared-memory size), queried once
template <typename T>
int gn_resident_ctas() {
  static int n = -1;
  if (n < 0) {
    int per_sm = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, gn_fused_kernel<T>, 512, kGnMaxSmem) != cudaSuccess) {
      per_sm = 0;
      cudaGetLastError();
    }
    n = per_sm * sm_count();
  }
  return n;
}

#ifdef DF_GN_TRACE
}  // namespace
extern "C" int df_debug_gn_trace(unsigned long long* out_host /* 16 */) {
  DF_CHECK_CUDA(cudaDeviceSynchronize());
  DF_CHECK_CUDA(cudaMemcpyFromSymbol(out_host, df_gn_trace, sizeof(unsigned long long) * 16));
  return 0;
}
namespace {
#endif

}  // namespace

extern "C" size_t df_groupnorm_scratch_bytes_dtype(int b, int groups, int h, int w, int C, int dtype) {
  GnPlan p = dtype == DF_F32 ? gn_plan<float>(b, h, w, C) : gn_plan<__half>(b, h, w, C);
  return (size_t)b * p.nchunk * groups * sizeof(float2) + 256;
}

extern "C" size_t df_groupnorm_scratch_bytes(int b, int groups, int h, int w, int C) {
  return df_groupnorm_scratch_bytes_dtype(b, groups, h, w, C, DF_F16);
}

namespace {
template <typename T>
int groupnorm_impl(df_comm_t comm, const void* x, const void* addend, int64_t addend_pitch, void* y, const void* gamma,
                   const void* beta, int b, int h, int w, int C, int groups, float eps, int mode, int bessel,
                   int neg_var_fallback, int fuse_silu, int idx, uint64_t tensor_off, uint64_t slot_bytes,
                   uint32_t group_mask, const int32_t* src_weight_host, void* scratch, void* stream, GnHalo halo) {
  constexpr int E = GnVec<T>::E;
  DF_REQUIRE(C % E == 0 && C % groups == 0 && C / E <= 512, "df_groupnorm_fwd: unsupported channel count %d", C);
  DF_REQUIRE(((uintptr_t)x % 16) == 0 && ((uintptr_t)y % 16) == 0 && ((uintptr_t)addend % 16) == 0 && addend_pitch % E == 0,
             "df_groupnorm_fwd: x / y / addend must be 16-byte aligned (addend pitch a multiple of %d elements)", E);
  if (addend == nullptr) addend_pitch = 0;
  else if (addend_pitch == 0) addend_pitch = C;
  DF_REQUIRE(mode >= 0 && mode <= 3, "df_groupnorm_fwd: bad mode %d", mode);
  DF_REQUIRE(!kGnShift<T> || mode <= 1, "df_groupnorm_fwd: fp32 statistics are local (mode 0) or synchronous (mode 1), not mode %d",
             mode);
  DF_REQUIRE(b * groups <= 512 && groups <= 128, "df_groupnorm_fwd: b*groups = %d exceeds the exchange buffer", b * groups);
  DF_REQUIRE(mode == 0 || (slot_bytes >= (uint64_t)b * groups * 8 && (group_mask >> comm.rank & 1)),
             "df_groupnorm_fwd: statistics slot too small or rank outside its own group");
  cudaStream_t st = (cudaStream_t)stream;
  GnPlan p = gn_plan<T>(b, h, w, C);
  // scratch: [tickets (256 B, zero-initialised by the caller once)] [partials]
  unsigned int* ticket = (unsigned int*)scratch;
  halo.ticket2 = ticket + 2;
  float2* partial = (float2*)((char*)scratch + 256);
  const int hw = h * w;
  const long long ne = (long long)(C / groups) * hw;
  GnExchange ex;
  ex.c = comm; ex.ticket = ticket; ex.bG = b * groups; ex.nchunk_total = p.nchunk * b;
  ex.inv_ne = (float)(1.0 / (double)ne);
  ex.bessel = bessel ? (float)((double)ne / (double)(ne - 1)) : 1.f;
  ex.eps = eps; ex.mode = mode; ex.neg_fb = neg_var_fallback; ex.idx = idx;
  ex.tensor_off = tensor_off; ex.slot_bytes = slot_bytes; ex.group_mask = group_mask;
  {                                                             // source weights reduced by their gcd; null = equal
    int64_t gcd = 0, sum = 0;
    for (int p = 0; p < DF_MAX_WORLD; ++p) {
      ex.wgt[p] = 0;
      if (p >= comm.world || !(group_mask >> p & 1)) continue;
      const int64_t w = src_weight_host ? src_weight_host[p] : 1;
      DF_REQUIRE(w >= 1, "df_groupnorm_fwd: weight %lld of source %d must be positive", (long long)w, p);
      int64_t a = gcd, c = w;
      while (c) { const int64_t t = a % c; a = c; c = t; }
      gcd = a;
    }
    for (int p = 0; p < comm.world && p < DF_MAX_WORLD; ++p) {
      if (!(group_mask >> p & 1)) continue;
      ex.wgt[p] = (int32_t)((src_weight_host ? src_weight_host[p] : 1) / gcd);
      sum += ex.wgt[p];
    }
    ex.inv_w = sum > 0 ? 1.f / (float)sum : 1.f;
  }
  size_t smem = (size_t)p.lanes * C * sizeof(float2);
  {                                                             // after the fold: 2 x (red[G*tpp] + mine[G]) + coef[G]
    int tpp = p.threads / groups; if (tpp > 16) tpp = 16; if (tpp < 1) tpp = 1;
    const size_t need = (size_t)(2 * (groups * tpp + groups) + groups) * sizeof(float2);
    if (smem < need) smem = need;
  }
  // the grid barrier spins on CTAs that have not arrived: all of them must be resident at once
  DF_REQUIRE(p.nchunk * b <= gn_resident_ctas<T>(), "df_groupnorm_fwd: grid of %d CTAs exceeds the %d this device holds at once",
             p.nchunk * b, gn_resident_ctas<T>());
  DF_REQUIRE(smem <= (size_t)kGnMaxSmem, "df_groupnorm_fwd: %zu bytes of shared memory exceed %d", smem, kGnMaxSmem);
  unsigned int* gen = ticket + 1;
  gn_fused_kernel<T><<<dim3(p.nchunk, b), p.threads, smem, st>>>((const T*)x, (const T*)addend, addend_pitch, (T*)y,
                                                                 (const T*)gamma, (const T*)beta, partial, hw, C, groups,
                                                                 p.V, p.lanes, p.ppc, fuse_silu, ex, gen, halo);
  DF_CHECK_LAUNCH();
  return 0;
}

int groupnorm_dispatch(int dtype, df_comm_t comm, const void* x, const void* addend, int64_t addend_pitch, void* y,
                       const void* gamma, const void* beta, int b, int h, int w, int C, int groups, float eps, int mode, int bessel,
                       int neg_var_fallback, int fuse_silu, int idx, uint64_t tensor_off, uint64_t slot_bytes,
                       uint32_t group_mask, const int32_t* src_weight_host, void* scratch, void* stream, GnHalo halo) {
  DF_REQUIRE(dtype == DF_F16 || dtype == DF_F32, "df_groupnorm_fwd: unknown element type %d", dtype);
  auto impl = dtype == DF_F32 ? groupnorm_impl<float> : groupnorm_impl<__half>;
  return impl(comm, x, addend, addend_pitch, y, gamma, beta, b, h, w, C, groups, eps, mode, bessel, neg_var_fallback, fuse_silu,
              idx, tensor_off, slot_bytes, group_mask, src_weight_host, scratch, stream, halo);
}
}  // namespace

extern "C" int df_groupnorm_fwd_dtype(df_comm_t comm, const void* x, const void* addend, int64_t addend_pitch, void* y,
                                      const void* gamma, const void* beta, int b, int h, int w, int C, int groups, float eps,
                                      int mode, int bessel, int neg_var_fallback, int fuse_silu, int idx, uint64_t tensor_off,
                                      uint64_t slot_bytes, uint32_t group_mask, const int32_t* src_weight_host, void* scratch,
                                      int dtype, void* stream) {
  GnHalo halo;
  memset(&halo, 0, sizeof(halo));
  return groupnorm_dispatch(dtype, comm, x, addend, addend_pitch, y, gamma, beta, b, h, w, C, groups, eps, mode, bessel,
                            neg_var_fallback, fuse_silu, idx, tensor_off, slot_bytes, group_mask, src_weight_host, scratch, stream,
                            halo);
}

extern "C" int df_groupnorm_fwd_weighted(df_comm_t comm, const void* x, const void* addend, int64_t addend_pitch, void* y,
                                         const void* gamma, const void* beta, int b, int h, int w, int C, int groups, float eps,
                                         int mode, int bessel, int neg_var_fallback, int fuse_silu, int idx, uint64_t tensor_off,
                                         uint64_t slot_bytes, uint32_t group_mask, const int32_t* src_weight_host, void* scratch,
                                         void* stream) {
  return df_groupnorm_fwd_dtype(comm, x, addend, addend_pitch, y, gamma, beta, b, h, w, C, groups, eps, mode, bessel,
                                neg_var_fallback, fuse_silu, idx, tensor_off, slot_bytes, group_mask, src_weight_host, scratch,
                                DF_F16, stream);
}

extern "C" int df_groupnorm_fwd(df_comm_t comm, const void* x, const void* addend, int64_t addend_pitch, void* y, const void* gamma,
                                const void* beta, int b, int h, int w, int C, int groups, float eps, int mode, int bessel,
                                int neg_var_fallback, int fuse_silu, int idx, uint64_t tensor_off, uint64_t slot_bytes,
                                uint32_t group_mask, void* scratch, void* stream) {
  return df_groupnorm_fwd_weighted(comm, x, addend, addend_pitch, y, gamma, beta, b, h, w, C, groups, eps, mode, bessel,
                                   neg_var_fallback, fuse_silu, idx, tensor_off, slot_bytes, group_mask, nullptr, scratch, stream);
}

extern "C" int df_groupnorm_halo_fwd_dtype(df_comm_t comm, const void* x, const void* addend, int64_t addend_pitch,
                                           void* y_padded, const void* gamma, const void* beta, int b, int h, int w, int C,
                                           int groups, float eps, int mode, int bessel, int neg_var_fallback, int fuse_silu,
                                           int idx, uint64_t tensor_off, uint64_t slot_bytes, uint32_t group_mask,
                                           const int32_t* src_weight_host, void* scratch, int halo_idx, uint64_t halo_off,
                                           uint64_t halo_slot_bytes, int up_rank, int down_rank, int push, int wait_flags,
                                           int dtype, void* stream) {
  const uint64_t esize = dtype == DF_F32 ? 4 : 2;
  DF_REQUIRE(halo_slot_bytes >= 2ull * b * w * C * esize, "df_groupnorm_halo_fwd: halo slot too small");
  DF_REQUIRE(up_rank < comm.world && down_rank < comm.world, "df_groupnorm_halo_fwd: neighbour outside the communicator");
  GnHalo halo;
  memset(&halo, 0, sizeof(halo));
  halo.enabled = 1; halo.h = h; halo.w = w; halo.up = up_rank; halo.down = down_rank; halo.push = push; halo.wait_flags = wait_flags;
  halo.idx = halo_idx; halo.off = halo_off; halo.slot_bytes = halo_slot_bytes; halo.c = comm;
  return groupnorm_dispatch(dtype, comm, x, addend, addend_pitch, y_padded, gamma, beta, b, h, w, C, groups, eps, mode, bessel,
                            neg_var_fallback, fuse_silu, idx, tensor_off, slot_bytes, group_mask, src_weight_host, scratch, stream,
                            halo);
}

extern "C" int df_groupnorm_halo_fwd_weighted(df_comm_t comm, const void* x, const void* addend, int64_t addend_pitch,
                                              void* y_padded, const void* gamma, const void* beta, int b, int h, int w, int C,
                                              int groups, float eps, int mode, int bessel, int neg_var_fallback, int fuse_silu,
                                              int idx, uint64_t tensor_off, uint64_t slot_bytes, uint32_t group_mask,
                                              const int32_t* src_weight_host, void* scratch, int halo_idx, uint64_t halo_off,
                                              uint64_t halo_slot_bytes, int up_rank, int down_rank, int push, int wait_flags,
                                              void* stream) {
  return df_groupnorm_halo_fwd_dtype(comm, x, addend, addend_pitch, y_padded, gamma, beta, b, h, w, C, groups, eps, mode, bessel,
                                     neg_var_fallback, fuse_silu, idx, tensor_off, slot_bytes, group_mask, src_weight_host, scratch,
                                     halo_idx, halo_off, halo_slot_bytes, up_rank, down_rank, push, wait_flags, DF_F16, stream);
}

extern "C" int df_groupnorm_halo_fwd(df_comm_t comm, const void* x, const void* addend, int64_t addend_pitch, void* y_padded, const void* gamma,
                                     const void* beta, int b, int h, int w, int C, int groups, float eps, int mode, int bessel,
                                     int neg_var_fallback, int fuse_silu, int idx, uint64_t tensor_off, uint64_t slot_bytes,
                                     uint32_t group_mask, void* scratch, int halo_idx, uint64_t halo_off,
                                     uint64_t halo_slot_bytes, int up_rank, int down_rank, int push, int wait_flags, void* stream) {
  return df_groupnorm_halo_fwd_weighted(comm, x, addend, addend_pitch, y_padded, gamma, beta, b, h, w, C, groups, eps, mode, bessel,
                                        neg_var_fallback, fuse_silu, idx, tensor_off, slot_bytes, group_mask, nullptr, scratch,
                                        halo_idx, halo_off, halo_slot_bytes, up_rank, down_rank, push, wait_flags, stream);
}
