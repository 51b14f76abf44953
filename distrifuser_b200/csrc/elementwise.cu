// distrifuser_b200 -- fused GEGLU gate for the transformer feed-forward (diffusers FeedForward.net[0], untouched by the
// reference's wrappers but 13 % of a 1024^2 SDXL step as two eager torch kernels: gelu(gate) then hidden * gelu).
// One pass: reads the [rows, 2*cols] projection once, writes [rows, cols].   Bound: HBM (3 * rows * cols * 2 B).
#include "common.cuh"

using namespace df;

namespace {

// gelu_erf(x) = x * Phi(x).  erf through Abramowitz-Stegun 7.1.26 (|error| < 1.5e-7: far below the fp16 rounding of the
// result): 5 FMAs + one MUFU.RCP + one MUFU.EX2 instead of libdevice erff's two-branch polynomial -- the kernel was
// ALU-bound at 3.1 TB/s with erff.
__device__ __forceinline__ float gelu_erf(float x) {
  const float z = fabsf(x) * 0.70710678118654752f;
  const float t = __fdividef(1.f, fmaf(0.3275911f, z, 1.f));
  float p = fmaf(1.061405429f, t, -1.453152027f);
  p = fmaf(p, t, 1.421413741f);
  p = fmaf(p, t, -0.284496736f);
  p = fmaf(p, t, 0.254829592f);
  const float e = p * t * __expf(-z * z);            // 1 - erf(|x|/sqrt2)
  const float phi = x >= 0.f ? 1.f - 0.5f * e : 0.5f * e;
  return x * phi;
}

__global__ void __launch_bounds__(256) geglu_kernel(const __half* __restrict__ in, __half* __restrict__ out, int64_t rows,
                                                    int vec_per_row, int64_t in_pitch, int64_t out_pitch, int cols) {
  const int64_t total = rows * vec_per_row;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / vec_per_row;
    const int q = (int)(i - r * vec_per_row);
    const __half* src = in + r * in_pitch + (int64_t)q * 8;
    int4 hv = ld_nc_v4(src), gv = ld_nc_v4(src + cols);
    const __half2* h2 = reinterpret_cast<const __half2*>(&hv);
    const __half2* g2 = reinterpret_cast<const __half2*>(&gv);
    int4 o;
    __half2* o2 = reinterpret_cast<__half2*>(&o);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float2 h = __half22float2(h2[j]), g = __half22float2(g2[j]);
      o2[j] = __floats2half2_rn(h.x * gelu_erf(g.x), h.y * gelu_erf(g.y));
    }
    st_v4(out + r * out_pitch + (int64_t)q * 8, o);
  }
}

}  // namespace

extern "C" int df_geglu(const void* in, void* out, int64_t rows, int cols, int64_t in_pitch, int64_t out_pitch, void* stream) {
  DF_REQUIRE(cols % 8 == 0 && in_pitch % 8 == 0 && out_pitch % 8 == 0 && ((uintptr_t)in % 16) == 0 && ((uintptr_t)out % 16) == 0,
             "df_geglu: 16-byte alignment required (cols=%d)", cols);
  if (rows == 0) return 0;
  const int64_t total = rows * (cols / 8);
  int64_t g = (total + 255) / 256;
  if (g > kSmCount * 16) g = kSmCount * 16;
  geglu_kernel<<<(unsigned)g, 256, 0, (cudaStream_t)stream>>>((const __half*)in, (__half*)out, rows, cols / 8, in_pitch,
                                                               out_pitch, cols);
  DF_CHECK_LAUNCH();
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------------
// out = a + bias[channel] (+ r) on NHWC activations, 16-byte vectors.  cuDNN's convolution has no bias epilogue through
// torch (`conv2d` = cudnn_convolution + a broadcast `add_`, a NON-vectorised element-wise kernel: 16 us on a 21 MB activation),
// and ResnetBlock2D then adds the residual in a third pass.  The convs run without bias and this kernel does both additions
// in one pass (conv2.bias + conv_shortcut.bias + residual), or just the bias, in place.   Bound: HBM.
namespace {
__global__ void __launch_bounds__(256) bias_residual_add_kernel(const __half* __restrict__ a, const __half* __restrict__ r,
                                                                const __half* __restrict__ bias, __half* __restrict__ out,
                                                                int64_t total_vec, int vec_per_row) {
  constexpr int U = 4;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i0 < total_vec; i0 += U * stride) {
    int4 av[U], rv[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t i = i0 + u * stride;
      if (i < total_vec) {
        av[u] = ld_nc_v4(a + i * 8);
        if (r) rv[u] = ld_nc_v4(r + i * 8);
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t i = i0 + u * stride;
      if (i >= total_vec) break;
      const int q = (int)(i % vec_per_row);
      const int4 bv = ld_v4(bias + (int64_t)q * 8);
      const __half2* a2 = reinterpret_cast<const __half2*>(&av[u]);
      const __half2* r2 = reinterpret_cast<const __half2*>(&rv[u]);
      const __half2* b2 = reinterpret_cast<const __half2*>(&bv);
      int4 o;
      __half2* o2 = reinterpret_cast<__half2*>(&o);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float2 x = __half22float2(a2[j]);
        const float2 b = __half22float2(b2[j]);
        x.x += b.x; x.y += b.y;
        if (r) { const float2 y = __half22float2(r2[j]); x.x += y.x; x.y += y.y; }
        o2[j] = __floats2half2_rn(x.x, x.y);
      }
      st_v4(out + i * 8, o);
    }
  }
}
}  // namespace

extern "C" int df_bias_residual_add(const void* a, const void* residual, const void* bias, void* out, int64_t rows, int C,
                                    void* stream) {
  DF_REQUIRE(C % 8 == 0 && ((uintptr_t)a % 16) == 0 && ((uintptr_t)residual % 16) == 0 && ((uintptr_t)bias % 16) == 0 &&
                 ((uintptr_t)out % 16) == 0, "df_bias_residual_add: 16-byte alignment required (C=%d)", C);
  if (rows == 0) return 0;
  const int64_t total = rows * (C / 8);
  int64_t g = (total + 256 * 4 - 1) / (256 * 4);
  if (g > kSmCount * 8) g = kSmCount * 8;
  bias_residual_add_kernel<<<(unsigned)g, 256, 0, (cudaStream_t)stream>>>((const __half*)a, (const __half*)residual,
                                                                           (const __half*)bias, (__half*)out, total, C / 8);
  DF_CHECK_LAUNCH();
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------------
// Fused residual add + LayerNorm for BasicTransformerBlock:  s = x + r (written back, fp16);  y = LN(s) * gamma + beta.
// One warp per token row, the row lives in registers between the statistics and the normalisation, so the pair
// `x + attn(...)` / `norm(x)` (two torch kernels, 5 HBM passes) becomes one kernel with 4 passes (2 reads, 2 writes).
namespace {

template <int MAXV>   // MAXV 16-byte vectors per lane: C <= 32 * 8 * MAXV
__global__ void __launch_bounds__(256) add_layernorm_kernel(const __half* __restrict__ x, const __half* __restrict__ r,
                                                            __half* __restrict__ s_out, __half* __restrict__ y,
                                                            const __half* __restrict__ gamma, const __half* __restrict__ beta,
                                                            int64_t rows, int C, float eps) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int nvec = C >> 3;
  const __half* xr = x + row * C;
  const __half* rr = r ? r + row * C : nullptr;
  float v[MAXV][8];
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int q = lane + 32 * i;
    if (q < nvec) {
      int4 a = ld_nc_v4(xr + q * 8);
      const __half2* a2 = reinterpret_cast<const __half2*>(&a);
      if (rr) {
        int4 b = ld_nc_v4(rr + q * 8);
        const __half2* b2 = reinterpret_cast<const __half2*>(&b);
        int4 o;
        __half2* o2 = reinterpret_cast<__half2*>(&o);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          o2[j] = __hadd2(a2[j], b2[j]);                 // same fp16 rounding as the eager `x + r`
          float2 f = __half22float2(o2[j]);
          v[i][2 * j] = f.x; v[i][2 * j + 1] = f.y;
        }
        if (s_out) st_v4(s_out + row * C + q * 8, o);
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          float2 f = __half22float2(a2[j]);
          v[i][2 * j] = f.x; v[i][2 * j + 1] = f.y;
        }
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) sum += v[i][j];
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  const float mean = sum / (float)C;
  float var = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    if (lane + 32 * i < nvec) {
#pragma unroll
      for (int j = 0; j < 8; ++j) { float d = v[i][j] - mean; var = fmaf(d, d, var); }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) var += __shfl_xor_sync(0xffffffffu, var, o);
  const float rstd = rsqrtf(var / (float)C + eps);
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int q = lane + 32 * i;
    if (q < nvec) {
      int4 g = ld_v4(gamma + q * 8), bt = ld_v4(beta + q * 8);
      const __half2* g2 = reinterpret_cast<const __half2*>(&g);
      const __half2* b2 = reinterpret_cast<const __half2*>(&bt);
      int4 o;
      __half2* o2 = reinterpret_cast<__half2*>(&o);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float2 gg = __half22float2(g2[j]), bb = __half22float2(b2[j]);
        o2[j] = __floats2half2_rn((v[i][2 * j] - mean) * rstd * gg.x + bb.x, (v[i][2 * j + 1] - mean) * rstd * gg.y + bb.y);
      }
      st_v4(y + row * C + q * 8, o);
    }
  }
}

}  // namespace

extern "C" int df_add_layernorm(const void* x, const void* r, void* s_out, void* y, const void* gamma, const void* beta,
                                int64_t rows, int C, float eps, void* stream) {
  DF_REQUIRE(C % 8 == 0 && C <= 32 * 8 * 8, "df_add_layernorm: C=%d not supported (multiple of 8, <= 2048)", C);
  DF_REQUIRE(((uintptr_t)x % 16) == 0 && ((uintptr_t)r % 16) == 0 && ((uintptr_t)s_out % 16) == 0 && ((uintptr_t)y % 16) == 0 &&
                 ((uintptr_t)gamma % 16) == 0 && ((uintptr_t)beta % 16) == 0, "df_add_layernorm: 16-byte alignment required");
  if (rows == 0) return 0;
  const int warps = 8;
  const unsigned grid = (unsigned)((rows + warps - 1) / warps);
  cudaStream_t st = (cudaStream_t)stream;
  const int nvec = C / 8;
#define DF_LN(MV) add_layernorm_kernel<MV><<<grid, warps * 32, 0, st>>>((const __half*)x, (const __half*)r, (__half*)s_out, \
      (__half*)y, (const __half*)gamma, (const __half*)beta, rows, C, eps)
  if (nvec <= 32 * 2) DF_LN(2); else if (nvec <= 32 * 3) DF_LN(3); else if (nvec <= 32 * 5) DF_LN(5); else DF_LN(8);
#undef DF_LN
  DF_CHECK_LAUNCH();
  return 0;
}
