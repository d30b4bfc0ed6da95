// Internal helpers shared by the rtti_b200 translation units (not part of the C ABI).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#ifdef __CUDACC__
#include <cuda_fp16.h>
#endif

#include "../../include/rtti_b200.h"

namespace rtti {

// cuTensorMapEncodeTiled resolved through the runtime (no link-time dependency on libcuda).
int encode_tiled_f16(CUtensorMap* map, const void* base, int rank, const cuuint64_t* dims,
                     const cuuint64_t* strides_bytes, const cuuint32_t* box, const cuuint32_t* elem_strides);

// 4-D map {head_dim, heads, rows, batch} over a [batch, rows, heads*head_dim] fp16 tensor with element
// strides bs (batch) and rs (row); box = {64, 1, box_rows, 1}, SWIZZLE_128B, zero OOB fill.
int make_head_map(CUtensorMap* m, const void* ptr, int head_dim, int heads, int rows, int batch, long long bs,
                  long long rs, int box_rows);

inline int ceil_div(long long a, long long b) { return (int)((a + b - 1) / b); }

// the buffers of a multistep (DDIM / DPM-Solver++) blend step: d_out required, d_prev required when cp != 0, both
// 16-byte aligned
inline int ms_step_args(float cp, const float* d_prev, const float* d_out) {
  if (!d_out || (cp != 0.f && !d_prev)) return RTTI_ERR_ARG;
  return (((uintptr_t)d_prev | (uintptr_t)d_out) & 15) ? RTTI_ERR_ALIGN : RTTI_OK;
}

// the noise of an ancestral blend step: required when s_up != 0, 16-byte aligned
inline int anc_step_args(float s_up, const void* z) {
  if (s_up != 0.f && !z) return RTTI_ERR_ARG;
  return ((uintptr_t)z & 15) ? RTTI_ERR_ALIGN : RTTI_OK;
}

// the buffers of a UniPC blend step: m_out and xl_out required; xl required when ul != 0, m1 when u1 or v1 != 0, m2
// when u2 != 0; all 16-byte aligned
inline int unipc_step_args(float ul, float u1, float u2, float v1, const float* xl, const float* m1, const float* m2,
                           const float* m_out, const float* xl_out) {
  if (!m_out || !xl_out || (ul != 0.f && !xl) || ((u1 != 0.f || v1 != 0.f) && !m1) || (u2 != 0.f && !m2))
    return RTTI_ERR_ARG;
  return (((uintptr_t)xl | (uintptr_t)m1 | (uintptr_t)m2 | (uintptr_t)m_out | (uintptr_t)xl_out) & 15) ? RTTI_ERR_ALIGN
                                                                                                      : RTTI_OK;
}

// the saved state of a Heun blend step: xs required when cs != 0, ds when cd != 0; both 16-byte aligned
inline int heun_step_args(float cs, float cd, const void* xs, const void* ds) {
  if ((cs != 0.f && !xs) || (cd != 0.f && !ds)) return RTTI_ERR_ARG;
  return (((uintptr_t)xs | (uintptr_t)ds) & 15) ? RTTI_ERR_ALIGN : RTTI_OK;
}

// the prediction history of an LMS blend step: d_k required when c_k != 0; each 16-byte aligned when given
inline int lms_step_args(float c1, float c2, float c3, const void* d1, const void* d2, const void* d3) {
  if ((c1 != 0.f && !d1) || (c2 != 0.f && !d2) || (c3 != 0.f && !d3)) return RTTI_ERR_ARG;
  return (((uintptr_t)d1 | (uintptr_t)d2 | (uintptr_t)d3) & 15) ? RTTI_ERR_ALIGN : RTTI_OK;
}

// the buffers of a singlestep (DPM-Solver++(2S)) blend step: those of the multistep step, and the block's starting
// latents xs, required when cs != 0 and 16-byte aligned
inline int ss_step_args(float cs, float cp, const void* xs, const float* d_prev, const float* d_out) {
  const int rc = ms_step_args(cp, d_prev, d_out);
  if (rc != RTTI_OK) return rc;
  if (cs != 0.f && !xs) return RTTI_ERR_ARG;
  return ((uintptr_t)xs & 15) ? RTTI_ERR_ALIGN : RTTI_OK;
}

#ifdef __CUDACC__
// GroupNorm statistics of a set of values as (count n, mean, m2 = sum of squared deviations from the mean), merged with
// the pairwise update of Chan, Golub & LeVeque. Unlike a one-pass E[x^2] - E[x]^2 in fp32, which loses about
// log10((mean/std)^2) digits of the variance, this keeps the variance as accurate as the inputs whatever their offset.
// Merging into an empty partial (n = 0) copies the other operand; an empty b is a no-op. The weight nb/(n+nb) uses the
// fast division (2 ulp): it only scales the correction term, and the merge sits on the serial tail of the reductions.
__device__ __forceinline__ void stats_merge(int& n, float& mean, float& m2, int nb, float mean_b, float m2_b) {
  if (nb == 0) return;
  if (n == 0) { n = nb; mean = mean_b; m2 = m2_b; return; }
  const int nt = n + nb;
  const float f = __fdividef((float)nb, (float)nt), d = mean_b - mean;
  mean = fmaf(d, f, mean);
  m2 = m2 + m2_b + d * d * ((float)n * f);
  n = nt;
}

// (count, mean, m2) of group g over chunks lane, lane+32, ... of a GroupNorm statistics workspace laid out
// [batch][chunks][groups][2] = (mean, m2); ws_bg points at (b, chunk 0, g). Chunk k holds
// min(rows_per_chunk, hw - k*rows_per_chunk) rows of cpg channels. The loads of 8 chunks are issued before they are
// merged (the merge order is still k ascending): the merges form a dependent chain, and one load per merge would put
// the memory latency on it.
__device__ __forceinline__ void gn_lane_stats(const float* __restrict__ ws_bg, int groups, int chunks, int hw,
                                              int rows_per_chunk, int cpg, int lane, int& n, float& mean, float& m2) {
  n = 0; mean = 0.f; m2 = 0.f;
  for (int k0 = lane; k0 < chunks; k0 += 32 * 8) {
    float2 v[8];
    int nk[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const int k = k0 + 32 * u;
      nk[u] = k < chunks ? min(rows_per_chunk, hw - k * rows_per_chunk) * cpg : 0;
      v[u] = k < chunks ? *reinterpret_cast<const float2*>(ws_bg + (size_t)k * groups * 2) : make_float2(0.f, 0.f);
    }
#pragma unroll
    for (int u = 0; u < 8; ++u) stats_merge(n, mean, m2, nk[u], v[u].x, v[u].y);
  }
}

// The step policies of the blend kernels (elementwise.cu, gather_blend.cu, blend_rescale.cu): each family has one body,
// instantiated with the Euler update (x' = x + dt_sigma * eps) or with the multistep update of DDIM / DPM-Solver++(2M)
// in data-prediction form (schedulers.py, StepCoeffs):
//   D  = hx * x + he * eps            written to d_out in fp32
//   x' = cx * x + cd * D + cp * D_prev    D_prev read from d_prev only when cp != 0
// eps is the fp16-rounded noise prediction the kernel stores, x the fp16 latents. d_prev may alias d_out: each thread
// reads its 8 elements of d_prev before it writes the same 8 elements of d_out.
struct MsStep {
  float hx, he, cx, cd, cp;
  const float* d_prev;
  float* d_out;
};

__device__ __forceinline__ void ms_step8(const MsStep& s, long long v, const float* e16, float* x) {
  float dp[8];
  if (s.cp != 0.f) {
    const float4 p0 = *reinterpret_cast<const float4*>(s.d_prev + v * 8);
    const float4 p1 = *reinterpret_cast<const float4*>(s.d_prev + v * 8 + 4);
    dp[0] = p0.x; dp[1] = p0.y; dp[2] = p0.z; dp[3] = p0.w; dp[4] = p1.x; dp[5] = p1.y; dp[6] = p1.z; dp[7] = p1.w;
  }
  float d[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) d[i] = fmaf(s.he, e16[i], s.hx * x[i]);
  *reinterpret_cast<float4*>(s.d_out + v * 8) = make_float4(d[0], d[1], d[2], d[3]);
  *reinterpret_cast<float4*>(s.d_out + v * 8 + 4) = make_float4(d[4], d[5], d[6], d[7]);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    float o = fmaf(s.cd, d[i], s.cx * x[i]);
    if (s.cp != 0.f) o = fmaf(s.cp, dp[i], o);
    x[i] = o;
  }
}

// The ancestral (Euler a) update: x' = x + dt_sigma * eps + s_up * z, with dt_sigma = sigma_down - sigma and z the
// fp16 noise of the step, [n] (schedulers.py, EulerAncestralDiscreteScheduler.ancestral_coeffs). The Euler update is
// formed first, exactly as EulerStep forms it; z is read (128-bit) only when s_up != 0, so s_up = 0 gives the Euler bits.
struct AncStep {
  float dt_sigma, s_up;
  const __half* z;
};

__device__ __forceinline__ void anc_step8(const AncStep& s, long long v, const float* e16, float* x) {
#pragma unroll
  for (int i = 0; i < 8; ++i) x[i] = fmaf(e16[i], s.dt_sigma, x[i]);
  if (s.s_up != 0.f) {
    const uint4 u = *reinterpret_cast<const uint4*>(s.z + v * 8);
    const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 t = __half22float2(h[i]);
      x[2 * i] = fmaf(t.x, s.s_up, x[2 * i]);
      x[2 * i + 1] = fmaf(t.y, s.s_up, x[2 * i + 1]);
    }
  }
}

// The UniPC (bh2, order 2) update in data-prediction form (schedulers.py, UniPCMultistepScheduler.unipc_coeffs):
//   m  = hx * x + he * eps                                   written to m_out
//   xc = ux * x + ul * xl + u0 * m + u1 * m1 + u2 * m2       the corrected sample, written to xl_out
//   x' = vx * xc + v0 * m + v1 * m1                          the predictor, rounded to fp16 by the caller
// with xl = xc of the previous step, m1 / m2 = m of the previous two steps, fp32 [n] each. A history is read (128-bit)
// only when one of its coefficients is non-zero; an unread one counts as 0. m_out may alias m2 and xl_out may alias xl:
// each thread loads its 8 elements of every history before it stores any.
struct UniPCStep {
  float hx, he, ux, ul, u0, u1, u2, vx, v0, v1;
  const float* xl;
  const float* m1;
  const float* m2;
  float* m_out;
  float* xl_out;
};

__device__ __forceinline__ void ld8f(const float* p, float* f) {
  const float4 a = *reinterpret_cast<const float4*>(p), b = *reinterpret_cast<const float4*>(p + 4);
  f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w; f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
}
__device__ __forceinline__ void st8f(float* p, const float* f) {
  *reinterpret_cast<float4*>(p) = make_float4(f[0], f[1], f[2], f[3]);
  *reinterpret_cast<float4*>(p + 4) = make_float4(f[4], f[5], f[6], f[7]);
}

__device__ __forceinline__ void unipc_step8(const UniPCStep& s, long long v, const float* e16, float* x) {
  float l[8], a[8], b[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) { l[i] = 0.f; a[i] = 0.f; b[i] = 0.f; }
  if (s.ul != 0.f) ld8f(s.xl + v * 8, l);
  if (s.u1 != 0.f || s.v1 != 0.f) ld8f(s.m1 + v * 8, a);
  if (s.u2 != 0.f) ld8f(s.m2 + v * 8, b);
  float m[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    m[i] = fmaf(s.he, e16[i], s.hx * x[i]);
    float c = fmaf(s.u0, m[i], s.ux * x[i]);
    c = fmaf(s.ul, l[i], c);
    c = fmaf(s.u1, a[i], c);
    c = fmaf(s.u2, b[i], c);
    l[i] = c;
    x[i] = fmaf(s.v1, a[i], fmaf(s.v0, m[i], s.vx * c));
  }
  st8f(s.m_out + v * 8, m);
  st8f(s.xl_out + v * 8, l);
}

// The Heun update (schedulers.py, HeunDiscreteScheduler.heun_coeffs), in fp32:
//   x' = cx * x + ce * eps + cd * ds + cs * xs
// with xs / ds the fp16 [n] latents and stepped noise prediction saved at the first stage: (1, dt, 0, 0) at a first
// stage, (0, dt/2, 1, dt/2) at a second. ds is read (128-bit) only when cd != 0 and xs only when cs != 0. The Euler
// update is formed first (cx * x is exact for cx = 1), so a first stage gives the Euler bits with dt_sigma = ce; the
// two dt/2 terms are summed before the latents xs are added.
struct HeunStep {
  float cx, ce, cs, cd;
  const __half* xs;
  const __half* ds;
};

__device__ __forceinline__ void heun_ld8(const __half* p, float* f) {
  const uint4 u = *reinterpret_cast<const uint4*>(p);
  const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) { const float2 t = __half22float2(h[i]); f[2 * i] = t.x; f[2 * i + 1] = t.y; }
}

__device__ __forceinline__ void heun_step8(const HeunStep& s, long long v, const float* e16, float* x) {
#pragma unroll
  for (int i = 0; i < 8; ++i) x[i] = fmaf(e16[i], s.ce, s.cx * x[i]);
  if (s.cd != 0.f) {
    float d[8];
    heun_ld8(s.ds + v * 8, d);
#pragma unroll
    for (int i = 0; i < 8; ++i) x[i] = fmaf(d[i], s.cd, x[i]);
  }
  if (s.cs != 0.f) {
    float p[8];
    heun_ld8(s.xs + v * 8, p);
#pragma unroll
    for (int i = 0; i < 8; ++i) x[i] = fmaf(p[i], s.cs, x[i]);
  }
}

// The LMS update (schedulers.py, LMSDiscreteScheduler.lms_coeffs), in fp32:
//   x' = x + c0 * eps + c1 * d1 + c2 * d2 + c3 * d3
// with d1, d2, d3 the fp16 [n] noise predictions of the last three steps of the trajectory, newest first. d_k is read
// (128-bit) only when c_k != 0; the history loads are all issued before the first FMA so that their latencies overlap.
// The terms are added in the order above, the Euler update first, so (c0, 0, 0, 0) gives the Euler bits with
// dt_sigma = c0.
struct LmsStep {
  float c0, c1, c2, c3;
  const __half* d1;
  const __half* d2;
  const __half* d3;
};

__device__ __forceinline__ void lms_fma8(const uint4& u, float c, float* x) {
  const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 t = __half22float2(h[i]);
    x[2 * i] = fmaf(t.x, c, x[2 * i]);
    x[2 * i + 1] = fmaf(t.y, c, x[2 * i + 1]);
  }
}

__device__ __forceinline__ void lms_step8(const LmsStep& s, long long v, const float* e16, float* x) {
  uint4 h1, h2, h3;
  if (s.c1 != 0.f) h1 = *reinterpret_cast<const uint4*>(s.d1 + v * 8);
  if (s.c2 != 0.f) h2 = *reinterpret_cast<const uint4*>(s.d2 + v * 8);
  if (s.c3 != 0.f) h3 = *reinterpret_cast<const uint4*>(s.d3 + v * 8);
#pragma unroll
  for (int i = 0; i < 8; ++i) x[i] = fmaf(e16[i], s.c0, x[i]);
  if (s.c1 != 0.f) lms_fma8(h1, s.c1, x);
  if (s.c2 != 0.f) lms_fma8(h2, s.c2, x);
  if (s.c3 != 0.f) lms_fma8(h3, s.c3, x);
}

// The DPM-Solver++(2S) update (schedulers.py, DPMSolverSinglestepScheduler.singlestep_coeffs), in fp32:
//   D  = hx * x + he * eps                              written to d_out
//   x' = cx * x + cd * D + cp * D_prev + cs * xs
// with xs the fp16 [n] latents that entered the first step of the current two-step block: (hx, he, cx, cd, 0, 0) on a
// first step, (hx, he, 0, cd, cp, cs) on the second. The multistep update is formed first, exactly as ms_step8 forms it
// (d_prev may alias d_out), and cs * xs added last; xs is read (128-bit, issued before the multistep arithmetic) only
// when cs != 0, so cs = 0 gives the multistep bits.
struct SsStep {
  MsStep ms;
  float cs;
  const __half* xs;
};

__device__ __forceinline__ void ss_step8(const SsStep& s, long long v, const float* e16, float* x) {
  uint4 u;
  if (s.cs != 0.f) u = *reinterpret_cast<const uint4*>(s.xs + v * 8);
  ms_step8(s.ms, v, e16, x);
  if (s.cs != 0.f) lms_fma8(u, s.cs, x);
}

// fixed-order tree over the 32 lanes of a warp; lane 0 ends with the statistics of every lane
__device__ __forceinline__ void stats_warp_merge(int& n, float& mean, float& m2) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const int nb = __shfl_down_sync(0xffffffffu, n, o);
    const float mb = __shfl_down_sync(0xffffffffu, mean, o);
    const float qb = __shfl_down_sync(0xffffffffu, m2, o);
    stats_merge(n, mean, m2, nb, mb, qb);
  }
}
#endif

}  // namespace rtti
