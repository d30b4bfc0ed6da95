// HBM-bound kernels of the region-diffusion step: GroupNorm(+temb)(+SiLU) on channels-last
// activations, LayerNorm, GEGLU, region blend + CFG (+ Euler update), colour-guidance loss
// forward/backward, guidance update, background injection, x0 prediction.
// All are coalesced 128-bit vectorised (ld8 / st8 below), fp32 math, deterministic (no atomics).
#include <cuda_fp16.h>

#include "rtti_internal.h"

namespace rtti {

struct alignas(16) Half8 { __half2 v[4]; };

__device__ __forceinline__ void unpack8(const Half8& h, float* f) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 t = __half22float2(h.v[i]);
    f[2 * i] = t.x; f[2 * i + 1] = t.y;
  }
}
__device__ __forceinline__ Half8 pack8(const float* f) {
  Half8 h;
#pragma unroll
  for (int i = 0; i < 4; ++i) h.v[i] = __floats2half2_rn(f[2 * i], f[2 * i + 1]);
  return h;
}
// 128-bit global accesses. A plain `*reinterpret_cast<const Half8*>(p)` is a memberwise struct copy that nvcc 12.9 lowers
// to FOUR 32-bit LDG / STG (cuobjdump: LDG.E, STG.E without .128 in every fp16 kernel of round 1 — four times the LSU
// wavefronts, l1tex pipe 83 % busy at 18 % of the DRAM bandwidth); going through uint4 gives LDG.E.128 / STG.E.128.
__device__ __forceinline__ Half8 ld8(const __half* p) {
  const uint4 u = *reinterpret_cast<const uint4*>(p);
  return *reinterpret_cast<const Half8*>(&u);
}
__device__ __forceinline__ void st8(__half* p, const Half8& h) {
  *reinterpret_cast<uint4*>(p) = *reinterpret_cast<const uint4*>(&h);
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float silu(float x) { return x / (1.f + __expf(-x)); }

// ============================================================================ GroupNorm
// x[b, hw, c] fp16. Thread t owns channel vector (t % nvec) for the rows (t / nvec) + k*rowlanes of its chunk.
struct GNPlan { int nvec, rowlanes, threads, chunks, rows_per_chunk; };

static GNPlan gn_plan(int batch, int hw, int c) {
  GNPlan p;
  p.nvec = c / 8;
  p.rowlanes = p.nvec >= 256 ? 1 : (256 / p.nvec);
  if (p.rowlanes < 1) p.rowlanes = 1;
  p.threads = p.nvec * p.rowlanes;
  int want = (592 + batch - 1) / batch;                 // ~4 CTAs per SM across the batch
  int maxc = (hw + p.rowlanes * 4 - 1) / (p.rowlanes * 4);  // at least 4 rows per thread
  if (maxc < 1) maxc = 1;
  p.chunks = want < maxc ? want : maxc;
  if (p.chunks > 128) p.chunks = 128;
  if (p.chunks < 1) p.chunks = 1;
  p.rows_per_chunk = (hw + p.chunks - 1) / p.chunks;
  p.rows_per_chunk = ((p.rows_per_chunk + p.rowlanes - 1) / p.rowlanes) * p.rowlanes;
  p.chunks = (hw + p.rows_per_chunk - 1) / p.rows_per_chunk;
  return p;
}

// partial (mean, m2) per (batch, chunk, group), m2 = sum of squared deviations from that mean: running (mean, m2) per
// thread, each batch of 4 rows reduced two-pass in registers and merged in (Chan et al.; Welford's update for the
// remainder rows), then the (thread, channel) partials merged into the group with stats_merge in a fixed order.
// No E[x^2] - E[x]^2 cancellation, whatever the offset of x. Up to c/8 = 1024 threads per CTA (rowlanes = 1 once
// nvec >= 256): the launch bound keeps it within 64 registers, so that every shape the entry point accepts launches.
__global__ void __launch_bounds__(1024) gn_stats_kernel(const __half* __restrict__ x, const __half* __restrict__ chan_bias,
                                float* __restrict__ ws, int hw, int c, int groups, int nvec, int rowlanes,
                                int rows_per_chunk, int chunks) {
  extern __shared__ float sm[];  // [rowlanes][c][2]
  const int b = blockIdx.y, chunk = blockIdx.x;
  const int vec = threadIdx.x % nvec, rl = threadIdx.x / nvec;
  const int r0 = chunk * rows_per_chunk;
  const int r1 = min(hw, r0 + rows_per_chunk);
  float s[8], ss[8], tb[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) { s[i] = 0.f; ss[i] = 0.f; tb[i] = 0.f; }
  if (chan_bias) unpack8(ld8(chan_bias + (size_t)b * c + vec * 8), tb);
  const __half* base = x + ((size_t)b * hw) * c + vec * 8;
  int cnt = 0;   // rows seen by this thread; s = running mean, ss = running m2
  int r = r0 + rl;
  for (; r + 3 * rowlanes < r1; r += 4 * rowlanes) {  // 4 independent 128-bit loads in flight per thread
    Half8 v[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) v[u] = ld8(base + (size_t)(r + u * rowlanes) * c);
    // the 4 rows as one batch (mean, m2), merged into the running statistics: one reciprocal; the halves are
    // converted a channel pair at a time, which keeps the kernel within 64 registers
    const float w = 4.f / (float)(cnt + 4), nw = (float)cnt * w;
    cnt += 4;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float2 t[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) t[u] = __half22float2(v[u].v[j]);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int i = 2 * j + h;
        const float t0 = (h ? t[0].y : t[0].x) + tb[i], t1 = (h ? t[1].y : t[1].x) + tb[i];
        const float t2 = (h ? t[2].y : t[2].x) + tb[i], t3 = (h ? t[3].y : t[3].x) + tb[i];
        const float bm = ((t0 + t1) + (t2 + t3)) * 0.25f;
        const float bq = fmaf(t3 - bm, t3 - bm, fmaf(t2 - bm, t2 - bm, fmaf(t1 - bm, t1 - bm, (t0 - bm) * (t0 - bm))));
        const float d = bm - s[i];
        s[i] = fmaf(d, w, s[i]);
        ss[i] = fmaf(d * d, nw, ss[i] + bq);
      }
    }
  }
  for (; r < r1; r += rowlanes) {
    float f[8];
    unpack8(ld8(base + (size_t)r * c), f);
    const float rc = 1.f / (float)(++cnt);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float t = f[i] + tb[i], d = t - s[i];
      s[i] = fmaf(d, rc, s[i]); ss[i] = fmaf(d, t - s[i], ss[i]);
    }
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    sm[((size_t)rl * c + vec * 8 + i) * 2] = s[i];
    sm[((size_t)rl * c + vec * 8 + i) * 2 + 1] = ss[i];
  }
  __syncthreads();
  const int cpg = c / groups;
  const int nrow = r1 - r0;
  for (int ch = threadIdx.x; ch < c; ch += blockDim.x) {   // each channel over its row lanes, into row lane 0's slot
    int n = 0;
    float mean = 0.f, m2 = 0.f;
    for (int l = 0; l < rowlanes && l < nrow; ++l)   // row lane l holds ceil((nrow - l) / rowlanes) rows
      stats_merge(n, mean, m2, (nrow - l + rowlanes - 1) / rowlanes, sm[((size_t)l * c + ch) * 2],
                  sm[((size_t)l * c + ch) * 2 + 1]);
    sm[(size_t)ch * 2] = mean; sm[(size_t)ch * 2 + 1] = m2;
  }
  __syncthreads();
  for (int g = threadIdx.x; g < groups; g += blockDim.x) {   // then the group's channels, nrow rows each
    int n = 0;
    float mean = 0.f, m2 = 0.f;
    for (int ch = g * cpg; ch < (g + 1) * cpg; ++ch) stats_merge(n, mean, m2, nrow, sm[(size_t)ch * 2], sm[(size_t)ch * 2 + 1]);
    float* o = ws + (((size_t)b * chunks + chunk) * groups + g) * 2;
    o[0] = mean; o[1] = m2;
  }
}

// one warp per (batch, group): fixed-order Chan merge of the chunk (mean, m2) -> (mean, rstd); chunk k holds
// min(rows_per_chunk, hw - k*rows_per_chunk) rows of cpg channels
__global__ void gn_finalize_kernel(const float* __restrict__ ws, float* __restrict__ mean_rstd, int groups, int chunks,
                                   int hw, int rows_per_chunk, int cpg, float n, float eps) {
  const int b = blockIdx.y;
  const int g = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (g >= groups) return;
  int cnt;
  float mean, m2;
  gn_lane_stats(ws + ((size_t)b * chunks * groups + g) * 2, groups, chunks, hw, rows_per_chunk, cpg, lane, cnt, mean, m2);
  stats_warp_merge(cnt, mean, m2);
  if (lane == 0) {
    mean_rstd[((size_t)b * groups + g) * 2] = mean;
    mean_rstd[((size_t)b * groups + g) * 2 + 1] = rsqrtf(m2 / n + eps);
  }
}

__global__ void gn_apply_kernel(const __half* __restrict__ x, const __half* __restrict__ chan_bias,
                                const __half* __restrict__ gamma, const __half* __restrict__ beta,
                                const float* __restrict__ mean_rstd, __half* __restrict__ y, int hw, int c, int groups,
                                int nvec, int rowlanes, int rows_per_chunk, int apply_silu) {
  const int b = blockIdx.y, chunk = blockIdx.x;
  const int cpg = c / groups;
  const float* sm = mean_rstd + (size_t)b * groups * 2;  // written by gn_finalize_kernel
  const int vec = threadIdx.x % nvec, rl = threadIdx.x / nvec;
  float sc[8], sh[8], ga[8], be[8], tb[8];
  unpack8(ld8(gamma + vec * 8), ga);
  unpack8(ld8(beta + vec * 8), be);
#pragma unroll
  for (int i = 0; i < 8; ++i) tb[i] = 0.f;
  if (chan_bias) unpack8(ld8(chan_bias + (size_t)b * c + vec * 8), tb);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int g = (vec * 8 + i) / cpg;
    sc[i] = ga[i] * sm[2 * g + 1];
    sh[i] = be[i] + (tb[i] - sm[2 * g]) * sc[i];
  }
  const int r0 = chunk * rows_per_chunk;
  const int r1 = min(hw, r0 + rows_per_chunk);
  const size_t base = ((size_t)b * hw) * c + vec * 8;
  int r = r0 + rl;
  for (; r + 3 * rowlanes < r1; r += 4 * rowlanes) {
    Half8 v[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) v[u] = ld8(x + base + (size_t)(r + u * rowlanes) * c);
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      float f[8];
      unpack8(v[u], f);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float t = fmaf(f[i], sc[i], sh[i]);
        f[i] = apply_silu ? silu(t) : t;
      }
      st8(y + base + (size_t)(r + u * rowlanes) * c, pack8(f));
    }
  }
  for (; r < r1; r += rowlanes) {
    float f[8];
    unpack8(ld8(x + base + (size_t)r * c), f);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float t = fmaf(f[i], sc[i], sh[i]);
      f[i] = apply_silu ? silu(t) : t;
    }
    st8(y + base + (size_t)r * c, pack8(f));
  }
}

// ============================================================================ LayerNorm
template <int VPL>  // vectors (8 halfs) per lane; one warp per row (measured faster than persistent warps)
__global__ void layernorm_kernel(const __half* __restrict__ x, const __half* __restrict__ gamma,
                                 const __half* __restrict__ beta, __half* __restrict__ y, int rows, int c,
                                 float eps) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= rows) return;
  const int nvec = c / 8;
  const __half* xr = x + (size_t)warp * c;
  Half8 raw[VPL];
#pragma unroll
  for (int k = 0; k < VPL; ++k)
    if (lane + 32 * k < nvec) raw[k] = ld8(xr + (lane + 32 * k) * 8);
  float f[VPL][8];
  float sum = 0.f;
#pragma unroll
  for (int k = 0; k < VPL; ++k)
    if (lane + 32 * k < nvec) {
      unpack8(raw[k], f[k]);
#pragma unroll
      for (int i = 0; i < 8; ++i) sum += f[k][i];
    }
  const float mean = warp_sum(sum) / (float)c;
  float sq = 0.f;
#pragma unroll
  for (int k = 0; k < VPL; ++k)
    if (lane + 32 * k < nvec) {
#pragma unroll
      for (int i = 0; i < 8; ++i) { const float d = f[k][i] - mean; sq += d * d; }
    }
  const float rstd = rsqrtf(warp_sum(sq) / (float)c + eps);
  __half* yr = y + (size_t)warp * c;
#pragma unroll
  for (int k = 0; k < VPL; ++k) {
    const int v = lane + 32 * k;
    if (v < nvec) {
      float ga[8], be[8], o[8];
      unpack8(ld8(gamma + v * 8), ga);
      unpack8(ld8(beta + v * 8), be);
#pragma unroll
      for (int i = 0; i < 8; ++i) o[i] = (f[k][i] - mean) * rstd * ga[i] + be[i];
      st8(yr + v * 8, pack8(o));
    }
  }
}

// ============================================================================ residual + bias + LayerNorm
// h = fp16(a + resid + bias[c]);  y = LayerNorm(h) * gamma + beta      (attention.py:155-181: `attn(...) + hidden_states`
// followed by the next norm). One pass over DRAM: reads a and resid, writes h (may alias resid) and y. The statistics
// are taken on the fp16-rounded h, i.e. on exactly the tensor later layers read.
template <int VPL>
__global__ void add_bias_layernorm_kernel(const __half* __restrict__ a, const __half* resid,
                                          const __half* __restrict__ bias, const __half* __restrict__ gamma,
                                          const __half* __restrict__ beta, __half* h_out, __half* __restrict__ y,
                                          int rows, int c, float eps) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= rows) return;
  const int nvec = c / 8;
  const size_t off = (size_t)warp * c;
  Half8 ra[VPL], rr[VPL];
#pragma unroll
  for (int k = 0; k < VPL; ++k)
    if (lane + 32 * k < nvec) {
      ra[k] = ld8(a + off + (lane + 32 * k) * 8);
      rr[k] = ld8(resid + off + (lane + 32 * k) * 8);
    }
  float f[VPL][8];
  float sum = 0.f;
#pragma unroll
  for (int k = 0; k < VPL; ++k) {
    const int v = lane + 32 * k;
    if (v < nvec) {
      float fa[8], fr[8], fb[8];
      unpack8(ra[k], fa);
      unpack8(rr[k], fr);
      if (bias != nullptr) unpack8(ld8(bias + v * 8), fb);
#pragma unroll
      for (int i = 0; i < 8; ++i) f[k][i] = fa[i] + fr[i] + (bias != nullptr ? fb[i] : 0.f);
      const Half8 hv = pack8(f[k]);
      st8(h_out + off + v * 8, hv);
      unpack8(hv, f[k]);   // the rounded values
#pragma unroll
      for (int i = 0; i < 8; ++i) sum += f[k][i];
    }
  }
  const float mean = warp_sum(sum) / (float)c;
  float sq = 0.f;
#pragma unroll
  for (int k = 0; k < VPL; ++k)
    if (lane + 32 * k < nvec) {
#pragma unroll
      for (int i = 0; i < 8; ++i) { const float d = f[k][i] - mean; sq += d * d; }
    }
  const float rstd = rsqrtf(warp_sum(sq) / (float)c + eps);
#pragma unroll
  for (int k = 0; k < VPL; ++k) {
    const int v = lane + 32 * k;
    if (v < nvec) {
      float ga[8], be[8], o[8];
      unpack8(ld8(gamma + v * 8), ga);
      unpack8(ld8(beta + v * 8), be);
#pragma unroll
      for (int i = 0; i < 8; ++i) o[i] = (f[k][i] - mean) * rstd * ga[i] + be[i];
      st8(y + off + v * 8, pack8(o));
    }
  }
}

// ============================================================================ GEGLU
__global__ void geglu_kernel(const __half* __restrict__ proj, __half* __restrict__ y, long long rows, int inner) {
  const int nvec = inner / 8;
  const long long total = rows * nvec;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const long long r = idx / nvec;
    const int v = (int)(idx - r * nvec);
    const __half* pr = proj + r * 2 * inner;
    float a[8], g[8];
    unpack8(ld8(pr + v * 8), a);
    unpack8(ld8(pr + inner + v * 8), g);
#pragma unroll
    for (int i = 0; i < 8; ++i) a[i] *= 0.5f * g[i] * (1.f + erff(g[i] * 0.70710678118654752f));
    st8(y + r * inner + v * 8, pack8(a));
  }
}

// ============================================================================ region blend + CFG
struct BlendPtrs { const __half* eps[16]; };

// step policies (rtti_internal.h): Euler, the multistep update of MsStep, the ancestral update of AncStep, the UniPC
// update of UniPCStep, the Heun update of HeunStep, the LMS update of LmsStep, or the DPM-Solver++(2S) update of SsStep
struct EulerStep { float dt_sigma; };
__device__ __forceinline__ void apply_step(const EulerStep& s, long long, const float* e16, float* x) {
#pragma unroll
  for (int i = 0; i < 8; ++i) x[i] = fmaf(e16[i], s.dt_sigma, x[i]);
}
__device__ __forceinline__ void apply_step(const MsStep& s, long long v, const float* e16, float* x) { ms_step8(s, v, e16, x); }
__device__ __forceinline__ void apply_step(const AncStep& s, long long v, const float* e16, float* x) { anc_step8(s, v, e16, x); }
__device__ __forceinline__ void apply_step(const UniPCStep& s, long long v, const float* e16, float* x) {
  unipc_step8(s, v, e16, x);
}
__device__ __forceinline__ void apply_step(const HeunStep& s, long long v, const float* e16, float* x) { heun_step8(s, v, e16, x); }
__device__ __forceinline__ void apply_step(const LmsStep& s, long long v, const float* e16, float* x) { lms_step8(s, v, e16, x); }
__device__ __forceinline__ void apply_step(const SsStep& s, long long v, const float* e16, float* x) { ss_step8(s, v, e16, x); }

template <class Step>
__device__ __forceinline__ void region_blend_body(const __half* __restrict__ eps_uncond, const BlendPtrs& ptrs,
                                                  const float* __restrict__ masks, int n_regions, long long n,
                                                  float guidance, __half* __restrict__ eps_out,
                                                  const __half* __restrict__ latents, __half* __restrict__ latents_out,
                                                  const Step& st) {
  const long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (v * 8 >= n) return;
  float eu[8], msum[8], et[8];
  unpack8(ld8(eps_uncond + v * 8), eu);
#pragma unroll
  for (int i = 0; i < 8; ++i) { msum[i] = 0.f; et[i] = 0.f; }
  for (int r = 0; r < n_regions; ++r) {
    float e[8];
    unpack8(ld8(ptrs.eps[r] + v * 8), e);
    const float4 m0 = *reinterpret_cast<const float4*>(masks + (size_t)r * n + v * 8);
    const float4 m1 = *reinterpret_cast<const float4*>(masks + (size_t)r * n + v * 8 + 4);
    const float m[8] = {m0.x, m0.y, m0.z, m0.w, m1.x, m1.y, m1.z, m1.w};
#pragma unroll
    for (int i = 0; i < 8; ++i) { msum[i] += m[i]; et[i] = fmaf(e[i], m[i], et[i]); }
  }
  float o[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const float u = eu[i] * msum[i];
    o[i] = u + guidance * (et[i] - u);
  }
  const Half8 oh = pack8(o);
  st8(eps_out + v * 8, oh);
  if (latents != nullptr) {
    float x[8], e16[8];
    unpack8(ld8(latents + v * 8), x);
    unpack8(oh, e16);  // the scheduler consumes the fp16-rounded noise prediction
    apply_step(st, v, e16, x);
    st8(latents_out + v * 8, pack8(x));
  }
}

__global__ void region_blend_kernel(const __half* __restrict__ eps_uncond, BlendPtrs ptrs,
                                    const float* __restrict__ masks, int n_regions, long long n, float guidance,
                                    __half* __restrict__ eps_out, const __half* __restrict__ latents,
                                    __half* __restrict__ latents_out, float dt_sigma) {
  region_blend_body(eps_uncond, ptrs, masks, n_regions, n, guidance, eps_out, latents, latents_out, EulerStep{dt_sigma});
}

__global__ void region_blend_ms_kernel(const __half* __restrict__ eps_uncond, BlendPtrs ptrs,
                                       const float* __restrict__ masks, int n_regions, long long n, float guidance,
                                       __half* __restrict__ eps_out, const __half* __restrict__ latents,
                                       __half* __restrict__ latents_out, const MsStep st) {
  region_blend_body(eps_uncond, ptrs, masks, n_regions, n, guidance, eps_out, latents, latents_out, st);
}

__global__ void region_blend_anc_kernel(const __half* __restrict__ eps_uncond, BlendPtrs ptrs,
                                        const float* __restrict__ masks, int n_regions, long long n, float guidance,
                                        __half* __restrict__ eps_out, const __half* __restrict__ latents,
                                        __half* __restrict__ latents_out, const AncStep st) {
  region_blend_body(eps_uncond, ptrs, masks, n_regions, n, guidance, eps_out, latents, latents_out, st);
}

__global__ void region_blend_unipc_kernel(const __half* __restrict__ eps_uncond, BlendPtrs ptrs,
                                          const float* __restrict__ masks, int n_regions, long long n, float guidance,
                                          __half* __restrict__ eps_out, const __half* __restrict__ latents,
                                          __half* __restrict__ latents_out, const UniPCStep st) {
  region_blend_body(eps_uncond, ptrs, masks, n_regions, n, guidance, eps_out, latents, latents_out, st);
}

__global__ void region_blend_heun_kernel(const __half* __restrict__ eps_uncond, BlendPtrs ptrs,
                                         const float* __restrict__ masks, int n_regions, long long n, float guidance,
                                         __half* __restrict__ eps_out, const __half* __restrict__ latents,
                                         __half* __restrict__ latents_out, const HeunStep st) {
  region_blend_body(eps_uncond, ptrs, masks, n_regions, n, guidance, eps_out, latents, latents_out, st);
}

__global__ void region_blend_lms_kernel(const __half* __restrict__ eps_uncond, BlendPtrs ptrs,
                                        const float* __restrict__ masks, int n_regions, long long n, float guidance,
                                        __half* __restrict__ eps_out, const __half* __restrict__ latents,
                                        __half* __restrict__ latents_out, const LmsStep st) {
  region_blend_body(eps_uncond, ptrs, masks, n_regions, n, guidance, eps_out, latents, latents_out, st);
}

__global__ void region_blend_ss_kernel(const __half* __restrict__ eps_uncond, BlendPtrs ptrs,
                                       const float* __restrict__ masks, int n_regions, long long n, float guidance,
                                       __half* __restrict__ eps_out, const __half* __restrict__ latents,
                                       __half* __restrict__ latents_out, const SsStep st) {
  region_blend_body(eps_uncond, ptrs, masks, n_regions, n, guidance, eps_out, latents, latents_out, st);
}

// ============================================================================ colour guidance
constexpr int CL_BLOCKS = 296;
constexpr int CL_MAXC = 16;

// stage 1: per block partial sums  [block][color][4] = {sum m, sum img_r m, sum img_g m, sum img_b m}
__global__ void color_partial_kernel(const float* __restrict__ dec, const float* __restrict__ masks, int n_colors,
                                     long long hw, float* __restrict__ ws) {
  __shared__ float red[8][4];
  for (int col = 0; col < n_colors; ++col) {
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < hw; p += (long long)gridDim.x * blockDim.x) {
      const float m = masks[(size_t)col * hw + p];
      acc[0] += m;
#pragma unroll
      for (int ch = 0; ch < 3; ++ch) {
        const float img = fminf(fmaxf(dec[(size_t)ch * hw + p] * 0.5f + 0.5f, 0.f), 1.f);
        acc[1 + ch] = fmaf(img, m, acc[1 + ch]);
      }
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) acc[k] = warp_sum(acc[k]);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0) { red[warp][0] = acc[0]; red[warp][1] = acc[1]; red[warp][2] = acc[2]; red[warp][3] = acc[3]; }
    __syncthreads();
    if (threadIdx.x < 4) {
      float t = 0.f;
      for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += red[w][threadIdx.x];
      ws[((size_t)blockIdx.x * n_colors + col) * 4 + threadIdx.x] = t;
    }
    __syncthreads();
  }
}
// stage 2: one block — reduce partials in fixed order, loss, and gradient coefficients coef[color][3]
__global__ void color_finalize_kernel(const float* __restrict__ ws, const float* __restrict__ target, int n_colors,
                                      int blocks, float* __restrict__ loss_out, float* __restrict__ coef) {
  __shared__ float loss_terms[CL_MAXC];
  const int col = threadIdx.x;
  if (col < n_colors) {
    float t[4] = {0.f, 0.f, 0.f, 0.f};
    for (int b = 0; b < blocks; ++b)
#pragma unroll
      for (int k = 0; k < 4; ++k) t[k] += ws[((size_t)b * n_colors + col) * 4 + k];
    float lt = 0.f;
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
      const float avg = t[1 + ch] / t[0];
      const float d = avg - target[col * 3 + ch];
      lt += d * d;
      coef[col * 3 + ch] = 100.f * (2.f / 3.f) * d / t[0];
    }
    loss_terms[col] = lt * (100.f / 3.f);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int i = 0; i < n_colors; ++i) s += loss_terms[i];
    *loss_out = s;
  }
}
// stage 3: d loss / d decoded  (clamp passes gradient on the closed interval, as torch.clamp does)
__global__ void color_grad_kernel(const float* __restrict__ dec, const float* __restrict__ masks,
                                  const float* __restrict__ coef, int n_colors, long long hw,
                                  float* __restrict__ grad) {
  __shared__ float cf[CL_MAXC * 3];
  if (threadIdx.x < n_colors * 3) cf[threadIdx.x] = coef[threadIdx.x];
  __syncthreads();
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < hw; p += (long long)gridDim.x * blockDim.x) {
    float g[3] = {0.f, 0.f, 0.f};
    for (int col = 0; col < n_colors; ++col) {
      const float m = masks[(size_t)col * hw + p];
#pragma unroll
      for (int ch = 0; ch < 3; ++ch) g[ch] = fmaf(cf[col * 3 + ch], m, g[ch]);
    }
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
      const float img = dec[(size_t)ch * hw + p] * 0.5f + 0.5f;
      grad[(size_t)ch * hw + p] = (img >= 0.f && img <= 1.f) ? 0.5f * g[ch] : 0.f;
    }
  }
}

// ============================================================================ small latent-space kernels
__global__ void guidance_update_kernel(const __half* __restrict__ lat, const float* __restrict__ grad,
                                       const float* __restrict__ atten, float weight, __half* __restrict__ out,
                                       long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = __float2half_rn(__half2float(lat[i]) - grad[i] * weight * atten[i]);
}
__global__ void bg_inject_kernel(const __half* __restrict__ lat, const __half* __restrict__ ref,
                                 const float* __restrict__ m, __half* __restrict__ out, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    const float mm = m[i];
    out[i] = __float2half_rn(__half2float(ref[i]) * mm + __half2float(lat[i]) * (1.f - mm));
  }
}
__global__ void predict_x0_kernel(const __half* __restrict__ xt, const __half* __restrict__ eps, float sq1ma,
                                  float inv_sqa, __half* __restrict__ x0, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) x0[i] = __float2half_rn((__half2float(xt[i]) - __half2float(eps[i]) * sq1ma) * inv_sqa);
}

// out[r, c] = a[r, c] + b[r, c] + bias[c]  (fp16; residual add of a resnet block fused with the conv2 bias, which
// PyTorch otherwise adds to a channels-last convolution output in a separate broadcast pass)
__global__ void add_bias_f16_kernel(const __half* __restrict__ a, const __half* __restrict__ b,
                                    const __half* __restrict__ bias, __half* __restrict__ out, long long nvec, int cvec) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (long long)gridDim.x * blockDim.x) {
    float x[8], y[8], z[8];
    unpack8(ld8(a + (size_t)(i) * 8), x);
    unpack8(ld8(b + (size_t)(i) * 8), y);
#pragma unroll
    for (int k = 0; k < 8; ++k) z[k] = 0.f;
    if (bias) unpack8(ld8(bias + (size_t)(i % cvec) * 8), z);
#pragma unroll
    for (int k = 0; k < 8; ++k) x[k] = x[k] + y[k] + z[k];
    st8(out + (size_t)(i) * 8, pack8(x));
  }
}

static inline int ok_or_cuda() { return cudaGetLastError() == cudaSuccess ? RTTI_OK : RTTI_ERR_CUDA; }

}  // namespace rtti

using namespace rtti;

extern "C" long long rtti_groupnorm_workspace_elems(int batch, int hw, int c, int groups) {
  if (batch < 1 || hw < 1 || c < 8 || groups < 1) return 0;
  const GNPlan p = gn_plan(batch, hw, c);
  return (long long)batch * p.chunks * groups * 2 + (long long)batch * groups * 2;
}

extern "C" int rtti_groupnorm_silu_fwd(const void* x, const void* chan_bias, const void* gamma, const void* beta,
                                       void* y, float* workspace, int batch, int hw, int c, int groups, float eps,
                                       int apply_silu, void* stream) {
  if (!x || !gamma || !beta || !y || !workspace) return RTTI_ERR_ARG;
  if (batch < 1 || hw < 1 || groups < 1) return RTTI_ERR_ARG;
  if (c % 8 != 0 || c % groups != 0 || c / 8 > 1024) return RTTI_ERR_SHAPE;
  if (((uintptr_t)x | (uintptr_t)y | (uintptr_t)gamma | (uintptr_t)beta | (uintptr_t)chan_bias) & 15) return RTTI_ERR_ALIGN;
  const GNPlan p = gn_plan(batch, hw, c);
  const size_t sm1 = (size_t)p.rowlanes * c * 2 * sizeof(float);
  if (sm1 > 200 * 1024) return RTTI_ERR_SHAPE;
  cudaStream_t st = (cudaStream_t)stream;
  if (sm1 > 48 * 1024) {
    if (cudaFuncSetAttribute(gn_stats_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm1) != cudaSuccess)
      return RTTI_ERR_CUDA;
  }
  dim3 grid(p.chunks, batch);
  gn_stats_kernel<<<grid, p.threads, sm1, st>>>((const __half*)x, (const __half*)chan_bias, workspace, hw, c, groups,
                                                p.nvec, p.rowlanes, p.rows_per_chunk, p.chunks);
  float* mean_rstd = workspace + (size_t)batch * p.chunks * groups * 2;
  gn_finalize_kernel<<<dim3((groups + 7) / 8, batch), 256, 0, st>>>(workspace, mean_rstd, groups, p.chunks, hw,
                                                                    p.rows_per_chunk, c / groups,
                                                                    (float)hw * (float)(c / groups), eps);
  gn_apply_kernel<<<grid, p.threads, 0, st>>>((const __half*)x, (const __half*)chan_bias, (const __half*)gamma,
                                              (const __half*)beta, mean_rstd, (__half*)y, hw, c, groups, p.nvec,
                                              p.rowlanes, p.rows_per_chunk, apply_silu);
  return ok_or_cuda();
}

extern "C" int rtti_layernorm_fwd(const void* x, const void* gamma, const void* beta, void* y, int rows, int c,
                                  float eps, void* stream) {
  if (!x || !gamma || !beta || !y) return RTTI_ERR_ARG;
  if (rows < 1) return RTTI_ERR_ARG;
  if (c % 8 != 0 || c > 8 * 32 * 8) return RTTI_ERR_SHAPE;
  if (((uintptr_t)x | (uintptr_t)y | (uintptr_t)gamma | (uintptr_t)beta) & 15) return RTTI_ERR_ALIGN;
  cudaStream_t st = (cudaStream_t)stream;
  const int vpl = (c / 8 + 31) / 32;
  const int blocks = (rows + 7) / 8;
#define LN(V) layernorm_kernel<V><<<blocks, 256, 0, st>>>((const __half*)x, (const __half*)gamma, (const __half*)beta, (__half*)y, rows, c, eps)
  if (vpl <= 1) LN(1); else if (vpl <= 2) LN(2); else if (vpl <= 3) LN(3); else if (vpl <= 4) LN(4);
  else if (vpl <= 5) LN(5); else if (vpl <= 6) LN(6); else LN(8);
#undef LN
  return ok_or_cuda();
}

extern "C" int rtti_add_bias_layernorm_fwd(const void* a, const void* resid, const void* bias, const void* gamma,
                                           const void* beta, void* h_out, void* y, int rows, int c, float eps,
                                           void* stream) {
  if (!a || !resid || !gamma || !beta || !h_out || !y) return RTTI_ERR_ARG;
  if (rows < 1) return RTTI_ERR_ARG;
  if (c % 8 != 0 || c > 8 * 32 * 8) return RTTI_ERR_SHAPE;
  if (((uintptr_t)a | (uintptr_t)resid | (uintptr_t)bias | (uintptr_t)gamma | (uintptr_t)beta | (uintptr_t)h_out | (uintptr_t)y) & 15)
    return RTTI_ERR_ALIGN;
  cudaStream_t st = (cudaStream_t)stream;
  const int vpl = (c / 8 + 31) / 32;
  const int blocks = (rows + 7) / 8;
#define ALN(V) add_bias_layernorm_kernel<V><<<blocks, 256, 0, st>>>((const __half*)a, (const __half*)resid, (const __half*)bias, \
    (const __half*)gamma, (const __half*)beta, (__half*)h_out, (__half*)y, rows, c, eps)
  if (vpl <= 1) ALN(1); else if (vpl <= 2) ALN(2); else if (vpl <= 3) ALN(3); else if (vpl <= 4) ALN(4);
  else if (vpl <= 5) ALN(5); else if (vpl <= 6) ALN(6); else ALN(8);
#undef ALN
  return ok_or_cuda();
}

extern "C" int rtti_geglu_fwd(const void* proj, void* y, int rows, int inner, void* stream) {
  if (!proj || !y) return RTTI_ERR_ARG;
  if (rows < 1 || inner < 8) return RTTI_ERR_ARG;
  if (inner % 8 != 0) return RTTI_ERR_SHAPE;
  if (((uintptr_t)proj | (uintptr_t)y) & 15) return RTTI_ERR_ALIGN;
  const long long total = (long long)rows * (inner / 8);
  long long blocks = (total + 255) / 256;
  if (blocks > 132 * 16) blocks = 132 * 16;
  geglu_kernel<<<(int)blocks, 256, 0, (cudaStream_t)stream>>>((const __half*)proj, (__half*)y, rows, inner);
  return ok_or_cuda();
}

// argument checks shared by rtti_region_blend_cfg and its _ms / _anc / _unipc forms; fills the region pointer table
static int region_blend_args(const void* eps_uncond, const void* const* eps_region, const float* masks, int n_regions,
                             long long n, void* eps_out, const void* latents, void* latents_out, BlendPtrs& ptrs) {
  if (!eps_uncond || !eps_region || !masks || !eps_out) return RTTI_ERR_ARG;
  if (n_regions < 1 || n_regions > 16 || n < 8) return RTTI_ERR_ARG;
  if (n % 8 != 0) return RTTI_ERR_SHAPE;
  if ((latents == nullptr) != (latents_out == nullptr)) return RTTI_ERR_ARG;
  uintptr_t al = (uintptr_t)eps_uncond | (uintptr_t)masks | (uintptr_t)eps_out | (uintptr_t)latents | (uintptr_t)latents_out;
  for (int i = 0; i < n_regions; ++i) {
    if (!eps_region[i]) return RTTI_ERR_ARG;
    ptrs.eps[i] = (const __half*)eps_region[i];
    al |= (uintptr_t)eps_region[i];
  }
  return (al & 15) ? RTTI_ERR_ALIGN : RTTI_OK;
}

extern "C" int rtti_region_blend_cfg(const void* eps_uncond, const void* const* eps_region, const float* masks,
                                     int n_regions, long long n, float guidance, void* eps_out, const void* latents,
                                     void* latents_out, float dt_sigma, void* stream) {
  BlendPtrs ptrs{};
  const int rc = region_blend_args(eps_uncond, eps_region, masks, n_regions, n, eps_out, latents, latents_out, ptrs);
  if (rc != RTTI_OK) return rc;
  const long long nv = n / 8;
  region_blend_kernel<<<(int)((nv + 127) / 128), 128, 0, (cudaStream_t)stream>>>(
      (const __half*)eps_uncond, ptrs, masks, n_regions, n, guidance, (__half*)eps_out, (const __half*)latents,
      (__half*)latents_out, dt_sigma);
  return ok_or_cuda();
}

extern "C" int rtti_region_blend_cfg_ms(const void* eps_uncond, const void* const* eps_region, const float* masks,
                                        int n_regions, long long n, float guidance, void* eps_out, const void* latents,
                                        void* latents_out, float hx, float he, float cx, float cd, float cp,
                                        const float* d_prev, float* d_out, void* stream) {
  if (!latents || !latents_out) return RTTI_ERR_ARG;
  BlendPtrs ptrs{};
  int rc = region_blend_args(eps_uncond, eps_region, masks, n_regions, n, eps_out, latents, latents_out, ptrs);
  if (rc == RTTI_OK) rc = ms_step_args(cp, d_prev, d_out);
  if (rc != RTTI_OK) return rc;
  const long long nv = n / 8;
  region_blend_ms_kernel<<<(int)((nv + 127) / 128), 128, 0, (cudaStream_t)stream>>>(
      (const __half*)eps_uncond, ptrs, masks, n_regions, n, guidance, (__half*)eps_out, (const __half*)latents,
      (__half*)latents_out, MsStep{hx, he, cx, cd, cp, d_prev, d_out});
  return ok_or_cuda();
}

extern "C" int rtti_region_blend_cfg_anc(const void* eps_uncond, const void* const* eps_region, const float* masks,
                                         int n_regions, long long n, float guidance, void* eps_out, const void* latents,
                                         void* latents_out, float dt_sigma, float s_up, const void* z, void* stream) {
  if (!latents || !latents_out) return RTTI_ERR_ARG;
  BlendPtrs ptrs{};
  int rc = region_blend_args(eps_uncond, eps_region, masks, n_regions, n, eps_out, latents, latents_out, ptrs);
  if (rc == RTTI_OK) rc = anc_step_args(s_up, z);
  if (rc != RTTI_OK) return rc;
  const long long nv = n / 8;
  region_blend_anc_kernel<<<(int)((nv + 127) / 128), 128, 0, (cudaStream_t)stream>>>(
      (const __half*)eps_uncond, ptrs, masks, n_regions, n, guidance, (__half*)eps_out, (const __half*)latents,
      (__half*)latents_out, AncStep{dt_sigma, s_up, (const __half*)z});
  return ok_or_cuda();
}

extern "C" int rtti_region_blend_cfg_unipc(const void* eps_uncond, const void* const* eps_region, const float* masks,
                                           int n_regions, long long n, float guidance, void* eps_out,
                                           const void* latents, void* latents_out, float hx, float he, float ux,
                                           float ul, float u0, float u1, float u2, float vx, float v0, float v1,
                                           const float* xl, const float* m1, const float* m2, float* m_out,
                                           float* xl_out, void* stream) {
  if (!latents || !latents_out) return RTTI_ERR_ARG;
  BlendPtrs ptrs{};
  int rc = region_blend_args(eps_uncond, eps_region, masks, n_regions, n, eps_out, latents, latents_out, ptrs);
  if (rc == RTTI_OK) rc = unipc_step_args(ul, u1, u2, v1, xl, m1, m2, m_out, xl_out);
  if (rc != RTTI_OK) return rc;
  const long long nv = n / 8;
  region_blend_unipc_kernel<<<(int)((nv + 127) / 128), 128, 0, (cudaStream_t)stream>>>(
      (const __half*)eps_uncond, ptrs, masks, n_regions, n, guidance, (__half*)eps_out, (const __half*)latents,
      (__half*)latents_out, UniPCStep{hx, he, ux, ul, u0, u1, u2, vx, v0, v1, xl, m1, m2, m_out, xl_out});
  return ok_or_cuda();
}

extern "C" int rtti_region_blend_cfg_heun(const void* eps_uncond, const void* const* eps_region, const float* masks,
                                          int n_regions, long long n, float guidance, void* eps_out,
                                          const void* latents, void* latents_out, float cx, float ce, float cs,
                                          float cd, const void* xs, const void* ds, void* stream) {
  if (!latents || !latents_out) return RTTI_ERR_ARG;
  BlendPtrs ptrs{};
  int rc = region_blend_args(eps_uncond, eps_region, masks, n_regions, n, eps_out, latents, latents_out, ptrs);
  if (rc == RTTI_OK) rc = heun_step_args(cs, cd, xs, ds);
  if (rc != RTTI_OK) return rc;
  const long long nv = n / 8;
  region_blend_heun_kernel<<<(int)((nv + 127) / 128), 128, 0, (cudaStream_t)stream>>>(
      (const __half*)eps_uncond, ptrs, masks, n_regions, n, guidance, (__half*)eps_out, (const __half*)latents,
      (__half*)latents_out, HeunStep{cx, ce, cs, cd, (const __half*)xs, (const __half*)ds});
  return ok_or_cuda();
}

extern "C" int rtti_region_blend_cfg_lms(const void* eps_uncond, const void* const* eps_region, const float* masks,
                                         int n_regions, long long n, float guidance, void* eps_out, const void* latents,
                                         void* latents_out, float c0, float c1, float c2, float c3, const void* d1,
                                         const void* d2, const void* d3, void* stream) {
  if (!latents || !latents_out) return RTTI_ERR_ARG;
  BlendPtrs ptrs{};
  int rc = region_blend_args(eps_uncond, eps_region, masks, n_regions, n, eps_out, latents, latents_out, ptrs);
  if (rc == RTTI_OK) rc = lms_step_args(c1, c2, c3, d1, d2, d3);
  if (rc != RTTI_OK) return rc;
  const long long nv = n / 8;
  region_blend_lms_kernel<<<(int)((nv + 127) / 128), 128, 0, (cudaStream_t)stream>>>(
      (const __half*)eps_uncond, ptrs, masks, n_regions, n, guidance, (__half*)eps_out, (const __half*)latents,
      (__half*)latents_out, LmsStep{c0, c1, c2, c3, (const __half*)d1, (const __half*)d2, (const __half*)d3});
  return ok_or_cuda();
}

extern "C" int rtti_region_blend_cfg_ss(const void* eps_uncond, const void* const* eps_region, const float* masks,
                                        int n_regions, long long n, float guidance, void* eps_out, const void* latents,
                                        void* latents_out, float hx, float he, float cx, float cs, float cd, float cp,
                                        const float* d_prev, float* d_out, const void* xs, void* stream) {
  if (!latents || !latents_out) return RTTI_ERR_ARG;
  BlendPtrs ptrs{};
  int rc = region_blend_args(eps_uncond, eps_region, masks, n_regions, n, eps_out, latents, latents_out, ptrs);
  if (rc == RTTI_OK) rc = ss_step_args(cs, cp, xs, d_prev, d_out);
  if (rc != RTTI_OK) return rc;
  const long long nv = n / 8;
  region_blend_ss_kernel<<<(int)((nv + 127) / 128), 128, 0, (cudaStream_t)stream>>>(
      (const __half*)eps_uncond, ptrs, masks, n_regions, n, guidance, (__half*)eps_out, (const __half*)latents,
      (__half*)latents_out, SsStep{MsStep{hx, he, cx, cd, cp, d_prev, d_out}, cs, (const __half*)xs});
  return ok_or_cuda();
}

extern "C" long long rtti_color_loss_workspace_elems(int n_colors, long long hw) {
  if (n_colors < 1 || n_colors > CL_MAXC || hw < 1) return 0;
  return (long long)CL_BLOCKS * n_colors * 4 + n_colors * 3;
}

extern "C" int rtti_color_loss_fwd_bwd(const float* decoded, const float* masks, const float* target_rgb,
                                       int n_colors, long long hw, float* loss_out, float* grad_decoded,
                                       float* workspace, void* stream) {
  if (!decoded || !masks || !target_rgb || !loss_out || !grad_decoded || !workspace) return RTTI_ERR_ARG;
  if (n_colors < 1 || n_colors > CL_MAXC || hw < 1) return RTTI_ERR_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  float* coef = workspace + (size_t)CL_BLOCKS * n_colors * 4;
  color_partial_kernel<<<CL_BLOCKS, 256, 0, st>>>(decoded, masks, n_colors, hw, workspace);
  color_finalize_kernel<<<1, 32, 0, st>>>(workspace, target_rgb, n_colors, CL_BLOCKS, loss_out, coef);
  color_grad_kernel<<<CL_BLOCKS * 4, 256, 0, st>>>(decoded, masks, coef, n_colors, hw, grad_decoded);
  return ok_or_cuda();
}

extern "C" int rtti_latent_guidance_update(const void* latents, const float* grad, const float* atten_all,
                                           float weight, void* latents_out, long long n, void* stream) {
  if (!latents || !grad || !atten_all || !latents_out || n < 1) return RTTI_ERR_ARG;
  guidance_update_kernel<<<(int)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      (const __half*)latents, grad, atten_all, weight, (__half*)latents_out, n);
  return ok_or_cuda();
}

extern "C" int rtti_bg_inject_blend(const void* latents, const void* latents_ref, const float* mask, void* out,
                                    long long n, void* stream) {
  if (!latents || !latents_ref || !mask || !out || n < 1) return RTTI_ERR_ARG;
  bg_inject_kernel<<<(int)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      (const __half*)latents, (const __half*)latents_ref, mask, (__half*)out, n);
  return ok_or_cuda();
}

extern "C" int rtti_predict_x0(const void* x_t, const void* eps, float alpha, void* x0, long long n, void* stream) {
  if (!x_t || !eps || !x0 || n < 1 || !(alpha > 0.f) || alpha > 1.f) return RTTI_ERR_ARG;
  predict_x0_kernel<<<(int)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      (const __half*)x_t, (const __half*)eps, sqrtf(1.f - alpha), 1.f / sqrtf(alpha), (__half*)x0, n);
  return ok_or_cuda();
}

extern "C" int rtti_add_bias_f16(const void* a, const void* b, const void* bias, void* out, long long rows, int c,
                                 void* stream) {
  if (!a || !b || !out || rows < 1 || c < 8) return RTTI_ERR_ARG;
  if (c % 8 != 0) return RTTI_ERR_SHAPE;
  if (((uintptr_t)a | (uintptr_t)b | (uintptr_t)out | (uintptr_t)bias) & 15) return RTTI_ERR_ALIGN;
  const long long nvec = rows * (c / 8);
  long long blocks = (nvec + 255) / 256;
  if (blocks > 132 * 16) blocks = 132 * 16;
  add_bias_f16_kernel<<<(int)blocks, 256, 0, (cudaStream_t)stream>>>((const __half*)a, (const __half*)b, (const __half*)bias,
                                                                     (__half*)out, nvec, c / 8);
  return ok_or_cuda();
}
