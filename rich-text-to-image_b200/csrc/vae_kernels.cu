// fp32 channels-last GroupNorm(+SiLU) forward and backward (input gradient only) for the VAE decoder that
// colour guidance differentiates through (reference: third-party AutoencoderKL called at
// models/region_diffusion_sdxl.py:856-865; SURVEY §8(f).1).  PyTorch's native GroupNorm copies a
// channels-last fp32 tensor to NCHW and back and reduces it row-wise (~100 ms of a 350 ms step in the
// first profile); these kernels work on the NHWC data in place: x [B, HW, C] fp32, groups of C/G channels.
//   forward : partial (mean, m2) per (b, chunk, g)  ->  finalize mean/rstd (Chan merge)  ->  y = silu?(xhat*gamma+beta)
//   backward: dy = dz * silu'(y) (y recomputed), partial (sum dy*gamma, sum dy*gamma*xhat) -> finalize ->
//             dx = rstd * (dy*gamma - c1 - xhat*c2)
// Deterministic (fixed-order two-stage reductions, no atomics); 128-bit vector accesses.
#include "peer_sync.cuh"
#include "rtti_internal.h"

namespace rtti {

struct GN32Plan { int nvec, rowlanes, threads, chunks, rows_per_chunk; };

static GN32Plan gn32_plan(int batch, int hw, int c) {
  GN32Plan p;
  p.nvec = c / 4;
  p.rowlanes = p.nvec >= 256 ? 1 : (256 / p.nvec);
  p.threads = p.nvec * p.rowlanes;
  int want = (132 * 8 + batch - 1) / batch;
  int maxc = (hw + p.rowlanes * 8 - 1) / (p.rowlanes * 8);  // at least 8 rows per thread
  if (maxc < 1) maxc = 1;
  p.chunks = want < maxc ? want : maxc;
  if (p.chunks < 1) p.chunks = 1;
  p.rows_per_chunk = (hw + p.chunks - 1) / p.chunks;
  p.rows_per_chunk = ((p.rows_per_chunk + p.rowlanes - 1) / p.rowlanes) * p.rowlanes;
  p.chunks = (hw + p.rows_per_chunk - 1) / p.rows_per_chunk;
  return p;
}

__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + __expf(-x)); }

// MODE 0: (mean, m2) of x per (b, chunk, g), m2 = sum of squared deviations from that mean. Each thread keeps running
//         (mean, m2) of its rows: each batch of 4 rows is reduced two-pass in registers and merged in (Chan et al.;
//         Welford's update for the remainder rows), then the (thread, channel) partials are merged into the group with
//         stats_merge in a fixed order. One read of x, no E[x^2] - E[x]^2 cancellation.
// MODE 1: backward sums (sum dy*gamma, sum dy*gamma*xhat).
template <int MODE>
__global__ void gn32_partial_kernel(const float* __restrict__ x, const float* __restrict__ cbias,
                                    const float* __restrict__ dz,
                                    const float* __restrict__ gamma, const float* __restrict__ beta,
                                    const float* __restrict__ mean_rstd, float* __restrict__ ws, int hw, int c,
                                    int groups, int nvec, int rowlanes, int rows_per_chunk, int chunks, int silu) {
  extern __shared__ float sm[];  // [rowlanes][c][2]
  const int b = blockIdx.y, chunk = blockIdx.x;
  const int vec = threadIdx.x % nvec, rl = threadIdx.x / nvec;
  const int cpg = c / groups;
  const int r0 = chunk * rows_per_chunk, r1 = min(hw, r0 + rows_per_chunk);
  float a[4] = {0.f, 0.f, 0.f, 0.f}, q[4] = {0.f, 0.f, 0.f, 0.f};
  float ga[4] = {1.f, 1.f, 1.f, 1.f}, be[4] = {0.f, 0.f, 0.f, 0.f}, mu[4], rs[4];
  float cb[4] = {0.f, 0.f, 0.f, 0.f};   // per-channel bias of the producing convolution, folded in (x := x + cb)
  if (cbias) { const float4 c4 = *reinterpret_cast<const float4*>(cbias + vec * 4); cb[0] = c4.x; cb[1] = c4.y; cb[2] = c4.z; cb[3] = c4.w; }
  if (MODE == 1) {
    const float4 g4 = *reinterpret_cast<const float4*>(gamma + vec * 4);
    const float4 b4 = *reinterpret_cast<const float4*>(beta + vec * 4);
    ga[0] = g4.x; ga[1] = g4.y; ga[2] = g4.z; ga[3] = g4.w;
    be[0] = b4.x; be[1] = b4.y; be[2] = b4.z; be[3] = b4.w;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int g = (vec * 4 + i) / cpg;
      mu[i] = mean_rstd[((size_t)b * groups + g) * 2];
      rs[i] = mean_rstd[((size_t)b * groups + g) * 2 + 1];
    }
  }
  const size_t base = ((size_t)b * hw) * c + vec * 4;
  int cnt = 0;   // MODE 0: rows seen by this thread; a = running mean, q = running m2
  auto accumulate = [&](const float4& xv, const float4& dv) {
    const float xs[4] = {xv.x + cb[0], xv.y + cb[1], xv.z + cb[2], xv.w + cb[3]};
    if (MODE == 0) {
      const float rc = 1.f / (float)(++cnt);
#pragma unroll
      for (int i = 0; i < 4; ++i) { const float d = xs[i] - a[i]; a[i] = fmaf(d, rc, a[i]); q[i] = fmaf(d, xs[i] - a[i], q[i]); }
    } else {
      const float ds[4] = {dv.x, dv.y, dv.z, dv.w};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float xh = (xs[i] - mu[i]) * rs[i];
        float dy = ds[i];
        if (silu) {
          const float y = fmaf(xh, ga[i], be[i]);
          const float s = sigmoidf_(y);
          dy *= s * (1.f + y * (1.f - s));
        }
        const float t = dy * ga[i];
        a[i] += t; q[i] += t * xh;
      }
    }
  };
  int r = r0 + rl;
  for (; r + 3 * rowlanes < r1; r += 4 * rowlanes) {  // 4 (x2 in backward) independent 128-bit loads in flight
    float4 xv[4], dv[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      xv[u] = *reinterpret_cast<const float4*>(x + base + (size_t)(r + u * rowlanes) * c);
      if (MODE == 1) dv[u] = *reinterpret_cast<const float4*>(dz + base + (size_t)(r + u * rowlanes) * c);
    }
    if (MODE == 0) {   // the 4 rows as one batch (mean, m2), merged into the running statistics: one reciprocal
      const float w = 4.f / (float)(cnt + 4), nw = (float)cnt * w;
      cnt += 4;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        float v[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) v[u] = reinterpret_cast<const float*>(&xv[u])[i] + cb[i];
        const float bm = ((v[0] + v[1]) + (v[2] + v[3])) * 0.25f;
        float bq = 0.f;
#pragma unroll
        for (int u = 0; u < 4; ++u) bq = fmaf(v[u] - bm, v[u] - bm, bq);
        const float d = bm - a[i];
        a[i] = fmaf(d, w, a[i]);
        q[i] = fmaf(d * d, nw, q[i] + bq);
      }
    } else {
#pragma unroll
      for (int u = 0; u < 4; ++u) accumulate(xv[u], dv[u]);
    }
  }
  for (; r < r1; r += rowlanes) {
    const float4 xv = *reinterpret_cast<const float4*>(x + base + (size_t)r * c);
    float4 dv = xv;
    if (MODE == 1) dv = *reinterpret_cast<const float4*>(dz + base + (size_t)r * c);
    accumulate(xv, dv);
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    sm[((size_t)rl * c + vec * 4 + i) * 2] = a[i];
    sm[((size_t)rl * c + vec * 4 + i) * 2 + 1] = q[i];
  }
  __syncthreads();
  const int nrow = r1 - r0;
  if (MODE == 0) {   // merge each channel over its row lanes (into row lane 0's slot), all channels in parallel
    for (int ch = threadIdx.x; ch < c; ch += blockDim.x) {
      int n = 0;
      float mean = 0.f, m2 = 0.f;
      for (int l = 0; l < rowlanes && l < nrow; ++l)   // row lane l holds ceil((nrow - l) / rowlanes) rows
        stats_merge(n, mean, m2, (nrow - l + rowlanes - 1) / rowlanes, sm[((size_t)l * c + ch) * 2],
                    sm[((size_t)l * c + ch) * 2 + 1]);
      sm[(size_t)ch * 2] = mean; sm[(size_t)ch * 2 + 1] = m2;
    }
    __syncthreads();
  }
  for (int g = threadIdx.x; g < groups; g += blockDim.x) {
    float s0 = 0.f, s1 = 0.f;
    if (MODE == 0) {   // then the group's channels, nrow rows each
      int n = 0;
      for (int ch = g * cpg; ch < (g + 1) * cpg; ++ch) stats_merge(n, s0, s1, nrow, sm[(size_t)ch * 2], sm[(size_t)ch * 2 + 1]);
    } else {
      for (int l = 0; l < rowlanes; ++l)
        for (int ch = g * cpg; ch < (g + 1) * cpg; ++ch) {
          s0 += sm[((size_t)l * c + ch) * 2];
          s1 += sm[((size_t)l * c + ch) * 2 + 1];
        }
    }
    float* o = ws + (((size_t)b * chunks + chunk) * groups + g) * 2;
    o[0] = s0; o[1] = s1;
  }
}

// one warp per (b, g): fixed-order reduction of the chunk partials.
// MODE 0 -> out = (mean, rstd) (Chan merge of the chunk (mean, m2));  MODE 1 -> out = (c1, c2) = sums / n
template <int MODE>
__global__ void gn32_finalize_kernel(const float* __restrict__ ws, float* __restrict__ out, int groups, int chunks,
                                     int hw, int rows_per_chunk, int cpg, float n, float eps) {
  const int b = blockIdx.y;
  const int g = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (g >= groups) return;
  if (MODE == 0) {
    int cnt; float mean, m2;
    gn_lane_stats(ws + ((size_t)b * chunks * groups + g) * 2, groups, chunks, hw, rows_per_chunk, cpg, lane, cnt,
                    mean, m2);
    stats_warp_merge(cnt, mean, m2);
    if (lane == 0) {
      float* d = out + ((size_t)b * groups + g) * 2;
      d[0] = mean; d[1] = rsqrtf(m2 / n + eps);
    }
    return;
  }
  float s0 = 0.f, s1 = 0.f;
  for (int k = lane; k < chunks; k += 32) {
    const float* o = ws + (((size_t)b * chunks + k) * groups + g) * 2;
    s0 += o[0]; s1 += o[1];
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s0 += __shfl_xor_sync(0xffffffffu, s0, o);
    s1 += __shfl_xor_sync(0xffffffffu, s1, o);
  }
  if (lane == 0) {
    float* d = out + ((size_t)b * groups + g) * 2;
    d[0] = s0 / n; d[1] = s1 / n;
  }
}

// MODE 0: y = silu?(xhat*gamma+beta).  MODE 1: dx = rstd*(dy*gamma - c1 - xhat*c2) (+ addend, e.g. the gradient
// reaching a resnet's identity / shortcut path, so the block's input gradient needs no separate add pass)
template <int MODE>
__global__ void gn32_apply_kernel(const float* __restrict__ x, const float* __restrict__ cbias,
                                  const float* __restrict__ dz,
                                  const float* __restrict__ gamma, const float* __restrict__ beta,
                                  const float* __restrict__ mean_rstd, const float* __restrict__ c12,
                                  const float* __restrict__ addend,
                                  float* __restrict__ out, int hw, int c, int groups, int nvec, int rowlanes,
                                  int rows_per_chunk, int silu) {
  const int b = blockIdx.y, chunk = blockIdx.x;
  const int vec = threadIdx.x % nvec, rl = threadIdx.x / nvec;
  const int cpg = c / groups;
  float ga[4], be[4], mu[4], rs[4], c1[4], c2[4];
  float cb[4] = {0.f, 0.f, 0.f, 0.f};
  if (cbias) { const float4 c4 = *reinterpret_cast<const float4*>(cbias + vec * 4); cb[0] = c4.x; cb[1] = c4.y; cb[2] = c4.z; cb[3] = c4.w; }
  const float4 g4 = *reinterpret_cast<const float4*>(gamma + vec * 4);
  const float4 b4 = *reinterpret_cast<const float4*>(beta + vec * 4);
  ga[0] = g4.x; ga[1] = g4.y; ga[2] = g4.z; ga[3] = g4.w;
  be[0] = b4.x; be[1] = b4.y; be[2] = b4.z; be[3] = b4.w;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int g = (vec * 4 + i) / cpg;
    mu[i] = mean_rstd[((size_t)b * groups + g) * 2];
    rs[i] = mean_rstd[((size_t)b * groups + g) * 2 + 1];
    if (MODE == 1) { c1[i] = c12[((size_t)b * groups + g) * 2]; c2[i] = c12[((size_t)b * groups + g) * 2 + 1]; }
  }
  const int r0 = chunk * rows_per_chunk, r1 = min(hw, r0 + rows_per_chunk);
  const size_t base = ((size_t)b * hw) * c + vec * 4;
  auto apply = [&](const float4& xv, const float4& dv) -> float4 {
    const float xs[4] = {xv.x + cb[0], xv.y + cb[1], xv.z + cb[2], xv.w + cb[3]};
    float o[4];
    if (MODE == 0) {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float y = fmaf((xs[i] - mu[i]) * rs[i], ga[i], be[i]);
        o[i] = silu ? y * sigmoidf_(y) : y;
      }
    } else {
      const float ds[4] = {dv.x, dv.y, dv.z, dv.w};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float xh = (xs[i] - mu[i]) * rs[i];
        float dy = ds[i];
        if (silu) {
          const float y = fmaf(xh, ga[i], be[i]);
          const float s = sigmoidf_(y);
          dy *= s * (1.f + y * (1.f - s));
        }
        o[i] = rs[i] * (dy * ga[i] - c1[i] - xh * c2[i]);
      }
    }
    return make_float4(o[0], o[1], o[2], o[3]);
  };
  auto store = [&](int row, float4 v) {
    const size_t off = base + (size_t)row * c;
    if (MODE == 1 && addend) {
      const float4 a = *reinterpret_cast<const float4*>(addend + off);
      v.x += a.x; v.y += a.y; v.z += a.z; v.w += a.w;
    }
    *reinterpret_cast<float4*>(out + off) = v;
  };
  int r = r0 + rl;
  for (; r + 3 * rowlanes < r1; r += 4 * rowlanes) {
    float4 xv[4], dv[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      xv[u] = *reinterpret_cast<const float4*>(x + base + (size_t)(r + u * rowlanes) * c);
      if (MODE == 1) dv[u] = *reinterpret_cast<const float4*>(dz + base + (size_t)(r + u * rowlanes) * c);
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) store(r + u * rowlanes, apply(xv[u], dv[u]));
  }
  for (; r < r1; r += rowlanes) {
    const float4 xv = *reinterpret_cast<const float4*>(x + base + (size_t)r * c);
    float4 dv = xv;
    if (MODE == 1) dv = *reinterpret_cast<const float4*>(dz + base + (size_t)r * c);
    store(r, apply(xv, dv));
  }
}

static int gn32_check(const void* a, const void* b_, const void* c_, const void* d, int batch, int hw, int c, int groups) {
  if (!a || !b_ || !c_ || !d) return RTTI_ERR_ARG;
  if (batch < 1 || hw < 1 || groups < 1) return RTTI_ERR_ARG;
  // c/4 threads per row lane, so up to c/4 threads per CTA: at most 512, as gn32_partial_kernel<1> and
  // gn32_apply_kernel<0/1> use 70-82 registers (ptxas, sm_90a) and 1024 x 72+ exceeds the 64K registers of a CTA
  if (c % 4 != 0 || c % groups != 0 || c / 4 > 512) return RTTI_ERR_SHAPE;
  if (((uintptr_t)a | (uintptr_t)b_ | (uintptr_t)c_ | (uintptr_t)d) & 15) return RTTI_ERR_ALIGN;
  return RTTI_OK;
}

// ---- stripe-parallel variant (multi-GPU colour guidance, see stripe_exchange.cu) -----------------------------
struct PeerSums {
  float* sums[PEER_MAX_WORLD];          // per rank: float [2 parities][3 * groups], peer-mapped
  unsigned int* flags[PEER_MAX_WORLD];  // per rank: [0] sequence word, [1] error word, [8] sequence base (local rank only)
  int world, rank;
  unsigned int seq;
};

// One CTA, one warp per group, batch 1: reduce this rank's chunk partials, publish them, wait for every peer, merge
// the slots in RANK ORDER (bit-identical statistics on all ranks). Slot of group g: MODE 0 (count as int bits, mean,
// m2), merged with stats_merge; MODE 1 (sum, sum, -), added.
// MODE 0 -> out = (mean, rstd);  MODE 1 -> out = (c1, c2) = sums / n_total
template <int MODE>
__global__ void __launch_bounds__(1024) gn32_finalize_peer_kernel(const float* __restrict__ ws, float* __restrict__ out,
                                                                  const PeerSums pp, int groups, int chunks, int hw,
                                                                  int rows_per_chunk, int cpg, float n_total,
                                                                  float eps) {
  const int g = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // effective sequence number = argument + the sequence base word next to this rank's flags (stripe_exchange.cu)
  const unsigned int seq = pp.seq + *reinterpret_cast<const volatile unsigned int*>(pp.flags[pp.rank] + 8);
  const int par = (int)(seq & 1u);
  if (g < groups) {
    float* mine = pp.sums[pp.rank] + (size_t)par * 3 * groups + 3 * g;
    if (MODE == 0) {
      int cnt; float mean, m2;
      gn_lane_stats(ws + (size_t)g * 2, groups, chunks, hw, rows_per_chunk, cpg, lane, cnt, mean, m2);
      stats_warp_merge(cnt, mean, m2);
      if (lane == 0) { mine[0] = __int_as_float(cnt); mine[1] = mean; mine[2] = m2; }
    } else {
      float s0 = 0.f, s1 = 0.f;
      for (int k = lane; k < chunks; k += 32) {
        const float* o = ws + ((size_t)k * groups + g) * 2;
        s0 += o[0]; s1 += o[1];
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        s0 += __shfl_xor_sync(0xffffffffu, s0, o);
        s1 += __shfl_xor_sync(0xffffffffu, s1, o);
      }
      if (lane == 0) { mine[0] = s0; mine[1] = s1; }
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence_system();
    st_release_sys(pp.flags[pp.rank], seq);
  }
  if (threadIdx.x < pp.world && threadIdx.x != pp.rank) {
    if (!wait_seq(pp.flags[threadIdx.x], seq)) pp.flags[pp.rank][1] = 0xDEADu;
  }
  __syncthreads();
  if (g < groups && lane == 0) {
    float* d = out + (size_t)g * 2;
    if (MODE == 0) {
      int cnt = 0; float mean = 0.f, m2 = 0.f;
      for (int r = 0; r < pp.world; ++r) {
        const float* p = pp.sums[r] + (size_t)par * 3 * groups + 3 * g;
        stats_merge(cnt, mean, m2, __float_as_int(ld_volatile_f32(p)), ld_volatile_f32(p + 1), ld_volatile_f32(p + 2));
      }
      d[0] = mean; d[1] = rsqrtf(m2 / n_total + eps);
    } else {
      float t0 = 0.f, t1 = 0.f;
      for (int r = 0; r < pp.world; ++r) {
        const float* p = pp.sums[r] + (size_t)par * 3 * groups + 3 * g;
        t0 += ld_volatile_f32(p);
        t1 += ld_volatile_f32(p + 1);
      }
      d[0] = t0 / n_total; d[1] = t1 / n_total;
    }
  }
}

static int fill_peer_sums(PeerSums& pp, void* const* peer_sums, void* const* peer_flags, int world, int rank,
                          unsigned int seq) {
  if (!peer_sums || !peer_flags) return RTTI_ERR_ARG;
  if (world < 1 || world > PEER_MAX_WORLD || rank < 0 || rank >= world) return RTTI_ERR_ARG;
  for (int r = 0; r < world; ++r) {
    if (!peer_sums[r] || !peer_flags[r]) return RTTI_ERR_ARG;
    if (((uintptr_t)peer_sums[r] | (uintptr_t)peer_flags[r]) & 3) return RTTI_ERR_ALIGN;
    pp.sums[r] = (float*)peer_sums[r];
    pp.flags[r] = (unsigned int*)peer_flags[r];
  }
  pp.world = world; pp.rank = rank; pp.seq = seq;
  return RTTI_OK;
}

}  // namespace rtti

using namespace rtti;

extern "C" long long rtti_gn32_workspace_elems(int batch, int hw, int c, int groups) {
  if (batch < 1 || hw < 1 || c < 4 || groups < 1) return 0;
  const GN32Plan p = gn32_plan(batch, hw, c);
  return (long long)batch * p.chunks * groups * 2 + (long long)batch * groups * 2;
}

extern "C" int rtti_gn32_silu_fwd(const float* x, const float* chan_bias, const float* gamma, const float* beta, float* y, float* mean_rstd,
                                  float* workspace, int batch, int hw, int c, int groups, float eps, int apply_silu,
                                  void* stream) {
  int rc = gn32_check(x, gamma, beta, y, batch, hw, c, groups);
  if (rc != RTTI_OK) return rc;
  if (!mean_rstd || !workspace) return RTTI_ERR_ARG;
  const GN32Plan p = gn32_plan(batch, hw, c);
  const size_t smem = (size_t)p.rowlanes * c * 2 * sizeof(float);
  if (smem > 48 * 1024) return RTTI_ERR_SHAPE;
  cudaStream_t st = (cudaStream_t)stream;
  dim3 grid(p.chunks, batch);
  gn32_partial_kernel<0><<<grid, p.threads, smem, st>>>(x, chan_bias, nullptr, gamma, beta, nullptr, workspace, hw, c, groups,
                                                        p.nvec, p.rowlanes, p.rows_per_chunk, p.chunks, 0);
  gn32_finalize_kernel<0><<<dim3((groups + 7) / 8, batch), 256, 0, st>>>(workspace, mean_rstd, groups, p.chunks, hw,
                                                                         p.rows_per_chunk, c / groups,
                                                                         (float)hw * (float)(c / groups), eps);
  gn32_apply_kernel<0><<<grid, p.threads, 0, st>>>(x, chan_bias, nullptr, gamma, beta, mean_rstd, nullptr, nullptr, y, hw, c,
                                                   groups, p.nvec, p.rowlanes, p.rows_per_chunk, apply_silu);
  return cudaGetLastError() == cudaSuccess ? RTTI_OK : RTTI_ERR_CUDA;
}

extern "C" int rtti_gn32_silu_bwd(const float* x, const float* chan_bias, const float* dz, const float* gamma, const float* beta,
                                  const float* mean_rstd, const float* addend, float* dx, float* workspace, int batch,
                                  int hw, int c, int groups, int apply_silu, void* stream) {
  int rc = gn32_check(x, gamma, beta, dx, batch, hw, c, groups);
  if (rc != RTTI_OK) return rc;
  if (!dz || !mean_rstd || !workspace || ((uintptr_t)dz & 15)) return RTTI_ERR_ARG;
  if ((uintptr_t)addend & 15) return RTTI_ERR_ALIGN;
  const GN32Plan p = gn32_plan(batch, hw, c);
  const size_t smem = (size_t)p.rowlanes * c * 2 * sizeof(float);
  if (smem > 48 * 1024) return RTTI_ERR_SHAPE;
  cudaStream_t st = (cudaStream_t)stream;
  dim3 grid(p.chunks, batch);
  float* c12 = workspace + (size_t)batch * p.chunks * groups * 2;
  gn32_partial_kernel<1><<<grid, p.threads, smem, st>>>(x, chan_bias, dz, gamma, beta, mean_rstd, workspace, hw, c, groups, p.nvec,
                                                        p.rowlanes, p.rows_per_chunk, p.chunks, apply_silu);
  gn32_finalize_kernel<1><<<dim3((groups + 7) / 8, batch), 256, 0, st>>>(workspace, c12, groups, p.chunks, hw,
                                                                         p.rows_per_chunk, c / groups,
                                                                         (float)hw * (float)(c / groups), 0.f);
  gn32_apply_kernel<1><<<grid, p.threads, 0, st>>>(x, chan_bias, dz, gamma, beta, mean_rstd, c12, addend, dx, hw, c, groups,
                                                   p.nvec, p.rowlanes, p.rows_per_chunk, apply_silu);
  return cudaGetLastError() == cudaSuccess ? RTTI_OK : RTTI_ERR_CUDA;
}


extern "C" int rtti_gn32_silu_fwd_striped(const float* x, const float* chan_bias, const float* gamma, const float* beta,
                                          float* y, float* mean_rstd, float* workspace, int hw_local, long long hw_total,
                                          int c, int groups, float eps, int apply_silu, void* const* peer_sums,
                                          void* const* peer_flags, int world, int rank, unsigned int seq, void* stream) {
  int rc = gn32_check(x, gamma, beta, y, 1, hw_local, c, groups);
  if (rc != RTTI_OK) return rc;
  if (!mean_rstd || !workspace || hw_total < hw_local) return RTTI_ERR_ARG;
  if (groups > 32) return RTTI_ERR_SHAPE;
  PeerSums pp{};
  rc = fill_peer_sums(pp, peer_sums, peer_flags, world, rank, seq);
  if (rc != RTTI_OK) return rc;
  const GN32Plan p = gn32_plan(1, hw_local, c);
  const size_t smem = (size_t)p.rowlanes * c * 2 * sizeof(float);
  if (smem > 48 * 1024) return RTTI_ERR_SHAPE;
  cudaStream_t st = (cudaStream_t)stream;
  dim3 grid(p.chunks, 1);
  gn32_partial_kernel<0><<<grid, p.threads, smem, st>>>(x, chan_bias, nullptr, gamma, beta, nullptr, workspace, hw_local, c,
                                                        groups, p.nvec, p.rowlanes, p.rows_per_chunk, p.chunks, 0);
  gn32_finalize_peer_kernel<0><<<1, 32 * groups, 0, st>>>(workspace, mean_rstd, pp, groups, p.chunks, hw_local,
                                                          p.rows_per_chunk, c / groups,
                                                          (float)hw_total * (float)(c / groups), eps);
  gn32_apply_kernel<0><<<grid, p.threads, 0, st>>>(x, chan_bias, nullptr, gamma, beta, mean_rstd, nullptr, nullptr, y, hw_local,
                                                   c, groups, p.nvec, p.rowlanes, p.rows_per_chunk, apply_silu);
  return cudaGetLastError() == cudaSuccess ? RTTI_OK : RTTI_ERR_CUDA;
}

extern "C" int rtti_gn32_silu_bwd_striped(const float* x, const float* chan_bias, const float* dz, const float* gamma,
                                          const float* beta, const float* mean_rstd, float* dx, float* workspace,
                                          int hw_local, long long hw_total, int c, int groups, int apply_silu,
                                          void* const* peer_sums, void* const* peer_flags, int world, int rank,
                                          unsigned int seq, void* stream) {
  int rc = gn32_check(x, gamma, beta, dx, 1, hw_local, c, groups);
  if (rc != RTTI_OK) return rc;
  if (!dz || !mean_rstd || !workspace || ((uintptr_t)dz & 15) || hw_total < hw_local) return RTTI_ERR_ARG;
  if (groups > 32) return RTTI_ERR_SHAPE;
  PeerSums pp{};
  rc = fill_peer_sums(pp, peer_sums, peer_flags, world, rank, seq);
  if (rc != RTTI_OK) return rc;
  const GN32Plan p = gn32_plan(1, hw_local, c);
  const size_t smem = (size_t)p.rowlanes * c * 2 * sizeof(float);
  if (smem > 48 * 1024) return RTTI_ERR_SHAPE;
  cudaStream_t st = (cudaStream_t)stream;
  dim3 grid(p.chunks, 1);
  float* c12 = workspace + (size_t)p.chunks * groups * 2;
  gn32_partial_kernel<1><<<grid, p.threads, smem, st>>>(x, chan_bias, dz, gamma, beta, mean_rstd, workspace, hw_local, c,
                                                        groups, p.nvec, p.rowlanes, p.rows_per_chunk, p.chunks, apply_silu);
  gn32_finalize_peer_kernel<1><<<1, 32 * groups, 0, st>>>(workspace, c12, pp, groups, p.chunks, hw_local,
                                                          p.rows_per_chunk, c / groups,
                                                          (float)hw_total * (float)(c / groups), 0.f);
  gn32_apply_kernel<1><<<grid, p.threads, 0, st>>>(x, chan_bias, dz, gamma, beta, mean_rstd, c12, nullptr, dx, hw_local, c,
                                                   groups, p.nvec, p.rowlanes, p.rows_per_chunk, apply_silu);
  return cudaGetLastError() == cudaSuccess ? RTTI_OK : RTTI_ERR_CUDA;
}

// out[r, c] = a[r, c] + b[r, c] + bias[c]   (residual add fused with the bias of the convolution that produced b)
__global__ void add_bias_f32_kernel(const float* __restrict__ a, const float* __restrict__ b,
                                    const float* __restrict__ bias, float* __restrict__ out, long long nvec, int cvec) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (long long)gridDim.x * blockDim.x) {
    const float4 x = reinterpret_cast<const float4*>(a)[i];
    const float4 y = reinterpret_cast<const float4*>(b)[i];
    float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
    if (bias) z = reinterpret_cast<const float4*>(bias)[i % cvec];
    reinterpret_cast<float4*>(out)[i] = make_float4(x.x + y.x + z.x, x.y + y.y + z.y, x.z + y.z + z.z, x.w + y.w + z.w);
  }
}

extern "C" int rtti_add_bias_f32(const float* a, const float* b, const float* bias, float* out, long long rows, int c,
                                 void* stream) {
  if (!a || !b || !out || rows < 1 || c < 4) return RTTI_ERR_ARG;
  if (c % 4 != 0) return RTTI_ERR_SHAPE;
  if (((uintptr_t)a | (uintptr_t)b | (uintptr_t)out | (uintptr_t)bias) & 15) return RTTI_ERR_ALIGN;
  const long long nvec = rows * (c / 4);
  long long blocks = (nvec + 255) / 256;
  if (blocks > 132 * 16) blocks = 132 * 16;
  add_bias_f32_kernel<<<(int)blocks, 256, 0, (cudaStream_t)stream>>>(a, b, bias, out, nvec, c / 4);
  return cudaGetLastError() == cudaSuccess ? RTTI_OK : RTTI_ERR_CUDA;
}

// ---- nearest x2 upsample + 3x3 convolution, evaluated at low resolution --------------------------------------------
// High-res output pixel (2i+a, 2j+b) of conv3x3(upsample2x(x)) is a 2x2 convolution of the low-res x with a folded
// filter per phase (a, b). One 2x2, pad-1 convolution with the four folded filters stacked along Cout yields
// y4 [B, h+1, w+1, 4c], where phase k = 2a+b of pixel (i, j) sits at low-res position (i+a, j+b), channels k*c.
// These two kernels move between that layout and the high-res tensor [B, 2h, 2w, c].

// out[b, 2i+a, 2j+bb, ch] = y4[b, i+a, j+bb, (2a+bb)*c + ch] + bias[ch]
__global__ void upsample_phase_interleave_kernel(const float* __restrict__ y4, const float* __restrict__ bias,
                                                 float* __restrict__ out, long long nvec, int h, int w, int cvec) {
  const int H = 2 * h, W = 2 * w;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (long long)gridDim.x * blockDim.x) {
    const int cv = (int)(i % cvec);
    long long pix = i / cvec;
    const int x = (int)(pix % W); pix /= W;
    const int y = (int)(pix % H);
    const long long b = pix / H;
    const int a = y & 1, bb = x & 1;
    const long long src = ((b * (h + 1) + (y >> 1) + a) * (w + 1) + (x >> 1) + bb) * (4LL * cvec) + (2 * a + bb) * cvec + cv;
    float4 v = reinterpret_cast<const float4*>(y4)[src];
    if (bias) {
      const float4 z = reinterpret_cast<const float4*>(bias)[cv];
      v.x += z.x; v.y += z.y; v.z += z.z; v.w += z.w;
    }
    reinterpret_cast<float4*>(out)[i] = v;
  }
}

// adjoint of the interleave: dy4[b, p, q, (2a+bb)*c + ch] = g[b, 2(p-a)+a, 2(q-bb)+bb, ch], 0 where (p-a, q-bb) falls
// outside the low-res image (those positions of y4 are never read by the interleave)
__global__ void upsample_phase_scatter_kernel(const float* __restrict__ g, float* __restrict__ dy4, long long nvec, int h,
                                              int w, int cvec) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (long long)gridDim.x * blockDim.x) {
    const int cv = (int)(i % (4 * cvec));
    long long pix = i / (4 * cvec);
    const int q = (int)(pix % (w + 1)); pix /= (w + 1);
    const int p = (int)(pix % (h + 1));
    const long long b = pix / (h + 1);
    const int k = cv / cvec, a = k >> 1, bb = k & 1;
    const int li = p - a, lj = q - bb;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (li >= 0 && li < h && lj >= 0 && lj < w)
      v = reinterpret_cast<const float4*>(g)[((b * 2 * h + 2 * li + a) * (2LL * w) + 2 * lj + bb) * cvec + cv % cvec];
    reinterpret_cast<float4*>(dy4)[i] = v;
  }
}

static int upsample_phase_check(const void* a, const void* b, int batch, int h, int w, int c) {
  if (!a || !b || batch < 1 || h < 1 || w < 1 || c < 4) return RTTI_ERR_ARG;
  if (c % 4 != 0) return RTTI_ERR_SHAPE;
  if (((uintptr_t)a | (uintptr_t)b) & 15) return RTTI_ERR_ALIGN;
  return RTTI_OK;
}

static int elementwise_blocks(long long nvec) {
  const long long blocks = (nvec + 255) / 256;
  return (int)(blocks < 132 * 16 ? blocks : 132 * 16);
}

extern "C" int rtti_upsample_phase_interleave(const float* y4, const float* bias, float* out, int batch, int h, int w, int c,
                                              void* stream) {
  int rc = upsample_phase_check(y4, out, batch, h, w, c);
  if (rc != RTTI_OK) return rc;
  if ((uintptr_t)bias & 15) return RTTI_ERR_ALIGN;
  const long long nvec = (long long)batch * 4 * h * w * (c / 4);
  upsample_phase_interleave_kernel<<<elementwise_blocks(nvec), 256, 0, (cudaStream_t)stream>>>(y4, bias, out, nvec, h, w, c / 4);
  return cudaGetLastError() == cudaSuccess ? RTTI_OK : RTTI_ERR_CUDA;
}

extern "C" int rtti_upsample_phase_scatter(const float* g, float* dy4, int batch, int h, int w, int c, void* stream) {
  int rc = upsample_phase_check(g, dy4, batch, h, w, c);
  if (rc != RTTI_OK) return rc;
  const long long nvec = (long long)batch * (h + 1) * (w + 1) * c;
  upsample_phase_scatter_kernel<<<elementwise_blocks(nvec), 256, 0, (cudaStream_t)stream>>>(g, dy4, nvec, h, w, c / 4);
  return cudaGetLastError() == cudaSuccess ? RTTI_OK : RTTI_ERR_CUDA;
}
