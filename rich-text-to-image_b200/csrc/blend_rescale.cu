// Region blend + classifier-free guidance + guidance rescale (+ Euler update), one launch per image, on one GPU
// (rtti_region_blend_cfg_rescale) or fused with the NVLink all-gather of the noise predictions
// (rtti_gather_blend_step_rescale).
//
// The rescale of diffusers' rescale_noise_cfg (models/region_diffusion_sdxl.py:42-53) scales the CFG prediction by
//   f = 1 - phi + phi * std(eps_text) / std(eps_cfg)      (unbiased std over all n elements of the image)
// so no output element can be written before both standard deviations are known. One thread-block cluster of
// RS_CL CTAs covers the image:
//   1. every thread forms eps_text / eps_cfg of its 8-element vectors once (loading each slot once, over NVLink in the
//      gather form), keeps eps_cfg in fp32 in shared memory and accumulates (count, mean, m2) of both;
//   2. the statistics are merged in a fixed order: per thread in vector order, stats_warp_merge, the warps of a CTA
//      in index order, then every CTA reads the CTA partials of ranks 0..RS_CL-1 through distributed shared memory,
//      so all CTAs hold bit-identical standard deviations without a second launch, a workspace or atomics;
//   3. eps = fp16(eps_cfg * f) is written and the Euler update consumes that fp16-rounded prediction.
// The vector layout depends on n only and both entry points run the same body, so for the same inputs the gather form
// is bit-identical to the single-GPU form whatever the world size. The gather form rescales the reference-latent pair
// (passes C/D: eps_text = eps_D, eps_cfg = eps_C + g (eps_D - eps_C)) as a second, independent reduction in the same
// launch, after the main blend, re-using the shared memory.
// The publish / wait / timeout protocol and the double-buffered slots are those of gather_blend.cu.
#include <cooperative_groups.h>
#include <cuda_fp16.h>

#include <type_traits>

#include "rtti_internal.h"

namespace rtti {
namespace {

namespace cg = cooperative_groups;

constexpr int RS_CL = 8;          // CTAs per cluster: the portable maximum
constexpr int RS_THREADS = 1024;
constexpr int RS_MAX_VPT = 4;     // 8-element vectors per thread at the largest n
constexpr long long RS_MAX_N = 8LL * RS_CL * RS_THREADS * RS_MAX_VPT;  // 262144: an SDXL 2048^2 latent
constexpr int RS_SMEM = RS_MAX_VPT * RS_THREADS * 32;                  // fp32 eps_cfg of the vectors of one CTA
constexpr int RS_MAX_WORLD = 16;
constexpr int RS_MAX_SLOTS = 24;
constexpr int RS_MAX_REGIONS = 16;

struct RescaleParams {
  const __half* slot[RS_MAX_SLOTS];  // [n] each: 0 uncond, 1..n_regions regions (base last), n_regions+1 / +2 = C / D
  const float* masks;                // [n_regions, n]
  int n_regions, threads, vpt;
  long long n;
  float guidance, phi, dt_sigma;
  __half* eps_out;
  const __half* latents;
  __half* latents_out;
  const __half* latents_ref;         // gather form only; null to skip the C/D pair
  __half* latents_ref_out;
  unsigned int* peer_flags[RS_MAX_WORLD];  // gather form only
  int world, rank;
  unsigned int step_id;
};

// the multistep form: the parameters of the Euler form (dt_sigma unused) + the step of each trajectory
struct RescaleMsParams : RescaleParams {
  MsStep ms, ms_ref;
};

// the ancestral form: the parameters of the Euler form + the noise of each trajectory
struct RescaleAncParams : RescaleParams {
  float s_up;
  const __half* z;
  const __half* z_ref;
};

// the UniPC form: the parameters of the Euler form (dt_sigma unused) + the step of each trajectory
struct RescaleUniPCParams : RescaleParams {
  UniPCStep up, up_ref;
};

// the Heun form: the parameters of the Euler form (dt_sigma unused) + the step of each trajectory, and where the
// reference trajectory's rescaled fp16 prediction goes (gather form only; null: not written)
struct RescaleHeunParams : RescaleParams {
  HeunStep hs, hs_ref;
  __half* eps_ref_out;
};

// the LMS form: the parameters of the Euler form (dt_sigma unused) + the step of each trajectory, and where the
// reference trajectory's rescaled fp16 prediction goes (gather form only; null: not written)
struct RescaleLmsParams : RescaleParams {
  LmsStep ls, ls_ref;
  __half* eps_ref_out;
};

// the DPM-Solver++(2S) form: the parameters of the Euler form (dt_sigma unused) + the step of each trajectory
struct RescaleSsParams : RescaleParams {
  SsStep ss, ss_ref;
};

// step policies (rtti_internal.h): the Euler update, or the multistep / ancestral / UniPC / Heun / LMS /
// DPM-Solver++(2S) update of the main (REF false) / reference (REF true) trajectory
template <bool REF>
__device__ __forceinline__ void rs_step(const RescaleParams& p, long long, const float* e16, float* x) {
#pragma unroll
  for (int i = 0; i < 8; ++i) x[i] = fmaf(e16[i], p.dt_sigma, x[i]);
}
template <bool REF>
__device__ __forceinline__ void rs_step(const RescaleMsParams& p, long long v, const float* e16, float* x) {
  ms_step8(REF ? p.ms_ref : p.ms, v, e16, x);
}
template <bool REF>
__device__ __forceinline__ void rs_step(const RescaleAncParams& p, long long v, const float* e16, float* x) {
  anc_step8(AncStep{p.dt_sigma, p.s_up, REF ? p.z_ref : p.z}, v, e16, x);
}
template <bool REF>
__device__ __forceinline__ void rs_step(const RescaleUniPCParams& p, long long v, const float* e16, float* x) {
  unipc_step8(REF ? p.up_ref : p.up, v, e16, x);
}
template <bool REF>
__device__ __forceinline__ void rs_step(const RescaleHeunParams& p, long long v, const float* e16, float* x) {
  heun_step8(REF ? p.hs_ref : p.hs, v, e16, x);
}
template <bool REF>
__device__ __forceinline__ void rs_step(const RescaleLmsParams& p, long long v, const float* e16, float* x) {
  lms_step8(REF ? p.ls_ref : p.ls, v, e16, x);
}
template <bool REF>
__device__ __forceinline__ void rs_step(const RescaleSsParams& p, long long v, const float* e16, float* x) {
  ss_step8(REF ? p.ss_ref : p.ss, v, e16, x);
}

// the output of the reference trajectory's prediction: only the Heun form (the ds of its first stage) and the LMS form
// (the newest entry of its history) store it
__device__ __forceinline__ __half* rs_ref_eps(const RescaleParams&) { return nullptr; }
__device__ __forceinline__ __half* rs_ref_eps(const RescaleHeunParams& p) { return p.eps_ref_out; }
__device__ __forceinline__ __half* rs_ref_eps(const RescaleLmsParams& p) { return p.eps_ref_out; }

// (count, mean, m2) of eps_text and of eps_cfg over the same elements
struct PairStats { int n; float mt, qt, mc, qc; };

__device__ __forceinline__ void pair_merge(PairStats& a, const PairStats& b) {
  int nt = a.n;
  stats_merge(nt, a.mt, a.qt, b.n, b.mt, b.qt);
  stats_merge(a.n, a.mc, a.qc, b.n, b.mc, b.qc);
}

__device__ __forceinline__ void unpack8(const uint4& u, float* f) {
  const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) { const float2 t = __half22float2(h[i]); f[2 * i] = t.x; f[2 * i + 1] = t.y; }
}
__device__ __forceinline__ uint4 pack8(const float* f) {
  uint4 u;
  __half2* h = reinterpret_cast<__half2*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) h[i] = __floats2half2_rn(f[2 * i], f[2 * i + 1]);
  return u;
}
// 128-bit loads: plain for local slots; volatile for peer slots (never served from a stale L1 line)
template <bool PEER>
__device__ __forceinline__ void load8(const __half* p, float* f) {
  uint4 r;
  if constexpr (PEER) {
    asm volatile("ld.volatile.global.v4.u32 {%0, %1, %2, %3}, [%4];\n" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  } else {
    r = *reinterpret_cast<const uint4*>(p);
  }
  unpack8(r, f);
}

// eps_text = sum_r m_r eps_r and eps_cfg = u + g (eps_text - u), u = eps_uncond * sum_r m_r, for vector v: the
// arithmetic of region_blend_kernel. ONES: every mask is 1 (the C/D pair, as the single-GPU path blends it).
template <bool PEER, bool ONES, class P>
__device__ __forceinline__ void blend_vec(const P& p, int s0, int n_reg, long long v, float* et, float* ec) {
  float msum[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) { msum[i] = 0.f; et[i] = 0.f; }
  for (int r = 0; r < n_reg; ++r) {
    float e[8];
    load8<PEER>(p.slot[s0 + 1 + r] + v * 8, e);
    float m[8];
    if constexpr (ONES) {
#pragma unroll
      for (int i = 0; i < 8; ++i) m[i] = 1.f;
    } else {
      const float4 m0 = *reinterpret_cast<const float4*>(p.masks + (size_t)r * p.n + v * 8);
      const float4 m1 = *reinterpret_cast<const float4*>(p.masks + (size_t)r * p.n + v * 8 + 4);
      m[0] = m0.x; m[1] = m0.y; m[2] = m0.z; m[3] = m0.w; m[4] = m1.x; m[5] = m1.y; m[6] = m1.z; m[7] = m1.w;
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) { msum[i] += m[i]; et[i] = fmaf(e[i], m[i], et[i]); }
  }
  float eu[8];  // loaded last: not live across the region loop (the kernel runs at 64 registers per thread)
  load8<PEER>(p.slot[s0] + v * 8, eu);
#pragma unroll
  for (int i = 0; i < 8; ++i) { const float u = eu[i] * msum[i]; ec[i] = u + p.guidance * (et[i] - u); }
}

__device__ __forceinline__ void vec_stats(const float* x, float& mean, float& m2) {
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) s += x[i];
  mean = s * 0.125f;
  m2 = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) { const float d = x[i] - mean; m2 = fmaf(d, d, m2); }
}

struct RescaleSmem {
  PairStats warp[RS_THREADS / 32];
  PairStats cta;
  float factor;
};

// One reduction + apply over the whole image: slots s0 (uncond) and s0+1..s0+n_reg, outputs eps_out (may be null) and
// lat_out = lat stepped with eps (when lat is non-null; the reference trajectory's step when ONES). Vector
// v = (k * RS_CL + cta rank) * threads + thread, k < vpt.
template <bool PEER, bool ONES, class P>
__device__ void rescale_job(const P& p, int s0, int n_reg, __half* eps_out, const __half* lat,
                            __half* lat_out, float4* cfg_s, RescaleSmem& sm) {
  cg::cluster_group cluster = cg::this_cluster();
  const int tid = threadIdx.x, T = p.threads, crank = (int)cluster.block_rank();
  const long long nv = p.n / 8;
  PairStats acc{0, 0.f, 0.f, 0.f, 0.f};
  for (int k = 0; k < p.vpt; ++k) {
    const long long v = ((long long)k * RS_CL + crank) * T + tid;
    if (v < nv) {
      float et[8], ec[8];
      blend_vec<PEER, ONES>(p, s0, n_reg, v, et, ec);
      cfg_s[(2 * k) * T + tid] = make_float4(ec[0], ec[1], ec[2], ec[3]);
      cfg_s[(2 * k + 1) * T + tid] = make_float4(ec[4], ec[5], ec[6], ec[7]);
      PairStats b;
      b.n = 8;
      vec_stats(et, b.mt, b.qt);
      vec_stats(ec, b.mc, b.qc);
      pair_merge(acc, b);
    }
  }
  {
    int nt = acc.n;
    stats_warp_merge(nt, acc.mt, acc.qt);
    stats_warp_merge(acc.n, acc.mc, acc.qc);
  }
  if ((tid & 31) == 0) sm.warp[tid >> 5] = acc;
  __syncthreads();
  if (tid == 0) {
    PairStats c = sm.warp[0];
    for (int w = 1; w < T / 32; ++w) pair_merge(c, sm.warp[w]);
    sm.cta = c;
  }
  cluster.sync();
  if (tid == 0) {
    PairStats tot = *cluster.map_shared_rank(&sm.cta, 0);
    for (int r = 1; r < RS_CL; ++r) pair_merge(tot, *cluster.map_shared_rank(&sm.cta, r));
    const float dof = (float)(tot.n - 1);  // unbiased, as torch.std
    const float sd_t = sqrtf(tot.qt / dof), sd_c = sqrtf(tot.qc / dof);
    sm.factor = fmaf(p.phi, sd_t / sd_c, 1.f - p.phi);
  }
  cluster.sync();  // also: no CTA reads a peer's partial after this point, so the next job may overwrite it
  const float f = sm.factor;
  for (int k = 0; k < p.vpt; ++k) {
    const long long v = ((long long)k * RS_CL + crank) * T + tid;
    if (v < nv) {
      const float4 c0 = cfg_s[(2 * k) * T + tid], c1 = cfg_s[(2 * k + 1) * T + tid];
      const float o[8] = {c0.x * f, c0.y * f, c0.z * f, c0.w * f, c1.x * f, c1.y * f, c1.z * f, c1.w * f};
      const uint4 oh = pack8(o);
      if (eps_out != nullptr) *reinterpret_cast<uint4*>(eps_out + v * 8) = oh;
      if (lat != nullptr) {
        float x[8], e16[8];
        unpack8(*reinterpret_cast<const uint4*>(lat + v * 8), x);
        unpack8(oh, e16);  // the scheduler consumes the fp16-rounded noise prediction
        rs_step<ONES>(p, v, e16, x);
        *reinterpret_cast<uint4*>(lat_out + v * 8) = pack8(x);
      }
    }
  }
}

template <bool PEER, class P>
__device__ __forceinline__ void blend_rescale_body(const P& p, float4* cfg_s, RescaleSmem& sm) {
  if constexpr (PEER) {
    // gather_blend.cu's protocol: publish this rank's step, wait (acquire, ~4 s timeout) for every peer's
    if (blockIdx.x == 0 && threadIdx.x == 0) {
      __threadfence_system();
      asm volatile("st.release.sys.global.u32 [%0], %1;\n" ::"l"(p.peer_flags[p.rank]), "r"(p.step_id) : "memory");
    }
    if (threadIdx.x < p.world && threadIdx.x != p.rank) {
      unsigned int v;
      long long spins = 0;
      do {
        asm volatile("ld.acquire.sys.global.u32 %0, [%1];\n" : "=r"(v) : "l"(p.peer_flags[threadIdx.x]) : "memory");
        if ((int)(v - p.step_id) < 0) {
          __nanosleep(500);
          if (++spins > 8000000LL) {  // ~4 s: a peer never published; raise the error word the host checks
            asm volatile("st.relaxed.sys.global.u32 [%0], %1;\n" ::"l"(p.peer_flags[p.rank] + 1), "r"(0xDEADu) : "memory");
            break;
          }
        }
      } while ((int)(v - p.step_id) < 0);
    }
    __syncthreads();
  }
  rescale_job<PEER, false>(p, 0, p.n_regions, p.eps_out, p.latents, p.latents_out, cfg_s, sm);
  if (p.latents_ref != nullptr)
    rescale_job<PEER, true>(p, p.n_regions + 1, 1, rs_ref_eps(p), p.latents_ref, p.latents_ref_out, cfg_s, sm);
}

template <bool PEER>
__global__ void __cluster_dims__(RS_CL, 1, 1) __launch_bounds__(RS_THREADS, 1)
    blend_rescale_kernel(const __grid_constant__ RescaleParams p) {
  extern __shared__ float4 cfg_s[];
  __shared__ RescaleSmem sm;
  blend_rescale_body<PEER>(p, cfg_s, sm);
}

template <bool PEER>
__global__ void __cluster_dims__(RS_CL, 1, 1) __launch_bounds__(RS_THREADS, 1)
    blend_rescale_ms_kernel(const __grid_constant__ RescaleMsParams p) {
  extern __shared__ float4 cfg_s[];
  __shared__ RescaleSmem sm;
  blend_rescale_body<PEER>(p, cfg_s, sm);
}

template <bool PEER>
__global__ void __cluster_dims__(RS_CL, 1, 1) __launch_bounds__(RS_THREADS, 1)
    blend_rescale_anc_kernel(const __grid_constant__ RescaleAncParams p) {
  extern __shared__ float4 cfg_s[];
  __shared__ RescaleSmem sm;
  blend_rescale_body<PEER>(p, cfg_s, sm);
}

template <bool PEER>
__global__ void __cluster_dims__(RS_CL, 1, 1) __launch_bounds__(RS_THREADS, 1)
    blend_rescale_unipc_kernel(const __grid_constant__ RescaleUniPCParams p) {
  extern __shared__ float4 cfg_s[];
  __shared__ RescaleSmem sm;
  blend_rescale_body<PEER>(p, cfg_s, sm);
}

template <bool PEER>
__global__ void __cluster_dims__(RS_CL, 1, 1) __launch_bounds__(RS_THREADS, 1)
    blend_rescale_heun_kernel(const __grid_constant__ RescaleHeunParams p) {
  extern __shared__ float4 cfg_s[];
  __shared__ RescaleSmem sm;
  blend_rescale_body<PEER>(p, cfg_s, sm);
}

template <bool PEER>
__global__ void __cluster_dims__(RS_CL, 1, 1) __launch_bounds__(RS_THREADS, 1)
    blend_rescale_lms_kernel(const __grid_constant__ RescaleLmsParams p) {
  extern __shared__ float4 cfg_s[];
  __shared__ RescaleSmem sm;
  blend_rescale_body<PEER>(p, cfg_s, sm);
}

template <bool PEER>
__global__ void __cluster_dims__(RS_CL, 1, 1) __launch_bounds__(RS_THREADS, 1)
    blend_rescale_ss_kernel(const __grid_constant__ RescaleSsParams p) {
  extern __shared__ float4 cfg_s[];
  __shared__ RescaleSmem sm;
  blend_rescale_body<PEER>(p, cfg_s, sm);
}

// the kernel of each parameter type
template <bool PEER>
const void* rescale_kernel(const RescaleParams&) { return (const void*)blend_rescale_kernel<PEER>; }
template <bool PEER>
const void* rescale_kernel(const RescaleMsParams&) { return (const void*)blend_rescale_ms_kernel<PEER>; }
template <bool PEER>
const void* rescale_kernel(const RescaleAncParams&) { return (const void*)blend_rescale_anc_kernel<PEER>; }
template <bool PEER>
const void* rescale_kernel(const RescaleUniPCParams&) { return (const void*)blend_rescale_unipc_kernel<PEER>; }
template <bool PEER>
const void* rescale_kernel(const RescaleHeunParams&) { return (const void*)blend_rescale_heun_kernel<PEER>; }
template <bool PEER>
const void* rescale_kernel(const RescaleLmsParams&) { return (const void*)blend_rescale_lms_kernel<PEER>; }
template <bool PEER>
const void* rescale_kernel(const RescaleSsParams&) { return (const void*)blend_rescale_ss_kernel<PEER>; }

// threads per CTA and vectors per thread: a function of n only
void rescale_plan(long long n, int& threads, int& vpt) {
  const long long nv = n / 8, per_cta = (nv + RS_CL - 1) / RS_CL;
  if (per_cta <= RS_THREADS) {
    threads = (int)((per_cta + 31) / 32 * 32);
    vpt = 1;
  } else {
    threads = RS_THREADS;
    vpt = (int)((nv + (long long)RS_CL * RS_THREADS - 1) / ((long long)RS_CL * RS_THREADS));
  }
}

template <bool PEER, class P>
int launch_rescale(P& p, void* stream) {
  static const bool configured = cudaFuncSetAttribute(rescale_kernel<PEER>(p), cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                      RS_SMEM) == cudaSuccess;
  if (!configured) return RTTI_ERR_CUDA;
  rescale_plan(p.n, p.threads, p.vpt);
  if constexpr (std::is_same<P, RescaleMsParams>::value)
    blend_rescale_ms_kernel<PEER><<<RS_CL, p.threads, (size_t)p.vpt * p.threads * 32, (cudaStream_t)stream>>>(p);
  else if constexpr (std::is_same<P, RescaleAncParams>::value)
    blend_rescale_anc_kernel<PEER><<<RS_CL, p.threads, (size_t)p.vpt * p.threads * 32, (cudaStream_t)stream>>>(p);
  else if constexpr (std::is_same<P, RescaleUniPCParams>::value)
    blend_rescale_unipc_kernel<PEER><<<RS_CL, p.threads, (size_t)p.vpt * p.threads * 32, (cudaStream_t)stream>>>(p);
  else if constexpr (std::is_same<P, RescaleHeunParams>::value)
    blend_rescale_heun_kernel<PEER><<<RS_CL, p.threads, (size_t)p.vpt * p.threads * 32, (cudaStream_t)stream>>>(p);
  else if constexpr (std::is_same<P, RescaleLmsParams>::value)
    blend_rescale_lms_kernel<PEER><<<RS_CL, p.threads, (size_t)p.vpt * p.threads * 32, (cudaStream_t)stream>>>(p);
  else if constexpr (std::is_same<P, RescaleSsParams>::value)
    blend_rescale_ss_kernel<PEER><<<RS_CL, p.threads, (size_t)p.vpt * p.threads * 32, (cudaStream_t)stream>>>(p);
  else
    blend_rescale_kernel<PEER><<<RS_CL, p.threads, (size_t)p.vpt * p.threads * 32, (cudaStream_t)stream>>>(p);
  return cudaGetLastError() == cudaSuccess ? RTTI_OK : RTTI_ERR_CUDA;
}

// argument checks of the single-GPU entry points; fills everything but the step and the rescale factor
int rescale_args(const void* eps_uncond, const void* const* eps_region, const float* masks, int n_regions, long long n,
                 float guidance, void* eps_out, const void* latents, void* latents_out, RescaleParams& p) {
  if (!eps_uncond || !eps_region || !masks || !eps_out) return RTTI_ERR_ARG;
  if (n_regions < 1 || n_regions > RS_MAX_REGIONS || n < 8) return RTTI_ERR_ARG;
  if (n % 8 != 0 || n > RS_MAX_N) return RTTI_ERR_SHAPE;
  if ((latents == nullptr) != (latents_out == nullptr)) return RTTI_ERR_ARG;
  uintptr_t al = (uintptr_t)eps_uncond | (uintptr_t)masks | (uintptr_t)eps_out | (uintptr_t)latents | (uintptr_t)latents_out;
  p.slot[0] = (const __half*)eps_uncond;
  for (int i = 0; i < n_regions; ++i) {
    if (!eps_region[i]) return RTTI_ERR_ARG;
    p.slot[1 + i] = (const __half*)eps_region[i];
    al |= (uintptr_t)eps_region[i];
  }
  if (al & 15) return RTTI_ERR_ALIGN;
  p.masks = masks; p.n_regions = n_regions; p.n = n; p.guidance = guidance;
  p.eps_out = (__half*)eps_out; p.latents = (const __half*)latents; p.latents_out = (__half*)latents_out;
  return RTTI_OK;
}

// argument checks of the gather entry points; fills everything but the step and the rescale factor
int gather_rescale_args(const void* const* peer_slots, void* const* peer_flags, int world, int rank,
                        const int* slot_owner, int n_slots, int n_regions, const float* masks, long long n,
                        float guidance, void* eps_out, const void* latents, void* latents_out, const void* latents_ref,
                        void* latents_ref_out, unsigned int step_id, RescaleParams& p) {
  if (!peer_slots || !peer_flags || !slot_owner || !masks || !eps_out) return RTTI_ERR_ARG;
  if (world < 1 || world > RS_MAX_WORLD || rank < 0 || rank >= world) return RTTI_ERR_ARG;
  if (n_regions < 1 || n_slots < n_regions + 1 || n_slots > RS_MAX_SLOTS || n < 8) return RTTI_ERR_ARG;
  if (n % 8 != 0 || n > RS_MAX_N) return RTTI_ERR_SHAPE;
  if ((latents == nullptr) != (latents_out == nullptr)) return RTTI_ERR_ARG;
  if ((latents_ref == nullptr) != (latents_ref_out == nullptr)) return RTTI_ERR_ARG;
  if (latents_ref != nullptr && n_slots < n_regions + 3) return RTTI_ERR_ARG;
  if (((uintptr_t)masks | (uintptr_t)eps_out | (uintptr_t)latents | (uintptr_t)latents_out | (uintptr_t)latents_ref |
       (uintptr_t)latents_ref_out) & 15)
    return RTTI_ERR_ALIGN;
  for (int r = 0; r < world; ++r) {
    if (!peer_slots[r] || !peer_flags[r]) return RTTI_ERR_ARG;
    if ((uintptr_t)peer_slots[r] & 15) return RTTI_ERR_ALIGN;
    p.peer_flags[r] = (unsigned int*)peer_flags[r];
  }
  const size_t par = (size_t)(step_id & 1u) * n_slots * n;  // double buffer by step parity (gather_blend.cu)
  for (int s = 0; s < n_slots; ++s) {
    if (slot_owner[s] < 0 || slot_owner[s] >= world) return RTTI_ERR_ARG;
    p.slot[s] = (const __half*)peer_slots[slot_owner[s]] + par + (size_t)s * n;
  }
  p.world = world; p.rank = rank; p.step_id = step_id;
  p.masks = masks; p.n_regions = n_regions; p.n = n; p.guidance = guidance;
  p.eps_out = (__half*)eps_out; p.latents = (const __half*)latents; p.latents_out = (__half*)latents_out;
  p.latents_ref = (const __half*)latents_ref; p.latents_ref_out = (__half*)latents_ref_out;
  return RTTI_OK;
}

}  // namespace
}  // namespace rtti

using namespace rtti;

extern "C" int rtti_region_blend_cfg_rescale(const void* eps_uncond, const void* const* eps_region, const float* masks,
                                             int n_regions, long long n, float guidance, void* eps_out,
                                             const void* latents, void* latents_out, float dt_sigma,
                                             float guidance_rescale, void* stream) {
  RescaleParams p{};
  const int rc = rescale_args(eps_uncond, eps_region, masks, n_regions, n, guidance, eps_out, latents, latents_out, p);
  if (rc != RTTI_OK) return rc;
  p.phi = guidance_rescale; p.dt_sigma = dt_sigma;
  return launch_rescale<false>(p, stream);
}

extern "C" int rtti_region_blend_cfg_rescale_ms(const void* eps_uncond, const void* const* eps_region,
                                                const float* masks, int n_regions, long long n, float guidance,
                                                void* eps_out, const void* latents, void* latents_out, float hx,
                                                float he, float cx, float cd, float cp, const float* d_prev,
                                                float* d_out, float guidance_rescale, void* stream) {
  if (!latents || !latents_out) return RTTI_ERR_ARG;
  RescaleMsParams p{};
  int rc = rescale_args(eps_uncond, eps_region, masks, n_regions, n, guidance, eps_out, latents, latents_out, p);
  if (rc == RTTI_OK) rc = ms_step_args(cp, d_prev, d_out);
  if (rc != RTTI_OK) return rc;
  p.phi = guidance_rescale;
  p.ms = MsStep{hx, he, cx, cd, cp, d_prev, d_out};
  return launch_rescale<false>(p, stream);
}

extern "C" int rtti_region_blend_cfg_rescale_anc(const void* eps_uncond, const void* const* eps_region,
                                                 const float* masks, int n_regions, long long n, float guidance,
                                                 void* eps_out, const void* latents, void* latents_out, float dt_sigma,
                                                 float s_up, const void* z, float guidance_rescale, void* stream) {
  if (!latents || !latents_out) return RTTI_ERR_ARG;
  RescaleAncParams p{};
  int rc = rescale_args(eps_uncond, eps_region, masks, n_regions, n, guidance, eps_out, latents, latents_out, p);
  if (rc == RTTI_OK) rc = anc_step_args(s_up, z);
  if (rc != RTTI_OK) return rc;
  p.phi = guidance_rescale; p.dt_sigma = dt_sigma;
  p.s_up = s_up; p.z = (const __half*)z;
  return launch_rescale<false>(p, stream);
}

extern "C" int rtti_gather_blend_step_rescale(const void* const* peer_slots, void* const* peer_flags, int world, int rank,
                                              const int* slot_owner, int n_slots, int n_regions, const float* masks,
                                              long long n, float guidance, void* eps_out, const void* latents,
                                              void* latents_out, const void* latents_ref, void* latents_ref_out,
                                              float dt_sigma, unsigned int step_id, float guidance_rescale,
                                              void* stream) {
  RescaleParams p{};
  const int rc = gather_rescale_args(peer_slots, peer_flags, world, rank, slot_owner, n_slots, n_regions, masks, n,
                                     guidance, eps_out, latents, latents_out, latents_ref, latents_ref_out, step_id, p);
  if (rc != RTTI_OK) return rc;
  p.phi = guidance_rescale; p.dt_sigma = dt_sigma;
  return launch_rescale<true>(p, stream);
}

extern "C" int rtti_gather_blend_step_rescale_ms(const void* const* peer_slots, void* const* peer_flags, int world,
                                                 int rank, const int* slot_owner, int n_slots, int n_regions,
                                                 const float* masks, long long n, float guidance, void* eps_out,
                                                 const void* latents, void* latents_out, const void* latents_ref,
                                                 void* latents_ref_out, float hx, float he, float cx, float cd,
                                                 float cp, const float* d_prev, float* d_out, const float* d_prev_ref,
                                                 float* d_out_ref, unsigned int step_id, float guidance_rescale,
                                                 void* stream) {
  if (!latents || !latents_out) return RTTI_ERR_ARG;
  RescaleMsParams p{};
  int rc = gather_rescale_args(peer_slots, peer_flags, world, rank, slot_owner, n_slots, n_regions, masks, n, guidance,
                               eps_out, latents, latents_out, latents_ref, latents_ref_out, step_id, p);
  if (rc == RTTI_OK) rc = ms_step_args(cp, d_prev, d_out);
  if (rc == RTTI_OK && latents_ref != nullptr) rc = ms_step_args(cp, d_prev_ref, d_out_ref);
  if (rc != RTTI_OK) return rc;
  p.phi = guidance_rescale;
  p.ms = MsStep{hx, he, cx, cd, cp, d_prev, d_out};
  p.ms_ref = MsStep{hx, he, cx, cd, cp, d_prev_ref, d_out_ref};
  return launch_rescale<true>(p, stream);
}

extern "C" int rtti_gather_blend_step_rescale_anc(const void* const* peer_slots, void* const* peer_flags, int world,
                                                  int rank, const int* slot_owner, int n_slots, int n_regions,
                                                  const float* masks, long long n, float guidance, void* eps_out,
                                                  const void* latents, void* latents_out, const void* latents_ref,
                                                  void* latents_ref_out, float dt_sigma, float s_up, const void* z,
                                                  const void* z_ref, unsigned int step_id, float guidance_rescale,
                                                  void* stream) {
  if (!latents || !latents_out) return RTTI_ERR_ARG;
  RescaleAncParams p{};
  int rc = gather_rescale_args(peer_slots, peer_flags, world, rank, slot_owner, n_slots, n_regions, masks, n, guidance,
                               eps_out, latents, latents_out, latents_ref, latents_ref_out, step_id, p);
  if (rc == RTTI_OK) rc = anc_step_args(s_up, z);
  if (rc == RTTI_OK && latents_ref != nullptr) rc = anc_step_args(s_up, z_ref);
  if (rc != RTTI_OK) return rc;
  p.phi = guidance_rescale; p.dt_sigma = dt_sigma;
  p.s_up = s_up; p.z = (const __half*)z; p.z_ref = (const __half*)z_ref;
  return launch_rescale<true>(p, stream);
}

extern "C" int rtti_region_blend_cfg_rescale_unipc(const void* eps_uncond, const void* const* eps_region,
                                                   const float* masks, int n_regions, long long n, float guidance,
                                                   void* eps_out, const void* latents, void* latents_out, float hx,
                                                   float he, float ux, float ul, float u0, float u1, float u2,
                                                   float vx, float v0, float v1, const float* xl, const float* m1,
                                                   const float* m2, float* m_out, float* xl_out,
                                                   float guidance_rescale, void* stream) {
  if (!latents || !latents_out) return RTTI_ERR_ARG;
  RescaleUniPCParams p{};
  int rc = rescale_args(eps_uncond, eps_region, masks, n_regions, n, guidance, eps_out, latents, latents_out, p);
  if (rc == RTTI_OK) rc = unipc_step_args(ul, u1, u2, v1, xl, m1, m2, m_out, xl_out);
  if (rc != RTTI_OK) return rc;
  p.phi = guidance_rescale;
  p.up = UniPCStep{hx, he, ux, ul, u0, u1, u2, vx, v0, v1, xl, m1, m2, m_out, xl_out};
  return launch_rescale<false>(p, stream);
}

extern "C" int rtti_gather_blend_step_rescale_unipc(const void* const* peer_slots, void* const* peer_flags, int world,
                                                    int rank, const int* slot_owner, int n_slots, int n_regions,
                                                    const float* masks, long long n, float guidance, void* eps_out,
                                                    const void* latents, void* latents_out, const void* latents_ref,
                                                    void* latents_ref_out, float hx, float he, float ux, float ul,
                                                    float u0, float u1, float u2, float vx, float v0, float v1,
                                                    const float* xl, const float* m1, const float* m2, float* m_out,
                                                    float* xl_out, const float* xl_ref, const float* m1_ref,
                                                    const float* m2_ref, float* m_out_ref, float* xl_out_ref,
                                                    unsigned int step_id, float guidance_rescale, void* stream) {
  if (!latents || !latents_out) return RTTI_ERR_ARG;
  RescaleUniPCParams p{};
  int rc = gather_rescale_args(peer_slots, peer_flags, world, rank, slot_owner, n_slots, n_regions, masks, n, guidance,
                               eps_out, latents, latents_out, latents_ref, latents_ref_out, step_id, p);
  if (rc == RTTI_OK) rc = unipc_step_args(ul, u1, u2, v1, xl, m1, m2, m_out, xl_out);
  if (rc == RTTI_OK && latents_ref != nullptr)
    rc = unipc_step_args(ul, u1, u2, v1, xl_ref, m1_ref, m2_ref, m_out_ref, xl_out_ref);
  if (rc != RTTI_OK) return rc;
  p.phi = guidance_rescale;
  p.up = UniPCStep{hx, he, ux, ul, u0, u1, u2, vx, v0, v1, xl, m1, m2, m_out, xl_out};
  p.up_ref = UniPCStep{hx, he, ux, ul, u0, u1, u2, vx, v0, v1, xl_ref, m1_ref, m2_ref, m_out_ref, xl_out_ref};
  return launch_rescale<true>(p, stream);
}

extern "C" int rtti_region_blend_cfg_rescale_heun(const void* eps_uncond, const void* const* eps_region,
                                                  const float* masks, int n_regions, long long n, float guidance,
                                                  void* eps_out, const void* latents, void* latents_out, float cx,
                                                  float ce, float cs, float cd, const void* xs, const void* ds,
                                                  float guidance_rescale, void* stream) {
  if (!latents || !latents_out) return RTTI_ERR_ARG;
  RescaleHeunParams p{};
  int rc = rescale_args(eps_uncond, eps_region, masks, n_regions, n, guidance, eps_out, latents, latents_out, p);
  if (rc == RTTI_OK) rc = heun_step_args(cs, cd, xs, ds);
  if (rc != RTTI_OK) return rc;
  p.phi = guidance_rescale;
  p.hs = HeunStep{cx, ce, cs, cd, (const __half*)xs, (const __half*)ds};
  return launch_rescale<false>(p, stream);
}

extern "C" int rtti_gather_blend_step_rescale_heun(const void* const* peer_slots, void* const* peer_flags, int world,
                                                   int rank, const int* slot_owner, int n_slots, int n_regions,
                                                   const float* masks, long long n, float guidance, void* eps_out,
                                                   const void* latents, void* latents_out, const void* latents_ref,
                                                   void* latents_ref_out, float cx, float ce, float cs, float cd,
                                                   const void* xs, const void* ds, const void* xs_ref,
                                                   const void* ds_ref, void* eps_ref_out, unsigned int step_id,
                                                   float guidance_rescale, void* stream) {
  if (!latents || !latents_out) return RTTI_ERR_ARG;
  if (eps_ref_out != nullptr && latents_ref == nullptr) return RTTI_ERR_ARG;
  RescaleHeunParams p{};
  int rc = gather_rescale_args(peer_slots, peer_flags, world, rank, slot_owner, n_slots, n_regions, masks, n, guidance,
                               eps_out, latents, latents_out, latents_ref, latents_ref_out, step_id, p);
  if (rc == RTTI_OK) rc = heun_step_args(cs, cd, xs, ds);
  if (rc == RTTI_OK && latents_ref != nullptr) rc = heun_step_args(cs, cd, xs_ref, ds_ref);
  if (rc == RTTI_OK && ((uintptr_t)eps_ref_out & 15)) rc = RTTI_ERR_ALIGN;
  if (rc != RTTI_OK) return rc;
  p.phi = guidance_rescale;
  p.hs = HeunStep{cx, ce, cs, cd, (const __half*)xs, (const __half*)ds};
  p.hs_ref = HeunStep{cx, ce, cs, cd, (const __half*)xs_ref, (const __half*)ds_ref};
  p.eps_ref_out = (__half*)eps_ref_out;
  return launch_rescale<true>(p, stream);
}

extern "C" int rtti_region_blend_cfg_rescale_lms(const void* eps_uncond, const void* const* eps_region,
                                                 const float* masks, int n_regions, long long n, float guidance,
                                                 void* eps_out, const void* latents, void* latents_out, float c0,
                                                 float c1, float c2, float c3, const void* d1, const void* d2,
                                                 const void* d3, float guidance_rescale, void* stream) {
  if (!latents || !latents_out) return RTTI_ERR_ARG;
  RescaleLmsParams p{};
  int rc = rescale_args(eps_uncond, eps_region, masks, n_regions, n, guidance, eps_out, latents, latents_out, p);
  if (rc == RTTI_OK) rc = lms_step_args(c1, c2, c3, d1, d2, d3);
  if (rc != RTTI_OK) return rc;
  p.phi = guidance_rescale;
  p.ls = LmsStep{c0, c1, c2, c3, (const __half*)d1, (const __half*)d2, (const __half*)d3};
  return launch_rescale<false>(p, stream);
}

extern "C" int rtti_gather_blend_step_rescale_lms(const void* const* peer_slots, void* const* peer_flags, int world,
                                                  int rank, const int* slot_owner, int n_slots, int n_regions,
                                                  const float* masks, long long n, float guidance, void* eps_out,
                                                  const void* latents, void* latents_out, const void* latents_ref,
                                                  void* latents_ref_out, float c0, float c1, float c2, float c3,
                                                  const void* d1, const void* d2, const void* d3, const void* d1_ref,
                                                  const void* d2_ref, const void* d3_ref, void* eps_ref_out,
                                                  unsigned int step_id, float guidance_rescale, void* stream) {
  if (!latents || !latents_out) return RTTI_ERR_ARG;
  if (eps_ref_out != nullptr && latents_ref == nullptr) return RTTI_ERR_ARG;
  RescaleLmsParams p{};
  int rc = gather_rescale_args(peer_slots, peer_flags, world, rank, slot_owner, n_slots, n_regions, masks, n, guidance,
                               eps_out, latents, latents_out, latents_ref, latents_ref_out, step_id, p);
  if (rc == RTTI_OK) rc = lms_step_args(c1, c2, c3, d1, d2, d3);
  if (rc == RTTI_OK && latents_ref != nullptr) rc = lms_step_args(c1, c2, c3, d1_ref, d2_ref, d3_ref);
  if (rc == RTTI_OK && ((uintptr_t)eps_ref_out & 15)) rc = RTTI_ERR_ALIGN;
  if (rc != RTTI_OK) return rc;
  p.phi = guidance_rescale;
  p.ls = LmsStep{c0, c1, c2, c3, (const __half*)d1, (const __half*)d2, (const __half*)d3};
  p.ls_ref = LmsStep{c0, c1, c2, c3, (const __half*)d1_ref, (const __half*)d2_ref, (const __half*)d3_ref};
  p.eps_ref_out = (__half*)eps_ref_out;
  return launch_rescale<true>(p, stream);
}

extern "C" int rtti_region_blend_cfg_rescale_ss(const void* eps_uncond, const void* const* eps_region,
                                                const float* masks, int n_regions, long long n, float guidance,
                                                void* eps_out, const void* latents, void* latents_out, float hx,
                                                float he, float cx, float cs, float cd, float cp, const float* d_prev,
                                                float* d_out, const void* xs, float guidance_rescale, void* stream) {
  if (!latents || !latents_out) return RTTI_ERR_ARG;
  RescaleSsParams p{};
  int rc = rescale_args(eps_uncond, eps_region, masks, n_regions, n, guidance, eps_out, latents, latents_out, p);
  if (rc == RTTI_OK) rc = ss_step_args(cs, cp, xs, d_prev, d_out);
  if (rc != RTTI_OK) return rc;
  p.phi = guidance_rescale;
  p.ss = SsStep{MsStep{hx, he, cx, cd, cp, d_prev, d_out}, cs, (const __half*)xs};
  return launch_rescale<false>(p, stream);
}

extern "C" int rtti_gather_blend_step_rescale_ss(const void* const* peer_slots, void* const* peer_flags, int world,
                                                 int rank, const int* slot_owner, int n_slots, int n_regions,
                                                 const float* masks, long long n, float guidance, void* eps_out,
                                                 const void* latents, void* latents_out, const void* latents_ref,
                                                 void* latents_ref_out, float hx, float he, float cx, float cs,
                                                 float cd, float cp, const float* d_prev, float* d_out, const void* xs,
                                                 const float* d_prev_ref, float* d_out_ref, const void* xs_ref,
                                                 unsigned int step_id, float guidance_rescale, void* stream) {
  if (!latents || !latents_out) return RTTI_ERR_ARG;
  RescaleSsParams p{};
  int rc = gather_rescale_args(peer_slots, peer_flags, world, rank, slot_owner, n_slots, n_regions, masks, n, guidance,
                               eps_out, latents, latents_out, latents_ref, latents_ref_out, step_id, p);
  if (rc == RTTI_OK) rc = ss_step_args(cs, cp, xs, d_prev, d_out);
  if (rc == RTTI_OK && latents_ref != nullptr) rc = ss_step_args(cs, cp, xs_ref, d_prev_ref, d_out_ref);
  if (rc != RTTI_OK) return rc;
  p.phi = guidance_rescale;
  p.ss = SsStep{MsStep{hx, he, cx, cd, cp, d_prev, d_out}, cs, (const __half*)xs};
  p.ss_ref = SsStep{MsStep{hx, he, cx, cd, cp, d_prev_ref, d_out_ref}, cs, (const __half*)xs_ref};
  return launch_rescale<true>(p, stream);
}
