// Fused all-gather + region blend + CFG + Euler update over NVLink peer memory (multi-GPU region parallelism).
//
// After the sharded UNet passes of a step every rank owns the noise predictions of its passes
// ("slots", [n] fp16 each) in a symmetric buffer that all peers have mapped. Instead of
// ncclAllGather followed by a blend kernel, ONE kernel per rank
//   1. publishes "my slots of step s are written" (release store of s to its flag word),
//   2. waits (acquire loads over NVLink) until every owner it reads from has published step s,
//   3. PULLS each slot straight from its owner's memory with 128-bit peer loads while computing
//      the masked region sums + classifier-free guidance + Euler update of
//      models/region_diffusion_sdxl.py:810-845 — replicated on every rank, bit-identical results,
//      so no broadcast of the latents is needed.
// A peer that never publishes makes the wait give up after ~4 s and raise the error word flags[1] (checked by the host).
// Slot buffers are double-buffered by step parity, which makes re-use safe without a trailing barrier:
// a rank overwrites parity p at step s+2 only after its step s+1 kernel saw every peer publish s+1,
// and a peer publishes s+1 only after its step-s kernel (the last reader of parity p) has finished.
#include <cuda_fp16.h>

#include "rtti_internal.h"

namespace rtti {

constexpr int GB_MAX_WORLD = 16;
constexpr int GB_MAX_SLOTS = 24;

struct GatherBlendParams {
  const __half* peer_slots[GB_MAX_WORLD];  // per rank: fp16 [2][n_slots][n]
  unsigned int* peer_flags[GB_MAX_WORLD];  // per rank: one uint32 step counter
  int slot_owner[GB_MAX_SLOTS];
  int world, rank, n_slots, n_regions;
  long long n;
  float guidance, dt_sigma;
  unsigned int step_id;
  const float* masks;        // [n_regions, n]
  __half* eps_out;           // [n]
  const __half* latents;     // [n] or null
  __half* latents_out;
  const __half* latents_ref; // [n] or null: needs slots n_regions+1 (C) and n_regions+2 (D)
  __half* latents_ref_out;
};

struct alignas(16) H8 { __half2 v[4]; };

__device__ __forceinline__ H8 ld_peer(const __half* p) {
  // volatile: never served from a stale L1 line (peer memory bypasses L2, B300_MICROARCH.md NVLink section)
  uint4 r;
  asm volatile("ld.volatile.global.v4.u32 {%0, %1, %2, %3}, [%4];\n" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  return *reinterpret_cast<H8*>(&r);
}
__device__ __forceinline__ void up8(const H8& h, float* f) {
#pragma unroll
  for (int i = 0; i < 4; ++i) { const float2 t = __half22float2(h.v[i]); f[2 * i] = t.x; f[2 * i + 1] = t.y; }
}
__device__ __forceinline__ H8 pk8(const float* f) {
  H8 h;
#pragma unroll
  for (int i = 0; i < 4; ++i) h.v[i] = __floats2half2_rn(f[2 * i], f[2 * i + 1]);
  return h;
}

// the multistep form: the parameters of the Euler form (dt_sigma unused) + the step of each trajectory
struct GatherBlendMsParams : GatherBlendParams {
  MsStep ms, ms_ref;
};

// the ancestral form: the parameters of the Euler form + the noise of each trajectory
struct GatherBlendAncParams : GatherBlendParams {
  float s_up;
  const __half* z;
  const __half* z_ref;
};

// the UniPC form: the parameters of the Euler form (dt_sigma unused) + the step of each trajectory
struct GatherBlendUniPCParams : GatherBlendParams {
  UniPCStep up, up_ref;
};

// the Heun form: the parameters of the Euler form (dt_sigma unused) + the step of each trajectory, and where the
// reference trajectory's fp16 prediction goes (null: not written)
struct GatherBlendHeunParams : GatherBlendParams {
  HeunStep hs, hs_ref;
  __half* eps_ref_out;
};

// the LMS form: the parameters of the Euler form (dt_sigma unused) + the step of each trajectory, and where the
// reference trajectory's fp16 prediction goes (null: not written)
struct GatherBlendLmsParams : GatherBlendParams {
  LmsStep ls, ls_ref;
  __half* eps_ref_out;
};

// the DPM-Solver++(2S) form: the parameters of the Euler form (dt_sigma unused) + the step of each trajectory
struct GatherBlendSsParams : GatherBlendParams {
  SsStep ss, ss_ref;
};

// step policies (rtti_internal.h): the Euler update, or the multistep / ancestral / UniPC / Heun / LMS /
// DPM-Solver++(2S) update of the main / reference trajectory
__device__ __forceinline__ void gb_step(const GatherBlendParams& p, bool, long long, const float* e16, float* x) {
#pragma unroll
  for (int i = 0; i < 8; ++i) x[i] = fmaf(e16[i], p.dt_sigma, x[i]);
}
__device__ __forceinline__ void gb_step(const GatherBlendMsParams& p, bool ref, long long v, const float* e16, float* x) {
  ms_step8(ref ? p.ms_ref : p.ms, v, e16, x);
}
__device__ __forceinline__ void gb_step(const GatherBlendAncParams& p, bool ref, long long v, const float* e16, float* x) {
  anc_step8(AncStep{p.dt_sigma, p.s_up, ref ? p.z_ref : p.z}, v, e16, x);
}
__device__ __forceinline__ void gb_step(const GatherBlendUniPCParams& p, bool ref, long long v, const float* e16,
                                        float* x) {
  unipc_step8(ref ? p.up_ref : p.up, v, e16, x);
}
__device__ __forceinline__ void gb_step(const GatherBlendHeunParams& p, bool ref, long long v, const float* e16, float* x) {
  heun_step8(ref ? p.hs_ref : p.hs, v, e16, x);
}
__device__ __forceinline__ void gb_step(const GatherBlendLmsParams& p, bool ref, long long v, const float* e16, float* x) {
  lms_step8(ref ? p.ls_ref : p.ls, v, e16, x);
}
__device__ __forceinline__ void gb_step(const GatherBlendSsParams& p, bool ref, long long v, const float* e16, float* x) {
  ss_step8(ref ? p.ss_ref : p.ss, v, e16, x);
}

// the reference trajectory's fp16 prediction: only the Heun form (the ds of its first stage) and the LMS form (the
// newest entry of its history) store it
__device__ __forceinline__ void gb_ref_eps(const GatherBlendParams&, long long, const H8&) {}
__device__ __forceinline__ void gb_ref_eps(const GatherBlendHeunParams& p, long long v8, const H8& h) {
  if (p.eps_ref_out != nullptr) *reinterpret_cast<H8*>(p.eps_ref_out + v8 * 8) = h;
}
__device__ __forceinline__ void gb_ref_eps(const GatherBlendLmsParams& p, long long v8, const H8& h) {
  if (p.eps_ref_out != nullptr) *reinterpret_cast<H8*>(p.eps_ref_out + v8 * 8) = h;
}

// steps 1 and 2: publish this rank's step, wait for every peer it reads from. A macro rather than a function: written
// out in the kernel it compiles to the same code as before the multistep form existed (an inlined call does not).
#define GB_PUBLISH_AND_WAIT(p) \
  if (blockIdx.x == 0 && threadIdx.x == 0) {                                                                            \
    __threadfence_system();                                                                                             \
    asm volatile("st.release.sys.global.u32 [%0], %1;\n" ::"l"(p.peer_flags[p.rank]), "r"(p.step_id) : "memory");       \
  }                                                                                                                     \
  if (threadIdx.x < p.world && threadIdx.x != p.rank) {                                                                 \
    unsigned int v;                                                                                                     \
    long long spins = 0;                                                                                                \
    do {                                                                                                                \
      asm volatile("ld.acquire.sys.global.u32 %0, [%1];\n" : "=r"(v) : "l"(p.peer_flags[threadIdx.x]) : "memory");      \
      if ((int)(v - p.step_id) < 0) {                                                                                   \
        __nanosleep(500);                                                                                               \
        if (++spins > 8000000LL) { /* ~4 s: a peer never published (crashed / diverged): flag it, do not hang */ \
          p.peer_flags[p.rank][1] = 0xDEADu;                                                                            \
          break;                                                                                                        \
        }                                                                                                               \
      }                                                                                                                 \
    } while ((int)(v - p.step_id) < 0);                                                                                 \
  }                                                                                                                     \
  __syncthreads();

// step 3: pull the slots, blend, CFG, step
template <class P>
__device__ __forceinline__ void gather_blend_body(const P& p) {
  const long long v8 = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (v8 * 8 >= p.n) return;
  const size_t par = (size_t)(p.step_id & 1u) * p.n_slots * p.n;
  auto slot = [&](int s) { return p.peer_slots[p.slot_owner[s]] + par + (size_t)s * p.n + v8 * 8; };
  float eu[8], msum[8], et[8];
  up8(ld_peer(slot(0)), eu);
#pragma unroll
  for (int i = 0; i < 8; ++i) { msum[i] = 0.f; et[i] = 0.f; }
  for (int r = 0; r < p.n_regions; ++r) {
    float e[8];
    up8(ld_peer(slot(1 + r)), e);
    const float4 m0 = *reinterpret_cast<const float4*>(p.masks + (size_t)r * p.n + v8 * 8);
    const float4 m1 = *reinterpret_cast<const float4*>(p.masks + (size_t)r * p.n + v8 * 8 + 4);
    const float m[8] = {m0.x, m0.y, m0.z, m0.w, m1.x, m1.y, m1.z, m1.w};
#pragma unroll
    for (int i = 0; i < 8; ++i) { msum[i] += m[i]; et[i] = fmaf(e[i], m[i], et[i]); }
  }
  float o[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) { const float u = eu[i] * msum[i]; o[i] = u + p.guidance * (et[i] - u); }
  const H8 oh = pk8(o);
  *reinterpret_cast<H8*>(p.eps_out + v8 * 8) = oh;
  if (p.latents != nullptr) {
    float x[8], e16[8];
    up8(*reinterpret_cast<const H8*>(p.latents + v8 * 8), x);
    up8(oh, e16);
    gb_step(p, false, v8, e16, x);
    *reinterpret_cast<H8*>(p.latents_out + v8 * 8) = pk8(x);
  }
  if (p.latents_ref != nullptr) {
    float c[8], d[8], x[8], e16[8];
    up8(ld_peer(slot(p.n_regions + 1)), c);
    up8(ld_peer(slot(p.n_regions + 2)), d);
#pragma unroll
    for (int i = 0; i < 8; ++i) c[i] = c[i] + p.guidance * (d[i] - c[i]);
    const H8 ch = pk8(c);
    gb_ref_eps(p, v8, ch);
    up8(ch, e16);
    up8(*reinterpret_cast<const H8*>(p.latents_ref + v8 * 8), x);
    gb_step(p, true, v8, e16, x);
    *reinterpret_cast<H8*>(p.latents_ref_out + v8 * 8) = pk8(x);
  }
}

__global__ void __launch_bounds__(128) gather_blend_kernel(const GatherBlendParams p) {
  GB_PUBLISH_AND_WAIT(p);
  gather_blend_body(p);
}
__global__ void __launch_bounds__(128) gather_blend_ms_kernel(const GatherBlendMsParams p) {
  GB_PUBLISH_AND_WAIT(p);
  gather_blend_body(p);
}
__global__ void __launch_bounds__(128) gather_blend_anc_kernel(const GatherBlendAncParams p) {
  GB_PUBLISH_AND_WAIT(p);
  gather_blend_body(p);
}
__global__ void __launch_bounds__(128) gather_blend_unipc_kernel(const GatherBlendUniPCParams p) {
  GB_PUBLISH_AND_WAIT(p);
  gather_blend_body(p);
}
__global__ void __launch_bounds__(128) gather_blend_heun_kernel(const GatherBlendHeunParams p) {
  GB_PUBLISH_AND_WAIT(p);
  gather_blend_body(p);
}
__global__ void __launch_bounds__(128) gather_blend_lms_kernel(const GatherBlendLmsParams p) {
  GB_PUBLISH_AND_WAIT(p);
  gather_blend_body(p);
}
__global__ void __launch_bounds__(128) gather_blend_ss_kernel(const GatherBlendSsParams p) {
  GB_PUBLISH_AND_WAIT(p);
  gather_blend_body(p);
}

}  // namespace rtti

using namespace rtti;

// argument checks shared by the Euler and multistep entry points; fills everything but the step
static int gather_blend_args(const void* const* peer_slots, void* const* peer_flags, int world, int rank,
                             const int* slot_owner, int n_slots, int n_regions, const float* masks, long long n,
                             float guidance, void* eps_out, const void* latents, void* latents_out,
                             const void* latents_ref, void* latents_ref_out, unsigned int step_id, GatherBlendParams& p) {
  if (!peer_slots || !peer_flags || !slot_owner || !masks || !eps_out) return RTTI_ERR_ARG;
  if (world < 1 || world > GB_MAX_WORLD || rank < 0 || rank >= world) return RTTI_ERR_ARG;
  if (n_regions < 1 || n_slots < n_regions + 1 || n_slots > GB_MAX_SLOTS || n < 8) return RTTI_ERR_ARG;
  if (n % 8 != 0) return RTTI_ERR_SHAPE;
  if ((latents == nullptr) != (latents_out == nullptr)) return RTTI_ERR_ARG;
  if ((latents_ref == nullptr) != (latents_ref_out == nullptr)) return RTTI_ERR_ARG;
  if (latents_ref != nullptr && n_slots < n_regions + 3) return RTTI_ERR_ARG;
  for (int r = 0; r < world; ++r) {
    if (!peer_slots[r] || !peer_flags[r]) return RTTI_ERR_ARG;
    if ((uintptr_t)peer_slots[r] & 15) return RTTI_ERR_ALIGN;
    p.peer_slots[r] = (const __half*)peer_slots[r];
    p.peer_flags[r] = (unsigned int*)peer_flags[r];
  }
  for (int s = 0; s < n_slots; ++s) {
    if (slot_owner[s] < 0 || slot_owner[s] >= world) return RTTI_ERR_ARG;
    p.slot_owner[s] = slot_owner[s];
  }
  p.world = world; p.rank = rank; p.n_slots = n_slots; p.n_regions = n_regions; p.n = n;
  p.guidance = guidance; p.step_id = step_id;
  p.masks = masks; p.eps_out = (__half*)eps_out;
  p.latents = (const __half*)latents; p.latents_out = (__half*)latents_out;
  p.latents_ref = (const __half*)latents_ref; p.latents_ref_out = (__half*)latents_ref_out;
  return RTTI_OK;
}

extern "C" int rtti_gather_blend_step(const void* const* peer_slots, void* const* peer_flags, int world, int rank,
                                      const int* slot_owner, int n_slots, int n_regions, const float* masks,
                                      long long n, float guidance, void* eps_out, const void* latents,
                                      void* latents_out, const void* latents_ref, void* latents_ref_out,
                                      float dt_sigma, unsigned int step_id, void* stream) {
  GatherBlendParams p{};
  const int rc = gather_blend_args(peer_slots, peer_flags, world, rank, slot_owner, n_slots, n_regions, masks, n, guidance,
                                   eps_out, latents, latents_out, latents_ref, latents_ref_out, step_id, p);
  if (rc != RTTI_OK) return rc;
  p.dt_sigma = dt_sigma;
  const long long nv = n / 8;
  gather_blend_kernel<<<(int)((nv + 127) / 128), 128, 0, (cudaStream_t)stream>>>(p);
  return cudaGetLastError() == cudaSuccess ? RTTI_OK : RTTI_ERR_CUDA;
}

extern "C" int rtti_gather_blend_step_ms(const void* const* peer_slots, void* const* peer_flags, int world, int rank,
                                         const int* slot_owner, int n_slots, int n_regions, const float* masks,
                                         long long n, float guidance, void* eps_out, const void* latents,
                                         void* latents_out, const void* latents_ref, void* latents_ref_out, float hx,
                                         float he, float cx, float cd, float cp, const float* d_prev, float* d_out,
                                         const float* d_prev_ref, float* d_out_ref, unsigned int step_id,
                                         void* stream) {
  if (!latents || !latents_out) return RTTI_ERR_ARG;
  GatherBlendMsParams p{};
  int rc = gather_blend_args(peer_slots, peer_flags, world, rank, slot_owner, n_slots, n_regions, masks, n, guidance,
                             eps_out, latents, latents_out, latents_ref, latents_ref_out, step_id, p);
  if (rc == RTTI_OK) rc = ms_step_args(cp, d_prev, d_out);
  if (rc == RTTI_OK && latents_ref != nullptr) rc = ms_step_args(cp, d_prev_ref, d_out_ref);
  if (rc == RTTI_OK && (((uintptr_t)masks | (uintptr_t)eps_out | (uintptr_t)latents | (uintptr_t)latents_out |
                         (uintptr_t)latents_ref | (uintptr_t)latents_ref_out) & 15))
    rc = RTTI_ERR_ALIGN;
  if (rc != RTTI_OK) return rc;
  p.ms = MsStep{hx, he, cx, cd, cp, d_prev, d_out};
  p.ms_ref = MsStep{hx, he, cx, cd, cp, d_prev_ref, d_out_ref};
  const long long nv = n / 8;
  gather_blend_ms_kernel<<<(int)((nv + 127) / 128), 128, 0, (cudaStream_t)stream>>>(p);
  return cudaGetLastError() == cudaSuccess ? RTTI_OK : RTTI_ERR_CUDA;
}

extern "C" int rtti_gather_blend_step_anc(const void* const* peer_slots, void* const* peer_flags, int world, int rank,
                                          const int* slot_owner, int n_slots, int n_regions, const float* masks,
                                          long long n, float guidance, void* eps_out, const void* latents,
                                          void* latents_out, const void* latents_ref, void* latents_ref_out,
                                          float dt_sigma, float s_up, const void* z, const void* z_ref,
                                          unsigned int step_id, void* stream) {
  if (!latents || !latents_out) return RTTI_ERR_ARG;
  GatherBlendAncParams p{};
  int rc = gather_blend_args(peer_slots, peer_flags, world, rank, slot_owner, n_slots, n_regions, masks, n, guidance,
                             eps_out, latents, latents_out, latents_ref, latents_ref_out, step_id, p);
  if (rc == RTTI_OK) rc = anc_step_args(s_up, z);
  if (rc == RTTI_OK && latents_ref != nullptr) rc = anc_step_args(s_up, z_ref);
  if (rc == RTTI_OK && (((uintptr_t)masks | (uintptr_t)eps_out | (uintptr_t)latents | (uintptr_t)latents_out |
                         (uintptr_t)latents_ref | (uintptr_t)latents_ref_out) & 15))
    rc = RTTI_ERR_ALIGN;
  if (rc != RTTI_OK) return rc;
  p.dt_sigma = dt_sigma;
  p.s_up = s_up; p.z = (const __half*)z; p.z_ref = (const __half*)z_ref;
  const long long nv = n / 8;
  gather_blend_anc_kernel<<<(int)((nv + 127) / 128), 128, 0, (cudaStream_t)stream>>>(p);
  return cudaGetLastError() == cudaSuccess ? RTTI_OK : RTTI_ERR_CUDA;
}

extern "C" int rtti_gather_blend_step_unipc(const void* const* peer_slots, void* const* peer_flags, int world, int rank,
                                            const int* slot_owner, int n_slots, int n_regions, const float* masks,
                                            long long n, float guidance, void* eps_out, const void* latents,
                                            void* latents_out, const void* latents_ref, void* latents_ref_out,
                                            float hx, float he, float ux, float ul, float u0, float u1, float u2,
                                            float vx, float v0, float v1, const float* xl, const float* m1,
                                            const float* m2, float* m_out, float* xl_out, const float* xl_ref,
                                            const float* m1_ref, const float* m2_ref, float* m_out_ref,
                                            float* xl_out_ref, unsigned int step_id, void* stream) {
  if (!latents || !latents_out) return RTTI_ERR_ARG;
  GatherBlendUniPCParams p{};
  int rc = gather_blend_args(peer_slots, peer_flags, world, rank, slot_owner, n_slots, n_regions, masks, n, guidance,
                             eps_out, latents, latents_out, latents_ref, latents_ref_out, step_id, p);
  if (rc == RTTI_OK) rc = unipc_step_args(ul, u1, u2, v1, xl, m1, m2, m_out, xl_out);
  if (rc == RTTI_OK && latents_ref != nullptr)
    rc = unipc_step_args(ul, u1, u2, v1, xl_ref, m1_ref, m2_ref, m_out_ref, xl_out_ref);
  if (rc == RTTI_OK && (((uintptr_t)masks | (uintptr_t)eps_out | (uintptr_t)latents | (uintptr_t)latents_out |
                         (uintptr_t)latents_ref | (uintptr_t)latents_ref_out) & 15))
    rc = RTTI_ERR_ALIGN;
  if (rc != RTTI_OK) return rc;
  p.up = UniPCStep{hx, he, ux, ul, u0, u1, u2, vx, v0, v1, xl, m1, m2, m_out, xl_out};
  p.up_ref = UniPCStep{hx, he, ux, ul, u0, u1, u2, vx, v0, v1, xl_ref, m1_ref, m2_ref, m_out_ref, xl_out_ref};
  const long long nv = n / 8;
  gather_blend_unipc_kernel<<<(int)((nv + 127) / 128), 128, 0, (cudaStream_t)stream>>>(p);
  return cudaGetLastError() == cudaSuccess ? RTTI_OK : RTTI_ERR_CUDA;
}

extern "C" int rtti_gather_blend_step_heun(const void* const* peer_slots, void* const* peer_flags, int world, int rank,
                                           const int* slot_owner, int n_slots, int n_regions, const float* masks,
                                           long long n, float guidance, void* eps_out, const void* latents,
                                           void* latents_out, const void* latents_ref, void* latents_ref_out, float cx,
                                           float ce, float cs, float cd, const void* xs, const void* ds,
                                           const void* xs_ref, const void* ds_ref, void* eps_ref_out,
                                           unsigned int step_id, void* stream) {
  if (!latents || !latents_out) return RTTI_ERR_ARG;
  if (eps_ref_out != nullptr && latents_ref == nullptr) return RTTI_ERR_ARG;
  GatherBlendHeunParams p{};
  int rc = gather_blend_args(peer_slots, peer_flags, world, rank, slot_owner, n_slots, n_regions, masks, n, guidance,
                             eps_out, latents, latents_out, latents_ref, latents_ref_out, step_id, p);
  if (rc == RTTI_OK) rc = heun_step_args(cs, cd, xs, ds);
  if (rc == RTTI_OK && latents_ref != nullptr) rc = heun_step_args(cs, cd, xs_ref, ds_ref);
  if (rc == RTTI_OK && (((uintptr_t)masks | (uintptr_t)eps_out | (uintptr_t)latents | (uintptr_t)latents_out |
                         (uintptr_t)latents_ref | (uintptr_t)latents_ref_out | (uintptr_t)eps_ref_out) & 15))
    rc = RTTI_ERR_ALIGN;
  if (rc != RTTI_OK) return rc;
  p.hs = HeunStep{cx, ce, cs, cd, (const __half*)xs, (const __half*)ds};
  p.hs_ref = HeunStep{cx, ce, cs, cd, (const __half*)xs_ref, (const __half*)ds_ref};
  p.eps_ref_out = (__half*)eps_ref_out;
  const long long nv = n / 8;
  gather_blend_heun_kernel<<<(int)((nv + 127) / 128), 128, 0, (cudaStream_t)stream>>>(p);
  return cudaGetLastError() == cudaSuccess ? RTTI_OK : RTTI_ERR_CUDA;
}

extern "C" int rtti_gather_blend_step_lms(const void* const* peer_slots, void* const* peer_flags, int world, int rank,
                                          const int* slot_owner, int n_slots, int n_regions, const float* masks,
                                          long long n, float guidance, void* eps_out, const void* latents,
                                          void* latents_out, const void* latents_ref, void* latents_ref_out, float c0,
                                          float c1, float c2, float c3, const void* d1, const void* d2, const void* d3,
                                          const void* d1_ref, const void* d2_ref, const void* d3_ref,
                                          void* eps_ref_out, unsigned int step_id, void* stream) {
  if (!latents || !latents_out) return RTTI_ERR_ARG;
  if (eps_ref_out != nullptr && latents_ref == nullptr) return RTTI_ERR_ARG;
  GatherBlendLmsParams p{};
  int rc = gather_blend_args(peer_slots, peer_flags, world, rank, slot_owner, n_slots, n_regions, masks, n, guidance,
                             eps_out, latents, latents_out, latents_ref, latents_ref_out, step_id, p);
  if (rc == RTTI_OK) rc = lms_step_args(c1, c2, c3, d1, d2, d3);
  if (rc == RTTI_OK && latents_ref != nullptr) rc = lms_step_args(c1, c2, c3, d1_ref, d2_ref, d3_ref);
  if (rc == RTTI_OK && (((uintptr_t)masks | (uintptr_t)eps_out | (uintptr_t)latents | (uintptr_t)latents_out |
                         (uintptr_t)latents_ref | (uintptr_t)latents_ref_out | (uintptr_t)eps_ref_out) & 15))
    rc = RTTI_ERR_ALIGN;
  if (rc != RTTI_OK) return rc;
  p.ls = LmsStep{c0, c1, c2, c3, (const __half*)d1, (const __half*)d2, (const __half*)d3};
  p.ls_ref = LmsStep{c0, c1, c2, c3, (const __half*)d1_ref, (const __half*)d2_ref, (const __half*)d3_ref};
  p.eps_ref_out = (__half*)eps_ref_out;
  const long long nv = n / 8;
  gather_blend_lms_kernel<<<(int)((nv + 127) / 128), 128, 0, (cudaStream_t)stream>>>(p);
  return cudaGetLastError() == cudaSuccess ? RTTI_OK : RTTI_ERR_CUDA;
}

extern "C" int rtti_gather_blend_step_ss(const void* const* peer_slots, void* const* peer_flags, int world, int rank,
                                         const int* slot_owner, int n_slots, int n_regions, const float* masks,
                                         long long n, float guidance, void* eps_out, const void* latents,
                                         void* latents_out, const void* latents_ref, void* latents_ref_out, float hx,
                                         float he, float cx, float cs, float cd, float cp, const float* d_prev,
                                         float* d_out, const void* xs, const float* d_prev_ref, float* d_out_ref,
                                         const void* xs_ref, unsigned int step_id, void* stream) {
  if (!latents || !latents_out) return RTTI_ERR_ARG;
  GatherBlendSsParams p{};
  int rc = gather_blend_args(peer_slots, peer_flags, world, rank, slot_owner, n_slots, n_regions, masks, n, guidance,
                             eps_out, latents, latents_out, latents_ref, latents_ref_out, step_id, p);
  if (rc == RTTI_OK) rc = ss_step_args(cs, cp, xs, d_prev, d_out);
  if (rc == RTTI_OK && latents_ref != nullptr) rc = ss_step_args(cs, cp, xs_ref, d_prev_ref, d_out_ref);
  if (rc == RTTI_OK && (((uintptr_t)masks | (uintptr_t)eps_out | (uintptr_t)latents | (uintptr_t)latents_out |
                         (uintptr_t)latents_ref | (uintptr_t)latents_ref_out) & 15))
    rc = RTTI_ERR_ALIGN;
  if (rc != RTTI_OK) return rc;
  p.ss = SsStep{MsStep{hx, he, cx, cd, cp, d_prev, d_out}, cs, (const __half*)xs};
  p.ss_ref = SsStep{MsStep{hx, he, cx, cd, cp, d_prev_ref, d_out_ref}, cs, (const __half*)xs_ref};
  const long long nv = n / 8;
  gather_blend_ss_kernel<<<(int)((nv + 127) / 128), 128, 0, (cudaStream_t)stream>>>(p);
  return cudaGetLastError() == cudaSuccess ? RTTI_OK : RTTI_ERR_CUDA;
}
