// Self-attention token-map capture for sm_90a: accum[q, k] += mean_h softmax(scale Q_h K_h^T)[q, k].
//
// The reference materialises the full probability tensor of every attention call and averages it
// over heads on every call (models/attention_processor.py:1157-1159, 166-171, 1181), then the
// token-map hook copies the conditional row to the CPU and sums it there
// (models/region_diffusion_sdxl.py:986-992). Here the flash kernel (attn_fwd.cu) leaves only the
// per-row log-sum-exp; this kernel recomputes the 128x128 score tiles with wgmma,
// loops over the heads inside the CTA (so the head mean needs no atomics and is deterministic) and
// adds the tile into an fp32 accumulator that stays on the device.
//
// CTA = one (128 query rows) x (128 keys) tile, all heads; two warpgroups of 64 rows. Thread 0 keeps the
// Q and K tiles of the next head in flight in a two-stage TMA ring.
#include "ptx.cuh"
#include "rtti_internal.h"

namespace rtti {

struct ProbsMeanParams {
  int heads, head_dim, n_q, n_k;
  float scale_log2, inv_heads;
  const float* lse;  // [heads, n_q]
  float* accum;      // [n_q, n_k]
};

template <int NDCH>
struct PMCfg {
  static constexpr int TILE = 128 * 128;
  static constexpr int STAGE = 2 * NDCH * TILE;   // Q chunks, then K chunks
  static constexpr int OFF_BAR = 2 * STAGE;
  static constexpr int SMEM_BYTES = OFF_BAR + 64 + 1024;
};

template <int NDCH>
__global__ void __launch_bounds__(256, 1)
attn_probs_mean_kernel(const __grid_constant__ CUtensorMap tm_q, const __grid_constant__ CUtensorMap tm_k,
                       const __grid_constant__ ProbsMeanParams p) {
  using C = PMCfg<NDCH>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + C::OFF_BAR);   // [2]

  const int tid = threadIdx.x, wg = tid >> 7, w = (tid >> 5) & 3, lane = tid & 31;
  const int k0 = blockIdx.x * 128, q0 = blockIdx.y * 128;

  auto load = [&](int h) {   // thread 0
    const int s = h & 1;
    uint8_t* st = smem + s * C::STAGE;
    mbar_expect_tx(&full[s], C::STAGE);
#pragma unroll
    for (int c = 0; c < NDCH; ++c) {
      tma_load_4d(st + c * C::TILE, &tm_q, &full[s], 64 * c, h, q0, 0);
      tma_load_4d(st + (NDCH + c) * C::TILE, &tm_k, &full[s], 64 * c, h, k0, 0);
    }
  };
  if (tid == 0) {
    tma_prefetch_desc(&tm_q); tma_prefetch_desc(&tm_k);
    mbar_init(&full[0], 1); mbar_init(&full[1], 1);
    mbar_fence_init();
    load(0);
    if (p.heads > 1) load(1);
  }
  __syncthreads();

  const int r0 = 64 * wg + 16 * w + (lane >> 2), r1 = r0 + 8;
  const int cq = 2 * (lane & 3);
  const bool ok0 = q0 + r0 < p.n_q, ok1 = q0 + r1 < p.n_q;
  const uint32_t sbase = smem_u32(smem);
  float acc[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) acc[i] = 0.f;
  for (int h = 0; h < p.heads; ++h) {
    const int s = h & 1;
    const float nl0 = ok0 ? -p.lse[static_cast<size_t>(h) * p.n_q + q0 + r0] : 0.f;
    const float nl1 = ok1 ? -p.lse[static_cast<size_t>(h) * p.n_q + q0 + r1] : 0.f;
    const uint32_t qa = sbase + s * C::STAGE + wg * 64 * 128;
    const uint32_t ka = sbase + s * C::STAGE + NDCH * C::TILE;
    mbar_wait(&full[s], (h >> 1) & 1);
    float sc[64];
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4 * NDCH; ++kk) {
      const uint32_t off = (kk >> 2) * C::TILE + (kk & 3) * 32;
      wgmma_ss<128>(sc, wgmma_desc_sw128(qa + off, 16, 1024), wgmma_desc_sw128(ka + off, 16, 1024), kk > 0 ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait_all<64>(sc);
    __syncthreads();   // both warpgroups are done with stage s
    if (tid == 0 && h + 2 < p.heads) load(h + 2);
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      // the reference averages fp16 probabilities (attention_processor.py:405, 1181)
      const float2 a = __half22float2(__floats2half2_rn(ex2_approx(fmaf(sc[4 * i], p.scale_log2, nl0)),
                                                        ex2_approx(fmaf(sc[4 * i + 1], p.scale_log2, nl0))));
      const float2 c = __half22float2(__floats2half2_rn(ex2_approx(fmaf(sc[4 * i + 2], p.scale_log2, nl1)),
                                                        ex2_approx(fmaf(sc[4 * i + 3], p.scale_log2, nl1))));
      acc[4 * i] += a.x; acc[4 * i + 1] += a.y; acc[4 * i + 2] += c.x; acc[4 * i + 3] += c.y;
    }
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    if (!(r ? ok1 : ok0)) continue;
    float* dst = p.accum + static_cast<size_t>(q0 + (r ? r1 : r0)) * p.n_k + k0;
#pragma unroll
    for (int i = 0; i < 16; ++i)
#pragma unroll
      for (int j = 0; j < 2; ++j)
        if (k0 + 8 * i + cq + j < p.n_k) dst[8 * i + cq + j] += acc[4 * i + 2 * r + j] * p.inv_heads;
  }
}

template <int NDCH>
static int launch_pm(const CUtensorMap& tq, const CUtensorMap& tk, const ProbsMeanParams& p, dim3 grid,
                     cudaStream_t stream) {
  using C = PMCfg<NDCH>;
  auto kern = attn_probs_mean_kernel<NDCH>;
  static const bool configured =
      cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES) == cudaSuccess;
  if (!configured) return RTTI_ERR_CUDA;
  kern<<<grid, 256, C::SMEM_BYTES, stream>>>(tq, tk, p);
  return cudaGetLastError() == cudaSuccess ? RTTI_OK : RTTI_ERR_CUDA;
}

}  // namespace rtti

using namespace rtti;

extern "C" int rtti_attn_probs_mean_accum(const void* q, const void* k, const float* lse, float* accum, int heads,
                                          int head_dim, int n_q, int n_k, long long q_rs, long long k_rs,
                                          float scale, void* stream) {
  if (!q || !k || !lse || !accum) return RTTI_ERR_ARG;
  if (heads < 1 || n_q < 1 || n_k < 1) return RTTI_ERR_ARG;
  if (head_dim < 8 || head_dim > 192 || (head_dim % 8) != 0) return RTTI_ERR_SHAPE;
  if (((uintptr_t)q | (uintptr_t)k) & 15) return RTTI_ERR_ALIGN;
  if ((q_rs | k_rs) & 7) return RTTI_ERR_ALIGN;
  int rc = rtti_arch_ok();
  if (rc != RTTI_OK) return rc;
  ProbsMeanParams p{};
  p.heads = heads; p.head_dim = head_dim; p.n_q = n_q; p.n_k = n_k;
  p.scale_log2 = scale * 1.4426950408889634f;
  p.inv_heads = 1.f / (float)heads;
  p.lse = lse; p.accum = accum;
  CUtensorMap tq, tk;
  if ((rc = make_head_map(&tq, q, head_dim, heads, n_q, 1, (long long)n_q * q_rs, q_rs, 128)) != RTTI_OK) return rc;
  if ((rc = make_head_map(&tk, k, head_dim, heads, n_k, 1, (long long)n_k * k_rs, k_rs, 128)) != RTTI_OK) return rc;
  dim3 grid((n_k + 127) / 128, (n_q + 127) / 128, 1);
  const int ndch = (head_dim + 63) / 64;
  cudaStream_t st = (cudaStream_t)stream;
  if (ndch == 1) return launch_pm<1>(tq, tk, p, grid, st);
  if (ndch == 2) return launch_pm<2>(tq, tk, p, grid, st);
  return launch_pm<3>(tq, tk, p, grid, st);
}
