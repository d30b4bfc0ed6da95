// Feed-forward input projection with the GEGLU gate fused into the GEMM epilogue (sm_90a: wgmma + TMA + mbarrier).
//
// Reference: models/attention.py:283-304 (GEGLU.forward): `hidden_states, gate = proj(x).chunk(2, dim=-1);
// return hidden_states * gelu(gate)` — a [M, C] x [C, 8C] GEMM whose [M, 8C] result is written, read back, gated and
// written again as [M, 4C]. Here the value and the gate columns of one output tile are accumulated side by side in
// registers (per k step two wgmma M64 N128 K16 per warpgroup: B tile rows 0-127 = value weights, rows 128-255 = the
// matching gate weights) and the epilogue computes y = (v + b_v) * gelu(g + b_g) straight from the accumulators: the
// [M, 8C] intermediate never exists.
//
//   y[M, N] = (x[M, K] W[0:N, :]^T + bias[0:N]) * gelu(x[M, K] W[N:2N, :]^T + bias[N:2N]),   exact (erf) GELU
//
// CTA = one 128 x 128 output tile, two warpgroups of 64 rows. A 4-stage ring of {A 128 x 64, value 128 x 64, gate
// 128 x 64} tiles (SWIZZLE_128B) is filled by TMA from thread 0, which refills a stage after the barrier that ends the
// k block that read it.
#include "ptx.cuh"
#include "rtti_internal.h"

namespace rtti {
namespace gg {
constexpr int BM = 128, BN = 128, BK = 64;
constexpr int STAGES = 4;
constexpr int A_TILE = BM * BK * 2;        // 16 KB
constexpr int B_TILE = 2 * BN * BK * 2;    // 32 KB: value rows then gate rows
constexpr int STAGE = A_TILE + B_TILE;
constexpr int OFF_BAR = STAGES * STAGE;
constexpr int SMEM_BYTES = OFF_BAR + 64 + 1024;
constexpr int THREADS = 256;
}  // namespace gg

struct GegluParams {
  const __half* bias;   // [2N] or nullptr
  __half* y;            // [M, N]
  int M, N, K;
  int n_blocks, k_blocks;
};

__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.f + erff(x * 0.70710678118654752f)); }

__global__ void __launch_bounds__(gg::THREADS, 1)
ff_geglu_kernel(const __grid_constant__ CUtensorMap tm_a, const __grid_constant__ CUtensorMap tm_b,
                const __grid_constant__ GegluParams p) {
  using namespace gg;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + OFF_BAR);   // [STAGES]

  const int tid = threadIdx.x, wg = tid >> 7, w = (tid >> 5) & 3, lane = tid & 31;
  const int m0 = (blockIdx.x / p.n_blocks) * BM, n0 = (blockIdx.x % p.n_blocks) * BN;

  auto load = [&](int kb) {   // thread 0
    const int s = kb % STAGES;
    uint8_t* st = smem + s * STAGE;
    mbar_expect_tx(&full[s], STAGE);
    tma_load_2d(st, &tm_a, &full[s], kb * BK, m0);
    tma_load_2d(st + A_TILE, &tm_b, &full[s], kb * BK, n0);
    tma_load_2d(st + A_TILE + B_TILE / 2, &tm_b, &full[s], kb * BK, p.N + n0);
  };
  if (tid == 0) {
    tma_prefetch_desc(&tm_a); tma_prefetch_desc(&tm_b);
    for (int i = 0; i < STAGES; ++i) mbar_init(&full[i], 1);
    mbar_fence_init();
    for (int kb = 0; kb < STAGES && kb < p.k_blocks; ++kb) load(kb);
  }
  __syncthreads();

  const uint32_t sbase = smem_u32(smem);
  float v[64], g[64];
  for (int kb = 0; kb < p.k_blocks; ++kb) {
    const int s = kb % STAGES;
    const uint32_t aa = sbase + s * STAGE + wg * 64 * 128;
    const uint32_t ba = sbase + s * STAGE + A_TILE;
    mbar_wait(&full[s], (kb / STAGES) & 1);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < BK / 16; ++kk) {
      const uint64_t da = wgmma_desc_sw128(aa + kk * 32, 16, 1024);
      const uint32_t acc = (kb > 0 || kk > 0) ? 1u : 0u;
      wgmma_ss<128>(v, da, wgmma_desc_sw128(ba + kk * 32, 16, 1024), acc);
      wgmma_ss<128>(g, da, wgmma_desc_sw128(ba + B_TILE / 2 + kk * 32, 16, 1024), acc);
    }
    wgmma_commit();
    wgmma_wait_all<64>(v);
    pin_regs<64>(g);
    __syncthreads();   // both warpgroups are done with stage s
    if (tid == 0 && kb + STAGES < p.k_blocks) load(kb + STAGES);
  }

  // ---- epilogue: bias, erf-GELU, product, fp16, straight from the accumulators
  const int r0 = m0 + 64 * wg + 16 * w + (lane >> 2), r1 = r0 + 8;
  const int cq = 2 * (lane & 3);
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    const int col = n0 + 8 * i + cq;
    float2 bv = make_float2(0.f, 0.f), bg = make_float2(0.f, 0.f);
    if (p.bias != nullptr) {
      bv = __half22float2(*reinterpret_cast<const __half2*>(p.bias + col));
      bg = __half22float2(*reinterpret_cast<const __half2*>(p.bias + p.N + col));
    }
    if (r0 < p.M)
      *reinterpret_cast<__half2*>(p.y + static_cast<size_t>(r0) * p.N + col) =
          __floats2half2_rn((v[4 * i] + bv.x) * gelu_erf(g[4 * i] + bg.x), (v[4 * i + 1] + bv.y) * gelu_erf(g[4 * i + 1] + bg.y));
    if (r1 < p.M)
      *reinterpret_cast<__half2*>(p.y + static_cast<size_t>(r1) * p.N + col) =
          __floats2half2_rn((v[4 * i + 2] + bv.x) * gelu_erf(g[4 * i + 2] + bg.x), (v[4 * i + 3] + bv.y) * gelu_erf(g[4 * i + 3] + bg.y));
  }
}

static int make_2d_map(CUtensorMap* m, const void* ptr, long long rows, long long cols, long long row_stride_elems,
                       int box_rows) {
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)row_stride_elems * 2};
  cuuint32_t box[2] = {64, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  return encode_tiled_f16(m, ptr, 2, dims, strides, box, estr);
}

}  // namespace rtti

using namespace rtti;

extern "C" int rtti_ff_geglu_fwd(const void* x, const void* w, const void* bias, void* y, long long m, int n, int k,
                                 void* stream) {
  if (!x || !w || !y) return RTTI_ERR_ARG;
  if (m < 1 || n < 1 || k < 1) return RTTI_ERR_ARG;
  if (n % gg::BN != 0 || k % gg::BK != 0) return RTTI_ERR_SHAPE;
  if (((uintptr_t)x | (uintptr_t)w | (uintptr_t)y | (uintptr_t)bias) & 15) return RTTI_ERR_ALIGN;
  int rc = rtti_arch_ok();
  if (rc != RTTI_OK) return rc;
  CUtensorMap ta, tb;
  if ((rc = make_2d_map(&ta, x, m, k, k, gg::BM)) != RTTI_OK) return rc;
  if ((rc = make_2d_map(&tb, w, 2LL * n, k, k, gg::BN)) != RTTI_OK) return rc;
  static const bool configured =
      cudaFuncSetAttribute(ff_geglu_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, gg::SMEM_BYTES) == cudaSuccess;
  if (!configured) return RTTI_ERR_CUDA;
  GegluParams p{};
  p.bias = (const __half*)bias; p.y = (__half*)y; p.M = (int)m; p.N = n; p.K = k;
  p.n_blocks = n / gg::BN; p.k_blocks = k / gg::BK;
  const long long tiles = ((m + gg::BM - 1) / gg::BM) * p.n_blocks;
  if (tiles > 0x7fffffffLL) return RTTI_ERR_SHAPE;
  ff_geglu_kernel<<<(unsigned)tiles, gg::THREADS, gg::SMEM_BYTES, (cudaStream_t)stream>>>(ta, tb, p);
  return cudaGetLastError() == cudaSuccess ? RTTI_OK : RTTI_ERR_CUDA;
}
