// Stripe-parallel colour guidance over NVLink peer memory (multi-GPU, SURVEY §8e).
//
// The VAE decoder that colour guidance differentiates through (models/region_diffusion_sdxl.py:849-867) has batch 1,
// so the only way to use more than one GPU for it is spatial: every rank owns a horizontal stripe of rows of every
// activation of the up-blocks. Two exchanges are needed and both are ONE kernel each over peer-mapped memory:
//
//   * halo_exchange_kernel — a 3x3 convolution (forward, or its data gradient) on a stripe needs one row from
//     each neighbour. Conv inputs live in padded buffers [1 + rows + 1][W][C] inside a symmetric arena; the kernel
//     PUSHES this rank's first / last interior row into the neighbours' halo rows with 128-bit peer stores, then the
//     last CTA publishes a sequence number to the neighbours' flag words (st.release.sys) and waits for theirs
//     (ld.acquire.sys on local memory). Ranks at the image border zero their outer halo (= the conv's zero padding).
//   * gn32_finalize_peer_kernel (vae_kernels.cu) — GroupNorm statistics (forward: sum, sum of squares; backward: the two
//     gradient sums) are global over the image: each rank reduces its stripe as before, stores the raw sums in its
//     symmetric slot, publishes, waits for all peers and adds the slots in RANK ORDER, so every rank gets
//     bit-identical statistics without a collective launch.
//
// Sequence numbers: `seq` is added to the SEQUENCE BASE word kept next to the local flags (flags[8], zero unless
// rtti_peer_seq_advance has been called). A caller that numbers the exchanges of one colour-guidance call 1..n and
// advances the base by n at the end of the call issues the same kernel arguments every call, so the whole call can be
// captured once in a CUDA graph and replayed; the base lives in device memory and keeps the flags monotonic.
//
// Re-use safety without trailing barriers: pad buffers and sum slots are double-buffered by sequence parity. A
// neighbour can push exchange s+2 only after its exchange s+1 completed, which needs this rank's push s+1, which
// is stream-ordered after this rank's consumer of exchange s. A peer that never arrives trips a ~4 s timeout that
// sets an error word checked by the host (never a hung GPU).
#include "peer_sync.cuh"
#include "rtti_internal.h"

namespace rtti {

// flags (uint32, local symmetric memory): [0] from_up, [1] from_down, [2] error, [3] CTA arrival counter, [8] sequence base
constexpr int SEQ_BASE_WORD = 8;
__device__ __forceinline__ unsigned int ld_seq_base(const unsigned int* flags) {
  return *reinterpret_cast<const volatile unsigned int*>(flags + SEQ_BASE_WORD);
}
__global__ void __launch_bounds__(256) halo_exchange_kernel(float* __restrict__ pad, float* __restrict__ up,
                                                            float* __restrict__ down, int rows, long long row_vec,
                                                            unsigned int* fl, unsigned int* fl_up,
                                                            unsigned int* fl_down, unsigned int seq) {
  const float4* top_src = reinterpret_cast<const float4*>(pad) + row_vec;                       // interior row 0
  const float4* bot_src = reinterpret_cast<const float4*>(pad) + (long long)rows * row_vec;     // interior row rows-1
  float4* top_dst = up ? reinterpret_cast<float4*>(up) + (long long)(rows + 1) * row_vec        // neighbour's bottom halo
                       : reinterpret_cast<float4*>(pad);                                        // my own top halo := 0
  float4* bot_dst = down ? reinterpret_cast<float4*>(down)                                      // neighbour's top halo
                         : reinterpret_cast<float4*>(pad) + (long long)(rows + 1) * row_vec;    // my own bottom halo := 0
  const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < row_vec; i += (long long)gridDim.x * blockDim.x) {
    top_dst[i] = up ? top_src[i] : zero;
    bot_dst[i] = down ? bot_src[i] : zero;
  }
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned int arrived = atomicAdd(&fl[3], 1u);
    if (arrived == gridDim.x - 1) {   // last CTA: every push of this rank is visible system-wide
      fl[3] = 0u;
      seq += ld_seq_base(fl);
      __threadfence_system();
      if (up) st_release_sys(fl_up + 1, seq);      // I am my upper neighbour's "down"
      if (down) st_release_sys(fl_down + 0, seq);  // and my lower neighbour's "up"
      bool ok = true;
      if (up) ok = wait_seq(fl + 0, seq) && ok;
      if (down) ok = wait_seq(fl + 1, seq) && ok;
      if (!ok) fl[2] = 0xDEADu;
    }
  }
}

}  // namespace rtti

namespace rtti {
__global__ void peer_seq_advance_kernel(unsigned int* a, unsigned int da, unsigned int* b, unsigned int db) {
  if (a) a[SEQ_BASE_WORD] += da;
  if (b) b[SEQ_BASE_WORD] += db;
}
}  // namespace rtti

using namespace rtti;

extern "C" int rtti_peer_seq_advance(void* flags_a, unsigned int da, void* flags_b, unsigned int db, void* stream) {
  if (!flags_a && !flags_b) return RTTI_ERR_ARG;
  if (((uintptr_t)flags_a | (uintptr_t)flags_b) & 3) return RTTI_ERR_ALIGN;
  peer_seq_advance_kernel<<<1, 1, 0, (cudaStream_t)stream>>>((unsigned int*)flags_a, da, (unsigned int*)flags_b, db);
  return cudaGetLastError() == cudaSuccess ? RTTI_OK : RTTI_ERR_CUDA;
}

extern "C" int rtti_halo_exchange(float* pad_local, float* pad_up, float* pad_down, int rows, long long row_elems,
                                  void* flags_local, void* flags_up, void* flags_down, unsigned int seq, void* stream) {
  if (!pad_local || !flags_local || rows < 1 || row_elems < 4) return RTTI_ERR_ARG;
  if ((pad_up && !flags_up) || (pad_down && !flags_down)) return RTTI_ERR_ARG;
  if (row_elems % 4 != 0) return RTTI_ERR_SHAPE;
  if (((uintptr_t)pad_local | (uintptr_t)pad_up | (uintptr_t)pad_down) & 15) return RTTI_ERR_ALIGN;
  const long long row_vec = row_elems / 4;
  long long blocks = (row_vec + 255) / 256;
  if (blocks > 132) blocks = 132;
  halo_exchange_kernel<<<(int)blocks, 256, 0, (cudaStream_t)stream>>>(pad_local, pad_up, pad_down, rows, row_vec,
                                                                      (unsigned int*)flags_local, (unsigned int*)flags_up,
                                                                      (unsigned int*)flags_down, seq);
  return cudaGetLastError() == cudaSuccess ? RTTI_OK : RTTI_ERR_CUDA;
}
