// Fused region attention forward for sm_90a (wgmma + TMA + mbarrier).
//
// One kernel family covers both attention sites of the reference UNet
// (reference: models/attention_processor.py:1108-1183 AttnProcessor2_0.__call__,
//  :359-407 Attention.get_attention_scores, :166-171 head average):
//
//   * cross-attention (77 text keys, single key tile KT=80): softmax with the optional
//     font-size token re-weighting (attention_processor.py:387-399) and the optional capture of
//     the head-averaged probability map P-bar (attention_processor.py:1181 + the token-map hook
//     models/region_diffusion_sdxl.py:965-992) fused in-kernel; P is normalised BEFORE the fp16
//     rounding exactly as the reference does;
//   * self-attention (KT=64 key tiles, online softmax) with the self-attention *injection*
//     of the region passes (models/region_diffusion_sdxl.py:1018-1029: real_attn_probs replaces
//     softmax(QK^T)) expressed as a per-batch-entry Q/K source index `qk_src`: entry b attends with
//     the scores of entry qk_src[b] and its own V, which is what P_ref @ V_b computes.
//
// Layout: Q/K/V/O are [batch, tokens, heads*head_dim] fp16 with arbitrary batch/row strides
// (so fused QKV projections can be consumed in place); Q/K/V heads are addressed by a 4-D TMA tensor map
// {head_dim, heads, tokens, batch}, box {64, 1, rows, 1}, SWIZZLE_128B.  head_dim that is not a
// multiple of 64 is zero-padded by the TMA out-of-bounds fill, so 8/40/80/160 work as well.
//
// CTA = 128 query rows of one batch entry, 2 warpgroups of 64 rows each. Per pipeline item (one key tile; for the
// single-tile case one head with its Q) both warpgroups run S = Q K^T as wgmma with both operands in shared memory,
// the softmax on the register accumulators (a row is spread over the 4 threads of a quad), and O += P V as wgmma with
// P straight from registers (the S accumulator layout is the A-fragment layout) and V transposed from shared memory.
// Thread 0 keeps the next item's TMA loads in flight in a two-stage ring; a stage is refilled after the barrier that
// ends the item which read it. O is scaled, rounded and stored from the accumulators.
#include "ptx.cuh"
#include "rtti_internal.h"

namespace rtti {

struct AttnParams {
  int batch, heads, head_dim, n_q, n_k;
  int n_k_tiles, heads_per_cta;
  float scale_log2;     // softmax scale * log2(e)
  float inv_heads;
  int8_t qk_src[64];    // batch entry supplying Q and K for the scores (identity when no injection)
  int8_t cap_slot[64];  // slot of pbar to accumulate into, -1 = not captured
  unsigned long long fs_mask;  // batch entries that get the font-size re-weighting
  const int* word_pos;
  const float* font_size;
  int n_fs;
  float* pbar;  // [n_slots, n_q, n_k] fp32, += mean over heads of P
  float* lse;   // [batch, heads, n_q] fp32, log2-domain log-sum-exp of the scaled scores (optional)
  __half* o;
  long long o_bs, o_rs;
};

template <int KT, int NDCH>
struct AttnCfg {
  static constexpr bool SINGLE = KT == 80;       // whole key row in one tile: a pipeline item is one head (Q, K, V)
  static constexpr int Q_TILE = 128 * 128;       // bytes per 64-wide d-chunk of 128 query rows
  static constexpr int KV_TILE = KT * 128;
  static constexpr int STAGE = (SINGLE ? NDCH * Q_TILE : 0) + 2 * NDCH * KV_TILE;
  static constexpr int OFF_Q = 0;                // multi-tile: Q of the CTA's head, loaded once
  static constexpr int OFF_ST = SINGLE ? 0 : NDCH * Q_TILE;
  static constexpr int OFF_BAR = OFF_ST + 2 * STAGE;
  static constexpr int OFF_FS = OFF_BAR + 64;
  static constexpr int SMEM_BYTES = OFF_FS + 128 * 4 + 1024 /*alignment slack*/;
};

template <int KT, int NDCH, bool CAPTURE>
__global__ void __launch_bounds__(256, 1)
attn_fwd_kernel(const __grid_constant__ CUtensorMap tm_q, const __grid_constant__ CUtensorMap tm_k,
                const __grid_constant__ CUtensorMap tm_v, const __grid_constant__ AttnParams p) {
  using C = AttnCfg<KT, NDCH>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + C::OFF_BAR);   // [2] stage loaded
  uint64_t* q_full = full + 2;
  float* fs_w = reinterpret_cast<float*>(smem + C::OFF_FS);          // signed font-size weight per key

  const int tid = threadIdx.x, wg = tid >> 7, w = (tid >> 5) & 3, lane = tid & 31;
  const int q0 = blockIdx.x * 128;
  const int b = blockIdx.z;
  const int h_begin = blockIdx.y * p.heads_per_cta;
  const int h_end = min(p.heads, h_begin + p.heads_per_cta);
  const int b_qk = p.qk_src[b];
  const int n_items = C::SINGLE ? h_end - h_begin : p.n_k_tiles;

  auto load_item = [&](int it) {   // thread 0
    const int s = it & 1;
    uint8_t* st = smem + C::OFF_ST + s * C::STAGE;
    const int h = C::SINGLE ? h_begin + it : h_begin;
    const int k0 = C::SINGLE ? 0 : it * KT;
    uint8_t* kp = st + (C::SINGLE ? NDCH * C::Q_TILE : 0);
    uint8_t* vp = kp + NDCH * C::KV_TILE;
    mbar_expect_tx(&full[s], C::STAGE);
#pragma unroll
    for (int c = 0; c < NDCH; ++c) {
      if (C::SINGLE) tma_load_4d(st + c * C::Q_TILE, &tm_q, &full[s], 64 * c, h, q0, b_qk);
      tma_load_4d(kp + c * C::KV_TILE, &tm_k, &full[s], 64 * c, h, k0, b_qk);
      tma_load_4d(vp + c * C::KV_TILE, &tm_v, &full[s], 64 * c, h, k0, b);
    }
  };

  if (tid == 0) {
    tma_prefetch_desc(&tm_q); tma_prefetch_desc(&tm_k); tma_prefetch_desc(&tm_v);
    mbar_init(&full[0], 1); mbar_init(&full[1], 1); mbar_init(q_full, 1);
    mbar_fence_init();
    if (!C::SINGLE) {
      mbar_expect_tx(q_full, NDCH * C::Q_TILE);
#pragma unroll
      for (int c = 0; c < NDCH; ++c) tma_load_4d(smem + C::OFF_Q + c * C::Q_TILE, &tm_q, q_full, 64 * c, h_begin, q0, b_qk);
    }
    load_item(0);
    if (n_items > 1) load_item(1);
  }
  const bool use_fs = C::SINGLE && p.n_fs > 0 && ((p.fs_mask >> b) & 1ull);
  if (C::SINGLE && tid < 128) fs_w[tid] = 1.f;
  __syncthreads();
  if (use_fs && tid == 0) {
    // dense signed weight per key; duplicates in word_pos: last write wins, as the reference's
    // advanced-index assignment does on CPU (attention_processor.py:393-396)
    for (int i = 0; i < p.n_fs; ++i) {
      const int pos = p.word_pos[i];
      if (pos >= 0 && pos < p.n_k) fs_w[pos] = p.font_size[i];   // the reference would raise an index error beyond the 77 keys
    }
  }
  if (C::SINGLE) __syncthreads();

  // this thread's two rows (of the CTA's 128) and the first of its two columns in every 8-column group
  const int r0 = 64 * wg + 16 * w + (lane >> 2), r1 = r0 + 8;
  const int cq = 2 * (lane & 3);
  const uint32_t sbase = smem_u32(smem);
  const float sl2 = p.scale_log2;

  float o[NDCH][32];
  float pb[CAPTURE ? KT / 2 : 1];
  if (CAPTURE) {
#pragma unroll
    for (int i = 0; i < KT / 2; ++i) pb[i] = 0.f;
  }
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;

  // O / l -> fp16 -> global, and the log-sum-exp of head h
  auto epilogue = [&](int h) {
    const float inv0 = C::SINGLE ? 1.f : 1.f / l0, inv1 = C::SINGLE ? 1.f : 1.f / l1;
    const size_t rowbase = static_cast<size_t>(b) * p.o_bs + static_cast<size_t>(h) * p.head_dim;
#pragma unroll
    for (int c = 0; c < NDCH; ++c) {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int col = 64 * c + 8 * i + cq;
        if (col >= p.head_dim) continue;
        if (q0 + r0 < p.n_q)
          *reinterpret_cast<__half2*>(p.o + rowbase + static_cast<size_t>(q0 + r0) * p.o_rs + col) =
              __floats2half2_rn(o[c][4 * i] * inv0, o[c][4 * i + 1] * inv0);
        if (q0 + r1 < p.n_q)
          *reinterpret_cast<__half2*>(p.o + rowbase + static_cast<size_t>(q0 + r1) * p.o_rs + col) =
              __floats2half2_rn(o[c][4 * i + 2] * inv1, o[c][4 * i + 3] * inv1);
      }
    }
    if (p.lse != nullptr && (lane & 3) == 0) {
      float* dst = p.lse + (static_cast<size_t>(b) * p.heads + h) * p.n_q + q0;
      if (q0 + r0 < p.n_q) dst[r0] = m0 + log2f(l0);
      if (q0 + r1 < p.n_q) dst[r1] = m1 + log2f(l1);
    }
  };

  if (!C::SINGLE) {
#pragma unroll
    for (int c = 0; c < NDCH; ++c)
#pragma unroll
      for (int i = 0; i < 32; ++i) o[c][i] = 0.f;
    mbar_wait(q_full, 0);
  }

  for (int it = 0; it < n_items; ++it) {
    const int s = it & 1;
    const uint32_t st = sbase + C::OFF_ST + s * C::STAGE;
    const uint32_t qa = (C::SINGLE ? st : sbase + C::OFF_Q) + wg * 64 * 128;
    const uint32_t ka = st + (C::SINGLE ? NDCH * C::Q_TILE : 0);
    const uint32_t va = ka + NDCH * C::KV_TILE;
    mbar_wait(&full[s], (it >> 1) & 1);

    // ---- S = Q K^T (columns beyond head_dim are zero in both tiles)
    float sc[KT / 2];
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4 * NDCH; ++kk) {
      const uint32_t off = (kk & 3) * 32;   // +32 bytes per 16-element k step inside a 64-wide chunk
      wgmma_ss<KT>(sc, wgmma_desc_sw128(qa + (kk >> 2) * C::Q_TILE + off, 16, 1024),
                   wgmma_desc_sw128(ka + (kk >> 2) * C::KV_TILE + off, 16, 1024), kk > 0 ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait_all<KT / 2>(sc);

    // ---- softmax on the accumulators
    const int valid = p.n_k - (C::SINGLE ? 0 : it * KT);
    float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
    for (int i = 0; i < KT / 8; ++i) {
      const int col = 8 * i + cq;
      if (col >= valid) { sc[4 * i] = -INFINITY; sc[4 * i + 2] = -INFINITY; }
      if (col + 1 >= valid) { sc[4 * i + 1] = -INFINITY; sc[4 * i + 3] = -INFINITY; }
      mx0 = fmaxf(mx0, fmaxf(sc[4 * i], sc[4 * i + 1]));
      mx1 = fmaxf(mx1, fmaxf(sc[4 * i + 2], sc[4 * i + 3]));
    }
#pragma unroll
    for (int d = 1; d <= 2; d <<= 1) {
      mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, d));
      mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, d));
    }
    uint32_t pk[KT / 4];   // fp16 P: pk[2i] = row r0, pk[2i + 1] = row r1, columns 8i + cq + {0, 1}
    if (C::SINGLE) {
      // ---- whole row: P normalised before the fp16 rounding exactly as the reference (attention_processor.py:401-405)
      m0 = mx0 * sl2; m1 = mx1 * sl2;
      float e[KT / 2];
      float s0 = 0.f, s1 = 0.f;
#pragma unroll
      for (int i = 0; i < KT / 8; ++i) {
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const float wa = use_fs ? fabsf(fs_w[8 * i + cq + j]) : 1.f;
          e[4 * i + j] = ex2_approx(fmaf(sc[4 * i + j], sl2, -m0)) * wa;
          e[4 * i + 2 + j] = ex2_approx(fmaf(sc[4 * i + 2 + j], sl2, -m1)) * wa;
          s0 += e[4 * i + j];
          s1 += e[4 * i + 2 + j];
        }
      }
#pragma unroll
      for (int d = 1; d <= 2; d <<= 1) {
        s0 += __shfl_xor_sync(0xffffffffu, s0, d);
        s1 += __shfl_xor_sync(0xffffffffu, s1, d);
      }
      l0 = s0; l1 = s1;
      const float inv0 = 1.f / s0, inv1 = 1.f / s1;
#pragma unroll
      for (int i = 0; i < KT / 8; ++i) {
        float sg[2] = {1.f, 1.f};
        if (use_fs) {
#pragma unroll
          for (int j = 0; j < 2; ++j) {
            const float wv = fs_w[8 * i + cq + j];
            sg[j] = wv > 0.f ? 1.f : (wv < 0.f ? -1.f : 0.f);
          }
        }
        pk[2 * i] = pack_half2(e[4 * i] * inv0 * sg[0], e[4 * i + 1] * inv0 * sg[1]);
        pk[2 * i + 1] = pack_half2(e[4 * i + 2] * inv1 * sg[0], e[4 * i + 3] * inv1 * sg[1]);
      }
      if (CAPTURE) {
#pragma unroll
        for (int i = 0; i < KT / 4; ++i) {
          const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&pk[i]));
          pb[2 * i] += f.x;
          pb[2 * i + 1] += f.y;
        }
      }
#pragma unroll
      for (int c = 0; c < NDCH; ++c)
#pragma unroll
        for (int i = 0; i < 32; ++i) o[c][i] = 0.f;
    } else {
      // ---- online softmax over key tiles: rescale O and l when the row max grows
      const float mn0 = fmaxf(m0, mx0 * sl2), mn1 = fmaxf(m1, mx1 * sl2);
      const float a0 = ex2_approx(m0 - mn0), a1 = ex2_approx(m1 - mn1);
      m0 = mn0; m1 = mn1;
      l0 *= a0; l1 *= a1;
#pragma unroll
      for (int c = 0; c < NDCH; ++c)
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          o[c][4 * i] *= a0; o[c][4 * i + 1] *= a0;
          o[c][4 * i + 2] *= a1; o[c][4 * i + 3] *= a1;
        }
#pragma unroll
      for (int i = 0; i < KT / 8; ++i) {
        const float e0 = ex2_approx(fmaf(sc[4 * i], sl2, -m0)), e1 = ex2_approx(fmaf(sc[4 * i + 1], sl2, -m0));
        const float e2 = ex2_approx(fmaf(sc[4 * i + 2], sl2, -m1)), e3 = ex2_approx(fmaf(sc[4 * i + 3], sl2, -m1));
        l0 += e0 + e1;
        l1 += e2 + e3;
        pk[2 * i] = pack_half2(e0, e1);
        pk[2 * i + 1] = pack_half2(e2, e3);
      }
    }

    // ---- O += P V (V is MN-major: 16 keys further = +2048 bytes)
    wgmma_fence();
#pragma unroll
    for (int c = 0; c < NDCH; ++c) {
      pin_regs<32>(o[c]);
#pragma unroll
      for (int kk = 0; kk < KT / 16; ++kk)
        wgmma_rs_tb<64>(o[c], &pk[4 * kk], wgmma_desc_sw128(va + c * C::KV_TILE + kk * 2048, C::KV_TILE, 1024), 1u);
    }
    wgmma_commit();
    wgmma_wait_all<32>(o[0]);
#pragma unroll
    for (int c = 1; c < NDCH; ++c) pin_regs<32>(o[c]);

    if (C::SINGLE) epilogue(h_begin + it);
    __syncthreads();   // every warpgroup is done with stage s
    if (tid == 0 && it + 2 < n_items) load_item(it + 2);
  }

  if (!C::SINGLE) {
#pragma unroll
    for (int d = 1; d <= 2; d <<= 1) {
      l0 += __shfl_xor_sync(0xffffffffu, l0, d);
      l1 += __shfl_xor_sync(0xffffffffu, l1, d);
    }
    epilogue(h_begin);
  }
  if (CAPTURE) {
    const int slot = p.cap_slot[b];
    if (slot >= 0) {
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const int row = q0 + (r ? r1 : r0);
        if (row >= p.n_q) continue;
        float* dst = p.pbar + (static_cast<size_t>(slot) * p.n_q + row) * p.n_k;
#pragma unroll
        for (int i = 0; i < KT / 8; ++i)
#pragma unroll
          for (int j = 0; j < 2; ++j)
            if (8 * i + cq + j < p.n_k) dst[8 * i + cq + j] += pb[4 * i + 2 * r + j] * p.inv_heads;
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
template <int KT, int NDCH, bool CAPTURE>
static int launch(const CUtensorMap& tq, const CUtensorMap& tk, const CUtensorMap& tv, const AttnParams& p, dim3 grid,
                  cudaStream_t stream) {
  using C = AttnCfg<KT, NDCH>;
  auto kern = attn_fwd_kernel<KT, NDCH, CAPTURE>;
  static const bool configured =
      cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES) == cudaSuccess;
  if (!configured) return RTTI_ERR_CUDA;
  kern<<<grid, 256, C::SMEM_BYTES, stream>>>(tq, tk, tv, p);
  return cudaGetLastError() == cudaSuccess ? RTTI_OK : RTTI_ERR_CUDA;
}

}  // namespace rtti

using namespace rtti;

extern "C" int rtti_attn_fwd(const void* q, const void* k, const void* v, void* o, int batch, int heads,
                             int head_dim, int n_q, int n_k, long long q_bs, long long q_rs, long long k_bs,
                             long long k_rs, long long v_bs, long long v_rs, long long o_bs, long long o_rs,
                             float scale, const int* qk_src, const int* word_pos, const float* font_size,
                             int n_fs, unsigned long long fs_batch_mask, float* pbar_accum,
                             const int* cap_slot, float* lse, void* stream) {
  if (!q || !k || !v || !o) return RTTI_ERR_ARG;
  if (batch < 1 || batch > 64 || heads < 1 || n_q < 1 || n_k < 1) return RTTI_ERR_ARG;
  if (head_dim < 8 || head_dim > 192 || (head_dim % 8) != 0) return RTTI_ERR_SHAPE;
  if (((uintptr_t)q | (uintptr_t)k | (uintptr_t)v | (uintptr_t)o) & 15) return RTTI_ERR_ALIGN;
  if ((q_bs | q_rs | k_bs | k_rs | v_bs | v_rs | o_bs | o_rs) & 7) return RTTI_ERR_ALIGN;
  const bool want_fs = (n_fs > 0 && fs_batch_mask != 0);
  const bool want_cap = (pbar_accum != nullptr && cap_slot != nullptr);
  if ((want_fs || want_cap) && n_k > 80) return RTTI_ERR_SHAPE;  // normalised-P features need one key tile
  if (want_fs && (!word_pos || !font_size)) return RTTI_ERR_ARG;
  if (qk_src)
    for (int i = 0; i < batch; ++i)
      if (qk_src[i] < 0 || qk_src[i] >= batch) return RTTI_ERR_ARG;
  if (want_cap) {
    // pbar_accum[slot] += is a plain read-modify-write by the CTAs of one entry: two entries naming the same slot
    // would race and lose updates, so every captured entry needs a slot of its own (and one that fits the int8 copy)
    unsigned long long used[2] = {0ull, 0ull};
    for (int i = 0; i < batch; ++i) {
      const int s = cap_slot[i];
      if (s < -1 || s > 127) return RTTI_ERR_ARG;
      if (s < 0) continue;
      if ((used[s >> 6] >> (s & 63)) & 1ull) return RTTI_ERR_ARG;
      used[s >> 6] |= 1ull << (s & 63);
    }
  }
  int rc = rtti_arch_ok();
  if (rc != RTTI_OK) return rc;
  static const int n_sm = [] {
    int dev = 0, v = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev);
    return v;
  }();

  const int ndch = (head_dim + 63) / 64;
  // up to 80 keys (77 text keys, or an 8x8 self-attention level): one 80-key tile; longer rows: 64-key tiles
  const int KT = (n_k <= 80) ? 80 : 64;
  AttnParams p{};
  p.batch = batch; p.heads = heads; p.head_dim = head_dim; p.n_q = n_q; p.n_k = n_k;
  p.n_k_tiles = (n_k + KT - 1) / KT;
  p.heads_per_cta = want_cap ? heads : 1;   // capture: the head mean stays inside one CTA (no atomics, deterministic)
  if (!want_cap && KT == 80) {
    // single key tile: several heads per CTA so the TMA loads of head h+1 overlap the softmax/epilogue of
    // head h (two-stage ring), while keeping at least two CTAs per SM worth of work
    const long long ctas1 = (long long)((n_q + 127) / 128) * heads * batch;
    const int cand[] = {10, 8, 5, 4, 2};
    for (int c : cand)
      if (heads % c == 0 && ctas1 / c >= 2 * n_sm) { p.heads_per_cta = c; break; }
  }
  p.scale_log2 = scale * 1.4426950408889634f;
  p.inv_heads = 1.f / (float)heads;
  for (int i = 0; i < 64; ++i) { p.qk_src[i] = (int8_t)i; p.cap_slot[i] = -1; }
  if (qk_src)
    for (int i = 0; i < batch; ++i) p.qk_src[i] = (int8_t)qk_src[i];   // range checked above
  if (want_cap)
    for (int i = 0; i < batch; ++i) p.cap_slot[i] = (int8_t)cap_slot[i];
  p.fs_mask = want_fs ? fs_batch_mask : 0ull;
  p.word_pos = word_pos; p.font_size = font_size; p.n_fs = want_fs ? n_fs : 0;
  p.pbar = want_cap ? pbar_accum : nullptr;
  p.lse = lse;
  p.o = (__half*)o; p.o_bs = o_bs; p.o_rs = o_rs;

  CUtensorMap tq, tk, tv;
  if ((rc = make_head_map(&tq, q, head_dim, heads, n_q, batch, q_bs, q_rs, 128)) != RTTI_OK) return rc;
  if ((rc = make_head_map(&tk, k, head_dim, heads, n_k, batch, k_bs, k_rs, KT)) != RTTI_OK) return rc;
  if ((rc = make_head_map(&tv, v, head_dim, heads, n_k, batch, v_bs, v_rs, KT)) != RTTI_OK) return rc;

  dim3 grid((n_q + 127) / 128, (heads + p.heads_per_cta - 1) / p.heads_per_cta, batch);
  cudaStream_t st = (cudaStream_t)stream;
#define RTTI_LAUNCH(KT_, ND_, CAP_) return launch<KT_, ND_, CAP_>(tq, tk, tv, p, grid, st)
  if (KT == 80) {
    if (want_cap) {
      if (ndch == 1) RTTI_LAUNCH(80, 1, true);
      if (ndch == 2) RTTI_LAUNCH(80, 2, true);
      RTTI_LAUNCH(80, 3, true);
    }
    if (ndch == 1) RTTI_LAUNCH(80, 1, false);
    if (ndch == 2) RTTI_LAUNCH(80, 2, false);
    RTTI_LAUNCH(80, 3, false);
  }
  if (ndch == 1) RTTI_LAUNCH(64, 1, false);
  if (ndch == 2) RTTI_LAUNCH(64, 2, false);
  RTTI_LAUNCH(64, 3, false);
#undef RTTI_LAUNCH
}
