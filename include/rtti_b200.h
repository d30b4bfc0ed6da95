/* rtti_b200 — C ABI of the region-diffusion hot path for the H100 (sm_90a).
 *
 * The reference (songweige/rich-text-to-image) has no FFI: its hot path is Python calling ATen.
 * Each entry point below replaces one (group of) reference call site(s); citations are
 * file:line in the reference tree.  A Python/ctypes (or any other FFI) host binds exactly these
 * symbols; see INTEGRATION.md for the reference-side stubs.
 *
 * Conventions
 *   - All pointers are DEVICE pointers unless marked "host".  The caller owns every buffer.
 *   - No entry point allocates, synchronises, or touches a stream other than `stream`
 *     (a cudaStream_t passed as void*); all are CUDA-graph capturable.
 *   - fp16 = IEEE binary16 (`__half`), row-major, innermost dimension contiguous.
 *   - Return value: RTTI_OK (0) or a negative RTTI_ERR_* code; nothing is launched on error.
 *   - The caller selects the device (cudaSetDevice) before the call; sm_90 is required.
 */
#ifndef RTTI_B200_H
#define RTTI_B200_H

#ifdef __cplusplus
extern "C" {
#endif

#define RTTI_OK 0
#define RTTI_ERR_ARG (-1)    /* null pointer / out-of-range argument */
#define RTTI_ERR_SHAPE (-2)  /* unsupported shape (e.g. head_dim not a multiple of 8 or > 192) */
#define RTTI_ERR_ALIGN (-3)  /* pointer not 16-byte aligned / stride not a multiple of 8 elements */
#define RTTI_ERR_ARCH (-4)   /* device is not sm_90 */
#define RTTI_ERR_CUDA (-5)   /* CUDA runtime / driver call failed (see cudaGetLastError) */

/* Library version: major*10000 + minor*100 + patch. */
int rtti_version(void);
/* RTTI_OK when the current device can run these kernels (compute capability 10.x). */
int rtti_arch_ok(void);

/* Fused attention forward: O = softmax(scale * Q K^T) V per head, on wgmma tensor cores.
 * Replaces Attention.get_attention_scores + torch.bmm + reshape_batch_dim_to_heads_and_average
 * (models/attention_processor.py:359-407, 1157-1163, 166-171, 1181) and the hook passes that
 * sit around them (models/region_diffusion_sdxl.py:959-1140).
 *
 *   q [batch, n_q, heads*head_dim], k/v [batch, n_k, heads*head_dim], o like q; fp16.
 *   *_bs / *_rs: batch and row strides in ELEMENTS (multiples of 8); head h starts at column h*head_dim.
 *   scale: softmax scale (head_dim^-0.5 in the reference, attention_processor.py:90).
 *   qk_src (host, [batch] or NULL): batch entry whose Q and K produce the probabilities applied to
 *       entry b's V — the self-attention injection of the region passes
 *       (real_attn_probs, attention_processor.py:1160-1163; region_diffusion_sdxl.py:1023-1029).
 *   word_pos [n_fs] int32, font_size [n_fs] fp32 (device), fs_batch_mask (bit b = apply to entry b):
 *       font-size re-weighting  E[:, pos] *= |fs|;  P = E / sum(E);  P[:, pos] *= sign(fs)
 *       (attention_processor.py:387-399; hooks region_diffusion_sdxl.py:1112-1140). Needs n_k <= 80.
 *   pbar_accum [n_slots, n_q, n_k] fp32 (device), cap_slot (host, [batch], -1 = skip):
 *       pbar_accum[cap_slot[b]] += mean over heads of P[b]  — the token-map capture of
 *       region_diffusion_sdxl.py:965-992 without the D2H copy. Deterministic. Needs n_k <= 80.
 *       Each slot is -1..127 and no two entries may name the same slot >= 0 (their updates would race);
 *       RTTI_ERR_ARG otherwise, as for a qk_src[b] outside [0, batch). Both host arrays are checked
 *       before the device is queried, so the rule holds without a GPU.
 *   lse [batch, heads, n_q] fp32 or NULL: log2-domain log-sum-exp of the scaled scores
 *       (consumed by rtti_attn_probs_mean_accum).
 */
int rtti_attn_fwd(const void* q, const void* k, const void* v, void* o, int batch, int heads, int head_dim,
                  int n_q, int n_k, long long q_bs, long long q_rs, long long k_bs, long long k_rs,
                  long long v_bs, long long v_rs, long long o_bs, long long o_rs, float scale,
                  const int* qk_src, const int* word_pos, const float* font_size, int n_fs,
                  unsigned long long fs_batch_mask, float* pbar_accum, const int* cap_slot, float* lse,
                  void* stream);

/* Self-attention token-map capture: accum[n_q, n_k] += mean_h exp2(scale*log2e * Q_h K_h^T - lse_h)
 * for ONE batch entry (the conditional row the reference keeps, region_diffusion_sdxl.py:989-992),
 * recomputing QK^T on tensor cores instead of materialising P (attention_processor.py:1181).
 *   q/k: [n_q|n_k, heads*head_dim] fp16 of that batch entry, row strides in elements;
 *   lse: [heads, n_q] fp32 as written by rtti_attn_fwd for that entry.
 */
int rtti_attn_probs_mean_accum(const void* q, const void* k, const float* lse, float* accum, int heads,
                               int head_dim, int n_q, int n_k, long long q_rs, long long k_rs, float scale,
                               void* stream);

/* GroupNorm (+ optional SiLU) over channels-last activations x[batch, hw, c] fp16.
 * Replaces norm1/norm2 + nonlinearity of ResnetBlock2D (models/resnet.py:597-600, 624-629),
 * Transformer2DModel.norm (models/transformer_2d.py:272) and conv_norm_out + conv_act
 * (models/unet_2d_condition.py:975-977).  gamma/beta fp16 [c]; stats in fp32. c a multiple of 8 and of groups,
 * c <= 8192 (RTTI_ERR_SHAPE otherwise).
 *   chan_bias: optional fp16 [batch, c] added to x before the statistics — the time-embedding add
 *   `hidden_states + temb` that precedes norm2 (models/resnet.py:621-622), fused; NULL to skip.
 *   workspace: fp32 [batch * ceil(hw/rows_per_block) * groups * 2] partial (mean, sum of squared deviations),
 *   merged pairwise (Chan et al.) so the variance keeps its accuracy for inputs with |mean| >> std; query the element
 *   count with rtti_groupnorm_workspace_elems.  Deterministic (no atomics).
 */
long long rtti_groupnorm_workspace_elems(int batch, int hw, int c, int groups);
int rtti_groupnorm_silu_fwd(const void* x, const void* chan_bias, const void* gamma, const void* beta, void* y,
                            float* workspace, int batch, int hw, int c, int groups, float eps, int apply_silu,
                            void* stream);

/* out[rows, c] = a + b + bias[c] (fp16; bias may be NULL): the residual add of ResnetBlock2D
 * (models/resnet.py:637-643) fused with the bias of conv2. */
int rtti_add_bias_f16(const void* a, const void* b, const void* bias, void* out, long long rows, int c, void* stream);

/* LayerNorm over the last dimension of x[rows, c] fp16 (models/attention.py:150,168,181). */
int rtti_layernorm_fwd(const void* x, const void* gamma, const void* beta, void* y, int rows, int c, float eps,
                       void* stream);

/* Feed-forward input projection with the GEGLU gate fused into the GEMM epilogue (wgmma GEMM, register accumulators):
 *   y[m, n] = (x[m, k] w[0:n, :]^T + bias[0:n]) * gelu(x w[n:2n, :]^T + bias[n:2n])     (exact erf GELU)
 * x [m, k], w [2n, k] (the nn.Linear weight of ff.net.0.proj: value rows first, gate rows second), y [m, n], all fp16
 * row-major contiguous; bias [2n] fp16 or NULL. Replaces models/attention.py:283-304 (GEGLU.forward: proj -> chunk ->
 * hidden * gelu(gate)); the [m, 2n] intermediate is never written. n % 128 == 0, k % 64 == 0. */
int rtti_ff_geglu_fwd(const void* x, const void* w, const void* bias, void* y, long long m, int n, int k, void* stream);

/* h_out = fp16(a + resid + bias[c]);  y = LayerNorm(h_out) * gamma + beta, rows x c fp16, one pass over DRAM.
 * Replaces the residual add after an attention / feed-forward projection together with the LayerNorm that follows it:
 * models/attention.py:155-160, 172-178 (`attn(...) + hidden_states`) + :168, :181 (norm2 / norm3); the projection's
 * bias (models/attention_processor.py:1167) is folded in. h_out may alias resid; bias may be NULL. c % 8 == 0, c <= 2048. */
int rtti_add_bias_layernorm_fwd(const void* a, const void* resid, const void* bias, const void* gamma, const void* beta,
                                void* h_out, void* y, int rows, int c, float eps, void* stream);

/* GEGLU gate: y[rows, inner] = proj[rows, :inner] * gelu_erf(proj[rows, inner:])
 * (models/attention.py:283-304). */
int rtti_geglu_fwd(const void* proj, void* y, int rows, int inner, void* stream);

/* Region blend + classifier-free guidance (+ optional Euler update), one launch.
 * Replaces models/region_diffusion_sdxl.py:810-825 (and :845 when dt_sigma != 0):
 *   eps_u = sum_i eps_uncond * m_i ; eps_t = sum_i eps_region[i] * m_i   (i over all n_regions masks,
 *   eps_region[n_regions-1] is the base-prompt pass, masks[n_regions-1] the remainder mask)
 *   eps = eps_u + guidance * (eps_t - eps_u)
 *   latents_out = latents + dt_sigma * eps            (only when latents/latents_out non-NULL)
 * eps_* fp16 [n], masks fp32 [n_regions, n], n = 4*h*w. eps_region rows may live in different
 * buffers: `eps_region` is a host array of n_regions device pointers.
 */
int rtti_region_blend_cfg(const void* eps_uncond, const void* const* eps_region, const float* masks,
                          int n_regions, long long n, float guidance, void* eps_out, const void* latents,
                          void* latents_out, float dt_sigma, void* stream);

/* rtti_region_blend_cfg with the CFG rescale of diffusers' rescale_noise_cfg (models/region_diffusion_sdxl.py:42-53,
 * applied at :903-905; the rich-text loop's call left as a TODO at :827-830):
 *   eps = eps_cfg * (1 - guidance_rescale + guidance_rescale * std(eps_t) / std(eps_cfg))
 * with eps_t the blended text prediction and eps_cfg = eps_u + guidance * (eps_t - eps_u), the unbiased standard
 * deviations taken over all n elements in fp32 from the fp32 values; eps is rounded to fp16 before it is stored and
 * before the Euler update consumes it. std(eps_cfg) = 0 gives a non-finite result, as the formula does.
 * One launch of one 8-CTA thread-block cluster (the statistics are merged in a fixed order through distributed shared
 * memory: deterministic, no workspace, no atomics). n a multiple of 8 and <= 262144 (RTTI_ERR_SHAPE otherwise),
 * n_regions <= 16; all pointers 16-byte aligned. */
int rtti_region_blend_cfg_rescale(const void* eps_uncond, const void* const* eps_region, const float* masks,
                                  int n_regions, long long n, float guidance, void* eps_out, const void* latents,
                                  void* latents_out, float dt_sigma, float guidance_rescale, void* stream);

/* Multistep forms ("_ms") of the blend entry points, for DDIM and DPM-Solver++(2M) (rich-text-to-image_b200/schedulers.py,
 * StepCoeffs). The blend, CFG and rescale arithmetic is that of the Euler form; the update of the latents is
 *   D  = hx * x + he * eps                (fp32, written to d_out[n])
 *   x' = cx * x + cd * D + cp * D_prev    (D_prev = d_prev[n], read only when cp != 0; x' rounded to fp16)
 * with x the fp16 latents and eps the fp16-rounded noise prediction written to eps_out. latents, latents_out and d_out
 * are required; d_prev may be null only when cp == 0, and it may alias d_out (every element is read before it is
 * written, by the same thread). d_prev / d_out 16-byte aligned. The other checks are those of the Euler form; on any
 * error nothing is launched. */
int rtti_region_blend_cfg_ms(const void* eps_uncond, const void* const* eps_region, const float* masks, int n_regions,
                             long long n, float guidance, void* eps_out, const void* latents, void* latents_out,
                             float hx, float he, float cx, float cd, float cp, const float* d_prev, float* d_out,
                             void* stream);
int rtti_region_blend_cfg_rescale_ms(const void* eps_uncond, const void* const* eps_region, const float* masks,
                                     int n_regions, long long n, float guidance, void* eps_out, const void* latents,
                                     void* latents_out, float hx, float he, float cx, float cd, float cp,
                                     const float* d_prev, float* d_out, float guidance_rescale, void* stream);

/* Ancestral forms ("_anc") of the blend entry points, for Euler Ancestral (rich-text-to-image_b200/schedulers.py,
 * EulerAncestralDiscreteScheduler.ancestral_coeffs). The blend, CFG and rescale arithmetic is that of the Euler form;
 * the update of the latents is, in fp32,
 *   x' = fma(z, s_up, fma(eps, dt_sigma, x))    (dt_sigma = sigma_down - sigma; x' rounded to fp16)
 * with x the fp16 latents, eps the fp16-rounded noise prediction written to eps_out and z[n] the fp16 noise of the step,
 * read only when s_up != 0 (with s_up == 0 the result equals the Euler form's with the same dt_sigma, bit for bit).
 * latents and latents_out are required; z is required when s_up != 0 and must be 16-byte aligned. The other checks are
 * those of the Euler form; on any error nothing is launched. */
int rtti_region_blend_cfg_anc(const void* eps_uncond, const void* const* eps_region, const float* masks, int n_regions,
                              long long n, float guidance, void* eps_out, const void* latents, void* latents_out,
                              float dt_sigma, float s_up, const void* z, void* stream);
int rtti_region_blend_cfg_rescale_anc(const void* eps_uncond, const void* const* eps_region, const float* masks,
                                      int n_regions, long long n, float guidance, void* eps_out, const void* latents,
                                      void* latents_out, float dt_sigma, float s_up, const void* z,
                                      float guidance_rescale, void* stream);

/* UniPC forms ("_unipc") of the blend entry points, for UniPC bh2 of order 2 (rich-text-to-image_b200/schedulers.py,
 * UniPCMultistepScheduler.unipc_coeffs). The blend, CFG and rescale arithmetic is that of the Euler form; the update of
 * the latents is, in fp32,
 *   m  = hx * x + he * eps                                   (written to m_out[n])
 *   xc = ux * x + ul * xl + u0 * m + u1 * m1 + u2 * m2       (the corrected sample, written to xl_out[n])
 *   x' = vx * xc + v0 * m + v1 * m1                          (x' rounded to fp16)
 * with x the fp16 latents, eps the fp16-rounded noise prediction written to eps_out, and xl, m1, m2 the fp32 [n]
 * histories (xc of the previous step, m of the previous two steps). latents, latents_out, m_out and xl_out are required;
 * xl may be null only when ul == 0, m1 only when u1 == v1 == 0, m2 only when u2 == 0, and a history is read only when
 * one of its coefficients is non-zero. m_out may alias m2 and xl_out may alias xl (every element is read before it is
 * written, by the same thread). Histories 16-byte aligned. The other checks are those of the Euler form; on any error
 * nothing is launched. */
int rtti_region_blend_cfg_unipc(const void* eps_uncond, const void* const* eps_region, const float* masks,
                                int n_regions, long long n, float guidance, void* eps_out, const void* latents,
                                void* latents_out, float hx, float he, float ux, float ul, float u0, float u1,
                                float u2, float vx, float v0, float v1, const float* xl, const float* m1,
                                const float* m2, float* m_out, float* xl_out, void* stream);
int rtti_region_blend_cfg_rescale_unipc(const void* eps_uncond, const void* const* eps_region, const float* masks,
                                        int n_regions, long long n, float guidance, void* eps_out, const void* latents,
                                        void* latents_out, float hx, float he, float ux, float ul, float u0, float u1,
                                        float u2, float vx, float v0, float v1, const float* xl, const float* m1,
                                        const float* m2, float* m_out, float* xl_out, float guidance_rescale,
                                        void* stream);

/* Heun forms ("_heun") of the blend entry points, for Heun's method (rich-text-to-image_b200/schedulers.py,
 * HeunDiscreteScheduler.heun_coeffs). They replace the scheduler step of models/region_diffusion_sdxl.py:837-846 and
 * :908 with a HeunDiscreteScheduler assigned to the reference's scheduler. The blend, CFG and rescale arithmetic is
 * that of the Euler form; the update of the latents is, in fp32,
 *   x' = cx * x + ce * eps + cd * ds + cs * xs      (x' rounded to fp16)
 * with x the fp16 latents, eps the fp16-rounded (rescaled) noise prediction written to eps_out, and xs[n] / ds[n] the
 * fp16 latents and noise prediction of the last first stage: (cx, ce, cs, cd) = (1, dt, 0, 0) at a first stage,
 * (0, dt/2, 1, dt/2) at a second. ds is read only when cd != 0 and xs only when cs != 0; with (1, dt, 0, 0) the result
 * equals the Euler form's with dt_sigma = dt, bit for bit. latents and latents_out are required; xs is required when
 * cs != 0 and ds when cd != 0, both 16-byte aligned when given. The other checks are those of the Euler form; on any
 * error nothing is launched. */
int rtti_region_blend_cfg_heun(const void* eps_uncond, const void* const* eps_region, const float* masks,
                               int n_regions, long long n, float guidance, void* eps_out, const void* latents,
                               void* latents_out, float cx, float ce, float cs, float cd, const void* xs,
                               const void* ds, void* stream);
int rtti_region_blend_cfg_rescale_heun(const void* eps_uncond, const void* const* eps_region, const float* masks,
                                       int n_regions, long long n, float guidance, void* eps_out, const void* latents,
                                       void* latents_out, float cx, float ce, float cs, float cd, const void* xs,
                                       const void* ds, float guidance_rescale, void* stream);

/* LMS forms ("_lms") of the blend entry points, for k-LMS, the fourth-order linear multistep method on Euler's sigma
 * grid (rich-text-to-image_b200/schedulers.py, LMSDiscreteScheduler.lms_coeffs). They replace the scheduler step of
 * models/region_diffusion_sdxl.py:837-846 and :908 with an LMSDiscreteScheduler assigned to the reference's scheduler.
 * The blend, CFG and rescale arithmetic is that of the Euler form; the update of the latents is, in fp32,
 *   x' = x + c0 * eps + c1 * d1 + c2 * d2 + c3 * d3      (x' rounded to fp16)
 * with x the fp16 latents, eps the fp16-rounded (rescaled) noise prediction written to eps_out, and d1[n], d2[n], d3[n]
 * the fp16 eps_out of the trajectory's last three steps, newest first. The terms are added in that order. d_k is read
 * only when c_k != 0; with (c0, 0, 0, 0) the result equals the Euler form's with dt_sigma = c0, bit for bit. latents and
 * latents_out are required; d_k is required when c_k != 0, and each is 16-byte aligned when given. The histories are
 * only read: they must not overlap eps_out or latents_out. The other checks are those of the Euler form; on any error
 * nothing is launched. */
int rtti_region_blend_cfg_lms(const void* eps_uncond, const void* const* eps_region, const float* masks, int n_regions,
                              long long n, float guidance, void* eps_out, const void* latents, void* latents_out,
                              float c0, float c1, float c2, float c3, const void* d1, const void* d2, const void* d3,
                              void* stream);
int rtti_region_blend_cfg_rescale_lms(const void* eps_uncond, const void* const* eps_region, const float* masks,
                                      int n_regions, long long n, float guidance, void* eps_out, const void* latents,
                                      void* latents_out, float c0, float c1, float c2, float c3, const void* d1,
                                      const void* d2, const void* d3, float guidance_rescale, void* stream);

/* Singlestep forms ("_ss") of the blend entry points, for DPM-Solver++(2S) (rich-text-to-image_b200/schedulers.py,
 * DPMSolverSinglestepScheduler.singlestep_coeffs). They replace the scheduler step of
 * models/region_diffusion_sdxl.py:837-846 and :908 with a DPMSolverSinglestepScheduler assigned to the reference's
 * scheduler. The blend, CFG and rescale arithmetic is that of the Euler form; the update of the latents is, in fp32,
 *   D  = hx * x + he * eps                              (written to d_out[n])
 *   x' = cx * x + cd * D + cp * D_prev + cs * xs        (x' rounded to fp16)
 * with x the fp16 latents, eps the fp16-rounded (rescaled) noise prediction written to eps_out, D_prev = d_prev[n]
 * the D of the block's first step and xs[n] the fp16 latents that entered it. The multistep update is formed exactly as the
 * "_ms" forms form it and cs * xs is added last; xs is read only when cs != 0, so with cs == 0 the result (latents_out,
 * d_out and eps_out) equals the "_ms" form's bit for bit. latents, latents_out and d_out are required; d_prev may be
 * null only when cp == 0 and may alias d_out; xs may be null only when cs == 0. d_prev / d_out / xs 16-byte aligned.
 * The other checks are those of the Euler form; on any error nothing is launched. */
int rtti_region_blend_cfg_ss(const void* eps_uncond, const void* const* eps_region, const float* masks, int n_regions,
                             long long n, float guidance, void* eps_out, const void* latents, void* latents_out,
                             float hx, float he, float cx, float cs, float cd, float cp, const float* d_prev,
                             float* d_out, const void* xs, void* stream);
int rtti_region_blend_cfg_rescale_ss(const void* eps_uncond, const void* const* eps_region, const float* masks,
                                     int n_regions, long long n, float guidance, void* eps_out, const void* latents,
                                     void* latents_out, float hx, float he, float cx, float cs, float cd, float cp,
                                     const float* d_prev, float* d_out, const void* xs, float guidance_rescale,
                                     void* stream);

/* Colour-guidance loss forward + analytic backward w.r.t. the VAE decoder output.
 * Replaces models/region_diffusion_sdxl.py:857-865 (clamp, masked mean RGB, MSE*100, autograd of those).
 *   decoded [3, hw] fp32 (VAE output before /2+0.5), masks [n_colors, hw] fp32 (channel 0 of
 *   color_obj_atten), target_rgb [n_colors, 3] fp32.
 *   loss_out [1] fp32; grad_decoded [3, hw] fp32 = d loss / d decoded.
 *   workspace fp32 [rtti_color_loss_workspace_elems(n_colors, hw)].
 */
long long rtti_color_loss_workspace_elems(int n_colors, long long hw);
int rtti_color_loss_fwd_bwd(const float* decoded, const float* masks, const float* target_rgb, int n_colors,
                            long long hw, float* loss_out, float* grad_decoded, float* workspace, void* stream);

/* latents_out = latents - grad * weight * atten_all   (models/region_diffusion_sdxl.py:866-867).
 * latents fp16, grad fp32, atten_all fp32, all [n]. */
int rtti_latent_guidance_update(const void* latents, const float* grad, const float* atten_all, float weight,
                                void* latents_out, long long n, void* stream);

/* out = latents_ref * m + latents * (1 - m)   (models/region_diffusion_sdxl.py:870-872). fp16, m fp32. */
int rtti_bg_inject_blend(const void* latents, const void* latents_ref, const float* mask, void* out,
                         long long n, void* stream);

/* x0 = (x_t - eps * sqrt(1-alpha)) / sqrt(alpha)   (models/region_diffusion_sdxl.py:955-957). fp16. */
int rtti_predict_x0(const void* x_t, const void* eps, float alpha, void* x0, long long n, void* stream);

/* fp32 channels-last GroupNorm(+SiLU) forward / input-gradient backward for the VAE decoder that colour guidance
 * differentiates through (third-party AutoencoderKL, called at models/region_diffusion_sdxl.py:856-865 and
 * models/region_diffusion.py:157-165). x, y, dz, dx: [batch, hw, c] fp32; gamma/beta [c] fp32;
 * c a multiple of 4 and of groups, c <= 2048 (RTTI_ERR_SHAPE otherwise);
 * mean_rstd [batch, groups, 2] fp32 (written by fwd, read by bwd); workspace fp32
 * [rtti_gn32_workspace_elems(...)]. dx = d loss / d x given dz = d loss / d (silu?(GN(x))).
 * chan_bias: optional fp32 [c] added to x first (the bias of the convolution that produced x, folded in); NULL to skip.
 * addend (bwd): optional fp32 [batch, hw, c] added to dx (the gradient reaching a resnet block's shortcut path); NULL
 * to skip.
 */
long long rtti_gn32_workspace_elems(int batch, int hw, int c, int groups);
int rtti_gn32_silu_fwd(const float* x, const float* chan_bias, const float* gamma, const float* beta, float* y,
                       float* mean_rstd, float* workspace, int batch, int hw, int c, int groups, float eps,
                       int apply_silu, void* stream);
int rtti_gn32_silu_bwd(const float* x, const float* chan_bias, const float* dz, const float* gamma, const float* beta,
                       const float* mean_rstd, const float* addend, float* dx, float* workspace, int batch, int hw,
                       int c, int groups, int apply_silu, void* stream);
/* Nearest x2 upsample + 3x3 convolution of the VAE decoder (diffusers Upsample2D) evaluated at low resolution:
 * output pixel (2i+a, 2j+b) only sees low-res rows {i-1, i} (a = 0) or {i, i+1} (a = 1), likewise for columns, so
 * the layer is one 2x2, pad-1 convolution of the low-res input x [batch, h, w, c] with the four phase-folded filters
 * stacked along the output channels, y4 [batch, h+1, w+1, 4c] (phase k = 2a+b of pixel (i, j) at (i+a, j+b),
 * channels k*c..k*c+c-1): 16 instead of 36 multiply-adds per (output pixel, cin, cout).
 * rtti_upsample_phase_interleave: out [batch, 2h, 2w, c] = y4 re-ordered to pixels + bias[c] (bias may be NULL).
 * rtti_upsample_phase_scatter: its adjoint, g [batch, 2h, 2w, c] -> dy4 [batch, h+1, w+1, 4c] (zero where the
 * interleave reads nothing). fp32, c a multiple of 4, 16-byte aligned. */
int rtti_upsample_phase_interleave(const float* y4, const float* bias, float* out, int batch, int h, int w, int c,
                                   void* stream);
int rtti_upsample_phase_scatter(const float* g, float* dy4, int batch, int h, int w, int c, void* stream);
/* out[rows, c] = a + b + bias[c] (fp32): the residual add of a VAE resnet block fused with the bias of the
 * convolution that produced b; bias may be NULL. */
int rtti_add_bias_f32(const float* a, const float* b, const float* bias, float* out, long long rows, int c,
                      void* stream);

/* Multi-GPU region parallelism (new relative to the single-GPU reference loop,
 * models/region_diffusion_sdxl.py:779-845): fused all-gather + region blend + CFG + Euler update over NVLink
 * peer memory. Every rank calls it once per step on its own stream after writing the noise predictions of
 * the passes it owns into its slot buffer.
 *   peer_slots (host, [world]): device pointers, valid on THIS device, to each rank's slot buffer
 *       fp16 [2 (step parity)][n_slots][n]; slot 0 = unconditional pass, slots 1..n_regions = region passes
 *       in mask order (base-prompt pass last), slot n_regions+1 / +2 = reference-latent uncond / base passes.
 *   peer_flags (host, [world]): device pointers to each rank's uint32 step counter (zero-initialised).
 *   slot_owner (host, [n_slots]): rank that writes slot s.  step_id: 1, 2, 3, ... identical on all ranks.
 *   Outputs are written locally on every rank (replicated, bit-identical): eps_out [n]; latents_out =
 *   latents + dt_sigma*eps; latents_ref_out = latents_ref + dt_sigma*(eps_C + guidance*(eps_D - eps_C)).
 *   latents/latents_out and latents_ref/latents_ref_out may be NULL pairs.
 */
int rtti_gather_blend_step(const void* const* peer_slots, void* const* peer_flags, int world, int rank,
                           const int* slot_owner, int n_slots, int n_regions, const float* masks, long long n,
                           float guidance, void* eps_out, const void* latents, void* latents_out,
                           const void* latents_ref, void* latents_ref_out, float dt_sigma, unsigned int step_id,
                           void* stream);
/* rtti_gather_blend_step with the CFG rescale of rtti_region_blend_cfg_rescale, same protocol and slot layout. The
 * reference-latent pair, when latents_ref is given, is rescaled on its own statistics (eps_t = eps_D,
 * eps_cfg = eps_C + guidance * (eps_D - eps_C)). For the same noise predictions the outputs equal those of
 * rtti_region_blend_cfg_rescale (the C/D pair: called with one region and a mask of ones) bit for bit, whatever the
 * world size. n a multiple of 8 and <= 262144 (RTTI_ERR_SHAPE otherwise); masks and outputs 16-byte aligned. */
int rtti_gather_blend_step_rescale(const void* const* peer_slots, void* const* peer_flags, int world, int rank,
                                   const int* slot_owner, int n_slots, int n_regions, const float* masks, long long n,
                                   float guidance, void* eps_out, const void* latents, void* latents_out,
                                   const void* latents_ref, void* latents_ref_out, float dt_sigma,
                                   unsigned int step_id, float guidance_rescale, void* stream);

/* Multistep forms of the two gather entry points (see rtti_region_blend_cfg_ms). The reference-latent trajectory, when
 * latents_ref is given, is stepped with the same coefficients on its own history (d_prev_ref -> d_out_ref, required
 * then), so each trajectory keeps its own D. For the same noise predictions the outputs equal those of the single-GPU
 * forms (the C/D pair: one region and a mask of ones) bit for bit, whatever the world size. */
int rtti_gather_blend_step_ms(const void* const* peer_slots, void* const* peer_flags, int world, int rank,
                              const int* slot_owner, int n_slots, int n_regions, const float* masks, long long n,
                              float guidance, void* eps_out, const void* latents, void* latents_out,
                              const void* latents_ref, void* latents_ref_out, float hx, float he, float cx, float cd,
                              float cp, const float* d_prev, float* d_out, const float* d_prev_ref, float* d_out_ref,
                              unsigned int step_id, void* stream);
int rtti_gather_blend_step_rescale_ms(const void* const* peer_slots, void* const* peer_flags, int world, int rank,
                                      const int* slot_owner, int n_slots, int n_regions, const float* masks,
                                      long long n, float guidance, void* eps_out, const void* latents,
                                      void* latents_out, const void* latents_ref, void* latents_ref_out, float hx,
                                      float he, float cx, float cd, float cp, const float* d_prev, float* d_out,
                                      const float* d_prev_ref, float* d_out_ref, unsigned int step_id,
                                      float guidance_rescale, void* stream);

/* Ancestral forms of rtti_gather_blend_step / rtti_gather_blend_step_rescale (the update of rtti_region_blend_cfg_anc).
 * Both trajectories take the same dt_sigma and s_up; the reference latents take their own noise z_ref[n], required
 * (16-byte aligned) when latents_ref is given and s_up != 0. Same protocol and slot layout as the Euler forms. */
int rtti_gather_blend_step_anc(const void* const* peer_slots, void* const* peer_flags, int world, int rank,
                               const int* slot_owner, int n_slots, int n_regions, const float* masks, long long n,
                               float guidance, void* eps_out, const void* latents, void* latents_out,
                               const void* latents_ref, void* latents_ref_out, float dt_sigma, float s_up,
                               const void* z, const void* z_ref, unsigned int step_id, void* stream);
int rtti_gather_blend_step_rescale_anc(const void* const* peer_slots, void* const* peer_flags, int world, int rank,
                                       const int* slot_owner, int n_slots, int n_regions, const float* masks,
                                       long long n, float guidance, void* eps_out, const void* latents,
                                       void* latents_out, const void* latents_ref, void* latents_ref_out,
                                       float dt_sigma, float s_up, const void* z, const void* z_ref,
                                       unsigned int step_id, float guidance_rescale, void* stream);

/* UniPC forms of rtti_gather_blend_step / rtti_gather_blend_step_rescale (the update of rtti_region_blend_cfg_unipc).
 * The reference-latent trajectory, when latents_ref is given, is stepped with the same coefficients on its own three
 * histories (xl_ref, m1_ref, m2_ref -> m_out_ref, xl_out_ref, with the requirements of the main ones). For the same
 * noise predictions the outputs equal those of the single-GPU forms (the C/D pair: one region and a mask of ones) bit
 * for bit, whatever the world size. Same protocol and slot layout as the Euler forms. */
int rtti_gather_blend_step_unipc(const void* const* peer_slots, void* const* peer_flags, int world, int rank,
                                 const int* slot_owner, int n_slots, int n_regions, const float* masks, long long n,
                                 float guidance, void* eps_out, const void* latents, void* latents_out,
                                 const void* latents_ref, void* latents_ref_out, float hx, float he, float ux, float ul,
                                 float u0, float u1, float u2, float vx, float v0, float v1, const float* xl,
                                 const float* m1, const float* m2, float* m_out, float* xl_out, const float* xl_ref,
                                 const float* m1_ref, const float* m2_ref, float* m_out_ref, float* xl_out_ref,
                                 unsigned int step_id, void* stream);
int rtti_gather_blend_step_rescale_unipc(const void* const* peer_slots, void* const* peer_flags, int world, int rank,
                                         const int* slot_owner, int n_slots, int n_regions, const float* masks,
                                         long long n, float guidance, void* eps_out, const void* latents,
                                         void* latents_out, const void* latents_ref, void* latents_ref_out, float hx,
                                         float he, float ux, float ul, float u0, float u1, float u2, float vx,
                                         float v0, float v1, const float* xl, const float* m1, const float* m2,
                                         float* m_out, float* xl_out, const float* xl_ref, const float* m1_ref,
                                         const float* m2_ref, float* m_out_ref, float* xl_out_ref,
                                         unsigned int step_id, float guidance_rescale, void* stream);

/* Heun forms of rtti_gather_blend_step / rtti_gather_blend_step_rescale (the update of rtti_region_blend_cfg_heun;
 * they replace models/region_diffusion_sdxl.py:837-846 with a HeunDiscreteScheduler assigned to the reference's
 * scheduler). The reference-latent trajectory, when latents_ref is given, is stepped with the same coefficients on its
 * own saved state xs_ref / ds_ref (with the requirements of xs / ds). eps_ref_out[n], optional (null: not written;
 * given without latents_ref: RTTI_ERR_ARG; 16-byte aligned), receives that trajectory's fp16-rounded (rescaled) noise
 * prediction, the eps_out of the single-GPU form called on the C/D pair with one region and a mask of ones: its ds for
 * the next second stage. For the same noise predictions the outputs equal those of the single-GPU forms bit for bit,
 * whatever the world size. Same protocol and slot layout as the Euler forms. */
int rtti_gather_blend_step_heun(const void* const* peer_slots, void* const* peer_flags, int world, int rank,
                                const int* slot_owner, int n_slots, int n_regions, const float* masks, long long n,
                                float guidance, void* eps_out, const void* latents, void* latents_out,
                                const void* latents_ref, void* latents_ref_out, float cx, float ce, float cs, float cd,
                                const void* xs, const void* ds, const void* xs_ref, const void* ds_ref,
                                void* eps_ref_out, unsigned int step_id, void* stream);
int rtti_gather_blend_step_rescale_heun(const void* const* peer_slots, void* const* peer_flags, int world, int rank,
                                        const int* slot_owner, int n_slots, int n_regions, const float* masks,
                                        long long n, float guidance, void* eps_out, const void* latents,
                                        void* latents_out, const void* latents_ref, void* latents_ref_out, float cx,
                                        float ce, float cs, float cd, const void* xs, const void* ds,
                                        const void* xs_ref, const void* ds_ref, void* eps_ref_out,
                                        unsigned int step_id, float guidance_rescale, void* stream);

/* LMS forms of rtti_gather_blend_step / rtti_gather_blend_step_rescale (the update of rtti_region_blend_cfg_lms; they
 * replace models/region_diffusion_sdxl.py:837-846 with an LMSDiscreteScheduler assigned to the reference's scheduler).
 * The reference-latent trajectory, when latents_ref is given, is stepped with the same coefficients on its own history
 * d1_ref / d2_ref / d3_ref (with the requirements of d1 / d2 / d3). eps_ref_out[n], optional (null: not written; given
 * without latents_ref: RTTI_ERR_ARG; 16-byte aligned), receives that trajectory's fp16-rounded (rescaled) noise
 * prediction, the eps_out of the single-GPU form called on the C/D pair with one region and a mask of ones: the newest
 * entry of its history for the next step. For the same noise predictions the outputs equal those of the single-GPU
 * forms bit for bit, whatever the world size. Same protocol and slot layout as the Euler forms. */
int rtti_gather_blend_step_lms(const void* const* peer_slots, void* const* peer_flags, int world, int rank,
                               const int* slot_owner, int n_slots, int n_regions, const float* masks, long long n,
                               float guidance, void* eps_out, const void* latents, void* latents_out,
                               const void* latents_ref, void* latents_ref_out, float c0, float c1, float c2, float c3,
                               const void* d1, const void* d2, const void* d3, const void* d1_ref, const void* d2_ref,
                               const void* d3_ref, void* eps_ref_out, unsigned int step_id, void* stream);
int rtti_gather_blend_step_rescale_lms(const void* const* peer_slots, void* const* peer_flags, int world, int rank,
                                       const int* slot_owner, int n_slots, int n_regions, const float* masks,
                                       long long n, float guidance, void* eps_out, const void* latents,
                                       void* latents_out, const void* latents_ref, void* latents_ref_out, float c0,
                                       float c1, float c2, float c3, const void* d1, const void* d2, const void* d3,
                                       const void* d1_ref, const void* d2_ref, const void* d3_ref, void* eps_ref_out,
                                       unsigned int step_id, float guidance_rescale, void* stream);

/* Singlestep forms of rtti_gather_blend_step / rtti_gather_blend_step_rescale (the update of rtti_region_blend_cfg_ss;
 * they replace models/region_diffusion_sdxl.py:837-846 with a DPMSolverSinglestepScheduler assigned to the reference's
 * scheduler). The reference-latent trajectory, when latents_ref is given, is stepped with the same coefficients on its
 * own state d_prev_ref -> d_out_ref and xs_ref (with the requirements of d_prev / d_out / xs). For the same noise
 * predictions the outputs equal those of the single-GPU forms (the C/D pair: one region and a mask of ones) bit for
 * bit, whatever the world size. Same protocol and slot layout as the Euler forms. */
int rtti_gather_blend_step_ss(const void* const* peer_slots, void* const* peer_flags, int world, int rank,
                              const int* slot_owner, int n_slots, int n_regions, const float* masks, long long n,
                              float guidance, void* eps_out, const void* latents, void* latents_out,
                              const void* latents_ref, void* latents_ref_out, float hx, float he, float cx, float cs,
                              float cd, float cp, const float* d_prev, float* d_out, const void* xs,
                              const float* d_prev_ref, float* d_out_ref, const void* xs_ref, unsigned int step_id,
                              void* stream);
int rtti_gather_blend_step_rescale_ss(const void* const* peer_slots, void* const* peer_flags, int world, int rank,
                                      const int* slot_owner, int n_slots, int n_regions, const float* masks,
                                      long long n, float guidance, void* eps_out, const void* latents,
                                      void* latents_out, const void* latents_ref, void* latents_ref_out, float hx,
                                      float he, float cx, float cs, float cd, float cp, const float* d_prev,
                                      float* d_out, const void* xs, const float* d_prev_ref, float* d_out_ref,
                                      const void* xs_ref, unsigned int step_id, float guidance_rescale, void* stream);

/* Stripe-parallel colour guidance (multi-GPU; new relative to the single-GPU reference, which back-propagates
 * through the batch-1 VAE decoder on one device: models/region_diffusion_sdxl.py:849-867). Every activation of
 * the decoder's up-blocks is split by image rows over `world` ranks.
 *
 * rtti_gn32_silu_fwd/bwd_striped: GroupNorm(+SiLU) over a tensor of hw_total rows of which x holds this rank's
 *   hw_local rows (batch 1, groups <= 32). The statistics are reduced through peer memory inside the call:
 *   peer_sums (host, [world]): device pointers to each rank's fp32 [2 (seq parity)][3*groups] slot (forward: the
 *   rank's element count, mean and sum of squared deviations per group, merged in rank order; backward: two sums);
 *   peer_flags (host, [world]): device pointers to each rank's uint32[9] {sequence, error, -, ..., [8] sequence base}
 *   words (zero-initialised);
 *   seq: 1, 2, 3, ... the same on every rank for the same call; the kernels add the local rank's sequence base word
 *   to it (0 unless rtti_peer_seq_advance was called). All ranks obtain bit-identical statistics.
 *   workspace: fp32 [rtti_gn32_workspace_elems(1, hw_local, c, groups)].
 * rtti_halo_exchange: pad_local is this rank's conv input [1 + rows + 1][row_elems] fp32 with the interior rows
 *   already written; pushes the first / last interior row into the bottom / top halo row of pad_up / pad_down
 *   (peer-mapped pointers to the neighbours' buffers of the same shape; NULL at the image border, where the own
 *   halo row is zeroed instead), then waits until both neighbours have pushed theirs.
 *   flags_*: uint32[9] per rank {from_up, from_down, error, arrival counter, -, -, -, -, sequence base}, zero-initialised,
 *   peer-mapped; the effective sequence number is seq + flags_local[8].
 * rtti_peer_seq_advance: flags_a[8] += da; flags_b[8] += db (either pointer may be NULL), stream-ordered. A caller that
 *   numbers the exchanges of one colour-guidance evaluation 1..n and advances the bases by n afterwards passes the same
 *   arguments every evaluation, so the evaluation can be captured ONCE in a CUDA graph and replayed (the sequence numbers
 *   the ranks compare stay monotonic because the base lives in device memory).
 */
int rtti_gn32_silu_fwd_striped(const float* x, const float* chan_bias, const float* gamma, const float* beta, float* y,
                               float* mean_rstd, float* workspace, int hw_local, long long hw_total, int c, int groups,
                               float eps, int apply_silu, void* const* peer_sums, void* const* peer_flags, int world,
                               int rank, unsigned int seq, void* stream);
int rtti_gn32_silu_bwd_striped(const float* x, const float* chan_bias, const float* dz, const float* gamma,
                               const float* beta, const float* mean_rstd, float* dx, float* workspace, int hw_local,
                               long long hw_total, int c, int groups, int apply_silu, void* const* peer_sums,
                               void* const* peer_flags, int world, int rank, unsigned int seq, void* stream);
int rtti_halo_exchange(float* pad_local, float* pad_up, float* pad_down, int rows, long long row_elems,
                       void* flags_local, void* flags_up, void* flags_down, unsigned int seq, void* stream);
int rtti_peer_seq_advance(void* flags_a, unsigned int da, void* flags_b, unsigned int db, void* stream);

/* Producer -> consumers hand-off of one activation over peer memory (multi-GPU; new relative to the single-GPU
 * reference). On feature-injection steps the region passes consume the self-attention Q, K of the reference pass D in
 * every layer and one resnet feature map (models/region_diffusion_sdxl.py:1018-1061, models/resnet.py:639-641); with the
 * passes sharded over ranks, the rank that runs D pushes them to the ranks that run region passes.
 * rtti_peer_push: copy rows x row_bytes (row stride src_row_stride_bytes; 16-byte multiples) into dst[0..n_dst) (host
 *   array of peer-mapped pointers, n_dst <= 15), then publish event number seq + flags_local[8] to dst_flags[d][0].
 *   flags_local: uint32[9] {-, error, -, arrival counter, ..., [8] sequence base}, zero-initialised.
 * rtti_peer_wait: stream-ordered wait until flags_local[0] >= seq + flags_local[8] (~4 s timeout -> flags_local[1] =
 *   0xDEAD, after which waits return immediately). Events are numbered 1, 2, ... within one UNet pass and the base is
 *   advanced with rtti_peer_seq_advance at its end, so both calls are CUDA-graph replayable.
 */
int rtti_peer_push(const void* src, long long src_row_stride_bytes, int rows, int row_bytes, void* const* dst,
                   void* const* dst_flags, int n_dst, void* flags_local, unsigned int seq, void* stream);
int rtti_peer_wait(void* flags_local, unsigned int seq, void* stream);

/* k-means of the spectral embedding of the token-map affinity: the KMeans(n_clusters, n_init) that scikit-learn's
 * SpectralClustering(affinity="precomputed", assign_labels="kmeans") runs (utils/attention_utils.py:262-265), all
 * restarts in one launch (one CTA each). Each restart is k-means++ seeding followed by Lloyd iterations, step for step
 * as scikit-learn's dense KMeans.fit: centring on the column means, n_local_trials = 2 + floor(ln k), candidates drawn
 * from the float32 cumulative sum of the float64-formed squared distances (searchsorted side='left', clipped to n-1),
 * the candidate of lowest potential kept (first on a tie); nearest centre by ||c||^2 - 2 x.c (first on a tie), empty
 * clusters relocated to the farthest samples, stop when the labels repeat, when the summed squared centre shift is
 * <= tol * mean(var(x, axis=0)), or after max_iter, then a final assignment unless the labels repeated.
 *   x [n, k] fp32 row-major; 1 <= k <= 32, k <= n <= 4096 and 4*n*(k+2) + 18 KB <= 227 KB of shared memory
 *   (n = 4096 allows k <= 11; RTTI_ERR_SHAPE otherwise).
 *   draws [n_init, 1 + (k-1)*(2 + floor(ln k))] fp64: per restart the index of the first centre, then the uniforms
 *   in [0, 1) of the k-1 k-means++ steps, as scikit-learn takes them from its RandomState.
 *   labels [n_init, n] int32, inertia [n_init] fp64 (sum of squared distances to the assigned centres), n_iter [n_init]
 *   int32: per restart. Choosing among restarts is left to the caller.
 *   flags [n_init] int32: bit 0 set when the restart relocated empty clusters in a step where scikit-learn's choice is
 *   left to np.argpartition's unspecified order (two or more clusters empty at once, or distinct samples tied at the
 *   largest distance); that restart's labels may then differ from scikit-learn's by a renaming.
 *   n_init >= 1, max_iter >= 1, tol >= 0 (RTTI_ERR_ARG otherwise). Deterministic (no atomics).
 * rtti_kmeans_supported: host-only query, RTTI_OK when rtti_kmeans_fit accepts (n, k), RTTI_ERR_SHAPE otherwise.
 */
int rtti_kmeans_fit(const float* x, const double* draws, int n, int k, int n_init, int max_iter, double tol,
                    int* labels, double* inertia, int* n_iter, int* flags, void* stream);
int rtti_kmeans_supported(int n, int k);

#ifdef __cplusplus
}
#endif
#endif /* RTTI_B200_H */
