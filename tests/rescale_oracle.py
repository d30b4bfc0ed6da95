"""TEST INFRASTRUCTURE — CPU fp32 restatement of the SDXL sampling loops with guidance_rescale.

`rescale_noise_cfg` restates models/region_diffusion_sdxl.py:42-53. The loops are oracle/sampler_oracle.py's
plain_loop / rich_text_loop with the rescale applied where the reference applies it (plain pass, :903-905) or leaves it
as a TODO (rich pass, :827-830), only when guidance_scale > 1 and guidance_rescale > 0:
  - plain pass: eps_text = the cond prediction, eps_cfg = the CFG result;
  - rich pass: eps_text = the blended text prediction sum_j m_j eps_j, eps_cfg = the blended CFG result;
  - the reference-latent pair, when it is stepped: eps_text = eps_D, eps_cfg = eps_C + g (eps_D - eps_C).
The rescaled prediction is what the scheduler steps and what colour guidance's predict_x0 sees. With
guidance_rescale = 0 both loops compute exactly what oracle/sampler_oracle.py computes. Pinned against the unmodified
reference by tests/golden/xl_rescale.npz (tests/gen_xl_rescale.py)."""
import torch

from oracle import sampler_oracle as sam


def rescale_noise_cfg(noise_cfg, noise_pred_text, guidance_rescale=0.0):
    """Per batch entry: noise_cfg * (phi * std(text) / std(cfg) + 1 - phi), unbiased std over all other dims."""
    dims = list(range(1, noise_pred_text.ndim))
    std_text = noise_pred_text.std(dim=dims, keepdim=True)
    std_cfg = noise_cfg.std(dim=dims, keepdim=True)
    return guidance_rescale * (noise_cfg * (std_text / std_cfg)) + (1 - guidance_rescale) * noise_cfg


def _on(guidance_scale, guidance_rescale):
    return guidance_scale > 1.0 and guidance_rescale > 0.0


def plain_loop(unet, scheduler, text_embeddings, latents, num_inference_steps, guidance_scale, xl, added_cond=None,
               ctrl=None, guidance_rescale=0.0):
    """sam.plain_loop + rescale_noise_cfg(noise_pred, eps_text) (region_diffusion_sdxl.py:899-905)."""
    scheduler.set_timesteps(num_inference_steps)
    for t in scheduler.timesteps:
        x = torch.cat([latents] * 2)
        if xl:
            x = scheduler.scale_model_input(x, t)
        with torch.no_grad():
            eps = unet(x, t, text_embeddings, added_cond, ctrl)
        eu, et = eps.chunk(2)
        noise_pred = eu + guidance_scale * (et - eu)
        if _on(guidance_scale, guidance_rescale):
            noise_pred = rescale_noise_cfg(noise_pred, et, guidance_rescale)
        latents = scheduler.step(noise_pred, t, latents)["prev_sample"]
    return latents


def rich_text_loop(unet, scheduler, text_embeddings, masks, latents, num_inference_steps, guidance_scale,
                   added_cond=None, use_guidance=False, text_format_dict=None, inject_selfattn=0.0, inject_background=0.0,
                   vae_decode=None, scaling_factor=0.18215, guidance_rescale=0.0):
    """sam.rich_text_loop (xl=True, region_diffusion_sdxl.py:772-878) with the rescale of the blended prediction and of
    the reference-latent pair."""
    tfd = text_format_dict or {}
    scheduler.set_timesteps(num_inference_steps)
    timesteps = scheduler.timesteps
    inject = inject_selfattn > 0 or inject_background > 0
    latents_reference = latents.clone() if inject else None
    n_t = len(timesteps)
    rescale = _on(guidance_scale, guidance_rescale)

    def added(rows):
        if added_cond is None:
            return None
        return {"text_embeds": added_cond["text_embeds"][rows], "time_ids": added_cond["time_ids"][:1]}

    last = text_embeddings.shape[0] - 1
    for i, t in enumerate(timesteps):
        feat_inject_step = bool(t > (1 - inject_selfattn) * 1000)
        background_inject_step = i < inject_background * n_t
        with torch.no_grad():
            x_in = scheduler.scale_model_input(latents, t)
            eps_u = unet(x_in, t, text_embeddings[:1], added(slice(0, 1)), None)
            eps_text_cur = unet(x_in, t, text_embeddings[-1:], added(slice(last, last + 1)), sam.FontSizeControl(tfd))
            if inject:
                xr_in = scheduler.scale_model_input(latents_reference, t)
                eps_u_ref = unet(xr_in, t, text_embeddings[:1], added(slice(0, 1)), None)
                store = sam.SelfAttnStore(feat_inject_step)
                eps_t_ref = unet(xr_in, t, text_embeddings[-1:], added(slice(last, last + 1)), store)
            noise_pred_uncond = eps_u * masks[-1]
            noise_pred_text = eps_text_cur * masks[-1]
            for j, mask in enumerate(masks[:-1]):
                ctrl = sam.ReplaceControl(feat_inject_step, store.store) if inject else None
                eps_j = unet(x_in, t, text_embeddings[j + 1:j + 2], added(slice(j + 1, j + 2)), ctrl)
                noise_pred_uncond = noise_pred_uncond + eps_u * mask
                noise_pred_text = noise_pred_text + eps_j * mask
            noise_pred = noise_pred_uncond + guidance_scale * (noise_pred_text - noise_pred_uncond)
            if rescale:
                noise_pred = rescale_noise_cfg(noise_pred, noise_pred_text, guidance_rescale)
            if inject_selfattn > 0 or background_inject_step > 0:
                noise_pred_refer = eps_u_ref + guidance_scale * (eps_t_ref - eps_u_ref)
                if rescale:
                    noise_pred_refer = rescale_noise_cfg(noise_pred_refer, eps_t_ref, guidance_rescale)
                both = scheduler.step(torch.cat([noise_pred, noise_pred_refer]), t,
                                      torch.cat([latents, latents_reference]))["prev_sample"]
                latents, latents_reference = torch.chunk(both, 2, dim=0)
            else:
                latents = scheduler.step(noise_pred, t, latents)["prev_sample"]
        if use_guidance and bool(t < tfd["guidance_start_step"]):
            latents = sam.color_guidance(latents, noise_pred, t, scheduler.alphas_cumprod, vae_decode, scaling_factor, tfd,
                                         True)
        if (i == int(inject_background * n_t)) and inject_background > 0:
            latents = latents_reference * masks[-1] + latents * (1 - masks[-1])
    return latents
