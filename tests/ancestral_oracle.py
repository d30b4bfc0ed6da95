"""TEST INFRASTRUCTURE — restatement of diffusers 0.18.2's EulerAncestralDiscreteScheduler (epsilon prediction, the
SDXL config) in the form diffusers evaluates it, for the oracle loops and for tests/gen_ancestral.py.

PARITY UNPINNED: the diffusers source is not available here (the reference pins diffusers==0.18.2, environment.yaml).
The arithmetic follows that version's `schedulers/scheduling_euler_ancestral_discrete.py` step by step (fp32 torch
sigmas, pred_original_sample, derivative, sigma_up / sigma_down, randn_tensor), independently of the product's
`ancestral_coeffs`. The grid is oracle/schedulers_oracle.py's Euler grid. The same class is assigned to `m.scheduler` of
the unmodified reference by tests/gen_ancestral.py, so what the goldens pin is the reference's loop logic — which
scheduler calls it makes, with which shapes and in which order — with this scheduler.

Noise: z is drawn in fp16 (what diffusers' randn_tensor draws for the fp16 SDXL UNet's prediction; the reference runs
in fp32 on the CPU here) and then computed with in the prediction's dtype. Its source, in order: the `generator` the
caller passes to `step` (the reference's plain pass forwards `sample(generator=...)`), else the scheduler's own
`generator` (the reference's rich-text pass passes none: a seeded CPU generator stands in for the global RNG), else the
next tensor of `noises` (draws recorded on the GPU), else the global CPU RNG.
"""
import torch

from oracle import sampler_oracle as sam
from oracle import schedulers_oracle as so


class EulerAncestralSchedulerOracle(so.EulerDiscreteSchedulerOracle):
    def __init__(self, generator=None, noises=None):
        super().__init__()
        self.generator = generator
        self.noises = list(noises) if noises is not None else None
        self.draw_shapes = []

    def _noise(self, shape, dtype, device, generator):
        self.draw_shapes.append(tuple(shape))
        g = generator if generator is not None else self.generator
        if g is None and self.noises is not None:
            z = self.noises.pop(0)
            assert tuple(z.shape) == tuple(shape), (tuple(z.shape), tuple(shape))
            return z.to(device, dtype)
        return torch.randn(shape, dtype=torch.float16, generator=g).to(device, dtype)

    def step(self, model_output, timestep, sample, generator=None, return_dict=True, **kw):
        i = self._index(timestep)
        sigma = self.sigmas[i]
        pred_original_sample = sample - sigma * model_output
        sigma_from, sigma_to = self.sigmas[i], self.sigmas[i + 1]
        sigma_up = (sigma_to ** 2 * (sigma_from ** 2 - sigma_to ** 2) / sigma_from ** 2) ** 0.5
        sigma_down = (sigma_to ** 2 - sigma_up ** 2) ** 0.5
        derivative = (sample - pred_original_sample) / sigma
        dt = sigma_down - sigma
        prev_sample = sample + derivative * dt
        noise = self._noise(model_output.shape, model_output.dtype, model_output.device, generator)
        prev_sample = prev_sample + noise * sigma_up
        return {"prev_sample": prev_sample, "pred_original_sample": pred_original_sample} if return_dict \
            else (prev_sample,)


def plain_loop(unet, scheduler, text_embeddings, latents, num_inference_steps, guidance_scale, added_cond=None,
               generator=None):
    """oracle/sampler_oracle.py's XL plain loop with `generator` forwarded to every step (:908), from the latents as the
    reference's prepare_latents hands them over (scaled by init_noise_sigma)."""
    scheduler.set_timesteps(num_inference_steps)
    latents = latents * scheduler.init_noise_sigma
    for t in scheduler.timesteps:
        x = scheduler.scale_model_input(torch.cat([latents] * 2), t)
        with torch.no_grad():
            eps = unet(x, t, text_embeddings, added_cond, None)
        eu, et = eps.chunk(2)
        noise_pred = eu + guidance_scale * (et - eu)
        latents = scheduler.step(noise_pred, t, latents, generator=generator)["prev_sample"]
    return latents


def rich_text_loop(unet, scheduler, text_embeddings, masks, latents, num_inference_steps, *a, **kw):
    """oracle/sampler_oracle.py's rich-text loop (one scheduler, the joint batch-2 step of the reference, :831-846), from
    the latents scaled by init_noise_sigma as in plain_loop (the reference sets the timesteps before it scales them)."""
    scheduler.set_timesteps(num_inference_steps)
    return sam.rich_text_loop(unet, scheduler, text_embeddings, masks, latents * scheduler.init_noise_sigma,
                              num_inference_steps, *a, **kw)
