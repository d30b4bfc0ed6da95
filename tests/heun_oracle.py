"""TEST INFRASTRUCTURE — restatement of diffusers 0.18.2's HeunDiscreteScheduler (epsilon prediction, the SDXL config,
no Karras sigmas) in the form diffusers evaluates it, for the oracle loops and for tests/gen_heun.py.

PARITY UNPINNED: the diffusers source is not available here (the reference pins diffusers==0.18.2, environment.yaml).
The arithmetic follows that version's `schedulers/scheduling_heun_discrete.py` step by step (fp32 torch sigmas,
index_for_timestep with its first-/second-order position rule, sigma_hat with gamma = 0, pred_original_sample,
derivative, the saved prev_derivative / dt / sample), independently of the product's `heun_coeffs`. The grid is
oracle/schedulers_oracle.py's Euler grid (`leading` spacing, steps_offset 1), interleaved. The same class is assigned to
`m.scheduler` of the unmodified reference by tests/gen_heun.py, so what the goldens pin is the reference's loop logic —
which scheduler calls it makes, in which order, and when it calls back — with this scheduler.
"""
import torch

from oracle import sampler_oracle as sam
from oracle import schedulers_oracle as so


class HeunSchedulerOracle:
    order = 2

    def __init__(self):
        self._euler = so.EulerDiscreteSchedulerOracle()
        self.alphas_cumprod = self._euler.alphas_cumprod
        self.sigmas, self.timesteps = self._euler.sigmas, self._euler.timesteps
        self.prev_derivative = self.dt = self.sample = None
        self.step_batches = []   # the batch size of every step call, in order

    @property
    def init_noise_sigma(self):
        return (self.sigmas.max() ** 2 + 1) ** 0.5

    def set_timesteps(self, num_inference_steps, device=None):
        e = self._euler
        e.set_timesteps(num_inference_steps)
        self.num_inference_steps = num_inference_steps
        self.sigmas = torch.cat([e.sigmas[:1], e.sigmas[1:-1].repeat_interleave(2), e.sigmas[-1:]])
        self.timesteps = torch.cat([e.timesteps[:1], e.timesteps[1:].repeat_interleave(2)])
        self.prev_derivative = self.dt = self.sample = None

    @property
    def state_in_first_order(self):
        return self.dt is None

    def index_for_timestep(self, timestep):
        indices = (self.timesteps == timestep).nonzero()
        pos = -1 if self.state_in_first_order else 0
        return int(indices[pos].item())

    def scale_model_input(self, sample, timestep):
        sigma = self.sigmas[self.index_for_timestep(timestep)]
        return sample / ((sigma ** 2 + 1) ** 0.5)

    def step(self, model_output, timestep, sample, return_dict=True, **kw):
        self.step_batches.append(int(sample.shape[0]))
        step_index = self.index_for_timestep(timestep)
        if self.state_in_first_order:
            sigma, sigma_next = self.sigmas[step_index], self.sigmas[step_index + 1]
        else:
            sigma, sigma_next = self.sigmas[step_index - 1], self.sigmas[step_index]
        sigma_hat = sigma * (0 + 1)   # gamma = 0
        sigma_input = sigma_hat if self.state_in_first_order else sigma_next
        pred_original_sample = sample - sigma_input * model_output
        if self.state_in_first_order:
            derivative = (sample - pred_original_sample) / sigma_hat
            dt = sigma_next - sigma_hat
            self.prev_derivative, self.dt, self.sample = derivative, dt, sample
        else:
            derivative = (sample - pred_original_sample) / sigma_next
            derivative = (self.prev_derivative + derivative) / 2
            dt, sample = self.dt, self.sample
            self.prev_derivative = self.dt = self.sample = None
        prev_sample = sample + derivative * dt
        return {"prev_sample": prev_sample, "pred_original_sample": pred_original_sample} if return_dict \
            else (prev_sample,)


class PerTrajectoryHeunOracle(HeunSchedulerOracle):
    """The product's rule for the rich-text loop: a batch-2 step (main, reference) steps each trajectory on its own
    HeunSchedulerOracle, a batch-1 step the main one alone. Where the reference loop steps both jointly on every
    iteration it equals one batch-2 scheduler; where it stops stepping the reference latents right after a first stage,
    the reference latents keep their first-stage value here instead of meeting a batch-2 saved state."""

    def __init__(self):
        super().__init__()
        self.main, self.ref = HeunSchedulerOracle(), HeunSchedulerOracle()

    def set_timesteps(self, num_inference_steps, device=None):
        super().set_timesteps(num_inference_steps, device)
        self.main.set_timesteps(num_inference_steps, device)
        self.ref.set_timesteps(num_inference_steps, device)

    def scale_model_input(self, sample, timestep):
        return self.main.scale_model_input(sample, timestep)

    def step(self, model_output, timestep, sample, return_dict=True, **kw):
        self.step_batches.append(int(sample.shape[0]))
        out = self.main.step(model_output[:1], timestep, sample[:1])["prev_sample"]
        if sample.shape[0] == 2:
            out = torch.cat([out, self.ref.step(model_output[1:], timestep, sample[1:])["prev_sample"]])
        return {"prev_sample": out} if return_dict else (out,)


def plain_loop(unet, scheduler, text_embeddings, latents, num_inference_steps, guidance_scale, added_cond=None):
    """oracle/sampler_oracle.py's XL plain loop from the latents as the reference's prepare_latents hands them over
    (scaled by init_noise_sigma, after set_timesteps)."""
    scheduler.set_timesteps(num_inference_steps)
    return sam.plain_loop(unet, scheduler, text_embeddings, latents * scheduler.init_noise_sigma, num_inference_steps,
                          guidance_scale, xl=True, added_cond=added_cond)


def rich_text_loop(unet, scheduler, text_embeddings, masks, latents, num_inference_steps, *a, **kw):
    """oracle/sampler_oracle.py's rich-text loop (one scheduler, the joint batch-2 step of the reference, :831-846), from
    the latents scaled by init_noise_sigma as in plain_loop."""
    scheduler.set_timesteps(num_inference_steps)
    return sam.rich_text_loop(unet, scheduler, text_embeddings, masks, latents * scheduler.init_noise_sigma,
                              num_inference_steps, *a, **kw)


def callback_iterations(n_iterations, num_inference_steps, order, callback_steps):
    """The reference's callback rule (models/region_diffusion_sdxl.py:770, :874-877, :910-914)."""
    num_warmup_steps = n_iterations - num_inference_steps * order
    return [i for i in range(n_iterations)
            if (i == n_iterations - 1 or ((i + 1) > num_warmup_steps and (i + 1) % order == 0)) and i % callback_steps == 0]
