"""TEST INFRASTRUCTURE — restatement of diffusers 0.18.2's DDIMScheduler (eta = 0) and DPMSolverMultistepScheduler
(DPM-Solver++(2M)) in the form diffusers evaluates them, and the sampling loops that drive them.

PARITY UNPINNED: the diffusers sources are not available here (the reference pins diffusers==0.18.2,
environment.yaml). The arithmetic below follows that version's `schedulers/scheduling_ddim.py` and
`schedulers/scheduling_dpmsolver_multistep.py` step by step (fp32 torch, `exp(-h) - 1`, the stateful model-output
list and lower_order_nums counter), independently of the product's closed-form `step_coeffs`. The same classes are
assigned to `m.scheduler` of the unmodified reference by tests/gen_multistep.py, so what the goldens pin is the
reference's loop logic with these schedulers.

Loops: `plain_loop` is oracle/sampler_oracle.py's (the schedulers' scale_model_input is the identity). `rich_text_loop`
is sampler_oracle's xl loop with one scheduler state per trajectory: the main latents step on `scheduler`, the
reference latents on `scheduler_ref`. When the reference latents are stepped on every step (inject_selfattn > 0, or
the SD1.5 loop) this equals the reference's joint batch-2 step; with inject_selfattn = 0 and 0 < inject_background < 1
the reference would mix a batch-2 history with a batch-1 sample, which this loop does not.
"""
import numpy as np
import torch

from oracle import sampler_oracle as sam

# latent sides of the sampler fixtures (tests/golden/multistep.npz). The plain pass takes any multiple of 4 (tiny XL has
# 3 levels); 32^2 keeps a fixture at 16 KB. The rich loops are fixed by the reference's feature-injection hook, which
# asserts the width of up_blocks.1.resnets.1: 128^2 for tiny XL (models/region_diffusion_sdxl.py:1091), 64^2 for tiny SD
# (models/region_diffusion.py:339).
LATENT_XL_PLAIN, LATENT_XL_RICH, LATENT_SD = 32, 128, 64


def _alphas_cumprod(beta_start=0.00085, beta_end=0.012, n=1000):
    betas = torch.linspace(beta_start ** 0.5, beta_end ** 0.5, n, dtype=torch.float32) ** 2
    return torch.cumprod(1.0 - betas, dim=0)


class _Out(dict):
    def __getattr__(self, k):
        return self[k]

    def __getitem__(self, k):
        if isinstance(k, int):
            return list(self.values())[k]
        return dict.__getitem__(self, k)


class DDIMSchedulerOracle:
    """DDIMScheduler(steps_offset=1, set_alpha_to_one=False, clip_sample=False), eta = 0."""
    order = 1
    init_noise_sigma = 1.0

    def __init__(self, num_train_timesteps=1000):
        self.num_train_timesteps = num_train_timesteps
        self.alphas_cumprod = _alphas_cumprod(n=num_train_timesteps)
        self.final_alpha_cumprod = self.alphas_cumprod[0]
        self.timesteps = None

    def set_timesteps(self, num_inference_steps, device=None):
        self.num_inference_steps = num_inference_steps
        ratio = self.num_train_timesteps // num_inference_steps
        ts = (np.arange(0, num_inference_steps) * ratio).round()[::-1].copy().astype(np.int64)
        self.timesteps = torch.from_numpy(ts) + 1

    def scale_model_input(self, sample, timestep=None):
        return sample

    def step(self, model_output, timestep, sample, eta=0.0, use_clipped_model_output=False, generator=None,
             variance_noise=None, return_dict=True):
        assert eta == 0.0, "the oracle restates eta = 0 only"
        timestep = int(timestep)
        prev_timestep = timestep - self.num_train_timesteps // self.num_inference_steps
        a_t = self.alphas_cumprod[timestep]
        a_prev = self.alphas_cumprod[prev_timestep] if prev_timestep >= 0 else self.final_alpha_cumprod
        x0 = (sample - (1 - a_t) ** 0.5 * model_output) / a_t ** 0.5
        prev = a_prev ** 0.5 * x0 + (1 - a_prev) ** 0.5 * model_output
        return _Out(prev_sample=prev, pred_original_sample=x0) if return_dict else (prev,)


class DPMSolverMultistepSchedulerOracle:
    """DPMSolverMultistepScheduler: dpmsolver++, solver_order 2, midpoint, lower_order_final, no Karras sigmas."""
    order = 1
    init_noise_sigma = 1.0

    def __init__(self, num_train_timesteps=1000):
        self.num_train_timesteps = num_train_timesteps
        self.alphas_cumprod = _alphas_cumprod(n=num_train_timesteps)
        self.alpha_t = torch.sqrt(self.alphas_cumprod)
        self.sigma_t = torch.sqrt(1 - self.alphas_cumprod)
        self.lambda_t = torch.log(self.alpha_t) - torch.log(self.sigma_t)
        self.timesteps = None

    def set_timesteps(self, num_inference_steps, device=None):
        ts = np.linspace(0, self.num_train_timesteps - 1, num_inference_steps + 1).round()[::-1][:-1].copy().astype(np.int64)
        _, idx = np.unique(ts, return_index=True)
        ts = ts[np.sort(idx)]
        self.timesteps = torch.from_numpy(ts)
        self.num_inference_steps = len(ts)
        self.model_outputs = [None, None]
        self.lower_order_nums = 0

    def scale_model_input(self, sample, timestep=None):
        return sample

    def _x0(self, model_output, timestep, sample):
        return (sample - self.sigma_t[timestep] * model_output) / self.alpha_t[timestep]

    def _first(self, m0, timestep, prev_timestep, sample):
        lt, ls = self.lambda_t[prev_timestep], self.lambda_t[timestep]
        h = lt - ls
        return (self.sigma_t[prev_timestep] / self.sigma_t[timestep]) * sample \
            - (self.alpha_t[prev_timestep] * (torch.exp(-h) - 1.0)) * m0

    def _second(self, timestep_list, prev_timestep, sample):
        t, s0, s1 = prev_timestep, timestep_list[-1], timestep_list[-2]
        m0, m1 = self.model_outputs[-1], self.model_outputs[-2]
        h, h0 = self.lambda_t[t] - self.lambda_t[s0], self.lambda_t[s0] - self.lambda_t[s1]
        r0 = h0 / h
        D0, D1 = m0, (1.0 / r0) * (m0 - m1)
        a = self.alpha_t[t] * (torch.exp(-h) - 1.0)
        return (self.sigma_t[t] / self.sigma_t[s0]) * sample - a * D0 - 0.5 * a * D1

    def step(self, model_output, timestep, sample, generator=None, return_dict=True, **kw):
        timestep = int(timestep)
        idx = (self.timesteps == timestep).nonzero()
        step_index = len(self.timesteps) - 1 if len(idx) == 0 else int(idx.item())
        prev_timestep = 0 if step_index == len(self.timesteps) - 1 else int(self.timesteps[step_index + 1])
        lower_order_final = step_index == len(self.timesteps) - 1 and len(self.timesteps) < 15
        m = self._x0(model_output, timestep, sample)
        self.model_outputs = [self.model_outputs[1], m]
        if self.lower_order_nums < 1 or lower_order_final:
            prev = self._first(m, timestep, prev_timestep, sample)
        else:
            prev = self._second([int(self.timesteps[step_index - 1]), timestep], prev_timestep, sample)
        if self.lower_order_nums < 2:
            self.lower_order_nums += 1
        return _Out(prev_sample=prev) if return_dict else (prev,)


SCHEDULERS = {"ddim": DDIMSchedulerOracle, "dpmpp_2m": DPMSolverMultistepSchedulerOracle}


# ------------------------------------------------------------------------------------------------ float64 steps
def coeffs64(kind, N, i):
    """(timestep t, target s, x' as a function of (x, eps, D_prev)) of step i, evaluated in float64 straight from the
    scheduler definitions (not through the affine coefficients): the reference for step_coeffs."""
    ac = _alphas_cumprod().double()
    al, sg = ac.sqrt(), (1 - ac).sqrt()
    lam = al.log() - sg.log()
    if kind == "ddim":
        ts = (np.arange(N) * (1000 // N))[::-1] + 1
        t = int(ts[i])
        s = t - 1000 // N
        ap = ac[s] if s >= 0 else ac[0]

        def f(x, eps, d_prev=None):
            x0 = (x - sg[t] * eps) / al[t]
            return ap.sqrt() * x0 + (1 - ap).sqrt() * eps, x0
        return t, s, f
    ts = np.linspace(0, 999, N + 1).round()[::-1][:-1].astype(np.int64)
    _, idx = np.unique(ts, return_index=True)
    ts = ts[np.sort(idx)]
    n = len(ts)
    t = int(ts[i])
    s = 0 if i == n - 1 else int(ts[i + 1])
    h = lam[s] - lam[t]
    first = i == 0 or (i == n - 1 and n < 15)

    def f(x, eps, d_prev=None):
        D = (x - sg[t] * eps) / al[t]
        if first:
            return (sg[s] / sg[t]) * x - al[s] * torch.expm1(-h) * D, D
        r = (lam[t] - lam[int(ts[i - 1])]) / h
        return (sg[s] / sg[t]) * x - al[s] * torch.expm1(-h) * (D + (D - d_prev) / (2 * r)), D
    return t, s, f


# ------------------------------------------------------------------------------------------------ loops
def plain_loop(unet, scheduler, text_embeddings, latents, num_inference_steps, guidance_scale, added_cond=None):
    return sam.plain_loop(unet, scheduler, text_embeddings, latents, num_inference_steps, guidance_scale, True,
                          added_cond=added_cond)


def rich_text_loop(unet, scheduler, scheduler_ref, text_embeddings, masks, latents, num_inference_steps, guidance_scale,
                   xl=True, added_cond=None, use_guidance=False, text_format_dict=None, inject_selfattn=0.0,
                   inject_background=0.0, vae_decode=None, scaling_factor=0.18215):
    """sampler_oracle.rich_text_loop with the reference latents stepped on their own scheduler state."""
    tfd = text_format_dict or {}
    scheduler.set_timesteps(num_inference_steps)
    scheduler_ref.set_timesteps(num_inference_steps)
    timesteps = scheduler.timesteps
    inject = inject_selfattn > 0 or inject_background > 0
    latents_reference = latents.clone() if inject else None
    n_t = len(timesteps)

    def added(rows):
        if added_cond is None:
            return None
        return {"text_embeds": added_cond["text_embeds"][rows], "time_ids": added_cond["time_ids"][:1]}

    last = text_embeddings.shape[0] - 1
    for i, t in enumerate(timesteps):
        feat_inject_step = bool(t > (1 - inject_selfattn) * 1000)
        if xl:
            background_inject_step = i < inject_background * n_t
        else:
            background_inject_step = (i == int(inject_background * n_t)) and inject_background > 0
        with torch.no_grad():
            eps_u = unet(latents, t, text_embeddings[:1], added(slice(0, 1)), None)
            eps_text_cur = unet(latents, t, text_embeddings[-1:], added(slice(last, last + 1)), sam.FontSizeControl(tfd))
            if inject:
                eps_u_ref = unet(latents_reference, t, text_embeddings[:1], added(slice(0, 1)), None)
                store = sam.SelfAttnStore(feat_inject_step)
                eps_t_ref = unet(latents_reference, t, text_embeddings[-1:], added(slice(last, last + 1)), store)
            noise_pred_uncond = eps_u * masks[-1]
            noise_pred_text = eps_text_cur * masks[-1]
            for j, mask in enumerate(masks[:-1]):
                ctrl = sam.ReplaceControl(feat_inject_step, store.store) if inject else None
                eps_j = unet(latents, t, text_embeddings[j + 1:j + 2], added(slice(j + 1, j + 2)), ctrl)
                noise_pred_uncond = noise_pred_uncond + eps_u * mask
                noise_pred_text = noise_pred_text + eps_j * mask
            noise_pred = noise_pred_uncond + guidance_scale * (noise_pred_text - noise_pred_uncond)
            joint = (inject_selfattn > 0 or background_inject_step > 0) if xl else inject
            latents = scheduler.step(noise_pred, t, latents)["prev_sample"]
            if joint:
                noise_pred_refer = eps_u_ref + guidance_scale * (eps_t_ref - eps_u_ref)
                latents_reference = scheduler_ref.step(noise_pred_refer, t, latents_reference)["prev_sample"]
        if use_guidance and bool(t < tfd["guidance_start_step"]):
            latents = sam.color_guidance(latents, noise_pred, t, scheduler.alphas_cumprod, vae_decode, scaling_factor,
                                         tfd, xl)
        if xl:
            do_bg = (i == int(inject_background * n_t)) and inject_background > 0
        else:
            do_bg = background_inject_step
        if do_bg:
            latents = latents_reference * masks[-1] + latents * (1 - masks[-1])
    return latents
