"""Device-side schedulers used by the samplers.

The reference delegates to the third-party diffusers 0.18.2 schedulers (PNDM/PLMS for SD1.5,
models/region_diffusion.py:35-37; EulerDiscrete for SDXL, models/region_diffusion_sdxl.py:120). Those
sources are not part of the reference tree, so the published algorithms are restated here; only the
calls the reference makes are provided: set_timesteps / timesteps / scale_model_input / step /
init_noise_sigma / alphas_cumprod.  All state lives on the sampling device; `step` never synchronises.

DDIMScheduler and DPMSolverMultistepScheduler (below) are the schedulers a diffusers user swaps in
(`model.scheduler = DPMSolverMultistepScheduler(...)`); the samplers run them through the fused blend kernels with
the per-step coefficients of `step_coeffs(i)`. EulerAncestralDiscreteScheduler ("Euler a", SDXL) adds fresh noise on
every step; the SDXL sampler runs it through the fused blend kernels with `ancestral_coeffs(i)`.
UniPCMultistepScheduler (bh2, order 2, the few-step sampler) runs through the fused blend kernels of both samplers
with `unipc_coeffs(i)`. HeunDiscreteScheduler (Heun's second-order method on Euler's sigma grid, two UNet evaluations
per step) runs through the fused blend kernels of the SDXL sampler with `heun_coeffs(k)`. LMSDiscreteScheduler (k-LMS,
the fourth-order linear multistep method on Euler's sigma grid) runs through the fused blend kernels of the SDXL sampler
with `lms_coeffs(i)`. DPMSolverSinglestepScheduler (DPM-Solver++(2S), two-step blocks that restart from the latents
that entered the block) runs through the fused blend kernels of both samplers with `singlestep_coeffs(i)`.
"""
import math
from typing import NamedTuple

import numpy as np
import torch


def _alphas_cumprod(beta_start, beta_end, n):
    betas = torch.linspace(beta_start ** 0.5, beta_end ** 0.5, n, dtype=torch.float32) ** 2
    return torch.cumprod(1.0 - betas, dim=0)


class _Config(dict):
    """Scheduler configuration: a dict with attribute access (diffusers' scheduler.config)."""
    __getattr__ = dict.get


class EulerDiscreteScheduler:
    """EulerDiscrete, epsilon prediction, scaled-linear betas, `leading` spacing, steps_offset=1 (SDXL config)."""
    order = 1

    def __init__(self, beta_start=0.00085, beta_end=0.012, num_train_timesteps=1000, steps_offset=1):
        self.num_train_timesteps, self.steps_offset = num_train_timesteps, steps_offset
        self.config = _Config(beta_start=beta_start, beta_end=beta_end, num_train_timesteps=num_train_timesteps,
                              steps_offset=steps_offset, beta_schedule="scaled_linear")
        self.alphas_cumprod = _alphas_cumprod(beta_start, beta_end, num_train_timesteps)  # host copy (predict_x0)
        self._sig_all = (((1 - self.alphas_cumprod) / self.alphas_cumprod) ** 0.5).numpy()
        self.sigmas_host = np.concatenate([self._sig_all[::-1], [0.0]]).astype(np.float32)
        self.timesteps_host = np.linspace(0, num_train_timesteps - 1, num_train_timesteps, dtype=float)[::-1].copy()
        self.timesteps = torch.from_numpy(self.timesteps_host)

    @property
    def init_noise_sigma(self):
        return float((self.sigmas_host.max() ** 2 + 1) ** 0.5)

    def set_timesteps(self, num_inference_steps, device=None):
        self.num_inference_steps = num_inference_steps
        ratio = self.num_train_timesteps // num_inference_steps
        ts = (np.arange(0, num_inference_steps) * ratio).round()[::-1].copy().astype(float) + self.steps_offset
        sig = np.interp(ts, np.arange(0, len(self._sig_all)), self._sig_all)
        self.sigmas_host = np.concatenate([sig, [0.0]]).astype(np.float32)
        self.timesteps_host = ts
        self.timesteps = torch.from_numpy(ts)  # host tensor: the loop's `t > ...` tests never touch the device

    def index_of(self, timestep):
        return int(np.nonzero(self.timesteps_host == float(timestep))[0][0])

    def sigma(self, timestep):
        return float(self.sigmas_host[self.index_of(timestep)])

    def dt(self, timestep):
        i = self.index_of(timestep)
        return float(self.sigmas_host[i + 1] - self.sigmas_host[i])

    def scale_model_input(self, sample, timestep):
        s = self.sigma(timestep)
        return sample / ((s * s + 1.0) ** 0.5)

    def step(self, model_output, timestep, sample, **kw):
        # x + eps * (sigma_next - sigma); the reference's `derivative` equals eps for epsilon prediction
        return {"prev_sample": (sample.float() + model_output.float() * self.dt(timestep)).to(sample.dtype)}


class PNDMScheduler:
    """PNDM with skip_prk_steps=True (pure PLMS), steps_offset=1 — N+1 model evaluations for N steps."""
    order = 1

    def __init__(self, beta_start=0.00085, beta_end=0.012, num_train_timesteps=1000, steps_offset=1):
        self.num_train_timesteps, self.steps_offset = num_train_timesteps, steps_offset
        self.config = _Config(beta_start=beta_start, beta_end=beta_end, num_train_timesteps=num_train_timesteps,
                              steps_offset=steps_offset, beta_schedule="scaled_linear")
        self.alphas_cumprod = _alphas_cumprod(beta_start, beta_end, num_train_timesteps)
        self.final_alpha_cumprod = float(self.alphas_cumprod[0])
        self.init_noise_sigma = 1.0
        self.ets, self.counter, self.cur_sample = [], 0, None
        self.timesteps = None

    def set_timesteps(self, num_inference_steps, device=None):
        self.num_inference_steps = num_inference_steps
        ratio = self.num_train_timesteps // num_inference_steps
        ts = (np.arange(0, num_inference_steps) * ratio).round() + self.steps_offset
        plms = np.concatenate([ts[:-1], ts[-2:-1], ts[-1:]])[::-1].copy().astype(np.int64)
        self.timesteps = torch.from_numpy(plms)
        self.ets, self.counter, self.cur_sample = [], 0, None

    def scale_model_input(self, sample, timestep=None):
        return sample

    def step(self, model_output, timestep, sample, **kw):
        timestep = int(timestep)
        ratio = self.num_train_timesteps // self.num_inference_steps
        prev_timestep = timestep - ratio
        model_output = model_output.float()
        sample = sample.float()
        if self.counter != 1:
            self.ets = self.ets[-3:]
            self.ets.append(model_output)
        else:
            prev_timestep = timestep
            timestep = timestep + ratio
        if len(self.ets) == 1 and self.counter == 0:
            self.cur_sample = sample
        elif len(self.ets) == 1 and self.counter == 1:
            model_output = (model_output + self.ets[-1]) / 2
            sample = self.cur_sample
            self.cur_sample = None
        elif len(self.ets) == 2:
            model_output = (3 * self.ets[-1] - self.ets[-2]) / 2
        elif len(self.ets) == 3:
            model_output = (23 * self.ets[-1] - 16 * self.ets[-2] + 5 * self.ets[-3]) / 12
        else:
            model_output = (1 / 24) * (55 * self.ets[-1] - 59 * self.ets[-2] + 37 * self.ets[-3] - 9 * self.ets[-4])
        a_t = float(self.alphas_cumprod[timestep])
        a_prev = float(self.alphas_cumprod[prev_timestep]) if prev_timestep >= 0 else self.final_alpha_cumprod
        b_t, b_prev = 1 - a_t, 1 - a_prev
        coeff = (a_prev / a_t) ** 0.5
        denom = a_t * b_prev ** 0.5 + (a_t * b_t * a_prev) ** 0.5
        self.counter += 1
        return {"prev_sample": coeff * sample - (a_prev - a_t) * model_output / denom}


# ---------------------------------------------------------------------------------------------------- multistep
class StepCoeffs(NamedTuple):
    """One step of DDIM / DPM-Solver++(2M) in data-prediction form (float64, host):
        D  = hx * x + he * eps                      (x0 prediction, hx = 1/alpha_t, he = -sigma_t/alpha_t)
        x' = cx * x + cd * D + cp * D_prev          (D_prev: the D of the previous step; cp = 0 on first-order steps)
    The blend kernels' multistep entry points (rtti_*_ms) evaluate exactly this with eps = the fp16-rounded prediction."""
    hx: float
    he: float
    cx: float
    cd: float
    cp: float


class _Configured:
    """Keyword configuration of the schedulers a diffusers user swaps in: `_defaults` (diffusers' keywords and defaults)
    and `_unsupported` (keyword -> the only value this restatement implements)."""
    _unsupported = {}

    def _configure(self, kw):
        for k, v in kw.items():
            if k in self._unsupported and v != self._unsupported[k]:
                raise NotImplementedError(f"{type(self).__name__}: {k}={v!r} is not supported "
                                          f"(only {k}={self._unsupported[k]!r})")
        cfg = dict(self._defaults)
        unknown = set(kw) - set(cfg)
        if unknown:
            raise TypeError(f"{type(self).__name__}: unexpected keyword arguments {sorted(unknown)}")
        cfg.update(kw)
        if cfg["beta_schedule"] != "scaled_linear":
            raise NotImplementedError(f"{type(self).__name__}: beta_schedule={cfg['beta_schedule']!r} is not supported")
        self.config = _Config(cfg)
        return self.config

    @classmethod
    def from_config(cls, config, **kw):
        """`config`: a dict, or any scheduler of this package (its `.config`); keys this class does not take are dropped,
        as diffusers' from_config does."""
        cfg = dict(config if isinstance(config, dict) else config.config)
        cfg.update(kw)
        return cls(**{k: v for k, v in cfg.items() if k in cls._defaults})


class _MultistepBase(_Configured):
    """Shared VP-space conventions of DDIMScheduler, DPMSolverMultistepScheduler and UniPCMultistepScheduler:
    scaled-linear betas, epsilon prediction, init_noise_sigma = 1, scale_model_input = identity (the UNet sees the
    latents unscaled),
    alphas_cumprod = the same host fp32 tensor as the other schedulers (colour guidance's predict_x0), host int64
    timesteps. Write a_t = alphas_cumprod[t], alpha_t = sqrt(a_t), sigma_t = sqrt(1 - a_t),
    lambda_t = log alpha_t - log sigma_t."""
    order = 1
    init_noise_sigma = 1.0

    def __init__(self, **kw):
        cfg = self._configure(kw)
        self.num_train_timesteps = int(cfg["num_train_timesteps"])
        self.alphas_cumprod = _alphas_cumprod(cfg["beta_start"], cfg["beta_end"], self.num_train_timesteps)
        ac = self.alphas_cumprod.double().numpy()
        self._alpha, self._sigma = np.sqrt(ac), np.sqrt(1.0 - ac)
        self._lambda = np.log(self._alpha) - np.log(self._sigma)
        self.timesteps = None
        self.num_inference_steps = None
        self._d_prev = None

    def scale_model_input(self, sample, timestep=None):
        return sample

    def index_of(self, timestep):
        return int(np.nonzero(self.timesteps_host == int(timestep))[0][0])

    def _first_order(self, t, s):
        """DPM-Solver-1 (= DDIM, eta 0) from timestep t to timestep s: (hx, he, cx, cd, h)."""
        h = float(self._lambda[s] - self._lambda[t])
        a_t, s_t, a_s, s_s = (float(v) for v in (self._alpha[t], self._sigma[t], self._alpha[s], self._sigma[s]))
        return 1.0 / a_t, -s_t / a_t, s_s / s_t, -a_s * math.expm1(-h), h

    def step(self, model_output, timestep, sample, eta=0.0, return_dict=True, **kw):
        """Stateful torch form of step_coeffs (the samplers use the fused kernels instead): keeps D of the last step."""
        if eta:
            raise NotImplementedError(f"{type(self).__name__}: eta > 0 is not supported")
        c = self.step_coeffs(self.index_of(timestep))
        x, e = sample.float(), model_output.float()
        d = c.hx * x + c.he * e
        prev = c.cx * x + c.cd * d
        if c.cp != 0.0:
            prev = prev + c.cp * self._d_prev
        self._d_prev = d
        prev = prev.to(sample.dtype)
        return {"prev_sample": prev} if return_dict else (prev,)


class DDIMScheduler(_MultistepBase):
    """DDIM, eta = 0, with the SD1.5 / SDXL scheduler configs (steps_offset=1, set_alpha_to_one=False,
    clip_sample=False), restating diffusers 0.18.2 (`schedulers/scheduling_ddim.py`). PARITY UNPINNED: that source is not
    available here; the conventions below are the definition.
      timesteps = arange(N) * (1000 // N), reversed, + steps_offset
      prev = t - 1000 // N;  a_prev = alphas_cumprod[prev], or alphas_cumprod[0] if prev < 0
      x' = sqrt(a_prev) * x0_hat + sqrt(1 - a_prev) * eps,   x0_hat = (x - sigma_t eps) / alpha_t
    which is DPM-Solver-1: cx = sigma_prev / sigma_t, cd = -alpha_prev * expm1(-h), cp = 0 (step_coeffs)."""
    _defaults = dict(num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear",
                     trained_betas=None, clip_sample=False, set_alpha_to_one=False, steps_offset=1,
                     prediction_type="epsilon", thresholding=False, dynamic_thresholding_ratio=0.995,
                     clip_sample_range=1.0, sample_max_value=1.0, timestep_spacing="leading")
    _unsupported = dict(trained_betas=None, clip_sample=False, set_alpha_to_one=False, prediction_type="epsilon",
                        thresholding=False, timestep_spacing="leading")

    def set_timesteps(self, num_inference_steps, device=None):
        self.num_inference_steps = num_inference_steps
        ratio = self.num_train_timesteps // num_inference_steps
        ts = (np.arange(0, num_inference_steps) * ratio).round()[::-1].astype(np.int64) + int(self.config.steps_offset)
        self.timesteps_host = ts.copy()
        self.timesteps = torch.from_numpy(self.timesteps_host.copy())
        self._d_prev = None

    def step_coeffs(self, i):
        t = int(self.timesteps_host[i])
        prev = t - self.num_train_timesteps // self.num_inference_steps
        hx, he, cx, cd, _ = self._first_order(t, max(prev, 0))   # set_alpha_to_one=False: prev < 0 lands on index 0
        return StepCoeffs(hx, he, cx, cd, 0.0)


class DPMSolverMultistepScheduler(_MultistepBase):
    """DPM-Solver++(2M): algorithm_type="dpmsolver++", solver_order=2, solver_type="midpoint", lower_order_final=True,
    no Karras sigmas, epsilon prediction — the defaults of diffusers 0.18.2 (`schedulers/scheduling_dpmsolver_multistep.py`),
    restated. PARITY UNPINNED: that source is not available here; the conventions below are the definition.
      timesteps = linspace(0, 999, N+1).round()[::-1][:-1], duplicates removed in order (N may shrink at N ~ 1000)
      step i: t = ts[i] -> s = ts[i+1] (s = 0 on the last step), h = lambda_s - lambda_t, D_i = x0_hat at step i
      first order (step 0, and the last step when len(ts) < 15): x' = (sigma_s/sigma_t) x - alpha_s expm1(-h) D_i
      otherwise, r = (lambda_t - lambda_{t_prev}) / h:
                  x' = (sigma_s/sigma_t) x - alpha_s expm1(-h) (D_i + (D_i - D_{i-1}) / (2r))"""
    _defaults = dict(num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear",
                     trained_betas=None, solver_order=2, prediction_type="epsilon", thresholding=False,
                     dynamic_thresholding_ratio=0.995, sample_max_value=1.0, algorithm_type="dpmsolver++",
                     solver_type="midpoint", lower_order_final=True, use_karras_sigmas=False, lambda_min_clipped=-float("inf"),
                     variance_type=None, steps_offset=1, set_alpha_to_one=False, clip_sample=False,
                     timestep_spacing="linspace")
    _unsupported = dict(trained_betas=None, solver_order=2, prediction_type="epsilon", thresholding=False,
                        algorithm_type="dpmsolver++", solver_type="midpoint", use_karras_sigmas=False,
                        lambda_min_clipped=-float("inf"), variance_type=None, timestep_spacing="linspace")

    def set_timesteps(self, num_inference_steps, device=None):
        ts = np.linspace(0, self.num_train_timesteps - 1, num_inference_steps + 1).round()[::-1][:-1].astype(np.int64)
        _, first = np.unique(ts, return_index=True)
        self.timesteps_host = ts[np.sort(first)].copy()
        self.timesteps = torch.from_numpy(self.timesteps_host.copy())
        self.num_inference_steps = len(self.timesteps_host)
        self._d_prev = None

    def step_coeffs(self, i):
        ts, n = self.timesteps_host, len(self.timesteps_host)
        t = int(ts[i])
        s = 0 if i == n - 1 else int(ts[i + 1])
        hx, he, cx, cd, h = self._first_order(t, s)
        if i == 0 or (i == n - 1 and self.config.lower_order_final and n < 15):
            return StepCoeffs(hx, he, cx, cd, 0.0)
        r = (self._lambda[t] - self._lambda[int(ts[i - 1])]) / h
        return StepCoeffs(hx, he, cx, cd * (1.0 + 0.5 / r), -cd * 0.5 / r)


MULTISTEP_SCHEDULERS = (DDIMScheduler, DPMSolverMultistepScheduler)


# ---------------------------------------------------------------------------------------------------- singlestep
class SinglestepCoeffs(NamedTuple):
    """One step of DPM-Solver++(2S) in data-prediction form (float64, host):
        D  = hx * x + he * eps                               (x0 prediction, as in StepCoeffs)
        x' = cx * x + cd * D + cp * D_prev + cs * xs         (D_prev: the D of the block's first step; xs: the latents
                                                              that entered it; cs = cp = 0 on a first step)
    The blend kernels' singlestep entry points (rtti_*_ss) evaluate exactly this with eps = the fp16-rounded prediction."""
    hx: float
    he: float
    cx: float
    cs: float
    cd: float
    cp: float


class DPMSolverSinglestepScheduler(_MultistepBase):
    """DPM-Solver++(2S): algorithm_type="dpmsolver++", solver_order=2, solver_type="midpoint", lower_order_final=True,
    no Karras sigmas, epsilon prediction, with the SD1.5 / SDXL betas — diffusers 0.18.2
    (`schedulers/scheduling_dpmsolver_singlestep.py`), restated. PARITY UNPINNED: that source is not available here; the
    conventions below are the definition.
      timesteps: those of DPMSolverMultistepScheduler (linspace grid, duplicates removed); N = len(timesteps)
      order list: [1, 2] * (N // 2), plus [1] when N is odd; step i goes from t_i = ts[i] to ts[i+1] (0 on the last
      step). order = 1: one UNet evaluation per step, so a sampling loop's callback fires on every iteration.
      D_i = (x_i - sigma_{t_i} eps_i) / alpha_{t_i}, with x_i the latents the UNet saw at step i
      order 1 (the first step of a two-step block, s1 = t_i -> s0 = ts[i+1]): DPM-Solver-1,
        x' = (sigma_s0 / sigma_s1) x_i - alpha_s0 expm1(-h) D_i;  the block keeps xs = x_i and D_i
      order 2 (the second step, s0 = t_i, from s1 = ts[i-1] to t = ts[i+1]): h = lambda_t - lambda_s1,
        r0 = (lambda_s0 - lambda_s1) / h,
        x' = (sigma_t / sigma_s1) xs - alpha_t expm1(-h) D_{i-1} - alpha_t expm1(-h) (D_i - D_{i-1}) / (2 r0)
    The second step restarts from xs, the latents that entered the block: the current latents x_i reach it only through
    eps_i (in D_i). Whatever a sampling loop does to the latents after a first step (colour guidance, background
    injection) therefore acts on the second step's update through the prediction alone, as in diffusers. The samplers run
    it through the fused blend kernels with the coefficients of `singlestep_coeffs(i)`, one fp32 D buffer and the fp16
    xs per trajectory (ops.SinglestepStep); `step` is the stateful torch form in diffusers' calling convention. Not a
    subclass of DPMSolverMultistepScheduler: the samplers dispatch on the class, and this update is not 2M's."""
    _defaults = dict(num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear",
                     trained_betas=None, solver_order=2, prediction_type="epsilon", thresholding=False,
                     dynamic_thresholding_ratio=0.995, sample_max_value=1.0, algorithm_type="dpmsolver++",
                     solver_type="midpoint", lower_order_final=True, use_karras_sigmas=False,
                     lambda_min_clipped=-float("inf"), variance_type=None)
    _unsupported = dict(trained_betas=None, solver_order=2, prediction_type="epsilon", thresholding=False,
                        algorithm_type="dpmsolver++", solver_type="midpoint", lower_order_final=True,
                        use_karras_sigmas=False, lambda_min_clipped=-float("inf"), variance_type=None)

    def __init__(self, **kw):
        if kw.get("solver_type") in ("bh1", "bh2", "logrho"):
            kw["solver_type"] = "midpoint"   # as diffusers does, so that from_config(UniPCMultistepScheduler) works
        super().__init__(**kw)
        self.order_list = []
        self._xs = None

    @staticmethod
    def get_order_list(n):
        """The order of each of n steps: [1, 2] * (n // 2), plus [1] when n is odd."""
        return [1, 2] * (n // 2) + [1] * (n % 2)

    def set_timesteps(self, num_inference_steps, device=None):
        DPMSolverMultistepScheduler.set_timesteps(self, num_inference_steps, device)
        self.order_list = self.get_order_list(len(self.timesteps_host))
        self._xs = None

    def is_first_step(self, i):
        """Whether step i is first order: it starts a two-step block (or is the odd last step), so its input latents
        become the xs of the block."""
        return self.order_list[i] == 1

    def singlestep_coeffs(self, i):
        ts, n = self.timesteps_host, len(self.timesteps_host)
        t_i = int(ts[i])
        s = 0 if i == n - 1 else int(ts[i + 1])
        hx, he, cx, cd, _ = self._first_order(t_i, s)
        if self.order_list[i] == 1:
            return SinglestepCoeffs(hx, he, cx, 0.0, cd, 0.0)
        s1 = int(ts[i - 1])
        lam = self._lambda
        h = float(lam[s] - lam[s1])
        r0 = float(lam[t_i] - lam[s1]) / h
        a_t, em = float(self._alpha[s]), math.expm1(-h)
        cs = float(self._sigma[s] / self._sigma[s1])
        return SinglestepCoeffs(hx, he, 0.0, cs, -0.5 * a_t * em / r0, -a_t * em * (1.0 - 0.5 / r0))

    def step(self, model_output, timestep, sample, return_dict=True, **kw):
        """Stateful torch form of singlestep_coeffs in diffusers' calling convention (the samplers use the fused kernels
        instead), in the precision of `sample` and at least fp32: a first step keeps `sample` as xs and its D."""
        i = self.index_of(timestep)
        c = self.singlestep_coeffs(i)
        dt = torch.promote_types(sample.dtype, torch.float32)
        x, e = sample.to(dt), model_output.to(dt)
        d = c.hx * x + c.he * e
        prev = c.cx * x + c.cd * d
        if c.cp != 0.0:
            prev = prev + c.cp * self._d_prev
        if c.cs != 0.0:
            prev = prev + c.cs * self._xs.to(dt)
        if self.is_first_step(i):
            self._xs = sample
        self._d_prev = d
        prev = prev.to(sample.dtype)
        return {"prev_sample": prev} if return_dict else (prev,)


# ---------------------------------------------------------------------------------------------------- UniPC
class UniPCCoeffs(NamedTuple):
    """One step of UniPC (bh2, order 2) in data-prediction form (float64, host):
        m  = hx * x + he * eps                                  (x0 prediction of this step)
        xc = ux * x + ul * xl + u0 * m + u1 * m1 + u2 * m2      (corrected sample; xl = xc of the previous step,
                                                                  m1 / m2 = m of the previous two steps)
        x' = vx * xc + v0 * m + v1 * m1                         (predictor)
    The blend kernels' UniPC entry points (rtti_*_unipc) evaluate exactly this with eps = the fp16-rounded prediction."""
    hx: float
    he: float
    ux: float
    ul: float
    u0: float
    u1: float
    u2: float
    vx: float
    v0: float
    v1: float


class UniPCMultistepScheduler(_MultistepBase):
    """UniPC: solver_type="bh2", solver_order=2, predict_x0=True, lower_order_final=True, no corrector disabled, no
    solver_p, epsilon prediction — the defaults of diffusers 0.18.2 (`schedulers/scheduling_unipc_multistep.py`) with
    the SD1.5 / SDXL betas, restated. PARITY UNPINNED: that source is not available here; the conventions below are the
    definition. Timesteps: those of DPMSolverMultistepScheduler. Step i goes from t = ts[i] to s = ts[i+1] (s = 0 on the
    last step); m_i = (x_i - sigma_t eps_i) / alpha_t, with x_i the latents the UNet saw at step i.
      orders: predictor p_i = min(2, n - i, i + 1); corrector at i >= 1 of order c_i = p_{i-1}
      corrector (UniC), i >= 1, t' = ts[i-1]: h = lambda_t - lambda_t', hh = -h, B = phi = expm1(hh),
        x^ = (sigma_t / sigma_t') xc_{i-1} - alpha_t phi m_{i-1}
        c_i = 1: xc_i = x^ - alpha_t B (m_i - m_{i-1}) / 2
        c_i = 2: r = (lambda_{ts[i-2]} - lambda_t') / h, D = (m_{i-2} - m_{i-1}) / r, (rho0, rho1) solves
                 [[1, 1], [r, 1]] rho = [g1, g2], g1 = (phi/hh - 1) / B, g2 = 2 ((phi/hh - 1)/hh - 1/2) / B;
                 xc_i = x^ - alpha_t B (rho0 D + rho1 (m_i - m_{i-1}))
        step 0: xc_0 = x_0
      predictor (UniP): h = lambda_s - lambda_t, hh, B, phi as above,
        x_{i+1} = (sigma_s / sigma_t) xc_i - alpha_s phi m_i - [p_i = 2] alpha_s B (m_{i-1} - m_i) / (2 r'),
        r' = (lambda_{ts[i-1]} - lambda_t) / h
    The corrector restarts from its own xc_{i-1}, so the current latents reach it only through m_i: whatever a sampling
    loop does to the latents between two steps (colour guidance, background injection) acts on the next update through
    the x0 prediction alone. The samplers run it through the fused blend kernels with the coefficients of
    `unipc_coeffs(i)` and three fp32 histories per trajectory (ops.UniPCHistory)."""
    _defaults = dict(num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear",
                     trained_betas=None, solver_order=2, prediction_type="epsilon", thresholding=False,
                     dynamic_thresholding_ratio=0.995, sample_max_value=1.0, predict_x0=True, solver_type="bh2",
                     lower_order_final=True, disable_corrector=[], solver_p=None, use_karras_sigmas=False,
                     timestep_spacing="linspace", steps_offset=1)
    _unsupported = dict(trained_betas=None, solver_order=2, prediction_type="epsilon", thresholding=False,
                        predict_x0=True, solver_type="bh2", lower_order_final=True, disable_corrector=[], solver_p=None,
                        use_karras_sigmas=False, timestep_spacing="linspace")

    def __init__(self, **kw):
        if kw.get("disable_corrector") is not None:
            kw["disable_corrector"] = list(kw["disable_corrector"])
        if kw.get("solver_type") in ("midpoint", "heun", "logrho"):
            kw["solver_type"] = "bh2"   # as diffusers does, so that from_config(DPMSolverMultistepScheduler) works
        super().__init__(**kw)
        self._xl = self._m1 = self._m2 = None

    def set_timesteps(self, num_inference_steps, device=None):
        DPMSolverMultistepScheduler.set_timesteps(self, num_inference_steps, device)
        self._xl = self._m1 = self._m2 = None

    def orders(self, i):
        """(predictor order p_i, corrector order c_i; 0 at step 0, which has no corrector)."""
        n = len(self.timesteps_host)
        p = lambda k: min(2, n - k, k + 1)
        return p(i), (p(i - 1) if i > 0 else 0)

    def unipc_coeffs(self, i):
        ts, n = self.timesteps_host, len(self.timesteps_host)
        al, sg, lam = self._alpha, self._sigma, self._lambda
        t = int(ts[i])
        s = 0 if i == n - 1 else int(ts[i + 1])
        p, c = self.orders(i)
        hx, he = 1.0 / al[t], -sg[t] / al[t]
        if c == 0:
            ux, ul, u0, u1, u2 = 1.0, 0.0, 0.0, 0.0, 0.0
        else:
            tp = int(ts[i - 1])
            h = lam[t] - lam[tp]
            hh = -h
            phi = math.expm1(hh)
            a = al[t] * phi                      # alpha_t * B (bh2: B = phi)
            ux, ul = 0.0, sg[t] / sg[tp]
            if c == 1:
                rho0, rho1, r = 0.0, 0.5, 1.0
            else:
                r = (lam[int(ts[i - 2])] - lam[tp]) / h
                g1 = (phi / hh - 1.0) / phi
                g2 = 2.0 * ((phi / hh - 1.0) / hh - 0.5) / phi
                rho0 = (g1 - g2) / (1.0 - r)
                rho1 = g1 - rho0
            # xc = ul xl - a m1 - a (rho0 (m2 - m1) / r + rho1 (m - m1))
            u0, u1, u2 = -a * rho1, -a * (1.0 - rho0 / r - rho1), -a * rho0 / r
        h = lam[s] - lam[t]
        phi = math.expm1(-h)
        b = al[s] * phi
        vx = sg[s] / sg[t]
        if p == 1:
            v0, v1 = -b, 0.0
        else:
            rp = (lam[int(ts[i - 1])] - lam[t]) / h
            v0, v1 = -b + 0.5 * b / rp, -0.5 * b / rp
        return UniPCCoeffs(*(float(v) for v in (hx, he, ux, ul, u0, u1, u2, vx, v0, v1)))

    def step(self, model_output, timestep, sample, return_dict=True, **kw):
        """Stateful torch form of unipc_coeffs (the samplers use the fused kernels instead), in the precision of
        `sample` and at least fp32: keeps xc of the last step and m of the last two."""
        c = self.unipc_coeffs(self.index_of(timestep))
        dt = torch.promote_types(sample.dtype, torch.float32)
        x, e = sample.to(dt), model_output.to(dt)
        m = c.hx * x + c.he * e
        xc = c.ux * x + c.u0 * m
        for coef, hist in ((c.ul, self._xl), (c.u1, self._m1), (c.u2, self._m2)):
            if coef != 0.0:
                xc = xc + coef * hist
        prev = c.vx * xc + c.v0 * m
        if c.v1 != 0.0:
            prev = prev + c.v1 * self._m1
        self._xl, self._m1, self._m2 = xc, m, self._m1
        prev = prev.to(sample.dtype)
        return {"prev_sample": prev} if return_dict else (prev,)


# ---------------------------------------------------------------------------------------------------- ancestral
class EulerAncestralDiscreteScheduler(_Configured):
    """Euler Ancestral ("Euler a"), epsilon prediction, with the SDXL config (scaled-linear betas 0.00085-0.012, `leading`
    spacing, steps_offset=1), restating diffusers 0.18.2 (`schedulers/scheduling_euler_ancestral_discrete.py`). PARITY
    UNPINNED: that source is not available here; the conventions below are the definition.
      timesteps, sigmas_host, init_noise_sigma, scale_model_input, alphas_cumprod: those of EulerDiscreteScheduler
      step i, sigma = sigmas_host[i] -> sigma' = sigmas_host[i + 1]:
        s_up = sqrt(sigma'^2 (sigma^2 - sigma'^2) / sigma^2),  s_down = sqrt(sigma'^2 - s_up^2)
        x' = x + (s_down - sigma) eps + s_up z
      z ~ N(0, 1), drawn as diffusers' randn_tensor draws it (`noise`), on every step: also on the last one, where
      sigma' = 0 and so s_up = 0.
    Not a subclass of EulerDiscreteScheduler: its `dt` is not this scheduler's step. The samplers run it through the
    fused blend kernels with the coefficients of `ancestral_coeffs(i)`."""
    order = 1
    _defaults = dict(num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear",
                     trained_betas=None, prediction_type="epsilon", timestep_spacing="leading", steps_offset=1)
    _unsupported = dict(trained_betas=None, prediction_type="epsilon", timestep_spacing="leading")

    def __init__(self, **kw):
        cfg = self._configure(kw)
        self._grid = EulerDiscreteScheduler(cfg["beta_start"], cfg["beta_end"], int(cfg["num_train_timesteps"]),
                                            int(cfg["steps_offset"]))
        self.num_train_timesteps = self._grid.num_train_timesteps
        self.alphas_cumprod = self._grid.alphas_cumprod
        self.num_inference_steps = None
        self._take_grid()

    def _take_grid(self):
        self.timesteps, self.timesteps_host, self.sigmas_host = \
            self._grid.timesteps, self._grid.timesteps_host, self._grid.sigmas_host

    @property
    def init_noise_sigma(self):
        return self._grid.init_noise_sigma

    def set_timesteps(self, num_inference_steps, device=None):
        self._grid.set_timesteps(num_inference_steps, device)
        self.num_inference_steps = num_inference_steps
        self._take_grid()

    def index_of(self, timestep):
        return self._grid.index_of(timestep)

    def sigma(self, timestep):
        return self._grid.sigma(timestep)

    def scale_model_input(self, sample, timestep):
        return self._grid.scale_model_input(sample, timestep)

    def ancestral_coeffs(self, i):
        """(dt, s_up) of step i in float64: x' = x + dt eps + s_up z, dt = s_down - sigma."""
        s, s_to = float(self.sigmas_host[i]), float(self.sigmas_host[i + 1])
        s_up = math.sqrt(s_to * s_to * (s * s - s_to * s_to) / (s * s))
        s_down = math.sqrt(s_to * s_to - s_up * s_up)
        return s_down - s, s_up

    @staticmethod
    def noise(shape, generator=None, device=None, dtype=torch.float16):
        """z of one step as diffusers' randn_tensor draws it: from `generator` on the generator's device (a CPU generator
        draws on the CPU and the result is copied to `device`), or, without one, from the global RNG of `device`."""
        if generator is None:
            return torch.randn(shape, dtype=dtype, device=device)
        return torch.randn(shape, dtype=dtype, generator=generator, device=generator.device).to(device)

    def step(self, model_output, timestep, sample, generator=None, return_dict=True, **kw):
        """Torch form of ancestral_coeffs (the samplers use the fused kernels instead); z has model_output's shape and
        dtype."""
        dt, s_up = self.ancestral_coeffs(self.index_of(timestep))
        z = self.noise(model_output.shape, generator, model_output.device, model_output.dtype)
        prev = (sample.float() + model_output.float() * dt + z.float() * s_up).to(sample.dtype)
        return {"prev_sample": prev} if return_dict else (prev,)


# ---------------------------------------------------------------------------------------------------- Heun
class HeunDiscreteScheduler(_Configured):
    """Heun's method (Karras et al., EDM, Algorithm 1 without churn), epsilon prediction, with the SDXL config
    (scaled-linear betas 0.00085-0.012, `leading` spacing, steps_offset=1), restating diffusers 0.18.2
    (`schedulers/scheduling_heun_discrete.py`). PARITY UNPINNED: that source is not available here; the conventions
    below are the definition.
      From Euler's grid for N steps, t_0..t_{N-1} and s_0..s_{N-1}, 0 (EulerDiscreteScheduler.set_timesteps):
        timesteps   = [t_0, t_1, t_1, ..., t_{N-1}, t_{N-1}]      2N - 1 loop iterations
        sigmas_host = [s_0, s_1, s_1, ..., s_{N-1}, s_{N-1}, 0]   2N entries
      num_inference_steps = N, order = 2; init_noise_sigma = sqrt(s_max^2 + 1), Euler's (the value of `leading`
      spacing, also unpinned); alphas_cumprod: Euler's.
      Iteration k, sigma_k = sigmas_host[k] (indexed by k: the timestep values repeat); the UNet sees
      x / sqrt(sigma_k^2 + 1).
        k even, first stage:  x' = x + (sigma_{k+1} - sigma_k) eps;  keeps xs = x, ds = eps, dt = sigma_{k+1} - sigma_k
        k odd, second stage:  x' = xs + dt/2 (ds + eps)
      The last iteration, k = 2N - 2, is a first stage to sigma = 0 (a plain Euler step); its saved state is never used.
    The second stage restarts from xs, so the current latents reach it only through eps: whatever a sampling loop does
    to the latents between the two stages (colour guidance, background injection) is overwritten, as in diffusers. The
    samplers run it through the fused blend kernels with the coefficients of `heun_coeffs(k)` and the fp16 xs and ds of
    each trajectory (ops.HeunStep); `step` is the stateful torch form in diffusers' calling convention."""
    order = 2
    _defaults = dict(num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear",
                     trained_betas=None, prediction_type="epsilon", use_karras_sigmas=False,
                     timestep_spacing="leading", steps_offset=1)
    _unsupported = dict(trained_betas=None, prediction_type="epsilon", use_karras_sigmas=False,
                        timestep_spacing="leading")

    def __init__(self, **kw):
        cfg = self._configure(kw)
        self._grid = EulerDiscreteScheduler(cfg["beta_start"], cfg["beta_end"], int(cfg["num_train_timesteps"]),
                                            int(cfg["steps_offset"]))
        self.num_train_timesteps = self._grid.num_train_timesteps
        self.alphas_cumprod = self._grid.alphas_cumprod
        self.num_inference_steps = None
        self.timesteps_host, self.sigmas_host = self._grid.timesteps_host, self._grid.sigmas_host
        self.timesteps = self._grid.timesteps
        self._reset()

    def _reset(self):
        self._k, self._xs, self._ds, self._dt = 0, None, None, None

    @property
    def init_noise_sigma(self):
        return self._grid.init_noise_sigma

    def set_timesteps(self, num_inference_steps, device=None):
        g = self._grid
        g.set_timesteps(num_inference_steps, device)
        self.num_inference_steps = num_inference_steps
        self.timesteps_host = np.concatenate([g.timesteps_host[:1], np.repeat(g.timesteps_host[1:], 2)])
        self.sigmas_host = np.concatenate([g.sigmas_host[:1], np.repeat(g.sigmas_host[1:-1], 2),
                                           g.sigmas_host[-1:]]).astype(np.float32)
        self.timesteps = torch.from_numpy(self.timesteps_host.copy())   # host tensor, as Euler's
        self._reset()

    @staticmethod
    def is_first_stage(k):
        return k % 2 == 0

    @property
    def state_in_first_order(self):
        """Whether the next `step` call is a first stage (diffusers' name)."""
        return self._dt is None

    def sigma_at(self, k):
        return float(self.sigmas_host[k])

    def scale_model_input(self, sample, timestep):
        """x / sqrt(sigma^2 + 1) at the iteration the next `step` call makes."""
        s = self.sigma_at(self._k)
        return sample / ((s * s + 1.0) ** 0.5)

    def heun_coeffs(self, k):
        """(cx, ce, cs, cd) of iteration k in float64: x' = cx x + ce eps + cs xs + cd ds; (1, dt, 0, 0) at a first
        stage, (0, dt/2, 1, dt/2) at a second, dt = sigma_{k+1} - sigma_k of the first stage."""
        if self.is_first_stage(k):
            return 1.0, float(self.sigmas_host[k + 1]) - float(self.sigmas_host[k]), 0.0, 0.0
        dt = float(self.sigmas_host[k]) - float(self.sigmas_host[k - 1])
        return 0.0, 0.5 * dt, 1.0, 0.5 * dt

    def step(self, model_output, timestep, sample, return_dict=True, **kw):
        """Stateful torch form of heun_coeffs in diffusers' calling convention (the samplers use the fused kernels
        instead): the stage follows from the calls made since set_timesteps, as diffusers' state_in_first_order, and
        `timestep` must be the loop's timestep of that call. Evaluated in the precision of `sample` and at least fp32."""
        k = self._k
        if float(timestep) != float(self.timesteps_host[k]):
            raise ValueError(f"HeunDiscreteScheduler.step: timestep {float(timestep)} is not that of iteration {k} "
                             f"({float(self.timesteps_host[k])})")
        cx, ce, cs, cd = self.heun_coeffs(k)
        dtype = torch.promote_types(sample.dtype, torch.float32)
        x, e = sample.to(dtype), model_output.to(dtype)
        if self.is_first_stage(k):
            prev = cx * x + ce * e
            self._xs, self._ds, self._dt = x, e, 2.0 * ce
        else:
            prev = self._xs + ce * (self._ds + e)
            self._xs = self._ds = self._dt = None
        self._k = k + 1
        prev = prev.to(sample.dtype)
        return {"prev_sample": prev} if return_dict else (prev,)


# ---------------------------------------------------------------------------------------------------- LMS
class LMSDiscreteScheduler(_Configured):
    """k-LMS, the linear multistep method of order 4 on the probability-flow ODE dx/dsigma = eps, epsilon prediction, with
    the SDXL config (scaled-linear betas 0.00085-0.012, `leading` spacing, steps_offset=1), restating diffusers 0.18.2
    (`schedulers/scheduling_lms_discrete.py`, `step(order=4)`). PARITY UNPINNED: that source is not available here; the
    conventions below are the definition.
      timesteps, sigmas_host (s_0..s_{N-1}, 0), init_noise_sigma, scale_model_input, alphas_cumprod: those of
      EulerDiscreteScheduler. order = 1: one UNet evaluation per step.
      step i, with eps_i the step's prediction and p = min(i + 1, 4):
        x' = x + sum_{k<p} c_k eps_{i-k},   c_k = integral from s_i to s_{i+1} of l_k(tau) dtau
      where l_k is the Lagrange basis polynomial on the nodes s_i, s_{i-1}, ..., s_{i-p+1} with l_k(s_{i-k}) = 1.
    diffusers integrates l_k with scipy.integrate.quad on a float32 integrand; `lms_coeffs` integrates it in closed form
    in float64 from the same float32 nodes. Every step starts from the current latents, so whatever a sampling loop does
    to the latents between steps (colour guidance, background injection) carries into the next update in full. Not a
    subclass of EulerDiscreteScheduler: its `dt` is not this scheduler's step. The samplers run it through the fused
    blend kernels with the coefficients of `lms_coeffs(i)` and the fp16 predictions of each trajectory's last three
    steps (ops.LMSStep); `step` is the stateful torch form in diffusers' calling convention."""
    order = 1
    max_order = 4
    _defaults = dict(num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear",
                     trained_betas=None, prediction_type="epsilon", use_karras_sigmas=False,
                     timestep_spacing="leading", steps_offset=1)
    _unsupported = dict(trained_betas=None, prediction_type="epsilon", use_karras_sigmas=False,
                        timestep_spacing="leading")

    def __init__(self, **kw):
        cfg = self._configure(kw)
        self._grid = EulerDiscreteScheduler(cfg["beta_start"], cfg["beta_end"], int(cfg["num_train_timesteps"]),
                                            int(cfg["steps_offset"]))
        self.num_train_timesteps = self._grid.num_train_timesteps
        self.alphas_cumprod = self._grid.alphas_cumprod
        self.num_inference_steps = None
        self._take_grid()

    def _take_grid(self):
        self.timesteps, self.timesteps_host, self.sigmas_host = \
            self._grid.timesteps, self._grid.timesteps_host, self._grid.sigmas_host
        self.derivatives = []

    @property
    def init_noise_sigma(self):
        return self._grid.init_noise_sigma

    def set_timesteps(self, num_inference_steps, device=None):
        self._grid.set_timesteps(num_inference_steps, device)
        self.num_inference_steps = num_inference_steps
        self._take_grid()

    def index_of(self, timestep):
        return self._grid.index_of(timestep)

    def sigma(self, timestep):
        return self._grid.sigma(timestep)

    def scale_model_input(self, sample, timestep):
        return self._grid.scale_model_input(sample, timestep)

    def lms_coeffs(self, i):
        """(c0, c1, c2, c3) of step i in float64: x' = x + c0 eps_i + c1 eps_{i-1} + c2 eps_{i-2} + c3 eps_{i-3};
        c_k = 0 for k >= min(i + 1, 4). Their sum is sigma_{i+1} - sigma_i."""
        sig = self.sigmas_host
        p = min(i + 1, self.max_order)
        nodes = [float(sig[i - j]) for j in range(p)]
        lo, hi = float(sig[i]), float(sig[i + 1])
        out = [0.0] * self.max_order
        for k in range(p):
            basis = np.array([1.0])
            for j in range(p):
                if j != k:
                    basis = np.polynomial.polynomial.polymul(basis, np.array([-nodes[j], 1.0]) / (nodes[k] - nodes[j]))
            prim = np.polynomial.polynomial.polyint(basis)
            out[k] = float(np.polynomial.polynomial.polyval(hi, prim) - np.polynomial.polynomial.polyval(lo, prim))
        return tuple(out)

    def step(self, model_output, timestep, sample, return_dict=True, **kw):
        """Stateful torch form of lms_coeffs in diffusers' calling convention (the samplers use the fused kernels
        instead): keeps the predictions of the last four calls since set_timesteps. Evaluated in the precision of
        `sample` and at least fp32."""
        i = self.index_of(timestep)
        dtype = torch.promote_types(sample.dtype, torch.float32)
        self.derivatives = [model_output.to(dtype)] + self.derivatives[:self.max_order - 1]
        prev = sample.to(dtype)
        for c, d in zip(self.lms_coeffs(i), self.derivatives):
            if c != 0.0:
                prev = prev + c * d
        prev = prev.to(sample.dtype)
        return {"prev_sample": prev} if return_dict else (prev,)
