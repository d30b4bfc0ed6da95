"""TEST INFRASTRUCTURE — restatement of diffusers 0.18.2's UniPCMultistepScheduler (solver_type "bh2", solver_order 2,
predict_x0, lower_order_final, no disabled corrector, no solver_p, epsilon prediction) in the form diffusers evaluates
it, with the SD1.5 / SDXL betas.

PARITY UNPINNED: the diffusers sources are not available here (the reference pins diffusers==0.18.2,
environment.yaml). The arithmetic below follows that version's `schedulers/scheduling_unipc_multistep.py` step by step:
the stateful `model_outputs` / `timestep_list` / `last_sample` / `lower_order_nums` / `this_order`, the UniC corrector
before the UniP predictor, the rks / R / b construction with the h_phi_k recursion, `rhos_c` from torch.linalg.solve
(order 2) or 0.5 (order 1), `rhos_p` = 0.5 at order 2. It is written independently of the product's closed-form
`unipc_coeffs`. diffusers keeps alpha_t / sigma_t / lambda_t in fp32; `dtype=torch.float64` builds them (from the same
fp32 alphas_cumprod) in float64 instead, for the float64 comparison with unipc_coeffs. The same class is assigned to
`m.scheduler` of the unmodified reference by tests/gen_unipc.py, so what the goldens pin is the reference's loop logic
with this scheduler.
"""
import numpy as np
import torch

from tests import multistep_oracle as mo


class UniPCSchedulerOracle:
    order = 1
    init_noise_sigma = 1.0

    def __init__(self, num_train_timesteps=1000, dtype=torch.float32):
        self.num_train_timesteps = num_train_timesteps
        self.alphas_cumprod = mo._alphas_cumprod(n=num_train_timesteps)
        ac = self.alphas_cumprod.to(dtype)
        self.alpha_t = torch.sqrt(ac)
        self.sigma_t = torch.sqrt(1 - ac)
        self.lambda_t = torch.log(self.alpha_t) - torch.log(self.sigma_t)
        self.solver_order = 2
        self.timesteps = None

    def set_timesteps(self, num_inference_steps, device=None):
        ts = np.linspace(0, self.num_train_timesteps - 1, num_inference_steps + 1).round()[::-1][:-1].copy()
        ts = ts.astype(np.int64)
        _, idx = np.unique(ts, return_index=True)
        ts = ts[np.sort(idx)]
        self.timesteps = torch.from_numpy(ts)
        self.num_inference_steps = len(ts)
        self.model_outputs = [None] * self.solver_order
        self.timestep_list = [None] * self.solver_order
        self.lower_order_nums = 0
        self.last_sample = None
        self.this_order = None

    def scale_model_input(self, sample, timestep=None):
        return sample

    def convert_model_output(self, model_output, timestep, sample):
        return (sample - self.sigma_t[timestep] * model_output) / self.alpha_t[timestep]

    def _b(self, hh, order):
        """b_k = h_phi_k * k! / B_h, k = 1..order (bh2: B_h = expm1(hh))."""
        h_phi_1 = torch.expm1(hh)
        h_phi_k = h_phi_1 / hh - 1
        factorial_i = 1
        B_h = torch.expm1(hh)
        b = []
        for i in range(1, order + 1):
            b.append(h_phi_k * factorial_i / B_h)
            factorial_i *= i + 1
            h_phi_k = h_phi_k / hh - 1 / factorial_i
        return h_phi_1, B_h, torch.stack(b)

    def multistep_uni_p_bh_update(self, model_output, prev_timestep, sample, order):
        s0, t = self.timestep_list[-1], prev_timestep
        m0 = self.model_outputs[-1]
        x = sample
        lambda_t, lambda_s0 = self.lambda_t[t], self.lambda_t[s0]
        alpha_t, sigma_t, sigma_s0 = self.alpha_t[t], self.sigma_t[t], self.sigma_t[s0]
        h = lambda_t - lambda_s0
        D1s = []
        for i in range(1, order):
            si = self.timestep_list[-(i + 1)]
            mi = self.model_outputs[-(i + 1)]
            rk = (self.lambda_t[si] - lambda_s0) / h
            D1s.append((mi - m0) / rk)
        hh = -h
        h_phi_1, B_h, _ = self._b(hh, order)
        x_t_ = sigma_t / sigma_s0 * x - alpha_t * h_phi_1 * m0
        if D1s:
            rhos_p = torch.tensor([0.5], dtype=x.dtype)      # order 2: diffusers' simplified form
            pred_res = sum(r * d for r, d in zip(rhos_p, D1s))   # diffusers' einsum over k
            x_t = x_t_ - alpha_t * B_h * pred_res
        else:
            x_t = x_t_
        return x_t.to(x.dtype)

    def multistep_uni_c_bh_update(self, this_model_output, this_timestep, last_sample, this_sample, order):
        s0, t = self.timestep_list[-1], this_timestep
        m0 = self.model_outputs[-1]
        x = last_sample
        model_t = this_model_output
        lambda_t, lambda_s0 = self.lambda_t[t], self.lambda_t[s0]
        alpha_t, sigma_t, sigma_s0 = self.alpha_t[t], self.sigma_t[t], self.sigma_t[s0]
        h = lambda_t - lambda_s0
        rks, D1s = [], []
        for i in range(1, order):
            si = self.timestep_list[-(i + 1)]
            mi = self.model_outputs[-(i + 1)]
            rk = (self.lambda_t[si] - lambda_s0) / h
            rks.append(rk)
            D1s.append((mi - m0) / rk)
        rks.append(torch.ones((), dtype=h.dtype))
        rks = torch.stack(rks)
        hh = -h
        h_phi_1, B_h, b = self._b(hh, order)
        R = torch.stack([torch.pow(rks, i - 1) for i in range(1, order + 1)])
        if order == 1:
            rhos_c = torch.tensor([0.5], dtype=x.dtype)
        else:
            rhos_c = torch.linalg.solve(R, b)
        x_t_ = sigma_t / sigma_s0 * x - alpha_t * h_phi_1 * m0
        corr_res = sum(r * d for r, d in zip(rhos_c[:-1], D1s)) if D1s else 0   # diffusers' einsum over k
        D1_t = model_t - m0
        x_t = x_t_ - alpha_t * B_h * (corr_res + rhos_c[-1] * D1_t)
        return x_t.to(x.dtype)

    def step(self, model_output, timestep, sample, return_dict=True, **kw):
        timestep = int(timestep)
        idx = (self.timesteps == timestep).nonzero()
        step_index = len(self.timesteps) - 1 if len(idx) == 0 else int(idx.item())
        use_corrector = step_index > 0 and self.last_sample is not None
        model_output_convert = self.convert_model_output(model_output, timestep, sample)
        if use_corrector:
            sample = self.multistep_uni_c_bh_update(model_output_convert, timestep, self.last_sample, sample,
                                                    self.this_order)
        prev_timestep = 0 if step_index == len(self.timesteps) - 1 else int(self.timesteps[step_index + 1])
        for i in range(self.solver_order - 1):
            self.model_outputs[i] = self.model_outputs[i + 1]
            self.timestep_list[i] = self.timestep_list[i + 1]
        self.model_outputs[-1] = model_output_convert
        self.timestep_list[-1] = timestep
        this_order = min(self.solver_order, len(self.timesteps) - step_index)     # lower_order_final
        self.this_order = min(this_order, self.lower_order_nums + 1)              # warm-up
        self.last_sample = sample
        prev_sample = self.multistep_uni_p_bh_update(model_output, prev_timestep, sample, self.this_order)
        if self.lower_order_nums < self.solver_order:
            self.lower_order_nums += 1
        return mo._Out(prev_sample=prev_sample) if return_dict else (prev_sample,)
