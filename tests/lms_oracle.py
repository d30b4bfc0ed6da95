"""TEST INFRASTRUCTURE — restatement of diffusers 0.18.2's LMSDiscreteScheduler (epsilon prediction, the SDXL config,
no Karras sigmas, `step(order=4)`) in the form diffusers evaluates it, for the oracle loops and for tests/gen_lms.py.

PARITY UNPINNED: the diffusers source is not available here (the reference pins diffusers==0.18.2, environment.yaml).
The arithmetic follows that version's `schedulers/scheduling_lms_discrete.py` step by step, independently of the
product's `lms_coeffs`: fp32 torch sigmas, the step index from the timestep, pred_original_sample = sample - sigma eps,
the derivative (sample - pred_original_sample) / sigma (eps up to rounding), a derivative list that drops its oldest
entry past 4, and each coefficient from scipy.integrate.quad (epsrel 1e-4) of the Lagrange basis evaluated on the
float32 sigmas. The grid is oracle/schedulers_oracle.py's Euler grid (`leading` spacing, steps_offset 1). The same class
is assigned to `m.scheduler` of the unmodified reference by tests/gen_lms.py, so what the goldens pin is the reference's
loop logic — which scheduler calls it makes, in which order, and when it calls back — with this scheduler.
"""
import torch
from scipy import integrate

from oracle import schedulers_oracle as so
from tests.heun_oracle import callback_iterations, plain_loop, rich_text_loop  # noqa: F401  (the same loops)


class LMSSchedulerOracle:
    order = 1

    def __init__(self):
        self._euler = so.EulerDiscreteSchedulerOracle()
        self.alphas_cumprod = self._euler.alphas_cumprod
        self.sigmas, self.timesteps = self._euler.sigmas, self._euler.timesteps
        self.derivatives = []
        self.step_batches = []   # the batch size of every step call, in order

    @property
    def init_noise_sigma(self):
        return (self.sigmas.max() ** 2 + 1) ** 0.5

    def set_timesteps(self, num_inference_steps, device=None):
        e = self._euler
        e.set_timesteps(num_inference_steps)
        self.num_inference_steps = num_inference_steps
        self.sigmas, self.timesteps = e.sigmas, e.timesteps
        self.derivatives = []

    def _index(self, timestep):
        return int((self.timesteps == timestep).nonzero().item())

    def scale_model_input(self, sample, timestep):
        sigma = self.sigmas[self._index(timestep)]
        return sample / ((sigma ** 2 + 1) ** 0.5)

    def get_lms_coefficient(self, order, t, current_order):
        def lms_derivative(tau):
            prod = 1.0
            for k in range(order):
                if current_order == k:
                    continue
                prod *= (tau - self.sigmas[t - k]) / (self.sigmas[t - current_order] - self.sigmas[t - k])
            return prod
        return integrate.quad(lms_derivative, self.sigmas[t], self.sigmas[t + 1], epsrel=1e-4)[0]

    def step(self, model_output, timestep, sample, order=4, return_dict=True, **kw):
        self.step_batches.append(int(sample.shape[0]))
        step_index = self._index(timestep)
        sigma = self.sigmas[step_index]
        pred_original_sample = sample - sigma * model_output
        derivative = (sample - pred_original_sample) / sigma
        self.derivatives.append(derivative)
        if len(self.derivatives) > order:
            self.derivatives.pop(0)
        order = min(step_index + 1, order)
        lms_coeffs = [self.get_lms_coefficient(order, step_index, cur) for cur in range(order)]
        prev_sample = sample + sum(coeff * d for coeff, d in zip(lms_coeffs, reversed(self.derivatives)))
        return {"prev_sample": prev_sample, "pred_original_sample": pred_original_sample} if return_dict \
            else (prev_sample,)


class PerTrajectoryLMSOracle(LMSSchedulerOracle):
    """The product's rule for the rich-text loop: a batch-2 step (main, reference) steps each trajectory on its own
    LMSSchedulerOracle, a batch-1 step the main one alone. Where the reference loop steps both jointly on every step it
    equals one batch-2 scheduler; where it steps them jointly only on a prefix, the main latents keep their own history
    here instead of continuing a batch-2 one."""

    def __init__(self):
        super().__init__()
        self.main, self.ref = LMSSchedulerOracle(), LMSSchedulerOracle()

    def set_timesteps(self, num_inference_steps, device=None):
        super().set_timesteps(num_inference_steps, device)
        self.main.set_timesteps(num_inference_steps, device)
        self.ref.set_timesteps(num_inference_steps, device)

    def step(self, model_output, timestep, sample, return_dict=True, **kw):
        self.step_batches.append(int(sample.shape[0]))
        out = self.main.step(model_output[:1], timestep, sample[:1])["prev_sample"]
        if sample.shape[0] == 2:
            out = torch.cat([out, self.ref.step(model_output[1:], timestep, sample[1:])["prev_sample"]])
        return {"prev_sample": out} if return_dict else (out,)
