"""TEST INFRASTRUCTURE — restatement of diffusers 0.18.2's DPMSolverSinglestepScheduler (DPM-Solver++(2S):
algorithm_type "dpmsolver++", solver_order 2, solver_type "midpoint", lower_order_final, no Karras sigmas, epsilon
prediction, the SD1.5 / SDXL betas) in the form diffusers evaluates it, for the oracle loops and for
tests/gen_singlestep.py.

PARITY UNPINNED: the diffusers source is not available here (the reference pins diffusers==0.18.2, environment.yaml).
The arithmetic follows that version's `schedulers/scheduling_dpmsolver_singlestep.py` step by step, independently of
the product's closed-form `singlestep_coeffs`: fp32 torch alpha_t / sigma_t / lambda_t, the order list, the stateful
model-output list, `self.sample` saved on first-order steps, `exp(-h) - 1`, and the second-order update written with
D0 = m1 and D1 = (m0 - m1) / r0. The timesteps are DPM-Solver++(2M)'s (tests/multistep_oracle.py). The same class is
assigned to `m.scheduler` of the unmodified reference by tests/gen_singlestep.py, so what the goldens pin is the
reference's loop logic — which scheduler calls it makes, in which order, and when it calls back — with this scheduler.
The loops are tests/multistep_oracle.py's (scale_model_input is the identity).
"""
import torch

from tests.multistep_oracle import DPMSolverMultistepSchedulerOracle, _Out, plain_loop, rich_text_loop  # noqa: F401


class DPMSolverSinglestepSchedulerOracle(DPMSolverMultistepSchedulerOracle):
    order = 1
    init_noise_sigma = 1.0

    def __init__(self, num_train_timesteps=1000):
        super().__init__(num_train_timesteps)
        self.step_batches = []   # the batch size of every step call, in order

    @staticmethod
    def get_order_list(steps):
        return [1, 2] * (steps // 2) + ([1] if steps % 2 else [])

    def set_timesteps(self, num_inference_steps, device=None):
        super().set_timesteps(num_inference_steps, device)
        self.order_list = self.get_order_list(len(self.timesteps))
        self.sample = None

    def _second_2s(self, timestep_list, prev_timestep, sample):
        t, s0, s1 = prev_timestep, timestep_list[-1], timestep_list[-2]
        m0, m1 = self.model_outputs[-1], self.model_outputs[-2]
        lambda_t, lambda_s0, lambda_s1 = self.lambda_t[t], self.lambda_t[s0], self.lambda_t[s1]
        alpha_t, sigma_t, sigma_s1 = self.alpha_t[t], self.sigma_t[t], self.sigma_t[s1]
        h, h_0 = lambda_t - lambda_s1, lambda_s0 - lambda_s1
        r0 = h_0 / h
        D0, D1 = m1, (1.0 / r0) * (m0 - m1)
        return (sigma_t / sigma_s1) * sample - (alpha_t * (torch.exp(-h) - 1.0)) * D0 \
            - 0.5 * (alpha_t * (torch.exp(-h) - 1.0)) * D1

    def step(self, model_output, timestep, sample, generator=None, return_dict=True, **kw):
        self.step_batches.append(int(sample.shape[0]))
        timestep = int(timestep)
        idx = (self.timesteps == timestep).nonzero()
        step_index = len(self.timesteps) - 1 if len(idx) == 0 else int(idx.item())
        prev_timestep = 0 if step_index == len(self.timesteps) - 1 else int(self.timesteps[step_index + 1])
        m = self._x0(model_output, timestep, sample)
        self.model_outputs = [self.model_outputs[1], m]
        order = self.order_list[step_index]
        while self.model_outputs[-order] is None:
            order -= 1
        if order == 1:
            self.sample = sample
            prev = self._first(m, timestep, prev_timestep, self.sample)
        else:
            timestep_list = [int(self.timesteps[step_index - 1]), timestep]
            prev = self._second_2s(timestep_list, prev_timestep, self.sample)
        return _Out(prev_sample=prev) if return_dict else (prev,)


def callback_iterations(n_iterations, callback_steps=1):
    """The iterations at which the reference calls back with an order-1 scheduler (:874-877)."""
    return [i for i in range(n_iterations) if i % callback_steps == 0]
