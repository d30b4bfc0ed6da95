"""The scheduler updates the region-blend kernels fuse, as the samplers drive them.

The blend kernels (ops.region_blend_cfg, ops.gather_blend_step) take the scheduler update of the latents in one of
seven forms (_lib.BLEND_FORMS): the plain Euler one, "_ms" for DDIM / DPM-Solver++(2M), which keep one fp32 history of
the x0 prediction per trajectory, "_anc" for Euler Ancestral, which adds the noise drawn for the step, "_unipc" for
UniPC, which keeps three fp32 histories per trajectory, "_heun" for Heun's method, which reads the fp16 latents and
prediction saved at the first stage, "_lms" for k-LMS, which reads the fp16 predictions of the last three steps, and
"_ss" for DPM-Solver++(2S), which keeps one fp32 history of the x0 prediction per trajectory and reads the fp16 latents
that entered the two-step block.

A Stepper owns what a sampling loop needs for one of them: the UNet input scaling, the state of each trajectory (the
main latents, and the reference latents of the rich-text pass), the ops step object of each blend call and the update
of the state after it. A loop calls, per step: input_norm() before the UNet pass, begin() after it, step() per
trajectory (split blends) or step_pair() (one fused gather-blend over both), and advance() for every trajectory that
stepped, with the contiguous latents handed to the blend and the stepped prediction it returned.
"""
import math

import torch

from . import ops
from .schedulers import (MULTISTEP_SCHEDULERS, DPMSolverSinglestepScheduler, EulerAncestralDiscreteScheduler,
                         EulerDiscreteScheduler, HeunDiscreteScheduler, LMSDiscreteScheduler, UniPCMultistepScheduler)


class Stepper:
    """The fused update of one sampling call for latents of `shape` (one trajectory's); `generator`: the source of
    Euler Ancestral's noise (None: the global RNG of `device`)."""
    scaled = True    # the UNet sees latents / sqrt(sigma^2 + 1) (scale_model_input)

    def __init__(self, scheduler, shape, device, generator=None):
        self.scheduler, self.shape, self.device, self.generator = scheduler, tuple(shape), device, generator
        self.n = math.prod(self.shape)

    def state(self):
        """A fresh state of one trajectory."""
        return None

    def input_norm(self, i, t):
        """sqrt(sigma^2 + 1), the divisor of the UNet input at iteration i, or None where the input is not scaled."""
        if not self.scaled:
            return None
        sigma = self.scheduler.sigma(t)
        return math.sqrt(sigma * sigma + 1.0)

    def begin(self, i, t, n_traj):
        """Start iteration i (after its UNet pass), which steps `n_traj` trajectories (main first)."""
        self.t = t

    def step(self, s, k=0):
        """The ops step of a blend call that steps trajectory k (0 = main, 1 = reference) in state s alone."""
        raise NotImplementedError

    def step_pair(self, s, s_ref, ref_steps, eps_ref_out=None):
        """The ops step of a gather-blend call over the main trajectory and the reference one (state s_ref, None when
        there is none), which steps only when `ref_steps`; eps_ref_out: an fp16 tensor of the reference latents' shape
        where writes_eps_ref(), else None."""
        raise NotImplementedError

    def writes_eps_ref(self):
        """Whether a fused call that steps the reference trajectory needs eps_ref_out (its stepped prediction)."""
        return False

    def advance(self, s, lat, eps):
        """The state after a blend stepped the trajectory: `lat` the latents handed to it, `eps` the stepped prediction
        it returned. States holding buffers may be updated in place."""
        return s


class _Euler(Stepper):
    def step(self, s, k=0):
        return ops.EulerStep(self.scheduler.dt(self.t))

    def step_pair(self, s, s_ref, ref_steps, eps_ref_out=None):
        return self.step(s)


class _Ancestral(Stepper):
    def begin(self, i, t, n_traj):
        # one draw per step, after the UNet pass: [2, ...] when both trajectories step as one batch (main first), as the
        # reference draws it; on CUDA one [2, n] draw differs from two [1, n] draws
        super().begin(i, t, n_traj)
        self.coeffs = self.scheduler.ancestral_coeffs(i)
        self.z = self.scheduler.noise((n_traj,) + self.shape[1:], self.generator, self.device)

    def step(self, s, k=0):
        return ops.AncestralStep(*self.coeffs, self.z[k:k + 1])

    def step_pair(self, s, s_ref, ref_steps, eps_ref_out=None):
        return ops.AncestralStep(*self.coeffs, self.z[0:1], self.z[1:2] if ref_steps else None)


class _Multistep(Stepper):
    """State: the fp32 D buffer (read and written in place)."""
    scaled = False

    def state(self):
        return torch.empty(self.n, dtype=torch.float32, device=self.device)

    def begin(self, i, t, n_traj):
        super().begin(i, t, n_traj)
        self.coeffs = self.scheduler.step_coeffs(i)

    def step(self, s, k=0):
        return ops.MultistepStep(self.coeffs, s, s)

    def step_pair(self, s, s_ref, ref_steps, eps_ref_out=None):
        # the reference D buffer goes along whenever the trajectory exists; the kernel reads it only when it steps
        return ops.MultistepStep(self.coeffs, s, s, s_ref, s_ref)


class _UniPC(Stepper):
    """State: an ops.UniPCHistory; the step's x0 prediction becomes its m1 after the blend."""
    scaled = False

    def state(self):
        return ops.UniPCHistory(self.n, self.device)

    def begin(self, i, t, n_traj):
        super().begin(i, t, n_traj)
        self.coeffs = self.scheduler.unipc_coeffs(i)

    def step(self, s, k=0):
        return ops.UniPCStep.of(self.coeffs, s)

    def step_pair(self, s, s_ref, ref_steps, eps_ref_out=None):
        return ops.UniPCStep.of(self.coeffs, s, s_ref if ref_steps else None)

    def advance(self, s, lat, eps):
        s.rotate()
        return s


class _Heun(Stepper):
    """State: (xs, ds), the latents and the stepped prediction of the trajectory's last first stage, fp16, referenced
    until the second stage reads them (the blend writes fresh outputs; nothing writes them in place). A first stage
    passes the previous block's (xs, ds) with cs = cd = 0, so they are not read."""

    def state(self):
        return None, None

    def input_norm(self, i, t):
        sigma = self.scheduler.sigma_at(i)
        return math.sqrt(sigma * sigma + 1.0)

    def begin(self, i, t, n_traj):
        super().begin(i, t, n_traj)
        self.coeffs = self.scheduler.heun_coeffs(i)
        self.first = self.scheduler.is_first_stage(i)

    def step(self, s, k=0):
        return ops.HeunStep(self.coeffs, *s)

    def step_pair(self, s, s_ref, ref_steps, eps_ref_out=None):
        return ops.HeunStep(self.coeffs, *s, *(s_ref if ref_steps else (None, None)), eps_ref_out)

    def writes_eps_ref(self):
        return self.first

    def advance(self, s, lat, eps):
        return (lat, eps) if self.first else s


class _LMS(Stepper):
    """State: the fp16 stepped predictions of the trajectory's last three steps, newest first (blend outputs,
    referenced while they are in the history; nothing writes them in place)."""

    def state(self):
        return None, None, None

    def begin(self, i, t, n_traj):
        super().begin(i, t, n_traj)
        self.coeffs = self.scheduler.lms_coeffs(i)

    def step(self, s, k=0):
        return ops.LMSStep(self.coeffs, *s)

    def step_pair(self, s, s_ref, ref_steps, eps_ref_out=None):
        return ops.LMSStep(self.coeffs, *s, *(s_ref if ref_steps else (None, None, None)), eps_ref_out)

    def writes_eps_ref(self):
        return True

    def advance(self, s, lat, eps):
        return (eps,) + s[:2]


class _Singlestep(Stepper):
    """State: (D, xs), the fp32 D buffer (read and written in place) and the fp16 latents that entered the current
    block's first step (referenced until its second step reads them)."""
    scaled = False

    def state(self):
        return torch.empty(self.n, dtype=torch.float32, device=self.device), None

    def begin(self, i, t, n_traj):
        super().begin(i, t, n_traj)
        self.coeffs = self.scheduler.singlestep_coeffs(i)
        self.first = self.scheduler.is_first_step(i)

    def step(self, s, k=0):
        d, xs = s
        return ops.SinglestepStep(self.coeffs, d, d, xs)

    def step_pair(self, s, s_ref, ref_steps, eps_ref_out=None):
        (d, xs), (d_ref, xs_ref) = s, (s_ref or (None, None))
        return ops.SinglestepStep(self.coeffs, d, d, xs, d_ref, d_ref, xs_ref if ref_steps else None)

    def advance(self, s, lat, eps):
        return (s[0], lat) if self.first else s


# checked in this order: a subclass before its base
_KINDS = ((DPMSolverSinglestepScheduler, "singlestep", _Singlestep), (LMSDiscreteScheduler, "lms", _LMS),
          (HeunDiscreteScheduler, "heun", _Heun), (UniPCMultistepScheduler, "unipc", _UniPC),
          (EulerAncestralDiscreteScheduler, "ancestral", _Ancestral), (EulerDiscreteScheduler, "euler", _Euler),
          (MULTISTEP_SCHEDULERS, "multistep", _Multistep))


def _step_kind(scheduler):
    """The fused update a scheduler runs as: "euler" (EulerDiscreteScheduler), "ancestral"
    (EulerAncestralDiscreteScheduler: the Euler update plus the noise term, ancestral_coeffs), "multistep"
    (DDIMScheduler / DPMSolverMultistepScheduler, step_coeffs), "unipc" (UniPCMultistepScheduler, unipc_coeffs),
    "heun" (HeunDiscreteScheduler, heun_coeffs), "lms" (LMSDiscreteScheduler, lms_coeffs) or "singlestep"
    (DPMSolverSinglestepScheduler, singlestep_coeffs). Any other scheduler has no fused update here."""
    for cls, kind, _ in _KINDS:
        if isinstance(scheduler, cls):
            return kind
    raise TypeError(f"RegionDiffusionXL: unsupported scheduler {type(scheduler).__name__}; supported: "
                    "EulerDiscreteScheduler, EulerAncestralDiscreteScheduler, DDIMScheduler, DPMSolverMultistepScheduler, "
                    "UniPCMultistepScheduler, HeunDiscreteScheduler, LMSDiscreteScheduler, DPMSolverSinglestepScheduler "
                    "(rtti_b200.schedulers)")


def stepper(scheduler, shape, device, generator=None, kinds=None):
    """The Stepper of `scheduler`. Without `kinds` a scheduler with no fused update raises (_step_kind); with them,
    a scheduler whose update is not among them gets None."""
    for cls, kind, make in _KINDS:
        if isinstance(scheduler, cls):
            return make(scheduler, shape, device, generator) if kinds is None or kind in kinds else None
    if kinds is None:
        _step_kind(scheduler)
    return None
