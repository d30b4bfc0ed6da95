"""Whole sampling trajectories of both samplers against float64, at full latent size, for every fused scheduler.

The kernel tests check one blend call each; what decides the image is the sequence of calls. An error that builds up
over the steps (a history kept at the wrong precision, a history handed to the wrong step or the wrong trajectory, the
reference trajectory stopping early, the ends of the schedule where sigma ~ 14.6 or the order drops) passes every
per-call test and shows here.

The denoiser is a stub with the product UNet's call signature that returns the ideal noise prediction for Gaussian data,
one Gaussian N(mu_b, S_DATA^2 I) per batch row:
    eps_b(x_in, t) = sqrt(1 - a_t) (x_in - sqrt(a_t) mu_b) / (a_t S_DATA^2 + 1 - a_t),   a_t = alphas_cumprod[t]
x_in is the UNet input, which both the sigma-scaled and the VP samplers hand over as the VP-scaled latent, so one formula
serves every scheduler. mu_b is a smooth [4, h, w] field: a fixed projection of the row's mean context vector onto a few
low-frequency cosines, so the uncond, base, region and reference passes differ and the blend matters. The fp16 stub
computes in fp32 from its fp16 input and returns fp16, as a UNet does; the float64 stub computes in float64. Its
projection, patterns and alphas_cumprod table are fp32 values, so both compute the same function. The stub ignores the
attention controls: injection acts through the background blend and the separate reference trajectory only. The
denoiser is linear and contracting, so errors neither blow up nor cancel, and the probability-flow ODE has a closed-form
solution (test_float64_reference_converges_to_the_ode_solution).

Three runs per case, from the same fp16 inputs, all on the GPU:
  * the product: RegionDiffusionXL's plain loop (sample) or rich-text loop (prepare_rich_text + rich_text_step, CUDA
    graphs on, the stub captured in the graph), or RegionDiffusion.produce_latents / produce_attn_maps;
  * the comparator, at the reference's precision: the oracle loop (tests/rescale_oracle.py for SDXL, which is
    oracle/sampler_oracle.py's loop with the CFG rescale; oracle/sampler_oracle.py for SD1.5) with the oracle scheduler
    of the kind (the classes test_oracle_*_matches_reference pins), everything in fp16;
  * the reference: the same loop and oracle scheduler on float64 latents, masks and contexts with the float64 stub, under
    Float64Guard (any op producing a floating-point tensor other than float64 fails the case). The oracle schedulers keep
    their tables in fp32; here every table is derived in float64 from the fp32 alphas_cumprod (the definition of the
    schedule): the sigma grid of Euler / Euler Ancestral / Heun / LMS (_Grid64), and alphas_cumprod, alpha_t, sigma_t and
    lambda_t of DDIM / DPM-Solver++(2M) / UniPC / DPM-Solver++(2S) (_vp64). The LMS coefficients are the oracle's
    quadratures of the Lagrange basis on the float64 sigmas (exact for these polynomials).
Euler Ancestral's noise comes from a seeded CPU generator in every run, drawn in fp16 as diffusers' randn_tensor draws
it; test_device_rng_draws_match_the_reference pins that the product draws the same.

Rule (tests/fp64_rule.py): every checked latent satisfies err_product <= 2 err_fp16 + half an fp16 ulp of max|ref|, on
the max and on the mean, at the first iteration, at the iteration where background injection happens (the middle one in
the plain loops), at the second-to-last and at the last. The reference trajectory of the SDXL rich loop is checked at the
same iterations but the last. Every product run is made twice and must be bit-identical.

At 1000 steps the fp16 rounding of the latents dominates. DPM-Solver++(2M) is checked there; DPM-Solver++(2S) is not,
because it fails the rule at 1000 steps while its fused update is exactly its own definition. With 3 SD1.5 regions
(produce_latents) or 5 SDXL regions (rich-text loop), injection 0.5 / 0.5, the latents at the second-to-last iteration
are, max / mean error against float64:
    SD1.5  product 0.318 / 0.0204   fp16 oracle on the GPU 0.130 / 0.0105   (0.148 / 0.0110 vs 0.154 / 0.0091 halfway)
    SDXL   product 0.367 / 0.0218   fp16 oracle on the GPU 0.160 / 0.0112   (0.176 / 0.0115 vs 0.176 / 0.0092 halfway)
The scheduler's own torch form (DPMSolverSinglestepScheduler.step: fp32 arithmetic, one fp16 rounding per step) in the
same SD1.5 loop gives 0.318 / 0.0202, and the fp16 oracle on the CPU, which rounds the coefficients to fp16, 0.319 /
0.0228. So the kernels compute what singlestep_coeffs defines; the gap lies between that form (one rounding of the
latents per step, each second step restarting from the block's fp16 input) and diffusers' fp16 form (several roundings
per step with fp32 coefficients), and opens in the second half of the trajectory. At 50 steps the product is at most
0.59x (SD1.5) and 1.2x (SDXL) the fp16 oracle's error.
"""
import math
import time
import types

import pytest
import torch

from oracle import sampler_oracle as sam
from oracle import schedulers_oracle as so
from tests import ancestral_oracle as ao
from tests import heun_oracle as ho
from tests import lms_oracle as lo
from tests import multistep_oracle as mo
from tests import rescale_oracle as ro
from tests import singlestep_oracle as sso
from tests import unipc_oracle as upo
from tests.fp64_rule import half_ulp16, maxerr, no_worse
from tests.test_unet_fp64 import Float64Guard

K = 2.0
F64 = torch.float64
S_DATA = 0.5                                          # standard deviation of the stub's data Gaussians
MU_STD = 0.5                                          # typical size of the mean field's cosine coefficients
FREQS = ((0, 0), (1, 0), (0, 1), (1, 1), (2, 1))      # (vertical, horizontal) half-periods of the mean field's patterns
SEED = 20261018
XL_DIM, SD_DIM, POOLED = 2048, 768, 1280
XL_G, SD_G = 7.0, 7.5
DEV = "cuda"
INJECT = (0.5, 0.5)                                   # inject_selfattn, inject_background of the rich-text cases

XL_KINDS = ("euler", "ancestral", "ddim", "dpm2m", "unipc", "heun", "lms", "dpm2s")


# ------------------------------------------------------------------------------------------------ the denoiser
class GaussianDenoiser:
    """The ideal noise prediction for Gaussian data (module docstring), for latents of [4, h, w]. `f64`: compute in
    float64 (the reference), else in fp32 from the input's dtype, returning the input's dtype. `keep`: iterations whose
    first batch row to record in `seen` (the SD1.5 loop's latents entering that call)."""

    def __init__(self, dim, h, w, device, f64=False, keep=()):
        g = torch.Generator().manual_seed(SEED)
        k = len(FREQS)
        proj = torch.randn(dim, 4 * k, generator=g) * (MU_STD * math.sqrt(77 / dim))
        yy = (torch.arange(h, dtype=F64) + 0.5) / h
        xx = (torch.arange(w, dtype=F64) + 0.5) / w
        pat = torch.stack([torch.cos(math.pi * fy * yy)[:, None] * torch.cos(math.pi * fx * xx)[None, :]
                           for fy, fx in FREQS]).float()
        self.dtype = F64 if f64 else torch.float32
        self.device = torch.device(device)
        self.proj, self.pat = proj.to(self.device, self.dtype), pat.to(self.device, self.dtype)
        self.ac = mo._alphas_cumprod().to(self.device, self.dtype)
        self.config = types.SimpleNamespace(sample_size=h, in_channels=4)
        self.in_channels = 4
        self.keep, self.seen, self.calls = set(keep), {}, 0

    def mu(self, ctx):
        """[B, 4, h, w]: the mean of the data Gaussian of each context row."""
        c = (ctx.to(self.dtype).mean(1) @ self.proj).view(ctx.shape[0], 4, len(FREQS))
        return torch.einsum("bck,khw->bchw", c, self.pat)

    def __call__(self, x, t, ctx, added, ctrl):
        if self.calls in self.keep:
            self.seen[self.calls] = x[:1].clone()
        self.calls += 1
        a = self.ac[torch.as_tensor(t, device=self.device).reshape(-1)[:1].long()]
        eps = (1 - a).sqrt() * (x.to(self.dtype) - a.sqrt() * self.mu(ctx)) / (a * (S_DATA * S_DATA) + (1 - a))
        return {"sample": eps.to(x.dtype)}

    def fn(self, x, t, ctx, added, ctrl):
        """The oracle loops' form: the prediction alone."""
        return self(x, t, ctx, added, ctrl)["sample"]


# ------------------------------------------------------------------------------------------------ float64 schedulers
class _Grid64:
    """An oracle scheduler on the Euler grid with its sigmas in float64 (from the fp32 alphas_cumprod). The grid is
    schedulers_oracle's (`leading` spacing, steps_offset 1): integer timesteps, where the interpolated sigma is the
    table's."""

    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        self.alphas_cumprod = self.alphas_cumprod.to(F64)

    def set_timesteps(self, num_inference_steps, device=None):
        self.num_inference_steps = num_inference_steps
        ts = torch.arange(num_inference_steps).flip(0) * (self.num_train_timesteps // num_inference_steps) \
            + self.steps_offset
        ac = self.alphas_cumprod
        sig = ((1 - ac) / ac).sqrt()
        self.timesteps = ts.to(F64)
        self.sigmas = torch.cat([sig[ts], sig.new_zeros(1)])


class _Euler64(_Grid64, so.EulerDiscreteSchedulerOracle):
    pass


class _Ancestral64(_Grid64, ao.EulerAncestralSchedulerOracle):
    """Draws z in fp16 from the same generator as the fp16 oracle and computes with it in float64."""

    def __init__(self, guard, **kw):
        super().__init__(**kw)
        self.guard = guard

    def _noise(self, shape, dtype, device, generator):
        with self.guard.allow_lower():
            z = torch.randn(shape, dtype=torch.float16, generator=self.generator)
        return z.to(device, F64)


def _vp64(s):
    """A VP oracle scheduler (DDIM, DPM-Solver++ 2M / 2S, UniPC) with its tables in float64."""
    ac = s.alphas_cumprod.to(F64)
    s.alphas_cumprod = ac
    if hasattr(s, "final_alpha_cumprod"):
        s.final_alpha_cumprod = ac[0]
    if hasattr(s, "alpha_t"):
        s.alpha_t, s.sigma_t = ac.sqrt(), (1 - ac).sqrt()
        s.lambda_t = s.alpha_t.log() - s.sigma_t.log()
    return s


def _oracle(kind, guard=None):
    """The oracle scheduler of `kind`: fp32 tables (the comparator) or, with the reference's Float64Guard, float64."""
    f64 = guard is not None
    if kind == "euler":
        return _Euler64() if f64 else so.EulerDiscreteSchedulerOracle()
    if kind == "ancestral":
        g = torch.Generator().manual_seed(SEED)
        return _Ancestral64(guard, generator=g) if f64 else ao.EulerAncestralSchedulerOracle(generator=g)
    if kind in ("heun", "lms"):
        s = ho.HeunSchedulerOracle() if kind == "heun" else lo.LMSSchedulerOracle()
        if f64:
            s._euler = _Euler64()
            s.alphas_cumprod = s._euler.alphas_cumprod
        return s
    s = {"ddim": mo.DDIMSchedulerOracle, "dpm2m": mo.DPMSolverMultistepSchedulerOracle,
         "unipc": upo.UniPCSchedulerOracle, "dpm2s": sso.DPMSolverSinglestepSchedulerOracle}[kind]()
    return _vp64(s) if f64 else s


def _product_scheduler(kind):
    from rtti_b200 import schedulers as S
    return {"euler": S.EulerDiscreteScheduler, "ancestral": S.EulerAncestralDiscreteScheduler,
            "ddim": S.DDIMScheduler, "dpm2m": S.DPMSolverMultistepScheduler, "unipc": S.UniPCMultistepScheduler,
            "heun": S.HeunDiscreteScheduler, "lms": S.LMSDiscreteScheduler,
            "dpm2s": S.DPMSolverSinglestepScheduler}[kind]()


class _Recorded:
    """An oracle scheduler that records the latents each step call starts from, for the calls in `keep` (call i + 1
    starts from the loop's latents at the end of iteration i; [main, reference] when the loop steps both)."""

    def __init__(self, s, keep):
        self.__dict__.update(_s=s, keep=set(keep), seen={}, calls=0)

    def __getattr__(self, name):
        return getattr(self._s, name)

    def step(self, model_output, timestep, sample, *a, **kw):
        if self.calls in self.keep:
            self.seen[self.calls] = sample
        self.__dict__["calls"] += 1
        return self._s.step(model_output, timestep, sample, *a, **kw)


# ------------------------------------------------------------------------------------------------ inputs
def _inputs(dim, n_prompts, h, w, seed=SEED):
    """fp16 latents [1, 4, h, w], contexts [n_prompts + 1, 77, dim] and pooled embeddings, and fp32 masks (a softmax
    over bicubically upsampled logits, as tests/synth.py makes them, at any h, w)."""
    g = torch.Generator().manual_seed(seed)
    lat = torch.randn(1, 4, h, w, generator=g).half()
    ctx = torch.randn(n_prompts + 1, 77, dim, generator=g).half()
    pooled = torch.randn(n_prompts + 1, POOLED, generator=g).half()
    logits = torch.randn(n_prompts, 1, 8, 8, generator=g)
    m = torch.softmax(torch.nn.functional.interpolate(logits, (h, w), mode="bicubic", align_corners=False) * 3.0, 0)
    return lat, ctx, pooled, [m[i:i + 1].repeat(1, 4, 1, 1) for i in range(n_prompts)]


def _checkpoints(n, inject_background):
    """The checked iterations: the first, the background-injection one (the middle one without injection), the
    second-to-last and the last."""
    mid = int(inject_background * n) if inject_background > 0 else n // 2
    return sorted({0, mid, n - 2, n - 1})


# ------------------------------------------------------------------------------------------------ the three runs
class Case(types.SimpleNamespace):
    """loop: "xl_plain", "xl_rich", "sd_latents" or "sd_attn_maps"."""

    @property
    def name(self):
        inj = f"/inject={self.inject}" if self.loop in ("xl_rich", "sd_latents") else ""
        return f"{self.loop}/{self.kind}/{self.h}x{self.w}/N={self.steps}/phi={self.phi}{inj}"


def _n_iterations(case):
    s = _oracle(case.kind)
    s.set_timesteps(case.steps)
    return len(s.timesteps)


def _product(case, keep):
    """{iteration: main latents at its end}, {iteration: reference latents at its end} of the product."""
    dev = DEV
    lat, ctx, pooled, masks = _inputs(case.dim, case.n_prompts, case.h, case.w)
    main, ref = {}, {}
    if case.loop.startswith("xl"):
        from rtti_b200.region_diffusion_sdxl import RegionDiffusionXL
        stub = GaussianDenoiser(case.dim, case.h, case.w, dev)
        model = RegionDiffusionXL(device=dev, unet=stub, vae=None, scheduler=_product_scheduler(case.kind))
        assert model.use_cuda_graphs
        gen = torch.Generator().manual_seed(SEED)
        if case.loop == "xl_plain":
            model._calls_back = lambda i, n, every: True     # a callback at every iteration, whatever the order

            def record(i, t, latents):
                if i in keep:
                    main[i] = latents.clone()
            model.sample(height=case.h * 8, width=case.w * 8, num_inference_steps=case.steps, guidance_scale=XL_G,
                         latents=lat, prompt_embeds=ctx[1:], negative_prompt_embeds=ctx[:1],
                         pooled_prompt_embeds=pooled[1:], negative_pooled_prompt_embeds=pooled[:1],
                         output_type="latent", guidance_rescale=case.phi, generator=gen, callback=record)
        else:
            model.masks = masks
            model.scheduler.set_timesteps(case.steps, device=dev)
            x = model.prepare_latents(case.h * 8, case.w * 8, None, lat)
            s = case.h * 8.0, case.w * 8.0
            time_ids = torch.tensor([[s[0], s[1], 0.0, 0.0, s[0], s[1]]], device=dev)
            st = model.prepare_rich_text(ctx.to(dev), pooled.to(dev), time_ids, x, model.scheduler.timesteps, XL_G,
                                         False, *case.inject, {}, case.phi, gen)
            for i in range(st.n_t):
                model.rich_text_step(st, i)
                if i in keep:
                    main[i] = st.latents.clone()
                    if i < st.n_t - 1:
                        ref[i] = st.latents_ref.clone()
            assert len(st.graphs) > 1, "the UNet pass ran outside a CUDA graph"
    else:
        from rtti_b200.region_diffusion import RegionDiffusion
        n = _n_iterations(case)
        stub = GaussianDenoiser(case.dim, case.h, case.w, dev, keep=[i + 1 for i in keep if i < n - 1])
        model = RegionDiffusion(device=dev, unet=stub)
        model.scheduler = _product_scheduler(case.kind)
        if case.loop == "sd_latents":
            model.masks = masks
            out = model.produce_latents(ctx, height=case.h * 8, width=case.w * 8, num_inference_steps=case.steps,
                                        guidance_scale=SD_G, latents=lat, inject_selfattn=case.inject[0],
                                        inject_background=case.inject[1])
        else:
            out = model.produce_attn_maps(None, height=case.h * 8, width=case.w * 8, num_inference_steps=case.steps,
                                          guidance_scale=SD_G, latents=lat, text_embeddings=ctx[[0, -1]], decode=False)
        main = {i - 1: x for i, x in stub.seen.items()}
        main[n - 1] = out.clone()
    torch.cuda.synchronize()
    return main, ref


def _oracle_run(case, keep, guard=None):
    """The same, from the oracle loop: fp16 (guard None) or float64 under `guard`."""
    dev = DEV
    f64 = guard is not None
    dt = F64 if f64 else torch.float16
    lat, ctx, pooled, masks = _inputs(case.dim, case.n_prompts, case.h, case.w)
    lat, ctx = lat.to(dev, dt), ctx.to(dev, dt)
    masks = [m.to(dev, dt) for m in masks]
    stub = GaussianDenoiser(case.dim, case.h, case.w, dev, f64=f64)
    sched = _oracle(case.kind, guard)
    sched.set_timesteps(case.steps)
    n = len(sched.timesteps)
    x = lat * sched.init_noise_sigma if case.loop.startswith("xl") else lat
    rec = _Recorded(sched, [i + 1 for i in keep if i < n - 1])
    ctx2 = torch.cat([ctx[:1], ctx[-1:]])
    with guard if f64 else torch.no_grad():
        if case.loop == "xl_plain":
            out = ro.plain_loop(stub.fn, rec, ctx2, x, case.steps, XL_G, True, guidance_rescale=case.phi)
        elif case.loop == "xl_rich":
            out = ro.rich_text_loop(stub.fn, rec, ctx, masks, x, case.steps, XL_G, inject_selfattn=case.inject[0],
                                    inject_background=case.inject[1], guidance_rescale=case.phi)
        elif case.loop == "sd_latents":
            out = sam.rich_text_loop(stub.fn, rec, ctx, masks, x, case.steps, SD_G, False,
                                     inject_selfattn=case.inject[0], inject_background=case.inject[1])
        else:
            out = ro.plain_loop(stub.fn, rec, ctx2, x, case.steps, SD_G, False)
    assert rec.calls == n, (rec.calls, n)
    main = {i - 1: s[:1] for i, s in rec.seen.items()}
    ref = {i - 1: s[1:2] for i, s in rec.seen.items() if s.shape[0] == 2}
    main[n - 1] = out
    return main, ref


def _run_case(case):
    t0 = time.perf_counter()
    n = _n_iterations(case)
    keep = _checkpoints(n, case.inject[1] if case.loop in ("xl_rich", "sd_latents") else 0.0)
    prod, prod_ref = _product(case, keep)
    again, again_ref = _product(case, keep)
    for i in keep:
        assert torch.equal(prod[i], again[i]), f"{case.name}: two runs differ at iteration {i}"
    for i in prod_ref:
        assert torch.equal(prod_ref[i], again_ref[i]), f"{case.name}: two runs differ at iteration {i} (reference)"
    comp, comp_ref = _oracle_run(case, keep)
    guard = Float64Guard()
    ref64, ref64_ref = _oracle_run(case, keep, guard)
    t1 = time.perf_counter()
    worst = 0.0
    checks = [(f"i={i}", prod[i], comp[i], ref64[i]) for i in keep]
    if case.loop == "xl_rich":
        assert sorted(prod_ref) == sorted(comp_ref) == sorted(ref64_ref) == [i for i in keep if i < n - 1]
        checks += [(f"i={i} reference", prod_ref[i], comp_ref[i], ref64_ref[i]) for i in sorted(prod_ref)]
    for what, got, fp16, r in checks:
        assert got.dtype == fp16.dtype == torch.float16 and r.dtype == F64 and got.shape == r.shape
        e_p, e_c = no_worse(f"{case.name} {what}", got, fp16, r, k=K, floor=half_ulp16(r), mean=True)
        worst = max(worst, e_p / max(e_c, 1e-30))
    print(f"[case] {case.name}: {n} iterations, worst max-error ratio product / fp16 {worst:.2f}, "
          f"{t1 - t0:.1f} s")


def _xl_plain(kind, phi, steps=50):
    return Case(loop="xl_plain", kind=kind, phi=phi, steps=steps, h=128, w=128, dim=XL_DIM, n_prompts=1,
                inject=(0.0, 0.0))


def _xl_rich(kind, phi, steps=50, h=128, w=128):
    return Case(loop="xl_rich", kind=kind, phi=phi, steps=steps, h=h, w=w, dim=XL_DIM, n_prompts=5, inject=INJECT)


def _sd(loop, kind, steps=50):
    return Case(loop=loop, kind=kind, phi=0.0, steps=steps, h=64, w=64, dim=SD_DIM,
                n_prompts=3 if loop == "sd_latents" else 1, inject=INJECT if loop == "sd_latents" else (0.0, 0.0))


CASES = ([_xl_plain(k, phi) for k in XL_KINDS for phi in (0.0, 0.7)]
         + [_xl_rich(k, phi) for k in XL_KINDS for phi in (0.0, 0.7)]
         + [_xl_rich("lms", 0.7, h=168, w=96)]
         + [_sd("sd_latents", k) for k in ("ddim", "dpm2m", "unipc", "dpm2s")]
         + [_sd("sd_attn_maps", k) for k in ("unipc", "dpm2s")]
         + [_xl_rich("dpm2m", 0.7, steps=1000)])


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=lambda c: c.name)
def test_trajectory_matches_float64(case):
    _run_case(case)


# ------------------------------------------------------------------------------------------------ CPU: the reference
T_STOP = 201   # a timestep of every grid of test_float64_reference_converges_to_the_ode_solution


def _ode_error(steps):
    """max |x - exact| at timestep T_STOP of the float64 Euler plain loop with the float64 stub at an 8 x 8 latent,
    under Float64Guard. With CFG the prediction is sigma (x - mu) / (S^2 + sigma^2) in the sigma variable x = latents,
    with mu = mu_u + g (mu_c - mu_u), so the probability-flow ODE dx/dsigma = eps gives
        x(sigma) = mu + (x(sigma_0) - mu) sqrt((S^2 + sigma^2) / (S^2 + sigma_0^2))."""
    h = w = 8
    lat, ctx, _, _ = _inputs(16, 1, h, w)
    lat, ctx = lat.to(F64), ctx.to(F64)
    stub = GaussianDenoiser(16, h, w, "cpu", f64=True)
    sched = _Euler64()
    sched.set_timesteps(steps)
    k = int((sched.timesteps == T_STOP).nonzero().item())
    x0, s0, s1 = lat * sched.init_noise_sigma, float(sched.sigmas[0]), float(sched.sigmas[k])
    rec = _Recorded(sched, [k])
    with Float64Guard():
        ro.plain_loop(stub.fn, rec, ctx, x0, steps, XL_G, True)
    mu_u, mu_c = stub.mu(ctx)
    mu = mu_u + XL_G * (mu_c - mu_u)
    exact = mu + (x0 - mu) * math.sqrt((S_DATA ** 2 + s1 ** 2) / (S_DATA ** 2 + s0 ** 2))
    return maxerr(rec.seen[k], exact)


def test_float64_reference_converges_to_the_ode_solution():
    """The float64 reference of the GPU cases runs under Float64Guard, and its Euler trajectory converges to the
    closed-form solution at first order: on nested grids, the error at a timestep they share falls about 2x per doubling
    of the step count (the last step, from timestep 1 to sigma = 0, is the same on every grid and so is not compared)."""
    Ns = (25, 50, 100, 200)
    for N in Ns:   # the float64 grid is the oracle's
        s32, s64 = so.EulerDiscreteSchedulerOracle(), _Euler64()
        s32.set_timesteps(N)
        s64.set_timesteps(N)
        assert torch.equal(s32.timesteps, s64.timesteps)
        assert torch.allclose(s32.sigmas.double(), s64.sigmas, rtol=1e-6, atol=0)
    errs = [_ode_error(N) for N in Ns]
    ratios = [errs[k] / errs[k + 1] for k in range(len(Ns) - 1)]
    print("[fp64] Euler error vs the ODE solution", [f"{e:.3e}" for e in errs], "ratios", [round(r, 2) for r in ratios])
    assert min(ratios) > 1.85 and max(ratios) < 2.15, ratios
