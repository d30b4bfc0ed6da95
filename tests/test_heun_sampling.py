"""Heun's method in RegionDiffusionXL, with both stages fused into the blend kernels (rtti_region_blend_cfg_heun,
rtti_region_blend_cfg_rescale_heun, rtti_gather_blend_step_heun, rtti_gather_blend_step_rescale_heun).

CPU: the interleaved grid, the configuration, the coefficients against float64 and the torch step against the
diffusers-form oracle (tests/heun_oracle.py), the convergence order on a Gaussian-data ODE with a closed-form solution,
the oracle loops against the unmodified reference (tests/golden/heun.npz, tests/gen_heun.py), the C-ABI argument checks
and the cubin. GPU: the kernels against float64 (tests/fp64_rule.py, K = 2, mean check on; the comparator is the fp16
torch expression diffusers evaluates), bit-identities, the sampler against the goldens and their callback iterations,
and the two-GPU exchanges (tests/multigpu_heun_check.py)."""
import ctypes
import math
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests import heun_oracle as ho
from tests import multistep_oracle as mo
from tests import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
ARG, SHAPE, ALIGN = -1, -2, -3


def _golden():
    return np.load(os.path.join(GOLDEN, "heun.npz"), allow_pickle=False)


def _heun(**kw):
    from rtti_b200.schedulers import HeunDiscreteScheduler
    return HeunDiscreteScheduler(**kw)


def _pooled(cfg):
    return cfg.projection_class_embeddings_input_dim - 6 * cfg.addition_time_embed_dim


# ------------------------------------------------------------------------------------------------ CPU: scheduler
@pytest.mark.parametrize("N", [10, 20, 41, 50])
def test_grid_interleaves_euler(N):
    from rtti_b200.schedulers import EulerDiscreteScheduler
    h, e = _heun(), EulerDiscreteScheduler()
    h.set_timesteps(N)
    e.set_timesteps(N)
    assert h.order == 2 and h.num_inference_steps == N
    t, s = e.timesteps.tolist(), e.sigmas_host
    assert h.timesteps.tolist() == [t[0]] + [v for v in t[1:] for _ in range(2)]
    assert len(h.timesteps) == 2 * N - 1
    want = np.concatenate([s[:1], np.repeat(s[1:-1], 2), [0.0]]).astype(np.float32)
    assert len(h.sigmas_host) == 2 * N and np.array_equal(h.sigmas_host, want) and h.sigmas_host.dtype == np.float32
    assert h.init_noise_sigma == e.init_noise_sigma and torch.equal(h.alphas_cumprod, e.alphas_cumprod)
    for k in range(2 * N - 1):
        assert h.sigma_at(k) == float(h.sigmas_host[k])
        assert h.sigma_at(k) == e.sigma(h.timesteps[k])   # both repeats of t_j sit at sigma_j


def test_config_and_dispatch():
    from rtti_b200 import schedulers as S
    from rtti_b200.region_diffusion_sdxl import _step_kind
    h = _heun()
    assert not isinstance(h, S.EulerDiscreteScheduler), "an Euler subclass would be stepped as Euler"
    assert _step_kind(h) == "heun"
    assert isinstance(S.HeunDiscreteScheduler.from_config(S.EulerDiscreteScheduler()), S.HeunDiscreteScheduler)
    assert S.HeunDiscreteScheduler.from_config(dict(h.config)).config == h.config
    for cfg in (S.DPMSolverMultistepScheduler().config, S.UniPCMultistepScheduler().config):
        with pytest.raises(NotImplementedError):   # the linspace grid is not this scheduler's
            S.HeunDiscreteScheduler.from_config(cfg)
    for kw in (dict(use_karras_sigmas=True), dict(timestep_spacing="trailing"), dict(prediction_type="v_prediction"),
               dict(trained_betas=[0.1] * 1000), dict(beta_schedule="linear")):
        with pytest.raises(NotImplementedError):
            _heun(**kw)
    with pytest.raises(TypeError):
        _heun(solver_order=2)
    with pytest.raises(TypeError, match="UniPCMultistepScheduler, HeunDiscreteScheduler"):
        _step_kind(S.PNDMScheduler())


@pytest.mark.parametrize("N", [1, 2, 4, 10, 41])
def test_coefficients_match_float64(N):
    """heun_coeffs(k) against the definitions evaluated in float64 on the grid, at every iteration; the last iteration
    is a first stage to sigma = 0."""
    s = _heun()
    s.set_timesteps(N)
    sig = s.sigmas_host.astype(np.float64)
    g = torch.Generator().manual_seed(N)
    x, e, xs, ds = (torch.randn(64, generator=g, dtype=torch.float64) * 3 for _ in range(4))
    for k in range(2 * N - 1):
        cx, ce, cs, cd = s.heun_coeffs(k)
        got = cx * x + ce * e + cs * xs + cd * ds
        if k % 2 == 0:
            want = x + (sig[k + 1] - sig[k]) * e
        else:
            want = xs + (sig[k] - sig[k - 1]) / 2 * (ds + e)
        torch.testing.assert_close(got, want, rtol=1e-14, atol=1e-14)
    assert s.heun_coeffs(2 * N - 2) == (1.0, -sig[2 * N - 2], 0.0, 0.0)


def test_torch_step_matches_coefficients_and_oracle():
    """step(), called by timestep value with its repeats (the stage from the call count, as diffusers), against the
    float64 affine form of heun_coeffs and against the diffusers-form oracle; a wrong timestep raises."""
    s, o = _heun(), ho.HeunSchedulerOracle()
    s.set_timesteps(10)
    o.set_timesteps(10)
    assert s.timesteps.tolist() == o.timesteps.tolist()
    g = torch.Generator().manual_seed(3)
    x = torch.randn(2, 4, 8, 8, generator=g) * 8
    xo, x64 = x.clone(), x.double()
    xs = ds = None
    for k, t in enumerate(s.timesteps):
        assert s.state_in_first_order == (k % 2 == 0) == o.state_in_first_order
        assert torch.equal(s.scale_model_input(x, t), x / math.sqrt(s.sigma_at(k) ** 2 + 1))
        torch.testing.assert_close(s.scale_model_input(x, t), o.scale_model_input(x, t), rtol=1e-6, atol=0)
        e = torch.randn(2, 4, 8, 8, generator=g)
        cx, ce, cs, cd = s.heun_coeffs(k)
        want = cx * x64 + ce * e.double() + (cs * xs + cd * ds if k % 2 else 0.0)
        if k % 2 == 0:
            xs, ds = x64, e.double()
        got = s.step(e, t, x)["prev_sample"]
        torch.testing.assert_close(got.double(), want, rtol=1e-6, atol=1e-6 * float(want.abs().max()))
        ref = o.step(e, t, xo)["prev_sample"]
        torch.testing.assert_close(got, ref, rtol=1e-5, atol=1e-5 * float(ref.abs().max()))
        x, xo, x64 = got, ref, want
    s.set_timesteps(4)
    s.step(torch.zeros(1), s.timesteps[0], torch.zeros(1))
    with pytest.raises(ValueError):
        s.step(torch.zeros(1), s.timesteps[0], torch.zeros(1))


def _ode_error(N, heun, var=0.25, x0=1.3, t_from=801, t_to=201):
    """Gaussian data of variance `var`: eps(x, sigma) = x sigma / (var + sigma^2) exactly, and the probability-flow ODE
    dx/dsigma = eps has x(sigma') = x(sigma) sqrt((var + sigma'^2) / (var + sigma^2)). Integrated from t_from to t_to, a
    point of every grid N = 5 * 2^m (ratio 200 / 2^m), so the grids are nested and the final Euler step is never taken."""
    from rtti_b200.schedulers import EulerDiscreteScheduler
    e = EulerDiscreteScheduler()
    e.set_timesteps(N)
    j0, j1 = (int(np.nonzero(e.timesteps_host == t)[0][0]) for t in (t_from, t_to))
    eps = lambda x, sg: x * sg / (var + sg * sg)
    s0, s1 = float(e.sigmas_host[j0]), float(e.sigmas_host[j1])
    exact = x0 * math.sqrt((var + s1 * s1) / (var + s0 * s0))
    x = x0
    if not heun:
        for j in range(j0, j1):
            sg = float(e.sigmas_host[j])
            x = x + (float(e.sigmas_host[j + 1]) - sg) * eps(x, sg)
        return x - exact
    h = _heun()
    h.set_timesteps(N)
    xs = ds = 0.0
    for k in range(2 * j0, 2 * j1):
        cx, ce, cs, cd = h.heun_coeffs(k)
        ek = eps(x, h.sigma_at(k))
        x, xs, ds = (cx * x + ce * ek + cs * xs + cd * ds, *((x, ek) if k % 2 == 0 else (xs, ds)))
    return x - exact


def test_convergence_orders():
    """Per doubling of N the error falls about 4x under Heun and about 2x under Euler."""
    Ns = (5, 10, 20, 40)
    ratios = {}
    for heun in (True, False):
        errs = [_ode_error(N, heun) for N in Ns]
        ratios[heun] = [errs[k] / errs[k + 1] for k in range(len(Ns) - 1)]
    print("error ratios per doubling: Heun", [round(r, 2) for r in ratios[True]], "Euler",
          [round(r, 2) for r in ratios[False]])
    assert min(ratios[True]) > 3.5 and max(ratios[True]) < 4.6, ratios[True]
    assert min(ratios[False]) > 1.7 and max(ratios[False]) < 2.3, ratios[False]


# ------------------------------------------------------------------------------------------------ CPU: goldens
def _xl_plain_oracle(steps):
    from oracle import sampler_oracle as sam, unet_oracle as uo
    cfg = uo.tiny_xl_config()
    S = mo.LATENT_XL_PLAIN
    unet = sam.make_unet_fn(uo.make_state_dict(cfg, 2), cfg)
    inp = synth.synth_inputs(cfg.cross_attention_dim, _pooled(cfg), 3, S, 31)
    ctx, te = inp["ctx"], inp["text_embeds"]
    added2 = {"text_embeds": torch.cat([te[:1], te[-1:]]), "time_ids": inp["time_ids"].repeat(2, 1)}
    return ho.plain_loop(unet, ho.HeunSchedulerOracle(), torch.cat([ctx[:1], ctx[-1:]]), inp["latents"].clone(), steps,
                         8.5, added_cond=added2)


def _xl_rich_oracle(inject_selfattn, inject_background, sched):
    from oracle import sampler_oracle as sam, unet_oracle as uo
    cfg = uo.tiny_xl_config()
    S = mo.LATENT_XL_RICH
    inp = synth.synth_inputs(cfg.cross_attention_dim, _pooled(cfg), 3, S, 31)
    ctx, te = inp["ctx"], inp["text_embeds"]
    tfd = synth.font_sizes()
    tfd.update(synth.color_dict(inp["masks"], S, 1.0))
    return ho.rich_text_loop(sam.make_unet_fn(uo.make_state_dict(cfg, 2), cfg), sched, ctx, inp["masks"],
                             inp["latents"].clone(), 4, 8.5, xl=True,
                             added_cond={"text_embeds": te, "time_ids": inp["time_ids"]}, use_guidance=True,
                             text_format_dict=tfd, inject_selfattn=inject_selfattn,
                             inject_background=inject_background, vae_decode=synth.TinyVAE(), scaling_factor=0.13025)


def _assert_golden(got, ref, what):
    np.testing.assert_allclose(np.asarray(got, np.float32), ref, atol=5e-4 * max(1.0, float(np.abs(ref).max()) / 10),
                               rtol=1e-4, err_msg=what)


@pytest.mark.parametrize("steps", [5, 10])
def test_oracle_xl_plain_matches_reference(steps):
    got = _xl_plain_oracle(steps)
    _assert_golden(got.numpy(), _golden()[f"xl_plain_{steps}"], f"xl plain {steps}")
    assert _golden()[f"xl_plain_{steps}_callbacks"].tolist() == ho.callback_iterations(2 * steps - 1, steps, 2, 1)


@pytest.mark.parametrize("sa,bg", [(0.5, 0.5), (0.0, 0.5)])
def test_oracle_xl_rich_matches_reference(sa, bg):
    """Joint batch-2 steps on every iteration (0.5 / 0.5), and on iterations 0..3 then batch-1 steps (0 / 0.5): the last
    joint iteration is a second stage."""
    sched = ho.HeunSchedulerOracle()
    got = _xl_rich_oracle(sa, bg, sched)
    joint = 7 if sa > 0 else 4
    assert sched.step_batches == [2] * joint + [1] * (7 - joint)
    _assert_golden(got.detach().numpy(), _golden()[f"xl_rich_{sa:g}_{bg:g}"], f"xl rich {sa} {bg}")


# ------------------------------------------------------------------------------------------------ CPU: C ABI, cubin
def test_heun_abi_rejects_bad_arguments_without_launching():
    """Every call below fails its argument checks; a launch without a device would return RTTI_ERR_CUDA instead."""
    from rtti_b200 import _lib
    lib = _lib.load()
    V = ctypes.c_void_p
    buf = (ctypes.c_char * 8192)()
    a = (ctypes.addressof(buf) + 15) // 16 * 16
    regions = (V * 3)(V(a), V(a), V(a))
    second = (0.0, -0.2, 1.0, -0.2)
    for fn, extra in ((lib.rtti_region_blend_cfg_heun, []), (lib.rtti_region_blend_cfg_rescale_heun, [0.7])):
        rb = lambda lat=a, xs=a, ds=a, n=64, c=second, eu=a, regs=regions, N=3: fn(
            V(eu), regs, V(a), N, n, 7.5, V(a), V(lat), V(lat), *c, V(xs), V(ds), *extra, V(0))
        assert rb(eu=0) == ARG
        assert rb(regs=(V * 3)(V(a), V(0), V(a))) == ARG
        assert rb(N=17) == ARG
        assert rb(lat=0) == ARG                  # the Heun update needs the latents
        assert rb(xs=0) == ARG                   # cs != 0 needs xs
        assert rb(ds=0) == ARG                   # cd != 0 needs ds
        assert rb(n=60) == SHAPE
        assert rb(xs=a + 2) == ALIGN
        assert rb(ds=a + 8, c=(1.0, -0.4, 0.0, 0.0)) == ALIGN   # a pointer that is given must be aligned
    peers = (V * 2)(V(a), V(a))
    owner = (ctypes.c_int * 6)(0, 0, 1, 1, 0, 1)
    for fn, extra in ((lib.rtti_gather_blend_step_heun, []), (lib.rtti_gather_blend_step_rescale_heun, [0.7])):
        gb = lambda world=2, rank=0, n=64, ref=0, xs=a, ds=a, xs_r=a, ds_r=a, er=0, lat=a, slots=peers: fn(
            slots, peers, world, rank, owner, 6, 3, V(a), n, 7.5, V(a), V(lat), V(lat), V(ref), V(ref), *second,
            V(xs), V(ds), V(xs_r), V(ds_r), V(er), 1, *extra, V(0))
        assert gb(world=17) == ARG
        assert gb(rank=2) == ARG
        assert gb(slots=(V * 2)(V(a), V(0))) == ARG
        assert gb(lat=0) == ARG
        assert gb(ds=0) == ARG
        assert gb(ref=a, xs_r=0) == ARG          # the reference trajectory needs its own saved state
        assert gb(ref=a, ds_r=0) == ARG
        assert gb(er=a) == ARG                   # eps_ref_out without the reference latents
        assert gb(n=60) == SHAPE
        assert gb(xs=a + 4) == ALIGN
        assert gb(ref=a, ds_r=a + 4) == ALIGN
        assert gb(ref=a, er=a + 8) == ALIGN
        assert gb(world=1) == ARG                # slot owned by rank 1 of a world of 1


def test_heun_step_python_checks():
    from rtti_b200 import _lib, ops
    x = torch.zeros(64, dtype=torch.float16)
    ops.HeunStep((1.0, -0.3, 0.0, 0.0), None, None)._check(64, False)   # a first stage reads no saved state
    ops.HeunStep((1.0, -0.3, 0.0, 0.0), None, None)._check(64, True)
    with pytest.raises(_lib.RttiError, match="xs is required"):
        ops.HeunStep((0.0, -0.1, 1.0, -0.1), None, None)._check(64, False)
    with pytest.raises(_lib.RttiError, match="ds is required"):
        ops.HeunStep((0.0, -0.1, 0.0, -0.1), None, None)._check(64, False)
    with pytest.raises(_lib.RttiError, match="must be a CUDA tensor"):
        ops.HeunStep((0.0, -0.1, 1.0, -0.1), x, x)._check(64, False)
    with pytest.raises(_lib.RttiError, match="eps_ref_out needs the reference latents"):
        ops.HeunStep((1.0, -0.3, 0.0, 0.0), None, None, eps_ref_out=x)._check(64, False)
    with pytest.raises(_lib.RttiError, match=r"\(cx, ce, cs, cd\)"):
        ops.HeunStep((1.0, -0.3, 0.0), None, None)


def _sass_by_kernel():
    from rtti_b200 import _lib
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    _lib.load()
    sass = subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True).stdout
    out = {}
    for f in re.split(r"\n\s*Function : ", sass)[1:]:
        name = f.split("\n", 1)[0]
        m = re.search(r"\d(region_blend|gather_blend|blend_rescale)(_heun)?_kernel(ILb[01]E)?", name)
        if m:
            out[(m.group(1), m.group(3) or "", bool(m.group(2)))] = (name, f)
    return out


def test_heun_kernels_in_the_cubin():
    """Each of the four families has its _heun kernel, whose 128-bit loads are those of its Euler kernel plus xs and ds
    (for each trajectory it steps); the rescale cluster kernels stay within 64 registers at 1024 threads, no spills."""
    from rtti_b200 import _lib
    k = _sass_by_kernel()
    fams = [("region_blend", "", 2), ("gather_blend", "", 4), ("blend_rescale", "ILb0E", 4), ("blend_rescale", "ILb1E", 4)]
    for fam, tpl, extra in fams:
        assert (fam, tpl, True) in k and (fam, tpl, False) in k, (fam, tpl, sorted(k))
        ld = {h: len(re.findall(r"\bLDG\.E\.128\b", k[(fam, tpl, h)][1])) for h in (False, True)}
        assert ld[True] >= ld[False] + extra, (fam, tpl, ld)
        if fam == "blend_rescale":
            assert not re.search(r"\bSTL", k[(fam, tpl, True)][1]), f"{fam}{tpl}: local-memory stores (spills)"
    out = subprocess.run(["cuobjdump", "-res-usage", _lib.LIB_PATH], capture_output=True, text=True).stdout
    regs = [int(r) for fn, r in re.findall(r"Function (\S+):\s*\n\s*REG:(\d+)", out) if "blend_rescale_heun_kernel" in fn]
    assert len(regs) == 2
    for r in regs:
        assert r <= 64 and ((r * 32 + 255) // 256 * 256) * 32 <= 65536, f"{r} registers x 32 warps"


# ------------------------------------------------------------------------------------------------ GPU: accuracy
def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _masks(N, n, g):
    m = torch.rand(N, n, device="cuda", generator=g)
    return (m / m.sum(0, keepdim=True)).half().float().contiguous()


def _coeffs(stage):
    """heun_coeffs of a 20-step grid: a first stage, a second stage, or the last iteration (a first stage to 0)."""
    s = _heun()
    s.set_timesteps(20)
    return s.heun_coeffs({"first": 12, "second": 13, "last": 38}[stage])


def _gather_world1(eu, er, m, guidance, lat, ref_pair, phi, step, dt=0.0, step_id=3):
    from rtti_b200 import ops
    n, N = eu.numel(), len(er)
    n_slots = N + 3
    slots = torch.zeros(2, n_slots, n, dtype=torch.float16, device="cuda")
    flags = torch.zeros(16, dtype=torch.int32, device="cuda")
    for s, e in enumerate([eu] + er + list(ref_pair[:2])):
        slots[step_id & 1, s].copy_(e)
    out = ops.gather_blend_step([slots.data_ptr()], [flags.data_ptr()], 0, [0] * n_slots, N, m, guidance, lat,
                                ref_pair[2], dt, step_id, guidance_rescale=phi, step=step)
    torch.cuda.synchronize()
    assert int(flags[0]) == step_id and int(flags[1]) == 0
    return out


def _inputs(n, N, seed):
    g = _gen(seed)
    rn = lambda s=1.0: (s * torch.randn(n, device="cuda", generator=g)).half()
    eu, er = rn(), [rn() for _ in range(N)]
    m = _masks(N, n, g)
    lat, ec, ed, lat_ref = rn(3.0), rn(), rn(), rn(3.0)
    xs, ds, xs_ref, ds_ref = rn(3.0), rn(), rn(3.0), rn()
    return eu, er, m, lat, ec, ed, lat_ref, (xs, ds), (xs_ref, ds_ref)


def _blend64(eu, er, m, guidance, phi):
    md = m.double()
    u64 = sum(eu.double() * md[k] for k in range(len(er)))
    t64 = sum(er[k].double() * md[k] for k in range(len(er)))
    e64 = u64 + guidance * (t64 - u64)
    if phi:
        e64 = e64 * (1 - phi + phi * t64.std() / e64.std())
    return e64


@pytest.mark.gpu
@pytest.mark.parametrize("stage", ["first", "second", "last"])
@pytest.mark.parametrize("with_ref", [False, True])
@pytest.mark.parametrize("phi", [0.0, 0.7])
@pytest.mark.parametrize("N", [2, 5, 16])
@pytest.mark.parametrize("n", [16384, 65536, 65528])
@pytest.mark.parametrize("family", ["single", "gather"])
def test_heun_kernels_vs_fp64(family, n, N, phi, with_ref, stage):
    """latents_out (and the reference latents with C/D) against float64 of x + dt eps (first stage, last iteration) or
    xs + dt/2 (ds + eps) (second stage) on the exact blend, with xs / ds the fp16 saved state."""
    from rtti_b200 import ops
    from tests.fp64_rule import half_ulp16, no_worse
    c = _coeffs(stage)
    cx, ce, cs, cd = c
    eu, er, m, lat, ec, ed, lat_ref, (xs, ds), (xs_ref, ds_ref) = _inputs(n, N, n + 13 * N + int(10 * phi) + 7 * with_ref)
    guidance = 5.0
    ones = torch.ones(1, n, device="cuda")
    st = (xs, ds) if cs else (None, None)
    st_ref = (xs_ref, ds_ref) if cs else (None, None)
    if family == "single":
        e1, x1 = ops.region_blend_cfg(eu, er, m, guidance, latents=lat, guidance_rescale=phi, step=ops.HeunStep(c, *st))
        xr = ops.region_blend_cfg(ec, [ed], ones, guidance, latents=lat_ref, guidance_rescale=phi,
                                  step=ops.HeunStep(c, *st_ref))[1] if with_ref else None
    else:
        step = ops.HeunStep(c, *st, *(st_ref if with_ref else (None, None)))
        e1, x1, xr = _gather_world1(eu, er, m, guidance, lat, (ec, ed, lat_ref if with_ref else None), phi, step)
    tag = f"heun {family} n{n} N{N} phi{phi:g} {stage}"
    trajectories = [(e1, x1, lat, xs, ds, _blend64(eu, er, m, guidance, phi), "latents")]
    if with_ref:
        e_ref16 = ops.region_blend_cfg(ec, [ed], ones, guidance, guidance_rescale=phi)   # the fp16 prediction stepped
        trajectories.append((e_ref16, xr, lat_ref, xs_ref, ds_ref, _blend64(ec, [ed], ones, guidance, phi),
                             "latents_ref"))
    for e16, got, x, xs_, ds_, e64, what in trajectories:
        if cs:
            want64 = xs_.double() + ce * (ds_.double() + e64)
            cmp16 = xs_ + (ds_ + e16) / 2 * (2 * ce)   # diffusers in fp16: sample + (prev_derivative + derivative) / 2 * dt
        else:
            want64 = x.double() + ce * e64
            cmp16 = x + e16 * ce
        no_worse(f"{tag} {what}", got, cmp16, want64, k=2.0, floor=half_ulp16(want64), mean=True)


# ------------------------------------------------------------------------------------------------ GPU: bit-identities
@pytest.mark.gpu
@pytest.mark.parametrize("phi", [0.0, 0.7])
@pytest.mark.parametrize("n,N", [(16384, 5), (65528, 2), (65536, 16)])
def test_heun_bit_identities(n, N, phi):
    """A first stage equals the Euler entry point with dt_sigma = dt (all four families, eps and latents); eps_ref_out
    equals the eps the single form computes for passes C/D; the gather form at world 1 equals the single form (both
    trajectories, both stages); a second stage does not read the current latents; a CUDA-graph replay equals eager."""
    from rtti_b200 import ops
    eu, er, m, lat, ec, ed, lat_ref, (xs, ds), (xs_ref, ds_ref) = _inputs(n, N, n + N + 1)
    ones = torch.ones(1, n, device="cuda")
    guidance = 8.5
    c1 = _coeffs("first")
    e_eu, x_eu = ops.region_blend_cfg(eu, er, m, guidance, latents=lat, dt_sigma=c1[1], guidance_rescale=phi)
    e_h, x_h = ops.region_blend_cfg(eu, er, m, guidance, latents=lat, guidance_rescale=phi,
                                    step=ops.HeunStep(c1, None, None))
    assert torch.equal(e_eu, e_h) and torch.equal(x_eu, x_h), "a first stage differs from the Euler form (single GPU)"
    eps_ref = torch.full_like(lat_ref, float("nan"))
    g_eu = _gather_world1(eu, er, m, guidance, lat, (ec, ed, lat_ref), phi, None, dt=c1[1])
    g_h = _gather_world1(eu, er, m, guidance, lat, (ec, ed, lat_ref), phi,
                         ops.HeunStep(c1, None, None, None, None, eps_ref))
    for a, b, what in zip(g_eu, g_h, ("eps", "latents", "latents_ref")):
        assert torch.equal(a, b), f"a first stage differs from the Euler form (gather): {what}"
    e_cd, _ = ops.region_blend_cfg(ec, [ed], ones, guidance, latents=lat_ref, guidance_rescale=phi,
                                   step=ops.HeunStep(c1, None, None))
    assert torch.equal(eps_ref, e_cd), "eps_ref_out differs from the single form's eps of C/D"
    c2 = _coeffs("second")

    def single(latents=lat):
        eps, lo = ops.region_blend_cfg(eu, er, m, guidance, latents=latents, guidance_rescale=phi,
                                       step=ops.HeunStep(c2, xs, ds))
        _, ro = ops.region_blend_cfg(ec, [ed], ones, guidance, latents=lat_ref, guidance_rescale=phi,
                                     step=ops.HeunStep(c2, xs_ref, ds_ref))
        return eps, lo, ro

    a = single()
    for x, y in zip(a, single()):
        assert torch.equal(x, y), "two calls differ"
    assert torch.equal(a[1], single(latents=(lat.float() * 0.5 + 1).half())[1]), "a second stage read the latents"
    gw = _gather_world1(eu, er, m, guidance, lat, (ec, ed, lat_ref), phi, ops.HeunStep(c2, xs, ds, xs_ref, ds_ref))
    for x, y, what in zip(a, gw, ("eps", "latents", "latents_ref")):
        assert torch.equal(x, y), f"gather world 1 vs single GPU: {what} differs"
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        single()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = single()
    for _ in range(2):
        graph.replay()
        torch.cuda.synchronize()
        for x, y in zip(a, captured):
            assert torch.equal(x, y), "graph replay differs from eager"


# ------------------------------------------------------------------------------------------------ GPU: sampler
def _close_range(got, ref, what):
    got, ref = np.asarray(got, np.float32), np.asarray(ref, np.float32)
    tol = 5e-3 * float(np.abs(ref).max()) + 3e-2 * np.abs(ref)
    err = np.abs(got - ref)
    assert np.isfinite(got).all(), f"{what}: non-finite values"
    assert (err <= tol).all(), f"{what}: {float((err > tol).mean()) * 100:.3f}% outside, max err {err.max():.4f}"
    print(f"{what}: max err {err.max():.4f} mean err {err.mean():.5f}")


def _xl_model(scheduler):
    from oracle import unet_oracle as uo
    from rtti_b200.region_diffusion_sdxl import RegionDiffusionXL
    from rtti_b200.unet import UNet2DConditionModel, UNetConfig
    cfg = uo.tiny_xl_config()
    unet = UNet2DConditionModel(UNetConfig.from_dict(cfg.__dict__))
    unet.load_state_dict(uo.make_state_dict(cfg, 2))
    return cfg, RegionDiffusionXL(device="cuda", unet=unet.finalize("cuda"), vae=synth.TinyVAE("cuda"),
                                  scheduler=scheduler)


def _xl_plain(steps, scheduler=None, calls=None):
    cfg, m = _xl_model(scheduler or _heun())
    S = mo.LATENT_XL_PLAIN
    inp = synth.synth_inputs(cfg.cross_attention_dim, _pooled(cfg), 3, S, 31)
    ctx, te = inp["ctx"].cuda(), inp["text_embeds"].cuda()
    cb = (lambda i, t, lat: calls.append(i)) if calls is not None else None
    return m.sample(height=S * 8, width=S * 8, num_inference_steps=steps, guidance_scale=8.5,
                    latents=inp["latents"].clone(), prompt_embeds=ctx[-1:], negative_prompt_embeds=ctx[:1],
                    pooled_prompt_embeds=te[-1:], negative_pooled_prompt_embeds=te[:1], output_type="latent",
                    run_rich_text=False, callback=cb, callback_steps=1).images.float().cpu().numpy()


def _xl_rich(sa, bg, scheduler=None, graphs=True, calls=None, callback_steps=1):
    cfg, m = _xl_model(scheduler or _heun())
    m.use_cuda_graphs = graphs
    S = mo.LATENT_XL_RICH
    inp = synth.synth_inputs(cfg.cross_attention_dim, _pooled(cfg), 3, S, 31)
    ctx, te = inp["ctx"], inp["text_embeds"]
    tfd = synth.font_sizes()
    tfd.update(synth.color_dict(inp["masks"], S, 1.0))
    m.masks = [x.cuda() for x in inp["masks"]]
    cb = (lambda i, t, lat: calls.append(i)) if calls is not None else None
    return m.sample(height=S * 8, width=S * 8, num_inference_steps=4, guidance_scale=8.5,
                    latents=inp["latents"].clone(), prompt_embeds=ctx[1:].cuda(), negative_prompt_embeds=ctx[:1].cuda(),
                    pooled_prompt_embeds=te[1:].cuda(), negative_pooled_prompt_embeds=te[:1].cuda(),
                    output_type="latent", run_rich_text=True, use_guidance=True, inject_selfattn=sa,
                    inject_background=bg, text_format_dict=tfd, callback=cb,
                    callback_steps=callback_steps).images.float().cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("steps", [5, 10])
def test_xl_plain_vs_reference_golden(steps):
    """The plain pass against the reference's, and its callback iterations; the Euler run of the same inputs lies
    outside the tolerance."""
    from rtti_b200.schedulers import EulerDiscreteScheduler
    ref = _golden()[f"xl_plain_{steps}"]
    calls = []
    _close_range(_xl_plain(steps, calls=calls), ref, f"xl plain {steps}")
    assert calls == _golden()[f"xl_plain_{steps}_callbacks"].tolist(), calls
    with pytest.raises(AssertionError):
        _close_range(_xl_plain(steps, EulerDiscreteScheduler()), ref, "xl plain, Euler")


@pytest.mark.gpu
@pytest.mark.parametrize("sa,bg", [(0.5, 0.5), (0.0, 0.5)])
def test_xl_rich_vs_reference_golden(sa, bg):
    """Injection, font sizes and colour guidance against the reference's loop, with its callback iterations; the Euler
    run lies outside the tolerance; CUDA-graph replayed UNet passes give the same bits as eager ones."""
    from rtti_b200.schedulers import EulerDiscreteScheduler
    ref = _golden()[f"xl_rich_{sa:g}_{bg:g}"]
    calls = []
    out = _xl_rich(sa, bg, calls=calls)
    _close_range(out, ref, f"xl rich {sa} {bg}")
    assert calls == _golden()[f"xl_rich_{sa:g}_{bg:g}_callbacks"].tolist(), calls
    with pytest.raises(AssertionError):
        _close_range(_xl_rich(sa, bg, EulerDiscreteScheduler()), ref, "xl rich, Euler")
    calls2 = []
    assert np.array_equal(out, _xl_rich(sa, bg, graphs=False, calls=calls2, callback_steps=2)), \
        "use_cuda_graphs on / off differ"
    assert calls2 == ho.callback_iterations(7, 4, 2, 2) == [6], calls2


@pytest.mark.gpu
def test_rich_loop_stops_the_reference_after_a_first_stage():
    """inject_selfattn = 0 with the last joint iteration a first stage (inject_background = 0.4: iterations 0..2 of 7):
    the reference latents keep their first-stage value and the main latents finish on their own saved state, as the
    per-trajectory oracle loop does; the reference loop would add a batch-1 prediction to a batch-2 state here."""
    sched = ho.PerTrajectoryHeunOracle()
    ref = _xl_rich_oracle(0.0, 0.4, sched)
    assert sched.step_batches == [2, 2, 2, 1, 1, 1, 1]
    _close_range(_xl_rich(0.0, 0.4), ref.detach().numpy(), "xl rich 0 / 0.4 vs the per-trajectory oracle")


@pytest.mark.gpu
def test_rich_loop_heun_two_gpus():
    """Heun on the fused peer exchange and on the NCCL path (tests/multigpu_heun_check.py)."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
                        "--master-addr", "127.0.0.1", "--master-port", "29543",
                        os.path.join(ROOT, "tests", "multigpu_heun_check.py")],
                       capture_output=True, text=True, timeout=900)
    print(r.stdout[-2000:], r.stderr[-2000:])
    assert r.returncode == 0 and "MULTIGPU_HEUN_CHECK PASS" in r.stdout
