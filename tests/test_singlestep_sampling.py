"""DPM-Solver++(2S) in both samplers, with the singlestep update fused into the blend kernels
(rtti_region_blend_cfg_ss, rtti_region_blend_cfg_rescale_ss, rtti_gather_blend_step_ss,
rtti_gather_blend_step_rescale_ss).

CPU: the grid and the order list, the configuration and the dispatch, singlestep_coeffs against a float64 evaluation of
diffusers' formulas, the torch step against the diffusers-form oracle (tests/singlestep_oracle.py), the convergence
order on a Gaussian-data ODE against DPM-Solver++(2M) at equal UNet evaluations, the oracle loops against the unmodified
reference (tests/golden/singlestep.npz, tests/gen_singlestep.py), the C-ABI argument checks and the cubin. GPU: the
kernels against float64 (tests/fp64_rule.py, K = 2, mean check on; the comparator is the fp16 torch expression
diffusers evaluates), bit-identities with the multistep ("_ms") forms, both samplers against the goldens, and the
two-GPU exchanges (tests/multigpu_singlestep_check.py)."""
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

from tests import multistep_oracle as mo
from tests import singlestep_oracle as so
from tests import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
ARG, SHAPE, ALIGN = -1, -2, -3


def _golden():
    return np.load(os.path.join(GOLDEN, "singlestep.npz"), allow_pickle=False)


def _ss(**kw):
    from rtti_b200.schedulers import DPMSolverSinglestepScheduler
    return DPMSolverSinglestepScheduler(**kw)


def _pooled(cfg):
    return cfg.projection_class_embeddings_input_dim - 6 * cfg.addition_time_embed_dim


def _ac64():
    ac = mo._alphas_cumprod().double()
    al, sg = ac.sqrt(), (1 - ac).sqrt()
    return al, sg, al.log() - sg.log()


# ------------------------------------------------------------------------------------------------ CPU: scheduler
@pytest.mark.parametrize("N", [1, 2, 3, 5, 10, 25, 1000])
def test_grid_and_order_list(N):
    from rtti_b200.schedulers import DPMSolverMultistepScheduler
    s, d = _ss(), DPMSolverMultistepScheduler()
    s.set_timesteps(N)
    d.set_timesteps(N)
    n = len(s.timesteps_host)
    assert s.timesteps.tolist() == d.timesteps.tolist() and n == s.num_inference_steps
    assert s.order_list == [1, 2] * (n // 2) + [1] * (n % 2)
    assert s.order_list == so.DPMSolverSinglestepSchedulerOracle.get_order_list(n)
    assert s.order == 1 and s.init_noise_sigma == 1.0 and torch.equal(s.alphas_cumprod, d.alphas_cumprod)
    x = torch.randn(1, 4, 8, 8)
    assert s.scale_model_input(x, s.timesteps[0]) is x
    o = so.DPMSolverSinglestepSchedulerOracle()
    o.set_timesteps(N)
    assert o.timesteps.tolist() == s.timesteps.tolist() and o.order_list == s.order_list


def test_config_and_dispatch():
    from rtti_b200 import schedulers as S
    from rtti_b200.region_diffusion_sdxl import _step_kind
    s = _ss()
    assert not isinstance(s, S.DPMSolverMultistepScheduler) and not isinstance(s, S.MULTISTEP_SCHEDULERS)
    assert _step_kind(s) == "singlestep"
    for src in (S.DPMSolverMultistepScheduler(), S.DDIMScheduler(), S.UniPCMultistepScheduler()):
        t = S.DPMSolverSinglestepScheduler.from_config(src)
        assert isinstance(t, S.DPMSolverSinglestepScheduler) and t.config.solver_type == "midpoint"
    assert S.DPMSolverSinglestepScheduler.from_config(dict(s.config)).config == s.config
    for kw in (dict(use_karras_sigmas=True), dict(solver_order=3), dict(solver_order=1),
               dict(algorithm_type="sde-dpmsolver++"), dict(algorithm_type="dpmsolver"), dict(solver_type="heun"),
               dict(thresholding=True), dict(prediction_type="v_prediction"), dict(trained_betas=[0.1] * 1000),
               dict(lower_order_final=False), dict(beta_schedule="linear")):
        with pytest.raises(NotImplementedError):
            _ss(**kw)
    with pytest.raises(NotImplementedError):
        S.DPMSolverSinglestepScheduler.from_config(S.DPMSolverMultistepScheduler(), use_karras_sigmas=True)
    with pytest.raises(TypeError):
        _ss(timestep_spacing="linspace")
    with pytest.raises(TypeError, match="LMSDiscreteScheduler, DPMSolverSinglestepScheduler"):
        _step_kind(S.PNDMScheduler())


def _diffusers64(ts, order_list, i, x, eps, xs, m_prev):
    """Step i in float64 as diffusers writes it (dpm_solver_first_order_update / singlestep_dpm_solver_second_order_update
    with solver_type "midpoint"): (x', D of this step)."""
    al, sg, lam = _ac64()
    n = len(ts)
    t_i = int(ts[i])
    s = 0 if i == n - 1 else int(ts[i + 1])
    m = (x - sg[t_i] * eps) / al[t_i]
    if order_list[i] == 1:
        h = lam[s] - lam[t_i]
        return (sg[s] / sg[t_i]) * x - (al[s] * (torch.exp(-h) - 1.0)) * m, m
    t, s0, s1 = s, t_i, int(ts[i - 1])
    h, h_0 = lam[t] - lam[s1], lam[s0] - lam[s1]
    r0 = h_0 / h
    D0, D1 = m_prev, (1.0 / r0) * (m - m_prev)
    a = al[t] * (torch.exp(-h) - 1.0)
    return (sg[t] / sg[s1]) * xs - a * D0 - 0.5 * a * D1, m


@pytest.mark.parametrize("N", [1, 2, 3, 5, 10, 25, 1000])
def test_singlestep_coeffs_match_float64(N):
    """singlestep_coeffs(i) applied to float64 (x, eps, xs, D_prev) against diffusers' formulas in float64, on every
    step: D to 1e-12 and x' to 1e-11 relative; a first step has cs = cp = 0 and equals DPM-Solver++(2M)'s first-order
    coefficients, a second step has cx = 0."""
    from rtti_b200.schedulers import DPMSolverMultistepScheduler
    s = _ss()
    s.set_timesteps(N)
    ts = s.timesteps_host
    g = torch.Generator().manual_seed(N)
    x = torch.randn(64, generator=g, dtype=torch.float64) * 3
    xs = m_prev = None
    worst = 0.0
    for i in range(len(ts)):
        c = s.singlestep_coeffs(i)
        assert len(c) == 6 and all(isinstance(v, float) for v in c)
        eps = torch.randn(64, generator=g, dtype=torch.float64)
        want, m = _diffusers64(ts, s.order_list, i, x, eps, xs, m_prev)
        d = c.hx * x + c.he * eps
        torch.testing.assert_close(d, m, rtol=1e-12, atol=1e-12 * float(m.abs().max()))
        got = c.cx * x + c.cd * d + (c.cp * m_prev if c.cp != 0.0 else 0.0) + (c.cs * xs if c.cs != 0.0 else 0.0)
        err = float((got - want).abs().max() / want.abs().max())
        worst = max(worst, err)
        assert err <= 1e-11, (i, err)
        if s.order_list[i] == 1:
            assert c.cs == 0.0 and c.cp == 0.0
            d2m = DPMSolverMultistepScheduler()._first_order(int(ts[i]), 0 if i == len(ts) - 1 else int(ts[i + 1]))
            assert (c.hx, c.he, c.cx, c.cd) == d2m[:4]
            xs = x
        else:
            assert c.cx == 0.0 and c.cs != 0.0 and c.cp != 0.0
        x, m_prev = want, m
    print(f"N={N}: max relative difference to diffusers' float64 form {worst:.2e}")


def test_torch_step_matches_oracle():
    """step() against the diffusers-form oracle in fp32 (even and odd N), with the latents moved between the two
    steps of a block (the second step restarts from the block's saved latents); set_timesteps clears the state."""
    s, o = _ss(), so.DPMSolverSinglestepSchedulerOracle()
    for N in (5, 10):
        s.set_timesteps(N)
        o.set_timesteps(N)
        assert s._xs is None
        g = torch.Generator().manual_seed(N)
        x = torch.randn(2, 4, 8, 8, generator=g) * 3
        xo = x.clone()
        for i, t in enumerate(s.timesteps):
            e = torch.randn(2, 4, 8, 8, generator=g)
            got = s.step(e, t, x)["prev_sample"]
            ref = o.step(e, t, xo)["prev_sample"]
            torch.testing.assert_close(got, ref, rtol=1e-5, atol=1e-5 * float(ref.abs().max()))
            kick = 0.1 * torch.randn(2, 4, 8, 8, generator=g)   # colour guidance / background injection stand-in
            x, xo = got + kick, ref + kick


def _ode_error(M, kind, var=0.25, x0=1.3, t_from=865, t_to=97):
    """Gaussian data of variance `var`: in VP space eps(x, t) = sigma_t x / (alpha_t^2 var + sigma_t^2) exactly, and the
    probability-flow ODE has x(t') = x(t) sqrt((alpha_t'^2 var + sigma_t'^2) / (alpha_t^2 var + sigma_t^2)). Integrated
    from t_from to t_to in M equal timestep strides (nested grids for M = 12 * 2^k) with the affine coefficients of the
    scheduler, each evaluation of eps counting one UNet call: equal M is equal work for 2S and 2M."""
    from rtti_b200.schedulers import DPMSolverMultistepScheduler
    s = _ss() if kind == "2s" else DPMSolverMultistepScheduler()
    s.set_timesteps(M + 1)
    assert (t_from - t_to) % M == 0
    s.timesteps_host = np.arange(t_from, t_to - 1, -((t_from - t_to) // M), dtype=np.int64)
    if kind == "2s":
        s.order_list = s.get_order_list(len(s.timesteps_host))
    al, sg, _ = _ac64()
    al, sg = al.numpy(), sg.numpy()
    var_t = lambda t: al[t] ** 2 * var + sg[t] ** 2
    exact = x0 * math.sqrt(var_t(t_to) / var_t(t_from))
    x, xs, d_prev = x0, 0.0, 0.0
    for i in range(M):
        t = int(s.timesteps_host[i])
        e = sg[t] * x / var_t(t)
        if kind == "2s":
            c = s.singlestep_coeffs(i)
            if s.is_first_step(i):
                xs = x
            d = c.hx * x + c.he * e
            x = c.cx * x + c.cd * d + c.cp * d_prev + c.cs * xs
        else:
            c = s.step_coeffs(i)
            d = c.hx * x + c.he * e
            x = c.cx * x + c.cd * d + c.cp * d_prev
        d_prev = d
    return x - exact


def test_convergence_order():
    """Per doubling of the UNet evaluations the DPM-Solver++(2S) error falls by more than 3.4x (second order: 3.5, 3.7,
    3.9). DPM-Solver++(2M) at the same number of evaluations converges faster still on this problem (its error crosses
    zero near M = 96), so it is only checked to fall at least second order over the three doublings."""
    Ms = (12, 24, 48, 96)
    e2s = [_ode_error(M, "2s") for M in Ms]
    e2m = [_ode_error(M, "2m") for M in Ms]
    r2s = [e2s[k] / e2s[k + 1] for k in range(len(Ms) - 1)]
    r2m = [e2m[k] / e2m[k + 1] for k in range(len(Ms) - 1)]
    print("2S errors", ["%.2e" % v for v in e2s], "ratios", [round(float(r), 2) for r in r2s])
    print("2M errors", ["%.2e" % v for v in e2m], "ratios", [round(float(r), 2) for r in r2m])
    assert min(r2s) > 3.4, r2s
    assert all(abs(e2s[k + 1]) < abs(e2s[k]) for k in range(len(Ms) - 1))
    assert abs(e2m[-1]) < abs(e2m[0]) / 64, e2m


# ------------------------------------------------------------------------------------------------ CPU: goldens
def _xl_plain_oracle(steps, sched=None):
    from oracle import sampler_oracle as sam, unet_oracle as uo
    cfg = uo.tiny_xl_config()
    S = mo.LATENT_XL_PLAIN
    unet = sam.make_unet_fn(uo.make_state_dict(cfg, 2), cfg)
    inp = synth.synth_inputs(cfg.cross_attention_dim, _pooled(cfg), 3, S, 31)
    ctx, te = inp["ctx"], inp["text_embeds"]
    added2 = {"text_embeds": torch.cat([te[:1], te[-1:]]), "time_ids": inp["time_ids"].repeat(2, 1)}
    return so.plain_loop(unet, sched or so.DPMSolverSinglestepSchedulerOracle(), torch.cat([ctx[:1], ctx[-1:]]),
                         inp["latents"].clone(), steps, 8.5, added_cond=added2)


# the colour guidance of each recorded rich loop (tests/gen_singlestep.py explains why 0 / 0 runs without it)
RICH_COLOUR = {(0.5, 0.5): False, (0.0, 0.0): False}


def _xl_rich_oracle(inject_selfattn, inject_background, steps=4, colour=True):
    """The oracle rich loop with one scheduler state per trajectory (tests/multistep_oracle.py): where the reference
    steps both trajectories jointly on every step this is the reference's loop."""
    from oracle import sampler_oracle as sam, unet_oracle as uo
    cfg = uo.tiny_xl_config()
    S = mo.LATENT_XL_RICH
    inp = synth.synth_inputs(cfg.cross_attention_dim, _pooled(cfg), 3, S, 31)
    ctx, te = inp["ctx"], inp["text_embeds"]
    tfd = synth.font_sizes()
    tfd.update(synth.color_dict(inp["masks"], S, 1.0))
    main, ref = so.DPMSolverSinglestepSchedulerOracle(), so.DPMSolverSinglestepSchedulerOracle()
    out = so.rich_text_loop(sam.make_unet_fn(uo.make_state_dict(cfg, 2), cfg), main, ref, ctx, inp["masks"],
                            inp["latents"].clone(), steps, 8.5, xl=True,
                            added_cond={"text_embeds": te, "time_ids": inp["time_ids"]}, use_guidance=colour,
                            text_format_dict=tfd, inject_selfattn=inject_selfattn,
                            inject_background=inject_background, vae_decode=synth.TinyVAE(), scaling_factor=0.13025)
    return out, main.step_batches, ref.step_batches


def _sd_rich_oracle(steps=5):
    from oracle import sampler_oracle as sam, unet_oracle as uo
    cfg = uo.tiny_sd_config()
    S = mo.LATENT_SD
    inp = synth.synth_inputs(cfg.cross_attention_dim, 0, 3, S, 21)
    tfd = synth.font_sizes()
    tfd.update(synth.color_dict(inp["masks"], S, 0.5))
    return so.rich_text_loop(sam.make_unet_fn(uo.make_state_dict(cfg, 1), cfg), so.DPMSolverSinglestepSchedulerOracle(),
                             so.DPMSolverSinglestepSchedulerOracle(), inp["ctx"], inp["masks"], inp["latents"].clone(),
                             steps, 8.5, xl=False, use_guidance=True, text_format_dict=tfd, inject_selfattn=0.3,
                             inject_background=0.5, vae_decode=synth.TinyVAE(), scaling_factor=0.18215)


def _assert_golden(got, ref, what):
    np.testing.assert_allclose(np.asarray(got, np.float32), ref, atol=5e-4 * max(1.0, float(np.abs(ref).max()) / 10),
                               rtol=1e-4, err_msg=what)


@pytest.mark.parametrize("steps", [5, 10])
def test_oracle_xl_plain_matches_reference(steps):
    """An odd (final first-order step) and an even step count; the reference calls back on every step."""
    _assert_golden(_xl_plain_oracle(steps).numpy(), _golden()[f"xl_plain_{steps}"], f"xl plain {steps}")
    assert _golden()[f"xl_plain_{steps}_callbacks"].tolist() == list(range(steps))


@pytest.mark.parametrize("sa,bg", [(0.5, 0.5), (0.0, 0.0)])
def test_oracle_xl_rich_matches_reference(sa, bg):
    """The reference latents stepped jointly on every step (0.5 / 0.5), and no reference latents (0 / 0); both without
    colour guidance (tests/gen_singlestep.py)."""
    got, main_b, ref_b = _xl_rich_oracle(sa, bg, colour=RICH_COLOUR[sa, bg])
    assert main_b == [1] * 4 and ref_b == ([1] * 4 if sa > 0 else [])
    _assert_golden(got.detach().numpy(), _golden()[f"xl_rich_{sa:g}_{bg:g}"], f"xl rich {sa} {bg}")
    assert _golden()[f"xl_rich_{sa:g}_{bg:g}_callbacks"].tolist() == [0, 1, 2, 3]


def test_oracle_sd_produce_latents_matches_reference():
    _assert_golden(_sd_rich_oracle().detach().numpy(), _golden()["sd_rich_5"], "sd rich")


# ------------------------------------------------------------------------------------------------ CPU: C ABI, cubin
def test_singlestep_abi_rejects_bad_arguments_without_launching():
    """Every call below fails its argument checks; a launch without a device would return RTTI_ERR_CUDA instead."""
    from rtti_b200 import _lib
    lib = _lib.load()
    V = ctypes.c_void_p
    buf = (ctypes.c_char * 8192)()
    a = (ctypes.addressof(buf) + 15) // 16 * 16
    regions = (V * 3)(V(a), V(a), V(a))
    second = (1.1, -0.4, 0.0, 0.9, 0.3, -0.2)   # (hx, he, cx, cs, cd, cp)
    first = (1.1, -0.4, 0.8, 0.0, 0.3, 0.0)
    for fn, extra in ((lib.rtti_region_blend_cfg_ss, []), (lib.rtti_region_blend_cfg_rescale_ss, [0.7])):
        rb = lambda lat=a, b=(a, a, a), n=64, c=second, eu=a, regs=regions, N=3: fn(
            V(eu), regs, V(a), N, n, 7.5, V(a), V(lat), V(lat), *c, *[V(x) for x in b], *extra, V(0))
        assert rb(eu=0) == ARG
        assert rb(regs=(V * 3)(V(a), V(0), V(a))) == ARG
        assert rb(N=17) == ARG
        assert rb(lat=0) == ARG                  # the update needs the latents
        assert rb(b=(a, 0, a)) == ARG            # d_out is always required
        assert rb(b=(0, a, a)) == ARG            # cp != 0 needs d_prev
        assert rb(b=(a, a, 0)) == ARG            # cs != 0 needs xs
        assert rb(b=(0, a, 0), c=first, n=60) == SHAPE   # a first step reads neither d_prev nor xs
        assert rb(n=60) == SHAPE
        assert rb(b=(a, a, a + 2)) == ALIGN
        assert rb(b=(a + 4, a, a)) == ALIGN
        assert rb(b=(0, a, a + 8), c=first) == ALIGN   # a pointer that is given must be aligned
    peers = (V * 2)(V(a), V(a))
    owner = (ctypes.c_int * 6)(0, 0, 1, 1, 0, 1)
    for fn, extra in ((lib.rtti_gather_blend_step_ss, []), (lib.rtti_gather_blend_step_rescale_ss, [0.7])):
        gb = lambda world=2, rank=0, n=64, ref=0, b=(a, a, a), br=(a, a, a), lat=a, slots=peers: fn(
            slots, peers, world, rank, owner, 6, 3, V(a), n, 7.5, V(a), V(lat), V(lat), V(ref), V(ref), *second,
            *[V(x) for x in b], *[V(x) for x in br], 1, *extra, V(0))
        assert gb(world=17) == ARG
        assert gb(rank=2) == ARG
        assert gb(slots=(V * 2)(V(a), V(0))) == ARG
        assert gb(lat=0) == ARG
        assert gb(b=(a, a, 0)) == ARG
        assert gb(ref=a, br=(a, a, 0)) == ARG    # the reference trajectory needs its own xs ...
        assert gb(ref=a, br=(a, 0, a)) == ARG    # ... and its own D buffer
        assert gb(n=60) == SHAPE
        assert gb(b=(a, a, a + 4)) == ALIGN
        assert gb(ref=a, br=(a, a, a + 4)) == ALIGN
        assert gb(world=1) == ARG                # slot owned by rank 1 of a world of 1


def test_singlestep_step_python_checks():
    from rtti_b200 import _lib, ops
    x = torch.zeros(64, dtype=torch.float16)
    d = torch.zeros(64, dtype=torch.float32)
    first = (1.1, -0.4, 0.8, 0.0, 0.3, 0.0)
    second = (1.1, -0.4, 0.0, 0.9, 0.3, -0.2)
    with pytest.raises(_lib.RttiError, match="must be a CUDA tensor"):
        ops.SinglestepStep(first, None, d, None)._check(64, False)
    with pytest.raises(_lib.RttiError, match="d_out is required"):
        ops.SinglestepStep(first, None, None, None)._check(64, False)
    with pytest.raises(_lib.RttiError, match="d_prev is required"):
        ops.SinglestepStep(second, None, d, x)._check(64, False)
    with pytest.raises(_lib.RttiError, match=r"\(hx, he, cx, cs, cd, cp\)"):
        ops.SinglestepStep(first[:5], None, d, None)
    assert len(ops.SinglestepStep(second, d, d, x).args()) == 9
    assert len(ops.SinglestepStep(second, d, d, x, d, d, x).args(ref=True)) == 12


def _sass_by_kernel():
    from rtti_b200 import _lib
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    _lib.load()
    sass = subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True).stdout
    out = {}
    for f in re.split(r"\n\s*Function : ", sass)[1:]:
        name = f.split("\n", 1)[0]
        m = re.search(r"\d(region_blend|gather_blend|blend_rescale)_(ss|ms)_kernel(ILb[01]E)?", name)
        if m:
            out[(m.group(1), m.group(3) or "", m.group(2))] = (name, f)
    return out


def test_singlestep_kernels_in_the_cubin():
    """The four entry points are exported; each of the four kernel families has its _ss kernel, whose 128-bit loads
    are those of its _ms kernel plus xs (for each trajectory it steps); the rescale cluster kernels stay within 64
    registers at 1024 threads, with no spills."""
    from rtti_b200 import _lib
    lib = _lib.load()
    for sym in ("rtti_region_blend_cfg_ss", "rtti_region_blend_cfg_rescale_ss", "rtti_gather_blend_step_ss",
                "rtti_gather_blend_step_rescale_ss"):
        assert hasattr(lib, sym), sym
    k = _sass_by_kernel()
    fams = [("region_blend", "", 1), ("gather_blend", "", 2), ("blend_rescale", "ILb0E", 2), ("blend_rescale", "ILb1E", 2)]
    for fam, tpl, extra in fams:
        assert (fam, tpl, "ss") in k and (fam, tpl, "ms") in k, (fam, tpl, sorted(k))
        ld = {h: len(re.findall(r"\bLDG\.E\.128\b", k[(fam, tpl, h)][1])) for h in ("ms", "ss")}
        assert ld["ss"] >= ld["ms"] + extra, (fam, tpl, ld)
        if fam == "blend_rescale":
            assert not re.search(r"\bSTL", k[(fam, tpl, "ss")][1]), f"{fam}{tpl}: local-memory stores (spills)"
    out = subprocess.run(["cuobjdump", "-res-usage", _lib.LIB_PATH], capture_output=True, text=True).stdout
    regs = [int(r) for fn, r in re.findall(r"Function (\S+):\s*\n\s*REG:(\d+)", out) if "blend_rescale_ss_kernel" in fn]
    assert len(regs) == 2
    for r in regs:
        assert r <= 64 and ((r * 32 + 255) // 256 * 256) * 32 <= 65536, f"{r} registers x 32 warps"


# ------------------------------------------------------------------------------------------------ GPU: accuracy
STEPS = {"first": 4, "second": 5, "last_second": 19}   # iterations of a 20-step grid


def _coeffs(kind):
    s = _ss()
    s.set_timesteps(20)
    i = STEPS[kind]
    assert s.is_first_step(i) == (kind == "first")
    return s.singlestep_coeffs(i)


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _masks(N, n, g):
    m = torch.rand(N, n, device="cuda", generator=g)
    return (m / m.sum(0, keepdim=True)).half().float().contiguous()


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
    xs, xs_ref = rn(3.0), rn(3.0)
    dp, dp_ref = (3.0 * torch.randn(n, device="cuda", generator=g)), (3.0 * torch.randn(n, device="cuda", generator=g))
    return eu, er, m, lat, ec, ed, lat_ref, (xs, dp), (xs_ref, dp_ref)


def _blend64(eu, er, m, guidance, phi):
    md = m.double()
    u64 = sum(eu.double() * md[k] for k in range(len(er)))
    t64 = sum(er[k].double() * md[k] for k in range(len(er)))
    e64 = u64 + guidance * (t64 - u64)
    if phi:
        e64 = e64 * (1 - phi + phi * t64.std() / e64.std())
    return e64


@pytest.mark.gpu
@pytest.mark.parametrize("kind", sorted(STEPS))
@pytest.mark.parametrize("with_ref", [False, True])
@pytest.mark.parametrize("phi", [0.0, 0.7])
@pytest.mark.parametrize("N", [2, 16])
@pytest.mark.parametrize("n", [16384, 65528])
@pytest.mark.parametrize("family", ["single", "gather"])
def test_singlestep_kernels_vs_fp64(family, n, N, phi, with_ref, kind):
    """latents_out (and the reference latents with C/D) against float64 of cx x + cd D + cp D_prev + cs xs on the exact
    blend, D = hx x + he eps; d_out against the fp32 evaluation of D on the fp16 prediction."""
    from rtti_b200 import ops
    from tests.fp64_rule import half_ulp16, no_worse
    c = _coeffs(kind)
    eu, er, m, lat, ec, ed, lat_ref, (xs, dp), (xs_ref, dp_ref) = _inputs(
        n, N, n + 13 * N + int(10 * phi) + 7 * with_ref + 101 * STEPS[kind])
    guidance = 5.0
    ones = torch.ones(1, n, device="cuda")
    d_out, d_out_ref = dp.clone(), dp_ref.clone()   # d_prev aliases d_out, as the samplers pass it
    dp0, dp0_ref = dp.clone(), dp_ref.clone()
    xs_in = xs if c.cs != 0.0 else None
    xs_ref_in = xs_ref if c.cs != 0.0 else None
    if family == "single":
        e1, x1 = ops.region_blend_cfg(eu, er, m, guidance, latents=lat, guidance_rescale=phi,
                                      step=ops.SinglestepStep(c, d_out, d_out, xs_in))
        xr = ops.region_blend_cfg(ec, [ed], ones, guidance, latents=lat_ref, guidance_rescale=phi,
                                  step=ops.SinglestepStep(c, d_out_ref, d_out_ref, xs_ref_in))[1] if with_ref else None
    else:
        ref_bufs = (d_out_ref, d_out_ref, xs_ref_in) if with_ref else (None,) * 3
        step = ops.SinglestepStep(c, d_out, d_out, xs_in, *ref_bufs)
        e1, x1, xr = _gather_world1(eu, er, m, guidance, lat, (ec, ed, lat_ref if with_ref else None), phi, step)
    tag = f"ss {family} n{n} N{N} phi{phi:g} {kind}"
    trajectories = [(e1, x1, lat, xs, dp0, d_out, _blend64(eu, er, m, guidance, phi), "latents")]
    if with_ref:
        e_ref16 = ops.region_blend_cfg(ec, [ed], ones, guidance, guidance_rescale=phi)   # the fp16 prediction stepped
        trajectories.append((e_ref16, xr, lat_ref, xs_ref, dp0_ref, d_out_ref, _blend64(ec, [ed], ones, guidance, phi),
                             "latents_ref"))
    for e16, got, x, xs_, dprev, dgot, e64, what in trajectories:
        D64 = c.hx * x.double() + c.he * e64
        want64 = c.cx * x.double() + c.cd * D64
        D16 = c.hx * x + c.he * e16   # diffusers in fp16: convert_model_output, then the update
        cmp16 = c.cx * x + c.cd * D16
        if c.cp != 0.0:
            want64 = want64 + c.cp * dprev.double()
            cmp16 = cmp16 + c.cp * dprev.half()
        if c.cs != 0.0:
            want64 = want64 + c.cs * xs_.double()
            cmp16 = cmp16 + c.cs * xs_
        no_worse(f"{tag} {what}", got, cmp16, want64, k=2.0, floor=half_ulp16(want64), mean=True)
        d32 = c.hx * x.float() + c.he * e16.float()
        torch.testing.assert_close(dgot, d32, rtol=1e-6, atol=1e-6 * float(d32.abs().max()))


# ------------------------------------------------------------------------------------------------ GPU: bit-identities
@pytest.mark.gpu
@pytest.mark.parametrize("phi", [0.0, 0.7])
@pytest.mark.parametrize("n,N", [(16384, 5), (65528, 2), (65536, 16)])
def test_singlestep_bit_identities(n, N, phi):
    """With cs = 0 every family equals its _ms form bit for bit (eps, latents, d_out, both trajectories), and xs is not
    read (NaN xs); on a second step the gather form at world 1 equals the single form (both trajectories); a CUDA-graph
    replay equals eager."""
    from rtti_b200 import ops
    eu, er, m, lat, ec, ed, lat_ref, (xs, dp), (xs_ref, dp_ref) = _inputs(n, N, n + N + 1)
    ones = torch.ones(1, n, device="cuda")
    guidance = 8.5
    nan = torch.full_like(lat, float("nan"))
    for kind in ("first", "second"):
        c = _coeffs(kind)
        ms_c = (c.hx, c.he, c.cx, c.cd, c.cp)
        cz = c._replace(cs=0.0)
        d_ms, d_ss = dp.clone(), dp.clone()
        e_ms, x_ms = ops.region_blend_cfg(eu, er, m, guidance, latents=lat, guidance_rescale=phi,
                                          step=ops.MultistepStep(ms_c, d_ms, d_ms))
        e_ss, x_ss = ops.region_blend_cfg(eu, er, m, guidance, latents=lat, guidance_rescale=phi,
                                          step=ops.SinglestepStep(cz, d_ss, d_ss, nan))
        assert torch.equal(e_ms, e_ss) and torch.equal(x_ms, x_ss) and torch.equal(d_ms, d_ss), \
            f"cs = 0 differs from the _ms form (single GPU, {kind})"
        bufs = [dp.clone() for _ in range(4)]
        g_ms = _gather_world1(eu, er, m, guidance, lat, (ec, ed, lat_ref), phi,
                              ops.MultistepStep(ms_c, bufs[0], bufs[0], bufs[1], bufs[1]))
        g_ss = _gather_world1(eu, er, m, guidance, lat, (ec, ed, lat_ref), phi,
                              ops.SinglestepStep(cz, bufs[2], bufs[2], nan, bufs[3], bufs[3], nan))
        for a, b, what in list(zip(g_ms, g_ss, ("eps", "latents", "latents_ref"))) + [
                (bufs[0], bufs[2], "d_out"), (bufs[1], bufs[3], "d_out_ref")]:
            assert torch.equal(a, b), f"cs = 0 differs from the _ms form (gather, {kind}): {what}"
    c = _coeffs("second")
    bufs = {}

    def single():
        bufs["m"], bufs["r"] = dp.clone(), dp_ref.clone()
        eps, lo_ = ops.region_blend_cfg(eu, er, m, guidance, latents=lat, guidance_rescale=phi,
                                        step=ops.SinglestepStep(c, bufs["m"], bufs["m"], xs))
        _, ro = ops.region_blend_cfg(ec, [ed], ones, guidance, latents=lat_ref, guidance_rescale=phi,
                                     step=ops.SinglestepStep(c, bufs["r"], bufs["r"], xs_ref))
        return eps, lo_, ro, bufs["m"], bufs["r"]

    a = single()
    for x, y in zip(a, single()):
        assert torch.equal(x, y), "two calls differ"
    gm, gr = dp.clone(), dp_ref.clone()
    gw = _gather_world1(eu, er, m, guidance, lat, (ec, ed, lat_ref), phi,
                        ops.SinglestepStep(c, gm, gm, xs, gr, gr, xs_ref))
    for x, y, what in zip(a, list(gw) + [gm, gr], ("eps", "latents", "latents_ref", "d_out", "d_out_ref")):
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


@pytest.mark.gpu
def test_singlestep_step_refuses_xs_overlapping_an_output():
    from rtti_b200 import _lib, ops
    n = 16384
    eu, er, m, lat, ec, ed, lat_ref, (xs, dp), _ = _inputs(n, 2, 5)
    from rtti_b200.ops import _overlap
    step = ops.SinglestepStep(_coeffs("second"), dp, dp, xs)
    step._check(n, False, (torch.empty_like(lat),))
    assert not _overlap(xs, lat)
    with pytest.raises(_lib.RttiError, match="xs overlaps"):
        step._check(n, False, (xs,))


# ------------------------------------------------------------------------------------------------ GPU: samplers
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


def _xl_plain(steps, scheduler=None, calls=None, phi=0.0):
    cfg, m = _xl_model(scheduler or _ss())
    S = mo.LATENT_XL_PLAIN
    inp = synth.synth_inputs(cfg.cross_attention_dim, _pooled(cfg), 3, S, 31)
    ctx, te = inp["ctx"].cuda(), inp["text_embeds"].cuda()
    cb = (lambda i, t, lat: calls.append(i)) if calls is not None else None
    return m.sample(height=S * 8, width=S * 8, num_inference_steps=steps, guidance_scale=8.5,
                    latents=inp["latents"].clone(), prompt_embeds=ctx[-1:], negative_prompt_embeds=ctx[:1],
                    pooled_prompt_embeds=te[-1:], negative_pooled_prompt_embeds=te[:1], output_type="latent",
                    run_rich_text=False, callback=cb, callback_steps=1,
                    guidance_rescale=phi).images.float().cpu().numpy()


def _xl_rich(sa, bg, scheduler=None, graphs=True, calls=None, callback_steps=1, colour=True):
    cfg, m = _xl_model(scheduler or _ss())
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
                    output_type="latent", run_rich_text=True, use_guidance=colour, inject_selfattn=sa,
                    inject_background=bg, text_format_dict=tfd, callback=cb,
                    callback_steps=callback_steps).images.float().cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("steps", [5, 10])
def test_xl_plain_vs_reference_golden(steps):
    """The plain pass against the reference's, and its callback iterations (every step); the DPM-Solver++(2M) run of
    the same inputs lies outside the tolerance; with guidance_rescale the rescale form runs and differs."""
    from rtti_b200.schedulers import DPMSolverMultistepScheduler
    ref = _golden()[f"xl_plain_{steps}"]
    calls = []
    out = _xl_plain(steps, calls=calls)
    _close_range(out, ref, f"xl plain {steps}")
    assert calls == _golden()[f"xl_plain_{steps}_callbacks"].tolist() == list(range(steps)), calls
    with pytest.raises(AssertionError):
        _close_range(_xl_plain(steps, DPMSolverMultistepScheduler()), ref, "xl plain, 2M")
    resc = _xl_plain(steps, phi=0.7)
    assert np.isfinite(resc).all() and not np.array_equal(resc, out)


@pytest.mark.gpu
@pytest.mark.parametrize("sa,bg", [(0.5, 0.5), (0.0, 0.0)])
def test_xl_rich_vs_reference_golden(sa, bg):
    """Injection and font sizes against the reference's loop, with its callback iterations; the DPM-Solver++(2M) run lies outside the tolerance; CUDA-graph replayed UNet passes give the same bits as eager ones."""
    from rtti_b200.schedulers import DPMSolverMultistepScheduler
    ref = _golden()[f"xl_rich_{sa:g}_{bg:g}"]
    calls = []
    colour = RICH_COLOUR[sa, bg]
    out = _xl_rich(sa, bg, calls=calls, colour=colour)
    _close_range(out, ref, f"xl rich {sa} {bg}")
    assert calls == _golden()[f"xl_rich_{sa:g}_{bg:g}_callbacks"].tolist(), calls
    with pytest.raises(AssertionError):
        _close_range(_xl_rich(sa, bg, DPMSolverMultistepScheduler(), colour=colour), ref, "xl rich, 2M")
    calls2 = []
    assert np.array_equal(out, _xl_rich(sa, bg, graphs=False, calls=calls2, callback_steps=2, colour=colour)), \
        "use_cuda_graphs on / off differ"
    assert calls2 == [0, 2], calls2


@pytest.mark.gpu
def test_rich_loop_keeps_a_state_per_trajectory():
    """inject_selfattn = 0, inject_background = 0.5: the reference latents are stepped on steps 0 and 1 only (one whole
    block); the main latents go on with their own state, as the per-trajectory oracle loop does."""
    ref, main_b, ref_b = _xl_rich_oracle(0.0, 0.5)
    assert main_b == [1, 1, 1, 1] and ref_b == [1, 1]
    _close_range(_xl_rich(0.0, 0.5), ref.detach().numpy(), "xl rich 0 / 0.5 vs the per-trajectory oracle")


def _sd_model(scheduler):
    from oracle import unet_oracle as uo
    from rtti_b200.region_diffusion import RegionDiffusion
    from rtti_b200.unet import UNet2DConditionModel, UNetConfig
    cfg = uo.tiny_sd_config()
    unet = UNet2DConditionModel(UNetConfig.from_dict(cfg.__dict__))
    unet.load_state_dict(uo.make_state_dict(cfg, 1))
    m = RegionDiffusion(device="cuda", unet=unet.finalize("cuda"), vae=synth.TinyVAE("cuda"))
    if scheduler is not None:
        m.scheduler = scheduler
    return cfg, m


def _sd_rich(scheduler):
    cfg, m = _sd_model(scheduler)
    S = mo.LATENT_SD
    inp = synth.synth_inputs(cfg.cross_attention_dim, 0, 3, S, 21)
    m.masks = [x.cuda() for x in inp["masks"]]
    tfd = synth.font_sizes()
    tfd.update(synth.color_dict(inp["masks"], S, 0.5))
    return m.produce_latents(inp["ctx"].cuda(), height=S * 8, width=S * 8, num_inference_steps=5, guidance_scale=8.5,
                             latents=inp["latents"].clone(), use_guidance=True, text_format_dict=tfd,
                             inject_selfattn=0.3, inject_background=0.5).float().cpu().numpy()


@pytest.mark.gpu
def test_sd_produce_latents_vs_reference_golden():
    """Against the reference's produce_latents; the PLMS run of the same inputs lies outside the tolerance."""
    out = _sd_rich(_ss())
    _close_range(out, _golden()["sd_rich_5"], "sd produce_latents 2S")
    with pytest.raises(AssertionError):
        _close_range(out, _sd_rich(None), "sd 2S vs PLMS")


@pytest.mark.gpu
@pytest.mark.parametrize("steps", [5, 6])
def test_sd_produce_attn_maps_vs_oracle(steps):
    """produce_attn_maps (the plain CFG loop of the SD1.5 sampler) against the oracle's plain loop."""
    from oracle import sampler_oracle as sam, unet_oracle as uo
    cfg, m = _sd_model(_ss())
    S = mo.LATENT_SD
    inp = synth.synth_inputs(cfg.cross_attention_dim, 0, 3, S, 21)
    ctx = torch.cat([inp["ctx"][:1], inp["ctx"][-1:]])
    out = m.produce_attn_maps(None, height=S * 8, width=S * 8, num_inference_steps=steps, guidance_scale=7.5,
                              latents=inp["latents"].clone(), text_embeddings=ctx.cuda(), decode=False)
    ref = so.plain_loop(sam.make_unet_fn(uo.make_state_dict(cfg, 1), cfg), so.DPMSolverSinglestepSchedulerOracle(),
                        ctx, inp["latents"].clone(), steps, 7.5)
    _close_range(out.float().cpu().numpy(), ref.numpy(), f"sd produce_attn_maps 2S {steps} vs oracle")


@pytest.mark.gpu
def test_rich_loop_singlestep_two_gpus():
    """DPM-Solver++(2S) on the fused peer exchange and on the NCCL path (tests/multigpu_singlestep_check.py)."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
                        "--master-addr", "127.0.0.1", "--master-port", "29549",
                        os.path.join(ROOT, "tests", "multigpu_singlestep_check.py")],
                       capture_output=True, text=True, timeout=900)
    print(r.stdout[-2000:], r.stderr[-2000:])
    assert r.returncode == 0 and "MULTIGPU_SINGLESTEP_CHECK PASS" in r.stdout
