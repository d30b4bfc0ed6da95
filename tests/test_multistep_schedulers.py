"""DDIM and DPM-Solver++(2M) in both samplers, with the multistep update fused into the blend kernels
(rtti_region_blend_cfg_ms, rtti_region_blend_cfg_rescale_ms, rtti_gather_blend_step_ms,
rtti_gather_blend_step_rescale_ms).

CPU: the timestep grids, invariants that do not rest on the restatement (a constant data prediction is carried exactly;
convergence orders on nested grids), step_coeffs against a float64 step of the scheduler definitions, the oracle loops
against the unmodified reference (tests/golden/multistep.npz, tests/gen_multistep.py), the C-ABI argument checks and
the cubin. GPU: the kernels against float64 (tests/fp64_rule.py, K = 2, mean check on; the comparator is the fp16 torch
expression diffusers evaluates), bit-identities, and both samplers against the goldens and the oracle."""
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
from tests import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
ARG, SHAPE, ALIGN = -1, -2, -3


def _golden(name="multistep.npz"):
    return np.load(os.path.join(GOLDEN, name), allow_pickle=False)


def _sched(kind):
    from rtti_b200 import schedulers as S
    return {"ddim": S.DDIMScheduler, "dpmpp_2m": S.DPMSolverMultistepScheduler, "euler": S.EulerDiscreteScheduler,
            "plms": S.PNDMScheduler}[kind]()


def _pooled(cfg):
    return cfg.projection_class_embeddings_input_dim - 6 * cfg.addition_time_embed_dim


# ------------------------------------------------------------------------------------------------ CPU: grids
GRIDS = {
    ("ddim", 10): [901, 801, 701, 601, 501, 401, 301, 201, 101, 1],
    ("ddim", 20): [951, 901, 851, 801, 751, 701, 651, 601, 551, 501, 451, 401, 351, 301, 251, 201, 151, 101, 51, 1],
    ("ddim", 41): [961, 937, 913, 889, 865, 841, 817, 793, 769, 745, 721, 697, 673, 649, 625, 601, 577, 553, 529, 505,
                   481, 457, 433, 409, 385, 361, 337, 313, 289, 265, 241, 217, 193, 169, 145, 121, 97, 73, 49, 25, 1],
    ("dpmpp_2m", 10): [999, 899, 799, 699, 599, 500, 400, 300, 200, 100],
    ("dpmpp_2m", 20): [999, 949, 899, 849, 799, 749, 699, 649, 599, 549, 500, 450, 400, 350, 300, 250, 200, 150, 100, 50],
    ("dpmpp_2m", 41): [999, 975, 950, 926, 902, 877, 853, 828, 804, 780, 755, 731, 707, 682, 658, 634, 609, 585, 560, 536,
                       512, 487, 463, 439, 414, 390, 365, 341, 317, 292, 268, 244, 219, 195, 171, 146, 122, 97, 73, 49,
                       24],
}


@pytest.mark.parametrize("kind,N", sorted(GRIDS))
def test_timestep_grid(kind, N):
    s = _sched(kind)
    s.set_timesteps(N)
    assert s.timesteps.dtype == torch.int64 and s.timesteps.device.type == "cpu"
    assert s.timesteps.tolist() == GRIDS[(kind, N)]
    assert s.init_noise_sigma == 1.0
    x = torch.randn(3)
    assert s.scale_model_input(x, s.timesteps[0]) is x


def test_timestep_grid_1000():
    """DDIM: every 1000//1000 = 1 step, 1000..1. DPM: round(linspace(0, 999, 1001)) has one duplicate pair (500 from both
    499.5 and 500.499); dropping it leaves the 999 timesteps 999..1."""
    d = _sched("ddim")
    d.set_timesteps(1000)
    assert d.timesteps.tolist() == list(range(1000, 0, -1))
    s = _sched("dpmpp_2m")
    s.set_timesteps(1000)
    assert s.timesteps.tolist() == list(range(999, 0, -1))
    assert s.num_inference_steps == 999
    c = s.step_coeffs(998)   # the last step lands on t = 0 and, at >= 15 steps, stays second order
    assert c.cp != 0.0


def test_alphas_cumprod_and_config():
    from rtti_b200 import schedulers as S
    e = S.EulerDiscreteScheduler()
    for cls in (S.DDIMScheduler, S.DPMSolverMultistepScheduler):
        s = cls()
        assert torch.equal(s.alphas_cumprod, e.alphas_cumprod)
        assert isinstance(cls.from_config(e), cls) and isinstance(cls.from_config(dict(s.config)), cls)
        assert cls.from_config(S.PNDMScheduler().config).config.steps_offset == 1
    with pytest.raises(NotImplementedError):
        S.DPMSolverMultistepScheduler(use_karras_sigmas=True)
    with pytest.raises(NotImplementedError):
        S.DPMSolverMultistepScheduler(solver_order=3)
    with pytest.raises(NotImplementedError):
        S.DPMSolverMultistepScheduler(algorithm_type="sde-dpmsolver++")
    with pytest.raises(NotImplementedError):
        S.DDIMScheduler(clip_sample=True)
    with pytest.raises(NotImplementedError):
        S.DDIMScheduler(prediction_type="v_prediction")


# ------------------------------------------------------------------------------------------------ CPU: invariants
def _ac64():
    from rtti_b200.schedulers import _alphas_cumprod
    ac = _alphas_cumprod(0.00085, 0.012, 1000).double().numpy()
    return np.sqrt(ac), np.sqrt(1 - ac)


def _run_coeffs(s, x, eps_fn, steps, first_order=False):
    """Step x with the scheduler's coefficients; eps_fn(i, t, x) gives the noise prediction."""
    d_prev = None
    for i in range(steps):
        c = s.step_coeffs(i)
        cd, cp = (c.cd + c.cp, 0.0) if first_order else (c.cd, c.cp)
        d = c.hx * x + c.he * eps_fn(i, int(s.timesteps_host[i]), x)
        x = c.cx * x + cd * d + (cp * d_prev if cp else 0.0)
        d_prev = d
    return x


@pytest.mark.parametrize("kind,N,first", [("ddim", 10, False), ("dpmpp_2m", 10, False), ("dpmpp_2m", 20, False),
                                          ("dpmpp_2m", 20, True)])
def test_constant_data_prediction_is_exact(kind, N, first):
    """With D constant every step lands on alpha_s D + (sigma_s / sigma_t)(x - alpha_t D), to round-off."""
    al, sg = _ac64()
    s = _sched(kind)
    s.set_timesteps(N)
    rng = np.random.default_rng(3)
    D = rng.standard_normal(64)
    x = rng.standard_normal(64)
    for i in range(len(s.timesteps_host)):
        t = int(s.timesteps_host[i])
        if kind == "ddim":
            tgt = max(t - 1000 // N, 0)
        else:
            tgt = 0 if i == len(s.timesteps_host) - 1 else int(s.timesteps_host[i + 1])
        eps = (x - al[t] * D) / sg[t]
        c = s.step_coeffs(i)
        cd, cp = (c.cd + c.cp, 0.0) if first else (c.cd, c.cp)
        d = c.hx * x + c.he * eps
        np.testing.assert_allclose(d, D, rtol=1e-12, atol=1e-12)
        xn = c.cx * x + cd * d + cp * D
        want = al[tgt] * D + (sg[tgt] / sg[t]) * (x - al[t] * D)
        np.testing.assert_allclose(xn, want, rtol=1e-12, atol=1e-12)
        x = xn


def test_convergence_orders():
    """Nested DPM grids N = 20, 40, 80, 160 stopped at t = 500 (the grid point all four share), with a smooth data
    prediction D(lambda) that ignores x: the exact solution is x_s = (sigma_s/sigma_t) x_t + sigma_s int e^l D(l) dl.
    The error falls ~4x per doubling for 2M and ~2x for the first-order update."""
    from scipy.integrate import quad
    al, sg = _ac64()
    lam = np.log(al) - np.log(sg)
    Dfn = np.sin
    x0 = 0.7
    t0, t1 = 999, 500
    exact = (sg[t1] / sg[t0]) * x0 + sg[t1] * quad(lambda l: math.exp(l) * Dfn(l), lam[t0], lam[t1], epsabs=1e-14,
                                                   epsrel=1e-14)[0]
    ratios = {}
    for first in (False, True):
        errs = []
        for N in (20, 40, 80, 160):
            s = _sched("dpmpp_2m")
            s.set_timesteps(N)
            steps = int(np.nonzero(s.timesteps_host == t1)[0][0])
            assert s.timesteps_host[0] == t0
            got = _run_coeffs(s, np.array([x0]), lambda i, t, x: (x - al[t] * Dfn(lam[t])) / sg[t], steps, first)[0]
            errs.append(abs(got - exact))
        ratios[first] = [errs[k] / errs[k + 1] for k in range(3)]
    print("error ratios per doubling: 2M", ratios[False], "first order", ratios[True])
    assert min(ratios[False]) > 3.5, ratios[False]
    assert min(ratios[True]) > 1.8, ratios[True]


@pytest.mark.parametrize("kind,N", [("ddim", 5), ("ddim", 41), ("dpmpp_2m", 2), ("dpmpp_2m", 5), ("dpmpp_2m", 14),
                                    ("dpmpp_2m", 15), ("dpmpp_2m", 20)])
def test_step_coeffs_match_float64_step(kind, N):
    """Every step index: first order, second order, and the last step (first order below 15 steps, second order from
    15). The oracle steps from the scheduler definitions in float64, not from the affine coefficients."""
    s = _sched(kind)
    s.set_timesteps(N)
    g = torch.Generator().manual_seed(N)
    x, e, dp = (torch.randn(256, generator=g, dtype=torch.float64) * 3 for _ in range(3))
    n = len(s.timesteps_host)
    for i in range(n):
        t, _, f = mo.coeffs64(kind, N, i)
        assert t == int(s.timesteps_host[i])
        want, D = f(x, e, dp)
        c = s.step_coeffs(i)
        d = c.hx * x + c.he * e
        got = c.cx * x + c.cd * d + c.cp * dp
        torch.testing.assert_close(d, D, rtol=1e-12, atol=1e-12)
        torch.testing.assert_close(got, want, rtol=1e-12, atol=1e-12)
        second = kind == "dpmpp_2m" and i > 0 and not (i == n - 1 and n < 15)
        assert (c.cp != 0.0) == second, (i, c)


def test_first_order_dpm_equals_ddim():
    """A first-order DPM step and a DDIM step between the same timesteps have the same coefficients."""
    al, sg = _ac64()
    s = _sched("dpmpp_2m")
    for N in (5, 10, 14):
        s.set_timesteps(N)
        ts = s.timesteps_host
        for i in (0, len(ts) - 1):
            t, tgt = int(ts[i]), (0 if i == len(ts) - 1 else int(ts[i + 1]))
            c = s.step_coeffs(i)
            # DDIM: x' = alpha_s x0 + sigma_s eps = alpha_s D + sigma_s (x - alpha_t D) / sigma_t
            assert c.cp == 0.0
            np.testing.assert_allclose([c.cx, c.cd], [sg[tgt] / sg[t], al[tgt] - sg[tgt] * al[t] / sg[t]], rtol=1e-12)


def test_product_step_matches_oracle_scheduler():
    """The schedulers' torch `step` (step_coeffs with a kept history) against the diffusers-form oracle, fp32."""
    for kind in ("ddim", "dpmpp_2m"):
        for N in (4, 16):
            s, o = _sched(kind), mo.SCHEDULERS[kind]()
            s.set_timesteps(N)
            o.set_timesteps(N)
            assert s.timesteps.tolist() == o.timesteps.tolist()
            g = torch.Generator().manual_seed(5)
            x = torch.randn(2, 4, 8, 8, generator=g)
            xo = x.clone()
            for t in s.timesteps:
                e = torch.randn(2, 4, 8, 8, generator=g)
                x = s.step(e, t, x)["prev_sample"]
                xo = o.step(e, t, xo)["prev_sample"]
            torch.testing.assert_close(x, xo, rtol=2e-5, atol=2e-5 * float(xo.abs().max()))


# ------------------------------------------------------------------------------------------------ CPU: goldens
def _xl_plain_oracle(kind, steps):
    from oracle import sampler_oracle as sam, unet_oracle as uo
    cfg = uo.tiny_xl_config()
    S = mo.LATENT_XL_PLAIN
    unet = sam.make_unet_fn(uo.make_state_dict(cfg, 2), cfg)
    inp = synth.synth_inputs(cfg.cross_attention_dim, _pooled(cfg), 3, S, 31)
    ctx, te = inp["ctx"], inp["text_embeds"]
    added2 = {"text_embeds": torch.cat([te[:1], te[-1:]]), "time_ids": inp["time_ids"].repeat(2, 1)}
    return mo.plain_loop(unet, mo.SCHEDULERS[kind](), torch.cat([ctx[:1], ctx[-1:]]), inp["latents"].clone(), steps, 8.5,
                         added_cond=added2)


def _xl_rich_oracle(kind, steps, inject_selfattn=0.5, inject_background=0.5, colour=True):
    from oracle import sampler_oracle as sam, unet_oracle as uo
    cfg = uo.tiny_xl_config()
    S = mo.LATENT_XL_RICH
    inp = synth.synth_inputs(cfg.cross_attention_dim, _pooled(cfg), 3, S, 31)
    ctx, te = inp["ctx"], inp["text_embeds"]
    tfd = synth.font_sizes()
    if colour:
        tfd.update(synth.color_dict(inp["masks"], S, 1.0))
    return mo.rich_text_loop(sam.make_unet_fn(uo.make_state_dict(cfg, 2), cfg), mo.SCHEDULERS[kind](),
                             mo.SCHEDULERS[kind](), ctx, inp["masks"], inp["latents"].clone(), steps, 8.5, xl=True,
                             added_cond={"text_embeds": te, "time_ids": inp["time_ids"]}, use_guidance=colour,
                             text_format_dict=tfd, inject_selfattn=inject_selfattn, inject_background=inject_background,
                             vae_decode=synth.TinyVAE(), scaling_factor=0.13025)


def _sd_rich_oracle(kind, steps):
    from oracle import sampler_oracle as sam, unet_oracle as uo
    cfg = uo.tiny_sd_config()
    S = mo.LATENT_SD
    inp = synth.synth_inputs(cfg.cross_attention_dim, 0, 3, S, 21)
    tfd = synth.font_sizes()
    tfd.update(synth.color_dict(inp["masks"], S, 0.5))
    return mo.rich_text_loop(sam.make_unet_fn(uo.make_state_dict(cfg, 1), cfg), mo.SCHEDULERS[kind](),
                             mo.SCHEDULERS[kind](), inp["ctx"], inp["masks"], inp["latents"].clone(), steps, 8.5, xl=False,
                             use_guidance=True, text_format_dict=tfd, inject_selfattn=0.3, inject_background=0.5,
                             vae_decode=synth.TinyVAE(), scaling_factor=0.18215)


def _assert_golden(got, ref, what):
    """test_xl_loops_match_reference's tolerance for the oracle against the reference."""
    np.testing.assert_allclose(np.asarray(got, np.float32), ref, atol=5e-4 * max(1.0, float(np.abs(ref).max()) / 10),
                               rtol=1e-4, err_msg=what)


@pytest.mark.parametrize("kind,steps", [("dpmpp_2m", 12), ("dpmpp_2m", 16), ("ddim", 10)])
def test_oracle_xl_plain_matches_reference(kind, steps):
    _assert_golden(_xl_plain_oracle(kind, steps).numpy(), _golden()[f"xl_plain_{kind}_{steps}"], f"xl plain {kind}")


def test_oracle_xl_rich_matches_reference():
    """inject_selfattn > 0: the reference steps both trajectories jointly on every step, which equals one scheduler
    state per trajectory. (The DDIM form of the loop has no fixture of its own: its step is pinned by the plain-pass
    fixture and the loop by this one.)"""
    _assert_golden(_xl_rich_oracle("dpmpp_2m", 4).detach().numpy(), _golden()["xl_rich_dpmpp_2m_4"], "xl rich dpm")


def test_oracle_sd_produce_latents_matches_reference():
    _assert_golden(_sd_rich_oracle("dpmpp_2m", 4).detach().numpy(), _golden()["sd_rich_dpmpp_2m_4"], "sd rich dpm")


# ------------------------------------------------------------------------------------------------ CPU: C ABI, cubin
def test_multistep_abi_rejects_bad_arguments_without_launching():
    from rtti_b200 import _lib
    lib = _lib.load()
    V = ctypes.c_void_p
    buf = (ctypes.c_char * 8192)()
    a = (ctypes.addressof(buf) + 15) // 16 * 16
    regions = (V * 3)(V(a), V(a), V(a))
    co = (1.5, -0.5, 0.9, 0.1, 0.2)
    for fn, extra in ((lib.rtti_region_blend_cfg_ms, []), (lib.rtti_region_blend_cfg_rescale_ms, [0.7])):
        rb = lambda lat=a, dprev=a, dout=a, n=64, cp=0.2, eu=a, regs=regions, N=3: fn(
            V(eu), regs, V(a), N, n, 7.5, V(a), V(lat), V(lat), *co[:4], cp, V(dprev), V(dout), *extra, V(0))
        assert rb(eu=0) == ARG
        assert rb(regs=(V * 3)(V(a), V(0), V(a))) == ARG
        assert rb(N=17) == ARG
        assert rb(lat=0) == ARG                   # the multistep update needs the latents
        assert rb(dout=0) == ARG                  # and a D output
        assert rb(dprev=0) == ARG                 # cp != 0 needs D_prev
        assert rb(n=60) == SHAPE
        assert rb(dprev=a + 4) == ALIGN
        assert rb(dout=a + 8) == ALIGN
    peers = (V * 2)(V(a), V(a))
    owner = (ctypes.c_int * 6)(0, 0, 1, 1, 0, 1)
    for fn, extra in ((lib.rtti_gather_blend_step_ms, []), (lib.rtti_gather_blend_step_rescale_ms, [0.7])):
        gb = lambda world=2, rank=0, n=64, ref=0, dprev=a, dout=a, dprev_ref=a, dout_ref=a, cp=0.2, lat=a, slots=peers: fn(
            slots, peers, world, rank, owner, 6, 3, V(a), n, 7.5, V(a), V(lat), V(lat), V(ref), V(ref), *co[:4], cp,
            V(dprev), V(dout), V(dprev_ref), V(dout_ref), 1, *extra, V(0))
        assert gb(world=17) == ARG
        assert gb(rank=2) == ARG
        assert gb(slots=(V * 2)(V(a), V(0))) == ARG
        assert gb(lat=0) == ARG
        assert gb(dout=0) == ARG
        assert gb(dprev=0) == ARG
        assert gb(ref=a, dout_ref=0) == ARG       # the reference trajectory needs its own history
        assert gb(ref=a, dprev_ref=0) == ARG
        assert gb(n=60) == SHAPE
        assert gb(dprev=a + 4) == ALIGN
        assert gb(world=1) == ARG                 # slot owned by rank 1 of a world of 1


def test_multistep_kernels_in_the_cubin():
    """LDG.E.128 / STG.E.128 in every multistep kernel, no 32-bit global store in the single-GPU and rescale ones, 128-bit
    accesses to both D histories in the gather one, and the rescale cluster kernels at
    64 registers or fewer (their 1024-thread CTAs fit the register file) without spills."""
    from rtti_b200 import _lib
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    _lib.load()
    sass = subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True).stdout
    seen = []
    for f in re.split(r"\n\s*Function : ", sass)[1:]:
        name = f.split("\n", 1)[0]
        if re.search(r"(region_blend_ms|gather_blend_ms|blend_rescale_ms)_kernel", name):
            seen.append(name)
            assert re.search(r"\bLDG\.E\.128", f) and re.search(r"\bSTG\.E\.128", f), f"{name}: no 128-bit accesses"
            if "gather_blend_ms" in name:
                # the fp16 slots / latents go through gather_blend's H8 copies (32-bit, as in the Euler form, which must
                # stay as it is); the fp32 histories of both trajectories are 128-bit: 2 loads + 2 stores each
                assert len(re.findall(r"@P\d LDG\.E\.128\b", f)) >= 4 and len(re.findall(r"\bSTG\.E\.128\b", f)) >= 4, name
            else:
                assert not re.search(r"\bSTG\.E\s", f), f"{name}: 32-bit global stores"
            if "blend_rescale_ms" in name:   # (region_blend's pointer table lives in local memory by design)
                assert not re.search(r"\bSTL", f), f"{name}: local-memory stores (spills)"
    assert len(seen) == 4, seen
    out = subprocess.run(["cuobjdump", "-res-usage", _lib.LIB_PATH], capture_output=True, text=True).stdout
    regs = [int(r) for fn, r in re.findall(r"Function (\S+):\s*\n\s*REG:(\d+)", out) if "blend_rescale_ms_kernel" in fn]
    assert len(regs) == 2
    for r in regs:
        assert r <= 64 and ((r * 32 + 255) // 256 * 256) * 32 <= 65536, f"{r} registers x 32 warps"


# ------------------------------------------------------------------------------------------------ GPU: accuracy
def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _masks(N, n, g):
    m = torch.rand(N, n, device="cuda", generator=g)
    return (m / m.sum(0, keepdim=True)).half().float().contiguous()


STEP_KINDS = {"first": ("dpmpp_2m", 16, 0), "second": ("dpmpp_2m", 16, 7), "ddim": ("ddim", 16, 3),
              "last": ("dpmpp_2m", 16, 15), "last_first": ("dpmpp_2m", 5, 4)}


def _scalars(kind, N, i):
    """(alpha_t, sigma_t, alpha_s, sigma_s, expm1(-h), r or None) of step i, float64."""
    al, sg = _ac64()
    s = _sched(kind)
    s.set_timesteps(N)
    ts = s.timesteps_host
    t = int(ts[i])
    if kind == "ddim":
        tgt = max(t - 1000 // N, 0)
    else:
        tgt = 0 if i == len(ts) - 1 else int(ts[i + 1])
    lam = lambda k: math.log(al[k]) - math.log(sg[k])
    h = lam(tgt) - lam(t)
    c = s.step_coeffs(i)
    r = (lam(t) - lam(int(ts[i - 1]))) / h if c.cp != 0.0 else None
    return s, c, (al[t], sg[t], al[tgt], sg[tgt], math.expm1(-h), r)


def _diffusers16(kind, x, e, dprev16, sc):
    """The fp16 torch expressions diffusers evaluates for this step: (x', x0 prediction)."""
    a_t, s_t, a_s, s_s, em, r = sc
    x0 = (x - s_t * e) / a_t
    if kind == "ddim":
        return a_s * x0 + s_s * e, x0
    a = a_s * em
    out = (s_s / s_t) * x - a * x0
    if r is not None:
        out = out - 0.5 * a * ((1.0 / r) * (x0 - dprev16))
    return out, x0


@pytest.mark.gpu
@pytest.mark.parametrize("phi", [0.0, 0.7])
@pytest.mark.parametrize("step_kind", sorted(STEP_KINDS))
@pytest.mark.parametrize("N", [2, 5, 16])
@pytest.mark.parametrize("n", [16384, 65536, 65528])
def test_region_blend_cfg_ms_vs_fp64(n, N, step_kind, phi):
    """latents_out and d_out against float64; eps_out bit-identical to the Euler entry point's."""
    from rtti_b200 import ops
    from tests.fp64_rule import half_ulp16, no_worse
    kind, nsteps, i = STEP_KINDS[step_kind]
    s, c, sc = _scalars(kind, nsteps, i)
    g = _gen(n + 13 * N + len(step_kind) + int(10 * phi))
    eu = torch.randn(n, device="cuda", generator=g).half()
    er = [torch.randn(n, device="cuda", generator=g).half() for _ in range(N)]
    m = _masks(N, n, g)
    a_t, s_t = sc[0], sc[1]
    lat = torch.randn(n, device="cuda", generator=g).half()
    dprev = (torch.randn(n, device="cuda", generator=g) * 1.5).float()
    guidance = 5.0

    def run():
        d = torch.full((n,), float("nan"), device="cuda")
        e, x = ops.region_blend_cfg(eu, er, m, guidance, latents=lat, guidance_rescale=phi,
                                    step=ops.MultistepStep(c, dprev, d))
        return e, x, d
    e1, x1, d1 = run()
    e2, x2, d2 = run()
    assert torch.equal(e1, e2) and torch.equal(x1, x2) and torch.equal(d1, d2), "two calls differ"
    e_euler, _ = ops.region_blend_cfg(eu, er, m, guidance, latents=lat, dt_sigma=-0.3, guidance_rescale=phi)
    assert torch.equal(e1, e_euler), "eps_out differs from the Euler entry point's"
    # float64: the exact blend (+ rescale), stepped without rounding
    md = m.double()
    u64 = sum(eu.double() * md[k] for k in range(N))
    t64 = sum(er[k].double() * md[k] for k in range(N))
    e64 = u64 + guidance * (t64 - u64)
    if phi:
        e64 = e64 * (1 - phi + phi * t64.std() / e64.std())
    x64 = lat.double()
    D64 = (x64 - s_t * e64) / a_t
    want64 = c.cx * x64 + c.cd * D64 + c.cp * dprev.double()
    # comparator: diffusers in fp16 on the fp16 prediction the reference would hold
    x16, D16 = _diffusers16(kind, lat, e1, dprev.half(), sc)
    tag = f"ms n{n} N{N} {step_kind} phi{phi:g}"
    no_worse(tag + " latents", x1, x16, want64, k=2.0, floor=half_ulp16(want64), mean=True)
    no_worse(tag + " d_out", d1, D16, D64, k=2.0, floor=half_ulp16(D64), mean=True)


# ------------------------------------------------------------------------------------------------ GPU: bit-identities
def _gather_world1(eu, er, m, guidance, lat, ref_pair, phi, step, step_id=3):
    from rtti_b200 import ops
    n, N = eu.numel(), len(er)
    n_slots = N + 3
    slots = torch.zeros(2, n_slots, n, dtype=torch.float16, device="cuda")
    flags = torch.zeros(16, dtype=torch.int32, device="cuda")
    for s, e in enumerate([eu] + er + list(ref_pair[:2])):
        slots[step_id & 1, s].copy_(e)
    out = ops.gather_blend_step([slots.data_ptr()], [flags.data_ptr()], 0, [0] * n_slots, N, m, guidance, lat,
                                ref_pair[2], 0.0, step_id, guidance_rescale=phi, step=step)
    torch.cuda.synchronize()
    assert int(flags[0]) == step_id and int(flags[1]) == 0
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("phi", [0.0, 0.7])
@pytest.mark.parametrize("n,N", [(16384, 5), (65528, 2), (65536, 16)])
def test_multistep_bit_identities(n, N, phi):
    """The gather form at world 1 equals the single-GPU form (both trajectories); d_prev aliasing d_out equals separate
    buffers; a CUDA-graph replay equals eager."""
    from rtti_b200 import ops
    s = _sched("dpmpp_2m")
    s.set_timesteps(10)
    c = s.step_coeffs(4)
    assert c.cp != 0.0
    g = _gen(n + N)
    eu = torch.randn(n, device="cuda", generator=g).half()
    er = [torch.randn(n, device="cuda", generator=g).half() for _ in range(N)]
    m = _masks(N, n, g)
    lat = (2 * torch.randn(n, device="cuda", generator=g)).half()
    ec, ed = torch.randn(n, device="cuda", generator=g).half(), torch.randn(n, device="cuda", generator=g).half()
    lat_ref = (2 * torch.randn(n, device="cuda", generator=g)).half()
    dp, dp_ref = torch.randn(n, device="cuda", generator=g), torch.randn(n, device="cuda", generator=g)
    ones = torch.ones(1, n, device="cuda")
    guidance = 8.5

    def single():
        d, dr = torch.empty(n, device="cuda"), torch.empty(n, device="cuda")
        eps, lo = ops.region_blend_cfg(eu, er, m, guidance, latents=lat, guidance_rescale=phi,
                                       step=ops.MultistepStep(c, dp, d))
        _, ro = ops.region_blend_cfg(ec, [ed], ones, guidance, latents=lat_ref, guidance_rescale=phi,
                                     step=ops.MultistepStep(c, dp_ref, dr))
        return eps, lo, ro, d, dr

    a = single()
    b = single()
    for x, y in zip(a, b):
        assert torch.equal(x, y), "two calls differ"
    d, dr = torch.empty(n, device="cuda"), torch.empty(n, device="cuda")
    eps, lo, ro = _gather_world1(eu, er, m, guidance, lat, (ec, ed, lat_ref), phi,
                                 ops.MultistepStep(c, dp, d, dp_ref, dr))
    for x, y, what in zip(a, (eps, lo, ro, d, dr), ("eps", "latents", "latents_ref", "d_out", "d_out_ref")):
        assert torch.equal(x, y), f"gather world 1 vs single GPU: {what} differs"
    # aliasing: D_prev and D_out in one buffer
    hist, hist_ref = dp.clone(), dp_ref.clone()
    _, lo2 = ops.region_blend_cfg(eu, er, m, guidance, latents=lat, guidance_rescale=phi,
                                  step=ops.MultistepStep(c, hist, hist))
    assert torch.equal(lo2, a[1]) and torch.equal(hist, a[3]), "aliased d_prev == d_out differs"
    hist = dp.clone()
    eps3, lo3, ro3 = _gather_world1(eu, er, m, guidance, lat, (ec, ed, lat_ref), phi,
                                    ops.MultistepStep(c, hist, hist, hist_ref, hist_ref))
    assert torch.equal(lo3, a[1]) and torch.equal(ro3, a[2]) and torch.equal(hist, a[3]) and torch.equal(hist_ref, a[4])
    # CUDA-graph capture + replay equals eager
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


# ------------------------------------------------------------------------------------------------ GPU: samplers
def _close_range(got, ref, what):
    got, ref = np.asarray(got, np.float32), np.asarray(ref, np.float32)
    tol = 5e-3 * float(np.abs(ref).max()) + 3e-2 * np.abs(ref)
    err = np.abs(got - ref)
    assert np.isfinite(got).all(), f"{what}: non-finite values"
    assert (err <= tol).all(), f"{what}: {float((err > tol).mean()) * 100:.3f}% outside, max err {err.max():.4f}"
    print(f"{what}: max err {err.max():.4f} mean err {err.mean():.5f}")


def _xl_model(kind):
    from oracle import unet_oracle as uo
    from rtti_b200.region_diffusion_sdxl import RegionDiffusionXL
    from rtti_b200.unet import UNet2DConditionModel, UNetConfig
    cfg = uo.tiny_xl_config()
    unet = UNet2DConditionModel(UNetConfig.from_dict(cfg.__dict__))
    unet.load_state_dict(uo.make_state_dict(cfg, 2))
    return cfg, RegionDiffusionXL(device="cuda", unet=unet.finalize("cuda"), vae=synth.TinyVAE("cuda"),
                                  scheduler=_sched(kind))


def _xl_plain(kind, steps, model=None):
    cfg, m = _xl_model(kind) if model is None else model
    S = mo.LATENT_XL_PLAIN
    inp = synth.synth_inputs(cfg.cross_attention_dim, _pooled(cfg), 3, S, 31)
    ctx, te = inp["ctx"].cuda(), inp["text_embeds"].cuda()
    return m.sample(height=S * 8, width=S * 8, num_inference_steps=steps, guidance_scale=8.5,
                    latents=inp["latents"].clone(), prompt_embeds=ctx[-1:], negative_prompt_embeds=ctx[:1],
                    pooled_prompt_embeds=te[-1:], negative_pooled_prompt_embeds=te[:1], output_type="latent",
                    run_rich_text=False).images.float().cpu().numpy()


def _xl_rich(kind, steps, inject_selfattn=0.5, inject_background=0.5, colour=True, graphs=True):
    cfg, m = _xl_model(kind)
    m.use_cuda_graphs = graphs
    S = mo.LATENT_XL_RICH
    inp = synth.synth_inputs(cfg.cross_attention_dim, _pooled(cfg), 3, S, 31)
    ctx, te = inp["ctx"], inp["text_embeds"]
    tfd = synth.font_sizes()
    if colour:
        tfd.update(synth.color_dict(inp["masks"], S, 1.0))
    m.masks = [x.cuda() for x in inp["masks"]]
    return m.sample(height=S * 8, width=S * 8, num_inference_steps=steps, guidance_scale=8.5,
                    latents=inp["latents"].clone(), prompt_embeds=ctx[1:].cuda(), negative_prompt_embeds=ctx[:1].cuda(),
                    pooled_prompt_embeds=te[1:].cuda(), negative_pooled_prompt_embeds=te[:1].cuda(),
                    output_type="latent", run_rich_text=True, use_guidance=colour, inject_selfattn=inject_selfattn,
                    inject_background=inject_background, text_format_dict=tfd).images.float().cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("kind,steps", [("dpmpp_2m", 12), ("dpmpp_2m", 16), ("ddim", 10)])
def test_xl_plain_vs_reference_golden(kind, steps):
    """Against the reference's plain pass. That the scheduler took effect: DPM lies outside the tolerance of the Euler
    run of the same inputs and step count (the path test_parity_gpu pins to the reference); DDIM, which is Euler's
    method in x / alpha, sigma / alpha and so lies close to that run, outside the tolerance of the DPM run."""
    out = _xl_plain(kind, steps)
    _close_range(out, _golden()[f"xl_plain_{kind}_{steps}"], f"xl plain {kind} {steps}")
    other = "euler" if kind == "dpmpp_2m" else "dpmpp_2m"
    with pytest.raises(AssertionError):
        _close_range(out, _xl_plain(other, steps), f"xl plain vs {other}")


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["dpmpp_2m", "ddim"])
def test_xl_rich_vs_reference(kind):
    """Injection (0.5 / 0.5), font sizes and colour guidance, against the reference's loop (DPM: the fixture; DDIM: the
    oracle loop that fixture pins); the CUDA-graph replayed UNet passes give the same bits as eager ones. DPM lies
    outside the tolerance of the Euler run of the same inputs. DDIM at eta 0 is Euler's method in the variables
    x / alpha, sigma / alpha on the same timesteps (only the last step's target differs), so its latents lie close to
    the Euler run; that it took effect is shown against the DPM fixture instead."""
    out = _xl_rich(kind, 4)
    ref = _golden()["xl_rich_dpmpp_2m_4"] if kind == "dpmpp_2m" else _xl_rich_oracle("ddim", 4).detach().numpy()
    _close_range(out, ref, f"xl rich {kind}")
    other = _xl_rich("euler", 4) if kind == "dpmpp_2m" else _golden()["xl_rich_dpmpp_2m_4"]
    with pytest.raises(AssertionError):
        _close_range(out, other, "xl rich vs Euler" if kind == "dpmpp_2m" else "xl rich ddim vs the DPM golden")
    assert np.array_equal(out, _xl_rich(kind, 4, graphs=False)), "use_cuda_graphs on / off differ"


@pytest.mark.gpu
def test_xl_rich_separate_histories_vs_oracle():
    """inject_selfattn = 0, inject_background = 0.5: the reference latents are stepped on the first half of the steps
    only. Against the oracle with one scheduler state per trajectory (5 DPM steps: second-order steps on both sides of
    the switch)."""
    out = _xl_rich("dpmpp_2m", 5, inject_selfattn=0.0, inject_background=0.5, colour=False)
    ref = _xl_rich_oracle("dpmpp_2m", 5, inject_selfattn=0.0, inject_background=0.5, colour=False)
    _close_range(out, ref.numpy(), "xl rich, separate histories, vs oracle")


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["dpmpp_2m", "ddim"])
def test_sd_produce_latents_vs_reference(kind):
    """Against the reference's produce_latents (DPM: the fixture; DDIM: the oracle loop that fixture pins); the PLMS
    run of the same inputs lies outside the tolerance."""
    out = _sd_rich(kind)
    ref = _golden()["sd_rich_dpmpp_2m_4"] if kind == "dpmpp_2m" else _sd_rich_oracle("ddim", 4).detach().numpy()
    _close_range(out, ref, f"sd produce_latents {kind}")
    with pytest.raises(AssertionError):
        _close_range(out, _sd_rich("plms"), "sd vs PLMS")


def _sd_rich(kind):
    from oracle import unet_oracle as uo
    from rtti_b200.region_diffusion import RegionDiffusion
    from rtti_b200.unet import UNet2DConditionModel, UNetConfig
    cfg = uo.tiny_sd_config()
    unet = UNet2DConditionModel(UNetConfig.from_dict(cfg.__dict__))
    unet.load_state_dict(uo.make_state_dict(cfg, 1))
    m = RegionDiffusion(device="cuda", unet=unet.finalize("cuda"), vae=synth.TinyVAE("cuda"))
    m.scheduler = _sched(kind)
    S = mo.LATENT_SD
    inp = synth.synth_inputs(cfg.cross_attention_dim, 0, 3, S, 21)
    m.masks = [x.cuda() for x in inp["masks"]]
    tfd = synth.font_sizes()
    tfd.update(synth.color_dict(inp["masks"], S, 0.5))
    return m.produce_latents(inp["ctx"].cuda(), height=S * 8, width=S * 8, num_inference_steps=4, guidance_scale=8.5,
                             latents=inp["latents"].clone(), use_guidance=True, text_format_dict=tfd,
                             inject_selfattn=0.3, inject_background=0.5).float().cpu().numpy()


@pytest.mark.gpu
def test_unsupported_scheduler_and_eta():
    from rtti_b200.schedulers import PNDMScheduler
    cfg, m = _xl_model("ddim")
    with pytest.raises(NotImplementedError):
        m.sample(height=256, width=256, num_inference_steps=2, prompt_embeds=torch.zeros(1, 77, 8, device="cuda"),
                 negative_prompt_embeds=torch.zeros(1, 77, 8, device="cuda"), pooled_prompt_embeds=None,
                 negative_pooled_prompt_embeds=None, eta=0.5, output_type="latent")
    m.scheduler = PNDMScheduler()
    with pytest.raises(TypeError, match="DPMSolverMultistepScheduler"):
        m.sample(height=256, width=256, num_inference_steps=2, prompt_embeds=torch.zeros(1, 77, 8, device="cuda"),
                 negative_prompt_embeds=torch.zeros(1, 77, 8, device="cuda"), pooled_prompt_embeds=None,
                 negative_pooled_prompt_embeds=None, output_type="latent")


@pytest.mark.gpu
def test_rich_loop_multistep_two_gpus():
    """DPM-Solver++(2M) on the fused peer-memory exchange and on the NCCL path (tests/multigpu_multistep_check.py)."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
                        "--master-addr", "127.0.0.1", "--master-port", "29539",
                        os.path.join(ROOT, "tests", "multigpu_multistep_check.py")],
                       capture_output=True, text=True, timeout=900)
    print(r.stdout[-2000:], r.stderr[-2000:])
    assert r.returncode == 0 and "MULTIGPU_MULTISTEP_CHECK PASS" in r.stdout
