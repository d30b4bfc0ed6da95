"""UniPC (bh2, order 2) in both samplers, with the predictor-corrector update fused into the blend kernels
(rtti_region_blend_cfg_unipc, rtti_region_blend_cfg_rescale_unipc, rtti_gather_blend_step_unipc,
rtti_gather_blend_step_rescale_unipc).

CPU: unipc_coeffs against the diffusers-form oracle (tests/unipc_oracle.py) in float64 on every step of several grids;
invariants that do not rest on the restatement (a constant data prediction is carried exactly; step 0 is DPM-Solver's
first-order step; the corrector sees the current latents only through m_i); the configuration; the oracle loops
against the unmodified reference (tests/golden/unipc.npz, tests/gen_unipc.py); the C-ABI argument checks and the
cubin. GPU: the kernels against float64 (tests/fp64_rule.py, K = 2, mean check on; the comparator is the fp16 torch
expression diffusers evaluates), bit-identities, and both samplers against the goldens and the oracle."""
import ctypes
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
from tests import unipc_oracle as uo_sched

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
ARG, SHAPE, ALIGN = -1, -2, -3


def _golden():
    return np.load(os.path.join(GOLDEN, "unipc.npz"), allow_pickle=False)


def _unipc(**kw):
    from rtti_b200.schedulers import UniPCMultistepScheduler
    return UniPCMultistepScheduler(**kw)


def _pooled(cfg):
    return cfg.projection_class_embeddings_input_dim - 6 * cfg.addition_time_embed_dim


def _ac64():
    from rtti_b200.schedulers import _alphas_cumprod
    ac = _alphas_cumprod(0.00085, 0.012, 1000).double().numpy()
    return np.sqrt(ac), np.sqrt(1 - ac)


def _apply(c, x, e, xl, m1, m2):
    """The fused form of UniPCCoeffs, evaluated on host tensors: (x', m, xc)."""
    m = c.hx * x + c.he * e
    xc = c.ux * x + c.ul * xl + c.u0 * m + c.u1 * m1 + c.u2 * m2
    return c.vx * xc + c.v0 * m + c.v1 * m1, m, xc


# ------------------------------------------------------------------------------------------------ CPU: configuration
def test_grid_and_config():
    from rtti_b200 import schedulers as S
    u, d = _unipc(), S.DPMSolverMultistepScheduler()
    for N in (1, 5, 10, 20, 1000):
        u.set_timesteps(N)
        d.set_timesteps(N)
        assert u.timesteps.tolist() == d.timesteps.tolist() and u.timesteps.dtype == torch.int64
        assert u.num_inference_steps == d.num_inference_steps
    assert u.init_noise_sigma == 1.0
    x = torch.randn(3)
    assert u.scale_model_input(x, u.timesteps[0]) is x
    assert torch.equal(u.alphas_cumprod, S.EulerDiscreteScheduler().alphas_cumprod)
    for src in (S.EulerDiscreteScheduler(), d, dict(u.config), u):
        assert isinstance(S.UniPCMultistepScheduler.from_config(src), S.UniPCMultistepScheduler)
    assert _unipc(disable_corrector=()).config.disable_corrector == []
    for k, v in dict(solver_order=3, solver_type="bh1", predict_x0=False, lower_order_final=False,
                     disable_corrector=[0], solver_p=S.DDIMScheduler(), use_karras_sigmas=True,
                     prediction_type="v_prediction", thresholding=True, timestep_spacing="leading",
                     trained_betas=[0.1] * 1000).items():
        with pytest.raises(NotImplementedError):
            _unipc(**{k: v})
    with pytest.raises(NotImplementedError):
        _unipc(beta_schedule="linear")
    with pytest.raises(TypeError):
        _unipc(no_such_option=1)
    assert S.MULTISTEP_SCHEDULERS == (S.DDIMScheduler, S.DPMSolverMultistepScheduler)


def test_orders():
    """p_i = min(2, n - i, i + 1) (warm-up, lower_order_final); c_i = p_{i-1}."""
    s = _unipc()
    s.set_timesteps(5)
    assert [s.orders(i) for i in range(5)] == [(1, 0), (2, 1), (2, 2), (2, 2), (1, 2)]
    s.set_timesteps(2)
    assert [s.orders(i) for i in range(2)] == [(1, 0), (1, 1)]
    s.set_timesteps(1)
    assert s.orders(0) == (1, 0)


# ------------------------------------------------------------------------------------------------ CPU: coefficients
@pytest.mark.parametrize("N", [1, 2, 3, 5, 10, 25, 1000])
def test_unipc_coeffs_match_oracle_float64(N):
    """Every step index: the oracle's stateful diffusers-form step (float64 tables) against unipc_coeffs with a kept
    history, on fresh random latents and predictions at each step, so every corrector and predictor term is exercised
    independently of the previous step's output."""
    s = _unipc()
    s.set_timesteps(N)
    o = uo_sched.UniPCSchedulerOracle(dtype=torch.float64)
    o.set_timesteps(N)
    assert s.timesteps.tolist() == o.timesteps.tolist()
    g = torch.Generator().manual_seed(N)
    xl = m1 = m2 = torch.zeros(64, dtype=torch.float64)
    worst = 0.0
    for i, t in enumerate(o.timesteps):
        x, e = (torch.randn(64, generator=g, dtype=torch.float64) * 2 for _ in range(2))
        want = o.step(e, t, x)["prev_sample"]
        got, m, xc = _apply(s.unipc_coeffs(i), x, e, xl, m1, m2)
        torch.testing.assert_close(m, o.model_outputs[-1], rtol=1e-12, atol=1e-12)
        torch.testing.assert_close(xc, o.last_sample, rtol=1e-12, atol=1e-12 * float(xc.abs().max()))
        torch.testing.assert_close(got, want, rtol=1e-12, atol=1e-12 * float(want.abs().max()))
        worst = max(worst, float(((got - want).abs() / want.abs().max()).max()))
        xl, m1, m2 = xc, m, m1
    print(f"N={N}: worst relative deviation {worst:.2e}")


def test_torch_step_matches_oracle():
    """The scheduler's stateful torch `step` against the oracle, in float64 (1e-12) and in fp32 (as diffusers runs)."""
    for dtype, tol in ((torch.float64, 1e-12), (torch.float32, 2e-5)):
        for N in (4, 12):
            s, o = _unipc(), uo_sched.UniPCSchedulerOracle()
            s.set_timesteps(N)
            o.set_timesteps(N)
            g = torch.Generator().manual_seed(5)
            x = torch.randn(2, 4, 8, 8, generator=g, dtype=dtype)
            xo = x.clone()
            o64 = uo_sched.UniPCSchedulerOracle(dtype=torch.float64) if dtype == torch.float64 else o
            o64.set_timesteps(N)
            for t in s.timesteps:
                e = torch.randn(2, 4, 8, 8, generator=g, dtype=dtype)
                x = s.step(e, t, x)["prev_sample"]
                xo = o64.step(e, t, xo)["prev_sample"]
                assert x.dtype == dtype
            torch.testing.assert_close(x, xo, rtol=tol, atol=tol * float(xo.abs().max()))


def test_step0_is_dpm_first_order():
    from rtti_b200.schedulers import DPMSolverMultistepScheduler
    for N in (1, 5, 20):
        s, d = _unipc(), DPMSolverMultistepScheduler()
        s.set_timesteps(N)
        d.set_timesteps(N)
        c, dc = s.unipc_coeffs(0), d.step_coeffs(0)
        assert (c.ux, c.ul, c.u0, c.u1, c.u2, c.v1) == (1.0, 0.0, 0.0, 0.0, 0.0, 0.0)
        np.testing.assert_allclose([c.hx, c.he, c.vx, c.v0], [dc.hx, dc.he, dc.cx, dc.cd], rtol=1e-15, atol=0)
        assert dc.cp == 0.0


@pytest.mark.parametrize("N", [3, 10, 25])
def test_constant_data_prediction_is_exact(N):
    """With m constant, every corrected sample and every predictor result lies on the exact solution
    alpha_s D + (sigma_s / sigma_T)(x_T - alpha_T D), to float64 rounding."""
    al, sg = _ac64()
    s = _unipc()
    s.set_timesteps(N)
    ts = s.timesteps_host
    rng = np.random.default_rng(3)
    D = rng.standard_normal(64)
    x0 = rng.standard_normal(64)
    T = int(ts[0])
    exact = lambda t: al[t] * D + (sg[t] / sg[T]) * (x0 - al[T] * D)
    x, xl, m1, m2 = x0, 0 * D, 0 * D, 0 * D
    for i in range(len(ts)):
        t = int(ts[i])
        e = (x - al[t] * D) / sg[t]
        xn, m, xc = _apply(s.unipc_coeffs(i), x, e, xl, m1, m2)
        np.testing.assert_allclose(m, D, rtol=1e-12, atol=1e-12)
        np.testing.assert_allclose(xc, exact(t), rtol=1e-12, atol=1e-12)
        s_ = 0 if i == len(ts) - 1 else int(ts[i + 1])
        np.testing.assert_allclose(xn, exact(s_), rtol=1e-12, atol=1e-12)
        x, xl, m1, m2 = xn, xc, m, m1


@pytest.mark.parametrize("N", [2, 5, 10])
def test_corrector_sees_latents_only_through_m(N):
    """For i >= 1, moving x_i while holding m_i fixed leaves x_{i+1} unchanged (ux = 0): the corrector restarts from
    its own last corrected sample. At step 0 (no corrector) the same move does change x_1."""
    al, sg = _ac64()
    s = _unipc()
    s.set_timesteps(N)
    ts = s.timesteps_host
    g = torch.Generator().manual_seed(11)
    xl, m1, m2 = (torch.randn(32, generator=g, dtype=torch.float64) for _ in range(3))
    for i in range(len(ts)):
        c = s.unipc_coeffs(i)
        t = int(ts[i])
        x, e = (torch.randn(32, generator=g, dtype=torch.float64) for _ in range(2))
        delta = torch.randn(32, generator=g, dtype=torch.float64)
        a, _, _ = _apply(c, x, e, xl, m1, m2)
        b, mb, _ = _apply(c, x + delta, e + delta / sg[t], xl, m1, m2)    # same m: delta / alpha - delta / alpha
        torch.testing.assert_close(mb, c.hx * x + c.he * e, rtol=1e-12, atol=1e-12)
        if i == 0:
            assert c.ux == 1.0 and not torch.allclose(a, b)
        else:
            assert c.ux == 0.0
            torch.testing.assert_close(a, b, rtol=1e-12, atol=1e-12)


# ------------------------------------------------------------------------------------------------ CPU: goldens
def _xl_plain_oracle(steps):
    from oracle import sampler_oracle as sam, unet_oracle as uo
    cfg = uo.tiny_xl_config()
    S = mo.LATENT_XL_PLAIN
    unet = sam.make_unet_fn(uo.make_state_dict(cfg, 2), cfg)
    inp = synth.synth_inputs(cfg.cross_attention_dim, _pooled(cfg), 3, S, 31)
    ctx, te = inp["ctx"], inp["text_embeds"]
    added2 = {"text_embeds": torch.cat([te[:1], te[-1:]]), "time_ids": inp["time_ids"].repeat(2, 1)}
    return mo.plain_loop(unet, uo_sched.UniPCSchedulerOracle(), torch.cat([ctx[:1], ctx[-1:]]), inp["latents"].clone(),
                         steps, 8.5, added_cond=added2)


def _xl_rich_oracle(steps, inject_selfattn=0.5, inject_background=0.5, colour=True):
    from oracle import sampler_oracle as sam, unet_oracle as uo
    cfg = uo.tiny_xl_config()
    S = mo.LATENT_XL_RICH
    inp = synth.synth_inputs(cfg.cross_attention_dim, _pooled(cfg), 3, S, 31)
    ctx, te = inp["ctx"], inp["text_embeds"]
    tfd = synth.font_sizes()
    if colour:
        tfd.update(synth.color_dict(inp["masks"], S, 1.0))
    return mo.rich_text_loop(sam.make_unet_fn(uo.make_state_dict(cfg, 2), cfg), uo_sched.UniPCSchedulerOracle(),
                             uo_sched.UniPCSchedulerOracle(), ctx, inp["masks"], inp["latents"].clone(), steps, 8.5,
                             xl=True, added_cond={"text_embeds": te, "time_ids": inp["time_ids"]}, use_guidance=colour,
                             text_format_dict=tfd, inject_selfattn=inject_selfattn, inject_background=inject_background,
                             vae_decode=synth.TinyVAE(), scaling_factor=0.13025)


def _sd_rich_oracle(steps):
    from oracle import sampler_oracle as sam, unet_oracle as uo
    cfg = uo.tiny_sd_config()
    S = mo.LATENT_SD
    inp = synth.synth_inputs(cfg.cross_attention_dim, 0, 3, S, 21)
    tfd = synth.font_sizes()
    tfd.update(synth.color_dict(inp["masks"], S, 0.5))
    return mo.rich_text_loop(sam.make_unet_fn(uo.make_state_dict(cfg, 1), cfg), uo_sched.UniPCSchedulerOracle(),
                             uo_sched.UniPCSchedulerOracle(), inp["ctx"], inp["masks"], inp["latents"].clone(), steps,
                             8.5, xl=False, use_guidance=True, text_format_dict=tfd, inject_selfattn=0.3,
                             inject_background=0.5, vae_decode=synth.TinyVAE(), scaling_factor=0.18215)


def _assert_golden(got, ref, what):
    """test_xl_loops_match_reference's tolerance for the oracle against the reference."""
    np.testing.assert_allclose(np.asarray(got, np.float32), ref, atol=5e-4 * max(1.0, float(np.abs(ref).max()) / 10),
                               rtol=1e-4, err_msg=what)


@pytest.mark.parametrize("steps", [5, 10])
def test_oracle_xl_plain_matches_reference(steps):
    _assert_golden(_xl_plain_oracle(steps).numpy(), _golden()[f"xl_plain_unipc_{steps}"], f"xl plain unipc {steps}")


def test_oracle_xl_rich_matches_reference():
    """inject_selfattn > 0: the reference steps both trajectories jointly on every step, which equals one scheduler
    state per trajectory; colour guidance and background injection move the latents between corrector steps."""
    _assert_golden(_xl_rich_oracle(5).detach().numpy(), _golden()["xl_rich_unipc_5"], "xl rich unipc")


def test_oracle_sd_produce_latents_matches_reference():
    _assert_golden(_sd_rich_oracle(5).detach().numpy(), _golden()["sd_rich_unipc_5"], "sd rich unipc")


# ------------------------------------------------------------------------------------------------ CPU: C ABI, cubin
def test_unipc_abi_rejects_bad_arguments_without_launching():
    from rtti_b200 import _lib
    lib = _lib.load()
    V = ctypes.c_void_p
    buf = (ctypes.c_char * 8192)()
    a = (ctypes.addressof(buf) + 15) // 16 * 16
    regions = (V * 3)(V(a), V(a), V(a))

    def co(ul=0.9, u1=0.2, u2=0.1, v1=0.3):
        return (1.5, -0.5, 0.0, ul, -0.1, u1, u2, 0.8, -0.2, v1)

    for fn, extra in ((lib.rtti_region_blend_cfg_unipc, []), (lib.rtti_region_blend_cfg_rescale_unipc, [0.7])):
        def rb(lat=a, xl=a, m1=a, m2=a, mo_=a, xo=a, n=64, eu=a, regs=regions, N=3, c=None):
            return fn(V(eu), regs, V(a), N, n, 7.5, V(a), V(lat), V(lat), *(c or co()), V(xl), V(m1), V(m2), V(mo_),
                      V(xo), *extra, V(0))
        assert rb(eu=0) == ARG
        assert rb(regs=(V * 3)(V(a), V(0), V(a))) == ARG
        assert rb(N=17) == ARG
        assert rb(lat=0) == ARG                      # the UniPC update needs the latents
        assert rb(mo_=0) == ARG and rb(xo=0) == ARG  # and both outputs
        assert rb(xl=0) == ARG                       # ul != 0 needs xl
        assert rb(m1=0) == ARG                       # u1 or v1 != 0 needs m1
        assert rb(m1=0, c=co(u1=0.0)) == ARG
        assert rb(m1=0, c=co(v1=0.0)) == ARG
        assert rb(m2=0) == ARG                       # u2 != 0 needs m2
        assert rb(n=60) == SHAPE
        assert rb(xl=a + 4) == ALIGN and rb(m1=a + 8) == ALIGN and rb(m2=a + 4) == ALIGN
        assert rb(mo_=a + 4) == ALIGN and rb(xo=a + 8) == ALIGN
    peers = (V * 2)(V(a), V(a))
    owner = (ctypes.c_int * 6)(0, 0, 1, 1, 0, 1)
    for fn, extra in ((lib.rtti_gather_blend_step_unipc, []), (lib.rtti_gather_blend_step_rescale_unipc, [0.7])):
        def gb(world=2, rank=0, n=64, ref=0, lat=a, slots=peers, main=(a,) * 5, refb=(a,) * 5):
            return fn(slots, peers, world, rank, owner, 6, 3, V(a), n, 7.5, V(a), V(lat), V(lat), V(ref), V(ref),
                      *co(), *[V(p) for p in main], *[V(p) for p in refb], 1, *extra, V(0))
        assert gb(world=17) == ARG
        assert gb(rank=2) == ARG
        assert gb(slots=(V * 2)(V(a), V(0))) == ARG
        assert gb(lat=0) == ARG
        assert gb(main=(a, a, a, 0, a)) == ARG
        assert gb(main=(0, a, a, a, a)) == ARG
        assert gb(ref=a, refb=(a, a, a, a, 0)) == ARG     # the reference trajectory needs its own histories
        assert gb(ref=a, refb=(a, 0, a, a, a)) == ARG
        assert gb(n=60) == SHAPE
        assert gb(main=(a, a + 4, a, a, a)) == ALIGN
        assert gb(ref=a, refb=(a, a, a, a + 8, a)) == ALIGN
        assert gb(world=1) == ARG                      # slot owned by rank 1 of a world of 1


def _unipc_sass():
    from rtti_b200 import _lib
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    _lib.load()
    sass = subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True).stdout
    out = {}
    for f in re.split(r"\n\s*Function : ", sass)[1:]:
        name = f.split("\n", 1)[0]
        m = re.search(r"\d(region_blend|gather_blend|blend_rescale)_unipc_kernel(ILb[01]E)?", name)
        if m:
            out[m.group(1) + (m.group(2) or "")] = f
    return out


def test_unipc_kernels_in_the_cubin():
    """Four _unipc kernels; the fp32 histories go through 128-bit loads and stores (loads predicated on their
    coefficients, two 128-bit stores per history written, per trajectory); no 32-bit global stores in the single-GPU
    and rescale kernels; the rescale cluster kernels within 64 registers at 1024 threads, without spills."""
    from rtti_b200 import _lib
    k = _unipc_sass()
    assert sorted(k) == ["blend_rescaleILb0E", "blend_rescaleILb1E", "gather_blend", "region_blend"], sorted(k)
    for name, f in k.items():
        trajectories = 1 if name == "region_blend" else 2
        assert len(re.findall(r"\bLDG\.E\.128\b", f)) >= 6 * trajectories, name
        assert len(re.findall(r"\bSTG\.E\.128\b", f)) >= 4 * trajectories, name
        if name != "gather_blend":   # gather_blend's fp16 latents go through the 32-bit H8 copies of its Euler form
            assert not re.search(r"\bSTG\.E\s", f), f"{name}: 32-bit global stores"
        if name.startswith("blend_rescale"):   # (region_blend's pointer table lives in local memory by design)
            assert not re.search(r"\bSTL", f), f"{name}: local-memory stores (spills)"
    out = subprocess.run(["cuobjdump", "-res-usage", _lib.LIB_PATH], capture_output=True, text=True).stdout
    regs = [int(r) for fn, r in re.findall(r"Function (\S+):\s*\n\s*REG:(\d+)", out) if "blend_rescale_unipc_kernel" in fn]
    assert len(regs) == 2
    for r in regs:
        assert r <= 64 and ((r * 32 + 255) // 256 * 256) * 32 <= 65536, f"{r} registers x 32 warps"


# ------------------------------------------------------------------------------------------------ GPU: accuracy
STEP_KINDS = {"first": 0, "corr1": 1, "corr2": 5, "last": 9}   # of a 10-step grid


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _masks(N, n, g):
    m = torch.rand(N, n, device="cuda", generator=g)
    return (m / m.sum(0, keepdim=True)).half().float().contiguous()


def _blend64(eu, er, m, guidance, phi):
    md = m.double()
    u64 = sum(eu.double() * md[k] for k in range(len(er)))
    t64 = sum(er[k].double() * md[k] for k in range(len(er)))
    e64 = u64 + guidance * (t64 - u64)
    if phi:
        e64 = e64 * (1 - phi + phi * t64.std() / e64.std())
    return e64


def _hist(n, g, scale):
    return [(torch.randn(n, device="cuda", generator=g) * scale).float() for _ in range(3)]   # xl, m1, m2


def _diffusers16(s, i, x16, e16, hist):
    """The fp16 torch expressions diffusers evaluates at step i (the oracle in fp32 tables on fp16 tensors, its state
    set to the fp16-rounded histories): (x', m, xc)."""
    ts = s.timesteps_host
    o = uo_sched.UniPCSchedulerOracle()
    o.set_timesteps(len(ts))
    xl, m1, m2 = (h.half() for h in hist)
    o.model_outputs = [m2, m1]
    o.timestep_list = [int(ts[i - 2]) if i >= 2 else None, int(ts[i - 1]) if i >= 1 else None]
    o.lower_order_nums = min(i, 2)
    o.this_order = s.orders(i)[1] if i > 0 else None
    o.last_sample = xl if i > 0 else None
    out = o.step(e16, int(ts[i]), x16)["prev_sample"]
    return out, o.model_outputs[-1], o.last_sample


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
@pytest.mark.parametrize("step_kind", sorted(STEP_KINDS))
@pytest.mark.parametrize("with_ref", [False, True])
@pytest.mark.parametrize("phi", [0.0, 0.7])
@pytest.mark.parametrize("N", [2, 5, 16])
@pytest.mark.parametrize("n", [16384, 65536, 65528])
@pytest.mark.parametrize("family", ["single", "gather"])
def test_unipc_kernels_vs_fp64(family, n, N, phi, with_ref, step_kind):
    """latents_out, m_out and xl_out of each trajectory against float64 of the fused form on the exact blend; the
    comparator is diffusers' fp16 evaluation on the fp16 prediction and fp16-rounded histories."""
    from rtti_b200 import ops
    from tests.fp64_rule import half_ulp16, no_worse
    i = STEP_KINDS[step_kind]
    s = _unipc()
    s.set_timesteps(10)
    c = s.unipc_coeffs(i)
    g = _gen(n + 13 * N + int(10 * phi) + 7 * with_ref + 3 * i)
    eu = torch.randn(n, device="cuda", generator=g).half()
    er = [torch.randn(n, device="cuda", generator=g).half() for _ in range(N)]
    m = _masks(N, n, g)
    lat = (2 * torch.randn(n, device="cuda", generator=g)).half()
    ec, ed = torch.randn(n, device="cuda", generator=g).half(), torch.randn(n, device="cuda", generator=g).half()
    lat_ref = (2 * torch.randn(n, device="cuda", generator=g)).half()
    hist, hist_ref = _hist(n, g, 2.0), _hist(n, g, 2.0)
    outs, outs_ref = [torch.full((n,), float("nan"), device="cuda") for _ in range(2)], \
        [torch.full((n,), float("nan"), device="cuda") for _ in range(2)]
    guidance = 5.0
    ones = torch.ones(1, n, device="cuda")
    step = ops.UniPCStep(c, *hist, *outs)
    step_ref = ops.UniPCStep(c, *hist_ref, *outs_ref)
    if family == "single":
        e1, x1 = ops.region_blend_cfg(eu, er, m, guidance, latents=lat, guidance_rescale=phi, step=step)
        xr = ops.region_blend_cfg(ec, [ed], ones, guidance, latents=lat_ref, guidance_rescale=phi,
                                  step=step_ref)[1] if with_ref else None
    else:
        e1, x1, xr = _gather_world1(eu, er, m, guidance, lat, (ec, ed, lat_ref if with_ref else None), phi,
                                    ops.UniPCStep(c, *hist, *outs, ref=(*hist_ref, *outs_ref)))
    e_euler, _ = ops.region_blend_cfg(eu, er, m, guidance, latents=lat, dt_sigma=-0.3, guidance_rescale=phi)
    assert torch.equal(e1, e_euler), "eps_out differs from the Euler entry point's"
    tag = f"unipc {family} n{n} N{N} phi{phi:g} {step_kind}"
    trajectories = [(e1, x1, lat, hist, outs, _blend64(eu, er, m, guidance, phi), "latents")]
    if with_ref:
        e_ref16 = ops.region_blend_cfg(ec, [ed], ones, guidance, guidance_rescale=phi)
        trajectories.append((e_ref16, xr, lat_ref, hist_ref, outs_ref, _blend64(ec, [ed], ones, guidance, phi),
                             "latents_ref"))
    for e16, got, x, (xl, m1, m2), (m_out, xl_out), e64, what in trajectories:
        x64 = x.double()
        m64 = c.hx * x64 + c.he * e64
        xc64 = c.ux * x64 + c.ul * xl.double() + c.u0 * m64 + c.u1 * m1.double() + c.u2 * m2.double()
        want64 = c.vx * xc64 + c.v0 * m64 + c.v1 * m1.double()
        x16, mm16, xc16 = _diffusers16(s, i, x, e16, (xl, m1, m2))
        no_worse(f"{tag} {what}", got, x16, want64, k=2.0, floor=half_ulp16(want64), mean=True)
        no_worse(f"{tag} {what} m_out", m_out, mm16, m64, k=2.0, floor=half_ulp16(m64), mean=True)
        no_worse(f"{tag} {what} xl_out", xl_out, xc16, xc64, k=2.0, floor=half_ulp16(xc64), mean=True)


# ------------------------------------------------------------------------------------------------ GPU: bit-identities
@pytest.mark.gpu
@pytest.mark.parametrize("phi", [0.0, 0.7])
@pytest.mark.parametrize("n,N", [(16384, 5), (65528, 2), (65536, 16)])
def test_unipc_bit_identities(n, N, phi):
    """The gather form at world 1 equals the single-GPU form (both trajectories, all outputs); m_out aliasing m2 and
    xl_out aliasing xl equal separate buffers; unread histories may be null; a CUDA-graph replay equals eager."""
    from rtti_b200 import ops
    s = _unipc()
    s.set_timesteps(10)
    c = s.unipc_coeffs(5)
    assert all(v != 0.0 for v in (c.ul, c.u1, c.u2, c.v1))
    g = _gen(n + N)
    eu = torch.randn(n, device="cuda", generator=g).half()
    er = [torch.randn(n, device="cuda", generator=g).half() for _ in range(N)]
    m = _masks(N, n, g)
    lat = (2 * torch.randn(n, device="cuda", generator=g)).half()
    ec, ed = torch.randn(n, device="cuda", generator=g).half(), torch.randn(n, device="cuda", generator=g).half()
    lat_ref = (2 * torch.randn(n, device="cuda", generator=g)).half()
    hist, hist_ref = _hist(n, g, 1.5), _hist(n, g, 1.5)
    ones = torch.ones(1, n, device="cuda")
    guidance = 8.5

    def single():
        o, orf = [torch.empty(n, device="cuda") for _ in range(2)], [torch.empty(n, device="cuda") for _ in range(2)]
        eps, lo = ops.region_blend_cfg(eu, er, m, guidance, latents=lat, guidance_rescale=phi,
                                       step=ops.UniPCStep(c, *hist, *o))
        _, ro = ops.region_blend_cfg(ec, [ed], ones, guidance, latents=lat_ref, guidance_rescale=phi,
                                     step=ops.UniPCStep(c, *hist_ref, *orf))
        return eps, lo, ro, *o, *orf

    a = single()
    b = single()
    for x, y in zip(a, b):
        assert torch.equal(x, y), "two calls differ"
    o, orf = [torch.empty(n, device="cuda") for _ in range(2)], [torch.empty(n, device="cuda") for _ in range(2)]
    gw = _gather_world1(eu, er, m, guidance, lat, (ec, ed, lat_ref), phi,
                        ops.UniPCStep(c, *hist, *o, ref=(*hist_ref, *orf)))
    for x, y, what in zip(a, (*gw, *o, *orf), ("eps", "latents", "latents_ref", "m_out", "xl_out", "m_out_ref",
                                               "xl_out_ref")):
        assert torch.equal(x, y), f"gather world 1 vs single GPU: {what} differs"
    # aliasing, as the samplers run it: m written over m2, xc over xl
    h = ops.UniPCHistory(n, "cuda")
    hr = ops.UniPCHistory(n, "cuda")
    for dst, src in ((h, hist), (hr, hist_ref)):
        dst.xl.copy_(src[0]); dst.m1.copy_(src[1]); dst.m2.copy_(src[2])
    _, lo2 = ops.region_blend_cfg(eu, er, m, guidance, latents=lat, guidance_rescale=phi, step=ops.UniPCStep.of(c, h))
    assert torch.equal(lo2, a[1]) and torch.equal(h.m2, a[3]) and torch.equal(h.xl, a[4]), "aliased buffers differ"
    h.rotate()
    assert torch.equal(h.m1, a[3]) and torch.equal(h.m2, hist[1])
    for dst, src in ((h, hist),):
        dst.xl.copy_(src[0]); dst.m1.copy_(src[1]); dst.m2.copy_(src[2])
    _, lo3, ro3 = _gather_world1(eu, er, m, guidance, lat, (ec, ed, lat_ref), phi, ops.UniPCStep.of(c, h, hr))
    assert torch.equal(lo3, a[1]) and torch.equal(ro3, a[2]) and torch.equal(h.xl, a[4]) and torch.equal(hr.xl, a[6])
    # first step: no history is read, so none is needed
    s0 = s.unipc_coeffs(0)
    o0 = [torch.empty(n, device="cuda") for _ in range(2)]
    _, l0 = ops.region_blend_cfg(eu, er, m, guidance, latents=lat, guidance_rescale=phi,
                                 step=ops.UniPCStep(s0, None, None, None, *o0))
    o1 = [torch.empty(n, device="cuda") for _ in range(2)]
    _, l1 = ops.region_blend_cfg(eu, er, m, guidance, latents=lat, guidance_rescale=phi,
                                 step=ops.UniPCStep(s0, *[torch.full((n,), float("nan"), device="cuda")] * 3, *o1))
    assert torch.equal(l0, l1) and torch.equal(o0[0], o1[0]) and torch.equal(o0[1], o1[1])
    assert torch.equal(o0[1], lat.float()), "step 0: the corrected sample is the latents"
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


def _sched(kind):
    from rtti_b200 import schedulers as S
    return {"unipc": S.UniPCMultistepScheduler, "dpmpp_2m": S.DPMSolverMultistepScheduler,
            "plms": S.PNDMScheduler}[kind]()


def _xl_model(kind):
    from oracle import unet_oracle as uo
    from rtti_b200.region_diffusion_sdxl import RegionDiffusionXL
    from rtti_b200.unet import UNet2DConditionModel, UNetConfig
    cfg = uo.tiny_xl_config()
    unet = UNet2DConditionModel(UNetConfig.from_dict(cfg.__dict__))
    unet.load_state_dict(uo.make_state_dict(cfg, 2))
    return cfg, RegionDiffusionXL(device="cuda", unet=unet.finalize("cuda"), vae=synth.TinyVAE("cuda"),
                                  scheduler=_sched(kind))


def _xl_plain(kind, steps):
    cfg, m = _xl_model(kind)
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
@pytest.mark.parametrize("steps", [5, 10])
def test_xl_plain_vs_reference_golden(steps):
    """Against the reference's plain pass; the DPM-Solver++(2M) run of the same inputs lies outside the tolerance."""
    out = _xl_plain("unipc", steps)
    _close_range(out, _golden()[f"xl_plain_unipc_{steps}"], f"xl plain unipc {steps}")
    with pytest.raises(AssertionError):
        _close_range(out, _xl_plain("dpmpp_2m", steps), "xl plain unipc vs dpm")


@pytest.mark.gpu
def test_xl_rich_vs_reference_golden():
    """Injection (0.5 / 0.5), font sizes and colour guidance, against the reference's loop; the DPM run of the same
    inputs lies outside the tolerance; CUDA-graph replayed UNet passes give the same bits as eager ones."""
    out = _xl_rich("unipc", 5)
    _close_range(out, _golden()["xl_rich_unipc_5"], "xl rich unipc")
    with pytest.raises(AssertionError):
        _close_range(out, _xl_rich("dpmpp_2m", 5), "xl rich unipc vs dpm")
    assert np.array_equal(out, _xl_rich("unipc", 5, graphs=False)), "use_cuda_graphs on / off differ"


@pytest.mark.gpu
@pytest.mark.parametrize("inject_selfattn", [0.0, 0.5])
def test_xl_rich_separate_states_vs_oracle(inject_selfattn):
    """inject_background = 0.5: with inject_selfattn = 0 the reference latents are stepped on the first half of the
    steps only, and each trajectory keeps its own UniPC state (the reference would carry a batch-2 state into batch-1
    steps). Against the oracle with one scheduler state per trajectory, 6 steps: order-2 corrector steps on both sides
    of the switch."""
    out = _xl_rich("unipc", 6, inject_selfattn=inject_selfattn, inject_background=0.5, colour=False)
    ref = _xl_rich_oracle(6, inject_selfattn=inject_selfattn, inject_background=0.5, colour=False)
    _close_range(out, ref.numpy(), f"xl rich unipc, inject {inject_selfattn} / 0.5, vs oracle")


def _sd_model(kind):
    from oracle import unet_oracle as uo
    from rtti_b200.region_diffusion import RegionDiffusion
    from rtti_b200.unet import UNet2DConditionModel, UNetConfig
    cfg = uo.tiny_sd_config()
    unet = UNet2DConditionModel(UNetConfig.from_dict(cfg.__dict__))
    unet.load_state_dict(uo.make_state_dict(cfg, 1))
    m = RegionDiffusion(device="cuda", unet=unet.finalize("cuda"), vae=synth.TinyVAE("cuda"))
    m.scheduler = _sched(kind)
    return cfg, m


def _sd_rich(kind):
    cfg, m = _sd_model(kind)
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
    out = _sd_rich("unipc")
    _close_range(out, _golden()["sd_rich_unipc_5"], "sd produce_latents unipc")
    with pytest.raises(AssertionError):
        _close_range(out, _sd_rich("plms"), "sd unipc vs PLMS")


@pytest.mark.gpu
def test_sd_produce_attn_maps_vs_oracle():
    """produce_attn_maps (the plain CFG loop of the SD1.5 sampler) with UniPC against the oracle's plain loop."""
    from oracle import sampler_oracle as sam, unet_oracle as uo
    cfg, m = _sd_model("unipc")
    S = mo.LATENT_SD
    inp = synth.synth_inputs(cfg.cross_attention_dim, 0, 3, S, 21)
    ctx = torch.cat([inp["ctx"][:1], inp["ctx"][-1:]])
    out = m.produce_attn_maps(None, height=S * 8, width=S * 8, num_inference_steps=6, guidance_scale=7.5,
                              latents=inp["latents"].clone(), text_embeddings=ctx.cuda(), decode=False)
    ref = mo.plain_loop(sam.make_unet_fn(uo.make_state_dict(cfg, 1), cfg), uo_sched.UniPCSchedulerOracle(), ctx,
                        inp["latents"].clone(), 6, 7.5)
    _close_range(out.float().cpu().numpy(), ref.numpy(), "sd produce_attn_maps unipc vs oracle")


@pytest.mark.gpu
def test_unsupported_scheduler_message_names_unipc():
    from rtti_b200.schedulers import PNDMScheduler
    cfg, m = _xl_model("unipc")
    m.scheduler = PNDMScheduler()
    with pytest.raises(TypeError, match="DPMSolverMultistepScheduler.*UniPCMultistepScheduler"):
        m.sample(height=256, width=256, num_inference_steps=2, prompt_embeds=torch.zeros(1, 77, 8, device="cuda"),
                 negative_prompt_embeds=torch.zeros(1, 77, 8, device="cuda"), pooled_prompt_embeds=None,
                 negative_pooled_prompt_embeds=None, output_type="latent")


@pytest.mark.gpu
def test_rich_loop_unipc_two_gpus():
    """UniPC on the fused peer-memory exchange and on the NCCL path (tests/multigpu_unipc_check.py)."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
                        "--master-addr", "127.0.0.1", "--master-port", "29541",
                        os.path.join(ROOT, "tests", "multigpu_unipc_check.py")],
                       capture_output=True, text=True, timeout=900)
    print(r.stdout[-2000:], r.stderr[-2000:])
    assert r.returncode == 0 and "MULTIGPU_UNIPC_CHECK PASS" in r.stdout
