"""k-LMS in RegionDiffusionXL, with the four-term linear multistep update fused into the blend kernels
(rtti_region_blend_cfg_lms, rtti_region_blend_cfg_rescale_lms, rtti_gather_blend_step_lms,
rtti_gather_blend_step_rescale_lms).

CPU: the grid, the configuration, the coefficients against scipy's quadrature and the diffusers-form oracle
(tests/lms_oracle.py), the order ramp, the convergence order on the Gaussian-data ODE of tests/test_heun_sampling.py,
the oracle loops against the unmodified reference (tests/golden/lms.npz, tests/gen_lms.py), the C-ABI argument checks
and the cubin. GPU: the kernels against float64 (tests/fp64_rule.py, K = 2, mean check on; the comparator is the fp16
torch expression diffusers evaluates), bit-identities, the sampler against the goldens and their callback iterations,
and the two-GPU exchanges (tests/multigpu_lms_check.py)."""
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

from tests import lms_oracle as lo
from tests import multistep_oracle as mo
from tests import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
ARG, SHAPE, ALIGN = -1, -2, -3


def _golden():
    return np.load(os.path.join(GOLDEN, "lms.npz"), allow_pickle=False)


def _lms(**kw):
    from rtti_b200.schedulers import LMSDiscreteScheduler
    return LMSDiscreteScheduler(**kw)


def _pooled(cfg):
    return cfg.projection_class_embeddings_input_dim - 6 * cfg.addition_time_embed_dim


# ------------------------------------------------------------------------------------------------ CPU: scheduler
@pytest.mark.parametrize("N", [10, 20, 41, 50])
def test_grid_is_eulers(N):
    from rtti_b200.schedulers import EulerDiscreteScheduler
    s, e = _lms(), EulerDiscreteScheduler()
    s.set_timesteps(N)
    e.set_timesteps(N)
    assert s.order == 1 and s.num_inference_steps == N
    assert s.timesteps.tolist() == e.timesteps.tolist()
    assert np.array_equal(s.sigmas_host, e.sigmas_host) and s.sigmas_host.dtype == np.float32 and s.sigmas_host[-1] == 0
    assert s.init_noise_sigma == e.init_noise_sigma and torch.equal(s.alphas_cumprod, e.alphas_cumprod)
    x = torch.randn(2, 4, 8, 8, generator=torch.Generator().manual_seed(N))
    for t in s.timesteps:
        assert s.sigma(t) == e.sigma(t)
        assert torch.equal(s.scale_model_input(x, t), e.scale_model_input(x, t))
        assert torch.equal(s.scale_model_input(x, t), x / math.sqrt(s.sigma(t) ** 2 + 1))


def test_config_and_dispatch():
    from rtti_b200 import schedulers as S
    from rtti_b200.region_diffusion_sdxl import _step_kind
    s = _lms()
    assert not isinstance(s, S.EulerDiscreteScheduler), "an Euler subclass would be stepped as Euler"
    assert _step_kind(s) == "lms"
    for src in (S.EulerDiscreteScheduler(), S.EulerAncestralDiscreteScheduler(), S.HeunDiscreteScheduler()):
        assert isinstance(S.LMSDiscreteScheduler.from_config(src), S.LMSDiscreteScheduler)
    assert S.LMSDiscreteScheduler.from_config(dict(s.config)).config == s.config
    for cfg in (S.DPMSolverMultistepScheduler().config, S.UniPCMultistepScheduler().config):
        with pytest.raises(NotImplementedError):   # the linspace grid is not this scheduler's
            S.LMSDiscreteScheduler.from_config(cfg)
    for kw in (dict(use_karras_sigmas=True), dict(timestep_spacing="trailing"), dict(timestep_spacing="linspace"),
               dict(prediction_type="v_prediction"), dict(trained_betas=[0.1] * 1000), dict(beta_schedule="linear")):
        with pytest.raises(NotImplementedError):
            _lms(**kw)
    with pytest.raises(TypeError):
        _lms(solver_order=2)
    with pytest.raises(TypeError, match="HeunDiscreteScheduler, LMSDiscreteScheduler"):
        _step_kind(S.PNDMScheduler())


def _quad64(sig, i, p, k):
    """c_k by scipy's quadrature of the float64 Lagrange basis."""
    from scipy import integrate
    nodes = [float(sig[i - j]) for j in range(p)]

    def basis(tau):
        out = 1.0
        for j in range(p):
            if j != k:
                out *= (tau - nodes[j]) / (nodes[k] - nodes[j])
        return out
    return integrate.quad(basis, float(sig[i]), float(sig[i + 1]), epsrel=1e-4)[0]


@pytest.mark.parametrize("N", [1, 2, 4, 10, 41])
def test_coefficients_match_quadrature(N):
    """lms_coeffs(i) against quad of the float64 basis (1e-9 relative) and against the oracle's quad of diffusers'
    float32 integrand (1e-5); the order ramps 1, 2, 3, 4, 4, ...; the unused coefficients are 0; sum c_k equals
    sigma_{i+1} - sigma_i."""
    s, o = _lms(), lo.LMSSchedulerOracle()
    s.set_timesteps(N)
    o.set_timesteps(N)
    assert torch.equal(o.sigmas, torch.from_numpy(s.sigmas_host))
    sig = s.sigmas_host
    w64 = w32 = 0.0
    for i in range(N):
        c = s.lms_coeffs(i)
        p = min(i + 1, 4)
        assert len(c) == 4 and all(x == 0.0 for x in c[p:]) and all(x != 0.0 for x in c[:p]), (i, c)
        for k in range(p):
            q64, q32 = _quad64(sig, i, p, k), o.get_lms_coefficient(p, i, k)
            w64 = max(w64, abs(c[k] - q64) / abs(q64))
            w32 = max(w32, abs(c[k] - q32) / abs(q32))
        dt = float(sig[i + 1]) - float(sig[i])
        assert abs(sum(c) - dt) <= 1e-11 * max(abs(x) for x in c), (i, sum(c), dt)   # up to cancellation
    print(f"N={N}: max relative difference to quad (float64 basis) {w64:.2e}, to quad (float32 integrand) {w32:.2e}")
    assert w64 <= 1e-9 and w32 <= 1e-5, (w64, w32)
    if N >= 5:
        assert [sum(x != 0.0 for x in s.lms_coeffs(i)) for i in range(5)] == [1, 2, 3, 4, 4]
    assert s.lms_coeffs(0) == (float(sig[1]) - float(sig[0]), 0.0, 0.0, 0.0)


def test_torch_step_matches_coefficients_and_oracle():
    """step() against the float64 affine form of lms_coeffs over the last four predictions, and against the
    diffusers-form oracle; set_timesteps clears the history."""
    s, o = _lms(), lo.LMSSchedulerOracle()
    for N in (3, 10):
        s.set_timesteps(N)
        o.set_timesteps(N)
        assert s.derivatives == []
        g = torch.Generator().manual_seed(N)
        x = torch.randn(2, 4, 8, 8, generator=g) * 8
        xo, x64, hist = x.clone(), x.double(), []
        for i, t in enumerate(s.timesteps):
            e = torch.randn(2, 4, 8, 8, generator=g)
            hist = [e.double()] + hist[:3]
            want = x64 + sum(c * d for c, d in zip(s.lms_coeffs(i), hist))
            got = s.step(e, t, x)["prev_sample"]
            torch.testing.assert_close(got.double(), want, rtol=1e-6, atol=1e-6 * float(want.abs().max()))
            ref = o.step(e, t, xo)["prev_sample"]
            torch.testing.assert_close(got, ref, rtol=1e-5, atol=1e-5 * float(ref.abs().max()))
            x, xo, x64 = got, ref, want


def _ode_error_lms(N, var=0.25, x0=1.3, t_from=801, t_to=201):
    """tests/test_heun_sampling.py's Gaussian-data ODE (eps(x, sigma) = x sigma / (var + sigma^2), exact solution
    x(sigma') = x(sigma) sqrt((var + sigma'^2) / (var + sigma^2))) integrated by LMS from t_from to t_to, with the order
    ramp restarted at t_from: the coefficients of step j are those lms_coeffs gives on the grid shifted to start there."""
    from rtti_b200.schedulers import EulerDiscreteScheduler
    e = EulerDiscreteScheduler()
    e.set_timesteps(N)
    j0, j1 = (int(np.nonzero(e.timesteps_host == t)[0][0]) for t in (t_from, t_to))
    s = _lms()
    s.set_timesteps(N)
    s.sigmas_host = s.sigmas_host[j0:]
    eps = lambda x, sg: x * sg / (var + sg * sg)
    s0, s1 = float(e.sigmas_host[j0]), float(e.sigmas_host[j1])
    exact = x0 * math.sqrt((var + s1 * s1) / (var + s0 * s0))
    x, hist = x0, []
    for i in range(j1 - j0):
        hist = [eps(x, float(s.sigmas_host[i]))] + hist[:3]
        x = x + sum(c * d for c, d in zip(s.lms_coeffs(i), hist))
    return x - exact


def test_convergence_order():
    """Per doubling of N the LMS error falls by more than 3.5x, and it is below Euler's at every N."""
    from tests.test_heun_sampling import _ode_error
    Ns = (5, 10, 20, 40)
    lms = [_ode_error_lms(N) for N in Ns]
    euler = [_ode_error(N, False) for N in Ns]
    ratios = [lms[k] / lms[k + 1] for k in range(len(Ns) - 1)]
    print("LMS errors", ["%.2e" % v for v in lms], "ratios", [round(r, 2) for r in ratios],
          "Euler errors", ["%.2e" % v for v in euler])
    assert all(abs(a) < abs(b) for a, b in zip(lms, euler)), (lms, euler)
    assert min(ratios) > 3.5, ratios


# ------------------------------------------------------------------------------------------------ CPU: goldens
def _xl_plain_oracle(steps):
    from oracle import sampler_oracle as sam, unet_oracle as uo
    cfg = uo.tiny_xl_config()
    S = mo.LATENT_XL_PLAIN
    unet = sam.make_unet_fn(uo.make_state_dict(cfg, 2), cfg)
    inp = synth.synth_inputs(cfg.cross_attention_dim, _pooled(cfg), 3, S, 31)
    ctx, te = inp["ctx"], inp["text_embeds"]
    added2 = {"text_embeds": torch.cat([te[:1], te[-1:]]), "time_ids": inp["time_ids"].repeat(2, 1)}
    return lo.plain_loop(unet, lo.LMSSchedulerOracle(), torch.cat([ctx[:1], ctx[-1:]]), inp["latents"].clone(), steps,
                         8.5, added_cond=added2)


def _xl_rich_oracle(inject_selfattn, inject_background, sched):
    from oracle import sampler_oracle as sam, unet_oracle as uo
    cfg = uo.tiny_xl_config()
    S = mo.LATENT_XL_RICH
    inp = synth.synth_inputs(cfg.cross_attention_dim, _pooled(cfg), 3, S, 31)
    ctx, te = inp["ctx"], inp["text_embeds"]
    tfd = synth.font_sizes()
    tfd.update(synth.color_dict(inp["masks"], S, 1.0))
    return lo.rich_text_loop(sam.make_unet_fn(uo.make_state_dict(cfg, 2), cfg), sched, ctx, inp["masks"],
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
    assert _golden()[f"xl_plain_{steps}_callbacks"].tolist() == list(range(steps))


@pytest.mark.parametrize("sa,bg", [(0.5, 0.5), (0.0, 0.0)])
def test_oracle_xl_rich_matches_reference(sa, bg):
    """The reference latents stepped jointly on every step (0.5 / 0.5), and no reference latents (0 / 0)."""
    sched = lo.LMSSchedulerOracle()
    got = _xl_rich_oracle(sa, bg, sched)
    assert sched.step_batches == [2 if sa > 0 else 1] * 4
    _assert_golden(got.detach().numpy(), _golden()[f"xl_rich_{sa:g}_{bg:g}"], f"xl rich {sa} {bg}")
    assert _golden()[f"xl_rich_{sa:g}_{bg:g}_callbacks"].tolist() == [0, 1, 2, 3]


# ------------------------------------------------------------------------------------------------ CPU: C ABI, cubin
def test_lms_abi_rejects_bad_arguments_without_launching():
    """Every call below fails its argument checks; a launch without a device would return RTTI_ERR_CUDA instead."""
    from rtti_b200 import _lib
    lib = _lib.load()
    V = ctypes.c_void_p
    buf = (ctypes.c_char * 8192)()
    a = (ctypes.addressof(buf) + 15) // 16 * 16
    regions = (V * 3)(V(a), V(a), V(a))
    full = (-0.3, 0.2, -0.1, 0.05)
    for fn, extra in ((lib.rtti_region_blend_cfg_lms, []), (lib.rtti_region_blend_cfg_rescale_lms, [0.7])):
        rb = lambda lat=a, d=(a, a, a), n=64, c=full, eu=a, regs=regions, N=3: fn(
            V(eu), regs, V(a), N, n, 7.5, V(a), V(lat), V(lat), *c, *[V(x) for x in d], *extra, V(0))
        assert rb(eu=0) == ARG
        assert rb(regs=(V * 3)(V(a), V(0), V(a))) == ARG
        assert rb(N=17) == ARG
        assert rb(lat=0) == ARG                  # the LMS update needs the latents
        for k in range(3):                       # c_k != 0 needs d_k
            assert rb(d=tuple(0 if j == k else a for j in range(3))) == ARG
        assert rb(d=(a, 0, 0), c=(-0.3, 0.2, 0.0, 0.0), n=60) == SHAPE   # null d2, d3 pass under c2 = c3 = 0
        assert rb(n=60) == SHAPE
        assert rb(d=(a, a, a + 2)) == ALIGN
        assert rb(d=(a + 8, 0, 0), c=(-0.3, 0.0, 0.0, 0.0)) == ALIGN   # a pointer that is given must be aligned
    peers = (V * 2)(V(a), V(a))
    owner = (ctypes.c_int * 6)(0, 0, 1, 1, 0, 1)
    for fn, extra in ((lib.rtti_gather_blend_step_lms, []), (lib.rtti_gather_blend_step_rescale_lms, [0.7])):
        gb = lambda world=2, rank=0, n=64, ref=0, d=(a, a, a), dr=(a, a, a), er=0, lat=a, slots=peers: fn(
            slots, peers, world, rank, owner, 6, 3, V(a), n, 7.5, V(a), V(lat), V(lat), V(ref), V(ref), *full,
            *[V(x) for x in d], *[V(x) for x in dr], V(er), 1, *extra, V(0))
        assert gb(world=17) == ARG
        assert gb(rank=2) == ARG
        assert gb(slots=(V * 2)(V(a), V(0))) == ARG
        assert gb(lat=0) == ARG
        assert gb(d=(a, a, 0)) == ARG
        assert gb(ref=a, dr=(0, a, a)) == ARG    # the reference trajectory needs its own history
        assert gb(ref=a, dr=(a, 0, a)) == ARG
        assert gb(er=a) == ARG                   # eps_ref_out without the reference latents
        assert gb(n=60) == SHAPE
        assert gb(d=(a + 4, a, a)) == ALIGN
        assert gb(ref=a, dr=(a, a, a + 4)) == ALIGN
        assert gb(ref=a, er=a + 8) == ALIGN
        assert gb(world=1) == ARG                # slot owned by rank 1 of a world of 1


def test_lms_step_python_checks():
    from rtti_b200 import _lib, ops
    x = torch.zeros(64, dtype=torch.float16)
    ops.LMSStep((-0.3, 0.0, 0.0, 0.0), None, None, None)._check(64, False)   # the first step reads no history
    ops.LMSStep((-0.3, 0.0, 0.0, 0.0), None, None, None)._check(64, True)
    for k in range(3):
        c = [-0.3, 0.0, 0.0, 0.0]
        c[k + 1] = 0.1
        with pytest.raises(_lib.RttiError, match=f"d{k + 1} is required"):
            ops.LMSStep(c, None, None, None)._check(64, False)
    with pytest.raises(_lib.RttiError, match="must be a CUDA tensor"):
        ops.LMSStep((-0.3, 0.2, 0.0, 0.0), x, None, None)._check(64, False)
    with pytest.raises(_lib.RttiError, match="eps_ref_out needs the reference latents"):
        ops.LMSStep((-0.3, 0.0, 0.0, 0.0), None, None, None, eps_ref_out=x)._check(64, False)
    with pytest.raises(_lib.RttiError, match=r"\(c0, c1, c2, c3\)"):
        ops.LMSStep((-0.3, 0.2, 0.0), None, None, None)
    big = torch.zeros(128, dtype=torch.float16)
    assert ops._overlap(big[:64], big[32:96]) and not ops._overlap(big[:64], big[64:])


def _sass_by_kernel():
    from rtti_b200 import _lib
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    _lib.load()
    sass = subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True).stdout
    out = {}
    for f in re.split(r"\n\s*Function : ", sass)[1:]:
        name = f.split("\n", 1)[0]
        m = re.search(r"\d(region_blend|gather_blend|blend_rescale)(_lms)?_kernel(ILb[01]E)?", name)
        if m:
            out[(m.group(1), m.group(3) or "", bool(m.group(2)))] = (name, f)
    return out


def test_lms_kernels_in_the_cubin():
    """Each of the four families has its _lms kernel, whose 128-bit loads are those of its Euler kernel plus d1, d2 and
    d3 (for each trajectory it steps); the rescale cluster kernels stay within 64 registers at 1024 threads, no spills."""
    from rtti_b200 import _lib
    k = _sass_by_kernel()
    fams = [("region_blend", "", 3), ("gather_blend", "", 6), ("blend_rescale", "ILb0E", 6), ("blend_rescale", "ILb1E", 6)]
    for fam, tpl, extra in fams:
        assert (fam, tpl, True) in k and (fam, tpl, False) in k, (fam, tpl, sorted(k))
        ld = {h: len(re.findall(r"\bLDG\.E\.128\b", k[(fam, tpl, h)][1])) for h in (False, True)}
        assert ld[True] >= ld[False] + extra, (fam, tpl, ld)
        if fam == "blend_rescale":
            assert not re.search(r"\bSTL", k[(fam, tpl, True)][1]), f"{fam}{tpl}: local-memory stores (spills)"
    out = subprocess.run(["cuobjdump", "-res-usage", _lib.LIB_PATH], capture_output=True, text=True).stdout
    regs = [int(r) for fn, r in re.findall(r"Function (\S+):\s*\n\s*REG:(\d+)", out) if "blend_rescale_lms_kernel" in fn]
    assert len(regs) == 2
    for r in regs:
        assert r <= 64 and ((r * 32 + 255) // 256 * 256) * 32 <= 65536, f"{r} registers x 32 warps"


# ------------------------------------------------------------------------------------------------ GPU: accuracy
def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _masks(N, n, g):
    m = torch.rand(N, n, device="cuda", generator=g)
    return (m / m.sum(0, keepdim=True)).half().float().contiguous()


def _coeffs(p):
    """lms_coeffs of a 20-step grid at order p: the first three steps, and a step of order 4."""
    s = _lms()
    s.set_timesteps(20)
    c = s.lms_coeffs({1: 0, 2: 1, 3: 2, 4: 12}[p])
    assert sum(x != 0.0 for x in c) == p
    return c


def _hist(h, c):
    """The history a caller passes: d_k where c_k != 0, None elsewhere."""
    return tuple(d if ck != 0.0 else None for d, ck in zip(h, c[1:]))


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
    h, h_ref = (rn(), rn(), rn()), (rn(), rn(), rn())
    return eu, er, m, lat, ec, ed, lat_ref, h, h_ref


def _blend64(eu, er, m, guidance, phi):
    md = m.double()
    u64 = sum(eu.double() * md[k] for k in range(len(er)))
    t64 = sum(er[k].double() * md[k] for k in range(len(er)))
    e64 = u64 + guidance * (t64 - u64)
    if phi:
        e64 = e64 * (1 - phi + phi * t64.std() / e64.std())
    return e64


@pytest.mark.gpu
@pytest.mark.parametrize("p", [1, 2, 3, 4])
@pytest.mark.parametrize("with_ref", [False, True])
@pytest.mark.parametrize("phi", [0.0, 0.7])
@pytest.mark.parametrize("N", [2, 5, 16])
@pytest.mark.parametrize("n", [16384, 65536, 65528])
@pytest.mark.parametrize("family", ["single", "gather"])
def test_lms_kernels_vs_fp64(family, n, N, phi, with_ref, p):
    """latents_out (and the reference latents with C/D) against float64 of x + c0 eps + c1 d1 + c2 d2 + c3 d3 on the
    exact blend, with d1..d3 the fp16 histories, at orders 1 to 4."""
    from rtti_b200 import ops
    from tests.fp64_rule import half_ulp16, no_worse
    c = _coeffs(p)
    eu, er, m, lat, ec, ed, lat_ref, h, h_ref = _inputs(n, N, n + 13 * N + int(10 * phi) + 7 * with_ref + 101 * p)
    guidance = 5.0
    ones = torch.ones(1, n, device="cuda")
    hm, hr = _hist(h, c), _hist(h_ref, c)
    if family == "single":
        e1, x1 = ops.region_blend_cfg(eu, er, m, guidance, latents=lat, guidance_rescale=phi, step=ops.LMSStep(c, *hm))
        xr = ops.region_blend_cfg(ec, [ed], ones, guidance, latents=lat_ref, guidance_rescale=phi,
                                  step=ops.LMSStep(c, *hr))[1] if with_ref else None
    else:
        step = ops.LMSStep(c, *hm, *(hr if with_ref else (None,) * 3))
        e1, x1, xr = _gather_world1(eu, er, m, guidance, lat, (ec, ed, lat_ref if with_ref else None), phi, step)
    tag = f"lms {family} n{n} N{N} phi{phi:g} p{p}"
    trajectories = [(e1, x1, lat, h, _blend64(eu, er, m, guidance, phi), "latents")]
    if with_ref:
        e_ref16 = ops.region_blend_cfg(ec, [ed], ones, guidance, guidance_rescale=phi)   # the fp16 prediction stepped
        trajectories.append((e_ref16, xr, lat_ref, h_ref, _blend64(ec, [ed], ones, guidance, phi), "latents_ref"))
    for e16, got, x, hist, e64, what in trajectories:
        want64 = x.double() + c[0] * e64
        cmp16 = x + c[0] * e16   # diffusers in fp16: sample + sum(coeff * derivative)
        for ck, d in zip(c[1:], hist):
            if ck != 0.0:
                want64 = want64 + ck * d.double()
                cmp16 = cmp16 + ck * d
        no_worse(f"{tag} {what}", got, cmp16, want64, k=2.0, floor=half_ulp16(want64), mean=True)


# ------------------------------------------------------------------------------------------------ GPU: bit-identities
@pytest.mark.gpu
@pytest.mark.parametrize("phi", [0.0, 0.7])
@pytest.mark.parametrize("n,N", [(16384, 5), (65528, 2), (65536, 16)])
def test_lms_bit_identities(n, N, phi):
    """Order 1 equals the Euler entry point with dt_sigma = c0 (all four families, eps and latents), with null
    histories; histories under zero coefficients are not read; eps_ref_out equals the eps the single form computes for
    passes C/D; the gather form at world 1 equals the single form at order 4 (both trajectories); a CUDA-graph replay
    equals eager."""
    from rtti_b200 import ops
    eu, er, m, lat, ec, ed, lat_ref, h, h_ref = _inputs(n, N, n + N + 1)
    ones = torch.ones(1, n, device="cuda")
    guidance = 8.5
    c1 = _coeffs(1)
    e_eu, x_eu = ops.region_blend_cfg(eu, er, m, guidance, latents=lat, dt_sigma=c1[0], guidance_rescale=phi)
    e_l, x_l = ops.region_blend_cfg(eu, er, m, guidance, latents=lat, guidance_rescale=phi,
                                    step=ops.LMSStep(c1, None, None, None))
    assert torch.equal(e_eu, e_l) and torch.equal(x_eu, x_l), "order 1 differs from the Euler form (single GPU)"
    nan = torch.full_like(lat, float("nan"))
    _, x_nan = ops.region_blend_cfg(eu, er, m, guidance, latents=lat, guidance_rescale=phi,
                                    step=ops.LMSStep(c1, nan, nan, nan))
    assert torch.equal(x_nan, x_l), "a history under a zero coefficient was read"
    c2 = _coeffs(2)
    _, x2 = ops.region_blend_cfg(eu, er, m, guidance, latents=lat, guidance_rescale=phi,
                                 step=ops.LMSStep(c2, h[0], None, None))
    _, x2n = ops.region_blend_cfg(eu, er, m, guidance, latents=lat, guidance_rescale=phi,
                                  step=ops.LMSStep(c2, h[0], nan, nan))
    assert torch.equal(x2, x2n), "d2 / d3 read at order 2"
    eps_ref = torch.full_like(lat_ref, float("nan"))
    g_eu = _gather_world1(eu, er, m, guidance, lat, (ec, ed, lat_ref), phi, None, dt=c1[0])
    g_l = _gather_world1(eu, er, m, guidance, lat, (ec, ed, lat_ref), phi,
                         ops.LMSStep(c1, None, None, None, None, None, None, eps_ref))
    for a, b, what in zip(g_eu, g_l, ("eps", "latents", "latents_ref")):
        assert torch.equal(a, b), f"order 1 differs from the Euler form (gather): {what}"
    e_cd, _ = ops.region_blend_cfg(ec, [ed], ones, guidance, latents=lat_ref, guidance_rescale=phi,
                                   step=ops.LMSStep(c1, None, None, None))
    assert torch.equal(eps_ref, e_cd), "eps_ref_out differs from the single form's eps of C/D"
    c4 = _coeffs(4)

    def single():
        eps, lo_ = ops.region_blend_cfg(eu, er, m, guidance, latents=lat, guidance_rescale=phi,
                                        step=ops.LMSStep(c4, *h))
        _, ro = ops.region_blend_cfg(ec, [ed], ones, guidance, latents=lat_ref, guidance_rescale=phi,
                                     step=ops.LMSStep(c4, *h_ref))
        return eps, lo_, ro

    a = single()
    for x, y in zip(a, single()):
        assert torch.equal(x, y), "two calls differ"
    eps_ref4 = torch.empty_like(lat_ref)
    gw = _gather_world1(eu, er, m, guidance, lat, (ec, ed, lat_ref), phi, ops.LMSStep(c4, *h, *h_ref, eps_ref4))
    for x, y, what in zip(a, gw, ("eps", "latents", "latents_ref")):
        assert torch.equal(x, y), f"gather world 1 vs single GPU: {what} differs"
    assert torch.equal(eps_ref4, e_cd), "eps_ref_out at order 4 differs from the single form's eps of C/D"
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
def test_lms_step_refuses_overlapping_outputs():
    """eps_ref_out may not share storage with a history it would overwrite."""
    from rtti_b200 import _lib, ops
    n = 16384
    eu, er, m, lat, ec, ed, lat_ref, h, h_ref = _inputs(n, 2, 5)
    with pytest.raises(_lib.RttiError, match="d2_ref overlaps"):
        _gather_world1(eu, er, m, 5.0, lat, (ec, ed, lat_ref), 0.0,
                       ops.LMSStep(_coeffs(4), *h, h_ref[0], h_ref[1], h_ref[2], h_ref[1]))


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
    cfg, m = _xl_model(scheduler or _lms())
    S = mo.LATENT_XL_PLAIN
    inp = synth.synth_inputs(cfg.cross_attention_dim, _pooled(cfg), 3, S, 31)
    ctx, te = inp["ctx"].cuda(), inp["text_embeds"].cuda()
    cb = (lambda i, t, lat: calls.append(i)) if calls is not None else None
    return m.sample(height=S * 8, width=S * 8, num_inference_steps=steps, guidance_scale=8.5,
                    latents=inp["latents"].clone(), prompt_embeds=ctx[-1:], negative_prompt_embeds=ctx[:1],
                    pooled_prompt_embeds=te[-1:], negative_pooled_prompt_embeds=te[:1], output_type="latent",
                    run_rich_text=False, callback=cb, callback_steps=1).images.float().cpu().numpy()


def _xl_rich(sa, bg, scheduler=None, graphs=True, calls=None, callback_steps=1):
    cfg, m = _xl_model(scheduler or _lms())
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
    """The plain pass against the reference's, and its callback iterations (every step); the Euler run of the same
    inputs lies outside the tolerance."""
    from rtti_b200.schedulers import EulerDiscreteScheduler
    ref = _golden()[f"xl_plain_{steps}"]
    calls = []
    _close_range(_xl_plain(steps, calls=calls), ref, f"xl plain {steps}")
    assert calls == _golden()[f"xl_plain_{steps}_callbacks"].tolist() == list(range(steps)), calls
    with pytest.raises(AssertionError):
        _close_range(_xl_plain(steps, EulerDiscreteScheduler()), ref, "xl plain, Euler")


@pytest.mark.gpu
@pytest.mark.parametrize("sa,bg", [(0.5, 0.5), (0.0, 0.0)])
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
    assert calls2 == [0, 2], calls2


@pytest.mark.gpu
def test_rich_loop_keeps_a_history_per_trajectory():
    """inject_selfattn = 0, inject_background = 0.5: the reference latents are stepped on steps 0 and 1 only; the main
    latents go on with their own history, as the per-trajectory oracle loop does; the reference loop would add a batch-1
    prediction to batch-2 ones here."""
    sched = lo.PerTrajectoryLMSOracle()
    ref = _xl_rich_oracle(0.0, 0.5, sched)
    assert sched.step_batches == [2, 2, 1, 1]
    _close_range(_xl_rich(0.0, 0.5), ref.detach().numpy(), "xl rich 0 / 0.5 vs the per-trajectory oracle")


@pytest.mark.gpu
def test_rich_loop_lms_two_gpus():
    """LMS on the fused peer exchange and on the NCCL path (tests/multigpu_lms_check.py)."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
                        "--master-addr", "127.0.0.1", "--master-port", "29547",
                        os.path.join(ROOT, "tests", "multigpu_lms_check.py")],
                       capture_output=True, text=True, timeout=900)
    print(r.stdout[-2000:], r.stderr[-2000:])
    assert r.returncode == 0 and "MULTIGPU_LMS_CHECK PASS" in r.stdout
