"""Euler Ancestral in RegionDiffusionXL, with the noise term fused into the blend kernels (rtti_region_blend_cfg_anc,
rtti_region_blend_cfg_rescale_anc, rtti_gather_blend_step_anc, rtti_gather_blend_step_rescale_anc).

CPU: the grid (Euler's), the coefficients (sigma_up^2 + sigma_down^2 = sigma'^2; a variance recursion that converges only
with sigma_up and sigma_down in their places), the torch step against float64, the generator semantics, the oracle loops
against the unmodified reference (tests/golden/ancestral.npz, tests/gen_ancestral.py), the C-ABI argument checks, the
cubin and the multi-rank noise-source check over gloo. GPU: the kernels against float64 (tests/fp64_rule.py, K = 2, mean
check on; the comparator is the fp16 torch expression diffusers evaluates), bit-identities, and the sampler against the
goldens and against the oracle fed the draws of the device RNG."""
import ctypes
import math
import os
import re
import shutil
import socket
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests import ancestral_oracle as ao
from tests import multistep_oracle as mo
from tests import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
ARG, SHAPE, ALIGN = -1, -2, -3
SEED = 1234   # tests/gen_ancestral.py


def _golden():
    return np.load(os.path.join(GOLDEN, "ancestral.npz"), allow_pickle=False)


def _anc(**kw):
    from rtti_b200.schedulers import EulerAncestralDiscreteScheduler
    return EulerAncestralDiscreteScheduler(**kw)


def _pooled(cfg):
    return cfg.projection_class_embeddings_input_dim - 6 * cfg.addition_time_embed_dim


# ------------------------------------------------------------------------------------------------ CPU: scheduler
@pytest.mark.parametrize("N", [10, 20, 41, 50])
def test_grid_equals_euler(N):
    from rtti_b200.schedulers import EulerDiscreteScheduler
    a, e = _anc(), EulerDiscreteScheduler()
    assert a.init_noise_sigma == e.init_noise_sigma and torch.equal(a.alphas_cumprod, e.alphas_cumprod)
    a.set_timesteps(N)
    e.set_timesteps(N)
    assert a.timesteps.tolist() == e.timesteps.tolist() and a.num_inference_steps == N
    assert np.array_equal(a.sigmas_host, e.sigmas_host) and a.sigmas_host.dtype == np.float32
    x = torch.randn(2, 4, 8, 8)
    for t in a.timesteps[:: max(1, N // 4)]:
        assert torch.equal(a.scale_model_input(x, t), e.scale_model_input(x, t))


def test_config_and_dispatch():
    from rtti_b200 import schedulers as S
    from rtti_b200.region_diffusion_sdxl import _step_kind
    a = _anc()
    assert not isinstance(a, S.EulerDiscreteScheduler), "an Euler subclass would be stepped as deterministic Euler"
    assert _step_kind(a) == "ancestral" and _step_kind(S.EulerDiscreteScheduler()) == "euler"
    assert isinstance(S.EulerAncestralDiscreteScheduler.from_config(S.EulerDiscreteScheduler()), S.EulerAncestralDiscreteScheduler)
    assert S.EulerAncestralDiscreteScheduler.from_config(dict(a.config)).config == a.config
    assert S.EulerAncestralDiscreteScheduler.from_config(S.DDIMScheduler().config).config.steps_offset == 1
    with pytest.raises(NotImplementedError):   # DPM-Solver's linspace grid is not this scheduler's
        S.EulerAncestralDiscreteScheduler.from_config(S.DPMSolverMultistepScheduler().config)
    for kw in (dict(timestep_spacing="trailing"), dict(prediction_type="v_prediction"), dict(trained_betas=[0.1] * 1000),
               dict(beta_schedule="linear")):
        with pytest.raises(NotImplementedError):
            _anc(**kw)
    with pytest.raises(TypeError):
        _anc(use_karras_sigmas=True)


@pytest.mark.parametrize("N", [4, 10, 41])
def test_coefficients(N):
    """sigma_up^2 + sigma_down^2 = sigma'^2 at every step; the last step (sigma' = 0) has sigma_up = sigma_down = 0, i.e.
    dt = -sigma."""
    s = _anc()
    s.set_timesteps(N)
    sig = s.sigmas_host.astype(np.float64)
    for i in range(N):
        dt, s_up = s.ancestral_coeffs(i)
        s_down = dt + sig[i]
        assert 0.0 <= s_up < sig[i + 1] + 1e-12 or sig[i + 1] == 0.0
        assert math.isclose(s_up ** 2 + s_down ** 2, sig[i + 1] ** 2, rel_tol=1e-12, abs_tol=1e-15)
    dt, s_up = s.ancestral_coeffs(N - 1)
    assert s_up == 0.0 and dt == -sig[N - 1]


def _variance_errors(N, swap=False):
    s = _anc()
    s.set_timesteps(N)
    sig = s.sigmas_host.astype(np.float64)
    v = sig[0] ** 2 + 1.0
    for i in range(N):
        dt, s_up = s.ancestral_coeffs(i)
        if swap:
            dt, s_up = s_up - sig[i], dt + sig[i]
        v = (1.0 + dt * sig[i] / (1.0 + sig[i] ** 2)) ** 2 * v + s_up ** 2
    return v - 1.0


def test_variance_converges_with_the_step_count():
    """Unit-variance Gaussian data: the exact eps of x at noise level sigma is x sigma / (1 + sigma^2), so the variance
    of the samples follows v' = (1 + dt sigma / (1 + sigma^2))^2 v + sigma_up^2 from sigma_0^2 + 1 and must end at 1.
    The error falls at least 1.6x per doubling of the step count; with sigma_up and sigma_down swapped it does not."""
    Ns = (10, 20, 40, 80, 160)
    errs = [_variance_errors(N) for N in Ns]
    ratios = [errs[k] / errs[k + 1] for k in range(len(Ns) - 1)]
    swapped = [_variance_errors(N, swap=True) for N in Ns]
    print("final-variance errors", [round(e, 4) for e in errs], "ratios", [round(r, 2) for r in ratios],
          "swapped", [round(e, 4) for e in swapped])
    assert min(ratios) >= 1.6, ratios
    assert abs(errs[-1]) < 0.05
    assert not min(swapped[k] / swapped[k + 1] for k in range(len(Ns) - 1)) >= 1.6, swapped
    assert min(abs(e) for e in swapped) > 0.25, swapped


def test_torch_step_matches_float64_and_draws_like_randn():
    """step() against float64 of x + (sigma_down - sigma) eps + sigma_up z, z drawn from the CPU generator as
    torch.randn(shape, dtype=fp16, generator=g) draws it; and against the diffusers-form oracle."""
    s = _anc()
    s.set_timesteps(10)
    o = ao.EulerAncestralSchedulerOracle()
    o.set_timesteps(10)
    assert s.timesteps.tolist() == o.timesteps.tolist()
    g0 = torch.Generator().manual_seed(3)
    x = torch.randn(2, 4, 8, 8, generator=g0) * 5
    for i, t in enumerate(s.timesteps):
        e = torch.randn(2, 4, 8, 8, generator=g0).half()
        got = s.step(e, t, x, generator=torch.Generator().manual_seed(100 + i))["prev_sample"]
        z = torch.randn(2, 4, 8, 8, dtype=torch.float16, generator=torch.Generator().manual_seed(100 + i))
        assert torch.equal(s.noise((2, 4, 8, 8), torch.Generator().manual_seed(100 + i), "cpu"), z)
        sg, sn = float(s.sigmas_host[i]), float(s.sigmas_host[i + 1])
        up = math.sqrt(sn ** 2 * (sg ** 2 - sn ** 2) / sg ** 2)
        want = x.double() + (math.sqrt(sn ** 2 - up ** 2) - sg) * e.double() + up * z.double()
        torch.testing.assert_close(got.double(), want, rtol=1e-6, atol=1e-6 * float(want.abs().max()))
        ref = o.step(e.float(), t, x, generator=torch.Generator().manual_seed(100 + i))["prev_sample"]
        torch.testing.assert_close(got, ref, rtol=1e-5, atol=1e-5 * float(ref.abs().max()))
        x = got


def test_joint_draw_is_split_main_first():
    """The rich-text loop's joint step: the oracle steps cat([main, ref]) with one [2, ...] draw; the product steps each
    trajectory with its half of the same draw, the main latents taking the first."""
    s = _anc()
    s.set_timesteps(4)
    o = ao.EulerAncestralSchedulerOracle(generator=torch.Generator().manual_seed(9))
    o.set_timesteps(4)
    g = torch.Generator().manual_seed(1)
    x, xr, e, er = (torch.randn(1, 4, 8, 8, generator=g) for _ in range(4))
    t = s.timesteps[1]
    both = o.step(torch.cat([e, er]), t, torch.cat([x, xr]))["prev_sample"]
    z = s.noise((2, 4, 8, 8), torch.Generator().manual_seed(9), "cpu")
    assert not torch.equal(z[0], z[1])
    dt, s_up = s.ancestral_coeffs(1)
    for k, (xx, ee) in enumerate(((x, e), (xr, er))):
        want = xx.double() + dt * ee.double() + s_up * z[k:k + 1].double()
        torch.testing.assert_close(both[k:k + 1].double(), want, rtol=1e-5, atol=1e-5 * float(want.abs().max()))


# ------------------------------------------------------------------------------------------------ CPU: goldens
def _xl_plain_oracle(steps, generator=None, noises=None):
    from oracle import sampler_oracle as sam, unet_oracle as uo
    cfg = uo.tiny_xl_config()
    S = mo.LATENT_XL_PLAIN
    unet = sam.make_unet_fn(uo.make_state_dict(cfg, 2), cfg)
    inp = synth.synth_inputs(cfg.cross_attention_dim, _pooled(cfg), 3, S, 31)
    ctx, te = inp["ctx"], inp["text_embeds"]
    added2 = {"text_embeds": torch.cat([te[:1], te[-1:]]), "time_ids": inp["time_ids"].repeat(2, 1)}
    return ao.plain_loop(unet, ao.EulerAncestralSchedulerOracle(noises=noises), torch.cat([ctx[:1], ctx[-1:]]),
                         inp["latents"].clone(), steps, 8.5, added_cond=added2, generator=generator)


def _xl_rich_oracle(inject_selfattn, inject_background, generator=None, noises=None, sched=None):
    from oracle import sampler_oracle as sam, unet_oracle as uo
    cfg = uo.tiny_xl_config()
    S = mo.LATENT_XL_RICH
    inp = synth.synth_inputs(cfg.cross_attention_dim, _pooled(cfg), 3, S, 31)
    ctx, te = inp["ctx"], inp["text_embeds"]
    tfd = synth.font_sizes()
    tfd.update(synth.color_dict(inp["masks"], S, 1.0))
    sched = sched or ao.EulerAncestralSchedulerOracle(generator=generator, noises=noises)
    return ao.rich_text_loop(sam.make_unet_fn(uo.make_state_dict(cfg, 2), cfg), sched, ctx, inp["masks"],
                             inp["latents"].clone(), 4, 8.5, xl=True,
                             added_cond={"text_embeds": te, "time_ids": inp["time_ids"]}, use_guidance=True,
                             text_format_dict=tfd, inject_selfattn=inject_selfattn,
                             inject_background=inject_background, vae_decode=synth.TinyVAE(), scaling_factor=0.13025)


def _assert_golden(got, ref, what):
    np.testing.assert_allclose(np.asarray(got, np.float32), ref, atol=5e-4 * max(1.0, float(np.abs(ref).max()) / 10),
                               rtol=1e-4, err_msg=what)


@pytest.mark.parametrize("steps", [10, 20])
def test_oracle_xl_plain_matches_reference(steps):
    got = _xl_plain_oracle(steps, generator=torch.Generator().manual_seed(SEED))
    _assert_golden(got.numpy(), _golden()[f"xl_plain_{steps}"], f"xl plain {steps}")


@pytest.mark.parametrize("sa,bg", [(0.5, 0.5), (0.0, 0.5)])
def test_oracle_xl_rich_matches_reference(sa, bg):
    """Joint [2, ...] draws on every step (0.5 / 0.5), and joint then main-only draws (0 / 0.5)."""
    sched = ao.EulerAncestralSchedulerOracle(generator=torch.Generator().manual_seed(SEED))
    got = _xl_rich_oracle(sa, bg, sched=sched)
    S = mo.LATENT_XL_RICH
    joint = 4 if sa > 0 else 2
    assert sched.draw_shapes == [(2, 4, S, S)] * joint + [(1, 4, S, S)] * (4 - joint)
    _assert_golden(got.detach().numpy(), _golden()[f"xl_rich_{sa:g}_{bg:g}"], f"xl rich {sa} {bg}")


# ------------------------------------------------------------------------------------------------ CPU: C ABI, cubin
def test_ancestral_abi_rejects_bad_arguments_without_launching():
    """Every call below fails its argument checks; a launch without a device would return RTTI_ERR_CUDA instead."""
    from rtti_b200 import _lib
    lib = _lib.load()
    V = ctypes.c_void_p
    buf = (ctypes.c_char * 8192)()
    a = (ctypes.addressof(buf) + 15) // 16 * 16
    regions = (V * 3)(V(a), V(a), V(a))
    for fn, extra in ((lib.rtti_region_blend_cfg_anc, []), (lib.rtti_region_blend_cfg_rescale_anc, [0.7])):
        rb = lambda lat=a, z=a, n=64, s_up=0.3, eu=a, regs=regions, N=3: fn(
            V(eu), regs, V(a), N, n, 7.5, V(a), V(lat), V(lat), -0.4, s_up, V(z), *extra, V(0))
        assert rb(eu=0) == ARG
        assert rb(regs=(V * 3)(V(a), V(0), V(a))) == ARG
        assert rb(N=17) == ARG
        assert rb(lat=0) == ARG                 # the ancestral update needs the latents
        assert rb(z=0) == ARG                   # s_up != 0 needs the noise
        assert rb(n=60) == SHAPE
        assert rb(z=a + 2) == ALIGN
        assert rb(z=a + 8, s_up=0.0) == ALIGN   # a noise pointer that is given must be aligned
    peers = (V * 2)(V(a), V(a))
    owner = (ctypes.c_int * 6)(0, 0, 1, 1, 0, 1)
    for fn, extra in ((lib.rtti_gather_blend_step_anc, []), (lib.rtti_gather_blend_step_rescale_anc, [0.7])):
        gb = lambda world=2, rank=0, n=64, ref=0, z=a, z_ref=a, s_up=0.3, lat=a, slots=peers: fn(
            slots, peers, world, rank, owner, 6, 3, V(a), n, 7.5, V(a), V(lat), V(lat), V(ref), V(ref), -0.4, s_up,
            V(z), V(z_ref), 1, *extra, V(0))
        assert gb(world=17) == ARG
        assert gb(rank=2) == ARG
        assert gb(slots=(V * 2)(V(a), V(0))) == ARG
        assert gb(lat=0) == ARG
        assert gb(z=0) == ARG
        assert gb(ref=a, z_ref=0) == ARG        # the reference trajectory needs its own noise
        assert gb(n=60) == SHAPE
        assert gb(z=a + 4) == ALIGN
        assert gb(ref=a, z_ref=a + 4) == ALIGN
        assert gb(world=1) == ARG               # slot owned by rank 1 of a world of 1


def _sass_by_kernel():
    from rtti_b200 import _lib
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    _lib.load()
    sass = subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True).stdout
    out = {}
    for f in re.split(r"\n\s*Function : ", sass)[1:]:
        name = f.split("\n", 1)[0]
        m = re.search(r"\d(region_blend|gather_blend|blend_rescale)(_anc)?_kernel(ILb[01]E)?", name)
        if m:
            out[(m.group(1), m.group(3) or "", bool(m.group(2)))] = (name, f)
    return out


def test_ancestral_kernels_in_the_cubin():
    """Each of the four families has its _anc kernel, whose 128-bit loads are those of its Euler kernel plus the noise
    (one per trajectory it steps); the rescale cluster kernels stay within 64 registers at 1024 threads, no spills."""
    from rtti_b200 import _lib
    k = _sass_by_kernel()
    fams = [("region_blend", "", 1), ("gather_blend", "", 2), ("blend_rescale", "ILb0E", 2), ("blend_rescale", "ILb1E", 2)]
    for fam, tpl, extra in fams:
        assert (fam, tpl, True) in k and (fam, tpl, False) in k, (fam, tpl, sorted(k))
        ld = {anc: len(re.findall(r"\bLDG\.E\.128\b", k[(fam, tpl, anc)][1])) for anc in (False, True)}
        assert ld[True] >= ld[False] + extra, (fam, tpl, ld)
        if fam == "blend_rescale":
            assert not re.search(r"\bSTL", k[(fam, tpl, True)][1]), f"{fam}{tpl}: local-memory stores (spills)"
    out = subprocess.run(["cuobjdump", "-res-usage", _lib.LIB_PATH], capture_output=True, text=True).stdout
    regs = [int(r) for fn, r in re.findall(r"Function (\S+):\s*\n\s*REG:(\d+)", out) if "blend_rescale_anc_kernel" in fn]
    assert len(regs) == 2
    for r in regs:
        assert r <= 64 and ((r * 32 + 255) // 256 * 256) * 32 <= 65536, f"{r} registers x 32 warps"


# ------------------------------------------------------------------------------------------------ CPU: ranks (gloo)
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _digest_worker(rank, world, port, q):
    import torch.distributed as dist
    sys.path.insert(0, ROOT)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from rtti_b200 import region_parallel as rp
    res = []
    for seeds in ((5, 5), (5, 6)):
        g = torch.Generator().manual_seed(seeds[rank])
        try:
            rp.check_noise_source(g, torch.device("cpu"))
            res.append("ok")
        except RuntimeError as e:
            res.append("raised" if "noise sources differ" in str(e) else repr(e))
    q.put((rank, res))
    dist.destroy_process_group()


def test_noise_source_check_gloo_world2():
    """Ranks whose generators agree pass; one rank seeded differently makes the check raise on both ranks."""
    import torch.multiprocessing as mp
    from rtti_b200 import region_parallel as rp
    assert rp.noise_source_digest(torch.Generator().manual_seed(5)) == rp.noise_source_digest(torch.Generator().manual_seed(5))
    assert rp.noise_source_digest(torch.Generator().manual_seed(5)) != rp.noise_source_digest(torch.Generator().manual_seed(6))
    g = torch.Generator().manual_seed(5)
    d0 = rp.noise_source_digest(g)
    torch.randn(3, generator=g)
    assert rp.noise_source_digest(g) != d0, "the digest must follow the state, not the seed"
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_digest_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = dict(q.get(timeout=120) for _ in procs)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    assert res == {0: ["ok", "raised"], 1: ["ok", "raised"]}, res


# ------------------------------------------------------------------------------------------------ GPU: accuracy
def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _masks(N, n, g):
    m = torch.rand(N, n, device="cuda", generator=g)
    return (m / m.sum(0, keepdim=True)).half().float().contiguous()


def _coeffs(kind):
    s = _anc()
    s.set_timesteps(20)
    return s.ancestral_coeffs(19 if kind == "last" else 6)


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
    eu = torch.randn(n, device="cuda", generator=g).half()
    er = [torch.randn(n, device="cuda", generator=g).half() for _ in range(N)]
    m = _masks(N, n, g)
    lat = (3 * torch.randn(n, device="cuda", generator=g)).half()
    ec, ed = torch.randn(n, device="cuda", generator=g).half(), torch.randn(n, device="cuda", generator=g).half()
    lat_ref = (3 * torch.randn(n, device="cuda", generator=g)).half()
    z, z_ref = torch.randn(n, device="cuda", generator=g).half(), torch.randn(n, device="cuda", generator=g).half()
    return eu, er, m, lat, ec, ed, lat_ref, z, z_ref


def _blend64(eu, er, m, guidance, phi):
    md = m.double()
    u64 = sum(eu.double() * md[k] for k in range(len(er)))
    t64 = sum(er[k].double() * md[k] for k in range(len(er)))
    e64 = u64 + guidance * (t64 - u64)
    if phi:
        e64 = e64 * (1 - phi + phi * t64.std() / e64.std())
    return e64


@pytest.mark.gpu
@pytest.mark.parametrize("step_kind", ["up", "last"])
@pytest.mark.parametrize("with_ref", [False, True])
@pytest.mark.parametrize("phi", [0.0, 0.7])
@pytest.mark.parametrize("N", [2, 5, 16])
@pytest.mark.parametrize("n", [16384, 65536, 65528])
@pytest.mark.parametrize("family", ["single", "gather"])
def test_anc_kernels_vs_fp64(family, n, N, phi, with_ref, step_kind):
    """latents_out (and the reference latents with C/D) against float64 of x + dt eps + s_up z on the exact blend;
    "last" is the step with s_up = 0."""
    from rtti_b200 import ops
    from tests.fp64_rule import half_ulp16, no_worse
    dt, s_up = _coeffs(step_kind)
    assert (s_up == 0.0) == (step_kind == "last")
    eu, er, m, lat, ec, ed, lat_ref, z, z_ref = _inputs(n, N, n + 13 * N + int(10 * phi) + 7 * with_ref)
    guidance = 5.0
    ones = torch.ones(1, n, device="cuda")
    if family == "single":
        e1, x1 = ops.region_blend_cfg(eu, er, m, guidance, latents=lat, guidance_rescale=phi,
                                      step=ops.AncestralStep(dt, s_up, z))
        xr = ops.region_blend_cfg(ec, [ed], ones, guidance, latents=lat_ref, guidance_rescale=phi,
                                  step=ops.AncestralStep(dt, s_up, z_ref))[1] if with_ref else None
    else:
        e1, x1, xr = _gather_world1(eu, er, m, guidance, lat, (ec, ed, lat_ref if with_ref else None), phi,
                                    ops.AncestralStep(dt, s_up, z, z_ref if with_ref else None))
    tag = f"anc {family} n{n} N{N} phi{phi:g} {step_kind}"
    trajectories = [(e1, x1, lat, z, _blend64(eu, er, m, guidance, phi), "latents")]
    if with_ref:
        e_ref16 = ops.region_blend_cfg(ec, [ed], ones, guidance, guidance_rescale=phi)   # the fp16 prediction stepped
        trajectories.append((e_ref16, xr, lat_ref, z_ref, _blend64(ec, [ed], ones, guidance, phi), "latents_ref"))
    for e16, got, x, zz, e64, what in trajectories:
        want64 = x.double() + dt * e64 + s_up * zz.double()
        cmp16 = (x + e16 * dt) + zz * s_up   # diffusers in fp16 on the fp16 prediction the reference would hold
        no_worse(f"{tag} {what}", got, cmp16, want64, k=2.0, floor=half_ulp16(want64), mean=True)


# ------------------------------------------------------------------------------------------------ GPU: bit-identities
@pytest.mark.gpu
@pytest.mark.parametrize("phi", [0.0, 0.7])
@pytest.mark.parametrize("n,N", [(16384, 5), (65528, 2), (65536, 16)])
def test_anc_bit_identities(n, N, phi):
    """s_up = 0 equals the Euler entry point with the same dt (all four families, z absent); the gather form at world 1
    equals the single-GPU form (both trajectories); repeated calls agree; a CUDA-graph replay equals eager."""
    from rtti_b200 import ops
    eu, er, m, lat, ec, ed, lat_ref, z, z_ref = _inputs(n, N, n + N + 1)
    ones = torch.ones(1, n, device="cuda")
    guidance = 8.5
    dt0, _ = _coeffs("last")
    e_eu, x_eu = ops.region_blend_cfg(eu, er, m, guidance, latents=lat, dt_sigma=dt0, guidance_rescale=phi)
    e_an, x_an = ops.region_blend_cfg(eu, er, m, guidance, latents=lat, guidance_rescale=phi,
                                      step=ops.AncestralStep(dt0, 0.0, None))
    assert torch.equal(e_eu, e_an) and torch.equal(x_eu, x_an), "s_up = 0 differs from the Euler form (single GPU)"
    g_eu = _gather_world1(eu, er, m, guidance, lat, (ec, ed, lat_ref), phi, None, dt=dt0)
    g_an = _gather_world1(eu, er, m, guidance, lat, (ec, ed, lat_ref), phi, ops.AncestralStep(dt0, 0.0, None, None))
    for a, b, what in zip(g_eu, g_an, ("eps", "latents", "latents_ref")):
        assert torch.equal(a, b), f"s_up = 0 differs from the Euler form (gather): {what}"
    dt, s_up = _coeffs("up")
    assert s_up > 0

    def single():
        eps, lo = ops.region_blend_cfg(eu, er, m, guidance, latents=lat, guidance_rescale=phi,
                                       step=ops.AncestralStep(dt, s_up, z))
        _, ro = ops.region_blend_cfg(ec, [ed], ones, guidance, latents=lat_ref, guidance_rescale=phi,
                                     step=ops.AncestralStep(dt, s_up, z_ref))
        return eps, lo, ro

    a = single()
    b = single()
    for x, y in zip(a, b):
        assert torch.equal(x, y), "two calls differ"
    assert not torch.equal(a[1], x_eu), "the noise was not added"
    gw = _gather_world1(eu, er, m, guidance, lat, (ec, ed, lat_ref), phi, ops.AncestralStep(dt, s_up, z, z_ref))
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


def _xl_plain(steps, generator, scheduler=None, cuda_seed=None):
    cfg, m = _xl_model(scheduler or _anc())
    S = mo.LATENT_XL_PLAIN
    inp = synth.synth_inputs(cfg.cross_attention_dim, _pooled(cfg), 3, S, 31)
    ctx, te = inp["ctx"].cuda(), inp["text_embeds"].cuda()
    if cuda_seed is not None:
        torch.cuda.manual_seed(cuda_seed)
    return m.sample(height=S * 8, width=S * 8, num_inference_steps=steps, guidance_scale=8.5,
                    latents=inp["latents"].clone(), prompt_embeds=ctx[-1:], negative_prompt_embeds=ctx[:1],
                    pooled_prompt_embeds=te[-1:], negative_pooled_prompt_embeds=te[:1], output_type="latent",
                    run_rich_text=False, generator=generator).images.float().cpu().numpy()


def _xl_rich(sa, bg, generator, scheduler=None, graphs=True, cuda_seed=None):
    cfg, m = _xl_model(scheduler or _anc())
    m.use_cuda_graphs = graphs
    S = mo.LATENT_XL_RICH
    inp = synth.synth_inputs(cfg.cross_attention_dim, _pooled(cfg), 3, S, 31)
    ctx, te = inp["ctx"], inp["text_embeds"]
    tfd = synth.font_sizes()
    tfd.update(synth.color_dict(inp["masks"], S, 1.0))
    m.masks = [x.cuda() for x in inp["masks"]]
    if cuda_seed is not None:
        torch.cuda.manual_seed(cuda_seed)
    return m.sample(height=S * 8, width=S * 8, num_inference_steps=4, guidance_scale=8.5,
                    latents=inp["latents"].clone(), prompt_embeds=ctx[1:].cuda(), negative_prompt_embeds=ctx[:1].cuda(),
                    pooled_prompt_embeds=te[1:].cuda(), negative_pooled_prompt_embeds=te[:1].cuda(),
                    output_type="latent", run_rich_text=True, use_guidance=True, inject_selfattn=sa,
                    inject_background=bg, text_format_dict=tfd, generator=generator).images.float().cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("steps", [10, 20])
def test_xl_plain_vs_reference_golden(steps):
    """A seeded CPU generator against the reference's plain pass; another seed, and the Euler run, lie outside the
    tolerance."""
    from rtti_b200.schedulers import EulerDiscreteScheduler
    ref = _golden()[f"xl_plain_{steps}"]
    _close_range(_xl_plain(steps, torch.Generator().manual_seed(SEED)), ref, f"xl plain {steps}")
    with pytest.raises(AssertionError):
        _close_range(_xl_plain(steps, torch.Generator().manual_seed(SEED + 1)), ref, "xl plain, other seed")
    with pytest.raises(AssertionError):
        _close_range(_xl_plain(steps, None, EulerDiscreteScheduler()), ref, "xl plain, Euler")


@pytest.mark.gpu
@pytest.mark.parametrize("sa,bg", [(0.5, 0.5), (0.0, 0.5)])
def test_xl_rich_vs_reference_golden(sa, bg):
    """Injection, font sizes and colour guidance with a seeded CPU generator against the reference's loop; another seed,
    and the Euler run, lie outside the tolerance; CUDA-graph replayed UNet passes give the same bits as eager ones."""
    from rtti_b200.schedulers import EulerDiscreteScheduler
    ref = _golden()[f"xl_rich_{sa:g}_{bg:g}"]
    out = _xl_rich(sa, bg, torch.Generator().manual_seed(SEED))
    _close_range(out, ref, f"xl rich {sa} {bg}")
    with pytest.raises(AssertionError):
        _close_range(_xl_rich(sa, bg, torch.Generator().manual_seed(SEED + 1)), ref, "xl rich, other seed")
    with pytest.raises(AssertionError):
        _close_range(_xl_rich(sa, bg, None, EulerDiscreteScheduler()), ref, "xl rich, Euler")
    assert np.array_equal(out, _xl_rich(sa, bg, torch.Generator().manual_seed(SEED), graphs=False)), \
        "use_cuda_graphs on / off differ"


def _recorded_draws(shapes, seed):
    torch.cuda.manual_seed(seed)
    return [torch.randn(s, dtype=torch.float16, device="cuda").cpu() for s in shapes]


@pytest.mark.gpu
def test_device_rng_draws_match_the_reference():
    """generator=None: the global RNG of the device. Two runs after torch.cuda.manual_seed(s) are bit-identical, and
    equal the oracle loop fed the draws recorded from the same seed with the reference's shapes in the reference's
    order ([1, ...] per plain step; [2, ...] on the joint rich steps, then [1, ...])."""
    S = mo.LATENT_XL_PLAIN
    a = _xl_plain(6, None, cuda_seed=77)
    assert np.array_equal(a, _xl_plain(6, None, cuda_seed=77)), "plain pass: two runs from the same device seed differ"
    ref = _xl_plain_oracle(6, noises=_recorded_draws([(1, 4, S, S)] * 6, 77))
    _close_range(a, ref.numpy(), "xl plain, device RNG, vs oracle")
    S = mo.LATENT_XL_RICH
    b = _xl_rich(0.0, 0.5, None, cuda_seed=78)
    assert np.array_equal(b, _xl_rich(0.0, 0.5, None, cuda_seed=78)), "rich loop: two runs from the same device seed differ"
    shapes = [(2, 4, S, S)] * 2 + [(1, 4, S, S)] * 2
    ref = _xl_rich_oracle(0.0, 0.5, noises=_recorded_draws(shapes, 78))
    _close_range(b, ref.detach().numpy(), "xl rich 0 / 0.5, device RNG, vs oracle")
    ones = _recorded_draws([(1, 4, S, S)] * 6, 78)   # two [1, ...] draws per joint step instead of one [2, ...] draw
    split = [torch.cat(ones[0:2]), torch.cat(ones[2:4])] + ones[4:]
    with pytest.raises(AssertionError):
        _close_range(b, _xl_rich_oracle(0.0, 0.5, noises=split).detach().numpy(), "rich loop, [1, ...] draws")


@pytest.mark.gpu
def test_rich_loop_ancestral_two_gpus():
    """Euler Ancestral on the fused peer exchange and on the NCCL path (tests/multigpu_ancestral_check.py)."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
                        "--master-addr", "127.0.0.1", "--master-port", "29541",
                        os.path.join(ROOT, "tests", "multigpu_ancestral_check.py")],
                       capture_output=True, text=True, timeout=900)
    print(r.stdout[-2000:], r.stderr[-2000:])
    assert r.returncode == 0 and "MULTIGPU_ANCESTRAL_CHECK PASS" in r.stdout
