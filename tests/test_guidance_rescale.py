"""guidance_rescale in RegionDiffusionXL: the CFG rescale of diffusers' rescale_noise_cfg fused into the blend kernels
(rtti_region_blend_cfg_rescale, rtti_gather_blend_step_rescale).

CPU: the restated oracle (tests/rescale_oracle.py) against the unmodified reference (tests/golden/xl_rescale.npz,
tests/gen_xl_rescale.py), the C-ABI argument checks and the kernels' SASS / register budget from the cubin.
GPU: the kernels against float64 (tests/fp64_rule.py, K = 2, mean check on; the comparator is the reference's
expression evaluated in fp16), bit-identities (repeat, phi = 0 vs the plain kernels, the gather form at world 1 vs the
single-GPU form, CUDA-graph replay vs eager), and the tiny-XL samplers against the fixture and the oracle."""
import ctypes
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
ARG, SHAPE = -1, -2
MAX_N = 262144


def _golden(name):
    return np.load(os.path.join(GOLDEN, name), allow_pickle=False)


def _pooled(cfg):
    return cfg.projection_class_embeddings_input_dim - 6 * cfg.addition_time_embed_dim


# ------------------------------------------------------------------------------------------------ CPU: oracle
def test_oracle_rescale_noise_cfg_matches_reference():
    from tests import rescale_oracle as ro
    from tests.gen_xl_rescale import PHIS, rescale_inputs
    g = _golden("xl_rescale.npz")
    cfg, text = rescale_inputs()
    for phi in PHIS:
        np.testing.assert_allclose(ro.rescale_noise_cfg(cfg, text, phi).numpy(), g[f"rescale_{phi:g}"], atol=2e-6,
                                   rtol=1e-6)


def test_oracle_plain_loop_with_rescale_matches_reference():
    """The oracle plain pass at phi = 0.7 against the reference, at test_xl_loops_match_reference's tolerance; and far
    from the phi = 0 result, so this cannot pass with phi ignored."""
    from oracle import sampler_oracle as sam, schedulers_oracle as so, unet_oracle as uo
    from tests import rescale_oracle as ro
    g = _golden("xl_rescale.npz")
    cfg = uo.tiny_xl_config()
    S = 128
    unet = sam.make_unet_fn(uo.make_state_dict(cfg, 2), cfg)
    inp = synth.synth_inputs(cfg.cross_attention_dim, _pooled(cfg), 3, S, 31)
    ctx, te = inp["ctx"], inp["text_embeds"]
    sch = so.EulerDiscreteSchedulerOracle()
    sch.set_timesteps(12)
    lat0 = inp["latents"].clone() * sch.init_noise_sigma
    added2 = {"text_embeds": torch.cat([te[:1], te[-1:]]), "time_ids": inp["time_ids"].repeat(2, 1)}
    lat = ro.plain_loop(unet, sch, torch.cat([ctx[:1], ctx[-1:]]), lat0, 12, 8.5, xl=True, added_cond=added2,
                        guidance_rescale=0.7).numpy()
    ref = g["plain_latents_phi0.7"]
    np.testing.assert_allclose(lat, ref, atol=5e-4, rtol=1e-4)
    plain0 = _golden("xl_loops.npz")["plain_latents"]
    tol = 5e-4 + 1e-4 * np.abs(plain0)
    assert np.abs(ref - plain0).max() > 100 * tol.max(), "phi = 0.7 and phi = 0 give nearly the same latents"


# ------------------------------------------------------------------------------------------------ CPU: C ABI
def test_rescale_abi_rejects_bad_arguments_without_launching():
    from rtti_b200 import _lib
    lib = _lib.load()
    V = ctypes.c_void_p
    buf = (ctypes.c_char * 4096)()
    a = (ctypes.addressof(buf) + 15) // 16 * 16
    regions = (V * 3)(V(a), V(a), V(a))
    rb = lambda eu, masks, out, n, regs=regions, N=3: lib.rtti_region_blend_cfg_rescale(
        V(eu), regs, V(masks), N, n, 7.5, V(out), V(0), V(0), -0.1, 0.7, V(0))
    assert rb(0, a, a, 64) == ARG
    assert rb(a, 0, a, 64) == ARG
    assert rb(a, a, 0, 64) == ARG
    assert rb(a, a, a, 64, regs=(V * 3)(V(a), V(0), V(a))) == ARG
    assert rb(a, a, a, 64, N=17) == ARG
    assert rb(a, a, a, 60) == SHAPE
    assert rb(a, a, a, MAX_N + 8) == SHAPE
    peers = (V * 2)(V(a), V(a))
    owner = (ctypes.c_int * 6)(0, 0, 1, 1, 0, 1)
    gb = lambda world, rank, n, slots=peers, flags=peers, masks=a, ref=0: lib.rtti_gather_blend_step_rescale(
        slots, flags, world, rank, owner, 6, 3, V(masks), n, 7.5, V(a), V(0), V(0), V(ref), V(ref), -0.1, 1, 0.7, V(0))
    assert gb(17, 0, 64) == ARG                    # more ranks than the kernel's table
    assert gb(2, 2, 64) == ARG                     # rank outside the world
    assert gb(2, 0, 64, masks=0) == ARG
    assert gb(2, 0, 64, slots=(V * 2)(V(a), V(0))) == ARG
    assert gb(2, 0, 64, flags=(V * 2)(V(0), V(a))) == ARG
    assert gb(2, 0, 60) == SHAPE                   # n not a multiple of 8
    assert gb(2, 0, MAX_N + 8) == SHAPE            # larger than an SDXL 2048^2 latent
    assert gb(1, 0, 64) == ARG                     # slot owned by rank 1 of a world of 1


def _sass_functions():
    from rtti_b200 import _lib
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    _lib.load()
    return _lib.LIB_PATH


def test_rescale_kernels_use_128_bit_accesses_and_fit_the_register_check():
    """From the cubin: LDG.E.128 / STG.E.128 and no 32-bit global store in both instantiations, and the register demand
    at 1024 threads (32 warps, the largest CTA the kernels launch) within the 64K-register file."""
    lib_path = _sass_functions()
    sass = subprocess.run(["cuobjdump", "-sass", lib_path], capture_output=True, text=True).stdout
    seen = 0
    for f in re.split(r"\n\s*Function : ", sass)[1:]:
        name = f.split("\n", 1)[0]
        if "blend_rescale_kernel" in name:
            seen += 1
            assert re.search(r"\bLDG\.E\.128", f) and re.search(r"\bSTG\.E\.128", f), f"{name}: no 128-bit global accesses"
            assert not re.search(r"\bSTG\.E\s", f), f"{name}: 32-bit global stores"
    assert seen == 2, "blend_rescale_kernel<false> / <true> not found in the library"
    out = subprocess.run(["cuobjdump", "-res-usage", lib_path], capture_output=True, text=True).stdout
    regs = [int(r) for fn, r in re.findall(r"Function (\S+):\s*\n\s*REG:(\d+)", out) if "blend_rescale_kernel" in fn]
    assert len(regs) == 2
    for r in regs:
        per_warp = (r * 32 + 255) // 256 * 256
        assert per_warp * 32 <= 65536, f"{r} registers x 32 warps exceed the register file"


# ------------------------------------------------------------------------------------------------ GPU helpers
def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _masks(N, n, g, unit_sum):
    """fp16-representable masks: soft + one-hot mixture summing to 1 (test_unet_kernels_fp64._masks16), or independent
    uniforms in [0, 1) that do not."""
    if unit_sum:
        m = torch.rand(N, n, device="cuda", generator=g)
        m = m / m.sum(0, keepdim=True)
        hard = torch.rand(n, device="cuda", generator=g) < 1 / 3
        pick = torch.randint(0, N, (n,), device="cuda", generator=g)
        m = torch.where(hard[None], torch.nn.functional.one_hot(pick, N).T.float(), m)
    else:
        m = torch.rand(N, n, device="cuda", generator=g)
    return m.half().float().contiguous()


def _twice(fn):
    a = fn()
    b = fn()
    for x, y in zip(a, b):
        assert torch.equal(x, y), "two calls with the same inputs differ"
    return a


def _rescale64(e64, t64, phi):
    f = 1 - phi + phi * t64.std() / e64.std()
    return e64 * f


# ------------------------------------------------------------------------------------------------ GPU: accuracy
@pytest.mark.gpu
@pytest.mark.parametrize("variant", ["unit", "free", "unit+10", "free+10"])
@pytest.mark.parametrize("N", [1, 2, 5, 10, 16])
@pytest.mark.parametrize("n", [16384, 49152, 65536, 65528, MAX_N])
def test_region_blend_cfg_rescale_vs_fp64(n, N, variant):
    """eps = eps_cfg (1 - phi + phi std(eps_t) / std(eps_cfg)) (+ latents + dt_sigma * eps) at g in {1.5, 5, 8.5},
    phi in {0.3, 0.7, 1.0}, with and without the Euler update. Masks that sum to one or not; "+10": every noise
    prediction offset by 10 (the statistics must not cancel). Comparator: the reference's blend, CFG and
    rescale_noise_cfg evaluated in fp16."""
    from rtti_b200 import ops
    from tests.fp64_rule import half_ulp16, no_worse
    g = _gen(n * 31 + N * 7 + len(variant))
    off = 10.0 if variant.endswith("+10") else 0.0
    eu = (torch.randn(n, device="cuda", generator=g) + off).half()
    er = [(torch.randn(n, device="cuda", generator=g) + off).half() for _ in range(N)]
    m = _masks(N, n, g, variant.startswith("unit"))
    lat = (3 * torch.randn(n, device="cuda", generator=g)).half()
    dt = -0.37
    m16, md = m.half(), m.double()
    u64 = sum(eu.double() * md[i] for i in range(N))
    t64 = sum(er[i].double() * md[i] for i in range(N))
    nu, nt = eu * m16[-1], er[-1] * m16[-1]
    for i in range(N - 1):
        nu = nu + eu * m16[i]
        nt = nt + er[i] * m16[i]
    for guidance in (1.5, 5.0, 8.5):
        e64 = u64 + guidance * (t64 - u64)
        e16 = nu + guidance * (nt - nu)
        for phi in (0.3, 0.7, 1.0):
            r64 = _rescale64(e64, t64, phi)
            r16 = (phi * (e16 * (nt.std() / e16.std())) + (1 - phi) * e16)
            tag = f"rescale n{n} N{N} {variant} g{guidance:g} phi{phi:g}"
            for euler in (False, True):
                def run():
                    r = ops.region_blend_cfg(eu, er, m, guidance, latents=lat if euler else None,
                                             dt_sigma=dt if euler else 0.0, guidance_rescale=phi)
                    return r if euler else (r,)
                res = _twice(run)
                no_worse(tag + (" eps+euler" if euler else " eps"), res[0], r16, r64, k=2.0, floor=half_ulp16(r64),
                         mean=True)
                if euler:
                    want64 = lat.double() + dt * r64
                    no_worse(tag + " latents", res[1], lat + r16 * dt, want64, k=2.0, floor=half_ulp16(want64), mean=True)


# ------------------------------------------------------------------------------------------------ GPU: bit-identities
def _gather_world1(eu, er, m, guidance, lat, ref_pair, dt, phi, step_id=3):
    """rtti_gather_blend_step(_rescale) at world 1: this device's own slot buffer is the only peer and holds every
    slot (uncond, regions, C, D) in the step_id parity half."""
    from rtti_b200 import ops
    n, N = eu.numel(), len(er)
    n_slots = N + 3
    slots = torch.zeros(2, n_slots, n, dtype=torch.float16, device="cuda")
    flags = torch.zeros(16, dtype=torch.int32, device="cuda")
    par = step_id & 1
    for s, e in enumerate([eu] + er + (list(ref_pair[:2]) if ref_pair is not None else [eu, eu])):
        slots[par, s].copy_(e)
    eps, lat_out, ref_out = ops.gather_blend_step([slots.data_ptr()], [flags.data_ptr()], 0, [0] * n_slots, N, m,
                                                  guidance, lat, ref_pair[2] if ref_pair is not None else None, dt,
                                                  step_id, guidance_rescale=phi)
    torch.cuda.synchronize()
    assert int(flags[0]) == step_id and int(flags[1]) == 0
    return eps, lat_out, ref_out


@pytest.mark.gpu
@pytest.mark.parametrize("n,N", [(16384, 5), (65536, 10), (65528, 2), (MAX_N, 16)])
def test_rescale_bit_identities(n, N):
    """Repeated calls, phi = 0 through the new entry points vs the plain kernels, the gather form at world 1 vs the
    single-GPU form (the C/D pair against a one-region blend with a mask of ones), and a CUDA-graph replay vs eager."""
    from rtti_b200 import _lib, ops
    g = _gen(n + N)
    eu = torch.randn(n, device="cuda", generator=g).half()
    er = [torch.randn(n, device="cuda", generator=g).half() for _ in range(N)]
    m = _masks(N, n, g, True)
    lat = (3 * torch.randn(n, device="cuda", generator=g)).half()
    ec, ed = torch.randn(n, device="cuda", generator=g).half(), torch.randn(n, device="cuda", generator=g).half()
    lat_ref = (3 * torch.randn(n, device="cuda", generator=g)).half()
    ones = torch.ones(1, n, device="cuda")
    dt, guidance = -0.37, 8.5
    lib = _lib.load()

    def single(phi):
        eps, lo = ops.region_blend_cfg(eu, er, m, guidance, latents=lat, dt_sigma=dt, guidance_rescale=phi)
        _, ro = ops.region_blend_cfg(ec, [ed], ones, guidance, latents=lat_ref, dt_sigma=dt, guidance_rescale=phi)
        return eps, lo, ro

    for phi in (0.3, 0.7, 1.0):
        a = _twice(lambda: single(phi))
        b = _twice(lambda: _gather_world1(eu, er, m, guidance, lat, (ec, ed, lat_ref), dt, phi))
        for x, y, what in zip(a, b, ("eps", "latents", "latents_ref")):
            assert torch.equal(x, y), f"gather world 1 vs single GPU, phi {phi}: {what} differs"
        assert not torch.equal(a[0], ops.region_blend_cfg(eu, er, m, guidance)), "phi > 0 left eps unchanged"

    # phi = 0 through the new entry points (raw C ABI: ops dispatches phi == 0 to the plain kernels)
    eps_old, lat_old = ops.region_blend_cfg(eu, er, m, guidance, latents=lat, dt_sigma=dt)
    eps_new, lat_new = torch.empty_like(eu), torch.empty_like(lat)
    ptrs = (ctypes.c_void_p * N)(*[e.data_ptr() for e in er])
    P = lambda t: ctypes.c_void_p(t.data_ptr())
    rc = lib.rtti_region_blend_cfg_rescale(P(eu), ptrs, P(m), N, n, guidance, P(eps_new), P(lat), P(lat_new), dt, 0.0,
                                           ops._stream())
    assert rc == 0
    assert torch.equal(eps_old, eps_new) and torch.equal(lat_old, lat_new)
    slots = torch.zeros(2, N + 3, n, dtype=torch.float16, device="cuda")
    for s, e in enumerate([eu] + er + [ec, ed]):
        slots[1, s].copy_(e)
    outs = []
    for fn in (lib.rtti_gather_blend_step, lib.rtti_gather_blend_step_rescale):
        flags = torch.zeros(16, dtype=torch.int32, device="cuda")
        o = [torch.empty_like(eu) for _ in range(3)]
        args = [(ctypes.c_void_p * 1)(slots.data_ptr()), (ctypes.c_void_p * 1)(flags.data_ptr()), 1, 0,
                (ctypes.c_int * (N + 3))(*([0] * (N + 3))), N + 3, N, P(m), n, guidance, P(o[0]), P(lat), P(o[1]),
                P(lat_ref), P(o[2]), dt, 1]
        rc = fn(*(args + ([0.0] if fn is lib.rtti_gather_blend_step_rescale else []) + [ops._stream()]))
        assert rc == 0
        torch.cuda.synchronize()
        outs.append(o)
    for x, y in zip(*outs):
        assert torch.equal(x, y), "phi = 0 gather rescale kernel differs from rtti_gather_blend_step"

    # CUDA-graph capture + replay equals eager
    eager = single(0.7)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        single(0.7)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = single(0.7)
    for _ in range(2):
        graph.replay()
        torch.cuda.synchronize()
        for x, y in zip(eager, captured):
            assert torch.equal(x, y), "graph replay differs from eager"


# ------------------------------------------------------------------------------------------------ GPU: samplers
def _close_range(got, ref, what):
    got, ref = np.asarray(got, np.float32), np.asarray(ref, np.float32)
    tol = 5e-3 * float(np.abs(ref).max()) + 3e-2 * np.abs(ref)
    err = np.abs(got - ref)
    assert np.isfinite(got).all(), f"{what}: non-finite values"
    assert (err <= tol).all(), f"{what}: {float((err > tol).mean()) * 100:.3f}% outside, max err {err.max():.4f}"
    print(f"{what}: max err {err.max():.4f} mean err {err.mean():.5f}")
    return err


def _xl_model(seed):
    from oracle import unet_oracle as uo
    from rtti_b200.region_diffusion_sdxl import RegionDiffusionXL
    from rtti_b200.unet import UNet2DConditionModel, UNetConfig
    cfg = uo.tiny_xl_config()
    unet = UNet2DConditionModel(UNetConfig.from_dict(cfg.__dict__))
    unet.load_state_dict(uo.make_state_dict(cfg, seed))
    return cfg, RegionDiffusionXL(device="cuda", unet=unet.finalize("cuda"), vae=synth.TinyVAE("cuda"))


@pytest.mark.gpu
def test_xl_plain_pass_with_rescale_vs_reference_golden():
    """The plain pass at phi = 0.7 (tiny XL, 128^2, 12 steps, g 8.5) against the reference's, at test_parity_gpu's
    latent tolerance; the phi = 0 golden lies outside that tolerance."""
    g = _golden("xl_rescale.npz")
    cfg, model = _xl_model(2)
    S = 128
    inp = synth.synth_inputs(cfg.cross_attention_dim, _pooled(cfg), 3, S, 31)
    ctx, te = inp["ctx"].cuda(), inp["text_embeds"].cuda()
    out = model.sample(height=S * 8, width=S * 8, num_inference_steps=12, guidance_scale=8.5, latents=inp["latents"].clone(),
                       prompt_embeds=ctx[-1:], negative_prompt_embeds=ctx[:1], pooled_prompt_embeds=te[-1:],
                       negative_pooled_prompt_embeds=te[:1], output_type="latent", run_rich_text=False,
                       guidance_rescale=0.7).images.float().cpu().numpy()
    _close_range(out, g["plain_latents_phi0.7"], "xl plain latents phi 0.7")
    with pytest.raises(AssertionError):
        _close_range(out, _golden("xl_loops.npz")["plain_latents"], "xl plain latents phi 0.7 vs phi 0 golden")


@pytest.mark.gpu
def test_xl_rich_loop_with_rescale_vs_oracle():
    """The rich loop at phi = 0.7 with injection, font sizes and colour guidance against the oracle's."""
    from oracle import sampler_oracle as sam, schedulers_oracle as so, unet_oracle as uo
    from tests import rescale_oracle as ro
    cfg, model = _xl_model(2)
    S = 128
    inp = synth.synth_inputs(cfg.cross_attention_dim, _pooled(cfg), 3, S, 31)
    ctx, te = inp["ctx"], inp["text_embeds"]
    tfd = synth.font_sizes()
    tfd.update(synth.color_dict(inp["masks"], S, 1.0))
    sch = so.EulerDiscreteSchedulerOracle()
    sch.set_timesteps(4)
    ref = ro.rich_text_loop(sam.make_unet_fn(uo.make_state_dict(cfg, 2), cfg), sch, ctx, inp["masks"],
                            inp["latents"].clone() * sch.init_noise_sigma, 4, 8.5,
                            added_cond={"text_embeds": te, "time_ids": inp["time_ids"]}, use_guidance=True,
                            text_format_dict=tfd, inject_selfattn=0.5, inject_background=0.5, vae_decode=synth.TinyVAE(),
                            scaling_factor=0.13025, guidance_rescale=0.7)
    model.masks = [m.cuda() for m in inp["masks"]]
    out = model.sample(height=S * 8, width=S * 8, num_inference_steps=4, guidance_scale=8.5, latents=inp["latents"].clone(),
                       prompt_embeds=ctx[1:].cuda(), negative_prompt_embeds=ctx[:1].cuda(),
                       pooled_prompt_embeds=te[1:].cuda(), negative_pooled_prompt_embeds=te[:1].cuda(),
                       output_type="latent", run_rich_text=True, use_guidance=True, inject_selfattn=0.5,
                       inject_background=0.5, text_format_dict=tfd, guidance_rescale=0.7).images
    _close_range(out.float().cpu().numpy(), ref.numpy(), "xl rich latents phi 0.7 vs oracle")


@pytest.mark.gpu
def test_rich_loop_with_rescale_two_gpus():
    """The rich loop at phi = 0.7 on the fused peer-memory exchange (tests/multigpu_rescale_check.py)."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
                        "--master-addr", "127.0.0.1", "--master-port", "29537",
                        os.path.join(ROOT, "tests", "multigpu_rescale_check.py")],
                       capture_output=True, text=True, timeout=900)
    print(r.stdout[-2000:], r.stderr[-2000:])
    assert r.returncode == 0 and "MULTIGPU_RESCALE_CHECK PASS" in r.stdout
