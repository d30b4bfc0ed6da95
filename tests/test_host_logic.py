"""CPU: host-side logic, the C-ABI surface (load + exported symbols, no compute) and the schedulers."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
    from rtti_b200 import _lib
    header = open(os.path.join(ROOT, "include", "rtti_b200.h")).read()
    declared = set(re.findall(r"\b(rtti_[a-z0-9_]+)\s*\(", header))
    assert declared, "no declarations parsed"
    assert declared == set(_lib.SIGNATURES), f"header vs binding mismatch: {declared ^ set(_lib.SIGNATURES)}"
    lib = _lib.load()
    for name in declared:
        assert getattr(lib, name) is not None
    assert lib.rtti_version() >= 100
    # pure host-side queries work without a GPU
    assert lib.rtti_groupnorm_workspace_elems(2, 4096, 640, 32) > 0
    assert lib.rtti_color_loss_workspace_elems(2, 1024 * 1024) > 0


_C_ABI = {"int": "int32", "int32_t": "int32", "long long": "int64", "int64_t": "int64", "unsigned": "uint32",
          "unsigned int": "uint32", "uint32_t": "uint32", "unsigned long long": "uint64", "uint64_t": "uint64",
          "size_t": "uint64", "float": "float", "double": "double"}


def _c_abi(decl):
    """ABI class of a C type, with or without a parameter name."""
    if "*" in decl:
        return "pointer"
    words = [w for w in decl.split() if w != "const"]
    base = " ".join(words[:-1]) if len(words) > 1 and " ".join(words) not in _C_ABI else " ".join(words)
    return _C_ABI[base]


def _ctypes_abi(ty):
    if ty is ctypes.c_void_p or issubclass(ty, ctypes._Pointer):
        return "pointer"
    if ty in (ctypes.c_float, ctypes.c_double):
        return ty.__name__[2:]
    return ("int" if ty(-1).value < 0 else "uint") + str(8 * ctypes.sizeof(ty))


def test_binding_argument_types_match_the_header():
    """Every prototype of the header against _lib.SIGNATURES, parameter by parameter: a miscounted or misplaced float
    or pointer would otherwise only show as wrong arguments on the GPU."""
    from rtti_b200 import _lib
    header = open(os.path.join(ROOT, "include", "rtti_b200.h")).read()
    header = re.sub(r"/\*.*?\*/|//[^\n]*|^\s*#[^\n]*", "", header, flags=re.S | re.M)
    protos = re.findall(r"([A-Za-z_][\w\s]*?)\s+(rtti_\w+)\s*\(([^)]*)\)\s*;", header)
    assert len(protos) == len(_lib.SIGNATURES)
    for ret, name, params in protos:
        params = [] if params.strip() in ("", "void") else [p.strip() for p in params.split(",")]
        restype, argtypes = _lib.SIGNATURES[name]
        assert _c_abi(ret) == _ctypes_abi(restype), name
        assert [_c_abi(p) for p in params] == [_ctypes_abi(t) for t in argtypes], name


def test_tensor_core_kernels_fit_the_launch_time_register_check():
    """The hardware verifies a launch's register demand with the CTA's warp count rounded up to the 4 SM sub-partitions
    (cuda_occupancy.h, "Hardware check"): a 9-warp CTA is checked as 12 warps. A kernel over the limit compiles and
    links but every launch fails with cudaErrorLaunchOutOfResources — found only on the GPU (round 2: attn_cross at
    9 warps x 210 registers). Checked here from the cubin resource usage, no GPU needed."""
    import shutil
    import subprocess
    from rtti_b200 import _lib
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    _lib.load()
    out = subprocess.run(["cuobjdump", "-res-usage", _lib.LIB_PATH], capture_output=True, text=True).stdout
    threads = {"attn_fwd_kernel": 256, "attn_probs_mean": 256, "ff_geglu_kernel": 256}
    seen = set()
    for fn, regs in re.findall(r"Function (\S+):\s*\n\s*REG:(\d+)", out):
        for key, nthreads in threads.items():
            if key in fn:
                seen.add(key)
                warps = (nthreads + 31) // 32
                per_warp = (int(regs) * 32 + 255) // 256 * 256
                assumed = per_warp * ((warps + 3) // 4 * 4)
                assert assumed <= 65536, f"{fn}: {regs} registers x {warps} warps is checked as {assumed} > 65536 registers"
    assert seen == set(threads), f"kernels not found in the library: {set(threads) - seen}"


def test_fp16_hbm_kernels_use_128_bit_global_accesses():
    """Round 2 found (ncu + SASS) that `*reinterpret_cast<const Half8*>(p)` had been lowered to FOUR 32-bit LDG/STG in
    every fp16 elementwise kernel. Checked from the cubin: the streaming kernels must move their tensors with
    LDG.E.128 / STG.E.128 and contain no plain 32-bit global store."""
    import shutil
    import subprocess
    from rtti_b200 import _lib
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    _lib.load()
    sass = subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True).stdout
    funcs = re.split(r"\n\s*Function : ", sass)[1:]
    want = ("layernorm_kernelILi5", "add_bias_layernorm_kernelILi5", "add_bias_layernorm_kernelILi3", "add_bias_f16_kernel",
            "4rtti12geglu_kernel", "gn_apply_kernel")
    seen = set()
    for f in funcs:
        name = f.split("\n", 1)[0]
        for w in want:
            if w in name:
                seen.add(w)
                assert re.search(r"\bLDG\.E\.128", f) and re.search(r"\bSTG\.E\.128", f), f"{name}: no 128-bit global accesses"
                assert not re.search(r"\bSTG\.E\s", f), f"{name}: 32-bit global stores"
    assert seen == set(want), f"kernels not found: {set(want) - seen}"


def test_ops_fail_loudly_without_gpu_or_library():
    from rtti_b200 import _lib, ops
    x = torch.zeros(1, 16, 64, dtype=torch.float16)
    with pytest.raises(_lib.RttiError):
        ops.attention(x, x, x, 1)          # CPU tensors: there is no CPU path
    saved, _lib._lib = _lib._lib, None
    saved_path, _lib.LIB_PATH = _lib.LIB_PATH, "/nonexistent/librtti_b200.so"
    try:
        with pytest.raises(_lib.RttiError):
            _lib.load()
    finally:
        _lib._lib, _lib.LIB_PATH = saved, saved_path


def test_pass_assignment_plans():
    from rtti_b200.region_parallel import assign_passes
    for n_regions in (1, 3, 5, 8, 10):
        kinds = ["A", "B", "C", "D"] + ["E"] * (n_regions - 1)
        for world in (1, 2, 4, 8):
            for feat in (False, True):
                assign, owner = assign_passes(kinds, world, feat)
                covered = sorted(set(p for a in assign for p in a))
                assert covered == list(range(len(kinds)))
                for p, o in enumerate(owner):
                    assert p in assign[o]
                for r, a in enumerate(assign):
                    if feat and any(kinds[p] == "E" for p in a):
                        assert kinds.index("D") in a, "E passes need the reference pass D on the same rank"
                    if not feat:
                        assert len(a) == len(set(a))
                if not feat:
                    assert sum(len(a) for a in assign) == len(kinds)
                    assert max(len(a) for a in assign) == -(-len(kinds) // world)
    assign, _ = assign_passes(list("ABCDEEEE"), 2, True)
    assert max(len(a) for a in assign) == 5


def test_remote_qk_assignment_roles_and_layout():
    """remote_qk: pass D runs on one rank and its Q|K / feature travel to the region-pass ranks, so the passes of an
    injection step are spread evenly (round 1 replicated D: 2 passes on the busiest of 8 ranks for the 8-pass step)."""
    from rtti_b200.region_parallel import RegionParallelPlan, assign_passes
    from rtti_b200.unet import UNet2DConditionModel, UNetConfig
    for n_regions in (3, 5, 8, 10):
        kinds = ["A", "B", "C", "D"] + ["E"] * (n_regions - 1)
        for world in (2, 4, 8):
            assign, owner = assign_passes(kinds, world, True, remote_qk=True)
            assert sorted(p for a in assign for p in a) == list(range(len(kinds))), "every pass exactly once"
            assert max(len(a) for a in assign) == -(-len(kinds) // world)
            assert all(a == sorted(a) for a in assign)
            roles = []
            for r in range(world):
                plan = RegionParallelPlan([dict(kind=k) for k in kinds], True, remote_qk=True)
                plan.world, plan.rank = world, r                       # no process group in this test
                local = plan.local_passes(True)
                role = plan.remote_role(local)
                roles.append(role)
                src = plan.injection_sources(local)
                has_d = kinds.index("D") in local
                has_e = any(kinds[p] == "E" for p in local)
                if has_e and not has_d:
                    assert role[0] == "dst" and src is None
                    assert [kinds[p] for p in local[role[1]:]] == ["E"] * (len(local) - role[1])
                elif has_d:
                    assert src is not None and all(src[k] == local.index(kinds.index("D")) for k, p in enumerate(local) if kinds[p] == "E")
            srcs = [r for r in roles if r is not None and r[0] == "src"]
            dsts = [i for i, r in enumerate(roles) if r is not None and r[0] == "dst"]
            if dsts:
                assert len(srcs) == 1 and srcs[0][2] == dsts
            else:
                assert not srcs
    # the 8-pass SDXL step on 8 ranks: one pass per rank
    assign, owner = assign_passes(list("ABCDEEEE"), 8, True, remote_qk=True)
    assert [len(a) for a in assign] == [1] * 8
    # layout: SDXL has 70 self-attention layers (10 at 64^2 with C=640, 60 at 32^2 with C=1280) + the injected feature
    with torch.device("meta"):
        unet = UNet2DConditionModel(UNetConfig.sdxl())
    lay = unet.injection_layout(128, 128)
    assert len(lay) == 71
    assert sorted(set(lay)) == [(1024, 2560), (4096, 640), (4096, 1280)]
    assert lay.count((4096, 1280)) == 10 and lay.count((1024, 2560)) == 60 and lay.count((4096, 640)) == 1
    assert sum(r * w * 2 for r, w in lay) == 10 * 4096 * 1280 * 2 + 60 * 1024 * 2560 * 2 + 4096 * 640 * 2


def test_injection_sources():
    from rtti_b200.region_parallel import RegionParallelPlan
    passes = [dict(kind=k) for k in "ABCDEE"]
    plan = RegionParallelPlan(passes, True)
    local = plan.local_passes(True)
    assert local == [0, 1, 2, 3, 4, 5]
    assert plan.injection_sources(local) == [0, 1, 2, 3, 3, 3]


def test_schedulers_match_oracle_restatement():
    from oracle import schedulers_oracle as so
    from rtti_b200.schedulers import EulerDiscreteScheduler, PNDMScheduler
    e, eo = EulerDiscreteScheduler(), so.EulerDiscreteSchedulerOracle()
    e.set_timesteps(41); eo.set_timesteps(41)
    np.testing.assert_allclose(e.timesteps.numpy(), eo.timesteps.numpy())
    np.testing.assert_allclose(e.sigmas_host, eo.sigmas.numpy(), rtol=1e-6)
    assert abs(e.init_noise_sigma - float(eo.init_noise_sigma)) < 1e-5
    g = torch.Generator().manual_seed(0)
    x, eps = torch.randn(1, 4, 8, 8, generator=g), torch.randn(1, 4, 8, 8, generator=g)
    t = e.timesteps[3]
    np.testing.assert_allclose(e.step(eps, t, x)["prev_sample"].numpy(), eo.step(eps, t, x)["prev_sample"].numpy(), atol=1e-5)
    np.testing.assert_allclose(e.scale_model_input(x, t).numpy(), eo.scale_model_input(x, t).numpy(), atol=1e-6)
    p, po = PNDMScheduler(), so.PNDMSchedulerOracle()
    p.set_timesteps(10); po.set_timesteps(10)
    assert p.timesteps.tolist() == po.timesteps.tolist() and len(p.timesteps) == 11
    xa, xb = x.clone(), x.clone()
    for t in p.timesteps:
        eps = torch.randn(1, 4, 8, 8, generator=g)
        xa = p.step(eps, t, xa)["prev_sample"]
        xb = po.step(eps, t, xb)["prev_sample"]
    np.testing.assert_allclose(xa.numpy(), xb.numpy(), atol=1e-5)


def test_schedulers_known_answers_and_analytic_properties():
    """The scheduler arithmetic is third-party (diffusers 0.18.2, not in the reference tree). Checks that do NOT rest on
    the repo's own restatement: (i) the published constants of the Stable Diffusion noise schedule (scaled-linear betas
    0.00085..0.012, 1000 steps: sigma_min 0.0292, sigma_max 14.6146 as quoted by k-diffusion / the SD model cards);
    (ii) Euler discrete integrates dx/dsigma = eps exactly for a constant eps: x_final = x_0 - eps * sigma_0 for any
    number of steps (telescoping); (iii) PLMS / DDIM transfer: with a constant eps the sample stays on the ray
    x_t = sqrt(a_t) x0 + sqrt(1 - a_t) eps, so after ALL steps it must equal sqrt(a_f) x0 + sqrt(1 - a_f) eps with
    a_f the cumulative alpha reached by the last step (the multistep combinations 3/2,-1/2 ... have coefficient sum 1)."""
    from rtti_b200.schedulers import EulerDiscreteScheduler, PNDMScheduler
    e = EulerDiscreteScheduler()
    ac = e.alphas_cumprod.double()
    sig = ((1 - ac) / ac).sqrt()
    assert abs(float(sig[-1]) - 14.6146) < 2e-3 and abs(float(sig[0]) - 0.0292) < 1e-4
    assert abs(float(ac[0]) - 0.99915) < 1e-6 and abs(float(ac[-1]) - 0.004660) < 2e-5
    g = torch.Generator().manual_seed(1)
    x0, eps = torch.randn(1, 4, 8, 8, generator=g), torch.randn(1, 4, 8, 8, generator=g)
    for n in (7, 41, 50):
        e.set_timesteps(n)
        assert float(e.timesteps[0]) == (n - 1) * (1000 // n) + 1 and float(e.timesteps[-1]) == 1.0   # `leading`, offset 1
        s0 = e.sigma(e.timesteps[0])
        x = x0 * e.init_noise_sigma
        for t in e.timesteps:
            x = e.step(eps, t, x)["prev_sample"]
        np.testing.assert_allclose(x.numpy(), (x0 * e.init_noise_sigma - eps * s0).numpy(), atol=2e-5)
        assert abs(e.init_noise_sigma - (s0 * s0 + 1) ** 0.5) < 1e-6
        xs = e.scale_model_input(x0, e.timesteps[0])
        np.testing.assert_allclose(xs.numpy(), (x0 / (s0 * s0 + 1) ** 0.5).numpy(), atol=1e-6)
    p = PNDMScheduler()
    acp = p.alphas_cumprod.double()
    for n in (10, 41):
        p.set_timesteps(n)
        ts = p.timesteps.tolist()
        assert len(ts) == n + 1 and ts[0] == (n - 1) * (1000 // n) + 1 and ts[-1] == 1
        a0 = float(acp[ts[0]])
        x = (a0 ** 0.5) * x0 + ((1 - a0) ** 0.5) * eps
        for t in p.timesteps:
            x = p.step(eps, t, x)["prev_sample"]
        prev = ts[-1] - 1000 // n                      # the last transfer goes to t = 1 - ratio < 0 -> final_alpha_cumprod
        af = float(acp[prev]) if prev >= 0 else float(acp[0])
        want = (af ** 0.5) * x0 + ((1 - af) ** 0.5) * eps
        np.testing.assert_allclose(x.numpy(), want.numpy(), atol=5e-5)


def test_token_map_accumulator_call_counting():
    from rtti_b200.unet import TokenMapAccumulator
    acc = TokenMapAccumulator(["c"], self_layers=["s"], start_after=2, sd_overwrite_bug=True, self_resolutions=None)
    assert acc.cross_target("c", 16, 77, "cpu") is None and acc.cross_target("c", 16, 77, "cpu") is None
    t = acc.cross_target("c", 16, 77, "cpu")
    assert t is not None and t.shape == (1, 16, 77) and acc.n_maps["c"] == 3
    assert acc.cross_target("other", 16, 77, "cpu") is None
    for _ in range(2):
        assert acc.self_target("s", 16, "cpu") is None
    s = acc.self_target("s", 16, "cpu")
    s += 1.0
    s2 = acc.self_target("s", 16, "cpu")   # 's' is never in crossattn_maps -> overwritten (reference quirk)
    assert s2 is s and float(s2.sum()) == 0.0


def test_richtext_parse_and_region_inputs():
    from rtti_b200 import richtext_utils as ru

    class Tok:
        def _tokenize(self, text):
            return text.lower().split()

    class M:
        tokenizer = Tok()

    delta = {"ops": [{"insert": "a church "}, {"attributes": {"color": "#fd6c9e"}, "insert": "garden"},
                     {"insert": " with "}, {"attributes": {"font": "slabo"}, "insert": "mountains"},
                     {"attributes": {"size": "60px"}, "insert": " snowy"}, {"attributes": {"link": "a red sun"}, "insert": " sky"},
                     {"insert": "\n"}]}
    base, styles, notes, note_t, cspans, cnames, crgbs, sizes, use_grad = ru.parse_json(delta, device="cpu")
    assert base == "a church garden with mountains snowy sky"
    assert styles == ["mountains in the style of Vincent Van Gogh"] and notes == ["a red sun"] and note_t == [" sky"]
    assert cspans == ["garden"] and cnames == ["pink"] and use_grad and sizes == [[" snowy", 20.0]]
    prompts, ids, base_tokens = ru.get_region_diffusion_input(M(), base, styles, notes, note_t, cspans, cnames)
    assert prompts == ["mountains in the style of Vincent Van Gogh", "a red sun", "pink garden", base]
    assert [i.tolist() for i in ids] == [[5], [7], [3], [1, 2, 4, 6]]
    tfd = ru.get_attention_control_input(M(), base_tokens, sizes, device="cpu")
    assert tfd["word_pos"].tolist() == [6] and tfd["font_size"].tolist() == [20.0]
    tfd, cids = ru.get_gradient_guidance_input(M(), base_tokens, cspans, crgbs, tfd, color_guidance_weight=0.5)
    assert [i.tolist() for i in cids] == [[3], [1, 2, 4, 5, 6, 7]] and tfd["color_guidance_weight"] == 0.5
    assert ru.find_nearest_color([250, 10, 5]) == "red"


def test_c_abi_rejects_bad_arguments_without_launching():
    """Error behaviour of the boundary (include/rtti_b200.h): bad pointers / shapes / alignment return the documented
    negative code before any CUDA call — checked through raw ctypes, which is what a foreign-language binding would do."""
    import ctypes
    from rtti_b200 import _lib
    lib = _lib.load()
    V = ctypes.c_void_p
    buf = (ctypes.c_char * 4096)()
    a = (ctypes.addressof(buf) + 15) // 16 * 16
    ARG, SHAPE, ALIGN = -1, -2, -3
    # rtti_halo_exchange(pad_local, pad_up, pad_down, rows, row_elems, flags_local, flags_up, flags_down, seq, stream)
    assert lib.rtti_halo_exchange(V(0), V(0), V(0), 4, 64, V(a), V(0), V(0), 1, V(0)) == ARG
    assert lib.rtti_halo_exchange(V(a), V(0), V(0), 4, 6, V(a), V(0), V(0), 1, V(0)) == SHAPE
    assert lib.rtti_halo_exchange(V(a + 4), V(0), V(0), 4, 64, V(a), V(0), V(0), 1, V(0)) == ALIGN
    assert lib.rtti_halo_exchange(V(a), V(a), V(0), 4, 64, V(a), V(0), V(0), 1, V(0)) == ARG      # neighbour without flags
    peers = (V * 2)(V(a), V(a))
    gn = lambda hw_local, hw_total, c, groups, world, rank: lib.rtti_gn32_silu_fwd_striped(
        V(a), V(0), V(a), V(a), V(a), V(a), V(a), hw_local, hw_total, c, groups, 1e-6, 1, peers, peers, world, rank, 1, V(0))
    assert gn(16, 32, 256, 64, 2, 0) == SHAPE      # more than 32 groups
    assert gn(16, 32, 64, 32, 2, 2) == ARG         # rank outside the world
    assert gn(16, 8, 64, 32, 2, 0) == ARG          # stripe larger than the tensor
    assert gn(16, 32, 66, 33, 2, 0) == SHAPE       # channels not a multiple of 4
    assert lib.rtti_add_bias_f32(V(a), V(a), V(0), V(a), 4, 6, V(0)) == SHAPE
    assert lib.rtti_add_bias_f32(V(0), V(a), V(0), V(a), 4, 8, V(0)) == ARG
    # rtti_gather_blend_step(peer_slots, peer_flags, world, rank, slot_owner, n_slots, n_regions, masks, n, ...)
    owner = (ctypes.c_int * 4)(0, 0, 1, 1)
    gb = lambda world, rank, n: lib.rtti_gather_blend_step(peers, peers, world, rank, owner, 4, 3, V(a), n, 7.5, V(a), V(0), V(0),
                                                            V(0), V(0), -0.1, 1, V(0))
    assert gb(17, 0, 64) == ARG                    # more ranks than the kernel's table
    assert gb(2, 0, 60) == SHAPE                   # n not a multiple of 8
    assert lib.rtti_version() >= 100


def test_pass_batch_matches_the_reference_call_sequence():
    """models/region_diffusion_sdxl.py:787-821 runs 2 + 2*inject + (N-1) UNet calls per step: uncond and base prompt on
    the latents, (uncond, base) on the reference latents when injecting, one call per region prompt."""
    from rtti_b200.region_diffusion_sdxl import RegionDiffusionXL
    for n_regions in (1, 3, 5, 8, 10):
        for inject in (False, True):
            passes = RegionDiffusionXL.build_pass_batch(None, n_regions, inject)
            assert len(passes) == 2 + 2 * inject + (n_regions - 1)
            kinds = "".join(p["kind"] for p in passes)
            assert kinds == "AB" + ("CD" if inject else "") + "E" * (n_regions - 1)
            assert [p["ctx"] for p in passes if p["kind"] in "AC"] == [0] * (1 + inject)          # unconditional row
            assert all(p["ctx"] == n_regions for p in passes if p["kind"] in "BD")                # base prompt = last row
            assert [p["ctx"] for p in passes if p["kind"] == "E"] == list(range(1, n_regions))    # region prompts in order
            assert [p["ref"] for p in passes] == [p["kind"] in "CD" for p in passes]              # reference-latent passes
    assert len(RegionDiffusionXL.build_pass_batch(None, 5, True)) == 8        # bench.py's workload
