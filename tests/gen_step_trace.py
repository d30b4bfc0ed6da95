"""Record the exact sequence of region-blend kernel calls the samplers make, on the CPU.

`_lib.load` is replaced by a fake library whose every symbol checks its argument count against `_lib.SIGNATURES` and
records the call; the UNet is a stub that returns fp16 tensors of its input's shape. Every tensor made during a case is
kept alive, so no address is reused, and pointers are recorded as ids in order of first appearance. The result pins
which entry point each step runs, its scalars and which buffer goes where (histories, saved latents, noise draws)
for every scheduler, both samplers and the fused peer-exchange path.

    python -m tests.gen_step_trace      # rewrites tests/golden/step_trace.json
"""
import contextlib
import ctypes
import itertools
import json
import os
import sys
import types

import torch
from torch.overrides import TorchFunctionMode

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden", "step_trace.json")
STEPS = 5
LATENT = 4                   # latents [1, 4, 4, 4]
N_PROMPTS = 3                # regions + base prompt


class _Recorder(TorchFunctionMode):
    """Keeps every tensor a torch function returns alive and logs the shapes of randn draws into `events`."""

    def __init__(self, events):
        super().__init__()
        self.events, self.keep = events, []

    def __torch_function__(self, func, types_, args=(), kwargs=None):
        out = func(*args, **(kwargs or {}))
        if func is torch.randn:
            self.events.append(["randn", list(out.shape)])
        for t in (out if isinstance(out, (tuple, list)) else (out,)):
            if isinstance(t, torch.Tensor):
                self.keep.append(t)
        return out


class _FakeLib:
    """Every symbol of `_lib.SIGNATURES`: checks the argument count and appends the canonical call to `events`."""

    def __init__(self, events):
        from rtti_b200 import _lib
        self._sigs, self._events, self._ids = _lib.SIGNATURES, events, {}

    def _pid(self, p):
        p = p.value if isinstance(p, ctypes.c_void_p) else p
        if not p:
            return 0
        return self._ids.setdefault(int(p), len(self._ids) + 1)

    def _canon(self, a, ty):
        if ty is ctypes.c_void_p:
            return self._pid(a)
        if ty is ctypes.POINTER(ctypes.c_void_p):
            return [self._pid(p) for p in a]
        if ty is ctypes.POINTER(ctypes.c_int):
            return None if a is None else [int(v) for v in a]
        if ty in (ctypes.c_float, ctypes.c_double):
            return ty(a.value if isinstance(a, ty) else a).value
        return int(a.value if isinstance(a, ctypes._SimpleCData) else a)

    def __getattr__(self, name):
        _, argtypes = self._sigs[name]

        def call(*args):
            assert len(args) == len(argtypes), f"{name}: {len(args)} arguments, the signature has {len(argtypes)}"
            self._events.append([name] + [self._canon(a, ty) for a, ty in zip(args, argtypes)])
            return 0
        return call


class _StubUNet:
    config = types.SimpleNamespace(sample_size=LATENT, in_channels=4)
    in_channels = 4

    def __init__(self):
        self.outs = []

    def __call__(self, x, t, ctx, added, ctrl):
        self.outs.append(torch.full(tuple(x.shape), 0.25, dtype=torch.float16))
        return {"sample": self.outs[-1]}


class _StubExchange:
    """The fused path's PeerExchange as rank 0 of 2 sees it, without peer memory."""
    slot_ptrs, flag_ptrs, rank = [0x10000, 0x20000], [0x30000, 0x40000], 0

    def __init__(self, passes):
        self.slot_of_pass = list(range(len(passes)))
        self.step_id = 0

    def publish(self, eps_local, local, owner):
        self.step_id += 1
        return self.step_id

    def slot_owner(self, owner):
        return list(owner)


@contextlib.contextmanager
def _traced():
    from rtti_b200 import _lib, ops
    events = []
    saved = _lib.load, ops._stream, ops._req

    def req(t, dtype, name):
        if t.dtype != dtype:
            raise _lib.RttiError(f"{name} must be {dtype}, got {t.dtype}")

    _lib.load, ops._stream, ops._req = (lambda: fake), (lambda: ctypes.c_void_p(0)), req
    fake = _FakeLib(events)
    try:
        with torch.no_grad(), _Recorder(events):
            yield events
    finally:
        _lib.load, ops._stream, ops._req = saved


def _schedulers():
    from rtti_b200 import schedulers as S
    return {"euler": S.EulerDiscreteScheduler, "ancestral": S.EulerAncestralDiscreteScheduler, "ddim": S.DDIMScheduler,
            "dpm2m": S.DPMSolverMultistepScheduler, "unipc": S.UniPCMultistepScheduler, "heun": S.HeunDiscreteScheduler,
            "lms": S.LMSDiscreteScheduler, "dpm2s": S.DPMSolverSinglestepScheduler, "plms": S.PNDMScheduler}


def _inputs():
    from tests import synth
    inp = synth.synth_inputs(8, 6, N_PROMPTS, LATENT, 3)
    return {k: (v.half() if k != "masks" else v) for k, v in inp.items()}


def _xl(sched):
    from rtti_b200.region_diffusion_sdxl import RegionDiffusionXL
    model = RegionDiffusionXL(device="cpu", unet=_StubUNet(), vae=None, scheduler=_schedulers()[sched]())
    model.use_cuda_graphs = False
    model.remote_qk = False
    return model


def xl_plain(sched, phi):
    inp = _inputs()
    model = _xl(sched)
    ctx, te = inp["ctx"], inp["text_embeds"]
    with _traced() as ev:
        model.sample(height=LATENT * 8, width=LATENT * 8, num_inference_steps=STEPS, guidance_scale=7.0,
                     latents=inp["latents"], prompt_embeds=ctx[1:], negative_prompt_embeds=ctx[:1],
                     pooled_prompt_embeds=te[1:], negative_pooled_prompt_embeds=te[:1], output_type="latent",
                     guidance_rescale=phi, generator=torch.Generator().manual_seed(0))
    return ev


def xl_rich(sched, sa, bg, fused, phi):
    inp = _inputs()
    model = _xl(sched)
    model.masks = inp["masks"]
    ctx, te = inp["ctx"], inp["text_embeds"]
    with _traced() as ev:
        model.scheduler.set_timesteps(STEPS)
        st = model.prepare_rich_text(ctx, te, inp["time_ids"].float(), inp["latents"], model.scheduler.timesteps, 7.0,
                                     False, sa, bg, {}, phi, torch.Generator().manual_seed(0))
        if fused:
            st.plan.world, st.plan.rank = 2, 0
            model._exchanges[(tuple(p["kind"] for p in st.passes), st.latents[0].numel())] = _StubExchange(st.passes)
        for i in range(st.n_t):
            model.rich_text_step(st, i)
    return ev


def sd_latents(sched, inject):
    from rtti_b200.region_diffusion import RegionDiffusion
    inp = _inputs()
    model = RegionDiffusion(device="cpu", unet=_StubUNet())
    model.scheduler = _schedulers()[sched]()
    model.masks = inp["masks"]
    with _traced() as ev:
        model.produce_latents(inp["ctx"], height=LATENT * 8, width=LATENT * 8, num_inference_steps=STEPS,
                              guidance_scale=7.0, latents=inp["latents"], inject_selfattn=0.5 if inject else 0,
                              inject_background=0.5 if inject else 0)
    return ev


def sd_attn_maps(sched):
    from rtti_b200.region_diffusion import RegionDiffusion
    inp = _inputs()
    model = RegionDiffusion(device="cpu", unet=_StubUNet())
    model.scheduler = _schedulers()[sched]()
    with _traced() as ev:
        model.produce_attn_maps(None, height=LATENT * 8, width=LATENT * 8, num_inference_steps=STEPS,
                                guidance_scale=7.0, latents=inp["latents"], text_embeddings=inp["ctx"][[0, -1]],
                                decode=False)
    return ev


XL = ("euler", "ancestral", "ddim", "dpm2m", "unipc", "heun", "lms", "dpm2s")
SD = ("plms", "ddim", "dpm2m", "unipc", "dpm2s")
INJECT = ((0.5, 0.5), (0.0, 0.5), (0.0, 0.0))


def cases():
    """name -> zero-argument function that returns the case's trace."""
    out = {}
    for s in XL:
        for phi in (0.0, 0.7):
            out[f"xl_plain/{s}/phi={phi}"] = lambda s=s, phi=phi: xl_plain(s, phi)
        for sa, bg in INJECT:
            for fused, phi in itertools.product((False, True), (0.0, 0.7)):
                name = f"xl_rich/{s}/sa={sa},bg={bg}/{'fused' if fused else 'split'}/phi={phi}"
                out[name] = lambda s=s, sa=sa, bg=bg, fused=fused, phi=phi: xl_rich(s, sa, bg, fused, phi)
    for s in SD:
        for inject in (True, False):
            out[f"sd_latents/{s}/inject={inject}"] = lambda s=s, inject=inject: sd_latents(s, inject)
        out[f"sd_attn_maps/{s}"] = lambda s=s: sd_attn_maps(s)
    return out


def main():
    golden = {name: fn() for name, fn in cases().items()}
    with open(GOLDEN, "w") as f:
        f.write("{\n" + ",\n".join(f"{json.dumps(k)}: [\n" + ",\n".join("  " + json.dumps(e) for e in v) + "\n]"
                                   for k, v in golden.items()) + "\n}\n")
    print(f"wrote {GOLDEN}: {len(golden)} cases, {sum(map(len, golden.values()))} events")


if __name__ == "__main__":
    main()
