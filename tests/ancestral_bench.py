"""Cost of the Euler Ancestral blend entry points against their Euler counterparts, and of drawing the noise, on one GPU:

    python tests/ancestral_bench.py [--launches 2000] [--out DIR]

1. Kernel time at the SDXL 128^2 latent (n = 65536), N = 5 and 10 regions, guidance_rescale 0 and 0.7, with and
   without the reference-latent pair C/D: rtti_region_blend_cfg(_rescale) vs its _anc form (with C/D: plus the C/D call,
   as the single-GPU rich loop runs it), and rtti_gather_blend_step(_rescale) vs its _anc form at world 1 (this device's
   slot buffer is the only peer). The ancestral cases take a step with s_up != 0, so the noise is read. Launches are
   captured in CUDA graphs of 100 and timed with CUDA events over >= 1000 launches.
2. The noise draw of one rich-text step, [2, 4, 128, 128] fp16: from the device's global RNG (CUDA events over 200
   draws), and from a CPU generator plus the host-to-device copy (host clock around 200 draws, each ending in a device
   synchronise).
Prints the card name and power limit, then the numbers; with --out also writes them as JSON there."""
import argparse
import ctypes
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests.guidance_rescale_bench import card, time_graph  # noqa: E402


def kernel_rows(lib, ops, launches):
    from rtti_b200.schedulers import EulerAncestralDiscreteScheduler
    s = EulerAncestralDiscreteScheduler()
    s.set_timesteps(41)
    dt, s_up = s.ancestral_coeffs(20)
    assert s_up > 0
    n = 65536
    P = lambda t: ctypes.c_void_p(t.data_ptr())
    st = ops._stream
    rows = []
    for N in (5, 10):
        g = torch.Generator(device="cuda").manual_seed(N)
        n_slots = N + 3
        slots = torch.randn(2, n_slots, n, device="cuda", generator=g).half()
        flags = torch.zeros(16, dtype=torch.int32, device="cuda")
        m = torch.softmax(torch.randn(N, n, device="cuda", generator=g), 0).contiguous()
        ones = torch.ones(1, n, device="cuda")
        lat, lat_ref = torch.randn(n, device="cuda", generator=g).half(), torch.randn(n, device="cuda", generator=g).half()
        z = torch.randn(2, n, device="cuda", generator=g).half()
        o = [torch.empty(n, dtype=torch.float16, device="cuda") for _ in range(4)]
        regions = (ctypes.c_void_p * N)(*[slots[1, 1 + i].data_ptr() for i in range(N)])
        ref_d = (ctypes.c_void_p * 1)(slots[1, N + 2].data_ptr())
        base = [P(slots[1, 0]), regions, P(m), N, n, 8.5, P(o[0]), P(lat), P(o[1])]
        ref_args = [P(slots[1, N + 1]), ref_d, P(ones), 1, n, 8.5, P(o[2]), P(lat_ref), P(o[3])]
        peer = (ctypes.c_void_p * 1)(slots.data_ptr())
        fl = (ctypes.c_void_p * 1)(flags.data_ptr())
        owner = (ctypes.c_int * n_slots)(*([0] * n_slots))

        def single(phi, anc, cd):
            def step():
                for a, zz in ((base, z[0]), (ref_args, z[1]))[:2 if cd else 1]:
                    if anc:
                        rc = (lib.rtti_region_blend_cfg_anc(*a, dt, s_up, P(zz), st()) if phi == 0 else
                              lib.rtti_region_blend_cfg_rescale_anc(*a, dt, s_up, P(zz), phi, st()))
                    else:
                        rc = (lib.rtti_region_blend_cfg(*a, dt, st()) if phi == 0 else
                              lib.rtti_region_blend_cfg_rescale(*a, dt, phi, st()))
                    assert rc == 0
            return step

        def gather(phi, anc, cd):
            def step():
                a = [peer, fl, 1, 0, owner, n_slots, N, P(m), n, 8.5, P(o[0]), P(lat), P(o[1])]
                a += [P(lat_ref), P(o[3])] if cd else [None, None]
                if anc:
                    a += [dt, s_up, P(z[0]), P(z[1]) if cd else None, 1]
                    rc = (lib.rtti_gather_blend_step_anc(*a, st()) if phi == 0 else
                          lib.rtti_gather_blend_step_rescale_anc(*a, phi, st()))
                else:
                    a += [dt, 1]
                    rc = (lib.rtti_gather_blend_step(*a, st()) if phi == 0 else
                          lib.rtti_gather_blend_step_rescale(*a, phi, st()))
                assert rc == 0
            return step

        for entry, fn in (("region_blend_cfg", single), ("gather_blend_step, world 1", gather)):
            for cd in (False, True):
                for phi in (0.0, 0.7):
                    res = {anc: time_graph(fn(phi, anc, cd), launches) for anc in (False, True)}
                    rows.append(dict(entry=entry, n=n, N=N, cd=cd, phi=phi, us_euler=res[False], us_anc=res[True]))
                    print(f"{entry:27s} n={n} N={N:2d} C/D={'yes' if cd else 'no ':3s} phi={phi:g}: "
                          f"Euler {res[False]:7.2f} us   ancestral {res[True]:7.2f} us", flush=True)
    return rows


def draw_rows(reps=200):
    from rtti_b200.schedulers import EulerAncestralDiscreteScheduler as A
    shape, dev = (2, 4, 128, 128), torch.device("cuda", torch.cuda.current_device())
    for _ in range(10):
        A.noise(shape, None, dev)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        A.noise(shape, None, dev)
    e1.record()
    torch.cuda.synchronize()
    device_us = e0.elapsed_time(e1) * 1e3 / reps
    g = torch.Generator().manual_seed(0)
    for _ in range(10):
        A.noise(shape, g, dev)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        A.noise(shape, g, dev)
        torch.cuda.synchronize()
    cpu_us = (time.perf_counter() - t0) * 1e6 / reps
    print(f"noise draw {shape} fp16: device RNG {device_us:.2f} us, CPU generator + copy {cpu_us:.1f} us", flush=True)
    return dict(shape=list(shape), device_rng_us=device_us, cpu_generator_and_copy_us=cpu_us)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=2000)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from rtti_b200 import _lib, ops
    lib = _lib.load()
    name, pl = card()
    print(f"card: {name}, power limit {pl}", flush=True)
    rows = kernel_rows(lib, ops, args.launches)
    draws = draw_rows()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "ancestral_bench.json"), "w") as f:
            json.dump({"card": name, "power_limit": pl, "kernels": rows, "noise_draw": draws}, f, indent=1)


if __name__ == "__main__":
    main()
