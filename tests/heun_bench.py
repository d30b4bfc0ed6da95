"""Cost of the second-stage Heun blend against the Euler blend, on one GPU:

    python tests/heun_bench.py [--launches 2000] [--out DIR]

At the SDXL 1024^2 shape (n = 65536 latent elements, 5 regions), guidance_rescale 0 and 0.7, with and without the
reference-latent pair C/D: rtti_region_blend_cfg(_rescale) vs its _heun form at a second stage (with C/D: plus the C/D
call, as the single-GPU rich loop runs it), and rtti_gather_blend_step(_rescale) vs its _heun form at world 1 (this
device's slot buffer is the only peer; with C/D it also writes eps_ref_out). A second stage reads the saved latents xs
and prediction ds of each trajectory it steps, two fp16 tensors more than Euler. Launches are captured in CUDA graphs
of 100 and timed with CUDA events over >= 1000 launches after a warm-up. Heun runs 2N - 1 UNet evaluations for N
steps: compare whole runs at equal evaluation counts, not equal step counts.
Prints the card name and power limit, then the numbers; with --out also writes them as JSON there."""
import argparse
import ctypes
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests.guidance_rescale_bench import card, time_graph  # noqa: E402


def kernel_rows(lib, ops, launches):
    from rtti_b200.schedulers import HeunDiscreteScheduler
    s = HeunDiscreteScheduler()
    s.set_timesteps(20)
    cx, ce, cs, cd = s.heun_coeffs(13)
    assert cs != 0.0 and cd != 0.0
    n, N = 65536, 5
    P = lambda t: ctypes.c_void_p(t.data_ptr())
    st = ops._stream
    g = torch.Generator(device="cuda").manual_seed(N)
    n_slots = N + 3
    slots = torch.randn(2, n_slots, n, device="cuda", generator=g).half()
    flags = torch.zeros(16, dtype=torch.int32, device="cuda")
    m = torch.softmax(torch.randn(N, n, device="cuda", generator=g), 0).contiguous()
    ones = torch.ones(1, n, device="cuda")
    lat, lat_ref = torch.randn(n, device="cuda", generator=g).half(), torch.randn(n, device="cuda", generator=g).half()
    xs, ds = torch.randn(2, n, device="cuda", generator=g).half(), torch.randn(2, n, device="cuda", generator=g).half()
    o = [torch.empty(n, dtype=torch.float16, device="cuda") for _ in range(5)]
    regions = (ctypes.c_void_p * N)(*[slots[1, 1 + i].data_ptr() for i in range(N)])
    ref_d = (ctypes.c_void_p * 1)(slots[1, N + 2].data_ptr())
    base = [P(slots[1, 0]), regions, P(m), N, n, 8.5, P(o[0]), P(lat), P(o[1])]
    ref_args = [P(slots[1, N + 1]), ref_d, P(ones), 1, n, 8.5, P(o[2]), P(lat_ref), P(o[3])]
    peer = (ctypes.c_void_p * 1)(slots.data_ptr())
    fl = (ctypes.c_void_p * 1)(flags.data_ptr())
    owner = (ctypes.c_int * n_slots)(*([0] * n_slots))

    def single(phi, heun, cd_pair):
        def step():
            for k, a in enumerate((base, ref_args)[:2 if cd_pair else 1]):
                if heun:
                    h = [cx, ce, cs, cd, P(xs[k]), P(ds[k])]
                    rc = (lib.rtti_region_blend_cfg_heun(*a, *h, st()) if phi == 0 else
                          lib.rtti_region_blend_cfg_rescale_heun(*a, *h, phi, st()))
                else:
                    rc = (lib.rtti_region_blend_cfg(*a, 2 * ce, st()) if phi == 0 else
                          lib.rtti_region_blend_cfg_rescale(*a, 2 * ce, phi, st()))
                assert rc == 0
        return step

    def gather(phi, heun, cd_pair):
        def step():
            a = [peer, fl, 1, 0, owner, n_slots, N, P(m), n, 8.5, P(o[0]), P(lat), P(o[1])]
            a += [P(lat_ref), P(o[3])] if cd_pair else [None, None]
            if heun:
                a += [cx, ce, cs, cd, P(xs[0]), P(ds[0])]
                a += [P(xs[1]), P(ds[1]), P(o[4])] if cd_pair else [None, None, None]
                a += [1]
                rc = (lib.rtti_gather_blend_step_heun(*a, st()) if phi == 0 else
                      lib.rtti_gather_blend_step_rescale_heun(*a, phi, st()))
            else:
                a += [2 * ce, 1]
                rc = (lib.rtti_gather_blend_step(*a, st()) if phi == 0 else
                      lib.rtti_gather_blend_step_rescale(*a, phi, st()))
            assert rc == 0
        return step

    rows = []
    for entry, fn in (("region_blend_cfg", single), ("gather_blend_step, world 1", gather)):
        for cd_pair in (False, True):
            for phi in (0.0, 0.7):
                res = {h: time_graph(fn(phi, h, cd_pair), launches) for h in (False, True)}
                rows.append(dict(entry=entry, n=n, N=N, cd=cd_pair, phi=phi, us_euler=res[False], us_heun=res[True]))
                print(f"{entry:27s} n={n} N={N} C/D={'yes' if cd_pair else 'no ':3s} phi={phi:g}: "
                      f"Euler {res[False]:7.2f} us   Heun second stage {res[True]:7.2f} us", flush=True)
    return rows


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
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "heun_bench.json"), "w") as f:
            json.dump({"card": name, "power_limit": pl, "kernels": rows}, f, indent=1)


if __name__ == "__main__":
    main()
