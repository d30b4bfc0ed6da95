"""Cost of the order-4 LMS blend against the Euler blend, on one GPU:

    python tests/lms_bench.py [--launches 2000] [--out DIR]

At the SDXL 1024^2 shape (n = 65536 latent elements, 5 regions), guidance_rescale 0 and 0.7, with and without the
reference-latent pair C/D: rtti_region_blend_cfg(_rescale) vs its _lms form at order 4 (with C/D: plus the C/D call, as
the single-GPU rich loop runs it), and rtti_gather_blend_step(_rescale) vs its _lms form at world 1 (this device's slot
buffer is the only peer; with C/D it also writes eps_ref_out). An order-4 step reads the fp16 predictions d1, d2, d3 of
each trajectory it steps, three fp16 tensors more than Euler. Launches are captured in CUDA graphs of 100 and timed with
CUDA events over >= 1000 launches after a warm-up.
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
    from rtti_b200.schedulers import LMSDiscreteScheduler
    s = LMSDiscreteScheduler()
    s.set_timesteps(20)
    c = s.lms_coeffs(12)
    assert all(x != 0.0 for x in c)
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
    hist = torch.randn(2, 3, n, device="cuda", generator=g).half()   # [trajectory, d1..d3]
    o = [torch.empty(n, dtype=torch.float16, device="cuda") for _ in range(5)]
    regions = (ctypes.c_void_p * N)(*[slots[1, 1 + i].data_ptr() for i in range(N)])
    ref_d = (ctypes.c_void_p * 1)(slots[1, N + 2].data_ptr())
    base = [P(slots[1, 0]), regions, P(m), N, n, 8.5, P(o[0]), P(lat), P(o[1])]
    ref_args = [P(slots[1, N + 1]), ref_d, P(ones), 1, n, 8.5, P(o[2]), P(lat_ref), P(o[3])]
    peer = (ctypes.c_void_p * 1)(slots.data_ptr())
    fl = (ctypes.c_void_p * 1)(flags.data_ptr())
    owner = (ctypes.c_int * n_slots)(*([0] * n_slots))
    d = lambda k: [P(hist[k, j]) for j in range(3)]

    def single(phi, lms, cd_pair):
        def step():
            for k, a in enumerate((base, ref_args)[:2 if cd_pair else 1]):
                if lms:
                    h = list(c) + d(k)
                    rc = (lib.rtti_region_blend_cfg_lms(*a, *h, st()) if phi == 0 else
                          lib.rtti_region_blend_cfg_rescale_lms(*a, *h, phi, st()))
                else:
                    rc = (lib.rtti_region_blend_cfg(*a, c[0], st()) if phi == 0 else
                          lib.rtti_region_blend_cfg_rescale(*a, c[0], phi, st()))
                assert rc == 0
        return step

    def gather(phi, lms, cd_pair):
        def step():
            a = [peer, fl, 1, 0, owner, n_slots, N, P(m), n, 8.5, P(o[0]), P(lat), P(o[1])]
            a += [P(lat_ref), P(o[3])] if cd_pair else [None, None]
            if lms:
                a += list(c) + d(0)
                a += d(1) + [P(o[4])] if cd_pair else [None] * 4
                a += [1]
                rc = (lib.rtti_gather_blend_step_lms(*a, st()) if phi == 0 else
                      lib.rtti_gather_blend_step_rescale_lms(*a, phi, st()))
            else:
                a += [c[0], 1]
                rc = (lib.rtti_gather_blend_step(*a, st()) if phi == 0 else
                      lib.rtti_gather_blend_step_rescale(*a, phi, st()))
            assert rc == 0
        return step

    rows = []
    for entry, fn in (("region_blend_cfg", single), ("gather_blend_step, world 1", gather)):
        for cd_pair in (False, True):
            for phi in (0.0, 0.7):
                res = {h: time_graph(fn(phi, h, cd_pair), launches) for h in (False, True)}
                rows.append(dict(entry=entry, n=n, N=N, cd=cd_pair, phi=phi, us_euler=res[False], us_lms=res[True]))
                print(f"{entry:27s} n={n} N={N} C/D={'yes' if cd_pair else 'no ':3s} phi={phi:g}: "
                      f"Euler {res[False]:7.2f} us   LMS order 4 {res[True]:7.2f} us", flush=True)
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
        with open(os.path.join(args.out, "lms_bench.json"), "w") as f:
            json.dump({"card": name, "power_limit": pl, "kernels": rows}, f, indent=1)


if __name__ == "__main__":
    main()
