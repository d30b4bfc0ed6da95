"""Kernel time of the region blend with and without the CFG rescale (guidance_rescale), on one GPU:

    python tests/guidance_rescale_bench.py [--launches 2000] [--out DIR]

At n = 65536 (an SDXL 1024^2 latent) and N = 5 / 10 regions it times
  - rtti_region_blend_cfg (phi = 0) and rtti_region_blend_cfg_rescale (phi = 0.7); "with C/D" adds the second call
    that steps the reference latents (one region, a mask of ones), as RegionDiffusionXL's single-GPU path does;
  - rtti_gather_blend_step (phi = 0) and rtti_gather_blend_step_rescale (phi = 0.7) at world 1 (this device's own slot
    buffer is the only peer), with and without the C/D pair in the same launch.
The launches of one case are captured in a CUDA graph (host launch cost excluded) and timed with CUDA events over
>= 1000 launches after a warm-up replay. Prints the card name and power limit, then one line per case (us per step);
with --out also writes the results as JSON there."""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    name = torch.cuda.get_device_name()
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                             str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    return name, pl


def time_graph(step, launches, per_graph=100):
    """us per call of step() (a list of raw C calls), from a CUDA graph of per_graph calls replayed."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(per_graph):
            step()
    reps = max(1, launches // per_graph)
    for _ in range(2):
        g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / (reps * per_graph)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=2000)
    ap.add_argument("--n", type=int, default=65536)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from rtti_b200 import _lib, ops
    lib = _lib.load()
    n = args.n
    g = torch.Generator(device="cuda").manual_seed(0)
    P = lambda t: ctypes.c_void_p(t.data_ptr())
    name, pl = card()
    print(f"card: {name}, power limit {pl}", flush=True)
    rows = []
    for N in (5, 10):
        n_slots = N + 3
        slots = torch.randn(2, n_slots, n, device="cuda", generator=g).half()
        flags = torch.zeros(16, dtype=torch.int32, device="cuda")
        m = torch.softmax(torch.randn(N, n, device="cuda", generator=g), 0).contiguous()
        ones = torch.ones(1, n, device="cuda")
        lat, lat_ref = torch.randn(n, device="cuda", generator=g).half(), torch.randn(n, device="cuda", generator=g).half()
        o = [torch.empty(n, dtype=torch.float16, device="cuda") for _ in range(4)]
        stream = lambda: ops._stream()
        regions = (ctypes.c_void_p * N)(*[slots[1, 1 + i].data_ptr() for i in range(N)])
        ref_d = (ctypes.c_void_p * 1)(slots[1, N + 2].data_ptr())
        base = [P(slots[1, 0]), regions, P(m), N, n, 8.5, P(o[0]), P(lat), P(o[1]), -0.1]
        ref_args = [P(slots[1, N + 1]), ref_d, P(ones), 1, n, 8.5, P(o[2]), P(lat_ref), P(o[3]), -0.1]
        peer = (ctypes.c_void_p * 1)(slots.data_ptr())
        fl = (ctypes.c_void_p * 1)(flags.data_ptr())
        owner = (ctypes.c_int * n_slots)(*([0] * n_slots))

        def single(phi, cd):
            def step():
                for a in ([base] + ([ref_args] if cd else [])):
                    rc = (lib.rtti_region_blend_cfg(*a, stream()) if phi == 0 else
                          lib.rtti_region_blend_cfg_rescale(*a, phi, stream()))
                    assert rc == 0
            return step

        def gather(phi, cd):
            def step():
                a = [peer, fl, 1, 0, owner, n_slots, N, P(m), n, 8.5, P(o[0]), P(lat), P(o[1]),
                     P(lat_ref) if cd else ctypes.c_void_p(0), P(o[3]) if cd else ctypes.c_void_p(0), -0.1, 1]
                rc = (lib.rtti_gather_blend_step(*a, stream()) if phi == 0 else
                      lib.rtti_gather_blend_step_rescale(*a, phi, stream()))
                assert rc == 0
            return step

        for entry, fn in (("region_blend_cfg", single), ("gather_blend_step (world 1)", gather)):
            for cd in (False, True):
                res = {}
                for phi in (0.0, 0.7):
                    res[phi] = time_graph(fn(phi, cd), args.launches)
                row = dict(entry=entry, n=n, N=N, cd_pair=cd, us_phi0=res[0.0], us_phi07=res[0.7])
                rows.append(row)
                print(f"{entry:28s} n={n} N={N:2d} C/D {'yes' if cd else 'no ':3s}: phi=0 {res[0.0]:7.2f} us   "
                      f"phi=0.7 {res[0.7]:7.2f} us", flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "guidance_rescale_bench.json"), "w") as f:
            json.dump({"card": name, "power_limit": pl, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
