"""Cost of the DPM-Solver++(2S) blend entry points against their multistep (DPM-Solver++(2M)) counterparts, on one GPU:

    python tests/singlestep_bench.py [--launches 2000] [--trials 3] [--steps 4] [--out DIR]

1. Kernel time at the SDXL 1024^2 shape (n = 65536 latent elements, 5 regions), guidance_rescale 0 and 0.7, with and
   without the reference-latent pair C/D: rtti_region_blend_cfg(_rescale)_ms vs its _ss form (with C/D: plus the C/D
   call, as the single-GPU rich loop runs it), and rtti_gather_blend_step(_rescale)_ms vs its _ss form at world 1 (this
   device's slot buffer is the only peer). Both take a second-order step that reads D_prev; the _ss form of the second
   step of a block also reads the fp16 latents xs of each trajectory it steps. Launches are captured in CUDA graphs of
   100 and timed with CUDA events over >= 1000 launches after a warm-up.
2. RegionDiffusionXL.rich_text_step at the bench.py --config 3 shape (SDXL 1024^2, random weights, 5 regions,
   injection 0.5 / 0.5, colour guidance), 41-step schedules, with DPMSolverMultistepScheduler and with
   DPMSolverSinglestepScheduler, alternated, median of --trials timings of --steps steps each.
Prints the card name and power limit, then the numbers; with --out also writes them as JSON there."""
import argparse
import ctypes
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests.guidance_rescale_bench import card, time_graph  # noqa: E402


def kernel_rows(lib, ops, launches):
    from rtti_b200.schedulers import DPMSolverSinglestepScheduler
    s = DPMSolverSinglestepScheduler()
    s.set_timesteps(20)
    c = s.singlestep_coeffs(11)
    assert c.cs != 0.0 and c.cp != 0.0
    ms_c = [c.hx, c.he, c.cx, c.cd, c.cp]
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
    xs = torch.randn(2, n, device="cuda", generator=g).half()     # [trajectory]
    dh = torch.randn(2, n, device="cuda", generator=g)            # [trajectory]: d_prev = d_out
    o = [torch.empty(n, dtype=torch.float16, device="cuda") for _ in range(4)]
    regions = (ctypes.c_void_p * N)(*[slots[1, 1 + i].data_ptr() for i in range(N)])
    ref_d = (ctypes.c_void_p * 1)(slots[1, N + 2].data_ptr())
    base = [P(slots[1, 0]), regions, P(m), N, n, 8.5, P(o[0]), P(lat), P(o[1])]
    ref_args = [P(slots[1, N + 1]), ref_d, P(ones), 1, n, 8.5, P(o[2]), P(lat_ref), P(o[3])]
    peer = (ctypes.c_void_p * 1)(slots.data_ptr())
    fl = (ctypes.c_void_p * 1)(flags.data_ptr())
    owner = (ctypes.c_int * n_slots)(*([0] * n_slots))

    def single(phi, ss, cd_pair):
        def step():
            for k, a in enumerate((base, ref_args)[:2 if cd_pair else 1]):
                if ss:
                    h = list(c) + [P(dh[k]), P(dh[k]), P(xs[k])]
                    rc = (lib.rtti_region_blend_cfg_ss(*a, *h, st()) if phi == 0 else
                          lib.rtti_region_blend_cfg_rescale_ss(*a, *h, phi, st()))
                else:
                    h = ms_c + [P(dh[k]), P(dh[k])]
                    rc = (lib.rtti_region_blend_cfg_ms(*a, *h, st()) if phi == 0 else
                          lib.rtti_region_blend_cfg_rescale_ms(*a, *h, phi, st()))
                assert rc == 0
        return step

    def gather(phi, ss, cd_pair):
        def step():
            a = [peer, fl, 1, 0, owner, n_slots, N, P(m), n, 8.5, P(o[0]), P(lat), P(o[1])]
            a += [P(lat_ref), P(o[3])] if cd_pair else [None, None]
            if ss:
                a += list(c) + [P(dh[0]), P(dh[0]), P(xs[0])]
                a += [P(dh[1]), P(dh[1]), P(xs[1])] if cd_pair else [None] * 3
                a += [1]
                rc = (lib.rtti_gather_blend_step_ss(*a, st()) if phi == 0 else
                      lib.rtti_gather_blend_step_rescale_ss(*a, phi, st()))
            else:
                a += ms_c + [P(dh[0]), P(dh[0])]
                a += [P(dh[1]), P(dh[1])] if cd_pair else [None] * 2
                a += [1]
                rc = (lib.rtti_gather_blend_step_ms(*a, st()) if phi == 0 else
                      lib.rtti_gather_blend_step_rescale_ms(*a, phi, st()))
            assert rc == 0
        return step

    rows = []
    for entry, fn in (("region_blend_cfg", single), ("gather_blend_step, world 1", gather)):
        for cd_pair in (False, True):
            for phi in (0.0, 0.7):
                res = {h: time_graph(fn(phi, h, cd_pair), launches) for h in (False, True)}
                rows.append(dict(entry=entry, n=n, N=N, cd=cd_pair, phi=phi, us_ms=res[False], us_ss=res[True]))
                print(f"{entry:27s} n={n} N={N} C/D={'yes' if cd_pair else 'no ':3s} phi={phi:g}: "
                      f"_ms {res[False]:7.2f} us   _ss {res[True]:7.2f} us", flush=True)
    return rows


def step_rows(trials, steps):
    import bench
    from rtti_b200.region_diffusion_sdxl import RegionDiffusionXL
    from rtti_b200.schedulers import DPMSolverMultistepScheduler, DPMSolverSinglestepScheduler
    cfg = bench.CONFIGS[3]
    dev = torch.device("cuda", torch.cuda.current_device())
    model = RegionDiffusionXL.from_synthetic(seed=0, device=dev, with_vae=cfg["color"])
    wl = bench.synth_workload(cfg)
    time_ids = torch.tensor([[1024.0, 1024, 0, 0, 1024, 1024]], device=dev)
    n_t = cfg["schedule"]
    schedulers = {"dpmpp_2m": DPMSolverMultistepScheduler(), "dpmpp_2s": DPMSolverSinglestepScheduler()}

    def fresh(name):
        model.scheduler = schedulers[name]
        model.scheduler.set_timesteps(n_t)
        tfd = dict(wl["tfd"])
        tfd["color_obj_atten"] = [x.to(dev) for x in tfd["color_obj_atten"]]
        tfd["target_RGB"] = [x.to(dev) for x in tfd["target_RGB"]]
        tfd["color_obj_atten_all"] = tfd["color_obj_atten_all"].to(dev)
        model.masks = [x.to(dev) for x in wl["masks"]]
        lat = wl["latents"].to(dev, torch.float16) * model.scheduler.init_noise_sigma
        return model.prepare_rich_text(wl["ctx"].to(dev, torch.float16), wl["pooled"].to(dev, torch.float16), time_ids,
                                       lat, model.scheduler.timesteps, bench.GUIDANCE, cfg["color"],
                                       cfg["inject_selfattn"], cfg["inject_background"], tfd)

    idx = bench.spread(steps, n_t)
    times = {k: [] for k in schedulers}
    with torch.no_grad():
        for name in schedulers:   # warm-up: graph capture, cuDNN / cuBLAS choices, both injection regimes
            st = fresh(name)
            for i in sorted({0, int(cfg["inject_background"] * n_t), n_t - 1}):
                model.rich_text_step(st, i)
        torch.cuda.synchronize()
        for _ in range(trials):
            for name in schedulers:
                st = fresh(name)
                # the state of step i - 1 is what step i reads: run every step up to the last timed one
                torch.cuda.synchronize()
                ev = []
                for i in range(idx[-1] + 1):
                    if i in idx:
                        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        e0.record()
                        model.rich_text_step(st, i)
                        e1.record()
                        ev.append((e0, e1))
                    else:
                        model.rich_text_step(st, i)
                torch.cuda.synchronize()
                times[name].append(sum(a.elapsed_time(b) for a, b in ev) / len(ev))
    res = {k: dict(ms_per_step_median=statistics.median(v), ms_per_step_trials=v) for k, v in times.items()}
    for k, v in res.items():
        print(f"rich_text_step, config 3 shape, {k:9s}: median {v['ms_per_step_median']:.2f} ms/step "
              f"({1e3 / v['ms_per_step_median']:.3f} steps/s)  trials {[round(x, 2) for x in v['ms_per_step_trials']]}",
              flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=2000)
    ap.add_argument("--trials", type=int, default=3)
    ap.add_argument("--steps", type=int, default=4)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from rtti_b200 import _lib, ops
    lib = _lib.load()
    name, pl = card()
    print(f"card: {name}, power limit {pl}", flush=True)
    rows = kernel_rows(lib, ops, args.launches)
    steps = step_rows(args.trials, args.steps)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "singlestep_bench.json"), "w") as f:
            json.dump({"card": name, "power_limit": pl, "kernels": rows, "rich_text_step": steps}, f, indent=1)


if __name__ == "__main__":
    main()
