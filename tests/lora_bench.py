"""Step time with and without a merged LoRA, and the cost of the merge, on one GPU:

    python tests/lora_bench.py [--trials 3] [--steps 4] [--rank 32] [--out DIR]

1. RegionDiffusionXL.rich_text_step at the bench.py --config 3 shape (SDXL 1024^2, random weights, 5 regions, injection
   0.5 / 0.5, colour guidance), 41-step schedule, without a LoRA and with a rank --rank LoRA on every linear and conv of
   the UNet's blocks merged at scale 0.8, alternated, median of --trials timings of --steps steps each. The merged model
   runs the same kernels on other weights, so the two should agree within the run-to-run spread.
2. The merge: load_lora_weights (state dict on the host -> device factors, W0 kept, merged), set_lora_scale (re-merge
   from W0) and unload_lora_weights, each timed with a device synchronise, median over --trials, and the device memory
   the loaded LoRA holds (W0 copies and factors).
Prints the card name and power limit, then the numbers; with --out also writes them as JSON there."""
import argparse
import json
import os
import statistics
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests.guidance_rescale_bench import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--trials", type=int, default=3)
    ap.add_argument("--steps", type=int, default=4)
    ap.add_argument("--rank", type=int, default=32)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import bench
    from rtti_b200 import lora
    from rtti_b200.region_diffusion_sdxl import RegionDiffusionXL
    from tests import lora_synth
    name, pl = card()
    print(f"card: {name}, power limit {pl}", flush=True)
    cfg = bench.CONFIGS[3]
    dev = torch.device("cuda", torch.cuda.current_device())
    model = RegionDiffusionXL.from_synthetic(seed=0, device=dev, with_vae=cfg["color"])
    targets = lora.unet_targets(model.unet)
    fac = lora_synth.lora_factors(targets, args.rank, seed=1)
    lsd = lora_synth.kohya_dict(fac, {n: lora_synth.diffusers_stem(n) for n in targets}, args.rank / 2)
    n_params = sum(m.weight.numel() for m in targets.values())
    n_lora = sum(d.numel() + u.numel() for d, u in fac.values())
    print(f"LoRA: rank {args.rank}, {len(targets)} target weights, {n_params / 1e9:.3f} B parameters of W0, "
          f"{n_lora / 1e6:.1f} M LoRA parameters", flush=True)
    wl = bench.synth_workload(cfg)
    time_ids = torch.tensor([[1024.0, 1024, 0, 0, 1024, 1024]], device=dev)
    n_t = cfg["schedule"]

    def fresh():
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

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3

    idx = bench.spread(args.steps, n_t)
    times = {"no_lora": [], "lora": []}
    merge = {"load_ms": [], "set_scale_ms": [], "unload_ms": []}
    held = 0
    with torch.no_grad():
        st = fresh()   # warm-up: graph capture, cuDNN / cuBLAS choices, both injection regimes
        for i in sorted({0, int(cfg["inject_background"] * n_t), n_t - 1}):
            model.rich_text_step(st, i)
        del st
        for _ in range(args.trials):
            for variant in ("no_lora", "lora"):
                if variant == "lora":
                    base = torch.cuda.memory_allocated()
                    merge["load_ms"].append(timed(lambda: model.load_lora_weights(lsd, scale=0.5)))
                    held = torch.cuda.memory_allocated() - base
                    merge["set_scale_ms"].append(timed(lambda: model.set_lora_scale(0.8)))
                st = fresh()
                torch.cuda.synchronize()
                ev = []
                for i in range(idx[-1] + 1):   # the state of step i - 1 is what step i reads
                    if i in idx:
                        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        e0.record()
                        model.rich_text_step(st, i)
                        e1.record()
                        ev.append((e0, e1))
                    else:
                        model.rich_text_step(st, i)
                torch.cuda.synchronize()
                times[variant].append(sum(a.elapsed_time(b) for a, b in ev) / len(ev))
                del st
                if variant == "lora":
                    merge["unload_ms"].append(timed(model.unload_lora_weights))
    res = {k: dict(ms_per_step_median=statistics.median(v), ms_per_step_trials=v) for k, v in times.items()}
    for k, v in res.items():
        print(f"rich_text_step, config 3 shape, {k:8s}: median {v['ms_per_step_median']:.2f} ms/step  "
              f"trials {[round(x, 2) for x in v['ms_per_step_trials']]}", flush=True)
    mres = {k: statistics.median(v) for k, v in merge.items()}
    print(f"merge, rank {args.rank}: load_lora_weights {mres['load_ms']:.1f} ms, set_lora_scale {mres['set_scale_ms']:.1f} ms, "
          f"unload_lora_weights {mres['unload_ms']:.1f} ms (medians of {merge}); "
          f"device memory held by the loaded LoRA {held / 2 ** 30:.2f} GiB", flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "lora_bench.json"), "w") as f:
            json.dump({"card": name, "power_limit": pl, "rank": args.rank, "targets": len(targets),
                       "w0_params": n_params, "rich_text_step": res, "merge_ms": mres, "merge_ms_trials": merge,
                       "held_bytes": held}, f, indent=1)


if __name__ == "__main__":
    main()
