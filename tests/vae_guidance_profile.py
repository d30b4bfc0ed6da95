"""Kernel table (GPU) of one colour-guidance evaluation: forward + data-gradient backward of the fp32 SDXL VAE decoder
(vae_guidance.DecoderFwdBwd) at a 128x128 latent (1024^2 image), under torch.profiler with CUDA activities.
Prints the wall time of the evaluation (CUDA events, profiler off), then every kernel grouped into
conv / groupnorm / elementwise / copy / attention with ms and share, then the top kernels.
    python tests/vae_guidance_profile.py [--latent 128] [--out DIR]"""
import argparse
import collections
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def category(name):
    n = name.lower()
    if "gn32" in n:
        return "groupnorm"
    if any(k in n for k in ("conv", "fprop", "dgrad", "implicit", "upsample_phase")):
        return "conv"
    if any(k in n for k in ("gemm", "softmax", "bmm")):
        return "attention"
    if any(k in n for k in ("copy", "reduce", "cat", "fill")):
        return "copy"
    return "elementwise"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--latent", type=int, default=128)
    ap.add_argument("--out", default=None, help="also write the table as JSON into this directory")
    args = ap.parse_args()
    from rtti_b200 import vae_guidance
    from rtti_b200.vae import AutoencoderKLDecoder, VAEConfig
    torch.backends.cudnn.benchmark = True
    vae = AutoencoderKLDecoder(VAEConfig.sdxl()).init_synthetic(0).finalize("cuda")
    eng = vae_guidance.DecoderFwdBwd(vae)
    h = args.latent
    z = torch.randn(1, 4, h, h, device="cuda", generator=torch.Generator("cuda").manual_seed(0))
    gimg = torch.randn(1, 3, 8 * h, 8 * h, device="cuda", generator=torch.Generator("cuda").manual_seed(1))

    def run():
        eng.forward(z)
        return eng.backward(gimg)

    for _ in range(3):
        run()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    n = 5
    e0.record()
    for _ in range(n):
        run()
    e1.record()
    torch.cuda.synchronize()
    wall = e0.elapsed_time(e1) / n
    print(f"{torch.cuda.get_device_name()}: decoder fwd+bwd at {8 * h}^2: {wall:.2f} ms per evaluation (mean of {n})")

    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run()
        torch.cuda.synchronize()
    per = collections.defaultdict(lambda: [0.0, 0])
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA:
            per[ev.name][0] += ev.device_time / 1e3
            per[ev.name][1] += 1
    total = sum(v[0] for v in per.values())
    cats = collections.defaultdict(float)
    for name, (ms, _) in per.items():
        cats[category(name)] += ms
    print(f"kernel time {total:.2f} ms")
    print(f"{'category':<12} {'ms':>9} {'share':>7}")
    for c, ms in sorted(cats.items(), key=lambda kv: -kv[1]):
        print(f"{c:<12} {ms:9.2f} {100 * ms / total:6.1f}%")
    print(f"\n{'ms':>9} {'calls':>6} {'cat':<12} kernel")
    for name, (ms, cnt) in sorted(per.items(), key=lambda kv: -kv[1][0])[:30]:
        print(f"{ms:9.2f} {cnt:6d} {category(name):<12} {name[:110]}")
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "vae_guidance_profile.json"), "w") as f:
            json.dump({"device": torch.cuda.get_device_name(), "wall_ms": wall, "kernel_ms": total, "categories": cats,
                       "kernels": {k: v for k, v in per.items()}}, f, indent=1)


if __name__ == "__main__":
    main()
