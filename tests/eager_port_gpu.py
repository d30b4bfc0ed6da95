"""Honest GPU baseline (SURVEY §8d): the reference's algorithm as plain PyTorch-eager on the SAME GPU —
the oracle restatement (oracle/unet_oracle.py: baddbmm -> softmax -> bmm with the probability tensor
materialised, head mean on every call, batch-1 passes run one after another as models/region_diffusion_sdxl.py:787-821
does), fp16 weights. Times UNet passes only (8 per step for the 5-region injected workload); prints one JSON line.

    python tests/eager_port_gpu.py > profiles/eager_port.json      # test infrastructure, not the product path
"""
import json
import math
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import unet_oracle as uo  # noqa: E402


def main():
    dev = "cuda"
    cfg = uo.sdxl_config()
    g = torch.Generator(device=dev).manual_seed(0)
    sd = {}
    for k, shp in uo.param_shapes(cfg).items():
        if len(shp) >= 2:
            sd[k] = (torch.randn(shp, generator=g, device=dev) / math.sqrt(float(torch.Size(shp[1:]).numel()))).half()
        else:
            sd[k] = (torch.ones(shp, device=dev) if k.endswith("weight") else torch.zeros(shp, device=dev)).half()
    x = torch.randn(1, 4, 128, 128, generator=g, device=dev).half()
    ctx = torch.randn(1, 77, 2048, generator=g, device=dev).half()
    added = {"text_embeds": torch.randn(1, 1280, generator=g, device=dev).half(),
             "time_ids": torch.tensor([[1024.0, 1024, 0, 0, 1024, 1024]], device=dev)}
    t = torch.tensor(981.0, device=dev)
    with torch.no_grad():
        for _ in range(2):
            uo.unet_forward(sd, cfg, x, t, ctx, added)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        n = 8
        for _ in range(n):
            uo.unet_forward(sd, cfg, x, t, ctx, added)
        e1.record()
        torch.cuda.synchronize()
    ms_pass = e0.elapsed_time(e1) / n
    print(json.dumps({"what": "PyTorch-eager port of the reference UNet pass on this GPU (fp16, batch 1, probabilities materialised)",
                      "ms_per_pass": ms_pass, "passes_per_step": 8, "steps_per_s_unet_only": 1000.0 / (8 * ms_pass),
                      "peak_mem_gb": torch.cuda.max_memory_allocated() / 2 ** 30}))


if __name__ == "__main__":
    main()
