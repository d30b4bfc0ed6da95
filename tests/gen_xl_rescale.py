"""TEST INFRASTRUCTURE — generates tests/golden/xl_rescale.npz (and nothing else) by running the UNMODIFIED reference
through oracle/ref_shim.py, with the helpers and inputs of oracle/gen_golden.py's gen_xl_loops.

Run where the reference tree exists (never on the GPU box):
    python -m tests.gen_xl_rescale
It records
  - the reference's rescale_noise_cfg (models/region_diffusion_sdxl.py:42-53) on seeded [2, 4, 16, 16] tensors at
    guidance_rescale 0.3, 0.7 and 1.0;
  - the reference's plain pass (:879-914) with the inputs of gen_xl_loops (tiny XL, 128^2 latent, 12 steps, guidance
    8.5) at guidance_rescale 0.7.
"""
import os

import numpy as np
import torch

from oracle import gen_golden as gg
from oracle import ref_shim, unet_oracle as uo

PHIS = (0.3, 0.7, 1.0)


def rescale_inputs():
    """Seeded CFG / text predictions with different per-entry scales and offsets."""
    g = torch.Generator().manual_seed(2305)
    cfg = torch.randn(2, 4, 16, 16, generator=g) * torch.tensor([3.0, 0.5]).reshape(2, 1, 1, 1) + 0.25
    text = torch.randn(2, 4, 16, 16, generator=g) * torch.tensor([1.0, 2.0]).reshape(2, 1, 1, 1) - 0.5
    return cfg, text


def gen_xl_rescale(ns):
    if ns.region_diffusion_sdxl is None:
        raise RuntimeError(ns.region_diffusion_sdxl_error)
    res = {}
    cfg_t, text_t = rescale_inputs()
    for phi in PHIS:
        res[f"rescale_{phi:g}"] = ns.region_diffusion_sdxl.rescale_noise_cfg(cfg_t, text_t, guidance_rescale=phi).numpy()
    cfg = uo.tiny_xl_config()
    S = 128
    inp = gg.synth_inputs(cfg, 3, S, 31)
    ctx, te = inp["ctx"], inp["text_embeds"]
    m = gg.make_xl_sampler(ns, cfg, 2, (ctx[-1:], ctx[:1], te[-1:], te[:1]))
    out = m.sample(["x"], height=S * 8, width=S * 8, num_inference_steps=12, guidance_scale=8.5, negative_prompt=[""],
                   latents=inp["latents"].clone(), output_type="latent", run_rich_text=False, guidance_rescale=0.7)
    res["plain_latents_phi0.7"] = out.images.numpy()
    np.savez_compressed(os.path.join(gg.GOLD, "xl_rescale.npz"), **res)
    print("xl rescale ok", {k: float(np.abs(v).mean()) for k, v in res.items()})


if __name__ == "__main__":
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    gen_xl_rescale(ref_shim.import_reference())
