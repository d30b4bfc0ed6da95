"""TEST INFRASTRUCTURE — generates tests/golden/unipc.npz (and nothing else) by running the UNMODIFIED reference through
oracle/ref_shim.py with the restated UniPC scheduler of tests/unipc_oracle.py assigned to its `scheduler`, on the
inputs of oracle/gen_golden.py's gen_xl_loops / gen_sd_loops (same seeds; latent sides multistep_oracle.LATENT_*).

Run where the reference tree exists (never on the GPU box):
    python -m tests.gen_unipc
It records
  - the SDXL plain pass (:879-914; tiny XL, 32^2 latent, guidance 8.5) at 5 and 10 steps;
  - the SDXL rich loop (:772-878; 128^2, 3 regions, inject_selfattn 0.5, inject_background 0.5, colour guidance, font
    sizes) at 5 steps: the corrector meets latents that colour guidance and background injection have moved. The
    reference latents are stepped jointly on every step there, so one batch-2 scheduler state is one state per
    trajectory;
  - SD1.5 produce_latents (models/region_diffusion.py:86-174; tiny SD, 64^2, the rich inputs of gen_sd_loops) at 5
    steps.
"""
import os

import numpy as np
import torch

from oracle import gen_golden as gg
from oracle import ref_shim, unet_oracle as uo
from tests import multistep_oracle as mo
from tests import unipc_oracle as uo_sched

PLAIN = (5, 10)
RICH = 5


def gen_unipc(ns):
    if ns.region_diffusion_sdxl is None:
        raise RuntimeError(ns.region_diffusion_sdxl_error)
    res = {}
    cfg = uo.tiny_xl_config()
    S = mo.LATENT_XL_PLAIN
    inp = gg.synth_inputs(cfg, 3, S, 31)
    ctx, te = inp["ctx"], inp["text_embeds"]
    for steps in PLAIN:
        m = gg.make_xl_sampler(ns, cfg, 2, (ctx[-1:], ctx[:1], te[-1:], te[:1]))
        m.scheduler = uo_sched.UniPCSchedulerOracle()
        out = m.sample(["x"], height=S * 8, width=S * 8, num_inference_steps=steps, guidance_scale=8.5,
                       negative_prompt=[""], latents=inp["latents"].clone(), output_type="latent", run_rich_text=False)
        res[f"xl_plain_unipc_{steps}"] = out.images.numpy()
    S = mo.LATENT_XL_RICH
    inp = gg.synth_inputs(cfg, 3, S, 31)
    ctx, te = inp["ctx"], inp["text_embeds"]
    m = gg.make_xl_sampler(ns, cfg, 2, (ctx[1:], ctx[:1], te[1:], te[:1]))
    m.scheduler = uo_sched.UniPCSchedulerOracle()
    m.masks = inp["masks"]
    tfd = gg.text_format(1, S, 31)
    tfd.update(gg.color_dict(inp["masks"], S, weight=1.0))
    out = m.sample(["a", "b", "c"], height=S * 8, width=S * 8, num_inference_steps=RICH, guidance_scale=8.5,
                   negative_prompt=[""], latents=inp["latents"].clone(), output_type="latent", use_guidance=True,
                   inject_selfattn=0.5, inject_background=0.5, text_format_dict=tfd, run_rich_text=True)
    res[f"xl_rich_unipc_{RICH}"] = out.images.detach().numpy()
    cfg = uo.tiny_sd_config()
    S = mo.LATENT_SD
    inp = gg.synth_inputs(cfg, 3, S, 21)
    m = gg.make_sd_sampler(ns, cfg, 1)
    m.scheduler = uo_sched.UniPCSchedulerOracle()
    m.masks = inp["masks"]
    m.vae = gg._TinyVAE()
    tfd = gg.text_format(1, S, 21)
    tfd.update(gg.color_dict(inp["masks"], S, weight=0.5))
    lat = m.produce_latents(inp["ctx"], height=S * 8, width=S * 8, num_inference_steps=RICH, guidance_scale=8.5,
                            latents=inp["latents"].clone(), use_guidance=True, text_format_dict=tfd,
                            inject_selfattn=0.3, inject_background=0.5)
    res[f"sd_rich_unipc_{RICH}"] = lat.detach().numpy()
    np.savez_compressed(os.path.join(gg.GOLD, "unipc.npz"), **res)
    print("unipc ok", {k: float(np.abs(v).mean()) for k, v in res.items()})


if __name__ == "__main__":
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    gen_unipc(ref_shim.import_reference())
