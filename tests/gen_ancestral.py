"""TEST INFRASTRUCTURE — generates tests/golden/ancestral.npz (and nothing else) by running the UNMODIFIED reference
through oracle/ref_shim.py with the restated Euler Ancestral scheduler of tests/ancestral_oracle.py assigned to its
`scheduler`, on the inputs of tests/gen_multistep.py (same seeds and latent sides).

Run where the reference tree exists (never on the GPU box):
    python -m tests.gen_ancestral
It records
  - the SDXL plain pass (:879-914; tiny XL, 32^2 latent, guidance 8.5) at 10 and 20 steps, with
    `sample(generator=torch.Generator().manual_seed(SEED))`, which the reference forwards to every step;
  - the SDXL rich loop (:772-878; 128^2, 3 regions, colour guidance, font sizes) at 4 steps with inject_selfattn =
    inject_background = 0.5 (the reference latents are stepped jointly on every step: one [2, ...] draw per step) and
    with inject_selfattn = 0, inject_background = 0.5 (joint draws on the first two steps, then [1, ...] draws). The
    reference passes no generator to these steps; the scheduler draws from its own CPU generator seeded SEED.
"""
import os

import numpy as np
import torch

from oracle import gen_golden as gg
from oracle import ref_shim, unet_oracle as uo
from tests import ancestral_oracle as ao
from tests import multistep_oracle as mo

SEED = 1234
PLAIN = (10, 20)
RICH = ((0.5, 0.5), (0.0, 0.5))   # (inject_selfattn, inject_background)


def gen_ancestral(ns):
    if ns.region_diffusion_sdxl is None:
        raise RuntimeError(ns.region_diffusion_sdxl_error)
    res = {}
    cfg = uo.tiny_xl_config()
    S = mo.LATENT_XL_PLAIN
    inp = gg.synth_inputs(cfg, 3, S, 31)
    ctx, te = inp["ctx"], inp["text_embeds"]
    for steps in PLAIN:
        m = gg.make_xl_sampler(ns, cfg, 2, (ctx[-1:], ctx[:1], te[-1:], te[:1]))
        m.scheduler = ao.EulerAncestralSchedulerOracle()
        out = m.sample(["x"], height=S * 8, width=S * 8, num_inference_steps=steps, guidance_scale=8.5,
                       negative_prompt=[""], latents=inp["latents"].clone(), output_type="latent", run_rich_text=False,
                       generator=torch.Generator().manual_seed(SEED))
        assert m.scheduler.draw_shapes == [(1, 4, S, S)] * steps
        res[f"xl_plain_{steps}"] = out.images.numpy()
    S = mo.LATENT_XL_RICH
    inp = gg.synth_inputs(cfg, 3, S, 31)
    ctx, te = inp["ctx"], inp["text_embeds"]
    for sa, bg in RICH:
        m = gg.make_xl_sampler(ns, cfg, 2, (ctx[1:], ctx[:1], te[1:], te[:1]))
        m.scheduler = ao.EulerAncestralSchedulerOracle(generator=torch.Generator().manual_seed(SEED))
        m.masks = inp["masks"]
        tfd = gg.text_format(1, S, 31)
        tfd.update(gg.color_dict(inp["masks"], S, weight=1.0))
        out = m.sample(["a", "b", "c"], height=S * 8, width=S * 8, num_inference_steps=4, guidance_scale=8.5,
                       negative_prompt=[""], latents=inp["latents"].clone(), output_type="latent", use_guidance=True,
                       inject_selfattn=sa, inject_background=bg, text_format_dict=tfd, run_rich_text=True)
        print("rich", sa, bg, "draws", m.scheduler.draw_shapes)
        res[f"xl_rich_{sa:g}_{bg:g}"] = out.images.detach().numpy()
    np.savez_compressed(os.path.join(gg.GOLD, "ancestral.npz"), **res)
    print("ancestral ok", {k: float(np.abs(v).mean()) for k, v in res.items()})


if __name__ == "__main__":
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    gen_ancestral(ref_shim.import_reference())
