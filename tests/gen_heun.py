"""TEST INFRASTRUCTURE — generates tests/golden/heun.npz (and nothing else) by running the UNMODIFIED reference through
oracle/ref_shim.py with the restated Heun scheduler of tests/heun_oracle.py assigned to its `scheduler`, on the inputs
of tests/gen_multistep.py (same seeds and latent sides).

Run where the reference tree exists (never on the GPU box):
    python -m tests.gen_heun
It records
  - the SDXL plain pass (:879-914; tiny XL, 32^2 latent, guidance 8.5) at 5 and 10 steps (9 and 19 UNet evaluations),
    with the iterations at which the reference calls back (callback_steps 1);
  - the SDXL rich loop (:772-878; 128^2, 3 regions, colour guidance, font sizes) at 4 steps (7 iterations), with
    inject_selfattn = inject_background = 0.5 (the reference latents are stepped jointly on every iteration) and with
    inject_selfattn = 0, inject_background = 0.5 (jointly on iterations 0..3, then the main latents alone), and its
    callback iterations. The last joint iteration, 3, is a second stage, so the reference's batch-2 saved state is
    consumed by a batch-2 step and the reference loop is well defined there: asserted below.
"""
import os

import numpy as np
import torch

from oracle import gen_golden as gg
from oracle import ref_shim, unet_oracle as uo
from tests import heun_oracle as ho
from tests import multistep_oracle as mo

PLAIN = (5, 10)
RICH_STEPS = 4
RICH = ((0.5, 0.5), (0.0, 0.5))   # (inject_selfattn, inject_background)


def gen_heun(ns):
    if ns.region_diffusion_sdxl is None:
        raise RuntimeError(ns.region_diffusion_sdxl_error)
    res = {}
    cfg = uo.tiny_xl_config()
    S = mo.LATENT_XL_PLAIN
    inp = gg.synth_inputs(cfg, 3, S, 31)
    ctx, te = inp["ctx"], inp["text_embeds"]
    for steps in PLAIN:
        m = gg.make_xl_sampler(ns, cfg, 2, (ctx[-1:], ctx[:1], te[-1:], te[:1]))
        m.scheduler = ho.HeunSchedulerOracle()
        calls = []
        out = m.sample(["x"], height=S * 8, width=S * 8, num_inference_steps=steps, guidance_scale=8.5,
                       negative_prompt=[""], latents=inp["latents"].clone(), output_type="latent", run_rich_text=False,
                       callback=lambda i, t, lat: calls.append(i), callback_steps=1)
        assert m.scheduler.step_batches == [1] * (2 * steps - 1)
        assert calls == ho.callback_iterations(2 * steps - 1, steps, 2, 1), calls
        res[f"xl_plain_{steps}"] = out.images.numpy()
        res[f"xl_plain_{steps}_callbacks"] = np.asarray(calls, np.int64)
    S = mo.LATENT_XL_RICH
    inp = gg.synth_inputs(cfg, 3, S, 31)
    ctx, te = inp["ctx"], inp["text_embeds"]
    n_it = 2 * RICH_STEPS - 1
    for sa, bg in RICH:
        m = gg.make_xl_sampler(ns, cfg, 2, (ctx[1:], ctx[:1], te[1:], te[:1]))
        m.scheduler = ho.HeunSchedulerOracle()
        m.masks = inp["masks"]
        tfd = gg.text_format(1, S, 31)
        tfd.update(gg.color_dict(inp["masks"], S, weight=1.0))
        calls = []
        out = m.sample(["a", "b", "c"], height=S * 8, width=S * 8, num_inference_steps=RICH_STEPS, guidance_scale=8.5,
                       negative_prompt=[""], latents=inp["latents"].clone(), output_type="latent", use_guidance=True,
                       inject_selfattn=sa, inject_background=bg, text_format_dict=tfd, run_rich_text=True,
                       callback=lambda i, t, lat: calls.append(i), callback_steps=1)
        joint = [i for i in range(n_it) if sa > 0 or i < bg * n_it]
        assert m.scheduler.step_batches == [2 if i in joint else 1 for i in range(n_it)], m.scheduler.step_batches
        assert joint[-1] % 2 == 1 or joint[-1] == n_it - 1, "the last joint iteration must not be a first stage"
        assert calls == ho.callback_iterations(n_it, RICH_STEPS, 2, 1), calls
        print("rich", sa, bg, "step batches", m.scheduler.step_batches, "callbacks", calls)
        res[f"xl_rich_{sa:g}_{bg:g}"] = out.images.detach().numpy()
        res[f"xl_rich_{sa:g}_{bg:g}_callbacks"] = np.asarray(calls, np.int64)
    np.savez_compressed(os.path.join(gg.GOLD, "heun.npz"), **res)
    print("heun ok", {k: float(np.abs(v).mean()) for k, v in res.items()})


if __name__ == "__main__":
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    gen_heun(ref_shim.import_reference())
