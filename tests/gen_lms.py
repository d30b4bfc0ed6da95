"""TEST INFRASTRUCTURE — generates tests/golden/lms.npz (and nothing else) by running the UNMODIFIED reference through
oracle/ref_shim.py with the restated LMS scheduler of tests/lms_oracle.py assigned to its `scheduler`, on the inputs
of tests/gen_multistep.py (same seeds and latent sides).

Run where the reference tree exists (never on the GPU box):
    python -m tests.gen_lms
It records
  - the SDXL plain pass (:879-914; tiny XL, 32^2 latent, guidance 8.5) at 5 and 10 steps (order 4 from step 3 on), with
    the iterations at which the reference calls back (callback_steps 1);
  - the SDXL rich loop (:772-878; 128^2, 3 regions, colour guidance, font sizes) at 4 steps with
    inject_selfattn = inject_background = 0.5 (the reference latents are stepped jointly on every step) and with
    inject_selfattn = inject_background = 0 (no reference latents), and its callback iterations.
In every recorded case the batch of the scheduler's step calls is constant, so the reference's single derivative list
never mixes batch-1 and batch-2 entries and the reference loop is well defined: asserted below.
"""
import os

import numpy as np
import torch

from oracle import gen_golden as gg
from oracle import ref_shim, unet_oracle as uo
from tests import lms_oracle as lo
from tests import multistep_oracle as mo

PLAIN = (5, 10)
RICH_STEPS = 4
RICH = ((0.5, 0.5), (0.0, 0.0))   # (inject_selfattn, inject_background)


def gen_lms(ns):
    if ns.region_diffusion_sdxl is None:
        raise RuntimeError(ns.region_diffusion_sdxl_error)
    res = {}
    cfg = uo.tiny_xl_config()
    S = mo.LATENT_XL_PLAIN
    inp = gg.synth_inputs(cfg, 3, S, 31)
    ctx, te = inp["ctx"], inp["text_embeds"]
    for steps in PLAIN:
        m = gg.make_xl_sampler(ns, cfg, 2, (ctx[-1:], ctx[:1], te[-1:], te[:1]))
        m.scheduler = lo.LMSSchedulerOracle()
        calls = []
        out = m.sample(["x"], height=S * 8, width=S * 8, num_inference_steps=steps, guidance_scale=8.5,
                       negative_prompt=[""], latents=inp["latents"].clone(), output_type="latent", run_rich_text=False,
                       callback=lambda i, t, lat: calls.append(i), callback_steps=1)
        assert m.scheduler.step_batches == [1] * steps
        assert calls == lo.callback_iterations(steps, steps, 1, 1) == list(range(steps)), calls
        res[f"xl_plain_{steps}"] = out.images.numpy()
        res[f"xl_plain_{steps}_callbacks"] = np.asarray(calls, np.int64)
    S = mo.LATENT_XL_RICH
    inp = gg.synth_inputs(cfg, 3, S, 31)
    ctx, te = inp["ctx"], inp["text_embeds"]
    for sa, bg in RICH:
        m = gg.make_xl_sampler(ns, cfg, 2, (ctx[1:], ctx[:1], te[1:], te[:1]))
        m.scheduler = lo.LMSSchedulerOracle()
        m.masks = inp["masks"]
        tfd = gg.text_format(1, S, 31)
        tfd.update(gg.color_dict(inp["masks"], S, weight=1.0))
        calls = []
        out = m.sample(["a", "b", "c"], height=S * 8, width=S * 8, num_inference_steps=RICH_STEPS, guidance_scale=8.5,
                       negative_prompt=[""], latents=inp["latents"].clone(), output_type="latent", use_guidance=True,
                       inject_selfattn=sa, inject_background=bg, text_format_dict=tfd, run_rich_text=True,
                       callback=lambda i, t, lat: calls.append(i), callback_steps=1)
        batches = m.scheduler.step_batches
        assert len(batches) == RICH_STEPS and len(set(batches)) == 1, batches   # well defined in the reference
        assert batches[0] == (2 if sa > 0 or bg > 0 else 1), batches
        assert calls == lo.callback_iterations(RICH_STEPS, RICH_STEPS, 1, 1), calls
        print("rich", sa, bg, "step batches", batches, "callbacks", calls)
        res[f"xl_rich_{sa:g}_{bg:g}"] = out.images.detach().numpy()
        res[f"xl_rich_{sa:g}_{bg:g}_callbacks"] = np.asarray(calls, np.int64)
    np.savez_compressed(os.path.join(gg.GOLD, "lms.npz"), **res)
    print("lms ok", {k: float(np.abs(v).mean()) for k, v in res.items()})


if __name__ == "__main__":
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    gen_lms(ref_shim.import_reference())
