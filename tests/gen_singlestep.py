"""TEST INFRASTRUCTURE — generates tests/golden/singlestep.npz (and nothing else) by running the UNMODIFIED reference
through oracle/ref_shim.py with the restated DPM-Solver++(2S) scheduler of tests/singlestep_oracle.py assigned to its
`scheduler`, on the inputs of tests/gen_unipc.py (same seeds and latent sides).

Run where the reference tree exists (never on the GPU box):
    python -m tests.gen_singlestep
It records
  - the SDXL plain pass (:879-914; tiny XL, 32^2 latent, guidance 8.5) at 5 steps (odd: a final first-order step) and 10
    (even), with the iterations at which the reference calls back (callback_steps 1);
  - the SDXL rich loop (:772-878; 128^2, 3 regions, font sizes, no colour guidance: see RICH) at 4 steps with
    inject_selfattn = inject_background = 0.5 (the reference latents are stepped jointly on every step, so one batch-2
    scheduler state is one state per trajectory) and with inject_selfattn = inject_background = 0 (no reference
    latents), and its callback iterations;
  - SD1.5 produce_latents (models/region_diffusion.py:86-174; tiny SD, 64^2, colour guidance, injection) at 5 steps.
In every recorded case the batch of the scheduler's step calls is constant: asserted below.
"""
import os

import numpy as np
import torch

from oracle import gen_golden as gg
from oracle import ref_shim, unet_oracle as uo
from tests import multistep_oracle as mo
from tests import singlestep_oracle as so

PLAIN = (5, 10)
RICH_STEPS = 4
# (inject_selfattn, inject_background) -> colour guidance on. Colour guidance differentiates through the clamp of the
# decoded image to [0, 1], a kink in the gradient. On these fixtures the decoded image spans about +-800, so thousands of
# pixels lie inside (0, 1) and some always sit within rounding (fp32 on another CPU: up to 2e-3; the fp16 product on
# the GPU: more) of the kink; the 0 / 0 run's nearest one is 3e-4 away. A pixel that crosses it changes the guidance
# gradient by a finite step, which the following steps carry on. The XL rich runs therefore pin the loop without
# guidance, a smooth function of its inputs; the SD1.5 run keeps colour guidance.
RICH = {(0.5, 0.5): False, (0.0, 0.0): False}
SD_STEPS = 5


def gen_singlestep(ns):
    if ns.region_diffusion_sdxl is None:
        raise RuntimeError(ns.region_diffusion_sdxl_error)
    res = {}
    cfg = uo.tiny_xl_config()
    S = mo.LATENT_XL_PLAIN
    inp = gg.synth_inputs(cfg, 3, S, 31)
    ctx, te = inp["ctx"], inp["text_embeds"]
    for steps in PLAIN:
        m = gg.make_xl_sampler(ns, cfg, 2, (ctx[-1:], ctx[:1], te[-1:], te[:1]))
        m.scheduler = so.DPMSolverSinglestepSchedulerOracle()
        calls = []
        out = m.sample(["x"], height=S * 8, width=S * 8, num_inference_steps=steps, guidance_scale=8.5,
                       negative_prompt=[""], latents=inp["latents"].clone(), output_type="latent", run_rich_text=False,
                       callback=lambda i, t, lat: calls.append(i), callback_steps=1)
        assert m.scheduler.step_batches == [1] * steps
        assert calls == so.callback_iterations(steps) == list(range(steps)), calls
        res[f"xl_plain_{steps}"] = out.images.numpy()
        res[f"xl_plain_{steps}_callbacks"] = np.asarray(calls, np.int64)
    S = mo.LATENT_XL_RICH
    inp = gg.synth_inputs(cfg, 3, S, 31)
    ctx, te = inp["ctx"], inp["text_embeds"]
    for (sa, bg), colour in RICH.items():
        m = gg.make_xl_sampler(ns, cfg, 2, (ctx[1:], ctx[:1], te[1:], te[:1]))
        m.scheduler = so.DPMSolverSinglestepSchedulerOracle()
        m.masks = inp["masks"]
        tfd = gg.text_format(1, S, 31)
        tfd.update(gg.color_dict(inp["masks"], S, weight=1.0))
        calls = []
        out = m.sample(["a", "b", "c"], height=S * 8, width=S * 8, num_inference_steps=RICH_STEPS, guidance_scale=8.5,
                       negative_prompt=[""], latents=inp["latents"].clone(), output_type="latent", use_guidance=colour,
                       inject_selfattn=sa, inject_background=bg, text_format_dict=tfd, run_rich_text=True,
                       callback=lambda i, t, lat: calls.append(i), callback_steps=1)
        batches = m.scheduler.step_batches
        assert len(batches) == RICH_STEPS and len(set(batches)) == 1, batches
        assert batches[0] == (2 if sa > 0 or bg > 0 else 1), batches
        assert calls == so.callback_iterations(RICH_STEPS), calls
        res[f"xl_rich_{sa:g}_{bg:g}"] = out.images.detach().numpy()
        res[f"xl_rich_{sa:g}_{bg:g}_callbacks"] = np.asarray(calls, np.int64)
    cfg = uo.tiny_sd_config()
    S = mo.LATENT_SD
    inp = gg.synth_inputs(cfg, 3, S, 21)
    m = gg.make_sd_sampler(ns, cfg, 1)
    m.scheduler = so.DPMSolverSinglestepSchedulerOracle()
    m.masks = inp["masks"]
    m.vae = gg._TinyVAE()
    tfd = gg.text_format(1, S, 21)
    tfd.update(gg.color_dict(inp["masks"], S, weight=0.5))
    lat = m.produce_latents(inp["ctx"], height=S * 8, width=S * 8, num_inference_steps=SD_STEPS, guidance_scale=8.5,
                            latents=inp["latents"].clone(), use_guidance=True, text_format_dict=tfd,
                            inject_selfattn=0.3, inject_background=0.5)
    assert m.scheduler.step_batches == [2] * SD_STEPS, m.scheduler.step_batches
    res[f"sd_rich_{SD_STEPS}"] = lat.detach().numpy()
    np.savez_compressed(os.path.join(gg.GOLD, "singlestep.npz"), **res)
    print("singlestep ok", {k: float(np.abs(v).mean()) for k, v in res.items()})


if __name__ == "__main__":
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    gen_singlestep(ref_shim.import_reference())
