"""Region-parallel rich-text loop with a LoRA, run under torchrun on >= 2 GPUs:

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29551 tests/multigpu_lora_check.py

Every rank loads the same synthetic LoRA (kohya SDXL-trainer naming, every linear and conv of the UNet's blocks, scale
0.8) into the tiny SDXL-shaped UNet and runs the rich-text loop (3 regions, injection 0.5 / 0.5, font sizes, colour
guidance) three ways: the fused peer-memory gather+blend exchange, the NCCL all-gather exchange, and as a single-GPU
run (a process group of its own rank). The ranks' latents must be bit-identical for both exchanges, and equal to the
single-GPU latents within bench.py --check's tolerance (0.5 % of the dynamic range + 3 %: the UNet passes run in other
batch compositions there)."""
import os
import re
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests import lora_synth, synth  # noqa: E402


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    from oracle import unet_oracle as uo
    from rtti_b200 import lora
    from rtti_b200.region_diffusion_sdxl import RegionDiffusionXL
    from rtti_b200.unet import UNet2DConditionModel, UNetConfig
    cfg = uo.tiny_xl_config()
    unet = UNet2DConditionModel(UNetConfig.from_dict(cfg.__dict__))
    unet.load_state_dict(uo.make_state_dict(cfg, 2))
    unet.finalize("cuda")
    stems = {n: k for k, (_, n) in lora.kohya_names(unet).items() if re.match(r"lora_unet_(input|middle|output)_block", k)}
    lsd = lora_synth.kohya_dict(lora_synth.lora_factors(lora.unet_targets(unet), 8, 3), stems, 4.0)
    S = 128
    pooled = cfg.projection_class_embeddings_input_dim - 6 * cfg.addition_time_embed_dim
    inp = synth.synth_inputs(cfg.cross_attention_dim, pooled, 3, S, 31)
    ctx, te = inp["ctx"].cuda(), inp["text_embeds"].cuda()
    tfd = synth.font_sizes()
    tfd.update(synth.color_dict(inp["masks"], S, 1.0))
    solo = [dist.new_group([r]) for r in range(world)][rank]
    out = {}
    for name, group, fused in (("fused", None, True), ("nccl", None, False), ("single", solo, True)):
        model = RegionDiffusionXL(device="cuda", unet=unet, vae=synth.TinyVAE("cuda"))
        model.load_lora_weights(lsd, scale=0.8)
        model.region_group = group
        model.fused_exchange = fused
        model.masks = [m.cuda() for m in inp["masks"]]
        out[name] = model.sample(height=S * 8, width=S * 8, num_inference_steps=4, guidance_scale=8.5,
                                 latents=inp["latents"].clone(), prompt_embeds=ctx[1:], negative_prompt_embeds=ctx[:1],
                                 pooled_prompt_embeds=te[1:], negative_pooled_prompt_embeds=te[:1], output_type="latent",
                                 run_rich_text=True, use_guidance=True, inject_selfattn=0.5, inject_background=0.5,
                                 text_format_dict=tfd).images.float()
        model.unload_lora_weights()   # the next run's model loads it into the same UNet
        if name == "fused":
            assert model.fused_exchange and model._exchanges, "the fused peer-memory exchange was not used"
    ok = True
    for name in ("fused", "nccl"):
        a = out[name]
        gathered = [torch.empty_like(a) for _ in range(world)]
        dist.all_gather(gathered, a.contiguous())
        same = all(torch.equal(gathered[0], x) for x in gathered)
        b = out["single"]
        equal_single = bool(((a - b).abs() <= 5e-3 * float(b.abs().max()) + 3e-2 * b.abs()).all())
        ok = ok and same and equal_single and bool(torch.isfinite(a).all())
        if rank == 0:
            print(f"world={world} LoRA {name} exchange: ranks bit-identical: {same}, equal to the single-GPU run: "
                  f"{equal_single} (max diff {(a - b).abs().max().item():.3g})", flush=True)
    t = torch.tensor([0.0 if ok else 1.0], device="cuda")
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    ok = float(t) == 0.0
    if rank == 0:
        print("MULTIGPU_LORA_CHECK", "PASS" if ok else "FAIL", flush=True)
    dist.barrier()
    dist.destroy_process_group()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
