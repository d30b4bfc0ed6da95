"""Region-parallel guidance_rescale check, run under torchrun on >= 2 GPUs:

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29537 tests/multigpu_rescale_check.py

Every rank runs the tiny SDXL-shaped rich-text loop (3 regions, injection, font sizes, colour guidance) at
guidance_rescale 0.7 with the fused peer-memory gather+blend kernel (rtti_gather_blend_step_rescale), then the same loop
as a single-GPU run (a process group of its own rank: all passes local, rtti_region_blend_cfg_rescale). The ranks'
region-parallel latents must be bit-identical and within bench.py --check's tolerance of the single-GPU latents
(0.5 % of the dynamic range + 3 %)."""
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests import synth  # noqa: E402


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    from oracle import unet_oracle as uo
    from rtti_b200 import ops
    from rtti_b200.region_diffusion_sdxl import RegionDiffusionXL
    from rtti_b200.unet import UNet2DConditionModel, UNetConfig
    cfg = uo.tiny_xl_config()
    unet = UNet2DConditionModel(UNetConfig.from_dict(cfg.__dict__))
    unet.load_state_dict(uo.make_state_dict(cfg, 2))
    unet.finalize("cuda")
    S = 128
    pooled = cfg.projection_class_embeddings_input_dim - 6 * cfg.addition_time_embed_dim
    inp = synth.synth_inputs(cfg.cross_attention_dim, pooled, 3, S, 31)
    ctx, te = inp["ctx"].cuda(), inp["text_embeds"].cuda()
    tfd = synth.font_sizes()
    tfd.update(synth.color_dict(inp["masks"], S, 1.0))
    solo = [dist.new_group([r]) for r in range(world)][rank]
    out = {}
    launches = {}
    for name, group in (("fused", None), ("single", solo)):
        model = RegionDiffusionXL(device="cuda", unet=unet, vae=synth.TinyVAE("cuda"))
        model.region_group = group
        model.masks = [m.cuda() for m in inp["masks"]]
        n0 = ops.LAUNCHES
        out[name] = model.sample(height=S * 8, width=S * 8, num_inference_steps=4, guidance_scale=8.5,
                                 latents=inp["latents"].clone(), prompt_embeds=ctx[1:], negative_prompt_embeds=ctx[:1],
                                 pooled_prompt_embeds=te[1:], negative_pooled_prompt_embeds=te[:1], output_type="latent",
                                 run_rich_text=True, use_guidance=True, inject_selfattn=0.5, inject_background=0.5,
                                 text_format_dict=tfd, guidance_rescale=0.7).images.float()
        launches[name] = ops.LAUNCHES - n0
        if name == "fused":
            assert model.fused_exchange and model._exchanges, "the fused peer-memory exchange was not used"
    gathered = [torch.empty_like(out["fused"]) for _ in range(world)]
    dist.all_gather(gathered, out["fused"].contiguous())
    same = all(torch.equal(gathered[0], x) for x in gathered)
    a, b = out["fused"], out["single"]
    err = (a - b).abs()
    tol = 5e-3 * float(b.abs().max()) + 3e-2 * b.abs()
    close = bool((err <= tol).all()) and bool(torch.isfinite(a).all())
    t = torch.tensor([0.0 if close and same else 1.0], device="cuda")
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    ok = float(t) == 0.0
    if rank == 0:
        print(f"world={world} guidance_rescale 0.7 fused exchange: ranks bit-identical: {same}, vs single-GPU run max err "
              f"{err.max().item():.4f} (ref absmax {b.abs().max().item():.3f}, {'OK' if close else 'FAIL'})", flush=True)
        print("MULTIGPU_RESCALE_CHECK", "PASS" if ok else "FAIL", flush=True)
    dist.barrier()
    dist.destroy_process_group()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
