"""sample.py — command-line entry with the reference's flags (sample.py:117-134 of the reference), driving
the H100 samplers. Flow = reference sample.py:17-114: parse the rich-text JSON, plain pass with token-map
capture, get_token_maps (twice: colour masks, region masks), rich-text pass.

Extra flags: --load_path (LOCAL diffusers-format directory; there is no hub access in this environment),
--synthetic (random weights + random prompt embeddings, for smoke runs without checkpoints) and
--scheduler {default,ddim,dpmpp_2m,dpmpp_2s,euler_a,unipc,heun,lms} (default: PLMS for SD1.5, Euler for SDXL;
DPM-Solver++(2M) is the usual choice at about 20 --sample_steps, UniPC the sampler built for 5-10, dpmpp_2s
DPM-Solver++(2S), the singlestep variant; euler_a, Euler Ancestral, heun, Heun's
second-order method, which evaluates the UNet 2N - 1 times for N --sample_steps, and lms, k-LMS, are for SDXL / AnimeXL
only), --lora_path (a LOCAL LoRA .safetensors file, kohya or diffusers format, merged into the UNet and text-encoder
weights) with --lora_scale (default 1.0), and --textual_inversion PATH[:TOKEN] (repeatable; a LOCAL textual-inversion
embedding, diffusers, A1111 or SDXL format, added to the tokenizers after the LoRA; TOKEN defaults to the token the file
names).
"""
import argparse
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from rtti_b200.attention_utils import get_token_maps  # noqa: E402
from rtti_b200.region_diffusion import RegionDiffusion  # noqa: E402
from rtti_b200.region_diffusion_sdxl import RegionDiffusionXL  # noqa: E402
from rtti_b200.schedulers import (DDIMScheduler, DPMSolverMultistepScheduler, DPMSolverSinglestepScheduler,  # noqa: E402
                                  EulerAncestralDiscreteScheduler, HeunDiscreteScheduler, LMSDiscreteScheduler,
                                  UniPCMultistepScheduler)
from rtti_b200.richtext_utils import (get_attention_control_input, get_gradient_guidance_input,  # noqa: E402
                                      get_region_diffusion_input, parse_json, seed_everything)

DEFAULT_JSON = ('{"ops":[{"insert":"A close-up 4k dslr photo of a "},{"attributes":{"link":"A cat wearing sunglasses '
                'and a bandana around its neck."},"insert":"cat"},{"insert":" riding a scooter. There are palm trees '
                'in the background."}]}')


def _save(img, path):
    from PIL import Image
    (img if hasattr(img, "save") else Image.fromarray(img)).save(path)


def main(args, param):
    os.makedirs(args.run_dir, exist_ok=True)
    xl = args.model in ("SDXL", "AnimeXL")
    if args.scheduler in ("euler_a", "heun", "lms") and not xl:
        # the SD1.5 loop, like the reference's, never calls scale_model_input: the Euler family does not apply there
        raise SystemExit(f"--scheduler {args.scheduler} needs --model SDXL or AnimeXL: the SD1.5 sampler never scales the model "
                         "input, which the Euler schedulers require")
    if args.load_path is None:
        raise SystemExit("--load_path <local diffusers-format directory> is required (no hub access here); "
                         "use bench.py / tests for synthetic-weight runs")
    model = RegionDiffusionXL(load_path=args.load_path) if xl else RegionDiffusion("cuda", load_path=args.load_path)
    if args.scheduler != "default":
        model.scheduler = {"ddim": DDIMScheduler, "dpmpp_2m": DPMSolverMultistepScheduler,
                           "dpmpp_2s": DPMSolverSinglestepScheduler,
                           "euler_a": EulerAncestralDiscreteScheduler, "unipc": UniPCMultistepScheduler,
                           "heun": HeunDiscreteScheduler, "lms": LMSDiscreteScheduler}[args.scheduler]()
    if args.lora_path is not None:
        model.load_lora_weights(args.lora_path, scale=args.lora_scale)
    for spec in args.textual_inversion:
        path, sep, token = spec.rpartition(":")
        if not (sep and os.path.exists(path)):   # no ":TOKEN" suffix (or a ':' inside the path)
            path, token = spec, None
        model.load_textual_inversion(path, token=token or None)

    (base_prompt, style_prompts, footnote_prompts, footnote_targets, color_prompts, color_names, color_rgbs,
     sizes, use_grad_guidance) = parse_json(param["text_input"])
    region_prompts, region_token_ids, base_tokens = get_region_diffusion_input(
        model, base_prompt, style_prompts, footnote_prompts, footnote_targets, color_prompts, color_names)
    tfd = get_attention_control_input(model, base_tokens, sizes)
    tfd, color_token_ids = get_gradient_guidance_input(model, base_tokens, color_prompts, color_rgbs, tfd,
                                                       color_guidance_weight=args.color_guidance_weight)
    height, width, seed, negative = param["height"], param["width"], param["noise_index"], param["negative_prompt"]

    seed_everything(seed)
    t0 = time.time()
    model.register_tokenmap_hooks()
    if xl:
        plain = model.sample([base_prompt], negative_prompt=[negative], height=height, width=width,
                             num_inference_steps=param["steps"], guidance_scale=param["guidance_weight"], run_rich_text=False)
        _save(plain.images[0], os.path.join(args.run_dir, f"seed{seed}_plain.jpg"))
    else:
        plain = model.produce_attn_maps([base_prompt], [negative], height=height, width=width,
                                        num_inference_steps=param["steps"], guidance_scale=param["guidance_weight"])
        _save(plain[0], os.path.join(args.run_dir, f"seed{seed}_plain.jpg"))
    print("time lapses to get attention maps: %.4f" % (time.time() - t0))

    seed_everything(seed)
    kw = dict(segment_threshold=args.segment_threshold, num_segments=args.num_segments)
    color_masks = get_token_maps(model.selfattn_maps, model.crossattn_maps, model.n_maps, args.run_dir, height // 8,
                                 width // 8, color_token_ids[:-1], seed, base_tokens, **kw)
    atten_all = torch.zeros_like(color_masks[-1])
    for m in color_masks[:-1]:
        atten_all += m
    tfd["color_obj_atten"] = [torch.nn.functional.interpolate(m, (height, width), mode="bicubic", antialias=True)
                              for m in color_masks]
    tfd["color_obj_atten_all"] = atten_all
    seed_everything(seed)
    model.masks = get_token_maps(model.selfattn_maps, model.crossattn_maps, model.n_maps, args.run_dir, height // 8,
                                 width // 8, region_token_ids[:-1], seed, base_tokens, **kw)
    model.remove_tokenmap_hooks()

    t0 = time.time()
    seed_everything(seed)
    common = dict(height=height, width=width, num_inference_steps=param["steps"], guidance_scale=param["guidance_weight"],
                  use_guidance=use_grad_guidance, inject_selfattn=args.inject_selfattn, text_format_dict=tfd,
                  inject_background=args.inject_background)
    if xl:
        rich = model.sample(region_prompts, negative_prompt=[negative], run_rich_text=True, **common).images[0]
    else:
        rich = model.prompt_to_img(region_prompts, [negative], **common)[0]
    _save(rich, os.path.join(args.run_dir, f"seed{seed}_rich.jpg"))
    print("time lapses to generate image from rich text: %.4f" % (time.time() - t0))


if __name__ == "__main__":
    p = argparse.ArgumentParser()
    p.add_argument("--run_dir", type=str, default="results/")
    p.add_argument("--height", type=int, default=None)
    p.add_argument("--width", type=int, default=None)
    p.add_argument("--seed", type=int, default=6)
    p.add_argument("--sample_steps", type=int, default=41)
    p.add_argument("--rich_text_json", type=str, default=DEFAULT_JSON)
    p.add_argument("--negative_prompt", type=str, default="")
    p.add_argument("--model", type=str, default="SD", choices=["SD", "SDXL", "AnimeXL"])
    p.add_argument("--guidance_weight", type=float, default=8.5)
    p.add_argument("--color_guidance_weight", type=float, default=0.5)
    p.add_argument("--inject_selfattn", type=float, default=0.0)
    p.add_argument("--segment_threshold", type=float, default=0.3)
    p.add_argument("--num_segments", type=int, default=9)
    p.add_argument("--inject_background", type=float, default=0.0)
    p.add_argument("--load_path", type=str, default=None)
    p.add_argument("--scheduler", type=str, default="default",
                   choices=["default", "ddim", "dpmpp_2m", "dpmpp_2s", "euler_a", "unipc", "heun", "lms"])
    p.add_argument("--lora_path", type=str, default=None)
    p.add_argument("--lora_scale", type=float, default=1.0)
    p.add_argument("--textual_inversion", action="append", default=[], metavar="PATH[:TOKEN]")
    a = p.parse_args()
    res = 512 if a.model == "SD" else 1024
    main(a, {"text_input": json.loads(a.rich_text_json), "height": a.height or res, "width": a.width or res,
             "guidance_weight": a.guidance_weight, "steps": a.sample_steps, "noise_index": a.seed,
             "negative_prompt": a.negative_prompt})
