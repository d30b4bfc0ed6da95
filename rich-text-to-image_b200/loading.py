"""Loading real checkpoints from a LOCAL diffusers-format directory (no network access here).

The reference pulls `runwayml/stable-diffusion-v1-5` / `stabilityai/stable-diffusion-xl-base-1.0` from the
hub (models/region_diffusion.py:24-33, models/region_diffusion_sdxl.py:105-120). Parameter names of
unet.UNet2DConditionModel and vae.AutoencoderKLDecoder match the diffusers checkpoints, so loading is a
plain `load_state_dict`. Text encoders / tokenizers are third-party `transformers` CLIP models.
"""
import json
import os

import torch

from .textual_inversion import expand_prompt
from .unet import UNet2DConditionModel, UNetConfig
from .vae import AutoencoderKLDecoder, VAEConfig


def _read_weights(folder, stems=("diffusion_pytorch_model", "model")):
    from safetensors.torch import load_file
    for stem in stems:
        for suffix in (".fp16.safetensors", ".safetensors"):
            p = os.path.join(folder, stem + suffix)
            if os.path.exists(p):
                return load_file(p)
    raise FileNotFoundError(f"no safetensors weights under {folder}")


def _need_dir(path):
    if not os.path.isdir(path):
        raise FileNotFoundError(
            f"{path!r} is not a local directory. This build has no network access: download the diffusers-format "
            "model once and pass its path, or use RegionDiffusion*.from_synthetic() for random weights.")


def load_unet(folder, device):
    with open(os.path.join(folder, "config.json")) as f:
        cfg = UNetConfig.from_dict(json.load(f))
    unet = UNet2DConditionModel(cfg)
    missing, unexpected = unet.load_state_dict(_read_weights(folder), strict=False)
    if missing:
        raise RuntimeError(f"UNet checkpoint is missing {len(missing)} tensors, e.g. {missing[:4]}")
    return unet.finalize(device)


_VAE_RENAMES = {"query": "to_q", "key": "to_k", "value": "to_v", "proj_attn": "to_out.0"}


def load_vae(folder, device, scaling_factor):
    with open(os.path.join(folder, "config.json")) as f:
        raw = json.load(f)
    cfg = VAEConfig(latent_channels=raw.get("latent_channels", 4), out_channels=raw.get("out_channels", 3),
                    block_out_channels=tuple(raw.get("block_out_channels", (128, 256, 512, 512))),
                    layers_per_block=raw.get("layers_per_block", 2), norm_num_groups=raw.get("norm_num_groups", 32),
                    scaling_factor=raw.get("scaling_factor", scaling_factor))
    vae = AutoencoderKLDecoder(cfg)
    sd = {}
    for k, v in _read_weights(folder).items():
        if not (k.startswith("decoder.") or k.startswith("post_quant_conv.")):
            continue
        for old, new in _VAE_RENAMES.items():  # pre-0.18 attention parameter names
            k = k.replace(f".attentions.0.{old}.", f".attentions.0.{new}.")
        sd[k] = v
    vae.load_state_dict(sd, strict=True)
    return vae.finalize(device)


class ClipTextEncoders:
    """CLIP tokenizer(s) + text encoder(s) (third-party `transformers`), as used by the reference at
    models/region_diffusion.py:53-83 and models/region_diffusion_sdxl.py:256-440."""

    def __init__(self, root, device, xl):
        from transformers import CLIPTextModel, CLIPTextModelWithProjection, CLIPTokenizer
        self.xl = xl
        self.tokenizer = CLIPTokenizer.from_pretrained(os.path.join(root, "tokenizer"))
        self.text_encoder = CLIPTextModel.from_pretrained(os.path.join(root, "text_encoder"), torch_dtype=torch.float16).to(device)
        if xl:
            self.tokenizer_2 = CLIPTokenizer.from_pretrained(os.path.join(root, "tokenizer_2"))
            self.text_encoder_2 = CLIPTextModelWithProjection.from_pretrained(
                os.path.join(root, "text_encoder_2"), torch_dtype=torch.float16).to(device)

    def _ids(self, tok, prompts, device):
        prompts = [expand_prompt(tok, p) for p in prompts]   # multi-vector textual-inversion tokens (textual_inversion.py)
        return tok(prompts, padding="max_length", max_length=tok.model_max_length, truncation=True,
                   return_tensors="pt").input_ids.to(device)

    @torch.no_grad()
    def encode_pair(self, prompt, negative_prompt, device):
        """SD1.5: cat([uncond, cond...]) of the last hidden state (region_diffusion.py:47-67)."""
        cond = self.text_encoder(self._ids(self.tokenizer, list(prompt), device))[0]
        unc = self.text_encoder(self._ids(self.tokenizer, list(negative_prompt), device))[0]
        return torch.cat([unc, cond])

    @torch.no_grad()
    def encode(self, prompt, negative_prompt, device, force_zeros_for_empty_prompt=True):
        """SDXL: penultimate hidden states of both encoders concatenated + pooled output of encoder 2
        (region_diffusion_sdxl.py:326-440). negative_prompt=[''] is encoded, not zeroed; negative_prompt=None with
        `force_zeros_for_empty_prompt` gives zero negative / negative-pooled embeddings (:368-373)."""
        def run(prompts):
            embs, pooled = [], None
            for tok, enc in ((self.tokenizer, self.text_encoder), (self.tokenizer_2, self.text_encoder_2)):
                out = enc(self._ids(tok, prompts, device), output_hidden_states=True)
                pooled = out[0]
                embs.append(out.hidden_states[-2])
            return torch.cat(embs, dim=-1), pooled
        prompt = [prompt] if isinstance(prompt, str) else list(prompt)
        zero_negative = negative_prompt is None and force_zeros_for_empty_prompt
        negative_prompt = [negative_prompt or ""] if not isinstance(negative_prompt, (list, tuple)) else list(negative_prompt)
        pe, pp = run(prompt)
        if zero_negative:
            return pe, torch.zeros_like(pe[:1]), pp, torch.zeros_like(pp[:1])
        ne, npool = run(negative_prompt[:1])
        return pe, ne, pp, npool


def load_sdxl_components(load_path, device):
    _need_dir(load_path)
    from .schedulers import EulerDiscreteScheduler
    unet = load_unet(os.path.join(load_path, "unet"), device)
    vae = load_vae(os.path.join(load_path, "vae"), device, 0.13025)
    return unet, vae, EulerDiscreteScheduler(), ClipTextEncoders(load_path, device, xl=True)


def load_sd15_components(load_path, device):
    _need_dir(load_path)
    unet = load_unet(os.path.join(load_path, "unet"), device)
    vae = load_vae(os.path.join(load_path, "vae"), device, 0.18215)
    return unet, vae, ClipTextEncoders(load_path, device, xl=False)
