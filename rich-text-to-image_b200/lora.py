"""LoRA checkpoints merged into the UNet and CLIP text-encoder weights.

One LoRA at a time is merged into the weights it targets, W = W0 + s * (alpha / r) * up @ down, so a denoising step runs
exactly the kernels it runs without one. The merge is computed on the weights' device: up @ down in fp32, added to the
fp32 upcast of the fp16 W0, rounded once to the weight's dtype and written with `copy_` into the existing parameter
(its memory layout is kept and `_version` moves on, which rebuilds Attention.fused_weight()). W0 is kept for every
module the LoRA touches, and every scale is computed from it: s -> s' -> s gives the bits of s, scale 0 and unloading
give W0's bits.

Formats:
  * kohya / A1111: `<stem>.lora_down.weight`, `<stem>.lora_up.weight`, optional `<stem>.alpha` (default: the rank).
    UNet stems are `lora_unet_` + a module path with `_` for `.`, either in diffusers' naming
    (`down_blocks_0_attentions_0_...`) or in the original UNet's (`input_blocks_N_M_...`, `middle_block_M_...`,
    `output_blocks_N_M_...`, with the resnets' `in_layers_2`, `emb_layers_1`, `out_layers_3`, `skip_connection` and the
    downsamplers' `op`), as kohya's SDXL trainer writes them. Text-encoder stems are `lora_te_` (SD1.5) or `lora_te1_` /
    `lora_te2_` (SDXL) + the `transformers` CLIP module path.
  * diffusers' UNet attention processors: `[unet.]<module path>.processor.to_{q,k,v,out}_lora.{down,up}.weight`
    (alpha = rank).
Targets: every nn.Linear and nn.Conv2d of the UNet's down, mid and up blocks (attention projections, feed-forward,
proj_in / proj_out, the resnets' convolutions, time_emb_proj and shortcut, the down- and upsampler convolutions), and the
linears of the CLIP encoder layers (self_attn q/k/v/out_proj, mlp.fc1 / fc2).
"""
import re

import torch
import torch.nn as nn

_KOHYA = re.compile(r"^(lora_unet|lora_te[12]?)_(.+)\.(lora_down\.weight|lora_up\.weight|alpha)$")
_DIFFUSERS = re.compile(r"^(?:unet\.)?(.+)\.processor\.(to_q|to_k|to_v|to_out)_lora\.(down|up)\.weight$")
_LYCORIS = ("hada_", "lokr_", "lora_mid", "dora_scale", ".diff", ".w_norm", ".b_norm")
# inner module names of the original (SGM) UNet blocks -> ours
_SGM_RESNET = {"conv1": "in_layers.2", "time_emb_proj": "emb_layers.1", "conv2": "out_layers.3",
               "conv_shortcut": "skip_connection"}


def _sgm_blocks(cfg):
    """Our block prefix -> the original UNet's (input_blocks / middle_block / output_blocks), from the config."""
    L = cfg.layers_per_block
    last = len(cfg.block_out_channels) - 1
    out = {}
    for i in range(len(cfg.down_block_types)):
        for l in range(L):
            n = 1 + i * (L + 1) + l
            out[f"down_blocks.{i}.resnets.{l}"] = f"input_blocks.{n}.0"
            out[f"down_blocks.{i}.attentions.{l}"] = f"input_blocks.{n}.1"
        if i != last:
            out[f"down_blocks.{i}.downsamplers.0"] = f"input_blocks.{(i + 1) * (L + 1)}.0"
    out.update({"mid_block.resnets.0": "middle_block.0", "mid_block.attentions.0": "middle_block.1",
                "mid_block.resnets.1": "middle_block.2"})
    for i, typ in enumerate(cfg.up_block_types):
        for l in range(L + 1):
            n = i * (L + 1) + l
            out[f"up_blocks.{i}.resnets.{l}"] = f"output_blocks.{n}.0"
            out[f"up_blocks.{i}.attentions.{l}"] = f"output_blocks.{n}.1"
        if i != last:   # the upsampler is the last entry of the block's last output_blocks row
            out[f"up_blocks.{i}.upsamplers.0"] = f"output_blocks.{i * (L + 1) + L}.{2 if typ == 'CrossAttnUpBlock2D' else 1}"
    return out


def _sgm_name(name, blocks):
    m = re.match(r"^((?:down_blocks|up_blocks)\.\d+\.(?:resnets|attentions|downsamplers|upsamplers)\.\d+"
                 r"|mid_block\.(?:resnets|attentions)\.\d+)\.(.+)$", name)
    prefix, rest = m.group(1), m.group(2)
    if ".resnets." in prefix:
        rest = _SGM_RESNET[rest]
    elif ".downsamplers." in prefix:
        rest = "op"
    return f"{blocks[prefix]}.{rest}"


def unet_targets(unet):
    """Module name -> module of every UNet layer a LoRA may target."""
    return {n: m for n, m in unet.named_modules() if isinstance(m, (nn.Linear, nn.Conv2d))
            and n.split(".")[0] in ("down_blocks", "mid_block", "up_blocks")}


def clip_targets(text_encoder):
    return {n: m for n, m in text_encoder.named_modules()
            if isinstance(m, nn.Linear) and n.startswith("text_model.encoder.layers.")}


def kohya_names(unet, text_encoders=()):
    """kohya stem -> (component, module name) for every target: the UNet in both naming schemes, then the text
    encoders in order (`lora_te` for one encoder, `lora_te1` / `lora_te2` for two)."""
    out = {}

    def add(stem, comp, name):
        if stem in out:
            raise AssertionError(f"two modules share the LoRA name {stem}")
        out[stem] = (comp, name)
    blocks = _sgm_blocks(unet.config)
    for name in unet_targets(unet):
        add("lora_unet_" + name.replace(".", "_"), "unet", name)
        add("lora_unet_" + _sgm_name(name, blocks).replace(".", "_"), "unet", name)
    tags = ["lora_te"] if len(text_encoders) == 1 else [f"lora_te{i + 1}" for i in range(len(text_encoders))]
    for i, (tag, enc) in enumerate(zip(tags, text_encoders)):
        for name in clip_targets(enc):
            add(f"{tag}_" + name.replace(".", "_"), f"te{i + 1}", name)
    return out


def read_lora(path_or_dict):
    """stem -> {"down", "up", "alpha"} and the format, from a .safetensors path or a state dict."""
    if isinstance(path_or_dict, dict):
        sd = path_or_dict
    else:
        from safetensors.torch import load_file
        sd = load_file(str(path_or_dict))
    groups, formats = {}, set()
    for key, t in sd.items():
        if any(s in key for s in _LYCORIS):
            raise ValueError(f"LoRA key {key!r}: LyCORIS (LoHa, LoKr, LoCon with a mid weight) and DoRA weights are not "
                             "supported; only plain LoRA (lora_down / lora_up) can be loaded")
        if key.startswith(("text_encoder.", "text_encoder_2.")):
            raise ValueError(f"LoRA key {key!r}: diffusers-format text-encoder weights are not supported; "
                             "use a kohya-format (lora_te*) file for text-encoder LoRA")
        m = _KOHYA.match(key)
        if m:
            formats.add("kohya")
            stem, part = f"{m.group(1)}_{m.group(2)}", {"lora_down.weight": "down", "lora_up.weight": "up"}.get(m.group(3), "alpha")
        elif _DIFFUSERS.match(key):
            m = _DIFFUSERS.match(key)
            formats.add("diffusers")
            proj = "to_out.0" if m.group(2) == "to_out" else m.group(2)
            stem, part = f"{m.group(1)}.{proj}", m.group(3)
        else:
            raise ValueError(f"LoRA key {key!r} is in no supported format (kohya lora_unet_* / lora_te*_*, "
                             "or diffusers' *.processor.to_*_lora.*)")
        groups.setdefault(stem, {})[part] = t
    if len(formats) > 1:
        raise ValueError("the LoRA mixes kohya and diffusers keys; load one LoRA at a time")
    for stem, g in groups.items():
        if "down" not in g or "up" not in g:
            raise ValueError(f"LoRA module {stem!r} has no {'down' if 'down' not in g else 'up'} weight")
    return groups, (formats.pop() if formats else None)


def _check_shapes(stem, mod, down, up):
    w = mod.weight
    r = down.shape[0]
    if isinstance(mod, nn.Conv2d):
        ok = (down.dim() == 4 and up.dim() == 4 and up.shape[2:] == (1, 1) and down.shape[1:] == w.shape[1:]
              and up.shape[:2] == (w.shape[0], r))
    else:
        ok = down.dim() == 2 and up.dim() == 2 and down.shape[1] == w.shape[1] and up.shape == (w.shape[0], r)
    if not ok:
        raise ValueError(f"LoRA module {stem!r}: down {tuple(down.shape)} / up {tuple(up.shape)} do not fit the weight "
                         f"{tuple(w.shape)} of its target ({type(mod).__name__})")


class MergedLora:
    """A LoRA merged into its target modules; holds W0 of each of them (on their device, in their dtype)."""

    def __init__(self, path_or_dict, unet, text_encoders=()):
        groups, fmt = read_lora(path_or_dict)
        comps = {"unet": unet, **{f"te{i + 1}": e for i, e in enumerate(text_encoders)}}
        names = kohya_names(unet, text_encoders) if fmt == "kohya" else None
        targets = {c: (unet_targets(m) if c == "unet" else clip_targets(m)) for c, m in comps.items()}
        self.entries = []   # (module name, module, W0, down fp32, up fp32, alpha / rank)
        seen = set()
        for stem, g in groups.items():
            if fmt == "kohya":
                if stem.startswith("lora_te") and not text_encoders:
                    raise ValueError(f"LoRA module {stem!r} targets a text encoder, and none is loaded")
                if stem not in names:
                    raise ValueError(f"LoRA module {stem!r} maps to no module of this model")
                comp, name = names[stem]
            else:
                comp, name = "unet", stem
                if name not in targets["unet"]:
                    raise ValueError(f"LoRA module {stem!r} maps to no module of this model")
            if (comp, name) in seen:
                raise ValueError(f"LoRA module {stem!r}: its target {name} is named twice (both UNet naming schemes)")
            seen.add((comp, name))
            mod = targets[comp][name]
            down, up = g["down"], g["up"]
            _check_shapes(stem, mod, down, up)
            r = down.shape[0]
            alpha = float(g["alpha"]) if "alpha" in g else float(r)
            dev = mod.weight.device
            self.entries.append((f"{comp}:{name}", mod, mod.weight.detach().clone(),
                                 down.to(dev, torch.float32).flatten(1), up.to(dev, torch.float32).flatten(1), alpha / r))
        self.scale = None

    @torch.no_grad()
    def set_scale(self, scale):
        """W = W0 + scale * (alpha / r) * up @ down for every target, from W0 (fp32 GEMM, no TF32)."""
        scale = float(scale)
        prev = torch.backends.cuda.matmul.allow_tf32
        torch.backends.cuda.matmul.allow_tf32 = False
        try:
            for _, mod, w0, down, up, f in self.entries:
                if scale == 0.0:
                    mod.weight.copy_(w0)
                else:
                    w = torch.addmm(w0.float().flatten(1), up, down, alpha=scale * f)
                    mod.weight.copy_(w.view(w0.shape))
        finally:
            torch.backends.cuda.matmul.allow_tf32 = prev
        self.scale = scale

    @torch.no_grad()
    def unload(self):
        for _, mod, w0, _, _, _ in self.entries:
            mod.weight.copy_(w0)
        self.entries = []


class LoraLoaderMixin:
    """load_lora_weights / set_lora_scale / unload_lora_weights of the samplers. The sampler gives the UNet and its CLIP
    text encoders (in kohya's lora_te1, lora_te2 order) through `_lora_components()`."""

    _lora = None

    def _lora_components(self):
        raise NotImplementedError

    def load_lora_weights(self, path_or_dict, scale=1.0):
        """Merge a LoRA (.safetensors path or state dict, kohya or diffusers format) into the UNet and, when the model
        has them, the text encoders, at `scale`. Raises ValueError for a key that maps to no module, a shape that does
        not fit its target, LyCORIS / DoRA weights, or while another LoRA is loaded."""
        if self._lora is not None:
            raise ValueError("a LoRA is already loaded; call unload_lora_weights() first (several LoRAs at once are "
                             "not supported)")
        unet, encoders = self._lora_components()
        lora = MergedLora(path_or_dict, unet, encoders)
        lora.set_scale(scale)
        self._lora = lora

    def set_lora_scale(self, scale):
        """Re-merge the loaded LoRA at `scale`, from the original weights."""
        if self._lora is None:
            raise RuntimeError("no LoRA is loaded")
        if float(scale) != self._lora.scale:
            self._lora.set_scale(scale)

    def unload_lora_weights(self):
        """Restore the original weights (bit for bit). No-op when no LoRA is loaded."""
        if self._lora is not None:
            self._lora.unload()
            self._lora = None
