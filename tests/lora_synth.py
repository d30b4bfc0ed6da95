"""Seeded synthetic LoRA state dicts for the LoRA tests, the multi-GPU check and the benchmark, and an unmerged
evaluation of the oracle UNet (W0 x + s (alpha / r) up(down(x)), as diffusers runs an adapter)."""
import math

import torch
import torch.nn.functional as F


def lora_factors(targets, rank, seed, device="cpu", up_gain=0.5):
    """name -> (down, up) fp32 for every target module: down ~ N(0, 1/fan_in) (conv: the target's kernel, 1x1 up),
    up ~ up_gain * N(0, 1/rank), so that (alpha / rank) up @ down is a sizeable fraction of W0 ~ N(0, 1/fan_in)."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    out = {}
    for name in sorted(targets):
        w = targets[name].weight
        o, fan_in = w.shape[0], w[0].numel()
        r = min(rank, o, fan_in)
        down = torch.randn((r, *w.shape[1:]), generator=g) / math.sqrt(fan_in)
        up = torch.randn((o, r) + ((1, 1) if w.dim() == 4 else ()), generator=g) * (up_gain / math.sqrt(r))
        out[name] = (down.to(device), up.to(device))
    return out


def kohya_dict(factors, stems, alpha=None):
    """kohya-format state dict; stems: name -> kohya stem. alpha=None writes no .alpha key."""
    sd = {}
    for name, (down, up) in factors.items():
        s = stems[name]
        sd[s + ".lora_down.weight"] = down
        sd[s + ".lora_up.weight"] = up
        if alpha is not None:
            sd[s + ".alpha"] = torch.tensor(float(alpha))
    return sd


def diffusers_stem(name):
    return "lora_unet_" + name.replace(".", "_")


class UnmergedF:
    """Stands in for torch.nn.functional inside oracle.unet_oracle: F.linear / F.conv2d with a weight that has a
    LoRA (looked up by identity) add f * up(down(x)), the down convolution taking the target's stride and padding."""

    def __init__(self, table):
        self.table = {id(w): v for w, v in table}   # [(weight tensor, (down, up, f))]

    def __getattr__(self, name):
        return getattr(F, name)

    def linear(self, x, w, b=None):
        y = F.linear(x, w, b)
        e = self.table.get(id(w))
        if e is not None:
            down, up, f = e
            y = y + f * F.linear(F.linear(x, down), up)
        return y

    def conv2d(self, x, w, b=None, stride=1, padding=0):
        y = F.conv2d(x, w, b, stride, padding)
        e = self.table.get(id(w))
        if e is not None:
            down, up, f = e
            y = y + f * F.conv2d(F.conv2d(x, down, None, stride, padding), up)
        return y


def unmerged_table(sd, factors, scale, alpha, dtype=None):
    """[(sd weight, (down, up, scale * alpha / rank))] for UnmergedF, factors cast to `dtype` (default: the weight's)."""
    out = []
    for name, (down, up) in factors.items():
        w = sd[name + ".weight"]
        dt = dtype or w.dtype
        out.append((w, (down.to(w.device, dt), up.to(w.device, dt), scale * alpha / down.shape[0])))
    return out
