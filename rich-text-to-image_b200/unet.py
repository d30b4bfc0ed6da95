"""UNet2DConditionModel on the H100 kernels for the region-diffusion sampler.

Mirrors the interface and parameter names of the reference's patched UNet (models/unet_2d_condition.py:703-983,
unet_2d_blocks.py, transformer_2d.py:270-310, attention.py:131-206, resnet.py:591-645) so diffusers-format
checkpoints load unchanged, but is organised for the hardware instead of for hooks:

  * activations are channels-last fp16 `[B, H*W, C]` end to end (no NCHW<->NHWC permute copies around the
    transformers, cuDNN NHWC tensor-core convolutions);
  * every normalisation / gating op and both attentions run in the hand-written sm_90a kernels of
    librtti_b200.so (ops.py); GEMMs and 3x3 convolutions are plain library calls (cuBLASLt / cuDNN);
  * the reference's per-pass PyTorch hooks (token-map capture, self-attention / feature injection,
    font-size re-weighting; models/region_diffusion_sdxl.py:959-1140) are a `RegionControl` argument:
    ALL passes of a denoising step run as ONE batched call, and "inject the reference pass's
    self-attention" is an index (`qk_src`) handed to the attention kernel;
  * K/V of the 77 text tokens depend only on the prompt, so they are projected once per sampling call
    (`CrossKVCache`) instead of once per layer per step.
"""
import math
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import ops

FEATURE_INJECT_RESNET = "up_blocks.1.resnets.1"  # models/region_diffusion_sdxl.py:1055,1104


@dataclass
class UNetConfig:
    """Constructor arguments of the reference UNet (models/unet_2d_condition.py:160-212) used by SD1.5 / SDXL."""
    sample_size: int = 64
    in_channels: int = 4
    out_channels: int = 4
    down_block_types: Tuple[str, ...] = ("CrossAttnDownBlock2D", "CrossAttnDownBlock2D", "CrossAttnDownBlock2D", "DownBlock2D")
    up_block_types: Tuple[str, ...] = ("UpBlock2D", "CrossAttnUpBlock2D", "CrossAttnUpBlock2D", "CrossAttnUpBlock2D")
    block_out_channels: Tuple[int, ...] = (320, 640, 1280, 1280)
    layers_per_block: int = 2
    transformer_layers_per_block: Tuple[int, ...] = (1, 1, 1, 1)
    attention_head_dim: Tuple[int, ...] = (8, 8, 8, 8)  # number of heads (unet_2d_condition.py:228)
    cross_attention_dim: int = 768
    use_linear_projection: bool = False
    addition_embed_type: Optional[str] = None
    addition_time_embed_dim: Optional[int] = None
    projection_class_embeddings_input_dim: Optional[int] = None
    norm_num_groups: int = 32
    norm_eps: float = 1e-5
    flip_sin_to_cos: bool = True
    freq_shift: int = 0

    @staticmethod
    def sd15():
        return UNetConfig()

    @staticmethod
    def sdxl():
        return UNetConfig(sample_size=128, down_block_types=("DownBlock2D", "CrossAttnDownBlock2D", "CrossAttnDownBlock2D"),
                          up_block_types=("CrossAttnUpBlock2D", "CrossAttnUpBlock2D", "UpBlock2D"),
                          block_out_channels=(320, 640, 1280), transformer_layers_per_block=(1, 2, 10),
                          attention_head_dim=(5, 10, 20), cross_attention_dim=2048, use_linear_projection=True,
                          addition_embed_type="text_time", addition_time_embed_dim=256,
                          projection_class_embeddings_input_dim=2816)

    @staticmethod
    def from_dict(d):
        keys = UNetConfig.__dataclass_fields__.keys()
        kw = {k: (tuple(v) if isinstance(v, list) else v) for k, v in d.items() if k in keys}
        n = len(kw.get("block_out_channels", (0,) * 4))
        for k in ("transformer_layers_per_block", "attention_head_dim"):
            if k in kw and isinstance(kw[k], int):
                kw[k] = (kw[k],) * n
        return UNetConfig(**kw)


class TokenMapAccumulator:
    """On-device replacement of the token-map capture hooks (models/region_diffusion_sdxl.py:959-1009,
    models/region_diffusion.py:397-443): fp32 accumulators written by the attention kernels, no D2H copy.

    Semantics kept from the reference: per-module call counter `n_maps`, capture starts at call 11, only the
    conditional batch row is kept, cross maps only for the allow-listed layers; `sd_overwrite_bug=True`
    reproduces region_diffusion.py:423 (`name in crossattn_maps` in the self branch: SD1.5 self maps are
    overwritten, not summed). `self_resolutions`: which self-attention sizes to keep — the reference keeps
    all of them but utils/attention_utils.py:243-248 only ever reads the 32x32 ones."""

    def __init__(self, cross_layers, self_layers=None, start_after=10, sd_overwrite_bug=False,
                 self_resolutions=(32,)):
        self.cross_layers = set(cross_layers)
        self.self_layers = None if self_layers is None else set(self_layers)
        self.start_after = start_after
        self.sd_overwrite_bug = sd_overwrite_bug
        self.self_resolutions = None if self_resolutions is None else set(self_resolutions)
        self.selfattn_maps: Dict[str, torch.Tensor] = {}
        self.crossattn_maps: Dict[str, torch.Tensor] = {}
        self.n_maps: Dict[str, int] = {}

    def tick(self, name):
        self.n_maps[name] = self.n_maps.get(name, 0) + 1
        return self.n_maps[name] > self.start_after

    def cross_target(self, name, n_q, n_k, device):
        """fp32 [1, n_q, n_k] accumulator for this call, or None."""
        if not self.tick(name) or name not in self.cross_layers:
            return None
        if name not in self.crossattn_maps:
            self.crossattn_maps[name] = torch.zeros(1, n_q, n_k, dtype=torch.float32, device=device)
        return self.crossattn_maps[name]

    def self_target(self, name, n_q, device):
        if not self.tick(name):
            return None
        if self.self_layers is not None and name not in self.self_layers:
            return None
        if self.self_resolutions is not None and int(round(math.sqrt(n_q))) not in self.self_resolutions:
            return None
        if name not in self.selfattn_maps:
            self.selfattn_maps[name] = torch.zeros(1, n_q, n_q, dtype=torch.float32, device=device)
        elif self.sd_overwrite_bug and name not in self.crossattn_maps:
            self.selfattn_maps[name].zero_()  # overwritten, not accumulated (region_diffusion.py:423-426)
        return self.selfattn_maps[name]


class CrossKVCache:
    """K/V projections of the text context per cross-attention layer; valid for one set of prompts."""

    def __init__(self):
        self.kv: Dict[str, torch.Tensor] = {}


@dataclass
class RegionControl:
    """Per-call description of what the reference does with hooks around each UNet pass."""
    qk_src: Optional[List[int]] = None          # self-attn injection: entry b uses Q,K of entry qk_src[b]
    feature_src: Optional[List[int]] = None     # up_blocks.1.resnets.1 hidden-state injection, same indexing
    feature_idx: Optional[torch.Tensor] = None  # the same as a device int64 tensor (avoids an H2D copy per call)
    word_pos: Optional[torch.Tensor] = None     # int32 [n]  (font-size re-weighting, attn2 only)
    font_size: Optional[torch.Tensor] = None    # fp32 [n]
    fs_batch_mask: int = 0                      # bit b set -> entry b gets the re-weighting (pass B only)
    capture: Optional[TokenMapAccumulator] = None
    capture_row: int = 1                        # batch row kept by the capture (the conditional one)
    kv_cache: Optional[CrossKVCache] = None
    # multi-GPU, injection steps: hand-off of pass D's self-attention Q|K and resnet feature between ranks
    # (region_parallel.RemoteQK role object: .is_src / .is_dst, push / wait / views), None = everything is local
    remote: Optional[object] = None


def _f16(t):
    return t.to(torch.float16)


class GroupNormCL(nn.Module):
    """GroupNorm parameters; applied by ops.groupnorm_silu on channels-last activations."""

    def __init__(self, groups, channels, eps):
        super().__init__()
        self.groups, self.eps = groups, eps
        self.weight = nn.Parameter(torch.ones(channels))
        self.bias = nn.Parameter(torch.zeros(channels))

    def forward(self, x, silu, chan_bias=None):
        return ops.groupnorm_silu(x, self.weight, self.bias, self.groups, self.eps, silu, chan_bias=chan_bias)


class LayerNormCL(nn.Module):
    def __init__(self, channels, eps=1e-5):
        super().__init__()
        self.eps = eps
        self.weight = nn.Parameter(torch.ones(channels))
        self.bias = nn.Parameter(torch.zeros(channels))

    def forward(self, x):
        return ops.layernorm(x, self.weight, self.bias, self.eps)


class Conv2dCL(nn.Conv2d):
    """nn.Conv2d over channels-last activations given as [B, H, W, C] (cuDNN NHWC path)."""

    def forward_cl(self, x, H, W, with_bias=True):
        """with_bias=False: the caller folds self.bias into the consumer (the next GroupNorm's per-channel bias or the
        fused residual add) — PyTorch adds the bias of a channels-last convolution in a separate broadcast pass."""
        B = x.shape[0]
        x4 = x.view(B, H, W, -1).permute(0, 3, 1, 2)  # logical NCHW, channels_last memory: no copy
        y = F.conv2d(x4, self.weight, self.bias if with_bias else None, self.stride, self.padding)
        Ho, Wo = y.shape[2], y.shape[3]
        y = y.permute(0, 2, 3, 1)
        if not y.is_contiguous():
            y = y.contiguous()
        return y.reshape(B, Ho * Wo, -1), Ho, Wo


class Attention(nn.Module):
    """Parameters of the reference `Attention` (models/attention_processor.py:35-160); the math is
    ops.attention (rtti_attn_fwd)."""

    def __init__(self, query_dim, cross_attention_dim, heads):
        super().__init__()
        self.heads = heads
        self.is_cross = cross_attention_dim is not None
        kv_dim = cross_attention_dim if self.is_cross else query_dim
        self.to_q = nn.Linear(query_dim, query_dim, bias=False)
        self.to_k = nn.Linear(kv_dim, query_dim, bias=False)
        self.to_v = nn.Linear(kv_dim, query_dim, bias=False)
        self.to_out = nn.ModuleList([nn.Linear(query_dim, query_dim)])
        self._fused = None

    def fused_weight(self):
        """[3C, C] (self) or [2C, ctx] (cross K,V) concatenation, rebuilt when parameters change."""
        ver = (self.to_k.weight._version, self.to_v.weight._version, self.to_q.weight._version,
               self.to_k.weight.data_ptr(), self.to_k.weight.dtype)
        if self._fused is None or self._fused[0] != ver:
            ws = [self.to_k.weight, self.to_v.weight] if self.is_cross else [self.to_q.weight, self.to_k.weight, self.to_v.weight]
            self._fused = (ver, torch.cat([w.detach() for w in ws], 0).contiguous())
        return self._fused[1]


class BasicTransformerBlock(nn.Module):
    def __init__(self, dim, heads, cross_attention_dim):
        super().__init__()
        self.norm1 = LayerNormCL(dim)
        self.attn1 = Attention(dim, None, heads)
        self.norm2 = LayerNormCL(dim)
        self.attn2 = Attention(dim, cross_attention_dim, heads)
        self.norm3 = LayerNormCL(dim)
        self.ff = nn.Module()
        self.ff.net = nn.ModuleList([nn.Module(), nn.Identity(), nn.Linear(dim * 4, dim)])
        self.ff.net[0].proj = nn.Linear(dim, dim * 8)

    def forward(self, h, n, ctx, ctrl: RegionControl, name):
        """h: residual stream [B, T, C]; n = norm1(h), already evaluated (fused into the previous block's last
        residual add). Returns (h, a, bias): the stream BEFORE the feed-forward residual add, the feed-forward output
        without its bias, and that bias — the caller fuses `h + a + bias` with whatever norm comes next.
        Every `x + sublayer(x)` of attention.py:155-204 is one rtti_add_bias_layernorm_fwd call together with the
        LayerNorm that follows it (the projections run without their bias epilogue)."""
        B, T, C = h.shape
        heads = self.attn1.heads
        # ---- self-attention (attention.py:150-160)
        cap = ctrl.capture
        rem = ctrl.remote
        if rem is not None and rem.is_dst:
            # region passes whose score source (pass D) runs on another rank: Q and K arrive in this layer's receive
            # buffer; the entries' own Q, K would be discarded (attention_processor.py:1160-1163), so only V is projected
            k0 = rem.n_own                                   # leading entries that compute their own scores
            w3 = self.attn1.fused_weight()
            o = torch.empty(B, T, C, dtype=h.dtype, device=h.device)
            if k0:
                qkv = F.linear(n[:k0], w3)
                ops.attention(qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:], heads, out=o[:k0])
            v = F.linear(n[k0:], w3[2 * C:])
            rqk = rem.wait(T, 2 * C)                         # [1, T, 2C] of pass D, stream-ordered behind the wait
            ops.attention(rqk[..., :C], rqk[..., C:], v, heads, qk_src=[0] * (B - k0), out=o[k0:])
        else:
            qkv = F.linear(n, self.attn1.fused_weight())
            q, k, v = qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:]
            if rem is not None and rem.is_src:
                rem.push(qkv[rem.d_index, :, :2 * C])        # side stream: overlaps the rest of this block (joined at its end)
            tgt = cap.self_target(name + ".attn1", T, h.device) if cap is not None else None
            lse = torch.empty(B, heads, T, dtype=torch.float32, device=h.device) if tgt is not None else None
            o = ops.attention(q, k, v, heads, qk_src=ctrl.qk_src, lse=lse)
            if tgt is not None:
                r = ctrl.capture_row
                ops.attn_probs_mean_accum(q[r], k[r], lse[r], tgt[0], heads)
        a = F.linear(o, self.attn1.to_out[0].weight)
        h, n = ops.add_bias_layernorm(a, h, self.attn1.to_out[0].bias, self.norm2.weight, self.norm2.bias, self.norm2.eps)
        # ---- cross-attention (attention.py:163-178)
        q = F.linear(n, self.attn2.to_q.weight)
        kv = None
        key = name + ".attn2"
        if ctrl.kv_cache is not None:
            kv = ctrl.kv_cache.kv.get(key)
        if kv is None:
            kv = F.linear(ctx, self.attn2.fused_weight())
            if ctrl.kv_cache is not None:
                ctrl.kv_cache.kv[key] = kv
        ck, cv = kv[..., :C], kv[..., C:]
        pbar, slots = None, None
        if cap is not None:
            pbar = cap.cross_target(key, T, ctx.shape[1], h.device)
            if pbar is not None:
                slots = [-1] * B
                slots[ctrl.capture_row] = 0
        o = ops.attention(q, ck, cv, heads, word_pos=ctrl.word_pos, font_size=ctrl.font_size,
                          fs_batch_mask=ctrl.fs_batch_mask, pbar_accum=pbar, cap_slot=slots)
        a = F.linear(o, self.attn2.to_out[0].weight)
        h, n = ops.add_bias_layernorm(a, h, self.attn2.to_out[0].bias, self.norm3.weight, self.norm3.bias, self.norm3.eps)
        # ---- feed-forward with GEGLU (attention.py:181-204, 283-304)
        proj = self.ff.net[0].proj
        if ops.FUSED_FF_GEGLU and C % 64 == 0:
            g = ops.ff_geglu(n, proj.weight, proj.bias)     # GEMM + bias + gate in one kernel; no [B, T, 8C] intermediate
        else:
            g = ops.geglu(F.linear(n, proj.weight, proj.bias))
        a = F.linear(g, self.ff.net[2].weight)
        if rem is not None and rem.is_src:
            # the push of this layer's Q|K has had the whole block to drain (at batch 1 it outlasts the attention kernel
            # it was forked next to: 21 MB to four consumers vs ~25 us); `qkv` is still referenced, so its memory was not
            # recycled by the allocator in between
            rem.join()
            del qkv
        return h, a, self.ff.net[2].bias


class Transformer2DModel(nn.Module):
    def __init__(self, channels, heads, layers, cross_attention_dim, groups, use_linear_projection):
        super().__init__()
        self.use_linear_projection = use_linear_projection
        self.norm = GroupNormCL(groups, channels, 1e-6)
        if use_linear_projection:
            self.proj_in = nn.Linear(channels, channels)
            self.proj_out = nn.Linear(channels, channels)
        else:
            self.proj_in = nn.Conv2d(channels, channels, 1)
            self.proj_out = nn.Conv2d(channels, channels, 1)
        self.transformer_blocks = nn.ModuleList([BasicTransformerBlock(channels, heads, cross_attention_dim) for _ in range(layers)])

    def _proj(self, mod, x):
        w = mod.weight if self.use_linear_projection else mod.weight.view(mod.weight.shape[0], -1)
        return F.linear(x, w, mod.bias)

    def forward(self, x, ctx, ctrl, name):
        # channels-last already: the permutes of transformer_2d.py:274-283, 299-307 are no-ops here
        h = self.norm(x, silu=False)
        h = self._proj(self.proj_in, h)
        blocks = self.transformer_blocks
        n = blocks[0].norm1(h)
        for i, blk in enumerate(blocks):
            h, a, bias = blk(h, n, ctx, ctrl, f"{name}.transformer_blocks.{i}")
            if i + 1 < len(blocks):   # feed-forward residual add + the next block's norm1 in one pass
                nxt = blocks[i + 1].norm1
                h, n = ops.add_bias_layernorm(a, h, bias, nxt.weight, nxt.bias, nxt.eps)
            else:
                h = ops.add_bias_f16(h, a, bias, out=a)
        w = self.proj_out.weight if self.use_linear_projection else self.proj_out.weight.view(self.proj_out.weight.shape[0], -1)
        y = F.linear(h, w)
        return ops.add_bias_f16(x, y, self.proj_out.bias, out=y)   # proj_out bias + transformer residual (transformer_2d.py:310)


class ResnetBlock2D(nn.Module):
    def __init__(self, cin, cout, temb_ch, groups, eps):
        super().__init__()
        self.norm1 = GroupNormCL(groups, cin, eps)
        self.conv1 = Conv2dCL(cin, cout, 3, padding=1)
        self.time_emb_proj = nn.Linear(temb_ch, cout)
        self.norm2 = GroupNormCL(groups, cout, eps)
        self.conv2 = Conv2dCL(cout, cout, 3, padding=1)
        self.conv_shortcut = nn.Conv2d(cin, cout, 1) if cin != cout else None

    def forward(self, x, H, W, temb_act, feature_idx=None, remote=None):
        """x [B, HW, Cin]; temb_act = silu(temb). Returns output [B, HW, Cout] (resnet.py:591-645).
        `remote` (multi-GPU): the injected feature of pass D is pushed to / received from another rank."""
        h = self.norm1(x, silu=True)
        h, _, _ = self.conv1.forward_cl(h, H, W, with_bias=False)
        # conv1 bias + `hidden_states + temb` (resnet.py:621-622) both folded into norm2 as a per-(batch, channel) bias
        t = F.linear(temb_act, self.time_emb_proj.weight, self.time_emb_proj.bias + self.conv1.bias)
        h = self.norm2(h, silu=True, chan_bias=t.contiguous())
        h, _, _ = self.conv2.forward_cl(h, H, W, with_bias=False)
        if remote is not None and remote.is_src:
            remote.push(h[remote.d_index])
            remote.join()
        if remote is not None and remote.is_dst:
            f = remote.wait(h.shape[1], h.shape[2])          # conv2 output of pass D, [1, HW, C]
            h = torch.cat([h[:remote.n_own], f.expand(h.shape[0] - remote.n_own, -1, -1)], 0)
        elif feature_idx is not None:
            # inject_states of the reference pass replaces the residual branch (resnet.py:639-641)
            h = h.index_select(0, feature_idx)
        if self.conv_shortcut is not None:
            x = F.linear(x, self.conv_shortcut.weight.view(self.conv_shortcut.weight.shape[0], -1), self.conv_shortcut.bias)
        return ops.add_bias_f16(x, h, self.conv2.bias, out=h)   # residual + conv2 bias in one pass


class Downsample2D(nn.Module):
    def __init__(self, ch):
        super().__init__()
        self.conv = Conv2dCL(ch, ch, 3, stride=2, padding=1)


class Upsample2D(nn.Module):
    def __init__(self, ch):
        super().__init__()
        self.conv = Conv2dCL(ch, ch, 3, padding=1)

    def forward(self, x, H, W):
        B, _, C = x.shape
        # nearest x2 (resnet.py:150-167) in channels-last: broadcast view + one copy
        x = x.view(B, H, 1, W, 1, C).expand(B, H, 2, W, 2, C).reshape(B, 4 * H * W, C)
        return self.conv.forward_cl(x, 2 * H, 2 * W)


class _Block(nn.Module):
    pass


class UNet2DConditionModel(nn.Module):
    def __init__(self, cfg: UNetConfig):
        super().__init__()
        self.config = cfg
        self.in_channels = cfg.in_channels
        boc = cfg.block_out_channels
        temb = boc[0] * 4
        g, eps = cfg.norm_num_groups, cfg.norm_eps
        self.conv_in = Conv2dCL(cfg.in_channels, boc[0], 3, padding=1)
        self.time_embedding = nn.Module()
        self.time_embedding.linear_1 = nn.Linear(boc[0], temb)
        self.time_embedding.linear_2 = nn.Linear(temb, temb)
        if cfg.addition_embed_type == "text_time":
            self.add_embedding = nn.Module()
            self.add_embedding.linear_1 = nn.Linear(cfg.projection_class_embeddings_input_dim, temb)
            self.add_embedding.linear_2 = nn.Linear(temb, temb)
        self.down_blocks = nn.ModuleList()
        out_c = boc[0]
        for i, typ in enumerate(cfg.down_block_types):
            in_c, out_c = out_c, boc[i]
            blk = _Block()
            blk.has_cross_attention = typ == "CrossAttnDownBlock2D"
            if blk.has_cross_attention:
                blk.attentions = nn.ModuleList([
                    Transformer2DModel(out_c, cfg.attention_head_dim[i], cfg.transformer_layers_per_block[i],
                                       cfg.cross_attention_dim, g, cfg.use_linear_projection)
                    for _ in range(cfg.layers_per_block)])
            blk.resnets = nn.ModuleList([ResnetBlock2D(in_c if l == 0 else out_c, out_c, temb, g, eps)
                                         for l in range(cfg.layers_per_block)])
            if i != len(boc) - 1:
                blk.downsamplers = nn.ModuleList([Downsample2D(out_c)])
            else:
                blk.downsamplers = None
            self.down_blocks.append(blk)
        self.mid_block = _Block()
        self.mid_block.attentions = nn.ModuleList([
            Transformer2DModel(boc[-1], cfg.attention_head_dim[-1], cfg.transformer_layers_per_block[-1],
                               cfg.cross_attention_dim, g, cfg.use_linear_projection)])
        self.mid_block.resnets = nn.ModuleList([ResnetBlock2D(boc[-1], boc[-1], temb, g, eps) for _ in range(2)])
        self.up_blocks = nn.ModuleList()
        rev = list(reversed(boc))
        rev_heads = list(reversed(cfg.attention_head_dim))
        rev_layers = list(reversed(cfg.transformer_layers_per_block))
        out_c = rev[0]
        for i, typ in enumerate(cfg.up_block_types):
            prev, out_c = out_c, rev[i]
            in_c = rev[min(i + 1, len(boc) - 1)]
            n = cfg.layers_per_block + 1
            blk = _Block()
            blk.has_cross_attention = typ == "CrossAttnUpBlock2D"
            if blk.has_cross_attention:
                blk.attentions = nn.ModuleList([
                    Transformer2DModel(out_c, rev_heads[i], rev_layers[i], cfg.cross_attention_dim, g, cfg.use_linear_projection)
                    for _ in range(n)])
            blk.resnets = nn.ModuleList([
                ResnetBlock2D((prev if l == 0 else out_c) + (in_c if l == n - 1 else out_c), out_c, temb, g, eps)
                for l in range(n)])
            blk.upsamplers = nn.ModuleList([Upsample2D(out_c)]) if i != len(boc) - 1 else None
            self.up_blocks.append(blk)
        self.conv_norm_out = GroupNormCL(g, boc[0], eps)
        self.conv_out = Conv2dCL(boc[0], cfg.out_channels, 3, padding=1)

    def injection_layout(self, H, W):
        """(tokens, width) of every activation the region passes take from pass D on a feature-injection step, in
        execution order: the Q|K slab [tokens, 2C] of each self-attention layer and the conv2 output [tokens, C] of
        FEATURE_INJECT_RESNET (models/region_diffusion_sdxl.py:1018-1061). Mirrors the traversal of forward()."""
        out = []

        def attn(tr, H, W):
            C = tr.proj_in.weight.shape[0]
            out.extend([(H * W, 2 * C)] * len(tr.transformer_blocks))

        for i, blk in enumerate(self.down_blocks):
            for l in range(len(blk.resnets)):
                if blk.has_cross_attention:
                    attn(blk.attentions[l], H, W)
            if blk.downsamplers is not None:
                H, W = (H + 1) // 2, (W + 1) // 2
        attn(self.mid_block.attentions[0], H, W)
        for i, blk in enumerate(self.up_blocks):
            for l, res in enumerate(blk.resnets):
                if f"up_blocks.{i}.resnets.{l}" == FEATURE_INJECT_RESNET:
                    out.append((H * W, res.conv2.weight.shape[0]))
                if blk.has_cross_attention:
                    attn(blk.attentions[l], H, W)
            if blk.upsamplers is not None:
                H, W = 2 * H, 2 * W
        return out

    # ------------------------------------------------------------------ weights
    def finalize(self, device="cuda"):
        """fp16, on device, 3x3 conv weights in channels_last so cuDNN picks NHWC tensor-core kernels."""
        self.to(device=device, dtype=torch.float16)
        for m in self.modules():
            if isinstance(m, nn.Conv2d) and m.kernel_size != (1, 1):
                m.weight.data = m.weight.data.contiguous(memory_format=torch.channels_last)
        self.requires_grad_(False)
        return self.eval()

    def init_synthetic(self, seed=0):
        """Random weights of the right shapes (no checkpoints in this environment): N(0, 1/fan_in) matrices,
        unit norm gains, small biases — keeps activations O(1) through the depth."""
        g = torch.Generator(device=self.conv_in.weight.device).manual_seed(seed)
        for name, p in self.named_parameters():
            if p.dim() >= 2:
                fan_in = p[0].numel()
                p.data.copy_(torch.randn(p.shape, generator=g, device=p.device, dtype=torch.float32) / math.sqrt(fan_in))
            elif name.endswith("weight"):
                p.data.fill_(1.0)
            else:
                p.data.copy_(0.05 * torch.randn(p.shape, generator=g, device=p.device, dtype=torch.float32))
        return self

    # ------------------------------------------------------------------ forward
    def _timestep_embedding(self, t, dim, device):
        half = dim // 2
        exponent = -math.log(10000) * torch.arange(half, dtype=torch.float32, device=device) / (half - self.config.freq_shift)
        emb = t[:, None].float() * torch.exp(exponent)[None, :]
        emb = torch.cat([torch.sin(emb), torch.cos(emb)], dim=-1)
        if self.config.flip_sin_to_cos:
            emb = torch.cat([emb[:, half:], emb[:, :half]], dim=-1)
        return emb

    def forward(self, sample, timestep, encoder_hidden_states, added_cond_kwargs=None, ctrl: Optional[RegionControl] = None,
                return_dict=True, **unused):
        """sample [B, 4, h, w] (NCHW, as the reference); timestep scalar or [B]; encoder_hidden_states [B, 77, D].
        Returns {'sample': [B, 4, h, w]} like models/unet_2d_condition.py:980-983."""
        cfg = self.config
        ctrl = ctrl or RegionControl()
        dev = sample.device
        B, _, H, W = sample.shape
        t = torch.as_tensor(timestep, device=dev)
        if t.dim() == 0:
            t = t[None]
        t = t.expand(B)
        mlp = lambda m, x: F.linear(F.silu(F.linear(x, m.linear_1.weight, m.linear_1.bias)), m.linear_2.weight, m.linear_2.bias)
        emb = mlp(self.time_embedding, _f16(self._timestep_embedding(t, cfg.block_out_channels[0], dev)))
        if cfg.addition_embed_type == "text_time":
            time_ids = added_cond_kwargs["time_ids"].to(dev)
            te = self._timestep_embedding(time_ids.flatten(), cfg.addition_time_embed_dim, dev)
            te = te.reshape(time_ids.shape[0], -1)
            if te.shape[0] != B:
                te = te[:1].expand(B, -1)  # the reference passes add_time_ids[:1] to every pass (sdxl.py:787-821)
            add = torch.cat([_f16(added_cond_kwargs["text_embeds"]), _f16(te)], dim=-1)
            emb = emb + mlp(self.add_embedding, add)
        temb_act = F.silu(emb)
        ctx = _f16(encoder_hidden_states).contiguous()
        feat_idx = ctrl.feature_idx
        if feat_idx is None and ctrl.feature_src is not None:
            feat_idx = torch.as_tensor(ctrl.feature_src, device=dev)

        x = _f16(sample).permute(0, 2, 3, 1).contiguous().view(B, H * W, -1)
        h, H, W = self.conv_in.forward_cl(x, H, W)
        skips = [(h, H, W)]
        for i, blk in enumerate(self.down_blocks):
            for l, res in enumerate(blk.resnets):
                h = res(h, H, W, temb_act)
                if blk.has_cross_attention:
                    h = blk.attentions[l](h, ctx, ctrl, f"down_blocks.{i}.attentions.{l}")
                skips.append((h, H, W))
            if blk.downsamplers is not None:
                h, H, W = blk.downsamplers[0].conv.forward_cl(h, H, W)
                skips.append((h, H, W))
        h = self.mid_block.resnets[0](h, H, W, temb_act)
        h = self.mid_block.attentions[0](h, ctx, ctrl, "mid_block.attentions.0")
        h = self.mid_block.resnets[1](h, H, W, temb_act)
        for i, blk in enumerate(self.up_blocks):
            for l, res in enumerate(blk.resnets):
                s, _, _ = skips.pop()
                h = torch.cat([h, s], dim=-1)
                rname = f"up_blocks.{i}.resnets.{l}"
                inj = rname == FEATURE_INJECT_RESNET
                h = res(h, H, W, temb_act, feat_idx if inj else None, ctrl.remote if inj else None)
                if blk.has_cross_attention:
                    h = blk.attentions[l](h, ctx, ctrl, f"up_blocks.{i}.attentions.{l}")
            if blk.upsamplers is not None:
                h, H, W = blk.upsamplers[0](h, H, W)
        h = self.conv_norm_out(h, silu=True)
        h, H, W = self.conv_out.forward_cl(h, H, W)
        out = h.view(B, H, W, -1).permute(0, 3, 1, 2).contiguous()
        return {"sample": out} if return_dict else (out,)
