"""Explicit forward + input-gradient backward of the VAE decoder for colour guidance.

The reference back-propagates `loss -> imgs -> vae.decode -> latents` with autograd through the third-party
fp32 AutoencoderKL (models/region_diffusion_sdxl.py:849-867, models/region_diffusion.py:151-168), including the
weight gradients it never uses. Here the decoder (vae.py, diffusers parameter names) is evaluated as an explicit
static sequence — no autograd graph, no autograd thread, CUDA-graph capturable:

  * channels-last fp32 activations [B, H*W, C] end to end;
  * GroupNorm(+SiLU) forward and backward in the sm_90a kernels of csrc/vae_kernels.cu
    (PyTorch's native GroupNorm round-trips channels-last tensors through NCHW copies);
  * 3x3 / 1x1 convolutions: cuDNN forward and `convolution_backward` with output_mask=(True, False, False)
    (data gradient only, TF32 tensor cores as in the reference's default PyTorch settings);
  * nearest x2 upsample + 3x3 convolution evaluated at low resolution: each output phase is a 2x2 convolution with a
    folded filter, so the layer is one 2x2 convolution of the low-res input with the four folded filters stacked
    (16 instead of 36 multiply-adds per output element, no 4x upsampled copy); its output is interleaved into the
    high-res tensor (and the gradient scattered back) by csrc/vae_kernels.cu;
  * the single-head 16384-token mid-block attention materialises its 1 GB probability matrix once
    and reuses it for the five backward GEMMs instead of recomputing it.

DecoderFwdBwd.forward / .backward are the one walk over the decoder's blocks. They hand the engine's activation from
layer to layer: here a [B, H*W, C] tensor; in the stripe-parallel engine, which overrides the per-layer methods
(stripe_parallel.py says which), this rank's stripe of rows.
"""
import contextlib
import math

import torch
import torch.nn.functional as F

from . import ops

_conv_bwd = torch.ops.aten.convolution_backward

# _PHASE_TAPS[a][t][k]: weight of 3x3 kernel row k in tap t of output phase a (rows 2i+a of the x2 nearest upsample
# read low-res rows i-1, i, i (a = 0) or i, i, i+1 (a = 1)); tap t of the 2x2, pad-1 phase convolution at low-res
# output position p reads row p-1+t, and phase a of row i sits at p = i+a. Columns likewise.
_PHASE_TAPS = (((1., 0., 0.), (0., 1., 1.)), ((1., 1., 0.), (0., 0., 1.)))


@contextlib.contextmanager
def _tf32_matmul():
    """fp32 matmuls (projections, attention) on TF32 tensor cores; the caller's setting is restored on exit."""
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = True
    try:
        yield
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev


def _nchw(x, H, W):
    """[B, HW, C] contiguous -> logical NCHW view with channels_last strides (no copy)."""
    return x.view(x.shape[0], H, W, x.shape[2]).permute(0, 3, 1, 2)


def _cl(y):
    """NCHW (channels_last memory) -> [B, HW, C] contiguous view."""
    B, C, H, W = y.shape
    y = y.permute(0, 2, 3, 1)
    if not y.is_contiguous():
        y = y.contiguous()
    return y.view(B, H * W, C), H, W


def _conv_f(conv, x, H, W, with_bias=True):
    """with_bias=False: the caller folds conv.bias into the consumer (GroupNorm kernel / fused residual add) —
    PyTorch otherwise adds the bias of a channels-last fp32 convolution in a separate broadcast pass."""
    y = F.conv2d(_nchw(x, H, W), conv.weight, conv.bias if with_bias else None, conv.stride, conv.padding)
    return _cl(y)[0]


class DecoderFwdBwd:
    """decode(z) -> image, then backward(d image) -> d z, for vae.AutoencoderKLDecoder parameters."""

    def __init__(self, vae):
        self.vae = vae
        self.groups = vae.config.norm_num_groups
        self._dummies = {}
        self._wphase = {}

    # ------------------------------------------------------------------ pieces
    def _gn_f(self, norm, x, silu, tape, chan_bias=None):
        y, stats = ops.gn32_silu_fwd(x, norm.weight, norm.bias, self.groups, norm.eps, silu, chan_bias=chan_bias)
        tape.append(("gn", norm, x, stats, silu, chan_bias))
        return y

    def _gn_b(self, rec, g, addend=None):
        _, norm, x, stats, silu, chan_bias = rec
        return ops.gn32_silu_bwd(x, g.contiguous(), norm.weight, norm.bias, stats, self.groups, silu, chan_bias=chan_bias,
                                 addend=addend)

    def _dummy(self, shape, dev):
        k = (tuple(shape), str(dev))
        if k not in self._dummies:
            self._dummies[k] = torch.empty(shape, dtype=torch.float32, device=dev, memory_format=torch.channels_last)
        return self._dummies[k]

    def _conv_b(self, conv, g, cin, H, W):
        g4 = _nchw(g, H, W)
        gi, _, _ = _conv_bwd(g4, self._dummy((g.shape[0], cin, H, W), g.device), conv.weight, None, list(conv.stride),
                             list(conv.padding), [1, 1], False, [0, 0], 1, [True, False, False])
        return _cl(gi)[0]

    def _phase_filter(self, conv):
        """[4*Cout, Cin, 2, 2] channels-last: the 3x3 filter of an upsampler folded into its four output phases,
        phase 2a+b in output channels (2a+b)*Cout.. (computed once per VAE in fp64: the weights are frozen).
        The fold is cached per module and never refreshed: changing conv.weight in place after the first call (e.g.
        load_state_dict) is not seen; build a new engine (vae._fwd_bwd = None) after loading other weights."""
        hit = self._wphase.get(id(conv))
        if hit is None or hit[0] is not conv:   # the module is kept with its filter: an id can be reused
            w = conv.weight.double()
            taps = torch.tensor(_PHASE_TAPS, dtype=w.dtype, device=w.device)
            wf = torch.einsum("atk,bul,oikl->aboitu", taps, taps, w).reshape(4 * w.shape[0], w.shape[1], 2, 2)
            hit = self._wphase[id(conv)] = (conv, wf.float().contiguous(memory_format=torch.channels_last))
        return hit[1]

    def _upsample_f(self, conv, x, H, W):
        """conv3x3(nearest_x2(x)) for x [B, H*W, C] -> [B, 4*H*W, Cout]."""
        y4 = F.conv2d(_nchw(x, H, W), self._phase_filter(conv), None, 1, 1)
        return ops.upsample_phase_interleave(_cl(y4)[0], conv.bias, H, W)

    def _upsample_b(self, conv, g, H, W, C):
        """Input gradient of _upsample_f: g [B, 4*H*W, Cout] -> [B, H*W, C]."""
        dy4 = ops.upsample_phase_scatter(g.contiguous(), H, W)
        gi, _, _ = _conv_bwd(_nchw(dy4, H + 1, W + 1), self._dummy((g.shape[0], C, H, W), g.device), self._phase_filter(conv),
                             None, [1, 1], [1, 1], [1, 1], False, [0, 0], 1, [True, False, False])
        return _cl(gi)[0]

    def _resnet_f(self, r, x, H, W, tape):
        h = self._gn_f(r.norm1, x, True, tape)
        h = _conv_f(r.conv1, h, H, W, with_bias=False)
        h = self._gn_f(r.norm2, h, True, tape, chan_bias=r.conv1.bias)   # conv1 bias folded into the norm
        h = _conv_f(r.conv2, h, H, W, with_bias=False)
        sc = _conv_f(r.conv_shortcut, x, H, W) if r.conv_shortcut is not None else x
        tape.append(("res", r, H, W))
        return ops.add_bias_f32(sc, h, r.conv2.bias)                      # residual + conv2 bias in one pass

    def _resnet_b(self, tape, g):
        _, r, H, W = tape.pop()
        cin, cout = r.conv1.in_channels, r.conv1.out_channels
        dh = self._conv_b(r.conv2, g, cout, H, W)
        dh = self._gn_b(tape.pop(), dh)
        dh = self._conv_b(r.conv1, dh, cin, H, W)
        sc = self._conv_b(r.conv_shortcut, g, cin, H, W) if r.conv_shortcut is not None else g.contiguous()
        return self._gn_b(tape.pop(), dh, addend=sc)                       # + the shortcut path's gradient

    def _attn_kv(self, hn):
        """Normalised tokens the keys and values are projected from."""
        return hn

    def _attn_dhn(self, a, dq, dk, dv):
        """Gradient of the attention's normalised input from those of q, k, v."""
        return dq @ a.to_q.weight + dk @ a.to_k.weight + dv @ a.to_v.weight

    def _attn_f(self, a, x, tape):
        """Single-head self-attention over all tokens (vae._MidAttention), probabilities materialised."""
        C = x.shape[2]
        hn = self._gn_f(a.group_norm, x, False, tape)
        kv = self._attn_kv(hn)
        q = F.linear(hn, a.to_q.weight, a.to_q.bias)
        k = F.linear(kv, a.to_k.weight, a.to_k.bias)
        v = F.linear(kv, a.to_v.weight, a.to_v.bias)
        scale = 1.0 / math.sqrt(C)
        # the softmax scale is applied to q ([T, C], 33 MB) instead of the [T, T] scores (1 GB at 1024^2: a 2 GB pass)
        p = torch.softmax(torch.bmm(q * scale, k.transpose(1, 2)), dim=-1)
        o = torch.bmm(p, v)
        tape.append(("attn", a, q, k, v, p, scale))
        return x + F.linear(o, a.to_out[0].weight, a.to_out[0].bias)

    def _attn_b(self, tape, g):
        _, a, q, k, v, p, scale = tape.pop()
        do = g @ a.to_out[0].weight                       # [B,T,C]
        dv = torch.bmm(p.transpose(1, 2), do)
        dp = torch.bmm(do, v.transpose(1, 2))
        ds = torch._softmax_backward_data(dp, p, -1, p.dtype)   # d/d(scaled scores); the scale goes onto the small operands
        dq = torch.bmm(ds, k * scale)
        dk = torch.bmm(ds.transpose(1, 2), q * scale)
        return g + self._gn_b(tape.pop(), self._attn_dhn(a, dq, dk, dv))

    def _entry(self, z):
        """z [B, 4, H, W] -> (activation after conv_in, H, W)."""
        vae, d = self.vae, self.vae.decoder
        B, _, H, W = z.shape
        x = z.permute(0, 2, 3, 1).contiguous().view(B, H * W, -1)
        x = _conv_f(vae.post_quant_conv, x, H, W)
        return _conv_f(d.conv_in, x, H, W), H, W

    def _out_f(self, x, H, W, tape):
        """conv_norm_out + SiLU + conv_out -> image [B, 3, H, W] (NCHW view of channels-last memory)."""
        d = self.vae.decoder
        x = self._gn_f(d.conv_norm_out, x, True, tape)
        return _nchw(_conv_f(d.conv_out, x, H, W), H, W)

    def _out_b(self, grad_image, H, W, tape):
        d = self.vae.decoder
        g = grad_image.permute(0, 2, 3, 1).contiguous().view(grad_image.shape[0], H * W, -1)
        g = self._conv_b(d.conv_out, g, d.conv_out.in_channels, H, W)
        return self._gn_b(tape.pop(), g)

    def _exit(self, g, H, W):
        """Gradient after conv_in's output -> d z [B, 4, H, W]."""
        vae, d = self.vae, self.vae.decoder
        g = self._conv_b(d.conv_in, g, d.conv_in.in_channels, H, W)
        g = self._conv_b(vae.post_quant_conv, g, vae.post_quant_conv.in_channels, H, W)
        return g.view(g.shape[0], H, W, -1).permute(0, 3, 1, 2).contiguous()

    # ------------------------------------------------------------------ whole decoder
    def forward(self, z):
        """z [B, 4, h, w] fp32 -> image [B, 3, 8h, 8w] fp32 (NCHW view of channels-last memory); keeps the tape."""
        d = self.vae.decoder
        with _tf32_matmul():
            tape = []
            x, H, W = self._entry(z)
            x = self._resnet_f(d.mid_block.resnets[0], x, H, W, tape)
            x = self._attn_f(d.mid_block.attentions[0], x, tape)
            x = self._resnet_f(d.mid_block.resnets[1], x, H, W, tape)
            for blk in d.up_blocks:
                for r in blk.resnets:
                    x = self._resnet_f(r, x, H, W, tape)
                if blk.upsamplers is not None:
                    conv, C = blk.upsamplers[0].conv, x.shape[2]
                    x = self._upsample_f(conv, x, H, W)
                    tape.append(("up", conv, H, W, C))
                    H, W = 2 * H, 2 * W
            img = self._out_f(x, H, W, tape)
            tape.append(("out", H, W))
            self.tape = tape
            return img

    def backward(self, grad_image):
        """grad_image [B, 3, H, W] -> d loss / d z [B, 4, h, w] fp32."""
        d = self.vae.decoder
        with _tf32_matmul():
            tape = self.tape
            _, H, W = tape.pop()
            g = self._out_b(grad_image, H, W, tape)
            for blk in reversed(d.up_blocks):
                if blk.upsamplers is not None:
                    _, conv, H, W, C = tape.pop()
                    g = self._upsample_b(conv, g, H, W, C)
                for _ in blk.resnets:
                    g = self._resnet_b(tape, g)
            g = self._resnet_b(tape, g)
            g = self._attn_b(tape, g)
            g = self._resnet_b(tape, g)
            self.tape = None
            return self._exit(g, H, W)


def default_engine(vae):
    """The single-GPU explicit forward/backward engine of `vae` (created once, kept on the module)."""
    eng = getattr(vae, "_fwd_bwd", None)
    if eng is None:
        eng = vae._fwd_bwd = DecoderFwdBwd(vae)
    return eng


def image_and_latent_grad(vae, z, grad_fn, engine=None):
    """image = decode(z); grad_image = grad_fn(image.detach()); returns d/dz of <grad_image, decode(z)>.
    Uses the explicit forward/backward for vae.AutoencoderKLDecoder and autograd for any other decoder object
    exposing decode_tensor() (e.g. the tiny stand-in of the parity fixtures). `engine`: a
    stripe_parallel.StripedDecoderFwdBwd to run the decoder split by rows over the ranks."""
    from .vae import AutoencoderKLDecoder
    if isinstance(vae, AutoencoderKLDecoder):
        eng = engine if engine is not None else default_engine(vae)
        img = eng.forward(z)
        return eng.backward(grad_fn(img))
    z = z.detach().requires_grad_(True)
    with torch.enable_grad():
        img = vae.decode_tensor(z)
    img.backward(grad_fn(img.detach()))
    return z.grad


class GuidanceGraph:
    """decode -> colour loss forward/backward -> decoder backward as ONE replayed CUDA graph.

    The evaluation is a static sequence of ~600 launches (the stripe-parallel engine adds one halo kernel per convolution
    and three NCCL collectives); on 4-8 GPUs each rank's share of the GPU work shrinks to 7-15 ms while the CPU issue time
    stays ~15 ms, i.e. the phase is launch-bound unless it is replayed. Protocol per (engine, shapes): the first call runs
    eagerly (cuDNN autotune, arena views, flipped filters), the second captures and replays, later calls replay. Inputs
    are copied into static buffers; the returned gradient and loss are static tensors overwritten by the next call.
    Every rank of a stripe group must make the same sequence of calls (they do: the guidance is replicated control flow).
    """

    def __init__(self, engine):
        self.engine = engine
        self.calls = 0
        self.graph = None
        self.launches = 0

    def _run(self, z, masks, tgt):
        img = self.engine.forward(z)
        loss, g = ops.color_loss_fwd_bwd(img[0].contiguous(), masks, tgt)
        return loss, self.engine.backward(g[None])

    def __call__(self, z, masks, tgt):
        self.calls += 1
        if self.calls == 1:
            return self._run(z, masks, tgt)
        if self.graph is None:
            self.z, self.masks, self.tgt = z.clone(), masks.clone(), tgt.clone()
            torch.cuda.synchronize(z.device)
            graph = torch.cuda.CUDAGraph()
            n0 = ops.LAUNCHES
            with torch.cuda.graph(graph, capture_error_mode="thread_local"):
                self.loss, self.grad = self._run(self.z, self.masks, self.tgt)
            self.launches = ops.LAUNCHES - n0
            self.graph = graph
        else:
            self.z.copy_(z); self.masks.copy_(masks); self.tgt.copy_(tgt)
        self.graph.replay()
        ops._count(self.launches)
        return self.loss, self.grad
