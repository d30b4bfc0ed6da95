"""Stripe-parallel colour guidance: the VAE decoder forward + input-gradient backward split by image rows over the
ranks (multi-GPU, SURVEY §8e; kernels in csrc/stripe_exchange.cu and csrc/vae_kernels.cu).

The reference back-propagates the colour loss through the batch-1 fp32 VAE decoder on one device
(models/region_diffusion_sdxl.py:849-867). With region-parallel UNet passes that replicated 51 ms is what limits
scaling (Amdahl), so here:

  * post_quant_conv and conv_in (0.6 GFLOP) stay replicated;
  * from the mid block on, every rank owns `rows` consecutive image rows of every activation. The 16 384-token
    mid-block attention runs this rank's query rows against all keys/values (normalised input all-gathered, the
    K/V-side gradient reduce-scattered after its projection: one 32 MB collective each way). 3x3 convolutions
    read padded buffers [1 + rows + 1, W, C] living in a symmetric (peer-mapped) arena whose halo rows the
    neighbours fill with ONE kernel per convolution (rtti_halo_exchange); GroupNorm statistics are reduced inside
    the GroupNorm call through peer memory (rtti_gn32_silu_*_striped); nearest-neighbour upsampling, SiLU, residual
    adds and 1x1 shortcuts are stripe-local;
  * the data gradient of a 3x3 convolution is evaluated as a forward convolution of the (haloed) output gradient
    with the flipped, transposed filter — the same halo machinery serves both directions;
  * two more NCCL all-gathers per call (the decoded image stripes: 12.6 MB, and the gradient entering conv_in:
    32 MB) and one 256 KB broadcast of the final latent gradient from rank 0, which keeps the replicated latents
    bit-identical on all ranks whatever algorithms cuDNN picked per rank.

PyTorch is used for the rendezvous (symmetric memory), cuDNN convolutions and the NCCL calls.

StripedDecoderFwdBwd runs the decoder walk of vae_guidance.DecoderFwdBwd.forward / .backward with this rank's stripe
as the activation (a _Pad in backward). It overrides _entry, _resnet_f/_b, _upsample_f/_b, _out_f/_b, _exit and
_gn_f/_b; of the attention, only where K/V come from (_attn_kv), how the input gradient is assembled (_attn_dhn), and
_attn_b to move the gradient in and out of its pad.
"""
import ctypes

import torch
import torch.nn.functional as F

from . import ops
from .vae_guidance import DecoderFwdBwd, _cl, _conv_f, _nchw


class _Pad:
    """A padded conv input [rows+2, W, C] in the arena whose interior is written but whose halo exchange is pending."""
    __slots__ = ("pad", "seq")

    def __init__(self, pad, seq):
        self.pad, self.seq = pad, seq


class StripeArena:
    """Symmetric arena: [4 KB control block][pad half 0][pad half 1], identical layout on every rank.

    Control block: +0 GroupNorm {sequence, error, ..., [8] sequence base} words; +64 halo flags {from_up, from_down,
    error, counter, ..., [8] sequence base}; +256 GroupNorm statistics slots fp32 [2 parities][3 * 32 groups]. Pads alternate
    between the two halves by exchange sequence parity (see csrc/stripe_exchange.cu for why two are enough).

    Sequence numbers are RELATIVE to one decoder evaluation (forward + backward): the host counts 1..n, the kernels add
    the device-side base words, and end_call() advances the bases by n with a stream-ordered kernel. Every evaluation
    therefore issues identical kernel arguments and can be replayed from one CUDA graph. Restarting the pad-half
    alternation at each evaluation is safe because an evaluation ends with collectives over all ranks (all-gather of the
    conv_in gradient, broadcast of the latent gradient) that order every rank's last pad consumer before any rank's
    next push."""
    HEADER = 4096

    def __init__(self, pad_bytes, device, group=None):
        import torch.distributed as dist
        import torch.distributed._symmetric_memory as symm
        self.dist = dist
        self.group = group or dist.group.WORLD
        self.world, self.rank = dist.get_world_size(self.group), dist.get_rank(self.group)
        self.pad_bytes = (int(pad_bytes) + 255) // 256 * 256
        self.buf = symm.empty(self.HEADER + 2 * self.pad_bytes, dtype=torch.uint8, device=device)
        self.handle = symm.rendezvous(self.buf, self.group.group_name)
        self.buf[:self.HEADER].zero_()
        torch.cuda.synchronize(device)
        dist.barrier(self.group)
        base = [int(p) for p in self.handle.buffer_ptrs]
        self.base = base
        self.gn_flag_ptrs = (ctypes.c_void_p * self.world)(*base)
        self.sum_ptrs = (ctypes.c_void_p * self.world)(*[b + 256 for b in base])
        self.halo_flags = [b + 64 for b in base]
        self.halves = [self.buf[self.HEADER:self.HEADER + self.pad_bytes],
                       self.buf[self.HEADER + self.pad_bytes:self.HEADER + 2 * self.pad_bytes]]
        self.gn_seq = 0
        self.halo_seq = 0
        self._views = {}

    def next_gn_seq(self):
        self.gn_seq += 1
        return self.gn_seq

    def pad(self, rows, W, C):
        """Reserve the pad of the next exchange: returns (pad [rows+2, W, C] fp32 view, seq)."""
        self.halo_seq += 1
        key = (self.halo_seq & 1, rows, W, C)
        v = self._views.get(key)
        if v is None:
            n = (rows + 2) * W * C * 4
            if n > self.pad_bytes:
                raise RuntimeError(f"stripe pad of {n} bytes exceeds the arena half ({self.pad_bytes})")
            v = self._views[key] = self.halves[key[0]][:n].view(torch.float32).view(rows + 2, W, C)
        return v, self.halo_seq

    def release(self, seq):
        """Give back the most recent pad() without exchanging it (its interior was only used as plain memory), so
        that exchanged pads keep alternating between the two halves."""
        assert seq == self.halo_seq
        self.halo_seq -= 1

    def exchange(self, pad, seq):
        assert seq == self.halo_seq, "pad()/exchange() must pair up in order"
        off = self.HEADER + (seq & 1) * self.pad_bytes
        up = self.rank - 1 if self.rank > 0 else None
        down = self.rank + 1 if self.rank + 1 < self.world else None
        ops.halo_exchange(pad,
                          self.base[up] + off if up is not None else 0,
                          self.base[down] + off if down is not None else 0,
                          self.halo_flags[self.rank],
                          self.halo_flags[up] if up is not None else 0,
                          self.halo_flags[down] if down is not None else 0, seq)

    def end_call(self):
        """End of one decoder evaluation: advance the device-side sequence bases by the exchanges issued and restart
        the relative numbering."""
        if self.halo_seq or self.gn_seq:
            ops.peer_seq_advance(self.halo_flags[self.rank], self.halo_seq, self.base[self.rank], self.gn_seq)
        self.halo_seq = 0
        self.gn_seq = 0

    def check(self):
        """Raise if a peer wait timed out (error words set by the kernels)."""
        words = self.buf[:80].view(torch.int32).cpu()
        if int(words[1]) != 0 or int(words[16 + 2]) != 0:
            raise RuntimeError("stripe-parallel colour guidance: timed out waiting for a peer rank")


def stripe_pad_elems(decoder, rows, W):
    """Largest padded conv input (elements) of the striped up-path for a latent stripe of `rows` x W."""
    best = 0
    for blk in decoder.up_blocks:
        for r in blk.resnets:
            best = max(best, (rows + 2) * W * max(r.conv1.in_channels, r.conv1.out_channels))
        if blk.upsamplers is not None:
            rows, W = 2 * rows, 2 * W
            best = max(best, (rows + 2) * W * blk.upsamplers[0].conv.in_channels)
    return max(best, (rows + 2) * W * decoder.conv_out.in_channels)


class StripedDecoderFwdBwd(DecoderFwdBwd):
    """decode(z) -> full image on every rank; backward(d image) -> d z on every rank (bit-identical)."""

    def __init__(self, vae, latent_h, latent_w, device, group=None, arena=None, dist=None):
        """`arena` / `dist`: injection points for the CPU emulation of the exchange (tests/test_stripe_emulation.py);
        the product path builds a StripeArena over torch.distributed's symmetric memory."""
        super().__init__(vae)
        if dist is None:
            import torch.distributed as dist
        self.dist = dist
        self.group = group or (arena.group if arena is not None else dist.group.WORLD)
        self.world, self.rank = dist.get_world_size(self.group), dist.get_rank(self.group)
        if latent_h % self.world != 0:
            raise ValueError(f"latent height {latent_h} is not divisible by {self.world} ranks")
        if self.groups > 32:
            raise ValueError("stripe-parallel GroupNorm supports at most 32 groups")
        self.latent_hw = (latent_h, latent_w)
        self.rows0 = latent_h // self.world
        self.arena = arena if arena is not None else StripeArena(stripe_pad_elems(vae.decoder, self.rows0, latent_w) * 4,
                                                                 device, self.group)
        self._wflip = {}

    # ------------------------------------------------------------------ striped pieces
    # x [1, rows*W, C] is this rank's stripe: the whole tensor has rows*W*world tokens.
    def _gn_f(self, norm, x, silu, tape, chan_bias=None, out=None):
        y, stats = ops.gn32_silu_fwd_striped(x, norm.weight, norm.bias, self.groups, norm.eps, silu, x.shape[1] * self.world,
                                             self.arena, self.arena.next_gn_seq(), chan_bias=chan_bias, out=out)
        tape.append(("gn", norm, x, stats, silu, chan_bias))
        return y

    def _gn_b(self, rec, g, out=None):
        _, norm, x, stats, silu, chan_bias = rec
        return ops.gn32_silu_bwd_striped(x, g.contiguous(), norm.weight, norm.bias, stats, self.groups, silu,
                                         x.shape[1] * self.world, self.arena, self.arena.next_gn_seq(), chan_bias=chan_bias,
                                         out=out)

    @staticmethod
    def _conv_pad(weight, bias, pad):
        """3x3 convolution of a haloed stripe: pad [rows+2, W, C] -> [1, rows*W, Cout] (zero padding along W only)."""
        R2, W, C = pad.shape
        y = F.conv2d(pad.view(1, R2, W, C).permute(0, 3, 1, 2), weight, bias, 1, (0, 1))
        return _cl(y)[0]

    def _flipped(self, conv):
        """Filter of the data-gradient-as-forward-convolution: wf[c, o, a, b] = w[o, c, 2-a, 2-b]."""
        k = id(conv)
        if k not in self._wflip:
            self._wflip[k] = conv.weight.flip(2, 3).transpose(0, 1).contiguous(memory_format=torch.channels_last)
        return self._wflip[k]

    def _new_pad(self, rows, W, C):
        """Pad of the NEXT exchange, to be filled by a producer kernel: (_Pad, interior view [1, rows*W, C])."""
        pad, seq = self.arena.pad(rows, W, C)
        return _Pad(pad, seq), pad[1:-1].view(1, rows * W, C)

    def _s_conv3_b(self, conv, g, rows, W):
        """d/d input of a striped 3x3 convolution. g: a _Pad whose interior already holds the output gradient
        (written there by its producer), or a plain [1, rows*W, Cout] tensor that is copied into a fresh pad."""
        if not isinstance(g, _Pad):
            gp, interior = self._new_pad(rows, W, g.shape[2])
            interior.copy_(g.view_as(interior))
            g = gp
        self.arena.exchange(g.pad, g.seq)
        return self._conv_pad(self._flipped(conv), None, g.pad)

    def _entry(self, z):
        """conv_in (0.6 GFLOP) and post_quant_conv are replicated; from their output on, this rank's stripe."""
        if z.shape[0] != 1 or tuple(z.shape[2:]) != self.latent_hw:
            raise ValueError(f"stripe-parallel decoder was built for a [1, C, {self.latent_hw}] latent, got {tuple(z.shape)}")
        x, _, W = super()._entry(z)
        rows = self.rows0
        return x[:, self.rank * rows * W:(self.rank + 1) * rows * W].contiguous(), rows, W

    def _resnet_f(self, r, x, rows, W, tape):
        cin, cout = r.conv1.in_channels, r.conv1.out_channels
        pad, seq = self.arena.pad(rows, W, cin)
        self._gn_f(r.norm1, x, True, tape, out=pad[1:-1].view(1, rows * W, cin))
        self.arena.exchange(pad, seq)
        h = self._conv_pad(r.conv1.weight, None, pad)
        pad, seq = self.arena.pad(rows, W, cout)
        self._gn_f(r.norm2, h, True, tape, chan_bias=r.conv1.bias, out=pad[1:-1].view(1, rows * W, cout))
        self.arena.exchange(pad, seq)
        h = self._conv_pad(r.conv2.weight, None, pad)
        sc = _conv_f(r.conv_shortcut, x, rows, W) if r.conv_shortcut is not None else x
        tape.append(("res", r, rows, W))
        return ops.add_bias_f32(sc, h, r.conv2.bias)

    def _resnet_b(self, tape, g):
        """g: _Pad (un-exchanged, interior = gradient of the block output). Returns a _Pad holding the gradient of
        the block input, again un-exchanged, so the consumer (the next resnet / upsampler gradient) needs no staging
        copy. Hazard rule for pads (two halves, alternating): anything that reads pad s other than its convolution
        must run before this rank pushes exchange s+1 — unless it reads only the interior and pad s+2 has the same
        shape (neighbours only ever write halo rows). Hence the 1x1 shortcut gradient is taken first, and the
        identity-shortcut add runs in place."""
        _, r, rows, W = tape.pop()
        cin, cout = r.conv1.in_channels, r.conv1.out_channels
        g_int = g.pad[1:-1].view(1, rows * W, cout)
        sc = self._conv_b(r.conv_shortcut, g_int, cin, rows, W) if r.conv_shortcut is not None else None
        dh = self._s_conv3_b(r.conv2, g, rows, W)
        p2, p2_int = self._new_pad(rows, W, cout)
        self._gn_b(tape.pop(), dh, out=p2_int)                      # straight into the next conv's pad
        dh = self._s_conv3_b(r.conv1, p2, rows, W)
        dx = self._gn_b(tape.pop(), dh)
        out, out_int = self._new_pad(rows, W, cin)                  # same half as g (two exchanges later)
        ops.add_bias_f32(dx, sc if sc is not None else g_int, out=out_int)   # identity case: in place over g
        return out

    def _attn_kv(self, hn):
        """Queries are this rank's stripe, keys/values come from all tokens: all-gather the normalised input (32 MB)."""
        hn_full = torch.empty(1, hn.shape[1] * self.world, hn.shape[2], dtype=torch.float32, device=hn.device)
        self.dist.all_gather_into_tensor(hn_full.view(-1), hn.reshape(-1), group=self.group)
        return hn_full

    def _attn_dhn(self, a, dq, dk, dv):
        """dk, dv are partial sums over the query stripes: project first (one reduction instead of two), then
        reduce-scatter over the ranks, keeping this rank's rows."""
        dkv = (dk @ a.to_k.weight + dv @ a.to_v.weight).contiguous()
        mine = torch.empty(1, dq.shape[1], dkv.shape[2], dtype=torch.float32, device=dq.device)
        self.dist.reduce_scatter_tensor(mine.view(-1), dkv.view(-1), group=self.group)
        return dq @ a.to_q.weight + mine

    def _attn_b(self, tape, g):
        """g: _Pad, returned with its interior overwritten by the attention's input gradient (the attention reads the
        interior only, and its result is a new tensor)."""
        g_int = g.pad[1:-1].view(1, -1, g.pad.shape[2])
        g_int.copy_(super()._attn_b(tape, g_int))
        return g

    def _upsample_f(self, conv, x, rows, W):
        """Nearest x2 into the pad, then the 3x3 convolution at high resolution."""
        C = x.shape[2]
        pad, seq = self.arena.pad(2 * rows, 2 * W, C)
        pad[1:-1].view(rows, 2, W, 2, C).copy_(x.view(rows, 1, W, 1, C).expand(rows, 2, W, 2, C))
        self.arena.exchange(pad, seq)
        return self._conv_pad(conv.weight, conv.bias, pad)

    def _upsample_b(self, conv, g, rows, W, C):
        g = self._s_conv3_b(conv, g, 2 * rows, 2 * W)
        gp, g_int = self._new_pad(rows, W, C)
        torch.sum(g.view(1, rows, 2, W, 2, C), dim=(2, 4), out=g_int.view(1, rows, W, C))   # adjoint of nearest x2
        return gp

    def _out_f(self, x, rows, W, tape):
        """The image stripes are all-gathered: every rank returns the full image."""
        d, C = self.vae.decoder, x.shape[2]
        pad, seq = self.arena.pad(rows, W, C)
        self._gn_f(d.conv_norm_out, x, True, tape, out=pad[1:-1].view(1, rows * W, C))
        self.arena.exchange(pad, seq)
        y = self._conv_pad(d.conv_out.weight, d.conv_out.bias, pad)       # [1, rows*W, 3]
        full = torch.empty(1, rows * W * self.world, y.shape[2], dtype=torch.float32, device=y.device)
        self.dist.all_gather_into_tensor(full.view(-1), y.reshape(-1), group=self.group)
        return _nchw(full, rows * self.world, W)

    def _out_b(self, grad_image, rows, W, tape):
        d, r0 = self.vae.decoder, self.rank * rows
        g = grad_image[:, :, r0:r0 + rows, :].permute(0, 2, 3, 1).contiguous().view(1, rows * W, -1)
        g = self._s_conv3_b(d.conv_out, g, rows, W)
        gp, g_int = self._new_pad(rows, W, g.shape[2])
        self._gn_b(tape.pop(), g, out=g_int)
        return gp

    def _exit(self, g, rows, W):
        """All-gather the gradient entering conv_in, run the replicated conv_in / post_quant_conv gradients, then
        broadcast rank 0's result so the replicated latents stay bit-identical on all ranks."""
        dist = self.dist
        g_int = g.pad[1:-1].view(1, rows * W, -1)
        full = torch.empty(1, rows * W * self.world, g_int.shape[2], dtype=torch.float32, device=g_int.device)
        dist.all_gather_into_tensor(full.view(-1), g_int.reshape(-1), group=self.group)
        self.arena.release(g.seq)
        out = super()._exit(full, rows * self.world, W)
        dist.broadcast(out, src=dist.get_global_rank(self.group, 0), group=self.group)
        end_call = getattr(self.arena, "end_call", None)   # emulated arenas (tests) count absolutely
        if end_call is not None:
            end_call()
        return out
