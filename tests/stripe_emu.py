"""Torch emulations of the colour-guidance decoder kernels' C-ABI contracts (include/rtti_b200.h: rtti_gn32_silu_fwd/bwd,
rtti_gn32_silu_*_striped, rtti_add_bias_f32, rtti_upsample_phase_interleave/_scatter) for the CPU tests of
rtti_b200/vae_guidance.py and rtti_b200/stripe_parallel.py. Test infrastructure only: the product path never imports
this module."""
import torch
import torch.nn.functional as F

from rtti_b200.vae import AutoencoderKLDecoder, VAEConfig


def make_vae():
    cfg = VAEConfig(block_out_channels=(8, 8, 16, 16), norm_num_groups=4)
    vae = AutoencoderKLDecoder(cfg).init_synthetic(seed=3).float().eval()
    g = torch.Generator().manual_seed(17)
    for p in vae.parameters():   # non-trivial biases / affine parameters
        if p.dim() == 1:
            p.data.add_(0.1 * torch.randn(p.shape, generator=g))
    vae.requires_grad_(False)
    return vae


def autograd_reference(vae, zs, grad_fn):
    want = []
    for z in zs:
        zz = z.clone().requires_grad_(True)
        with torch.enable_grad():
            img = vae.decode_tensor(zz)
        img.backward(grad_fn(img.detach()))
        want.append((img.detach(), zz.grad))
    return want


def _group_sums(v, groups):   # v [hw, C] -> [groups]
    return v.view(v.shape[0], groups, -1).sum(dim=(0, 2))


def fake_ops(reduce_over_ranks):
    """name -> emulation. reduce_over_ranks(key, tensor) returns the sum of `tensor` over the ranks (the peer
    reduction of gn32_finalize_peer_kernel); every rank must call it in the same order."""
    def gn_stats(x, cb, groups, n, eps, red):
        # per rank (count, mean, sum of squared deviations) merged over the ranks (Chan et al.), as the kernels do
        xs = x[0] + (cb if cb is not None else 0)
        n_r = xs.numel() // groups
        mean_r = _group_sums(xs, groups) / n_r
        m2_r = _group_sums((xs - mean_r.repeat_interleave(xs.shape[1] // groups)) ** 2, groups)
        mean = red(mean_r * n_r) / n
        m2 = red(m2_r + n_r * (mean_r - mean) ** 2)
        rstd = torch.rsqrt(m2 / n + eps)
        return xs, torch.stack([mean, rstd], 1)[None]

    def gn_fwd(x, gamma, beta, groups, eps, silu, n, red, chan_bias, out):
        xs, stats = gn_stats(x, chan_bias, groups, n, eps, red)
        cpg = x.shape[2] // groups
        y = (xs - stats[0, :, 0].repeat_interleave(cpg)) * stats[0, :, 1].repeat_interleave(cpg) * gamma + beta
        y = F.silu(y) if silu else y
        if out is None:
            out = torch.empty_like(x)
        out.view_as(x).copy_(y[None])
        return out.view_as(x), stats

    def gn_bwd(x, dz, gamma, beta, stats, groups, silu, n, red, chan_bias, out):
        cpg = x.shape[2] // groups
        xs = x[0] + (chan_bias if chan_bias is not None else 0)
        mu, rs = stats[0, :, 0].repeat_interleave(cpg), stats[0, :, 1].repeat_interleave(cpg)
        xh = (xs - mu) * rs
        dy = dz.reshape(xs.shape)
        if silu:
            y = xh * gamma + beta
            sg = torch.sigmoid(y)
            dy = dy * sg * (1 + y * (1 - sg))
        t = dy * gamma
        c1 = (red(_group_sums(t, groups)) / n).repeat_interleave(cpg)
        c2 = (red(_group_sums(t * xh, groups)) / n).repeat_interleave(cpg)
        dx = rs * (t - c1 - xh * c2)
        if out is None:
            out = torch.empty_like(x)
        out.view_as(x).copy_(dx[None])
        return out.view_as(x)

    ident = lambda v: v

    def add_bias(a, b, bias=None, out=None):
        r = a + b + (bias if bias is not None else 0)
        return r if out is None else out.copy_(r)

    def gn_bwd_addend(x, dz, g, b, stats, groups, silu, chan_bias=None, addend=None):
        dx = gn_bwd(x, dz, g, b, stats, groups, silu, x.shape[1] * x.shape[2] // groups, ident, chan_bias, None)
        return dx if addend is None else dx + addend

    return {
        "gn32_silu_fwd": lambda x, g, b, groups, eps, silu, chan_bias=None:
            gn_fwd(x, g, b, groups, eps, silu, x.shape[1] * x.shape[2] // groups, ident, chan_bias, None),
        "gn32_silu_bwd": gn_bwd_addend,
        "gn32_silu_fwd_striped": lambda x, g, b, groups, eps, silu, hw_total, peers, seq, chan_bias=None, out=None:
            gn_fwd(x, g, b, groups, eps, silu, hw_total * x.shape[2] // groups,
                   lambda v: reduce_over_ranks(("gn", seq), v), chan_bias, out),
        "gn32_silu_bwd_striped": lambda x, dz, g, b, stats, groups, silu, hw_total, peers, seq, chan_bias=None, out=None:
            gn_bwd(x, dz, g, b, stats, groups, silu, hw_total * x.shape[2] // groups,
                   lambda v: reduce_over_ranks(("gn", seq), v), chan_bias, out),
        "add_bias_f32": add_bias,
        "upsample_phase_interleave": upsample_phase_interleave,
        "upsample_phase_scatter": upsample_phase_scatter,
    }


def upsample_phase_interleave(y4, bias, h, w):
    """y4 [B, (h+1)*(w+1), 4C], phase 2a+b in channels (2a+b)*C.. -> [B, 4*h*w, C]: output pixel (2i+a, 2j+b) is
    phase (a, b) of low-res position (i+a, j+b), plus bias."""
    B, C = y4.shape[0], y4.shape[2] // 4
    t = y4.view(B, h + 1, w + 1, 2, 2, C)
    out = torch.empty(B, 2 * h, 2 * w, C, dtype=y4.dtype)
    for a in range(2):
        for b in range(2):
            out[:, a::2, b::2] = t[:, a:a + h, b:b + w, a, b] + (bias if bias is not None else 0)
    return out.view(B, 4 * h * w, C)


def upsample_phase_scatter(g, h, w):
    """Adjoint of upsample_phase_interleave: g [B, 4*h*w, C] -> [B, (h+1)*(w+1), 4C], zero where no pixel maps."""
    B, C = g.shape[0], g.shape[2]
    g5 = g.view(B, 2 * h, 2 * w, C)
    d4 = g.new_zeros(B, h + 1, w + 1, 2, 2, C)
    for a in range(2):
        for b in range(2):
            d4[:, a:a + h, b:b + w, a, b] = g5[:, a::2, b::2]
    return d4.view(B, (h + 1) * (w + 1), 4 * C)


class FakeArenaBase:
    """Interface of stripe_parallel.StripeArena on CPU tensors; subclasses implement exchange()."""

    def __init__(self, world, rank, pad_bytes, group=None):
        self.world, self.rank, self.group = world, rank, group
        self.pad_bytes = pad_bytes
        self.halves = [torch.full((pad_bytes // 4,), float("nan")) for _ in range(2)]   # NaN: an unwritten halo shows up
        self.gn_seq = self.halo_seq = 0

    def next_gn_seq(self):
        self.gn_seq += 1
        return self.gn_seq

    def pad(self, rows, W, C):
        self.halo_seq += 1
        n = (rows + 2) * W * C
        assert n * 4 <= self.pad_bytes
        return self.halves[self.halo_seq & 1][:n].view(rows + 2, W, C), self.halo_seq

    def release(self, seq):
        assert seq == self.halo_seq
        self.halo_seq -= 1

    def check(self):
        pass


def assert_matches(results, want, rank0_results=None):
    for k, ((img, g), (img_w, g_w)) in enumerate(zip(results, want)):
        assert torch.allclose(img, img_w, rtol=1e-4, atol=1e-4 * float(img_w.abs().max()))
        assert torch.allclose(g, g_w, rtol=1e-3, atol=1e-4 * float(g_w.abs().max()))
        if rank0_results is not None:
            assert torch.equal(g, rank0_results[k][1])   # broadcast: identical on all ranks
