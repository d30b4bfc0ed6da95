"""The colour-guidance kernels against float64 references at the shapes the SDXL decoder runs.

Tolerance rule, used throughout: for each op compute
  * a float64 reference on the GPU,
  * PyTorch's own fp32 implementation of the same op on the same inputs (F.group_norm (+ F.silu) with autograd, the
    reference colour-loss expression, vae.decode_tensor with TF32 convolutions),
  * the kernel / engine result,
and require err_kernel <= K * err_torch32 + floor with err = max|x - ref64| and floor a few fp32 ulps of the output
range (half an fp16 ulp for fp16 outputs). That is: no worse than the implementation it replaces, at the same
precision. A fixed absolute tolerance would let a kernel that is several times less accurate pass. The rule lives in
tests/fp64_rule.py, shared with tests/test_unet_kernels_fp64.py.
Every case prints both errors ("[fp64] ..." lines, visible with -s)."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

from tests.fp64_rule import EPS32, absmax as _absmax, half_ulp16, no_worse as _no_worse


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


# ------------------------------------------------------------------------------------------------ a. gn32 (fp32)
def _gn_ref(x, gamma, beta, G, eps, silu, chan_bias, dz, addend):
    """F.group_norm (+ F.silu) of x + chan_bias on channels-last [B, HW, C] in x's dtype; returns (y, dx (+ addend))."""
    xs = x if chan_bias is None else x + chan_bias
    xs = xs.detach().requires_grad_(True)
    with torch.enable_grad():
        y = F.group_norm(xs.permute(0, 2, 1), G, gamma, beta, eps).permute(0, 2, 1)
        if silu:
            y = F.silu(y)
        (dx,) = torch.autograd.grad(y, xs, dz)
    if addend is not None:
        dx = dx + addend
    return y.detach().contiguous(), dx.contiguous()


def _check_gn32(B, HW, C, G, silu, seed, bias=False, addend=False, scale=2.0, offset=0.3, offset_via_bias=False):
    from rtti_b200 import ops
    g = _gen(seed)
    eps = 1e-6
    x = torch.randn(B, HW, C, device="cuda", generator=g) * scale
    cb = None
    if offset_via_bias:
        cb = torch.full((C,), offset, device="cuda")
    else:
        x += offset
        if bias:
            cb = torch.randn(C, device="cuda", generator=g)
    ga = 1 + 0.5 * torch.randn(C, device="cuda", generator=g)
    be = 0.5 * torch.randn(C, device="cuda", generator=g)
    dz = torch.randn(B, HW, C, device="cuda", generator=g)
    add = torch.randn(B, HW, C, device="cuda", generator=g) if addend else None
    tag = f"gn32 B{B} HW{HW} C{C} G{G} silu={silu} bias={cb is not None} addend={addend} offset={offset:g}/{scale:g}"

    dd = lambda t: None if t is None else t.double()
    y64, dx64 = _gn_ref(x.double(), ga.double(), be.double(), G, eps, silu, dd(cb), dz.double(), dd(add))
    y32, dx32 = _gn_ref(x, ga, be, G, eps, silu, cb, dz, add)
    y, st = ops.gn32_silu_fwd(x, ga, be, G, eps, silu, chan_bias=cb)
    _no_worse(tag + " y", y, y32, y64)
    del y, y32, y64
    dx = ops.gn32_silu_bwd(x, dz, ga, be, st, G, silu, chan_bias=cb, addend=add)
    _no_worse(tag + " dx", dx, dx32, dx64)
    del dx, dx32, dx64, x, dz, add
    torch.cuda.empty_cache()


# (C, HW) of every GroupNorm of the SDXL decoder at a 1024^2 image (128^2 latent), G = 32, batch 1
SDXL_GN = [(512, 128 * 128), (512, 256 * 256), (512, 512 * 512), (256, 512 * 512), (256, 1024 * 1024),
           (128, 1024 * 1024)]


@pytest.mark.gpu
@pytest.mark.parametrize("C,HW", SDXL_GN)
def test_gn32_at_sdxl_decoder_shapes_vs_fp64(C, HW):
    """The chunk plan at hw up to 1M: ~1050 chunks, rows per chunk rounded to rowlanes, a ragged last chunk; SiLU with
    the folded conv bias and the shortcut-gradient addend as the resnet blocks use them."""
    _check_gn32(1, HW, C, 32, True, seed=C + HW, bias=True, addend=True)


@pytest.mark.gpu
def test_gn32_attention_norm_without_silu_vs_fp64():
    _check_gn32(1, 128 * 128, 512, 32, False, seed=5)


# (B, HW, C, G): hw not a multiple of anything, 1..3 channels per group (C = 96: one float4 spans two groups), C = 4,
# C = 2048 (c/4 = 512 threads, the kernels' limit), batch 2 and 3 (the chunk target of gn32_plan depends on batch)
ODD_GN = [(1, 1, 512, 32), (1, 7, 512, 32), (1, 255, 128, 32), (1, 257, 256, 32), (1, 1000, 64, 32),
          (1, 300, 32, 32), (1, 300, 64, 32), (1, 301, 96, 32), (1, 999, 4, 2), (1, 64, 2048, 32),
          (2, 1000, 512, 32), (3, 4097, 128, 32)]


@pytest.mark.gpu
@pytest.mark.parametrize("B,HW,C,G", ODD_GN)
@pytest.mark.parametrize("silu,bias,addend", [(True, False, False), (False, True, True)])
def test_gn32_odd_shapes_vs_fp64(B, HW, C, G, silu, bias, addend):
    _check_gn32(B, HW, C, G, silu, seed=B * 7 + HW + C, bias=bias, addend=addend)


def test_gn32_abi_rejects_more_channels_than_a_cta_can_hold_without_launching():
    """c/4 threads per row lane: above 512 (c > 2048) the backward kernels' registers do not fit a 1024-thread CTA, so
    the shape is refused instead of failing at launch."""
    from rtti_b200 import _lib
    lib = _lib.load()
    V = ctypes.c_void_p
    buf = (ctypes.c_char * 4096)()
    a = (ctypes.addressof(buf) + 15) // 16 * 16
    SHAPE = -2
    # rtti_gn32_silu_fwd(x, chan_bias, gamma, beta, y, mean_rstd, workspace, batch, hw, c, groups, eps, silu, stream)
    assert lib.rtti_gn32_silu_fwd(V(a), V(0), V(a), V(a), V(a), V(a), V(a), 1, 64, 4096, 32, 1e-6, 1, V(0)) == SHAPE
    # rtti_gn32_silu_bwd(x, chan_bias, dz, gamma, beta, mean_rstd, addend, dx, workspace, batch, hw, c, groups, silu, s)
    assert lib.rtti_gn32_silu_bwd(V(a), V(0), V(a), V(a), V(a), V(a), V(0), V(a), V(a), 1, 64, 2052, 36, 1, V(0)) == SHAPE


OFFSETS = [0.0, 10.0, 100.0, 1000.0]


@pytest.mark.gpu
@pytest.mark.parametrize("C,HW", [(512, 128 * 128), (256, 512 * 512)])
@pytest.mark.parametrize("via_bias", [False, True])
@pytest.mark.parametrize("offset", OFFSETS)
def test_gn32_statistics_hold_for_offset_inputs(C, HW, via_bias, offset):
    """x = randn + offset (mean/std = offset), in x itself or supplied through chan_bias as conv biases are. A
    variance computed as E[x^2] - E[x]^2 in fp32 loses log10(offset^2) digits; PyTorch's GroupNorm does not."""
    _check_gn32(1, HW, C, 32, True, seed=11, scale=1.0, offset=offset, offset_via_bias=via_bias)


# ------------------------------------------------------------------------------------------------ b. fp16 GroupNorm
def test_fp16_groupnorm_abi_rejects_more_than_1024_threads_without_launching():
    """rtti_groupnorm_silu_fwd runs c/8 threads per row lane: c = 8192 (1024 threads) is the largest accepted shape and
    is checked on the GPU below; one vector more is refused."""
    from rtti_b200 import _lib
    lib = _lib.load()
    V = ctypes.c_void_p
    buf = (ctypes.c_char * 4096)()
    a = (ctypes.addressof(buf) + 15) // 16 * 16
    # rtti_groupnorm_silu_fwd(x, chan_bias, gamma, beta, y, workspace, batch, hw, c, groups, eps, silu, stream)
    assert lib.rtti_groupnorm_silu_fwd(V(a), V(0), V(a), V(a), V(a), V(a), 1, 64, 8200, 8, 1e-5, 1, V(0)) == -2


@pytest.mark.gpu
@pytest.mark.parametrize("B,HW,C", [(2, 128 * 128, 320), (2, 32 * 32, 1280), (1, 64, 8192)])
@pytest.mark.parametrize("temb", [False, True])
@pytest.mark.parametrize("offset", OFFSETS)
def test_fp16_groupnorm_statistics_hold_for_offset_inputs(B, HW, C, temb, offset):
    """rtti_groupnorm_silu_fwd (UNet, fp16 in/out, fp32 statistics) on x = randn + offset, the offset in x or in the
    temb chan_bias, at two UNet shapes and at c = 8192 (1024 threads per CTA, the largest the entry point accepts)."""
    check_fp16_groupnorm(B, HW, C, temb, offset, seed=int(offset) + C + temb)


def check_fp16_groupnorm(B, HW, C, temb, offset, seed, k=4.0, mean=False):
    """ops.groupnorm_silu (G = 32, SiLU) on x = randn + offset, the offset in x or in the temb chan_bias. Reference:
    float64 on the same fp16 inputs; PyTorch: fp32 GroupNorm + SiLU rounded to fp16. Floor: the fp16 output rounding,
    half an fp16 ulp of max|y|."""
    from rtti_b200 import ops
    g = _gen(seed)
    G, eps = 32, 1e-5
    x = torch.randn(B, HW, C, device="cuda", generator=g)
    cb = None
    if temb:
        cb = (offset + 0.5 * torch.randn(B, C, device="cuda", generator=g)).half()
    else:
        x += offset
    x = x.half()
    ga = (1 + 0.5 * torch.randn(C, device="cuda", generator=g)).half()
    be = (0.5 * torch.randn(C, device="cuda", generator=g)).half()

    def ref(dt):
        xs = x.to(dt) + (cb.to(dt)[:, None, :] if cb is not None else 0)
        return F.silu(F.group_norm(xs.permute(0, 2, 1), G, ga.to(dt), be.to(dt), eps)).permute(0, 2, 1)

    y64 = ref(torch.float64)
    y32 = ref(torch.float32).half()
    y = ops.groupnorm_silu(x, ga, be, G, eps, True, chan_bias=cb)
    _no_worse(f"fp16 groupnorm B{B} HW{HW} C{C} temb={temb} offset={offset:g}", y, y32, y64, floor=half_ulp16(y64),
              k=k, mean=mean)


# ------------------------------------------------------------------------------------------------ c. striped, world 1
class _OnePeer:
    """This rank's own zeroed statistics slot and flag words: with world = 1 gn32_finalize_peer_kernel waits on nobody."""

    def __init__(self):
        self.sums = torch.zeros(2 * 3 * 32, dtype=torch.float32, device="cuda")
        self.flags = torch.zeros(16, dtype=torch.int32, device="cuda")
        self.sum_ptrs = (ctypes.c_void_p * 1)(self.sums.data_ptr())
        self.gn_flag_ptrs = (ctypes.c_void_p * 1)(self.flags.data_ptr())
        self.world, self.rank = 1, 0


@pytest.mark.gpu
@pytest.mark.parametrize("C,HW", [(512, 128 * 128), (128, 1024 * 1024), (64, 1000)])
def test_gn32_striped_world_one_is_bit_identical_to_unstriped(C, HW):
    """gn32_silu_{fwd,bwd}_striped with a single peer against the unstriped kernels: statistics, y and dx bit-identical
    (the rank-order merge of one slot is exact). Covers gn32_finalize_peer_kernel on one GPU."""
    from rtti_b200 import ops
    g = _gen(C)
    x = torch.randn(1, HW, C, device="cuda", generator=g) * 2 + 30
    ga, be, cb = (torch.randn(C, device="cuda", generator=g) for _ in range(3))
    dz = torch.randn_like(x)
    peers = _OnePeer()
    for silu in (False, True):
        y, st = ops.gn32_silu_fwd(x, ga, be, 32, 1e-6, silu, chan_bias=cb)
        dx = ops.gn32_silu_bwd(x, dz, ga, be, st, 32, silu, chan_bias=cb)
        ys, sts = ops.gn32_silu_fwd_striped(x, ga, be, 32, 1e-6, silu, HW, peers, 1 + 2 * silu, chan_bias=cb)
        dxs = ops.gn32_silu_bwd_striped(x, dz, ga, be, sts, 32, silu, HW, peers, 2 + 2 * silu, chan_bias=cb)
        torch.cuda.synchronize()
        assert int(peers.flags[1]) == 0, "peer wait reported an error"
        assert torch.equal(sts, st) and torch.equal(ys, y) and torch.equal(dxs, dx), (
            f"striped != unstriped: stats {(sts - st).abs().max():.3e} y {(ys - y).abs().max():.3e} "
            f"dx {(dxs - dx).abs().max():.3e}")


# ------------------------------------------------------------------------------------------------ d. colour loss
def test_color_loss_abi_rejects_more_than_16_colors_without_launching():
    from rtti_b200 import _lib
    lib = _lib.load()
    V = ctypes.c_void_p
    buf = (ctypes.c_char * 4096)()
    a = (ctypes.addressof(buf) + 15) // 16 * 16
    ARG = -1
    # rtti_color_loss_fwd_bwd(decoded, masks, target_rgb, n_colors, hw, loss, grad, workspace, stream)
    assert lib.rtti_color_loss_fwd_bwd(V(a), V(a), V(a), 17, 64, V(a), V(a), V(a), V(0)) == ARG
    assert lib.rtti_color_loss_fwd_bwd(V(a), V(a), V(a), 0, 64, V(a), V(a), V(a), V(0)) == ARG
    assert lib.rtti_color_loss_workspace_elems(17, 64) == 0
    assert lib.rtti_color_loss_workspace_elems(16, 64) > 0


def _color_loss_ref(dec, masks, tgt):
    """The reference expression: (dec/2 + 0.5).clamp(0, 1), masked mean colour, mse_loss * 100 summed over colours;
    returns (loss, d loss / d dec) by autograd in the dtype of the inputs."""
    d = dec.detach().requires_grad_(True)
    with torch.enable_grad():
        img = (d / 2 + 0.5).clamp(0, 1)
        loss = 0.
        for m, t in zip(masks, tgt):
            avg = (img * m).sum((1, 2)) / m.sum()
            loss = loss + F.mse_loss(avg, t) * 100
        (gd,) = torch.autograd.grad(loss, d)
    return loss.detach().reshape(1), gd


@pytest.mark.gpu
@pytest.mark.parametrize("H,W", [(1024, 1024), (1000, 1001)])
@pytest.mark.parametrize("R", [1, 2, 5, 16])
def test_color_loss_vs_fp64(H, W, R):
    """color_loss_fwd_bwd at the 1024^2 size guidance runs and an odd size, 1..16 colours (CL_MAXC), masks with exact
    zeros and one that is zero outside a small patch, decoder values exactly at -1 / +1 and one fp32 ulp beyond."""
    from rtti_b200 import ops
    g = _gen(R * 31 + H)
    dec = torch.randn(3, H, W, device="cuda", generator=g) * 0.7
    flat = dec.view(3, -1)
    n_edge = 64
    one = torch.tensor(1.0, device="cuda")
    for i, v in enumerate((-one, one, torch.nextafter(-one, -2 * one), torch.nextafter(one, 2 * one))):
        flat[:, i * 997:i * 997 + n_edge] = v   # -1, +1 and one fp32 ulp beyond each
    masks = torch.rand(R, H, W, device="cuda", generator=g)
    masks[masks < 0.3] = 0.0
    masks[0] = 0.0
    masks[0, H // 3:H // 3 + 9, W // 2:W // 2 + 13] = torch.rand(9, 13, device="cuda", generator=g) + 0.1
    tgt = torch.rand(R, 3, device="cuda", generator=g)

    loss, grad = ops.color_loss_fwd_bwd(dec, masks, tgt)
    l32, g32 = _color_loss_ref(dec, masks, tgt)
    l64, g64 = _color_loss_ref(dec.double(), masks.double(), tgt.double())
    # where fp32 rounding of dec/2 + 0.5 lands on the clamp edge (dec = 1 + 1 ulp -> exactly 1.0) the fp32 expression
    # passes the gradient and the exact one does not: there the kernel must do what torch.clamp does in fp32
    img32 = dec / 2 + 0.5
    edge = ((img32 >= 0) & (img32 <= 1)) != ((dec.double() / 2 + 0.5 >= 0) & (dec.double() / 2 + 0.5 <= 1))
    assert bool(edge.view(3, -1)[:, 3 * 997:3 * 997 + n_edge].all()) and bool((img32[edge] == 1).all())
    assert torch.equal(grad == 0, g32 == 0), "gradient passes the clamp where torch.clamp's does not (or vice versa)"
    ge, g32e = grad[edge], g32[edge]
    assert bool(((ge - g32e).abs() <= 1e-5 * g32e.abs() + 4 * EPS32 * _absmax(g32)).all()), "gradient at the clamp edge"
    keep = ~edge
    tag = f"color loss {H}x{W} R{R}"
    _no_worse(tag + " loss", loss, l32, l64)
    _no_worse(tag + " grad", grad[keep], g32[keep], g64[keep])


# ------------------------------------------------------------------------------------------------ e. add_bias
@pytest.mark.gpu
@pytest.mark.parametrize("with_bias", [True, False])
def test_add_bias_f32_and_f16_are_exact(with_bias):
    """out = (a + b) + bias: fp32 bit-exact; fp16 = the fp32 sum rounded once. C = 8*33 so that i % cvec wraps
    unevenly, and enough rows that the grid-stride loop wraps too."""
    from rtti_b200 import ops
    g = _gen(3 + with_bias)
    C = 8 * 33
    for rows, dt in ((10007, torch.float32), (20011, torch.float16), (3, torch.float32), (5, torch.float16)):
        a = (torch.randn(rows, C, device="cuda", generator=g) * 10).to(dt)
        b = torch.randn(rows, C, device="cuda", generator=g).to(dt)
        bias = (torch.randn(C, device="cuda", generator=g) * 3).to(dt) if with_bias else None
        if dt == torch.float32:
            got = ops.add_bias_f32(a, b, bias)
            want = a + b + (bias if with_bias else 0)
        else:
            got = ops.add_bias_f16(a, b, bias)
            want = (a.float() + b.float() + (bias.float() if with_bias else 0)).half()
        assert torch.equal(got, want), f"add_bias {dt} rows={rows}: max diff {(got.float() - want.float()).abs().max()}"


# ------------------------------------------------------------------------------------------------ f. whole decoder
def _sdxl_vae(seed):
    from rtti_b200.vae import AutoencoderKLDecoder, VAEConfig
    vae = AutoencoderKLDecoder(VAEConfig.sdxl()).init_synthetic(seed)
    g = torch.Generator().manual_seed(seed + 100)
    for p in vae.parameters():   # non-trivial biases and GroupNorm affines: conv biases reach the kernels as chan_bias
        if p.dim() == 1:
            p.data.add_(0.1 * torch.randn(p.shape, generator=g))
    return vae.finalize("cuda")


@pytest.mark.gpu
@pytest.mark.parametrize("latent", [32, 64])
def test_sdxl_decoder_vs_fp64(latent):
    """DecoderFwdBwd.forward / .backward of the SDXL decoder against float64 autograd through a .double() copy of the
    same module; image and dz errors within 2x of what TF32 autograd through decode_tensor achieves."""
    import copy
    from rtti_b200.vae_guidance import DecoderFwdBwd
    vae = _sdxl_vae(latent)
    g = _gen(latent)
    z = torch.randn(1, 4, latent, latent, device="cuda", generator=g)
    gi = torch.randn(1, 3, 8 * latent, 8 * latent, device="cuda", generator=g)

    def autograd(module, zz, gg):
        zz = zz.clone().requires_grad_(True)
        with torch.enable_grad():
            img = module.decode_tensor(zz)
        img.backward(gg)
        return img.detach(), zz.grad

    vae64 = copy.deepcopy(vae).double()
    img64, gz64 = autograd(vae64, z.double(), gi.double())
    del vae64
    torch.cuda.empty_cache()
    prev = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = True
    try:
        img32, gz32 = autograd(vae, z, gi)
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = prev
    torch.cuda.empty_cache()
    eng = DecoderFwdBwd(vae)
    img = eng.forward(z)
    gz = eng.backward(gi)
    _no_worse(f"SDXL decoder {latent}^2 image", img, img32, img64, k=2.0)
    _no_worse(f"SDXL decoder {latent}^2 dz", gz, gz32, gz64, k=2.0)


# ------------------------------------------------------------------------------------------------ g. GuidanceGraph
@pytest.mark.gpu
def test_guidance_graph_replays_match_eager_on_new_inputs():
    """vae_guidance.GuidanceGraph on one GPU: call 1 eager, call 2 captures + replays, call 3 replays after copying new
    z / masks / targets into the static buffers. Each call's loss and gradient must equal a fresh eager
    engine.forward -> color_loss_fwd_bwd -> engine.backward on the same inputs, bit for bit (the replay runs the same
    kernels on the same data; cuDNN is held to deterministic algorithms so that eager runs repeat too)."""
    from rtti_b200 import ops
    from rtti_b200.vae_guidance import DecoderFwdBwd, GuidanceGraph
    vae = _sdxl_vae(7)
    h, R = 32, 3
    g = _gen(9)
    inputs = [(torch.randn(1, 4, h, h, device="cuda", generator=g),
               torch.rand(R, 8 * h, 8 * h, device="cuda", generator=g),
               torch.rand(R, 3, device="cuda", generator=g)) for _ in range(3)]
    prev = torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
    try:
        gg = GuidanceGraph(DecoderFwdBwd(vae))
        fresh = DecoderFwdBwd(vae)
        got = []
        for z, m, t in inputs:
            loss, grad = gg(z, m, t)
            loss, grad = loss.clone(), grad.clone()
            img = fresh.forward(z)
            want_loss, gimg = ops.color_loss_fwd_bwd(img[0].contiguous(), m, t)
            want_grad = fresh.backward(gimg[None])
            k = len(got) + 1
            assert torch.equal(loss, want_loss), f"call {k}: loss {float(loss)} != eager {float(want_loss)}"
            assert torch.equal(grad, want_grad), f"call {k}: grad max diff {(grad - want_grad).abs().max():.3e}"
            got.append((loss, grad))
        assert gg.graph is not None and gg.calls == 3
        assert not torch.equal(got[2][1], got[1][1]) and float(got[2][0]) != float(got[1][0])
    finally:
        torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = prev
