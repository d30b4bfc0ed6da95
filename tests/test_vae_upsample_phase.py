"""The VAE decoder's upsampler evaluated at low resolution (vae_guidance.DecoderFwdBwd._upsample_f / _upsample_b with
rtti_upsample_phase_interleave / _scatter) and the addend of rtti_gn32_silu_bwd: C-ABI argument checks on CPU, then
the kernels and the layer against fp64 PyTorch on the GPU at small and real SDXL decoder shapes."""
import ctypes

import pytest
import torch
import torch.nn.functional as F


def test_upsample_phase_abi_rejects_bad_arguments_without_launching():
    from rtti_b200 import _lib
    lib = _lib.load()
    V = ctypes.c_void_p
    buf = (ctypes.c_char * 4096)()
    a = (ctypes.addressof(buf) + 15) // 16 * 16
    ARG, SHAPE, ALIGN = -1, -2, -3
    assert lib.rtti_upsample_phase_interleave(V(0), V(0), V(a), 1, 4, 4, 8, V(0)) == ARG
    assert lib.rtti_upsample_phase_interleave(V(a), V(0), V(a), 1, 0, 4, 8, V(0)) == ARG
    assert lib.rtti_upsample_phase_interleave(V(a), V(0), V(a), 1, 4, 4, 6, V(0)) == SHAPE
    assert lib.rtti_upsample_phase_interleave(V(a), V(a + 4), V(a), 1, 4, 4, 8, V(0)) == ALIGN
    assert lib.rtti_upsample_phase_scatter(V(a), V(0), 1, 4, 4, 8, V(0)) == ARG
    assert lib.rtti_upsample_phase_scatter(V(a), V(a), 0, 4, 4, 8, V(0)) == ARG
    assert lib.rtti_upsample_phase_scatter(V(a + 8), V(a), 1, 4, 4, 8, V(0)) == ALIGN
    # rtti_gn32_silu_bwd(x, chan_bias, dz, gamma, beta, mean_rstd, addend, dx, workspace, batch, hw, c, groups, silu, s)
    assert lib.rtti_gn32_silu_bwd(V(a), V(0), V(a), V(a), V(a), V(a), V(a + 4), V(a), V(a), 1, 16, 64, 32, 1, V(0)) == ALIGN


def _engine():
    from rtti_b200.vae import AutoencoderKLDecoder, VAEConfig
    from rtti_b200.vae_guidance import DecoderFwdBwd
    return DecoderFwdBwd(AutoencoderKLDecoder(VAEConfig(block_out_channels=(32, 64), layers_per_block=1,
                                                        norm_num_groups=8)))


def _rel(got, ref):
    return float((got.double() - ref).abs().max() / ref.abs().max())


# (low-res size, channels): the three upsamplers of the SDXL decoder at a 128x128 latent, and small odd shapes
SHAPES = [(5, 8), (7, 32), (128, 512), (256, 512), (512, 256)]


@pytest.mark.gpu
@pytest.mark.parametrize("h,C", SHAPES)
def test_upsample_phase_layer_matches_fp64(h, C):
    """_upsample_f against conv2d(interpolate(x)) and _upsample_b against its autograd input gradient, in fp64.
    TF32 products (10-bit mantissa) over 9*C terms: 2e-3 of the output range."""
    from rtti_b200 import ops
    eng = _engine()
    g = torch.Generator(device="cuda").manual_seed(h + C)
    w = h + 3 if h < 64 else h
    conv = torch.nn.Conv2d(C, C, 3, padding=1).cuda().requires_grad_(False)
    conv.weight.copy_(torch.randn(C, C, 3, 3, device="cuda", generator=g) / (9 * C) ** 0.5)
    conv.bias.copy_(torch.randn(C, device="cuda", generator=g))
    conv.to(memory_format=torch.channels_last)
    x = torch.randn(1, h * w, C, device="cuda", generator=g)
    gy = torch.randn(1, 4 * h * w, C, device="cuda", generator=g)
    xd = x.double().view(1, h, w, C).permute(0, 3, 1, 2).requires_grad_(True)
    with torch.enable_grad():
        ref = F.conv2d(F.interpolate(xd, scale_factor=2.0, mode="nearest"), conv.weight.double(), conv.bias.double(), 1, 1)
        (gx_ref,) = torch.autograd.grad(ref, xd, gy.double().view(1, 2 * h, 2 * w, C).permute(0, 3, 1, 2))
    ref = ref.detach().permute(0, 2, 3, 1).reshape(1, 4 * h * w, C)
    gx_ref = gx_ref.permute(0, 2, 3, 1).reshape(1, h * w, C)
    y = eng._upsample_f(conv, x, h, w)
    gx = eng._upsample_b(conv, gy, h, w, C)
    assert y.shape == ref.shape and gx.shape == gx_ref.shape
    assert _rel(y, ref) < 2e-3, _rel(y, ref)
    assert _rel(gx, gx_ref) < 2e-3, _rel(gx, gx_ref)
    # the interleave and scatter kernels move data exactly: compare against the same reordering in torch
    y4 = torch.randn(1, (h + 1) * (w + 1), 4 * C, device="cuda", generator=g)
    t = y4.view(h + 1, w + 1, 2, 2, C)
    want = torch.empty(2 * h, 2 * w, C, device="cuda")
    for a in range(2):
        for b in range(2):
            want[a::2, b::2] = t[a:a + h, b:b + w, a, b] + conv.bias
    assert torch.equal(ops.upsample_phase_interleave(y4, conv.bias, h, w).view(2 * h, 2 * w, C), want)
    d4 = ops.upsample_phase_scatter(gy, h, w).view(h + 1, w + 1, 2, 2, C)
    want = torch.zeros_like(d4)
    g5 = gy.view(2 * h, 2 * w, C)
    for a in range(2):
        for b in range(2):
            want[a:a + h, b:b + w, a, b] = g5[a::2, b::2]
    assert torch.equal(d4, want)


@pytest.mark.gpu
def test_gn32_bwd_addend():
    from rtti_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(4)
    x = torch.randn(1, 1000, 128, device="cuda", generator=g)
    dz, add = torch.randn_like(x), torch.randn_like(x)
    ga, be = torch.randn(128, device="cuda", generator=g), torch.randn(128, device="cuda", generator=g)
    _, st = ops.gn32_silu_fwd(x, ga, be, 32, 1e-6, True)
    dx = ops.gn32_silu_bwd(x, dz, ga, be, st, 32, True)
    assert torch.equal(ops.gn32_silu_bwd(x, dz, ga, be, st, 32, True, addend=add), dx + add)


@pytest.mark.gpu
def test_sdxl_decoder_forward_backward_at_128_latent_matches_autograd():
    """The whole SDXL decoder at the 1024^2 shape colour guidance runs, image and d/dz, against autograd through
    vae.decode_tensor (tolerances of test_vae_explicit_forward_backward_matches_autograd)."""
    from rtti_b200.vae import AutoencoderKLDecoder, VAEConfig
    from rtti_b200.vae_guidance import DecoderFwdBwd
    from tests.test_parity_gpu import _close
    vae = AutoencoderKLDecoder(VAEConfig.sdxl()).init_synthetic(0).finalize("cuda")
    g = torch.Generator(device="cuda").manual_seed(0)
    z = torch.randn(1, 4, 128, 128, device="cuda", generator=g)
    z1 = z.clone().requires_grad_(True)
    with torch.enable_grad():
        img = vae.decode_tensor(z1)
    gi = torch.randn(img.shape, device="cuda", generator=g)
    img.backward(gi)
    img_ref, gz_ref = img.detach().cpu(), z1.grad.cpu()
    del img, z1
    torch.cuda.empty_cache()
    eng = DecoderFwdBwd(vae)
    img2 = eng.forward(z)
    gz = eng.backward(gi)
    _close(img2.cpu(), img_ref, 2e-2, 2e-2, "SDXL decoder forward")
    _close(gz.cpu(), gz_ref, "range", 3e-2, "SDXL decoder backward (d/dz)")
