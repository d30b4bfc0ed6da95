"""Micro-benchmark (GPU): the three upsamplers of the SDXL VAE decoder at a 128x128 latent (nearest x2 + 3x3 conv),
forward and input gradient, evaluated (a) at high resolution: cuDNN on the materialised 4x copy, then the
`view.sum` adjoint, and (b) at low resolution: cuDNN 2x2 convolution with the phase-folded filters plus
rtti_upsample_phase_interleave / _scatter (vae_guidance.DecoderFwdBwd._upsample_f / _b). fp32 channels-last, TF32.
TFLOP/s counts the high-res 3x3 layer's FLOPs for both, so it is an effective rate.
    python tests/upsample_phase_bench.py"""
import json
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def bench(fn, n=10):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def main():
    from rtti_b200.vae import AutoencoderKLDecoder, VAEConfig
    from rtti_b200.vae_guidance import DecoderFwdBwd, _cl, _nchw
    torch.backends.cudnn.benchmark = True
    bwd = torch.ops.aten.convolution_backward
    # the upsampler pieces read only the conv they are given; the engine's VAE just supplies the GroupNorm config
    eng = DecoderFwdBwd(AutoencoderKLDecoder(VAEConfig(block_out_channels=(32, 64), layers_per_block=1, norm_num_groups=8)))
    print(torch.cuda.get_device_name())
    for (h, C) in ((128, 512), (256, 512), (512, 256)):
        conv = torch.nn.Conv2d(C, C, 3, padding=1).cuda().requires_grad_(False).to(memory_format=torch.channels_last)
        x = torch.randn(1, h * h, C, device="cuda")
        g = torch.randn(1, 4 * h * h, C, device="cuda")
        dummy = torch.empty(1, C, 2 * h, 2 * h, device="cuda").contiguous(memory_format=torch.channels_last)

        def hi_fwd():
            xu = x.view(1, h, 1, h, 1, C).expand(1, h, 2, h, 2, C).reshape(1, 4 * h * h, C)
            return _cl(F.conv2d(_nchw(xu, 2 * h, 2 * h), conv.weight, conv.bias, 1, 1))[0]

        def hi_bwd():
            gi = bwd(_nchw(g, 2 * h, 2 * h), dummy, conv.weight, None, [1, 1], [1, 1], [1, 1], False, [0, 0], 1,
                     [True, False, False])[0]
            return _cl(gi)[0].view(1, h, 2, h, 2, C).sum(dim=(2, 4)).reshape(1, h * h, C)

        t = {"hi_fwd": bench(hi_fwd), "hi_bwd": bench(hi_bwd),
             "phase_fwd": bench(lambda: eng._upsample_f(conv, x, h, h)),
             "phase_bwd": bench(lambda: eng._upsample_b(conv, g, h, h, C))}
        fl = 2.0 * 4 * h * h * C * C * 9
        rec = {"h": h, "C": C}
        for k, ms in t.items():
            rec[k + "_ms"] = round(ms, 3)
            rec[k + "_TFLOPs"] = round(fl / ms / 1e9, 1)
        print(json.dumps(rec), flush=True)
        del conv, x, g, dummy
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
