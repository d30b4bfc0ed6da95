"""Per-kernel timing of the rtti_b200 kernels at the SDXL 1024^2 shapes (batch 8 = the passes of one step).
CUDA events on the launching stream, 3 warm-ups, L2 flushed (256 MB write) before every timed launch,
median of 9. Prints one JSON line per kernel with achieved GB/s or TFLOP/s against MEASURED_PEAKS.json.

    python tests/kernel_bench.py > profiles/kernels.jsonl
"""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from rtti_b200 import ops  # noqa: E402


def peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        d = json.load(open(p))
        return d["hbm_gbs"], d["bf16_tflops"], "measured"
    return 6650.0, 1590.0, "fallback"


HBM, TF, SRC = peaks()
_flush = None


def timeit(fn, iters=9):
    global _flush
    if _flush is None:
        _flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    for _ in range(3):
        fn()
    ts = []
    for _ in range(iters):
        _flush.fill_(1)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2] * 1e-3


def report(name, sec, nbytes=None, flops=None, bound="hbm"):
    line = {"kernel": name, "us": round(sec * 1e6, 2), "bound": bound, "peak_source": SRC}
    if nbytes is not None:
        line["GBps"] = round(nbytes / sec / 1e9, 1); line["frac_hbm"] = round(nbytes / sec / 1e9 / HBM, 3)
    if flops is not None:
        line["TFLOPs"] = round(flops / sec / 1e12, 1); line["frac_tensor_burst"] = round(flops / sec / 1e12 / TF, 3)
    print(json.dumps(line), flush=True)


def main():
    g = torch.Generator(device="cuda").manual_seed(0)
    rn = lambda *s: torch.randn(*s, device="cuda", generator=g).half()
    B = 8
    for (H, T, tag) in ((10, 4096, "XL-64"), (20, 1024, "XL-32")):
        C = H * 64
        qkv = rn(B, T, 3 * C)
        q, k, v = qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:]
        o = torch.empty(B, T, C, device="cuda", dtype=torch.float16)
        full = 4.0 * B * H * T * T * 64
        sec = timeit(lambda: ops.attention(q, k, v, H, out=o))
        report(f"attn_self plain {tag} B{B} h{H} T{T}", sec, nbytes=2 * 4 * B * T * C, flops=full, bound="tensor")
        # injection step of the 5-region workload: entries 4..7 take the scores of entry 3 (models/region_diffusion_sdxl.py:1018-1029).
        # Algorithmic FLOPs = what the reference evaluates: QK^T only for entries that compute their own scores, PV for all.
        src = [0, 1, 2, 3, 3, 3, 3, 3]
        own = len(set(src))
        sec = timeit(lambda: ops.attention(q, k, v, H, out=o, qk_src=src))
        report(f"attn_self inject(5 share) {tag}", sec, flops=full * (own + B) / (2.0 * B), bound="tensor")
        if os.environ.get("RTTI_KBENCH_ONLY") == "self":   # A/B runs of the self-attention schedule switches
            continue
        kc, vc = rn(B, 77, C), rn(B, 77, C)
        qc = rn(B, T, C)
        sec = timeit(lambda: ops.attention(qc, kc, vc, H, out=o))
        report(f"attn_fwd cross {tag} B{B} h{H} T{T} K77", sec, nbytes=2 * (2 * B * T * C + 2 * B * 77 * C), flops=4.0 * B * H * T * 77 * 64)
        pos = torch.tensor([2, 5, 9], dtype=torch.int32, device="cuda"); fs = torch.tensor([2.0, 0.5, -1.5], device="cuda")
        sec = timeit(lambda: ops.attention(qc, kc, vc, H, out=o, word_pos=pos, font_size=fs, fs_batch_mask=2))
        report(f"attn_fwd cross+fontsize {tag}", sec, nbytes=2 * (2 * B * T * C + 2 * B * 77 * C))
        pbar = torch.zeros(1, T, 77, device="cuda")
        sec = timeit(lambda: ops.attention(qc[:2], kc[:2], vc[:2], H, pbar_accum=pbar, cap_slot=[-1, 0]))
        report(f"attn_fwd cross+capture {tag} B2", sec, nbytes=2 * (2 * 2 * T * C + 2 * 2 * 77 * C) + 8 * T * 77)
        if T == 1024:
            lse = torch.empty(2, H, T, device="cuda")
            ops.attention(q[:2], k[:2], v[:2], H, lse=lse)
            acc = torch.zeros(T, T, device="cuda")
            sec = timeit(lambda: ops.attn_probs_mean_accum(q[1], k[1], lse[1], acc, H))
            report(f"attn_probs_mean {tag}", sec, nbytes=8 * T * T + 4 * T * C, flops=2.0 * H * T * T * 64, bound="tensor")
    if os.environ.get("RTTI_KBENCH_ONLY") == "self":
        return
    if os.environ.get("RTTI_KBENCH_ONLY") == "geglu":
        for (rows, C) in ((B * 4096, 640), (B * 1024, 1280)):
            x = rn(rows, C); w = (rn(8 * C, C).float() / C ** 0.5).half(); bb = rn(8 * C)
            yo = torch.empty(rows, 4 * C, device="cuda", dtype=torch.float16)
            fl = 2.0 * rows * C * 8 * C
            sec = timeit(lambda: ops.ff_geglu(x, w, bb, out=yo))
            report(f"ff_geglu (wgmma GEMM + gate epilogue) rows{rows} C{C}", sec, flops=fl, bound="tensor")
            sec = timeit(lambda: ops.geglu(torch.nn.functional.linear(x, w, bb), out=yo))
            report(f"cuBLAS linear + geglu kernel rows{rows} C{C}", sec, flops=fl, bound="tensor")
            sec = timeit(lambda: torch.nn.functional.linear(x, w, bb))
            report(f"cuBLAS linear only rows{rows} C{C}", sec, flops=fl, bound="tensor")
        return
    for (HW, C) in ((16384, 320), (4096, 640), (4096, 1920), (1024, 1280), (1024, 2560)):
        x = rn(B, HW, C); ga, be = rn(C), rn(C); y = torch.empty_like(x); tb = rn(B, C)
        sec = timeit(lambda: ops.groupnorm_silu(x, ga, be, 32, 1e-5, True, chan_bias=tb, out=y))
        report(f"groupnorm+temb+silu B{B} HW{HW} C{C}", sec, nbytes=2 * 2 * x.numel())
    for (rows, C) in ((B * 4096, 640), (B * 1024, 1280)):
        x = rn(rows, C); ga, be = rn(C), rn(C); y = torch.empty_like(x)
        sec = timeit(lambda: ops.layernorm(x, ga, be, 1e-5, out=y))
        report(f"layernorm rows{rows} C{C}", sec, nbytes=2 * 2 * x.numel())
        pr = rn(rows, 8 * C); yo = torch.empty(rows, 4 * C, device="cuda", dtype=torch.float16)
        sec = timeit(lambda: ops.geglu(pr, out=yo))
        report(f"geglu rows{rows} inner{4 * C}", sec, nbytes=2 * (pr.numel() + yo.numel()))
    for (rows, C) in ((B * 4096, 640), (B * 1024, 1280)):   # feed-forward input projection of the two SDXL levels
        x = rn(rows, C); w = (rn(8 * C, C).float() / C ** 0.5).half(); bb = rn(8 * C)
        yo = torch.empty(rows, 4 * C, device="cuda", dtype=torch.float16)
        fl = 2.0 * rows * C * 8 * C
        sec = timeit(lambda: ops.ff_geglu(x, w, bb, out=yo))
        report(f"ff_geglu (wgmma GEMM + gate epilogue) rows{rows} C{C}", sec, flops=fl, bound="tensor")
        sec = timeit(lambda: ops.geglu(torch.nn.functional.linear(x, w, bb), out=yo))
        report(f"cuBLAS linear + geglu kernel rows{rows} C{C}", sec, flops=fl, bound="tensor")
        sec = timeit(lambda: torch.nn.functional.linear(x, w, bb))
        report(f"cuBLAS linear only rows{rows} C{C}", sec, flops=fl, bound="tensor")
    n = 4 * 128 * 128
    eu = rn(n); er = [rn(n) for _ in range(5)]; m = torch.rand(5, n, device="cuda"); lat = rn(n)
    sec = timeit(lambda: ops.region_blend_cfg(eu, er, m, 8.5, latents=lat, dt_sigma=-0.3))
    report("region_blend_cfg N5 n65536", sec, nbytes=2 * n * 8 + 4 * 5 * n, bound="latency")
    dec = torch.randn(3, 1024, 1024, device="cuda"); masks = torch.rand(1, 1024, 1024, device="cuda")
    tgt = torch.tensor([[0.99, 0.42, 0.62]], device="cuda")
    sec = timeit(lambda: ops.color_loss_fwd_bwd(dec, masks, tgt))
    report("color_loss_fwd_bwd 1024^2 R1 (3 kernels)", sec, nbytes=4 * (2 * 3 + 2 + 3) * 1024 * 1024)


if __name__ == "__main__":
    main()
