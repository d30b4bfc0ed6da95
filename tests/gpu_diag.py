"""GPU bring-up diagnostics: each kernel case runs in its own subprocess under a timeout so a
dead-locked kernel cannot hang the box. Prints one line per case plus error details.

    python tests/gpu_diag.py            # all cases
    python tests/gpu_diag.py case_name  # one case, in-process
"""
import math
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def ref_attention(q, k, v, heads, scale=None, qk_src=None, fs=None, fs_mask=0):
    import torch
    B, nq, C = q.shape
    nk = k.shape[1]
    D = C // heads
    scale = scale or 1.0 / math.sqrt(D)
    qf = q.float().view(B, nq, heads, D).permute(0, 2, 1, 3)
    kf = k.float().view(B, nk, heads, D).permute(0, 2, 1, 3)
    vf = v.float().view(B, nk, heads, D).permute(0, 2, 1, 3)
    if qk_src is not None:
        idx = torch.tensor(qk_src, device=q.device)
        qf, kf = qf[idx], kf[idx]
    s = torch.einsum("bhqd,bhkd->bhqk", qf, kf) * scale
    p = s.softmax(-1)
    if fs is not None:
        pos, size = fs
        e = (s - s.max(-1, keepdim=True)[0]).exp()
        w_abs = torch.ones(nk, device=q.device)
        w_sgn = torch.ones(nk, device=q.device)
        for pp, ss in zip(pos.tolist(), size.tolist()):
            w_abs[pp] = abs(ss)
            w_sgn[pp] = (ss > 0) - (ss < 0)
        e2 = e * w_abs
        p2 = e2 / e2.sum(-1, keepdim=True) * w_sgn
        for b in range(B):
            if (fs_mask >> b) & 1:
                p[b] = p2[b]
    o = torch.einsum("bhqk,bhkd->bhqd", p, vf)
    lse = torch.logsumexp(s, -1) / math.log(2.0)
    return o.permute(0, 2, 1, 3).reshape(B, nq, C), p, lse


def report(name, got, exp, atol, rtol):
    import torch
    got = got.float(); exp = exp.float()
    err = (got - exp).abs()
    tol = atol + rtol * exp.abs()
    bad = (err > tol)
    nbad = int(bad.sum())
    ok = nbad == 0 and bool(torch.isfinite(got).all())
    print(f"{'PASS' if ok else 'FAIL'} {name}: max_abs_err={err.max().item():.3e} mean_err={err.mean().item():.3e} "
          f"ref_absmax={exp.abs().max().item():.3e} nbad={nbad}/{err.numel()} nan={int(torch.isnan(got).sum())}", flush=True)
    if not ok:
        idx = torch.nonzero(bad)[:6].tolist()
        print("   first bad idx:", idx)
        flat_g = got.reshape(-1, got.shape[-1]); flat_e = exp.reshape(-1, exp.shape[-1])
        print("   got[0,:8] ", [round(x, 4) for x in flat_g[0, :8].tolist()])
        print("   exp[0,:8] ", [round(x, 4) for x in flat_e[0, :8].tolist()])
        print("   got[1,:8] ", [round(x, 4) for x in flat_g[1, :8].tolist()])
        print("   exp[1,:8] ", [round(x, 4) for x in flat_e[1, :8].tolist()])
        rows_bad = bad.reshape(-1, bad.shape[-1]).any(-1)
        cols_bad = bad.reshape(-1, bad.shape[-1]).any(0)
        print(f"   bad rows {int(rows_bad.sum())}/{rows_bad.numel()} first {torch.nonzero(rows_bad)[:8].flatten().tolist()}"
              f" | bad cols {int(cols_bad.sum())}/{cols_bad.numel()} first {torch.nonzero(cols_bad)[:8].flatten().tolist()}")
    return ok


def attn_case(B, H, D, nq, nk, qk_src=None, fs=False, cap=False, fused_qkv=False, seed=0, want_lse=False):
    import torch
    from rtti_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(seed)
    C = H * D
    if fused_qkv:
        qkv = torch.randn(B, nq, 3 * C, device="cuda", generator=g).half()
        q, k, v = qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:]
    else:
        q = torch.randn(B, nq, C, device="cuda", generator=g).half()
        k = torch.randn(B, nk, C, device="cuda", generator=g).half()
        v = torch.randn(B, nk, C, device="cuda", generator=g).half()
    kw = {}
    fsr = None
    if fs:
        pos = torch.tensor([3, 7, 7, 20], dtype=torch.int32, device="cuda")
        size = torch.tensor([2.5, 0.3, -1.7, 4.0], dtype=torch.float32, device="cuda")
        kw.update(word_pos=pos, font_size=size, fs_batch_mask=0b10 if B > 1 else 1)
        fsr = (pos, size)
    if cap:
        acc = torch.full((1, nq, nk), 0.25, dtype=torch.float32, device="cuda")
        slots = [-1] * B; slots[B - 1] = 0
        kw.update(pbar_accum=acc, cap_slot=slots)
    lse = torch.zeros(B, H, nq, dtype=torch.float32, device="cuda") if want_lse else None
    o = ops.attention(q, k, v, H, qk_src=qk_src, lse=lse, **kw)
    torch.cuda.synchronize()
    o_ref, p_ref, lse_ref = ref_attention(q, k, v, H, qk_src=qk_src, fs=fsr, fs_mask=kw.get("fs_batch_mask", 0))
    name = f"attn B{B} H{H} D{D} nq{nq} nk{nk} src={qk_src} fs={fs} cap={cap} fused={fused_qkv}"
    ok = report(name, o, o_ref, 2e-3, 2e-2)
    if cap:
        ok &= report(name + " [pbar]", acc[0] - 0.25, p_ref[B - 1].mean(0), 1e-3, 1e-2)
    if want_lse:
        ok &= report(name + " [lse]", lse, lse_ref, 2e-3, 1e-3)
        accum = torch.full((nq, nk), 0.5, dtype=torch.float32, device="cuda")
        sb = qk_src[B - 1] if qk_src is not None else B - 1     # the scores of entry B-1 come from its source entry
        ops.attn_probs_mean_accum(q[sb], k[sb], lse[B - 1], accum, H)
        torch.cuda.synchronize()
        ok &= report(name + " [probs_mean]", accum - 0.5, p_ref[B - 1].mean(0), 1e-3, 1e-2)
    return ok


def case_elementwise():
    import torch
    from rtti_b200 import ops
    torch.manual_seed(0)
    ok = True
    for (B, HW, C, G) in [(2, 1024, 320, 32), (3, 4096, 640, 32), (1, 256, 1280, 32), (2, 64, 2560, 32), (2, 100, 32, 8), (1, 16384, 320, 32)]:
        x = (torch.randn(B, HW, C, device="cuda") * 2 + 0.5).half()
        ga = torch.randn(C, device="cuda").half(); be = torch.randn(C, device="cuda").half()
        tb = torch.randn(B, C, device="cuda").half()
        for silu in (False, True):
            for bias in (None, tb):
                y = ops.groupnorm_silu(x, ga, be, G, 1e-5, silu, chan_bias=bias)
                xin = x.float() + (bias.float()[:, None, :] if bias is not None else 0)
                ref = torch.nn.functional.group_norm(xin.permute(0, 2, 1), G, ga.float(), be.float(), 1e-5).permute(0, 2, 1)
                if silu:
                    ref = torch.nn.functional.silu(ref)
                ok &= report(f"groupnorm B{B} HW{HW} C{C} G{G} silu={silu} bias={bias is not None}", y, ref, 4e-3, 1e-2)
    for (rows, C) in [(4096, 640), (1024, 1280), (77, 320), (5, 2048), (64, 32)]:
        x = (torch.randn(rows, C, device="cuda") * 3 + 1).half()
        ga = torch.randn(C, device="cuda").half(); be = torch.randn(C, device="cuda").half()
        y = ops.layernorm(x, ga, be, 1e-5)
        ref = torch.nn.functional.layer_norm(x.float(), (C,), ga.float(), be.float(), 1e-5)
        ok &= report(f"layernorm rows{rows} C{C}", y, ref, 4e-3, 1e-2)
    for (rows, C) in [(4096, 640), (1024, 1280), (77, 320), (5, 2048), (64, 32)]:
        a = torch.randn(rows, C, device="cuda").half(); r = (torch.randn(rows, C, device="cuda") * 2).half()
        bi = torch.randn(C, device="cuda").half(); ga = torch.randn(C, device="cuda").half(); be = torch.randn(C, device="cuda").half()
        for bias in (bi, None):
            h_ref = (a.float() + r.float() + (bias.float() if bias is not None else 0)).half()
            y_ref = torch.nn.functional.layer_norm(h_ref.float(), (C,), ga.float(), be.float(), 1e-5)
            r2 = r.clone()
            h, y = ops.add_bias_layernorm(a, r2, bias, ga, be, 1e-5)
            assert h.data_ptr() == r2.data_ptr()
            ok &= report(f"add_bias_layernorm h rows{rows} C{C} bias={bias is not None}", h, h_ref, 2e-3, 1e-3)
            ok &= report(f"add_bias_layernorm y rows{rows} C{C} bias={bias is not None}", y, y_ref, 4e-3, 1e-2)
    for (rows, inner) in [(4096, 2560), (1024, 5120), (77, 128)]:
        pr = torch.randn(rows, 2 * inner, device="cuda").half()
        y = ops.geglu(pr)
        ref = pr[:, :inner].float() * torch.nn.functional.gelu(pr[:, inner:].float())
        ok &= report(f"geglu rows{rows} inner{inner}", y, ref, 2e-3, 1e-2)
    n = 4 * 128 * 128
    N = 5
    eu = torch.randn(n, device="cuda").half()
    er = [torch.randn(n, device="cuda").half() for _ in range(N)]
    m = torch.rand(N, n, device="cuda"); m = m / m.sum(0, keepdim=True)
    lat = torch.randn(n, device="cuda").half()
    eps, lat2 = ops.region_blend_cfg(eu, er, m, 8.5, latents=lat, dt_sigma=-0.37)
    u = eu.float() * m.sum(0); t = sum(e.float() * mm for e, mm in zip(er, m))
    ref = u + 8.5 * (t - u)
    ok &= report("region_blend_cfg eps", eps, ref, 2e-2, 1e-2)
    ok &= report("region_blend_cfg latents", lat2, lat.float() + eps.float() * -0.37, 2e-3, 1e-2)
    H = W = 256
    dec = (torch.randn(3, H, W, device="cuda") * 1.5).requires_grad_(True)
    masks = torch.rand(2, H, W, device="cuda")
    tgt = torch.tensor([[0.99, 0.42, 0.62], [0.1, 0.9, 0.3]], device="cuda")
    loss, grad = ops.color_loss_fwd_bwd(dec.detach(), masks, tgt)
    img = (dec / 2 + 0.5).clamp(0, 1)
    lt = 0
    for r in range(2):
        avg = (img[None] * masks[r][None, None]).sum(2).sum(2) / masks[r].sum()
        lt = lt + torch.nn.functional.mse_loss(avg, tgt[r][None]) * 100
    lt.backward()
    ok &= report("color_loss loss", loss, lt.detach().reshape(1), 1e-3, 1e-4)
    ok &= report("color_loss grad", grad * 1e4, dec.grad * 1e4, 1e-4, 1e-3)
    g32 = torch.randn(n, device="cuda"); att = torch.rand(n, device="cuda")
    ok &= report("latent_guidance_update", ops.latent_guidance_update(lat, g32, att, 0.5), lat.float() - g32 * 0.5 * att, 2e-3, 1e-2)
    ok &= report("bg_inject_blend", ops.bg_inject_blend(lat, eu, att), eu.float() * att + lat.float() * (1 - att), 2e-3, 1e-2)
    ok &= report("predict_x0", ops.predict_x0(lat, eu, 0.3), (lat.float() - eu.float() * math.sqrt(0.7)) / math.sqrt(0.3), 4e-3, 1e-2)
    return ok


def case_ff_geglu():
    """wgmma GEMM with the GEGLU gate in the epilogue against torch (fp32 matmul of the fp16 operands)."""
    import torch
    from rtti_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(2)
    ok = True
    for (M, C, bias) in [(128, 64, True), (256, 128, False), (300, 320, True), (4096, 640, True), (8192, 1280, True), (77, 640, True)]:
        x = torch.randn(M, C, device="cuda", generator=g).half()
        w = (torch.randn(8 * C, C, device="cuda", generator=g) / C ** 0.5).half()
        b = (0.3 * torch.randn(8 * C, device="cuda", generator=g)).half() if bias else None
        y = ops.ff_geglu(x, w, b)
        torch.cuda.synchronize()
        pr = x.float() @ w.float().t() + (b.float() if b is not None else 0)
        ref = pr[:, :4 * C] * torch.nn.functional.gelu(pr[:, 4 * C:])
        ok &= report(f"ff_geglu M{M} C{C} bias={bias}", y, ref, 3e-3, 1e-2)
    return ok


CASES = {
    "elementwise": case_elementwise,
    "ff_geglu": case_ff_geglu,
    "cross_small": lambda: attn_case(1, 1, 64, 128, 77),
    "cross_basic": lambda: attn_case(2, 4, 64, 256, 77),
    "self_1tile": lambda: attn_case(1, 1, 64, 128, 128),
    "self_small": lambda: attn_case(2, 2, 64, 256, 256),
    "self_1024": lambda: attn_case(2, 4, 64, 1024, 1024, fused_qkv=True),
    "self_4096": lambda: attn_case(1, 10, 64, 4096, 4096, fused_qkv=True),
    "cross_fs": lambda: attn_case(2, 4, 64, 256, 77, fs=True),
    "cross_cap": lambda: attn_case(2, 4, 64, 256, 77, cap=True),
    "cross_fs_cap": lambda: attn_case(2, 4, 64, 320, 77, fs=True, cap=True),
    "self_inject": lambda: attn_case(4, 2, 64, 256, 256, qk_src=[0, 1, 1, 1]),
    "self_lse_pm": lambda: attn_case(2, 4, 64, 1024, 1024, want_lse=True),
    "self_ragged": lambda: attn_case(2, 2, 64, 200, 200, want_lse=True),
    "d40": lambda: attn_case(2, 8, 40, 256, 256),
    "d40_cross": lambda: attn_case(2, 8, 40, 256, 77, cap=True),
    "d80": lambda: attn_case(2, 8, 80, 256, 256, want_lse=True),
    "d160": lambda: attn_case(2, 8, 160, 256, 256),
    "d160_cross": lambda: attn_case(2, 8, 160, 64, 77, fs=True),
    "d32": lambda: attn_case(2, 2, 32, 64, 64),
    "d8": lambda: attn_case(2, 4, 8, 64, 77),
    # self-attention over <= 80 tokens (an 8x8 mid block) takes the single-key-tile path of attn_fwd.cu: with a
    # requested log-sum-exp / token-map capture recompute, and with injected probabilities
    "self_64tok_lse_pm": lambda: attn_case(2, 8, 32, 64, 64, want_lse=True),
    "self_64tok_inject": lambda: attn_case(4, 8, 32, 64, 64, qk_src=[0, 1, 1, 1]),
    # Q / K handed over from another tensor (pass D's slab in a RemoteQK receive buffer): q, k batch 1, v batch 3
    "self_remote_qk": lambda: remote_qk_case(),
    "cross_xl64": lambda: attn_case(8, 10, 64, 4096, 77),
    "self_xl32": lambda: attn_case(8, 20, 64, 1024, 1024, fused_qkv=True),
    # injection (qk_src): entries that share a score source, each recomputing its source's softmax for its own V
    "self_group5": lambda: attn_case(8, 2, 64, 512, 512, qk_src=[0, 1, 2, 3, 3, 3, 3, 3], fused_qkv=True),
    "self_group3": lambda: attn_case(6, 2, 64, 320, 320, qk_src=[0, 1, 2, 3, 3, 3]),
    "self_group2_lse": lambda: attn_case(3, 4, 64, 200, 200, qk_src=[0, 1, 1], want_lse=True),
    "self_group7_split": lambda: attn_case(8, 2, 64, 256, 256, qk_src=[1, 1, 1, 1, 1, 1, 1, 7]),
    "self_group_scattered": lambda: attn_case(6, 2, 64, 256, 256, qk_src=[4, 1, 4, 1, 4, 5]),
    "self_group5_d40": lambda: attn_case(6, 8, 40, 256, 256, qk_src=[0, 1, 1, 1, 1, 1]),
    "self_group5_xl32": lambda: attn_case(8, 20, 64, 1024, 1024, qk_src=[0, 1, 2, 3, 3, 3, 3, 3], fused_qkv=True),
    "self_rescale": lambda: rescale_case(),
    "sanitizer_small": lambda: case_sanitizer_small(),
}


def remote_qk_case():
    """ops.attention with q / k of batch 1 (another pass's Q|K slab, strided like a [1, T, 2C] receive buffer) and v of
    batch 3: every entry applies softmax(q k^T) of entry 0 to its own values — one entry and three entries."""
    import torch
    from rtti_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(5)
    H, D, T = 4, 64, 384
    C = H * D
    qk = torch.randn(1, T, 2 * C, device="cuda", generator=g).half()
    ok = True
    for B in (1, 3):
        v = torch.randn(B, T, C, device="cuda", generator=g).half()
        o = ops.attention(qk[..., :C], qk[..., C:], v, H, qk_src=[0] * B)
        torch.cuda.synchronize()
        o_ref, _, _ = ref_attention(qk[..., :C].expand(B, -1, -1).contiguous(), qk[..., C:].expand(B, -1, -1).contiguous(), v, H)
        ok &= report(f"remote qk B{B}", o, o_ref, 2e-3, 2e-2)
    return ok


def rescale_case():
    """Row maxima that grow by far more than 2^8 from key tile to key tile: exercises the online O rescale (with and
    without injection)."""
    import torch
    from rtti_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(3)
    B, H, D, T = 3, 2, 64, 384
    q = torch.randn(B, T, H * D, device="cuda", generator=g).half()
    k = torch.randn(B, T, H * D, device="cuda", generator=g).half()
    v = torch.randn(B, T, H * D, device="cuda", generator=g).half()
    ramp = torch.linspace(0.05, 3.0, T, device="cuda")[None, :, None]     # later keys score much higher
    k = (k.float() * ramp).half()
    ok = True
    for src in (None, [0, 1, 1]):
        o = ops.attention(q, k, v, H, qk_src=src, scale=1.0)
        torch.cuda.synchronize()
        o_ref, _, _ = ref_attention(q, k, v, H, scale=1.0, qk_src=src)
        ok &= report(f"rescale src={src}", o, o_ref, 2e-3, 2e-2)
    return ok


def case_sanitizer_small():
    """Small shapes of every kernel family in one process."""
    import torch
    from rtti_b200 import ops
    ok = True
    ok &= attn_case(2, 2, 64, 256, 256)                                  # self-attention, 64-key tiles
    ok &= attn_case(4, 2, 64, 192, 192, qk_src=[0, 1, 1, 1])             # self-attention with injection
    ok &= attn_case(2, 2, 64, 128, 77, fs=True, cap=True)                # cross-attention, font sizes + capture
    ok &= attn_case(1, 2, 80, 128, 128, want_lse=True)                   # head_dim 80 (two d-chunks) + probs mean
    x = (torch.randn(2, 256, 64, device="cuda") * 2).half(); ga = torch.randn(64, device="cuda").half(); be = torch.randn(64, device="cuda").half()
    ops.groupnorm_silu(x, ga, be, 8, 1e-5, True)
    ops.layernorm(x, ga, be, 1e-5)
    ops.add_bias_layernorm(x.clone(), x.clone(), ga, ga, be, 1e-5)
    ops.geglu(torch.randn(64, 128, device="cuda").half())
    w = torch.randn(8 * 64, 64, device="cuda").half() / 8
    ops.ff_geglu(x, w, torch.randn(8 * 64, device="cuda").half())
    n = 4 * 32 * 32
    eu = torch.randn(n, device="cuda").half(); m = torch.rand(2, n, device="cuda"); lat = torch.randn(n, device="cuda").half()
    ops.region_blend_cfg(eu, [eu, lat], m, 8.5, latents=lat, dt_sigma=-0.3)
    dec = torch.randn(3, 64, 64, device="cuda"); masks = torch.rand(1, 64, 64, device="cuda")
    ops.color_loss_fwd_bwd(dec, masks, torch.tensor([[0.9, 0.4, 0.6]], device="cuda"))
    ops.latent_guidance_update(lat, torch.randn(n, device="cuda"), torch.rand(n, device="cuda"), 0.5)
    ops.bg_inject_blend(lat, eu, torch.rand(n, device="cuda"))
    ops.predict_x0(lat, eu, 0.3)
    x32 = torch.randn(1, 256, 64, device="cuda")
    y, st = ops.gn32_silu_fwd(x32, torch.randn(64, device="cuda"), torch.randn(64, device="cuda"), 8, 1e-6, True)
    ops.gn32_silu_bwd(x32, torch.randn_like(x32), torch.randn(64, device="cuda"), torch.randn(64, device="cuda"), st, 8, True)
    torch.cuda.synchronize()
    return ok


if __name__ == "__main__":
    if len(sys.argv) > 2 and sys.argv[1] == "--many":   # several cases in ONE process (bring-up; wrap in `timeout`)
        bad = []
        for name in sys.argv[2:]:
            print(f"== {name}", flush=True)
            if not CASES[name]():
                bad.append(name)
        print("MANY", "ALL PASS" if not bad else f"FAILED {bad}", flush=True)
        sys.exit(1 if bad else 0)
    if len(sys.argv) > 1:
        ok = CASES[sys.argv[1]]()
        sys.exit(0 if ok else 1)
    summary = []
    for name in CASES:
        try:
            r = subprocess.run([sys.executable, os.path.abspath(__file__), name], timeout=120, capture_output=True, text=True)
            out = (r.stdout + r.stderr).strip()
            status = "ok" if r.returncode == 0 else f"rc={r.returncode}"
        except subprocess.TimeoutExpired as e:
            out = ((e.stdout or b"").decode() if isinstance(e.stdout, bytes) else (e.stdout or "")) + "\nTIMEOUT"
            status = "TIMEOUT"
        print(f"=== {name}: {status}")
        print("\n".join(out.splitlines()[-40:]), flush=True)
        summary.append((name, status))
    print("SUMMARY", summary)
