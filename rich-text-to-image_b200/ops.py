"""Torch-tensor front end of the C ABI (include/rtti_b200.h).

PyTorch is plumbing here: it owns the device memory and the stream; every op below hands raw
pointers, sizes and the current CUDA stream to librtti_b200.so. No op has a PyTorch fallback.
"""
import ctypes
import math

import torch

from . import _lib

_F16 = torch.float16

# number of kernels of librtti_b200.so launched since import (bench.py reports the count of a timed region)
LAUNCHES = 0
# feed-forward input projection: True = rtti_ff_geglu_fwd (hand-written wgmma GEMM with the gate in its epilogue),
# False = cuBLAS GEMM + rtti_geglu_fwd (kept for A/B measurements, profiles/)
FUSED_FF_GEGLU = True
# when a list: attention() appends (start_event, end_event, kind, flops, algorithmic_bytes) per launch
PROFILE = None


def _count(n):
    global LAUNCHES
    LAUNCHES += n


_raw_stream = getattr(torch._C, "_cuda_getCurrentRawStream", None)


def _stream():
    """Current CUDA stream handle (raw accessor when torch exposes it: ~5x cheaper than current_stream())."""
    if _raw_stream is not None:
        return ctypes.c_void_p(_raw_stream(torch.cuda.current_device()))
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)


def _req(t, dtype, name):
    if not t.is_cuda:
        raise _lib.RttiError(f"{name} must be a CUDA tensor (rtti_b200 has no CPU path)")
    if t.dtype != dtype:
        raise _lib.RttiError(f"{name} must be {dtype}, got {t.dtype}")


def _int_array(vals):
    return (ctypes.c_int * len(vals))(*[int(v) for v in vals])


def version():
    return _lib.load().rtti_version()


def arch_ok():
    return _lib.load().rtti_arch_ok() == 0


def _bsr(t):
    """(batch stride, row stride) in elements of a [B, T, C] view whose last dim is contiguous."""
    assert t.dim() == 3 and t.stride(2) == 1, "attention operands must be [B, T, heads*head_dim] with contiguous channels"
    return t.stride(0), t.stride(1)


def attention(q, k, v, heads, scale=None, qk_src=None, word_pos=None, font_size=None, fs_batch_mask=0,
              pbar_accum=None, cap_slot=None, lse=None, out=None):
    """Fused attention forward (rtti_attn_fwd). q [B,Nq,H*D], k/v [B,Nk,H*D] fp16 (strided views allowed)."""
    lib = _lib.load()
    for t, n in ((q, "q"), (k, "k"), (v, "v")):
        _req(t, _F16, n)
    B, nq, C = v.shape[0], q.shape[1], q.shape[2]
    nk = k.shape[1]
    D = C // heads
    if q.shape[0] != B or k.shape[0] != B:
        # Q / K handed over from another pass (e.g. the reference pass on a peer rank): every entry must name its source
        if qk_src is None or q.shape[0] != k.shape[0] or max(qk_src) >= q.shape[0] or len(qk_src) != B:
            raise _lib.RttiError("attention: q/k with a different batch than v need qk_src[b] < q.shape[0] for every entry of v")
    if out is None:
        out = torch.empty((B, nq, C), dtype=_F16, device=q.device)
    if scale is None:
        scale = 1.0 / math.sqrt(D)
    qb, qr = _bsr(q); kb, kr = _bsr(k); vb, vr = _bsr(v); ob, orr = _bsr(out)
    n_fs = 0
    if word_pos is not None and font_size is not None and fs_batch_mask:
        _req(word_pos, torch.int32, "word_pos"); _req(font_size, torch.float32, "font_size")
        n_fs = int(word_pos.numel())
        if font_size.numel() != n_fs:
            raise _lib.RttiError("attention: word_pos and font_size must have the same length")
    prof = PROFILE
    if prof is not None:
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record()
    rc = lib.rtti_attn_fwd(_ptr(q), _ptr(k), _ptr(v), _ptr(out), B, heads, D, nq, nk, qb, qr, kb, kr, vb, vr, ob, orr,
                           float(scale), _int_array(qk_src) if qk_src is not None else None,
                           _ptr(word_pos) if n_fs else None, _ptr(font_size) if n_fs else None, n_fs,
                           int(fs_batch_mask) if n_fs else 0,
                           _ptr(pbar_accum) if pbar_accum is not None else None,
                           _int_array(cap_slot) if cap_slot is not None else None,
                           _ptr(lse) if lse is not None else None, _stream())
    _lib.check(rc, "rtti_attn_fwd")
    _count(1)
    if prof is not None:
        ev1.record()
        # algorithmic work = what the reference evaluates: QK^T only for entries that compute their own scores (an entry
        # that is handed another entry's probabilities skips it, attention_processor.py:1160-1162), PV for every entry
        own = len(set(qk_src)) if qk_src is not None else B
        flops = 2.0 * (own + B) * heads * nq * nk * D
        nbytes = 2.0 * (2 * B * nq * C + 2 * B * nk * C)
        prof.append((ev0, ev1, "self" if nk > 80 else "cross", flops, nbytes, (B, heads, D, nq, nk)))
    return out


def attn_probs_mean_accum(q, k, lse, accum, heads, scale=None):
    """accum[Nq,Nk] += mean_h softmax(scale q_h k_h^T) for one batch entry (rtti_attn_probs_mean_accum)."""
    lib = _lib.load()
    _req(q, _F16, "q"); _req(k, _F16, "k"); _req(lse, torch.float32, "lse"); _req(accum, torch.float32, "accum")
    nq, C = q.shape
    nk = k.shape[0]
    D = C // heads
    assert q.stride(1) == 1 and k.stride(1) == 1 and lse.is_contiguous() and accum.is_contiguous()
    if scale is None:
        scale = 1.0 / math.sqrt(D)
    rc = lib.rtti_attn_probs_mean_accum(_ptr(q), _ptr(k), _ptr(lse), _ptr(accum), heads, D, nq, nk, q.stride(0),
                                        k.stride(0), float(scale), _stream())
    _lib.check(rc, "rtti_attn_probs_mean_accum")
    _count(1)
    return accum


_gn_ws = {}


def groupnorm_silu(x, gamma, beta, groups, eps, silu, chan_bias=None, out=None):
    """GroupNorm(+temb bias)(+SiLU) on channels-last x[B, HW, C] fp16 (rtti_groupnorm_silu_fwd)."""
    lib = _lib.load()
    _req(x, _F16, "x"); _req(gamma, _F16, "gamma"); _req(beta, _F16, "beta")
    assert x.dim() == 3 and x.is_contiguous()
    B, HW, C = x.shape
    if out is None:
        out = torch.empty_like(x)
    n = lib.rtti_groupnorm_workspace_elems(B, HW, C, groups)
    key = (x.device.index, torch.cuda.current_stream().cuda_stream)
    ws = _gn_ws.get(key)
    if ws is None or ws.numel() < n:
        ws = torch.empty(max(n, 1 << 16), dtype=torch.float32, device=x.device)
        _gn_ws[key] = ws
    if chan_bias is not None:
        _req(chan_bias, _F16, "chan_bias")
        assert chan_bias.shape == (B, C) and chan_bias.is_contiguous()
    rc = lib.rtti_groupnorm_silu_fwd(_ptr(x), _ptr(chan_bias), _ptr(gamma), _ptr(beta), _ptr(out), _ptr(ws), B, HW, C,
                                     groups, float(eps), 1 if silu else 0, _stream())
    _lib.check(rc, "rtti_groupnorm_silu_fwd")
    _count(3)
    return out


def layernorm(x, gamma, beta, eps, out=None):
    lib = _lib.load()
    _req(x, _F16, "x"); _req(gamma, _F16, "gamma"); _req(beta, _F16, "beta")
    assert x.is_contiguous()
    C = x.shape[-1]
    rows = x.numel() // C
    if out is None:
        out = torch.empty_like(x)
    _lib.check(lib.rtti_layernorm_fwd(_ptr(x), _ptr(gamma), _ptr(beta), _ptr(out), rows, C, float(eps), _stream()),
               "rtti_layernorm_fwd")
    _count(1)
    return out


def add_bias_layernorm(a, resid, bias, gamma, beta, eps, h_out=None, y=None):
    """h = a + resid + bias[c] (fp16, may be written over `resid`), y = LayerNorm(h) (rtti_add_bias_layernorm_fwd).
    Returns (h, y)."""
    lib = _lib.load()
    _req(a, _F16, "a"); _req(resid, _F16, "resid"); _req(gamma, _F16, "gamma"); _req(beta, _F16, "beta")
    assert a.is_contiguous() and resid.is_contiguous() and a.shape == resid.shape
    C = a.shape[-1]
    rows = a.numel() // C
    if h_out is None:
        h_out = resid
    if y is None:
        y = torch.empty_like(a)
    _lib.check(lib.rtti_add_bias_layernorm_fwd(_ptr(a), _ptr(resid), _ptr(bias), _ptr(gamma), _ptr(beta), _ptr(h_out), _ptr(y),
                                               rows, C, float(eps), _stream()), "rtti_add_bias_layernorm_fwd")
    _count(1)
    return h_out, y


def ff_geglu(x, weight, bias=None, out=None):
    """(x W_v^T + b_v) * gelu(x W_g^T + b_g) with weight [2n, k] = [W_v; W_g] (rtti_ff_geglu_fwd: wgmma GEMM with the
    gate in the epilogue). x [..., k] fp16 contiguous -> [..., n]."""
    lib = _lib.load()
    _req(x, _F16, "x"); _req(weight, _F16, "weight")
    assert x.is_contiguous() and weight.is_contiguous() and weight.shape[1] == x.shape[-1]
    k = x.shape[-1]
    n = weight.shape[0] // 2
    m = x.numel() // k
    if out is None:
        out = torch.empty(x.shape[:-1] + (n,), dtype=_F16, device=x.device)
    if bias is not None:
        _req(bias, _F16, "bias"); assert bias.is_contiguous() and bias.numel() == 2 * n
    _lib.check(lib.rtti_ff_geglu_fwd(_ptr(x), _ptr(weight), _ptr(bias), _ptr(out), m, n, k, _stream()), "rtti_ff_geglu_fwd")
    _count(1)
    return out


def geglu(proj, out=None):
    lib = _lib.load()
    _req(proj, _F16, "proj")
    assert proj.is_contiguous()
    inner = proj.shape[-1] // 2
    rows = proj.numel() // (2 * inner)
    if out is None:
        out = torch.empty(proj.shape[:-1] + (inner,), dtype=_F16, device=proj.device)
    _lib.check(lib.rtti_geglu_fwd(_ptr(proj), _ptr(out), rows, inner, _stream()), "rtti_geglu_fwd")
    _count(1)
    return out


def region_blend_cfg(eps_uncond, eps_regions, masks, guidance, latents=None, dt_sigma=0.0):
    """eps = eps_u + g (eps_t - eps_u) with the masked region sums; optionally latents + dt_sigma*eps.
    eps_regions: list of fp16 tensors (region passes in mask order, base-prompt pass last); masks fp32 [N, n]."""
    lib = _lib.load()
    _req(eps_uncond, _F16, "eps_uncond"); _req(masks, torch.float32, "masks")
    n = eps_uncond.numel()
    N = len(eps_regions)
    assert masks.is_contiguous() and masks.numel() == N * n
    for e in eps_regions:
        _req(e, _F16, "eps_region"); assert e.is_contiguous() and e.numel() == n
    ptrs = (ctypes.c_void_p * N)(*[e.data_ptr() for e in eps_regions])
    eps_out = torch.empty_like(eps_uncond)
    lat_out = torch.empty_like(latents) if latents is not None else None
    rc = lib.rtti_region_blend_cfg(_ptr(eps_uncond), ptrs, _ptr(masks), N, n, float(guidance), _ptr(eps_out),
                                   _ptr(latents), _ptr(lat_out), float(dt_sigma), _stream())
    _lib.check(rc, "rtti_region_blend_cfg")
    _count(1)
    return (eps_out, lat_out) if latents is not None else eps_out


_cl_ws = {}


def color_loss_fwd_bwd(decoded, masks, target_rgb):
    """decoded [3,H,W] fp32 (pre-clamp VAE output), masks [R,H,W] fp32, target_rgb [R,3] fp32 -> (loss[1], grad[3,H,W])."""
    lib = _lib.load()
    for t, nme in ((decoded, "decoded"), (masks, "masks"), (target_rgb, "target_rgb")):
        _req(t, torch.float32, nme); assert t.is_contiguous()
    R = masks.shape[0]
    hw = decoded.numel() // 3
    if decoded.shape[0] != 3 or masks[0].numel() != hw or tuple(target_rgb.shape) != (R, 3):
        raise _lib.RttiError(f"color_loss_fwd_bwd: decoded {tuple(decoded.shape)}, masks {tuple(masks.shape)}, "
                             f"target_rgb {tuple(target_rgb.shape)} do not agree (need [3,H,W], [R,H,W], [R,3])")
    n = lib.rtti_color_loss_workspace_elems(R, hw)
    ws = _cl_ws.get(decoded.device.index)
    if ws is None or ws.numel() < n:
        ws = torch.empty(n, dtype=torch.float32, device=decoded.device)
        _cl_ws[decoded.device.index] = ws
    loss = torch.empty(1, dtype=torch.float32, device=decoded.device)
    grad = torch.empty_like(decoded)
    rc = lib.rtti_color_loss_fwd_bwd(_ptr(decoded), _ptr(masks), _ptr(target_rgb), R, hw, _ptr(loss), _ptr(grad),
                                     _ptr(ws), _stream())
    _lib.check(rc, "rtti_color_loss_fwd_bwd")
    _count(3)
    return loss, grad


def latent_guidance_update(latents, grad, atten_all, weight):
    lib = _lib.load()
    _req(latents, _F16, "latents"); _req(grad, torch.float32, "grad"); _req(atten_all, torch.float32, "atten_all")
    if grad.numel() != latents.numel() or atten_all.numel() != latents.numel():
        raise _lib.RttiError("latent_guidance_update: latents, grad and atten_all must have the same number of elements")
    out = torch.empty_like(latents)
    rc = lib.rtti_latent_guidance_update(_ptr(latents), _ptr(grad.contiguous()), _ptr(atten_all.contiguous()),
                                         float(weight), _ptr(out), latents.numel(), _stream())
    _lib.check(rc, "rtti_latent_guidance_update")
    _count(1)
    return out


def bg_inject_blend(latents, latents_ref, mask):
    lib = _lib.load()
    _req(latents, _F16, "latents"); _req(latents_ref, _F16, "latents_ref"); _req(mask, torch.float32, "mask")
    if latents_ref.numel() != latents.numel() or mask.numel() != latents.numel():
        raise _lib.RttiError("bg_inject_blend: latents, latents_ref and mask must have the same number of elements")
    out = torch.empty_like(latents)
    rc = lib.rtti_bg_inject_blend(_ptr(latents), _ptr(latents_ref), _ptr(mask.contiguous()), _ptr(out),
                                  latents.numel(), _stream())
    _lib.check(rc, "rtti_bg_inject_blend")
    _count(1)
    return out


def predict_x0(x_t, eps, alpha):
    lib = _lib.load()
    _req(x_t, _F16, "x_t"); _req(eps, _F16, "eps")
    out = torch.empty_like(x_t)
    _lib.check(lib.rtti_predict_x0(_ptr(x_t), _ptr(eps), float(alpha), _ptr(out), x_t.numel(), _stream()),
               "rtti_predict_x0")
    _count(1)
    return out


def gather_blend_step(peer_slot_ptrs, peer_flag_ptrs, rank, slot_owner, n_regions, masks, guidance, latents, latents_ref,
                      dt_sigma, step_id):
    """Fused all-gather + blend + CFG + Euler over NVLink peer memory (rtti_gather_blend_step).
    Returns (eps, latents_out, latents_ref_out or None)."""
    lib = _lib.load()
    world = len(peer_slot_ptrs)
    n = latents.numel()
    _req(latents, _F16, "latents"); _req(masks, torch.float32, "masks")
    eps = torch.empty_like(latents)
    lat_out = torch.empty_like(latents)
    ref_out = torch.empty_like(latents_ref) if latents_ref is not None else None
    slots = (ctypes.c_void_p * world)(*peer_slot_ptrs)
    flags = (ctypes.c_void_p * world)(*peer_flag_ptrs)
    rc = lib.rtti_gather_blend_step(slots, flags, world, rank, _int_array(slot_owner), len(slot_owner), n_regions,
                                    _ptr(masks), n, float(guidance), _ptr(eps), _ptr(latents), _ptr(lat_out),
                                    _ptr(latents_ref), _ptr(ref_out), float(dt_sigma), int(step_id), _stream())
    _lib.check(rc, "rtti_gather_blend_step")
    _count(1)
    return eps, lat_out, ref_out


_gn32_ws = {}


_gn32_ws_elems = {}


def _gn32_workspace(x, groups):
    B, HW, C = x.shape
    n = _gn32_ws_elems.get((B, HW, C, groups))
    if n is None:
        n = _gn32_ws_elems[(B, HW, C, groups)] = _lib.load().rtti_gn32_workspace_elems(B, HW, C, groups)
    key = (x.device.index, _stream().value)
    ws = _gn32_ws.get(key)
    if ws is None or ws.numel() < n:
        ws = torch.empty(max(n, 1 << 18), dtype=torch.float32, device=x.device)
        _gn32_ws[key] = ws
    return ws


def gn32_silu_fwd(x, gamma, beta, groups, eps, silu, chan_bias=None):
    """fp32 channels-last GroupNorm(+SiLU): x [B, HW, C] -> (y, mean_rstd [B, G, 2])  (rtti_gn32_silu_fwd)."""
    lib = _lib.load()
    _req(x, torch.float32, "x"); _req(gamma, torch.float32, "gamma"); _req(beta, torch.float32, "beta")
    assert x.dim() == 3 and x.is_contiguous()
    B, HW, C = x.shape
    y = torch.empty_like(x)
    stats = torch.empty(B, groups, 2, dtype=torch.float32, device=x.device)
    rc = lib.rtti_gn32_silu_fwd(_ptr(x), _ptr(chan_bias), _ptr(gamma), _ptr(beta), _ptr(y), _ptr(stats), _ptr(_gn32_workspace(x, groups)),
                                B, HW, C, groups, float(eps), 1 if silu else 0, _stream())
    _lib.check(rc, "rtti_gn32_silu_fwd")
    _count(3)
    return y, stats


def gn32_silu_bwd(x, dz, gamma, beta, stats, groups, silu, chan_bias=None, addend=None):
    """Input gradient of gn32_silu_fwd (rtti_gn32_silu_bwd); `addend` (same shape as x) is added to it."""
    lib = _lib.load()
    _req(x, torch.float32, "x"); _req(dz, torch.float32, "dz")
    assert x.is_contiguous() and dz.is_contiguous() and dz.shape == x.shape
    if addend is not None:
        _req(addend, torch.float32, "addend")
        assert addend.is_contiguous() and addend.shape == x.shape
    B, HW, C = x.shape
    dx = torch.empty_like(x)
    rc = lib.rtti_gn32_silu_bwd(_ptr(x), _ptr(chan_bias), _ptr(dz), _ptr(gamma), _ptr(beta), _ptr(stats), _ptr(addend),
                                _ptr(dx), _ptr(_gn32_workspace(x, groups)), B, HW, C, groups, 1 if silu else 0, _stream())
    _lib.check(rc, "rtti_gn32_silu_bwd")
    _count(3)
    return dx


def gn32_silu_fwd_striped(x, gamma, beta, groups, eps, silu, hw_total, peers, seq, chan_bias=None, out=None):
    """Stripe-parallel gn32_silu_fwd: x [1, hw_local, C] holds this rank's rows of a [1, hw_total, C] tensor; the
    statistics are reduced over the ranks through peer memory (rtti_gn32_silu_fwd_striped). `peers` provides
    sum_ptrs / gn_flag_ptrs (ctypes arrays), world, rank. `out` may be a contiguous view (e.g. a pad interior)."""
    lib = _lib.load()
    _req(x, torch.float32, "x"); _req(gamma, torch.float32, "gamma"); _req(beta, torch.float32, "beta")
    assert x.dim() == 3 and x.shape[0] == 1 and x.is_contiguous()
    _, HW, C = x.shape
    y = torch.empty_like(x) if out is None else out
    assert y.is_contiguous() and y.numel() == x.numel() and y.dtype == torch.float32
    stats = torch.empty(1, groups, 2, dtype=torch.float32, device=x.device)
    rc = lib.rtti_gn32_silu_fwd_striped(_ptr(x), _ptr(chan_bias), _ptr(gamma), _ptr(beta), _ptr(y), _ptr(stats),
                                        _ptr(_gn32_workspace(x, groups)), HW, int(hw_total), C, groups, float(eps),
                                        1 if silu else 0, peers.sum_ptrs, peers.gn_flag_ptrs, peers.world, peers.rank,
                                        int(seq), _stream())
    _lib.check(rc, "rtti_gn32_silu_fwd_striped")
    _count(3)
    return y, stats


def gn32_silu_bwd_striped(x, dz, gamma, beta, stats, groups, silu, hw_total, peers, seq, chan_bias=None, out=None):
    """Input gradient of gn32_silu_fwd_striped (rtti_gn32_silu_bwd_striped)."""
    lib = _lib.load()
    _req(x, torch.float32, "x"); _req(dz, torch.float32, "dz")
    assert x.is_contiguous() and dz.is_contiguous() and dz.numel() == x.numel() and x.shape[0] == 1
    _, HW, C = x.shape
    dx = torch.empty_like(x) if out is None else out
    assert dx.is_contiguous() and dx.numel() == x.numel() and dx.dtype == torch.float32
    rc = lib.rtti_gn32_silu_bwd_striped(_ptr(x), _ptr(chan_bias), _ptr(dz), _ptr(gamma), _ptr(beta), _ptr(stats), _ptr(dx),
                                        _ptr(_gn32_workspace(x, groups)), HW, int(hw_total), C, groups, 1 if silu else 0,
                                        peers.sum_ptrs, peers.gn_flag_ptrs, peers.world, peers.rank, int(seq), _stream())
    _lib.check(rc, "rtti_gn32_silu_bwd_striped")
    _count(3)
    return dx


def halo_exchange(pad, pad_ptr_up, pad_ptr_down, flags_local, flags_up, flags_down, seq):
    """pad [rows + 2, W, C] fp32 (interior rows written): push the boundary rows into the neighbours' halo rows and
    wait for theirs (rtti_halo_exchange). pad_ptr_up / pad_ptr_down: peer-mapped addresses of the neighbours' pads
    (0 at the image border)."""
    lib = _lib.load()
    _req(pad, torch.float32, "pad")
    assert pad.dim() == 3 and pad.is_contiguous()
    rows = pad.shape[0] - 2
    rc = lib.rtti_halo_exchange(_ptr(pad), ctypes.c_void_p(pad_ptr_up or 0), ctypes.c_void_p(pad_ptr_down or 0), rows,
                                pad.shape[1] * pad.shape[2], ctypes.c_void_p(flags_local),
                                ctypes.c_void_p(flags_up or 0), ctypes.c_void_p(flags_down or 0), int(seq), _stream())
    _lib.check(rc, "rtti_halo_exchange")
    _count(1)


def peer_seq_advance(flags_a, da, flags_b=0, db=0):
    """flags_a[8] += da; flags_b[8] += db: advance the device-side sequence bases of the stripe exchange at the end of
    one colour-guidance evaluation (rtti_peer_seq_advance), which makes the evaluation CUDA-graph replayable."""
    lib = _lib.load()
    rc = lib.rtti_peer_seq_advance(ctypes.c_void_p(flags_a or 0), int(da), ctypes.c_void_p(flags_b or 0), int(db), _stream())
    _lib.check(rc, "rtti_peer_seq_advance")
    _count(1)


def peer_push(src, dst_ptrs, dst_flag_ptrs, flags_local, seq):
    """src [rows, width] fp16 view (unit column stride, any row stride): copy into every peer buffer of `dst_ptrs` and
    publish event `seq` to their flag words (rtti_peer_push). dst_ptrs / dst_flag_ptrs: ctypes c_void_p arrays."""
    lib = _lib.load()
    _req(src, _F16, "src")
    assert src.dim() == 2 and src.stride(1) == 1
    rc = lib.rtti_peer_push(_ptr(src), src.stride(0) * 2, src.shape[0], src.shape[1] * 2, dst_ptrs, dst_flag_ptrs,
                            len(dst_ptrs), ctypes.c_void_p(flags_local), int(seq), _stream())
    _lib.check(rc, "rtti_peer_push")
    _count(1)


def peer_wait(flags_local, seq):
    """Stream-ordered wait for event `seq` of the producer rank (rtti_peer_wait)."""
    lib = _lib.load()
    _lib.check(lib.rtti_peer_wait(ctypes.c_void_p(flags_local), int(seq), _stream()), "rtti_peer_wait")
    _count(1)


def add_bias_f32(a, b, bias=None, out=None):
    """a + b + bias[c] for fp32 [.., C] tensors (rtti_add_bias_f32); `out` may alias a or b."""
    lib = _lib.load()
    _req(a, torch.float32, "a"); _req(b, torch.float32, "b")
    assert a.is_contiguous() and b.is_contiguous() and a.shape == b.shape
    C = a.shape[-1]
    if out is None:
        out = torch.empty_like(a)
    _lib.check(lib.rtti_add_bias_f32(_ptr(a), _ptr(b), _ptr(bias), _ptr(out), a.numel() // C, C, _stream()), "rtti_add_bias_f32")
    _count(1)
    return out


def upsample_phase_interleave(y4, bias, h, w):
    """y4 [B, (h+1)*(w+1), 4C] (2x2 pad-1 convolution with the phase-folded filters of an upsampler, vae_guidance)
    -> [B, 4*h*w, C] high-res output + bias[C] (rtti_upsample_phase_interleave)."""
    lib = _lib.load()
    _req(y4, torch.float32, "y4")
    B, n, C4 = y4.shape
    assert y4.is_contiguous() and n == (h + 1) * (w + 1) and C4 % 4 == 0
    C = C4 // 4
    if bias is not None:
        _req(bias, torch.float32, "bias"); assert bias.is_contiguous() and bias.numel() == C
    out = torch.empty(B, 4 * h * w, C, dtype=torch.float32, device=y4.device)
    _lib.check(lib.rtti_upsample_phase_interleave(_ptr(y4), _ptr(bias), _ptr(out), B, h, w, C, _stream()),
               "rtti_upsample_phase_interleave")
    _count(1)
    return out


def upsample_phase_scatter(g, h, w):
    """Adjoint of upsample_phase_interleave: g [B, 4*h*w, C] -> [B, (h+1)*(w+1), 4C] (rtti_upsample_phase_scatter)."""
    lib = _lib.load()
    _req(g, torch.float32, "g")
    B, n, C = g.shape
    assert g.is_contiguous() and n == 4 * h * w
    dy4 = torch.empty(B, (h + 1) * (w + 1), 4 * C, dtype=torch.float32, device=g.device)
    _lib.check(lib.rtti_upsample_phase_scatter(_ptr(g), _ptr(dy4), B, h, w, C, _stream()), "rtti_upsample_phase_scatter")
    _count(1)
    return dy4


def add_bias_f16(a, b, bias=None, out=None):
    """a + b + bias[c] for fp16 [.., C] tensors (rtti_add_bias_f16); `out` may alias `b`."""
    lib = _lib.load()
    _req(a, _F16, "a"); _req(b, _F16, "b")
    assert a.is_contiguous() and b.is_contiguous() and a.shape == b.shape
    C = a.shape[-1]
    if out is None:
        out = torch.empty_like(a)
    _lib.check(lib.rtti_add_bias_f16(_ptr(a), _ptr(b), _ptr(bias), _ptr(out), a.numel() // C, C, _stream()), "rtti_add_bias_f16")
    _count(1)
    return out


def kmeans_fit(x, draws, max_iter=300, tol=1e-4):
    """k-means restarts of x [n, k] fp32 (rtti_kmeans_fit): draws [n_init, 1 + (k-1)*trials] fp64 from
    attention_utils.kmeans_draws. Returns (labels [n_init, n] int32, inertia [n_init] fp64, n_iter [n_init] int32,
    flags [n_init] int32); a non-zero flag marks a restart whose empty-cluster relocation scikit-learn leaves to an
    unspecified order."""
    _req(x, torch.float32, "x")
    _req(draws, torch.float64, "draws")
    x, draws = x.contiguous(), draws.contiguous()
    n, k = x.shape
    n_init = draws.shape[0]
    if draws.dim() != 2 or draws.shape[1] != 1 + (k - 1) * (2 + int(math.log(k))):
        raise _lib.RttiError(f"draws must be [n_init, 1 + (k-1)*trials] for k={k}, got {tuple(draws.shape)}")
    labels = torch.empty(n_init, n, dtype=torch.int32, device=x.device)
    inertia = torch.empty(n_init, dtype=torch.float64, device=x.device)
    n_iter = torch.empty(n_init, dtype=torch.int32, device=x.device)
    flags = torch.empty(n_init, dtype=torch.int32, device=x.device)
    lib = _lib.load()
    _lib.check(lib.rtti_kmeans_fit(_ptr(x), _ptr(draws), n, k, n_init, int(max_iter), float(tol), _ptr(labels),
                                   _ptr(inertia), _ptr(n_iter), _ptr(flags), _stream()), "rtti_kmeans_fit")
    _count(1)
    return labels, inertia, n_iter, flags


def kmeans_supported(n, k):
    """Whether rtti_kmeans_fit accepts an [n, k] embedding (host-only query, no GPU needed)."""
    return _lib.load().rtti_kmeans_supported(int(n), int(k)) == _lib.RTTI_OK
