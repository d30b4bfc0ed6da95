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


_DTYPE_NAME = {torch.float32: "fp32", _F16: "fp16"}


def _overlap(a, b):
    """Whether the storage spans of two tensors intersect."""
    a0, b0 = a.data_ptr(), b.data_ptr()
    return a0 < b0 + b.numel() * b.element_size() and b0 < a0 + a.numel() * a.element_size()


class _Step:
    """The fused scheduler update of one blend call: its floats `coeffs`, the [n] buffers of the main trajectory and
    those of the reference-latent trajectory (gather_blend_step only), in the order the entry points take them. `form`
    is the suffix of the entry points that run the update (_lib.BLEND_FORMS)."""
    form = ""
    what = ""               # the update's name in error messages
    coeff_names = None      # when given, the number of coeffs is checked
    names = dtypes = ()     # per buffer of one trajectory
    read_only = ()          # buffers the update only reads: no output of the call may overlap them
    has_eps_ref_out = False

    def __init__(self, coeffs, main=(), ref=None, eps_ref_out=None):
        self.coeffs = tuple(float(c) for c in coeffs)
        if self.coeff_names and len(self.coeffs) != len(self.coeff_names):
            raise _lib.RttiError(f"{self.what} blend: coeffs must be ({', '.join(self.coeff_names)}), got "
                                 f"{len(self.coeffs)} values")
        self.main = tuple(main)
        self.ref = tuple(ref) if ref is not None else (None,) * len(self.main)
        self.eps_ref_out = eps_ref_out

    def _needed(self):
        """Per buffer of one trajectory: whether this step reads or writes it (it may be None otherwise)."""
        return ()

    def _check(self, n, ref, outs=()):
        """Refuse a missing or malformed buffer. `outs`: the output tensors of the call."""
        if self.eps_ref_out is not None and not ref:
            raise _lib.RttiError(f"{self.what} blend: eps_ref_out needs the reference latents")
        need = self._needed()
        items = list(zip(self.main, need, self.dtypes, self.names))
        if ref:
            items += [(t, nd, dt, name + "_ref") for t, nd, dt, name in zip(self.ref, need, self.dtypes, self.names)]
            if self.has_eps_ref_out:
                items.append((self.eps_ref_out, False, _F16, "eps_ref_out"))
                outs = (*outs, self.eps_ref_out)
        outs = [o for o in outs if o is not None]
        for t, nd, dtype, name in items:
            if t is None:
                if nd:
                    raise _lib.RttiError(f"{self.what} blend: {name} is required")
                continue
            _req(t, dtype, name)
            if not t.is_contiguous() or t.numel() != n:
                raise _lib.RttiError(f"{self.what} blend: {name} must be a contiguous {_DTYPE_NAME[dtype]} tensor of "
                                     f"{n} elements")
            if name.removesuffix("_ref") in self.read_only and any(_overlap(t, o) for o in outs):
                raise _lib.RttiError(f"{self.what} blend: {name} overlaps an output of the call")

    def args(self, ref=False):
        a = [ctypes.c_float(c) for c in self.coeffs] + [_ptr(t) for t in self.main]
        if ref:
            a += [_ptr(t) for t in self.ref] + ([_ptr(self.eps_ref_out)] if self.has_eps_ref_out else [])
        return a


class EulerStep(_Step):
    """The Euler update of one blend call: x' = x + dt eps, with dt = sigma_next - sigma (EulerDiscreteScheduler.dt);
    both trajectories take the same dt."""
    what = "Euler"

    def __init__(self, dt):
        super().__init__((dt,))


class MultistepStep(_Step):
    """The multistep (DDIM / DPM-Solver++) update of one blend call: `coeffs` (schedulers.StepCoeffs: hx, he, cx, cd, cp)
    and the fp32 histories of D = hx x + he eps, [n] each: d_prev (read when cp != 0; may be the same tensor as d_out)
    and d_out (written). d_prev_ref / d_out_ref: the reference-latent trajectory's (gather_blend_step only)."""
    form, what, names, dtypes = "_ms", "multistep", ("d_prev", "d_out"), (torch.float32,) * 2

    def __init__(self, coeffs, d_prev, d_out, d_prev_ref=None, d_out_ref=None):
        super().__init__(coeffs, (d_prev, d_out), (d_prev_ref, d_out_ref))

    def _needed(self):
        return self.coeffs[4] != 0.0, True


class AncestralStep(_Step):
    """The Euler Ancestral update of one blend call: x' = x + dt eps + s_up z, with (dt, s_up) from
    schedulers.EulerAncestralDiscreteScheduler.ancestral_coeffs and z the fp16 noise of the step, [n] elements (read only
    when s_up != 0). z_ref: the reference-latent trajectory's noise (gather_blend_step only); both trajectories take the
    same dt and s_up."""
    form, what, names, dtypes = "_anc", "ancestral", ("z",), (_F16,)

    def __init__(self, dt, s_up, z, z_ref=None):
        super().__init__((dt, s_up), (z,), (z_ref,))

    def _needed(self):
        return (self.coeffs[1] != 0.0,)


class UniPCHistory:
    """The UniPC state of one trajectory: three fp32 [n] buffers, xl (the corrected sample of the last step) and the x0
    predictions of the last two steps, m1 (newest) and m2. A step writes its m over m2 and its corrected sample over
    xl; `rotate()` after the step makes that m the new m1."""

    def __init__(self, n, device):
        self.xl, self.m1, self.m2 = (torch.empty(n, dtype=torch.float32, device=device) for _ in range(3))

    def rotate(self):
        self.m1, self.m2 = self.m2, self.m1


class UniPCStep(_Step):
    """The UniPC update of one blend call: `coeffs` (schedulers.UniPCCoeffs) and the fp32 [n] buffers of one trajectory,
    (xl, m1, m2, m_out, xl_out): xl read when ul != 0, m1 when u1 or v1 != 0, m2 when u2 != 0; m_out (may be m2) and
    xl_out (may be xl) written. `ref`: the same five buffers of the reference-latent trajectory (gather_blend_step only).
    `UniPCStep.of(coeffs, hist, hist_ref)` steps UniPCHistory objects in place (call their rotate() afterwards)."""
    form, what = "_unipc", "UniPC"
    names, dtypes = ("xl", "m1", "m2", "m_out", "xl_out"), (torch.float32,) * 5

    def __init__(self, coeffs, xl, m1, m2, m_out, xl_out, ref=None):
        super().__init__(coeffs, (xl, m1, m2, m_out, xl_out), ref)

    @classmethod
    def of(cls, coeffs, hist, hist_ref=None):
        b = lambda h: (h.xl, h.m1, h.m2, h.m2, h.xl)
        return cls(coeffs, *b(hist), ref=b(hist_ref) if hist_ref is not None else None)

    def _needed(self):
        _, _, _, ul, _, u1, u2, _, _, v1 = self.coeffs
        return ul != 0.0, u1 != 0.0 or v1 != 0.0, u2 != 0.0, True, True


class HeunStep(_Step):
    """The Heun update of one blend call: `coeffs` (cx, ce, cs, cd) from schedulers.HeunDiscreteScheduler.heun_coeffs,
    x' = cx x + ce eps + cs xs + cd ds, with xs / ds the fp16 [n] latents and stepped noise prediction saved at the last
    first stage (xs read when cs != 0, ds when cd != 0; may be None otherwise). xs_ref / ds_ref: the reference-latent
    trajectory's; eps_ref_out: an fp16 [n] tensor that receives that trajectory's stepped prediction, or None
    (gather_blend_step only)."""
    form, what, names, dtypes, coeff_names = "_heun", "Heun", ("xs", "ds"), (_F16,) * 2, ("cx", "ce", "cs", "cd")
    has_eps_ref_out = True

    def __init__(self, coeffs, xs, ds, xs_ref=None, ds_ref=None, eps_ref_out=None):
        super().__init__(coeffs, (xs, ds), (xs_ref, ds_ref), eps_ref_out)

    def _needed(self):
        return self.coeffs[2] != 0.0, self.coeffs[3] != 0.0


class LMSStep(_Step):
    """The LMS update of one blend call: `coeffs` (c0, c1, c2, c3) from schedulers.LMSDiscreteScheduler.lms_coeffs,
    x' = x + c0 eps + c1 d1 + c2 d2 + c3 d3, with d1, d2, d3 the fp16 [n] stepped noise predictions of the trajectory's
    last three steps, newest first (d_k read when c_k != 0; may be None otherwise). d1_ref / d2_ref / d3_ref: the
    reference-latent trajectory's; eps_ref_out: an fp16 [n] tensor that receives that trajectory's stepped prediction,
    or None (gather_blend_step only). The histories are only read; no output may overlap them."""
    form, what, names, dtypes, coeff_names = "_lms", "LMS", ("d1", "d2", "d3"), (_F16,) * 3, ("c0", "c1", "c2", "c3")
    read_only, has_eps_ref_out = names, True

    def __init__(self, coeffs, d1, d2, d3, d1_ref=None, d2_ref=None, d3_ref=None, eps_ref_out=None):
        super().__init__(coeffs, (d1, d2, d3), (d1_ref, d2_ref, d3_ref), eps_ref_out)

    def _needed(self):
        return tuple(c != 0.0 for c in self.coeffs[1:])


class SinglestepStep(_Step):
    """The DPM-Solver++(2S) update of one blend call: `coeffs` (schedulers.SinglestepCoeffs: hx, he, cx, cs, cd, cp),
    D = hx x + he eps, x' = cx x + cd D + cp D_prev + cs xs. d_prev / d_out: the fp32 [n] D buffers as in MultistepStep
    (d_prev read when cp != 0, may be the same tensor as d_out); xs: the fp16 [n] latents that entered the block's first
    step (read when cs != 0; may be None otherwise; only read, so no output may overlap it). d_prev_ref / d_out_ref /
    xs_ref: the reference-latent trajectory's (gather_blend_step only)."""
    form, what, coeff_names = "_ss", "singlestep", ("hx", "he", "cx", "cs", "cd", "cp")
    names, dtypes, read_only = ("d_prev", "d_out", "xs"), (torch.float32, torch.float32, _F16), ("xs",)

    def __init__(self, coeffs, d_prev, d_out, xs, d_prev_ref=None, d_out_ref=None, xs_ref=None):
        super().__init__(coeffs, (d_prev, d_out, xs), (d_prev_ref, d_out_ref, xs_ref))

    def _needed(self):
        return self.coeffs[5] != 0.0, True, self.coeffs[3] != 0.0


def _blend_symbol(base, guidance_rescale, step):
    return f"rtti_{base}{'_rescale' if guidance_rescale != 0.0 else ''}{step.form}"


def region_blend_cfg(eps_uncond, eps_regions, masks, guidance, latents=None, dt_sigma=0.0, guidance_rescale=0.0,
                     step=None):
    """eps = eps_u + g (eps_t - eps_u) with the masked region sums; optionally latents + dt_sigma*eps.
    eps_regions: list of fp16 tensors (region passes in mask order, base-prompt pass last); masks fp32 [N, n].
    guidance_rescale = phi > 0 scales eps by 1 - phi + phi std(eps_t) / std(eps) before it is stored and stepped
    (rtti_region_blend_cfg_rescale*); phi == 0 runs rtti_region_blend_cfg*.
    step: the scheduler update of the latents (required then), one of EulerStep (dt_sigma is shorthand for
    EulerStep(dt_sigma)), MultistepStep, AncestralStep, UniPCStep, HeunStep, LMSStep or SinglestepStep; it selects the
    entry point by its form (rtti_region_blend_cfg_ms, ..._anc, ..._unipc, ..._heun, ..._lms, ..._ss). The buffers of
    the reference trajectory are not used here; eps_ref_out must be None."""
    lib = _lib.load()
    _req(eps_uncond, _F16, "eps_uncond"); _req(masks, torch.float32, "masks")
    n = eps_uncond.numel()
    N = len(eps_regions)
    assert masks.is_contiguous() and masks.numel() == N * n
    for e in eps_regions:
        _req(e, _F16, "eps_region"); assert e.is_contiguous() and e.numel() == n
    if step is None:
        step = EulerStep(dt_sigma)
    elif latents is None:
        raise _lib.RttiError(f"region_blend_cfg: a {type(step).__name__} needs the latents")
    ptrs = (ctypes.c_void_p * N)(*[e.data_ptr() for e in eps_regions])
    eps_out = torch.empty_like(eps_uncond)
    lat_out = torch.empty_like(latents) if latents is not None else None
    step._check(n, False, (eps_out, lat_out))
    symbol = _blend_symbol("region_blend_cfg", guidance_rescale, step)
    phi = [float(guidance_rescale)] if guidance_rescale != 0.0 else []
    rc = getattr(lib, symbol)(_ptr(eps_uncond), ptrs, _ptr(masks), N, n, float(guidance), _ptr(eps_out), _ptr(latents),
                              _ptr(lat_out), *step.args(), *phi, _stream())
    _lib.check(rc, symbol)
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
                      dt_sigma, step_id, guidance_rescale=0.0, step=None):
    """Fused all-gather + blend + CFG + scheduler update over NVLink peer memory (rtti_gather_blend_step*; with
    guidance_rescale > 0 the _rescale entry points, which also rescale the reference-latent pair).
    step: as for region_blend_cfg (None: EulerStep(dt_sigma)), with the reference trajectory's buffers (and, for Heun
    and LMS, optionally eps_ref_out) when latents_ref is given.
    Returns (eps, latents_out, latents_ref_out or None)."""
    lib = _lib.load()
    world = len(peer_slot_ptrs)
    n = latents.numel()
    _req(latents, _F16, "latents"); _req(masks, torch.float32, "masks")
    if step is None:
        step = EulerStep(dt_sigma)
    eps = torch.empty_like(latents)
    lat_out = torch.empty_like(latents)
    ref_out = torch.empty_like(latents_ref) if latents_ref is not None else None
    step._check(n, latents_ref is not None, (eps, lat_out, ref_out))
    slots = (ctypes.c_void_p * world)(*peer_slot_ptrs)
    flags = (ctypes.c_void_p * world)(*peer_flag_ptrs)
    symbol = _blend_symbol("gather_blend_step", guidance_rescale, step)
    phi = [float(guidance_rescale)] if guidance_rescale != 0.0 else []
    rc = getattr(lib, symbol)(slots, flags, world, rank, _int_array(slot_owner), len(slot_owner), n_regions, _ptr(masks),
                              n, float(guidance), _ptr(eps), _ptr(latents), _ptr(lat_out), _ptr(latents_ref),
                              _ptr(ref_out), *step.args(ref=True), int(step_id), *phi, _stream())
    _lib.check(rc, symbol)
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
