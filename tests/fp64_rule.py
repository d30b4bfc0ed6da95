"""The float64 tolerance rule of the kernel tests (test_guidance_fp64.py, test_unet_kernels_fp64.py).

For each op: a float64 reference computed on the GPU from the kernel's own inputs, the PyTorch implementation the
kernel replaces (at the precision the replaced code runs), and the kernel. The kernel passes when
    err_kernel <= k * err_torch + floor,   err = max |x - ref64|
and, with mean=True, the same for the mean |x - ref64| (a max-only check lets a bias spread over the whole output
through). The floor is a few fp32 ulps of the output range, or half an fp16 ulp for fp16 outputs; for the mean it is
scaled by mean|ref| / max|ref|. Every check prints its errors ("[fp64] ..." lines, visible with -s)."""
import math

import torch

EPS32 = torch.finfo(torch.float32).eps
_STEP = 1 << 25   # elements per slice: the SDXL activations are up to 256M elements


def _slices(got, ref):
    a, b = got.reshape(-1), ref.reshape(-1)
    for i in range(0, a.numel(), _STEP):
        yield a[i:i + _STEP].double() - b[i:i + _STEP].double()


def maxerr(got, ref):
    """max |got - ref| in float64."""
    return max(float(d.abs().max()) for d in _slices(got, ref))


def meanerr(got, ref):
    """mean |got - ref| in float64."""
    return sum(float(d.abs().sum()) for d in _slices(got, ref)) / got.numel()


def absmax(t):
    return float(t.abs().max())


def absmean(t):
    return sum(float(s.double().abs().sum()) for s in t.reshape(-1).split(_STEP)) / t.numel()


def half_ulp16(ref):
    """Half an fp16 ulp of max|ref|: the rounding of an fp16 output alone."""
    return 2.0 ** (math.floor(math.log2(absmax(ref))) - 11)


def no_worse(what, got, torch_, ref, k=4.0, floor_ulps=4.0, floor=None, mean=False):
    """Assert the rule for `got` against the PyTorch result(s) `torch_` (a tensor, or a list of tensors of which the
    most accurate counts). Returns (err_kernel, err_torch) of the max."""
    cmps = torch_ if isinstance(torch_, (list, tuple)) else [torch_]
    amax = absmax(ref)
    if floor is None:
        floor = floor_ulps * EPS32 * amax
    e_k = maxerr(got, ref)
    e_ts = [maxerr(t, ref) for t in cmps]
    e_t = min(e_ts)
    line = f"[fp64] {what}: kernel {e_k:.3e}  torch {' / '.join(f'{e:.3e}' for e in e_ts)}"
    if mean:
        m_k = meanerr(got, ref)
        m_ts = [meanerr(t, ref) for t in cmps]
        m_t = min(m_ts)
        floor_m = floor * absmean(ref) / amax if amax > 0 else floor
        line += f"  | mean kernel {m_k:.3e}  torch {' / '.join(f'{e:.3e}' for e in m_ts)}"
    print(line + f"  (ref absmax {amax:.3g})")
    assert math.isfinite(e_k) and e_k <= k * e_t + floor, (
        f"{what}: kernel err {e_k:.3e} > {k:g} x torch err {e_t:.3e} + floor {floor:.3e}")
    if mean:
        assert math.isfinite(m_k) and m_k <= k * m_t + floor_m, (
            f"{what}: kernel mean err {m_k:.3e} > {k:g} x torch mean err {m_t:.3e} + floor {floor_m:.3e}")
    return e_k, e_t
