"""ctypes binding of the C ABI declared in include/rtti_b200.h.

The product path has no CPU or PyTorch fallback: if the library is missing or the device is not
sm_90 every op raises.
"""
import ctypes
import os

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(PKG_DIR, "librtti_b200.so")

RTTI_OK = 0
_ERRORS = {
    -1: "RTTI_ERR_ARG (null pointer / out-of-range argument)",
    -2: "RTTI_ERR_SHAPE (unsupported shape)",
    -3: "RTTI_ERR_ALIGN (pointer or stride alignment)",
    -4: "RTTI_ERR_ARCH (device is not sm_90)",
    -5: "RTTI_ERR_CUDA (CUDA runtime/driver error)",
}

c_void_p, c_int, c_ll, c_float, c_ull = ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong, ctypes.c_float, ctypes.c_ulonglong
P_int = ctypes.POINTER(ctypes.c_int)

# symbol -> (restype, argtypes); must list every symbol include/rtti_b200.h declares
SIGNATURES = {
    "rtti_version": (c_int, []),
    "rtti_arch_ok": (c_int, []),
    "rtti_attn_fwd": (c_int, [c_void_p] * 4 + [c_int] * 5 + [c_ll] * 8 + [c_float, P_int, c_void_p, c_void_p, c_int,
                                                                         c_ull, c_void_p, P_int, c_void_p, c_void_p]),
    "rtti_attn_probs_mean_accum": (c_int, [c_void_p] * 4 + [c_int] * 4 + [c_ll] * 2 + [c_float, c_void_p]),
    "rtti_groupnorm_workspace_elems": (c_ll, [c_int] * 4),
    "rtti_groupnorm_silu_fwd": (c_int, [c_void_p] * 6 + [c_int] * 4 + [c_float, c_int, c_void_p]),
    "rtti_add_bias_f16": (c_int, [c_void_p] * 4 + [c_ll, c_int, c_void_p]),
    "rtti_layernorm_fwd": (c_int, [c_void_p] * 4 + [c_int, c_int, c_float, c_void_p]),
    "rtti_add_bias_layernorm_fwd": (c_int, [c_void_p] * 7 + [c_int, c_int, c_float, c_void_p]),
    "rtti_ff_geglu_fwd": (c_int, [c_void_p] * 4 + [c_ll, c_int, c_int, c_void_p]),
    "rtti_geglu_fwd": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p]),
    "rtti_color_loss_workspace_elems": (c_ll, [c_int, c_ll]),
    "rtti_color_loss_fwd_bwd": (c_int, [c_void_p] * 3 + [c_int, c_ll] + [c_void_p] * 4),
    "rtti_latent_guidance_update": (c_int, [c_void_p] * 3 + [c_float, c_void_p, c_ll, c_void_p]),
    "rtti_bg_inject_blend": (c_int, [c_void_p] * 4 + [c_ll, c_void_p]),
    "rtti_predict_x0": (c_int, [c_void_p, c_void_p, c_float, c_void_p, c_ll, c_void_p]),
    "rtti_gn32_workspace_elems": (c_ll, [c_int] * 4),
    "rtti_gn32_silu_fwd": (c_int, [c_void_p] * 7 + [c_int] * 4 + [c_float, c_int, c_void_p]),
    "rtti_gn32_silu_bwd": (c_int, [c_void_p] * 9 + [c_int] * 4 + [c_int, c_void_p]),
    "rtti_add_bias_f32": (c_int, [c_void_p] * 4 + [c_ll, c_int, c_void_p]),
    "rtti_upsample_phase_interleave": (c_int, [c_void_p] * 3 + [c_int] * 4 + [c_void_p]),
    "rtti_upsample_phase_scatter": (c_int, [c_void_p] * 2 + [c_int] * 4 + [c_void_p]),
    "rtti_gn32_silu_fwd_striped": (c_int, [c_void_p] * 7 + [c_int, c_ll, c_int, c_int, c_float, c_int,
                                           ctypes.POINTER(c_void_p), ctypes.POINTER(c_void_p), c_int, c_int, ctypes.c_uint,
                                           c_void_p]),
    "rtti_gn32_silu_bwd_striped": (c_int, [c_void_p] * 8 + [c_int, c_ll, c_int, c_int, c_int,
                                           ctypes.POINTER(c_void_p), ctypes.POINTER(c_void_p), c_int, c_int, ctypes.c_uint,
                                           c_void_p]),
    "rtti_halo_exchange": (c_int, [c_void_p] * 3 + [c_int, c_ll] + [c_void_p] * 3 + [ctypes.c_uint, c_void_p]),
    "rtti_peer_seq_advance": (c_int, [c_void_p, ctypes.c_uint, c_void_p, ctypes.c_uint, c_void_p]),
    "rtti_peer_push": (c_int, [c_void_p, c_ll, c_int, c_int, ctypes.POINTER(c_void_p), ctypes.POINTER(c_void_p), c_int,
                               c_void_p, ctypes.c_uint, c_void_p]),
    "rtti_peer_wait": (c_int, [c_void_p, ctypes.c_uint, c_void_p]),
    "rtti_kmeans_fit": (c_int, [c_void_p, c_void_p] + [c_int] * 4 + [ctypes.c_double] + [c_void_p] * 5),
    "rtti_kmeans_supported": (c_int, [c_int, c_int]),
}

# The region-blend entry points: one form per fused scheduler update, as (suffix, float count, pointer count of the
# main trajectory, pointer count of the reference trajectory). The update's floats and pointers follow the base
# arguments; gather_blend_step also takes the reference trajectory's pointers and the step id. Each form comes with
# and without the CFG rescale, whose φ is the last argument before the stream.
BLEND_FORMS = (("", 1, 0, 0), ("_ms", 5, 2, 2), ("_anc", 2, 1, 1), ("_unipc", 10, 5, 5), ("_heun", 4, 2, 3),
               ("_lms", 4, 3, 4), ("_ss", 6, 3, 3))
_P_void = ctypes.POINTER(c_void_p)
_BLEND_BASE = [c_void_p, _P_void, c_void_p, c_int, c_ll, c_float, c_void_p, c_void_p, c_void_p]
_GATHER_BASE = [_P_void, _P_void, c_int, c_int, P_int, c_int, c_int, c_void_p, c_ll, c_float] + [c_void_p] * 5
for _sfx, _nf, _np, _nr in BLEND_FORMS:
    for _rescale in ("", "_rescale"):
        _phi = [c_float] if _rescale else []
        SIGNATURES[f"rtti_region_blend_cfg{_rescale}{_sfx}"] = (
            c_int, _BLEND_BASE + [c_float] * _nf + [c_void_p] * _np + _phi + [c_void_p])
        SIGNATURES[f"rtti_gather_blend_step{_rescale}{_sfx}"] = (
            c_int, _GATHER_BASE + [c_float] * _nf + [c_void_p] * (_np + _nr) + [ctypes.c_uint] + _phi + [c_void_p])

_lib = None


class RttiError(RuntimeError):
    pass


def load():
    """Load librtti_b200.so (raises if it has not been built — there is no fallback)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RttiError(
            f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(the rtti_b200 product path has no CPU/PyTorch fallback)")
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is missing
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc, what):
    if rc != RTTI_OK:
        raise RttiError(f"{what} failed: {_ERRORS.get(rc, rc)}")
