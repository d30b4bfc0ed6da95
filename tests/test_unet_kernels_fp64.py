"""The denoising-path kernels against float64 references at the shapes the SD1.5 and SDXL UNets run.

Rule (tests/fp64_rule.py), with K = 2 for every case: the kernel's max and mean |x - ref64| are each at most twice
those of the PyTorch computation the kernel replaces, run at the reference project's precision, plus a floor of half
an fp16 ulp of max|ref| (fp16 outputs) or four fp32 ulps of the output range (fp32 outputs: lse, pbar, accum). The
float64 references are computed on the GPU from the kernel's own fp16 inputs, one (batch entry, head) or one batch
entry at a time (the SDXL 4096^2 score matrix of one head is 134 MB in float64). Every kernel call is made twice and
must give bit-identical results. Each case prints its errors ("[fp64] ..." lines, visible with -s).

Operands are laid out as the UNet hands them over: self-attention q, k, v are column slices of one [B, T, 3C]
projection, cross-attention k, v of one [B, 77, 2C] projection."""
import ctypes
import math
import zlib

import pytest
import torch
import torch.nn.functional as F

from tests.fp64_rule import half_ulp16, no_worse
from tests.test_guidance_fp64 import check_fp16_groupnorm

K = 2.0
F64 = torch.float64
LN2 = math.log(2.0)


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _rule(what, got, cmp, ref, fp16_out=True):
    if fp16_out:
        return no_worse(what, got, cmp, ref, k=K, floor=half_ulp16(ref), mean=True)
    return no_worse(what, got, cmp, ref, k=K, floor_ulps=4.0, mean=True)


# ------------------------------------------------------------------------------------------------ attention helpers
def _h2b(x, H):
    """[T, H*D] of one batch entry -> [H, T, D] (head_to_batch_dim for one entry)."""
    T, C = x.shape
    return x.reshape(T, H, C // H).permute(1, 0, 2)


def _fs_dense(word_pos, font_size, nk):
    """Per-key font-size weight, 1 where unset; for a repeated position the last entry wins."""
    w = torch.ones(nk, dtype=F64, device="cuda")
    for p, s in zip(word_pos.tolist(), font_size.tolist()):
        w[p] = s
    return w


def _fs_unique(word_pos, font_size):
    """(word_pos, font_size) with repeated positions resolved (last wins), for the reference's advanced indexing,
    whose order for repeated indices CUDA leaves unspecified."""
    last = {}
    for p, s in zip(word_pos.tolist(), font_size.tolist()):
        last[p] = s
    pos = sorted(last)
    return (torch.tensor(pos, dtype=torch.long, device="cuda"),
            torch.tensor([last[p] for p in pos], dtype=torch.float32, device="cuda"))


def _ref64(q, k, v, H, scale, src, fs_w=None, fs_mask=0, want_lse=False, want_pm=False):
    """float64 attention of the fp16 operands, one (head, score source) at a time: O [B, nq, C], lse [B, H, nq]
    (log2 domain) and the head mean of P [B, nq, nk]. Font-size entries use the expression of
    unet_oracle.attention_probs: E[:, pos] *= |fs|; P = E / sum(E); P[:, pos] *= sign(fs)."""
    B, nq, C = v.shape[0], q.shape[1], v.shape[2]
    nk, D = k.shape[1], C // H
    o = torch.empty(B, nq, C, dtype=F64, device="cuda")
    lse = torch.empty(B, H, nq, dtype=F64, device="cuda") if want_lse else None
    pm = torch.zeros(B, nq, nk, dtype=F64, device="cuda") if want_pm else None
    for h in range(H):
        cs = slice(h * D, (h + 1) * D)
        for s in sorted(set(src)):
            sc = (q[s, :, cs].double() @ k[s, :, cs].double().T) * scale
            if want_lse:
                ls = torch.logsumexp(sc, -1) / LN2
            e = (sc - sc.amax(-1, keepdim=True)).exp_()
            del sc
            p = e / e.sum(-1, keepdim=True)
            pf = None
            for b in range(B):
                if src[b] != s:
                    continue
                pb = p
                if fs_w is not None and (fs_mask >> b) & 1:
                    if pf is None:
                        ew = e * fs_w.abs()
                        pf = ew / ew.sum(-1, keepdim=True) * fs_w.sign()
                    pb = pf
                o[b, :, cs] = pb @ v[b, :, cs].double()
                if want_lse:
                    lse[b, h] = ls
                if want_pm:
                    pm[b] += pb / H
            del e, p, pf
    return o, lse, pm


def _oracle16(q, k, v, H, scale, src, fs=None, fs_mask=0, want_pm=False):
    """The reference's fp16 path, one batch entry at a time: unet_oracle.attention_probs (font-size branch included),
    torch.bmm(probs, v), and the head mean probs.mean over heads in fp16."""
    from oracle import unet_oracle as uo
    B, nq, C = v.shape[0], q.shape[1], v.shape[2]
    o = torch.empty(B, nq, C, dtype=torch.float16, device="cuda")
    pm = torch.empty(B, nq, k.shape[1], dtype=torch.float16, device="cuda") if want_pm else None
    aw = None
    if fs is not None:
        pos, size = _fs_unique(*fs)
        aw = {"word_pos": pos, "font_size": size}
    for b in range(B):
        s = src[b]
        p = uo.attention_probs(_h2b(q[s], H), _h2b(k[s], H), scale, aw if (fs_mask >> b) & 1 else None)
        o[b] = torch.bmm(p, _h2b(v[b], H)).permute(1, 0, 2).reshape(nq, C)
        if want_pm:
            pm[b] = p.mean(0)
        del p
    return o, pm


def _sdpa16(q, k, v, H, scale, src):
    B, nq, C = v.shape[0], q.shape[1], v.shape[2]
    o = torch.empty(B, nq, C, dtype=torch.float16, device="cuda")
    for b in range(B):
        s = src[b]
        o[b] = F.scaled_dot_product_attention(_h2b(q[s], H)[None], _h2b(k[s], H)[None], _h2b(v[b], H)[None],
                                              scale=scale)[0].permute(1, 0, 2).reshape(nq, C)
    return o


def _twice(fn):
    """Run a kernel call twice; every output must be bit-identical."""
    a, b = fn(), fn()
    for x, y in zip(a, b):
        if x is not None:
            assert torch.equal(x, y), "two runs of the same call differ"
    return a


def _peak(q, k, H, scale, target=30.0):
    """Scale q (float, before the fp16 rounding) so that the scaled scores of entry 0, head 0 span about +-target."""
    D = q.shape[-1] // H
    s = (q[0, :, :D] @ k[0, :, :D].T) * scale
    q *= target / float(s.abs().max())


def _last_key_wins(q, k, H, g):
    """Give every row its largest score at the last key: q += 6 u_h, k[:, -1] = 4 sqrt(D) u_h for a unit vector u_h
    per head. The last key then scores (6 + N(0, 1)) * 4 ~ 24, every other key ~ N(0, 1.25^2)."""
    C = q.shape[-1]
    D = C // H
    u = torch.randn(H, D, device="cuda", generator=g)
    u = (u / u.norm(dim=-1, keepdim=True)).reshape(C)
    q += 6.0 * u
    k[:, -1] = 4.0 * math.sqrt(D) * u


def _operands(B, nq, nk, C, H, g, dist):
    """fp16 (q, k, v) laid out as the UNet produces them. Self-attention (nq == nk): slices of one [B, T, 3C]
    tensor; otherwise q [B, nq, C] and k, v slices of one [B, nk, 2C] tensor."""
    scale = (C // H) ** -0.5
    fused = nq == nk
    if fused:
        qkv = torch.randn(B, nq, 3 * C, device="cuda", generator=g)
        q, k = qkv[..., :C], qkv[..., C:2 * C]
    else:
        q = torch.randn(B, nq, C, device="cuda", generator=g)
        kv = torch.randn(B, nk, 2 * C, device="cuda", generator=g)
        k = kv[..., :C]
    if dist == "peaked":
        _peak(q, k, H, scale)
    elif dist == "last":
        _last_key_wins(q, k, H, g)
    if fused:
        qkv = qkv.half()
        return qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:]
    kv = kv.half()
    return q.half(), kv[..., :C], kv[..., C:]


def _check_attention(tag, q, k, v, H, qk_src=None, fs=None, fs_mask=0, want_lse=False):
    """ops.attention against float64; comparator: the reference's fp16 path, and fp16 SDPA where no font size
    applies (the better of the two counts)."""
    from rtti_b200 import ops
    B, nq = v.shape[0], q.shape[1]
    scale = (v.shape[2] // H) ** -0.5
    src = list(qk_src) if qk_src is not None else list(range(B))
    kw = {}
    if fs is not None:
        kw = dict(word_pos=fs[0], font_size=fs[1], fs_batch_mask=fs_mask)

    def call():
        lse = torch.empty(B, H, nq, dtype=torch.float32, device="cuda") if want_lse else None
        return ops.attention(q, k, v, H, scale=scale, qk_src=qk_src, lse=lse, **kw), lse
    o, lse = _twice(call)
    fs_w = _fs_dense(*fs, k.shape[1]) if fs is not None else None
    o64, lse64, _ = _ref64(q, k, v, H, scale, src, fs_w, fs_mask, want_lse=want_lse)
    cmps = [_oracle16(q, k, v, H, scale, src, fs, fs_mask)[0]]
    if not fs_mask:
        cmps.append(_sdpa16(q, k, v, H, scale, src))
    _rule(tag + " o", o, cmps, o64)
    del cmps, o64
    if want_lse:
        lse32 = torch.empty_like(lse64)
        for h in range(H):
            cs = slice(h * (v.shape[2] // H), (h + 1) * (v.shape[2] // H))
            for b in range(B):
                lse32[b, h] = torch.logsumexp((q[src[b], :, cs].float() @ k[src[b], :, cs].float().T) * scale, -1) / LN2
        _rule(tag + " lse", lse, lse32.float(), lse64, fp16_out=False)
    torch.cuda.empty_cache()
    return lse


# (T, C, heads) of every attention level of SDXL at 1024^2 and SD1.5 at 512^2
SHAPES = {
    "xl64": (4096, 640, 10), "xl32": (1024, 1280, 20),
    "sd64": (4096, 320, 8), "sd32": (1024, 640, 8), "sd16": (256, 1280, 8), "sd8": (64, 1280, 8),
}
# injection sources of a rich step (RegionParallelPlan.injection_sources): SDXL with 5 regions, SD1.5 with 3
RICH = {"xl": [0, 1, 2, 3, 3, 3, 3, 3], "sd": [0, 1, 2, 3, 3, 3]}
# font sizes of pass B (entry 1) on a rich step
FS_PASS_B = ([4, 5, 9, 17], [2.0, -1.0, 0.5, 3.0])


def _fs_tensors(pos, size):
    return (torch.tensor(pos, dtype=torch.int32, device="cuda"), torch.tensor(size, dtype=torch.float32, device="cuda"))


# ------------------------------------------------------------------------------------------------ a. ops.attention
@pytest.mark.gpu
@pytest.mark.parametrize("dist", ["randn", "peaked"])
@pytest.mark.parametrize("batch", ["cfg", "rich"])
@pytest.mark.parametrize("kind", ["self", "cross"])
@pytest.mark.parametrize("shape", list(SHAPES))
def test_attention_at_unet_shapes_vs_fp64(shape, kind, batch, dist):
    """Self- and cross-attention at every UNet level, on the CFG batch of 2 and on the rich-step batch: self-attention
    with the injection sources, cross-attention with font sizes on pass B. `peaked` scales q so that the scaled scores
    span about +-30 (one key dominates each row); `randn` rows are nearly flat."""
    T, C, H = SHAPES[shape]
    src = RICH[shape[:2]] if batch == "rich" else None
    B = len(src) if src else 2
    g = _gen(zlib.crc32(f"{shape} {kind} {batch} {dist}".encode()))
    tag = f"attn {shape} {kind} {batch} {dist}"
    if kind == "self":
        q, k, v = _operands(B, T, T, C, H, g, dist)
        _check_attention(tag, q, k, v, H, qk_src=src)
    else:
        q, k, v = _operands(B, T, 77, C, H, g, dist)
        if batch == "rich":
            _check_attention(tag, q, k, v, H, fs=_fs_tensors(*FS_PASS_B), fs_mask=0b10)
        else:
            _check_attention(tag, q, k, v, H)


@pytest.mark.gpu
@pytest.mark.parametrize("dist", ["randn", "peaked"])
def test_attention_remote_qk_vs_fp64(dist):
    """q and k of one entry (pass D's [1, T, 2C] Q|K slab, received from another rank) applied to the values of four
    entries, at SDXL 64^2."""
    T, C, H = SHAPES["xl64"]
    g = _gen(41 + (dist == "peaked"))
    qk = torch.randn(1, T, 2 * C, device="cuda", generator=g)
    if dist == "peaked":
        _peak(qk[..., :C], qk[..., C:], H, (C // H) ** -0.5)
    qk = qk.half()
    v = torch.randn(4, T, C, device="cuda", generator=g).half()
    _check_attention(f"attn remote qk xl64 {dist}", qk[..., :C], qk[..., C:], v, H, qk_src=[0] * 4)


# (tag, batch, heads, head_dim, n_q, n_k, q distribution): n_k = 80 is the largest single tile; 81 / 129 / 4097 leave
# 17 / 1 / 1 valid keys in the last 64-key tile; "last" puts every row's largest score on the last key, so the
# online rescale happens on the final, partial tile
EDGES = [
    ("nk80", 2, 4, 64, 300, 80, "peaked"),
    ("nk81_last", 2, 4, 64, 300, 81, "last"),
    ("nk129_last", 2, 4, 64, 300, 129, "last"),
    ("nk4097_last", 2, 4, 64, 300, 4097, "last"),
    ("nk4097_peaked", 2, 4, 64, 300, 4097, "peaked"),
    ("nq1_self", 2, 8, 64, 1, 1024, "randn"),
    ("nq1_cross", 2, 8, 64, 1, 77, "peaked"),
    ("nq129_self", 2, 8, 64, 129, 1024, "peaked"),
    ("nq129_cross", 2, 8, 64, 129, 77, "peaked"),
    ("d192_self", 2, 4, 192, 1024, 1024, "peaked"),
    ("d192_cross", 2, 4, 192, 1024, 77, "peaked"),
    ("d72_self", 2, 4, 72, 1024, 1024, "last"),
    ("d72_cross", 2, 4, 72, 1024, 77, "randn"),
    ("b64_self", 64, 2, 64, 256, 256, "peaked"),
    ("b64_cross", 64, 2, 64, 256, 77, "randn"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("tag,B,H,D,nq,nk,dist", EDGES, ids=[e[0] for e in EDGES])
def test_attention_edges_vs_fp64(tag, B, H, D, nq, nk, dist):
    g = _gen(nk * 7 + nq + D + B)
    q, k, v = _operands(B, nq, nk, H * D, H, g, dist)
    src = None
    if B == 64:   # every entry draws its scores from a random entry: the full int8 range of qk_src
        src = torch.randint(0, 64, (64,), generator=torch.Generator().manual_seed(3)).tolist()
    _check_attention(f"attn edge {tag}", q, k, v, H, qk_src=src)


# ------------------------------------------------------------------------------------------------ b/c. capture
def _check_capture(tag, T, C, H, fs=None, fs_mask=0, calls=3, B=2, seed=0):
    """Cross-attention with P-bar capture, as the token-map hook runs it: `calls` successive calls (new q each time,
    the same text keys) accumulate into a prefilled buffer; every entry has its own slot (entry b -> slot B-1-b).
    O of every call and the buffer after every call against float64; comparator: the reference's fp16 path and
    its fp16 probs.mean over heads, summed into the buffer in fp32."""
    from rtti_b200 import ops
    g = _gen(seed)
    scale = (C // H) ** -0.5
    kv = torch.randn(B, 77, 2 * C, device="cuda", generator=g).half()
    k, v = kv[..., :C], kv[..., C:]
    qs = [torch.randn(B, T, C, device="cuda", generator=g) for _ in range(calls)]
    for i in range(1, calls, 2):
        _peak(qs[i], k.float(), H, scale)
    qs = [x.half() for x in qs]
    slots = list(range(B - 1, -1, -1))
    prefill = 0.5 + 0.25 * torch.rand(B, T, 77, device="cuda", generator=g)
    kw = dict(word_pos=fs[0], font_size=fs[1], fs_batch_mask=fs_mask) if fs is not None else {}

    def run():
        pbar = prefill.clone()
        outs = [ops.attention(q, k, v, H, scale=scale, pbar_accum=pbar, cap_slot=slots, **kw) for q in qs]
        return outs + [pbar]
    res = _twice(run)
    # the calls again, checking the buffer after each one
    pbar = prefill.clone()
    p64, p16 = prefill.double(), prefill.clone()
    fs_w = _fs_dense(*fs, 77) if fs is not None else None
    src = list(range(B))
    for i, q in enumerate(qs):
        o = ops.attention(q, k, v, H, scale=scale, pbar_accum=pbar, cap_slot=slots, **kw)
        assert torch.equal(o, res[i])
        o64, _, pm64 = _ref64(q, k, v, H, scale, src, fs_w, fs_mask, want_pm=True)
        o16, pm16 = _oracle16(q, k, v, H, scale, src, fs, fs_mask, want_pm=True)
        cmps = [o16] if fs_mask else [o16, _sdpa16(q, k, v, H, scale, src)]
        _rule(f"{tag} call {i} o", o, cmps, o64)
        p64 = p64 + pm64.flip(0)      # entry b lands in slot B-1-b
        p16 = p16 + pm16.float().flip(0)
        _rule(f"{tag} call {i} pbar", pbar, p16, p64, fp16_out=False)
    assert torch.equal(pbar, res[-1])


@pytest.mark.gpu
@pytest.mark.parametrize("shape", ["xl32", "sd32", "sd16"])
def test_cross_attention_capture_vs_fp64(shape):
    """P-bar capture at SDXL 32^2 (20 heads in one CTA), SD1.5 32^2 (head_dim 80) and SD1.5 16^2 (head_dim 160)."""
    T, C, H = SHAPES[shape]
    _check_capture(f"capture {shape}", T, C, H, seed=len(shape) * 100 + H)


# word_pos / font_size sets: the first and last text key; a repeated position (the last entry, negative, wins);
# zero, negative and 100; all 77 keys set with mixed signs
FONT_SIZES = {
    "ends": ([0, 76], [2.5, -1.7]),
    "repeated": ([5, 9, 5, 5], [3.0, 0.5, 1.5, -2.0]),
    "zero_neg_100": ([3, 10, 40], [0.0, -4.0, 100.0]),
    "all77": (list(range(77)), [((-1) ** i) * (0.2 + 0.05 * i) for i in range(77)]),
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(FONT_SIZES))
def test_font_size_reweighting_and_capture_vs_fp64(case):
    """Font-size re-weighting on entry 1 of a batch of 2 at SD1.5 32^2, output and P-bar capture against float64 of
    the expression in unet_oracle.attention_probs."""
    T, C, H = SHAPES["sd32"]
    _check_capture(f"font size {case}", T, C, H, fs=_fs_tensors(*FONT_SIZES[case]), fs_mask=0b10, seed=7)


@pytest.mark.gpu
def test_capture_at_batch_64_vs_fp64():
    """64 entries, each captured into its own slot (slots 63..0): the int8 limit of the slot table."""
    _check_capture("capture b64", 128, 128, 2, calls=1, B=64, seed=64)


# ------------------------------------------------------------------------------------------------ d. lse, probs mean
@pytest.mark.gpu
@pytest.mark.parametrize("dist", ["randn", "peaked"])
@pytest.mark.parametrize("T,H,D", [(1024, 20, 64), (1024, 8, 80), (4096, 8, 40), (1000, 10, 64)])
def test_lse_and_probs_mean_vs_fp64(T, H, D, dist):
    """The log-sum-exp of ops.attention (against float64 logsumexp / ln 2; comparator torch fp32) and
    ops.attn_probs_mean_accum of entry 1 into a prefilled buffer (against the float64 head mean of softmax;
    comparator the reference's fp16 probs.mean over heads), at the captured self-attention shapes, at T = 4096 with
    head_dim 40 and at a ragged T."""
    from oracle import unet_oracle as uo
    from rtti_b200 import ops
    C = H * D
    g = _gen(T + H + D + (dist == "peaked"))
    q, k, v = _operands(2, T, T, C, H, g, dist)
    scale = D ** -0.5
    tag = f"self T{T} H{H} D{D} {dist}"
    lse = _check_attention(tag, q, k, v, H, want_lse=True)
    prefill = 0.5 + 0.25 * torch.rand(T, T, device="cuda", generator=g)

    def run():
        acc = prefill.clone()
        ops.attn_probs_mean_accum(q[1], k[1], lse[1], acc, H, scale=scale)
        return (acc,)
    (acc,) = _twice(run)
    _, _, pm64 = _ref64(q[1:], k[1:], v[1:], H, scale, [0], want_pm=True)
    p16 = uo.attention_probs(_h2b(q[1], H), _h2b(k[1], H), scale).mean(0)
    _rule(tag + " probs_mean", acc, prefill + p16.float(), prefill.double() + pm64[0], fp16_out=False)


# ------------------------------------------------------------------------------------------------ e. ABI
def test_attn_abi_rejects_shared_or_out_of_range_slots_without_launching():
    """Two entries capturing into one slot would race on pbar_accum's read-modify-write, and a slot outside -1..127
    would not survive the kernel's int8 slot table: both are refused, as is a qk_src entry outside [0, batch). The
    host arrays are checked before the device is queried (fake aligned pointers; nothing is launched)."""
    from rtti_b200 import _lib
    lib = _lib.load()
    V = ctypes.c_void_p
    buf = (ctypes.c_char * 4096)()
    a = (ctypes.addressof(buf) + 15) // 16 * 16
    ARG = -1

    def ints(vals):
        return (ctypes.c_int * len(vals))(*vals)

    def call(B, qk_src=None, slots=None):
        # rtti_attn_fwd(q, k, v, o, batch, heads, head_dim, n_q, n_k, q_bs, q_rs, k_bs, k_rs, v_bs, v_rs, o_bs, o_rs,
        #               scale, qk_src, word_pos, font_size, n_fs, fs_batch_mask, pbar_accum, cap_slot, lse, stream)
        return lib.rtti_attn_fwd(V(a), V(a), V(a), V(a), B, 2, 64, 128, 77, 128 * 128, 128, 77 * 128, 128, 77 * 128,
                                 128, 128 * 128, 128, 0.125, ints(qk_src) if qk_src else None, None, None, 0, 0,
                                 V(a) if slots else None, ints(slots) if slots else None, None, None)
    assert call(2, slots=[0, 0]) == ARG
    assert call(3, slots=[1, -1, 1]) == ARG
    assert call(64, slots=list(range(63, 0, -1)) + [17]) == ARG
    assert call(2, slots=[127, 127]) == ARG
    assert call(2, slots=[128, -1]) == ARG
    assert call(2, slots=[-1, -2]) == ARG
    assert call(3, qk_src=[0, 1, 3]) == ARG
    assert call(3, qk_src=[0, -1, 1]) == ARG


# ------------------------------------------------------------------------------------------------ f. ops.ff_geglu
# (M = B*T, K, N) of every feed-forward of SDXL at 1024^2 (rich batch 8) and SD1.5 at 512^2 (rich batch 6), and
# row counts that leave a ragged last M tile
FF_SHAPES = [(8 * 4096, 640, 2560), (8 * 1024, 1280, 5120), (6 * 4096, 320, 1280), (6 * 1024, 640, 2560),
             (6 * 256, 1280, 5120), (6 * 64, 1280, 5120), (1, 640, 2560), (77, 640, 2560), (129, 640, 2560)]


@pytest.mark.gpu
@pytest.mark.parametrize("gate", ["std", "gate10"])
@pytest.mark.parametrize("bias", [True, False])
@pytest.mark.parametrize("M,Kd,N", FF_SHAPES)
def test_ff_geglu_vs_fp64(M, Kd, N, bias, gate):
    """y = (x Wv^T + bv) * gelu(x Wg^T + bg). Comparator: the reference's fp16 F.linear -> chunk -> a * F.gelu(gate)
    (the FUSED_FF_GEGLU = False route). W ~ N(0, 1/K); `gate10` gives the gate pre-activations a standard deviation
    of 10, where GELU is the identity or zero nearly everywhere."""
    from rtti_b200 import ops
    g = _gen(M + Kd + N + 2 * bias + (gate == "gate10"))
    x = torch.randn(M, Kd, device="cuda", generator=g).half()
    w = torch.randn(2 * N, Kd, device="cuda", generator=g) / math.sqrt(Kd)
    if gate == "gate10":
        w[N:] *= 10.0
    w = w.half()
    b = (0.3 * torch.randn(2 * N, device="cuda", generator=g)).half() if bias else None
    y = _twice(lambda: (ops.ff_geglu(x, w, b),))[0]
    a16, g16 = F.linear(x, w, b).chunk(2, dim=-1)
    y16 = a16 * F.gelu(g16)
    del a16, g16
    y64 = torch.empty(M, N, dtype=F64, device="cuda")
    w64 = w.double()
    b64 = b.double() if bias else None
    for r in range(0, M, 4096):
        a, gt = F.linear(x[r:r + 4096].double(), w64, b64).chunk(2, dim=-1)
        y64[r:r + 4096] = a * F.gelu(gt)
    _rule(f"ff_geglu M{M} K{Kd} N{N} bias={bias} {gate}", y, y16, y64)


# ------------------------------------------------------------------------------------------------ g. LayerNorm
# (C, rows): the UNet's transformer widths with rows = B*T of the levels above, and C = 2048, the kernels' limit
LN_SHAPES = [(320, 6 * 4096), (640, 8 * 4096), (640, 6 * 1024), (1280, 8 * 1024), (1280, 6 * 256), (1280, 6 * 64),
             (2048, 1000)]


def _ln_params(C, g):
    return ((1 + 0.1 * torch.randn(C, device="cuda", generator=g)).half(),
            (0.1 * torch.randn(C, device="cuda", generator=g)).half())


def _ln_ref(x, ga, be, dt):
    return F.layer_norm(x.to(dt), (x.shape[-1],), ga.to(dt), be.to(dt), 1e-5)


def _check_layernorm(C, rows, offset, seed):
    from rtti_b200 import ops
    g = _gen(seed)
    x = (torch.randn(rows, C, device="cuda", generator=g) + offset).half()
    ga, be = _ln_params(C, g)
    y = _twice(lambda: (ops.layernorm(x, ga, be, 1e-5),))[0]
    _rule(f"layernorm C{C} rows{rows} offset={offset:g}", y, _ln_ref(x, ga, be, torch.float16), _ln_ref(x, ga, be, F64))


def _check_add_bias_layernorm(C, rows, offset, bias, seed):
    """h = fp16((a + resid) + bias) bit for bit, written over resid as unet.py calls it; y = LayerNorm(h) against
    float64 of the fp16 h, comparator fp16 F.layer_norm."""
    from rtti_b200 import ops
    g = _gen(seed)
    a = torch.randn(rows, C, device="cuda", generator=g).half()
    resid = (2 * torch.randn(rows, C, device="cuda", generator=g) + offset).half()
    bi = (0.5 * torch.randn(C, device="cuda", generator=g)).half() if bias else None
    ga, be = _ln_params(C, g)

    def run():
        r = resid.clone()
        h, y = ops.add_bias_layernorm(a, r, bi, ga, be, 1e-5)
        assert h.data_ptr() == r.data_ptr()
        return h, y
    h, y = _twice(run)
    want = ((a.float() + resid.float()) + (bi.float() if bias else 0.0)).half()
    assert torch.equal(h, want), f"add_bias_layernorm h: max diff {(h.float() - want.float()).abs().max():.3e}"
    _rule(f"add_bias_layernorm C{C} rows{rows} offset={offset:g} bias={bias}", y, _ln_ref(h, ga, be, torch.float16),
          _ln_ref(h, ga, be, F64))


@pytest.mark.gpu
@pytest.mark.parametrize("C,rows", LN_SHAPES)
def test_layernorm_vs_fp64(C, rows):
    _check_layernorm(C, rows, 0.0, seed=C + rows)


@pytest.mark.gpu
@pytest.mark.parametrize("bias", [True, False])
@pytest.mark.parametrize("C,rows", LN_SHAPES)
def test_add_bias_layernorm_vs_fp64(C, rows, bias):
    _check_add_bias_layernorm(C, rows, 0.0, bias, seed=C + rows + bias)


@pytest.mark.gpu
@pytest.mark.parametrize("C", [640, 2048])
@pytest.mark.parametrize("offset", [0.0, 10.0, 100.0, 1000.0])
def test_layernorm_statistics_hold_for_offset_inputs(C, offset):
    """Rows with mean/std = offset (in x, or in the residual stream). The kernels take the variance in two passes;
    an E[x^2] - E[x]^2 variance in fp32 would lose log10(offset^2) digits here."""
    _check_layernorm(C, 4096, offset, seed=C + int(offset))
    _check_add_bias_layernorm(C, 4096, offset, True, seed=C + int(offset) + 1)


# ------------------------------------------------------------------------------------------------ h. GroupNorm
@pytest.mark.gpu
@pytest.mark.parametrize("HW,C", [(128 * 128, 320), (64 * 64, 640), (32 * 32, 1280),       # SDXL
                                  (64 * 64, 320), (16 * 16, 1280), (8 * 8, 1280)])           # SD1.5 (32^2 x 640 above)
def test_fp16_groupnorm_at_rich_batch_vs_fp64(HW, C):
    """ops.groupnorm_silu at every resnet GroupNorm of the two UNets, on the rich-step batch of 8 with the temb
    chan_bias."""
    check_fp16_groupnorm(8, HW, C, True, 0.0, seed=HW + C, k=K, mean=True)


# ------------------------------------------------------------------------------------------------ i. latent kernels
def _masks16(N, n, g):
    """N region masks over n latents, fp16-representable (the reference holds them in fp16): soft where random,
    exact one-hot on a third of the latents, exact zeros elsewhere in those."""
    m = torch.rand(N, n, device="cuda", generator=g)
    m = m / m.sum(0, keepdim=True)
    hard = torch.rand(n, device="cuda", generator=g) < 1 / 3
    pick = torch.randint(0, N, (n,), device="cuda", generator=g)
    oh = F.one_hot(pick, N).T.float()
    m = torch.where(hard[None], oh, m)
    return m.half().float().contiguous()


@pytest.mark.gpu
@pytest.mark.parametrize("euler", [False, True])
@pytest.mark.parametrize("guidance", [1.0, 8.5])
@pytest.mark.parametrize("N", [2, 5, 16])
@pytest.mark.parametrize("n", [4 * 128 * 128, 4 * 64 * 64])
def test_region_blend_cfg_vs_fp64(n, N, guidance, euler):
    """eps = eps_u + g (eps_t - eps_u) over the region masks (+ latents + dt_sigma * eps). Comparator: the reference's
    fp16 expressions (region_diffusion_sdxl.py: base pass times the last mask, then each region pass added in mask
    order; the Euler update in fp16)."""
    from rtti_b200 import ops
    g = _gen(n + N + int(guidance) + euler)
    eu = torch.randn(n, device="cuda", generator=g).half()
    er = [torch.randn(n, device="cuda", generator=g).half() for _ in range(N)]
    m = _masks16(N, n, g)
    lat = (3 * torch.randn(n, device="cuda", generator=g)).half() if euler else None
    dt = -0.37

    def run():
        r = ops.region_blend_cfg(eu, er, m, guidance, latents=lat, dt_sigma=dt if euler else 0.0)
        return r if euler else (r,)
    res = _twice(run)
    m16 = m.half()
    nu, nt = eu * m16[-1], er[-1] * m16[-1]
    for i in range(N - 1):
        nu = nu + eu * m16[i]
        nt = nt + er[i] * m16[i]
    e16 = nu + guidance * (nt - nu)
    md = m.double()
    u64 = sum(eu.double() * md[i] for i in range(N))
    t64 = sum(er[i].double() * md[i] for i in range(N))
    e64 = u64 + guidance * (t64 - u64)
    tag = f"region_blend_cfg n{n} N{N} g{guidance:g}"
    _rule(tag + " eps", res[0], e16, e64)
    if euler:
        _rule(tag + " latents", res[1], lat + e16 * dt, lat.double() + dt * e64)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [4 * 128 * 128, 4 * 64 * 64, 4 * 64 * 64 + 5])
def test_latent_kernels_vs_fp64(n):
    """predict_x0, bg_inject_blend and latent_guidance_update (one element per thread; n + 5 leaves a ragged last
    block). Comparators: the reference's expressions in its dtypes (fp16 latents with the fp32 alphas_cumprod scalar;
    fp16 masks; the guidance step in fp32 rounded to fp16)."""
    from rtti_b200 import ops
    g = _gen(n)
    x = (2 * torch.randn(n, device="cuda", generator=g)).half()
    e = torch.randn(n, device="cuda", generator=g).half()
    for alpha in (0.05, 0.9):
        got = _twice(lambda: (ops.predict_x0(x, e, alpha),))[0]
        a32 = torch.tensor(alpha, dtype=torch.float32, device="cuda")
        want16 = (x - e * torch.sqrt(1 - a32)) / torch.sqrt(a32)
        a = float(a32)
        want64 = (x.double() - e.double() * math.sqrt(1 - a)) / math.sqrt(a)
        _rule(f"predict_x0 n{n} alpha{alpha:g}", got, want16, want64)
    m = _masks16(2, n, g)[0]
    got = _twice(lambda: (ops.bg_inject_blend(x, e, m),))[0]
    m16 = m.half()
    _rule(f"bg_inject_blend n{n}", got, e * m16 + x * (1 - m16), e.double() * m.double() + x.double() * (1 - m.double()))
    grad = 0.05 * torch.randn(n, device="cuda", generator=g)
    att = torch.rand(n, device="cuda", generator=g)
    att[: n // 4] = 0.0
    got = _twice(lambda: (ops.latent_guidance_update(x, grad, att, 3.0),))[0]
    _rule(f"latent_guidance_update n{n}", got, (x.float() - grad * 3.0 * att).half(),
          x.double() - grad.double() * 3.0 * att.double())
