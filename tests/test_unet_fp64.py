"""The product UNet as a whole against float64, at the full SD1.5 and SDXL configurations.

The kernels each have a float64 test at the UNet's shapes (test_unet_kernels_fp64.py); this file holds the way they are
put together to the same rule (tests/fp64_rule.py, K = 2): folded biases, fused residual + LayerNorm chains, the
concatenated Q/K/V weights, the channels-last views, the x2 upsample, feature and self-attention injection, font sizes
and the token-map capture. Three results per case, all on the GPU, from the same fp16 weights and inputs:
  * the product UNet2DConditionModel (synthetic weights, every 1-D parameter perturbed so that norm gains and biases
    are not 1 and 0);
  * the comparator: oracle.unet_oracle.unet_forward on the product's own fp16 state_dict(), the fp16 PyTorch
    computation the kernels replace;
  * the reference: the same unet_forward on that state dict upcast to float64, with the fp16 inputs upcast, run one
    batch entry at a time under Float64Guard, which fails on any op producing a floating-point result other than
    float64.
Every output must satisfy err_product <= 2 err_fp16 + half an fp16 ulp of max|ref| (max and mean); the captured token
maps are fp32 outputs (floor 4 fp32 ulps). Every product call is made twice and must give bit-identical results, with
cuDNN held to deterministic algorithms. Each case prints its errors ("[fp64] ..." lines) and its wall time and peak
memory ("[case] ..." lines), visible with -s.

Cases: the plain CFG batch at square latents with token maps; the plain batch at non-square latents (a swapped H/W in a
channels-last view gives identical results when H == W); the rich-text step batch A, B, C, D, E1, E2 as one product
call against the passes in sequence; the cross K/V cache against no cache."""
import contextlib
import time

import pytest
import torch
from torch.utils._python_dispatch import TorchDispatchMode
from torch.utils._pytree import tree_leaves

from oracle import sampler_oracle as sam, unet_oracle as uo
from tests.fp64_rule import half_ulp16, no_worse

K = 2.0
F64 = torch.float64
T_STEPS = (981, 41)
N_REGIONS = 3
FS_POS, FS_SIZE = [4, 5, 9, 17], [2.0, -1.0, 0.5, 3.0]   # font sizes of pass B, one of them negative
GB = 2 ** 30
BOS_LOGIT_STD = 3.0  # standard deviation of the cross-attention logits of the first context token (see _inputs)


class Float64Guard(TorchDispatchMode):
    """Fails on any op that produces a floating-point tensor other than float64, outside `allow_lower()`."""

    def __init__(self):
        super().__init__()
        self.exempt = False

    @contextlib.contextmanager
    def allow_lower(self):
        prev, self.exempt = self.exempt, True
        try:
            yield
        finally:
            self.exempt = prev

    def __torch_dispatch__(self, func, types, args=(), kwargs=None):
        out = func(*args, **(kwargs or {}))
        if not self.exempt:
            for t in tree_leaves(out):
                if isinstance(t, torch.Tensor) and t.is_floating_point() and t.dtype != F64:
                    raise AssertionError(f"float64 reference: {func} returned {t.dtype}")
        return out


class _Store32(sam.SelfAttnStore):
    """Pass D's stores for the float64 reference, with the self-attention probabilities kept in float32 (exempt from
    the guard): SDXL's would take 23.5 GB in float64. Their 2^-24 relative rounding is far below the fp16 floor of
    the rule (2^-12 relative)."""

    def __init__(self, guard):
        super().__init__(True)
        self.guard = guard

    def post_attn(self, name, probs_avg, probs):
        if "attn2" not in name:
            with self.guard.allow_lower():
                self.store[name] = probs.float()


class _Replace64(sam.ReplaceControl):
    """ReplaceControl that upcasts the float32 probabilities of _Store32 at use."""

    def pre_attn(self, name):
        p, w = super().pre_attn(name)
        return (None if p is None else p.to(F64)), w


class _RowCapture(sam.TokenMapCapture):
    """TokenMapCapture for a batch of one: that entry stands in for the conditional row 1 of the CFG batch."""

    def post_attn(self, name, probs_avg, probs):
        super().post_attn(name, probs_avg.expand(2, -1, -1), probs)


# ------------------------------------------------------------------------------------------------ helpers
@pytest.fixture
def deterministic_cudnn():
    prev = torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
    try:
        yield
    finally:
        torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = prev


@contextlib.contextmanager
def _case(what, need_gb):
    """Skips when the GPU has less than `need_gb` free; prints the case's wall time and peak memory."""
    torch.cuda.empty_cache()   # blocks cached from the previous case are free for this one
    free, _ = torch.cuda.mem_get_info()
    if free < need_gb * GB:
        pytest.skip(f"{what}: needs {need_gb} GB of free GPU memory, {free / GB:.1f} GB free")
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    yield
    torch.cuda.synchronize()
    print(f"[case] {what}: wall {time.perf_counter() - t0:.1f} s, peak allocated "
          f"{torch.cuda.max_memory_allocated() / GB:.1f} GB, peak reserved {torch.cuda.max_memory_reserved() / GB:.1f} GB")


def _configs(kind):
    from rtti_b200.unet import UNetConfig
    if kind == "sdxl":
        return UNetConfig.sdxl(), uo.sdxl_config()
    return UNetConfig.sd15(), uo.sd15_config()


def _product(cfg, seed):
    """Synthetic weights made on the GPU, every 1-D parameter perturbed by 0.1 randn (GroupNorm and LayerNorm gains
    and biases are not 1 and 0, conv biases reach the kernels folded into chan_bias), then finalize."""
    from rtti_b200.unet import UNet2DConditionModel
    with torch.device("cuda"):
        unet = UNet2DConditionModel(cfg)
    unet.init_synthetic(seed)
    g = torch.Generator(device="cuda").manual_seed(seed + 100)
    for p in unet.parameters():
        if p.dim() == 1:
            p.data.add_(0.1 * torch.randn(p.shape, generator=g, device="cuda"))
    return unet.finalize("cuda")


def _inputs(ocfg, B, H, W, n_ctx, seed):
    """fp16 latents [B, 4, H, W], context [n_ctx, 77, D] with a dominant first token row, and SDXL's pooled text
    embeddings [n_ctx, P] and time ids [1, 6].

    Like CLIP's BOS row, the first row stands out, so that cross-attention rows are peaked. With N(0, 1/fan_in)
    weights a context row of norm r gives logits q.k/sqrt(d) of standard deviation about r/sqrt(D): the randn rows
    (norm ~sqrt(D)) give 1, which leaves rows nearly flat whatever r the first row has up to a few sqrt(D) (CLIP's
    BOS norm of ~28 is about sqrt(768)). The first row gets BOS_LOGIT_STD * sqrt(D): its logits span about +-13 against
    +-4 for the others, and the largest probability of a row averages 0.15 instead of 0.09. Larger scales (5, 8) make
    the UNet ill-conditioned: a row whose first logit sits at the tipping point amplifies upstream rounding through
    the large first value row, so the single largest map error of the product and of the fp16 comparator become
    draws from a heavy tail (ratios up to 2.6 and 6.4 at mean ratios below 0.95)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(B, 4, H, W, device="cuda", generator=g).half()
    D = ocfg.cross_attention_dim
    ctx = torch.randn(n_ctx, 77, D, device="cuda", generator=g)
    ctx[:, 0] *= BOS_LOGIT_STD * D ** 0.5 / ctx[:, 0].norm(dim=-1, keepdim=True)
    te = tid = None
    if ocfg.addition_embed_type:
        pooled = ocfg.projection_class_embeddings_input_dim - 6 * ocfg.addition_time_embed_dim
        te = torch.randn(n_ctx, pooled, device="cuda", generator=g).half()
        tid = torch.tensor([[8 * H, 8 * W, 0, 0, 8 * H, 8 * W]], dtype=torch.float16, device="cuda")
    return x, ctx.half(), te, tid


def _added(te, tid, rows, dtype=torch.float16):
    if te is None:
        return None
    return {"text_embeds": te[rows].to(dtype), "time_ids": tid.to(dtype)}


def _twice(fn):
    """Run a product call twice; the outputs (a tensor and a dict of tensors) must be bit-identical."""
    (ya, ma), (yb, mb) = fn(), fn()
    assert torch.equal(ya, yb), "two runs of the same UNet call differ"
    assert sorted(ma) == sorted(mb) and all(torch.equal(ma[k], mb[k]) for k in ma), "two runs' token maps differ"
    return ya, ma


def _rule(what, got, cmp, ref):
    return no_worse(what, got, cmp, ref, k=K, floor=half_ulp16(ref), mean=True)


def _rule32(what, got, cmp, ref):
    return no_worse(what, got, cmp, ref, k=K, floor_ulps=4.0, mean=True)


def _to64(sd16):
    return {k: v.to(F64) for k, v in sd16.items()}


# ------------------------------------------------------------------------------------------------ 1/2. plain CFG batch
def _plain(kind, H, W, t, maps, need_gb):
    from rtti_b200.attention_utils import CrossAttentionLayers, CrossAttentionLayers_XL, SelfAttentionLayers
    from rtti_b200.unet import RegionControl, TokenMapAccumulator
    xl = kind == "sdxl"
    pcfg, ocfg = _configs(kind)
    what = f"{kind} plain {H}x{W} t{t}"
    with _case(what, need_gb):
        x, ctx, te, tid = _inputs(ocfg, 2, H, W, 2, seed=H * 1000 + W + t)
        tid2 = tid.expand(2, -1) if xl else None
        unet = _product(pcfg, seed=7 if xl else 5)

        def run():
            cap = None
            if maps:
                cap = TokenMapAccumulator(CrossAttentionLayers_XL if xl else CrossAttentionLayers,
                                          self_layers=None if xl else SelfAttentionLayers, start_after=0,
                                          sd_overwrite_bug=not xl, self_resolutions=None)
            y = unet(x, t, ctx, _added(te, tid2, slice(0, 2)), RegionControl(capture=cap, capture_row=1))["sample"]
            return y, ({**cap.selfattn_maps, **cap.crossattn_maps} if maps else {})
        with torch.no_grad():
            y, pmaps = _twice(run)
            sd16 = unet.state_dict()
            cap16 = sam.TokenMapCapture(xl, start_after=0) if maps else None
            y16 = uo.unet_forward(sd16, ocfg, x, t, ctx, _added(te, tid2, slice(0, 2)), cap16)
            sd64 = _to64(sd16)
            del unet, sd16
            torch.cuda.empty_cache()
            y64 = torch.empty(y.shape, dtype=F64, device="cuda")
            cap64 = _RowCapture(xl, start_after=0) if maps else None
            for b in range(2):
                xb, cb, ab = x[b:b + 1].to(F64), ctx[b:b + 1].to(F64), _added(te, tid, slice(b, b + 1), F64)
                with Float64Guard():
                    y64[b:b + 1] = uo.unet_forward(sd64, ocfg, xb, t, cb, ab, cap64 if b == 1 else None)
            del sd64
        _rule(f"{what} eps", y, y16, y64)
        if maps:
            m16 = {**cap16.selfattn_maps, **cap16.crossattn_maps}
            m64 = {**cap64.selfattn_maps, **cap64.crossattn_maps}
            assert sorted(pmaps) == sorted(m16) == sorted(m64)
            for name in sorted(pmaps):
                _rule32(f"{what} map {name}", pmaps[name], m16[name], m64[name])


@pytest.mark.gpu
@pytest.mark.parametrize("t", T_STEPS)
@pytest.mark.parametrize("kind", ["sd15", "sdxl"])
def test_unet_cfg_batch_with_token_maps_vs_fp64(deterministic_cudnn, kind, t):
    """[uncond, cond] at SD1.5 64^2 / SDXL 128^2; every self and cross map the capture keeps (from the first call on)
    against the maps the oracle's TokenMapCapture takes."""
    S = 128 if kind == "sdxl" else 64
    _plain(kind, S, S, t, maps=True, need_gb=40 if kind == "sdxl" else 16)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["sd15", "sdxl"])
def test_unet_non_square_latents_vs_fp64(deterministic_cudnn, kind):
    """SD1.5 at 64x96 and SDXL at 96x168 (768x1344 images: levels of 4032 and 1008 tokens), H != W at every level."""
    H, W = (96, 168) if kind == "sdxl" else (64, 96)
    _plain(kind, H, W, T_STEPS[0], maps=False, need_gb=40 if kind == "sdxl" else 16)


# ------------------------------------------------------------------------------------------------ 3. rich-text step
def _rich_batch(ocfg, S, seed):
    """Inputs of one rich-text step with injection: passes A, B (font sizes), C, D (reference latents) and E1, E2."""
    from rtti_b200.region_parallel import RegionParallelPlan
    N = N_REGIONS
    passes = [dict(kind="A", ctx=0, ref=False), dict(kind="B", ctx=N, ref=False),
              dict(kind="C", ctx=0, ref=True), dict(kind="D", ctx=N, ref=True)]
    passes += [dict(kind="E", ctx=j + 1, ref=False, region=j) for j in range(N - 1)]
    plan = RegionParallelPlan(passes, True)
    local = plan.local_passes(True)
    assert local == list(range(len(passes)))
    src = plan.injection_sources(local)
    lat, ctx, te, tid = _inputs(ocfg, 2, S, S, N + 1, seed)   # lat[0]: latents, lat[1]: reference latents
    return passes, src, lat, ctx, te, tid


def _oracle_rich(sd, ocfg, passes, lat, t, ctx, te, tid, dtype, guard=None):
    """The reference's sequential pass order (sampler_oracle.rich_text_loop): A, B with FontSizeControl, C, D with
    SelfAttnStore, then each E with ReplaceControl on D's store."""
    fs = {"word_pos": torch.tensor(FS_POS, device="cuda"),
          "font_size": torch.tensor(FS_SIZE, dtype=torch.float32 if dtype == torch.float16 else F64, device="cuda")}
    store = sam.SelfAttnStore(True) if guard is None else _Store32(guard)
    out = []
    for p in passes:
        if p["kind"] == "B":
            ctrl = sam.FontSizeControl(fs)
        elif p["kind"] == "D":
            ctrl = store
        elif p["kind"] == "E":
            ctrl = (sam.ReplaceControl if guard is None else _Replace64)(True, store.store)
        else:
            ctrl = None
        r = p["ctx"]
        x = (lat[1:2] if p["ref"] else lat[:1]).to(dtype)
        c, a = ctx[r:r + 1].to(dtype), _added(te, tid, slice(r, r + 1), dtype)
        with guard if guard is not None else contextlib.nullcontext():
            out.append(uo.unet_forward(sd, ocfg, x, t, c, a, ctrl))
    return out


def _product_rich_ctrl(src, kv_cache=None):
    from rtti_b200.unet import RegionControl
    return RegionControl(qk_src=src, feature_src=src, feature_idx=torch.as_tensor(src, device="cuda"),
                         word_pos=torch.tensor(FS_POS, dtype=torch.int32, device="cuda"),
                         font_size=torch.tensor(FS_SIZE, dtype=torch.float32, device="cuda"), fs_batch_mask=0b10,
                         kv_cache=kv_cache)


def _product_rich_inputs(passes, lat, ctx, te, tid):
    rows = [p["ctx"] for p in passes]
    x = torch.cat([lat[1:2] if p["ref"] else lat[:1] for p in passes])
    return x, ctx[rows], _added(te, tid, rows)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["sd15", "sdxl"])
def test_unet_rich_text_step_batch_vs_fp64(deterministic_cudnn, kind):
    """One product call on the batch of a rich-text injection step (qk_src = feature_src from
    RegionParallelPlan.injection_sources, font sizes on pass B only) against the oracle's passes in sequence; the
    reference latents differ from the latents, so a pass reading the wrong entry shows."""
    xl = kind == "sdxl"
    pcfg, ocfg = _configs(kind)
    S = 128 if xl else 64
    t = T_STEPS[0]
    what = f"{kind} rich step {S}x{S} t{t}"
    with _case(what, 48 if xl else 20):
        passes, src, lat, ctx, te, tid = _rich_batch(ocfg, S, seed=S + 3)
        unet = _product(pcfg, seed=7 if xl else 5)
        x, c, added = _product_rich_inputs(passes, lat, ctx, te, tid)
        with torch.no_grad():
            y, _ = _twice(lambda: (unet(x, t, c, added, _product_rich_ctrl(src))["sample"], {}))
            sd16 = unet.state_dict()
            y16 = _oracle_rich(sd16, ocfg, passes, lat, t, ctx, te, tid, torch.float16)
            sd64 = _to64(sd16)
            del unet, sd16
            torch.cuda.empty_cache()
            y64 = _oracle_rich(sd64, ocfg, passes, lat, t, ctx, te, tid, F64, guard=Float64Guard())
            del sd64
        for i, p in enumerate(passes):
            _rule(f"{what} pass {p['kind']}{p.get('region', '')}", y[i:i + 1], y16[i], y64[i])


# ------------------------------------------------------------------------------------------------ 4. cross K/V cache
@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["sd15", "sdxl"])
def test_unet_cross_kv_cache_is_bit_exact(deterministic_cudnn, kind):
    """One RegionControl with a CrossKVCache, called twice with the same context (the second call reads every cross
    K/V from the cache), equals a call without the cache bit for bit, on the rich-text step batch."""
    from rtti_b200.unet import CrossKVCache
    xl = kind == "sdxl"
    pcfg, ocfg = _configs(kind)
    S = 128 if xl else 64
    with _case(f"{kind} cross K/V cache", 16 if xl else 8):
        passes, src, lat, ctx, te, tid = _rich_batch(ocfg, S, seed=S + 5)
        unet = _product(pcfg, seed=9)
        x, c, added = _product_rich_inputs(passes, lat, ctx, te, tid)
        with torch.no_grad():
            want = unet(x, 501, c, added, _product_rich_ctrl(src))["sample"]
            ctrl = _product_rich_ctrl(src, CrossKVCache())
            first = unet(x, 501, c, added, ctrl)["sample"]
            n_kv = len(ctrl.kv_cache.kv)
            second = unet(x, 501, c, added, ctrl)["sample"]
        assert n_kv == sum(len(tr.transformer_blocks) for blk in [*unet.down_blocks, unet.mid_block, *unet.up_blocks]
                           for tr in (getattr(blk, "attentions", None) or []))
        assert len(ctrl.kv_cache.kv) == n_kv
        assert torch.equal(first, want), "the call that fills the cache differs from a call without it"
        assert torch.equal(second, want), "the call that reads the cache differs from a call without it"


# ------------------------------------------------------------------------------------------------ guard (CPU)
@pytest.mark.parametrize("name", ["tiny_sd", "tiny_xl"])
def test_oracle_float64_reference_stays_float64(name):
    """The float64 reference of this file runs without a single lower-precision op: the tiny oracle configs in float64
    under Float64Guard, with font sizes (pass B), the stores of pass D (float32 probabilities, exempt) and injection
    (pass E). The guard fails on a float32 result: font sizes handed over in float32."""
    cfg = uo.tiny_sd_config() if name == "tiny_sd" else uo.tiny_xl_config()
    sd = uo.make_state_dict(cfg, 3, dtype=F64)
    g = torch.Generator().manual_seed(4)
    x = torch.randn(2, 4, 16, 16, generator=g, dtype=F64)            # latents, reference latents
    ctx = torch.randn(2, 77, cfg.cross_attention_dim, generator=g, dtype=F64)
    added = None
    if cfg.addition_embed_type:
        pooled = cfg.projection_class_embeddings_input_dim - 6 * cfg.addition_time_embed_dim
        added = {"text_embeds": torch.randn(1, pooled, generator=g, dtype=F64),
                 "time_ids": torch.tensor([[128.0, 128.0, 0.0, 0.0, 128.0, 128.0]], dtype=F64)}
    pos = torch.tensor(FS_POS)
    guard = Float64Guard()
    store = _Store32(guard)
    with torch.no_grad():
        with guard:
            outs = [uo.unet_forward(sd, cfg, x[:1], 981, ctx[1:], added,
                                    sam.FontSizeControl({"word_pos": pos, "font_size": torch.tensor(FS_SIZE, dtype=F64)})),
                    uo.unet_forward(sd, cfg, x[1:], 981, ctx[1:], added, store),
                    uo.unet_forward(sd, cfg, x[:1], 981, ctx[:1], added, _Replace64(True, store.store))]
        assert all(o.dtype == F64 and torch.isfinite(o).all() for o in outs)
        probs = [v for k, v in store.store.items() if k.endswith("attn1")]
        assert probs and all(p.dtype == torch.float32 for p in probs)
        assert store.store["up_blocks.1.resnets.1"].dtype == F64
        with pytest.raises(AssertionError, match="float32"), guard:
            uo.unet_forward(sd, cfg, x[:1], 981, ctx[1:], added,
                            sam.FontSizeControl({"word_pos": pos, "font_size": torch.tensor(FS_SIZE)}))
