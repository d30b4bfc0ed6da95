"""LoRA checkpoints (rtti_b200/lora.py) merged into the UNet and CLIP text-encoder weights.

CPU: the name mapping of both kohya UNet naming schemes, of diffusers' attention-processor format and of the CLIP
encoders is a bijection onto the targets (full SD1.5 / SDXL configurations on the meta device); malformed files raise
ValueError; the merge equals W0 + s (alpha / r) B A, a conv LoRA equals its down conv then its up conv; re-merging and
unloading give exact bits; the tiny UNets with a merged LoRA match the oracle run unmerged.
GPU: the full-size UNets with a merged rank-16 LoRA against a float64 unmerged evaluation (the rule of
test_unet_fp64.py); both samplers with a LoRA loaded against a model built from pre-merged weights, bit for bit, also
after a second call at another scale."""
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import unet_oracle as uo
from rtti_b200 import lora
from rtti_b200.unet import UNet2DConditionModel, UNetConfig
from tests import lora_synth as ls
from tests import synth

ALPHA = 3.0   # != rank: the alpha / rank factor is exercised
_SGM = re.compile(r"lora_unet_(input|middle|output)_block")


def _meta_unet(cfg):
    with torch.device("meta"):
        return UNet2DConditionModel(cfg)


def _cpu_unet(ocfg, seed, dtype=torch.float32):
    unet = UNet2DConditionModel(UNetConfig.from_dict(ocfg.__dict__))
    unet.load_state_dict(uo.make_state_dict(ocfg, seed))
    return unet.to(dtype).requires_grad_(False)


def _sgm_to_diffusers(stem, cfg):
    """The original UNet's block names -> ours, by the formulas of the SDXL block layout (independent of lora.py)."""
    L = cfg.layers_per_block
    res = {"in_layers_2": "conv1", "emb_layers_1": "time_emb_proj", "out_layers_3": "conv2", "skip_connection": "conv_shortcut"}
    m = re.match(r"lora_unet_input_blocks_(\d+)_(\d+)_(.+)$", stem)
    if m:
        n, j, rest = int(m.group(1)), int(m.group(2)), m.group(3)
        b, k = (n - 1) // (L + 1), (n - 1) % (L + 1)
        if k == L:
            assert j == 0 and rest == "op"
            return f"down_blocks.{b}.downsamplers.0.conv"
        return f"down_blocks.{b}.resnets.{k}.{res[rest]}" if j == 0 else \
            f"down_blocks.{b}.attentions.{k}.{rest.replace('_', '.')}"
    m = re.match(r"lora_unet_middle_block_(\d)_(.+)$", stem)
    if m:
        j, rest = int(m.group(1)), m.group(2)
        return (f"mid_block.resnets.{j // 2}.{res[rest]}" if j != 1 else f"mid_block.attentions.0.{rest.replace('_', '.')}")
    m = re.match(r"lora_unet_output_blocks_(\d+)_(\d)_(.+)$", stem)
    n, j, rest = int(m.group(1)), int(m.group(2)), m.group(3)
    b, k = n // (L + 1), n % (L + 1)
    attn = cfg.up_block_types[b] == "CrossAttnUpBlock2D"
    if j == 0:
        return f"up_blocks.{b}.resnets.{k}.{res[rest]}"
    if j == 1 and attn:
        return f"up_blocks.{b}.attentions.{k}.{rest.replace('_', '.')}"
    assert k == L and j == (2 if attn else 1) and rest == "conv"
    return f"up_blocks.{b}.upsamplers.0.conv"


def _unmangle(name):
    """Module names with `_` in a component, restored from the `.`-to-`_` mangling of the test's own formula."""
    for a in ("transformer.blocks", "to.q", "to.k", "to.v", "to.out", "proj.in", "proj.out"):
        name = name.replace(a, a.replace(".", "_"))
    return name


def _targets_from_oracle(ocfg):
    """Every 2-D / 4-D weight of the down, mid and up blocks in the oracle's parameter inventory."""
    return {k[:-len(".weight")] for k, s in uo.param_shapes(ocfg).items()
            if k.endswith(".weight") and len(s) >= 2 and k.split(".")[0] in ("down_blocks", "mid_block", "up_blocks")}


# ---------------------------------------------------------------------------------------------------- CPU: names
@pytest.mark.parametrize("kind", ["sd15", "sdxl"])
def test_kohya_names_are_a_bijection_onto_the_targets(kind):
    cfg, ocfg = (UNetConfig.sdxl(), uo.sdxl_config()) if kind == "sdxl" else (UNetConfig.sd15(), uo.sd15_config())
    unet = _meta_unet(cfg)
    targets = lora.unet_targets(unet)
    assert set(targets) == _targets_from_oracle(ocfg)
    names = lora.kohya_names(unet)
    diffusers_keys = {k: v for k, v in names.items() if not _SGM.match(k)}
    sgm_keys = {k: v for k, v in names.items() if k not in diffusers_keys}
    for keys in (diffusers_keys, sgm_keys):
        assert len(keys) == len(targets)
        assert sorted(n for _, n in keys.values()) == sorted(targets)   # onto, and no target named twice
    for k, (comp, n) in diffusers_keys.items():
        assert comp == "unet" and k == ls.diffusers_stem(n)
    for k, (comp, n) in sgm_keys.items():
        m = _sgm_to_diffusers(k, cfg)
        assert _unmangle(m) == n, (k, m, n)
    if kind == "sdxl":   # spot checks of kohya's SDXL names
        assert names["lora_unet_input_blocks_4_1_transformer_blocks_0_attn1_to_q"][1] == \
            "down_blocks.1.attentions.0.transformer_blocks.0.attn1.to_q"
        assert names["lora_unet_output_blocks_2_2_conv"][1] == "up_blocks.0.upsamplers.0.conv"
        assert names["lora_unet_input_blocks_3_0_op"][1] == "down_blocks.0.downsamplers.0.conv"
        assert names["lora_unet_middle_block_1_proj_in"][1] == "mid_block.attentions.0.proj_in"
        assert names["lora_unet_output_blocks_8_0_skip_connection"][1] == "up_blocks.2.resnets.2.conv_shortcut"
    else:
        assert names["lora_unet_output_blocks_2_1_conv"][1] == "up_blocks.0.upsamplers.0.conv"


@pytest.mark.parametrize("kind", ["sd15", "sdxl"])
def test_every_target_merges_from_both_kohya_schemes_and_diffusers_format(kind):
    """A rank-1 LoRA on every target loads (meta device) through each naming; diffusers' format covers exactly the
    attention projections."""
    cfg = UNetConfig.sdxl() if kind == "sdxl" else UNetConfig.sd15()
    unet = _meta_unet(cfg)
    targets = lora.unet_targets(unet)
    fac = ls.lora_factors(targets, 1, 0)
    names = lora.kohya_names(unet)
    for sgm in (False, True):
        stems = {n: k for k, (_, n) in names.items() if bool(_SGM.match(k)) == sgm}
        m = lora.MergedLora(ls.kohya_dict(fac, stems, ALPHA), unet)
        assert sorted(e[0] for e in m.entries) == sorted("unet:" + n for n in targets)
    attn = [n for n in targets if re.search(r"\.attn[12]\.(to_q|to_k|to_v|to_out\.0)$", n)]
    sd = {}
    for n in attn:
        path, proj = re.match(r"(.+)\.(to_q|to_k|to_v|to_out)", n).groups()
        down, up = fac[n]
        sd[f"unet.{path}.processor.{proj}_lora.down.weight"] = down
        sd[f"unet.{path}.processor.{proj}_lora.up.weight"] = up
    m = lora.MergedLora(sd, unet)
    assert sorted(e[0] for e in m.entries) == sorted("unet:" + n for n in attn)
    assert all(e[5] == 1.0 for e in m.entries)   # no alpha in this format: alpha = rank


def _tiny_clip(tmp_path):
    from tests.test_loading import _tiny_clip_dir
    from rtti_b200 import loading
    _tiny_clip_dir(str(tmp_path))
    return loading.ClipTextEncoders(str(tmp_path), "cpu", xl=True)


def test_clip_names_are_a_bijection(tmp_path):
    enc = _tiny_clip(tmp_path)
    unet = _meta_unet(UNetConfig.sd15())
    want = {f"text_model.encoder.layers.{i}.{p}" for i in range(3)
            for p in ("self_attn.q_proj", "self_attn.k_proj", "self_attn.v_proj", "self_attn.out_proj", "mlp.fc1", "mlp.fc2")}
    for encs, tags in (((enc.text_encoder,), ("lora_te",)), ((enc.text_encoder, enc.text_encoder_2), ("lora_te1", "lora_te2"))):
        names = lora.kohya_names(unet, encs)
        for i, tag in enumerate(tags):
            got = {k: n for k, (c, n) in names.items() if c == f"te{i + 1}"}
            assert set(got.values()) == want and len(got) == len(want)
            assert all(k == tag + "_" + n.replace(".", "_") for k, n in got.items())


# ---------------------------------------------------------------------------------------------------- CPU: errors
def _full_lora(unet, rank=2, seed=0):
    targets = lora.unet_targets(unet)
    fac = ls.lora_factors(targets, rank, seed)
    return fac, ls.kohya_dict(fac, {n: ls.diffusers_stem(n) for n in targets}, ALPHA)


def test_malformed_files_raise_value_error_naming_the_key():
    unet = _cpu_unet(uo.tiny_sd_config(), 1)
    _, sd = _full_lora(unet)
    k0 = "lora_unet_down_blocks_0_attentions_0_transformer_blocks_0_attn1_to_q"
    bad = dict(sd, **{"lora_unet_down_blocks_9_resnets_0_conv1.lora_down.weight": torch.zeros(2, 4, 3, 3),
                      "lora_unet_down_blocks_9_resnets_0_conv1.lora_up.weight": torch.zeros(4, 2, 1, 1)})
    with pytest.raises(ValueError, match="down_blocks_9_resnets_0_conv1"):
        lora.MergedLora(bad, unet)
    with pytest.raises(ValueError, match="lora_unet_conv_in"):      # not a target: the blocks only
        lora.MergedLora(dict(sd, **{"lora_unet_conv_in.lora_down.weight": torch.zeros(2, 4, 3, 3),
                                    "lora_unet_conv_in.lora_up.weight": torch.zeros(64, 2, 1, 1)}), unet)
    shp = dict(sd)
    shp[k0 + ".lora_up.weight"] = torch.zeros(65, 2)
    with pytest.raises(ValueError, match=k0):
        lora.MergedLora(shp, unet)
    conv = "lora_unet_down_blocks_0_resnets_0_conv1"
    shp = dict(sd)
    shp[conv + ".lora_down.weight"] = torch.zeros(2, 64, 1, 1)      # 1x1 down on a 3x3 conv
    with pytest.raises(ValueError, match=conv):
        lora.MergedLora(shp, unet)
    half = {k: v for k, v in sd.items() if not k.startswith(k0 + ".lora_up")}
    with pytest.raises(ValueError, match=k0):
        lora.MergedLora(half, unet)
    for key in (k0 + ".hada_w1_a", k0 + ".lokr_w1", k0 + ".dora_scale", k0 + ".lora_mid.weight"):
        with pytest.raises(ValueError, match="LyCORIS"):
            lora.MergedLora(dict(sd, **{key: torch.zeros(2, 2)}), unet)
    with pytest.raises(ValueError, match="text-encoder"):
        lora.MergedLora(dict(sd, **{"text_encoder.text_model.encoder.layers.0.self_attn.q_proj.lora_A.weight": torch.zeros(2, 2)}), unet)
    with pytest.raises(ValueError, match="no supported format"):
        lora.MergedLora({"down_blocks.0.attentions.0.transformer_blocks.0.attn1.to_q.lora_A.weight": torch.zeros(2, 64)}, unet)
    with pytest.raises(ValueError, match="no text encoder|none is loaded"):
        lora.MergedLora(dict(sd, **{"lora_te_text_model_encoder_layers_0_mlp_fc1.lora_down.weight": torch.zeros(2, 32),
                                    "lora_te_text_model_encoder_layers_0_mlp_fc1.lora_up.weight": torch.zeros(64, 2)}), unet)
    # the same module named in both UNet schemes
    twice = dict(sd, **{"lora_unet_input_blocks_1_1_transformer_blocks_0_attn1_to_q.lora_down.weight": sd[k0 + ".lora_down.weight"],
                        "lora_unet_input_blocks_1_1_transformer_blocks_0_attn1_to_q.lora_up.weight": sd[k0 + ".lora_up.weight"]})
    with pytest.raises(ValueError, match="named twice"):
        lora.MergedLora(twice, unet)
    w0 = _cpu_unet(uo.tiny_sd_config(), 1).state_dict()
    assert all(torch.equal(v, w0[k]) for k, v in unet.state_dict().items()), "a failed load merged weights"


def test_sampler_refuses_a_second_lora_and_a_scale_without_one():
    from rtti_b200.region_diffusion import RegionDiffusion
    unet = _cpu_unet(uo.tiny_sd_config(), 1)
    m = RegionDiffusion(device="cpu", unet=unet, vae=None)
    with pytest.raises(RuntimeError, match="no LoRA"):
        m.set_lora_scale(0.5)
    _, sd = _full_lora(unet)
    m.load_lora_weights(sd, 0.5)
    with pytest.raises(ValueError, match="already loaded"):
        m.load_lora_weights(sd)
    m.unload_lora_weights()
    m.unload_lora_weights()
    m.load_lora_weights(sd)


# ---------------------------------------------------------------------------------------------------- CPU: merge
def test_merge_equals_w0_plus_scaled_product_and_conv_lora_is_down_then_up(tmp_path):
    safetensors = pytest.importorskip("safetensors.torch")
    unet = _cpu_unet(uo.tiny_sd_config(), 1)
    w0 = {k: v.clone() for k, v in unet.state_dict().items()}
    fac, sd = _full_lora(unet, rank=3, seed=4)
    path = tmp_path / "lora.safetensors"
    safetensors.save_file({k: v.contiguous() for k, v in sd.items()}, str(path))
    s = 0.7
    m = lora.MergedLora(str(path), unet)
    m.set_scale(s)
    targets = lora.unet_targets(unet)
    assert len(m.entries) == len(targets)
    g = torch.Generator().manual_seed(0)
    for n, mod in targets.items():
        down, up = fac[n]
        d = (up.double().flatten(1) @ down.double().flatten(1)).view(mod.weight.shape)
        want = w0[n + ".weight"].double() + s * ALPHA / down.shape[0] * d
        np.testing.assert_allclose(mod.weight.double().numpy(), want.numpy(), rtol=1e-6, atol=1e-7, err_msg=n)
        if isinstance(mod, torch.nn.Conv2d):
            x = torch.randn(1, mod.weight.shape[1], 9, 7, generator=g, dtype=torch.float64)
            st, pad = mod.stride, mod.padding
            got = F.conv2d(x, mod.weight.double(), None, st, pad) - F.conv2d(x, w0[n + ".weight"].double(), None, st, pad)
            lo = s * ALPHA / down.shape[0] * F.conv2d(F.conv2d(x, down.double(), None, st, pad), up.double())
            np.testing.assert_allclose(got.numpy(), lo.numpy(), rtol=1e-5, atol=1e-6, err_msg=n)
    for k, v in unet.state_dict().items():   # biases and non-targets untouched
        if k[:-len(".weight")] not in targets or not k.endswith(".weight"):
            assert torch.equal(v, w0[k]), k


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_rescale_and_unload_are_bit_exact(dtype):
    unet = _cpu_unet(uo.tiny_xl_config(), 2, dtype)
    w0 = {k: v.clone() for k, v in unet.state_dict().items()}
    _, sd = _full_lora(unet, rank=4, seed=5)

    def weights():
        return {k: v.clone() for k, v in unet.state_dict().items()}
    m = lora.MergedLora(sd, unet)
    m.set_scale(0.8)
    at_s = weights()
    assert any(not torch.equal(at_s[k], w0[k]) for k in w0)
    m.set_scale(-0.3)
    assert any(not torch.equal(v, at_s[k]) for k, v in unet.state_dict().items())
    m.set_scale(0.8)
    assert all(torch.equal(v, at_s[k]) for k, v in unet.state_dict().items())
    m.set_scale(0.0)
    assert all(torch.equal(v, w0[k]) for k, v in unet.state_dict().items())
    m.set_scale(0.8)
    m.unload()
    assert all(torch.equal(v, w0[k]) for k, v in unet.state_dict().items())


def test_text_encoder_lora_merges_into_both_encoders(tmp_path):
    enc = _tiny_clip(tmp_path)
    from rtti_b200.region_diffusion_sdxl import RegionDiffusionXL
    unet = _cpu_unet(uo.tiny_xl_config(), 2)
    m = RegionDiffusionXL(device="cpu", unet=unet, vae=None, text_encoders=enc)
    t1, t2 = lora.clip_targets(enc.text_encoder), lora.clip_targets(enc.text_encoder_2)
    f1, f2 = ls.lora_factors(t1, 2, 1), ls.lora_factors(t2, 2, 2)
    sd = {**ls.kohya_dict(f1, {n: "lora_te1_" + n.replace(".", "_") for n in t1}, ALPHA),
          **ls.kohya_dict(f2, {n: "lora_te2_" + n.replace(".", "_") for n in t2}, ALPHA)}
    w0 = {n: mod.weight.clone() for n, mod in t2.items()}
    before = enc.encode(["a red cat"], None, "cpu")[0]
    m.load_lora_weights(sd, 0.5)
    for n, mod in t2.items():
        down, up = f2[n]
        want = w0[n].double() + 0.5 * ALPHA / 2 * (up.double() @ down.double())
        assert bool(((mod.weight.double() - want).abs() <= 2.0 ** -10 * want.abs() + 2.0 ** -24).all()), n
    assert not torch.equal(enc.encode(["a red cat"], None, "cpu")[0], before)
    m.unload_lora_weights()
    assert torch.equal(enc.encode(["a red cat"], None, "cpu")[0], before)


# ---------------------------------------------------------------------------------------------------- CPU: oracle
@pytest.mark.parametrize("name,cfg", [("tiny_sd", uo.tiny_sd_config()), ("tiny_xl", uo.tiny_xl_config())])
def test_tiny_unet_with_merged_lora_matches_the_unmerged_oracle(monkeypatch, name, cfg):
    """The merged weights in the oracle UNet against the oracle with the adapter run unmerged
    (W0 x + s (alpha / r) up(down(x)) at every target), fp32, at the tolerance of the tiny-UNet golden tests."""
    unet = _cpu_unet(cfg, 3)
    sd0 = uo.make_state_dict(cfg, 3)
    fac, lsd = _full_lora(unet, rank=4, seed=6)
    s = 0.9
    lora.MergedLora(lsd, unet).set_scale(s)
    merged = {k: v.clone() for k, v in unet.state_dict().items()}
    pooled = cfg.projection_class_embeddings_input_dim - 6 * cfg.addition_time_embed_dim if cfg.addition_embed_type else 0
    inp = synth.synth_inputs(cfg.cross_attention_dim, pooled, 1, 16, 8)
    x = torch.cat([inp["latents"], inp["latents"].flip(-1)])
    added = {"text_embeds": inp["text_embeds"], "time_ids": inp["time_ids"].repeat(2, 1)} if cfg.addition_embed_type else None
    with torch.no_grad():
        y_merged = uo.unet_forward(merged, cfg, x, torch.tensor(601), inp["ctx"], added)
        y_plain = uo.unet_forward(sd0, cfg, x, torch.tensor(601), inp["ctx"], added)
        monkeypatch.setattr(uo, "F", ls.UnmergedF(ls.unmerged_table(sd0, fac, s, ALPHA)))
        y_lora = uo.unet_forward(sd0, cfg, x, torch.tensor(601), inp["ctx"], added)
    np.testing.assert_allclose(y_merged.numpy(), y_lora.numpy(), atol=1e-5, rtol=1e-5)
    assert float((y_lora - y_plain).abs().max()) > 100 * 1e-5   # the LoRA changes the output well past the tolerance


# ---------------------------------------------------------------------------------------------------- GPU: full UNets
@pytest.fixture
def deterministic_cudnn():
    prev = torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
    try:
        yield
    finally:
        torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = prev


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["sd15", "sdxl"])
def test_lora_unet_vs_fp64_unmerged(deterministic_cudnn, kind):
    """Full-size UNet, random rank-16 LoRA on every linear and conv of the blocks, merged at scale 0.8, on the plain CFG
    batch (SD1.5 64^2, SDXL 128^2). The merged fp16 weights are within one fp16 rounding of the float64 merge; the
    product output satisfies the rule of test_unet_fp64.py against the UNet evaluated unmerged in float64, with the
    fp16 PyTorch computations (unmerged and merged) as comparators."""
    from tests import test_unet_fp64 as tf
    F64 = torch.float64
    xl = kind == "sdxl"
    pcfg, ocfg = tf._configs(kind)
    S, t, s = (128 if xl else 64), 981, 0.8
    what = f"{kind} LoRA plain {S}x{S} t{t}"
    with tf._case(what, 48 if xl else 16):
        x, ctx, te, tid = tf._inputs(ocfg, 2, S, S, 2, seed=S + 11)
        tid2 = tid.expand(2, -1) if xl else None
        unet = tf._product(pcfg, seed=7 if xl else 5)
        sd0 = {k: v.clone() for k, v in unet.state_dict().items()}
        targets = lora.unet_targets(unet)
        fac = ls.lora_factors(targets, 16, seed=21, device="cuda")
        m = lora.MergedLora(ls.kohya_dict(fac, {n: ls.diffusers_stem(n) for n in targets}, ALPHA), unet)
        m.set_scale(s)
        with torch.no_grad():
            worst = 0.0
            for n, mod in targets.items():
                down, up = fac[n]
                d = (up.double().flatten(1) @ down.double().flatten(1)).view(mod.weight.shape)
                ref = sd0[n + ".weight"].double() + s * ALPHA / down.shape[0] * d
                err = (mod.weight.double() - ref).abs()
                assert bool((err <= 2.0 ** -10 * ref.abs() + 2.0 ** -24).all()), f"{n}: merge off by more than an fp16 ulp"
                worst = max(worst, float((err / (ref.abs() + 2.0 ** -14)).max()))
            print(f"[merge] {kind}: {len(targets)} weights, max relative error {worst:.3e}")
            y, _ = tf._twice(lambda: (unet(x, t, ctx, tf._added(te, tid2, slice(0, 2)))["sample"], {}))
            sdm = unet.state_dict()
            y16m = uo.unet_forward(sdm, ocfg, x, t, ctx, tf._added(te, tid2, slice(0, 2)))
            del unet, m, sdm
            torch.cuda.empty_cache()
            prev = uo.F
            try:
                uo.F = ls.UnmergedF(ls.unmerged_table(sd0, fac, s, ALPHA))
                y16u = uo.unet_forward(sd0, ocfg, x, t, ctx, tf._added(te, tid2, slice(0, 2)))
                sd64 = tf._to64(sd0)
                del sd0
                torch.cuda.empty_cache()
                uo.F = ls.UnmergedF(ls.unmerged_table(sd64, fac, s, ALPHA))
                y64 = torch.empty(y.shape, dtype=F64, device="cuda")
                for b in range(2):
                    xb, cb, ab = x[b:b + 1].to(F64), ctx[b:b + 1].to(F64), tf._added(te, tid, slice(b, b + 1), F64)
                    with tf.Float64Guard():
                        y64[b:b + 1] = uo.unet_forward(sd64, ocfg, xb, t, cb, ab)
            finally:
                uo.F = prev
            del sd64
        tf._rule(f"{what} eps", y, [y16u, y16m], y64)


# ---------------------------------------------------------------------------------------------------- GPU: samplers
S_XL, S_SD = 64, 32


def _xl_unet(seed=2):
    cfg = uo.tiny_xl_config()
    unet = UNet2DConditionModel(UNetConfig.from_dict(cfg.__dict__))
    unet.load_state_dict(uo.make_state_dict(cfg, seed))
    return cfg, unet.finalize("cuda")


def _sd_unet(seed=1):
    cfg = uo.tiny_sd_config()
    unet = UNet2DConditionModel(UNetConfig.from_dict(cfg.__dict__))
    unet.load_state_dict(uo.make_state_dict(cfg, seed))
    return cfg, unet.finalize("cuda")


def _premerged(make, lsd, scale):
    """A UNet built from weights that had the merge applied before the model was made."""
    cfg, donor = make()
    lora.MergedLora(lsd, donor).set_scale(scale)
    sd = {k: v.float().contiguous() for k, v in donor.state_dict().items()}
    unet = UNet2DConditionModel(UNetConfig.from_dict(cfg.__dict__))
    unet.load_state_dict(sd)
    return unet.finalize("cuda")


def _sgm_lora(unet, seed):
    """kohya SDXL-trainer naming (input_blocks / middle_block / output_blocks) for every target."""
    names = lora.kohya_names(unet)
    stems = {n: k for k, (_, n) in names.items() if _SGM.match(k)}
    targets = lora.unet_targets(unet)
    return ls.kohya_dict(ls.lora_factors(targets, 8, seed), stems, ALPHA)


def _xl_runs(model, cfg, **kw):
    from tests import synth as sy
    pooled = cfg.projection_class_embeddings_input_dim - 6 * cfg.addition_time_embed_dim
    inp = sy.synth_inputs(cfg.cross_attention_dim, pooled, 3, S_XL, 31)
    ctx, te = inp["ctx"].cuda(), inp["text_embeds"].cuda()
    common = dict(height=S_XL * 8, width=S_XL * 8, num_inference_steps=4, guidance_scale=8.5,
                  latents=inp["latents"].clone(), negative_prompt_embeds=ctx[:1],
                  negative_pooled_prompt_embeds=te[:1], output_type="latent", **kw)
    plain = model.sample(prompt_embeds=ctx[-1:], pooled_prompt_embeds=te[-1:], **common).images.clone()
    tfd = sy.font_sizes()
    tfd.update(sy.color_dict(inp["masks"], S_XL, 1.0))
    model.masks = [x.cuda() for x in inp["masks"]]
    rich = model.sample(prompt_embeds=ctx[1:], pooled_prompt_embeds=te[1:], run_rich_text=True, use_guidance=True,
                        inject_selfattn=0.5, inject_background=0.5, text_format_dict=tfd, **common).images.clone()
    return plain, rich


def _xl_model(unet):
    from rtti_b200.region_diffusion_sdxl import RegionDiffusionXL
    m = RegionDiffusionXL(device="cuda", unet=unet, vae=synth.TinyVAE("cuda"))
    m.use_cuda_graphs = True
    return m


@pytest.mark.gpu
def test_lora_xl_sampler_is_bit_identical_to_premerged_weights():
    """RegionDiffusionXL (tiny SDXL-shaped UNet, CUDA graphs on): plain pass and rich-text pass (colour guidance,
    injection, font sizes) with a LoRA loaded equal a model built from pre-merged weights; a second call at another
    scale through cross_attention_kwargs equals a fresh model at that scale (no stale graph, K/V cache or fused
    weight); unloading equals the model without a LoRA."""
    cfg, unet = _xl_unet()
    lsd = _sgm_lora(unet, 3)
    model = _xl_model(unet)
    base = _xl_runs(model, cfg)
    model.load_lora_weights(lsd, scale=0.7)
    got = _xl_runs(model, cfg)
    want = _xl_runs(_xl_model(_premerged(_xl_unet, lsd, 0.7)), cfg)
    for a, b, c, what in zip(got, want, base, ("plain", "rich")):
        assert torch.equal(a, b), f"{what}: LoRA loaded vs pre-merged weights differ"
        assert not torch.equal(a, c), f"{what}: the LoRA changed nothing"
    got2 = _xl_runs(model, cfg, cross_attention_kwargs={"scale": 0.3})
    assert model._lora.scale == 0.3
    fresh = _xl_model(_xl_unet()[1])
    fresh.load_lora_weights(lsd, scale=0.3)
    want2 = _xl_runs(fresh, cfg)
    for a, b, what in zip(got2, want2, ("plain", "rich")):
        assert torch.equal(a, b), f"{what}: second call at scale 0.3 differs from a fresh model at 0.3"
    again = _xl_runs(model, cfg)   # the scale persists after the call
    assert all(torch.equal(a, b) for a, b in zip(again, got2))
    model.unload_lora_weights()
    assert all(torch.equal(a, b) for a, b in zip(_xl_runs(model, cfg), base)), "unloading did not restore the model"


def _sd_run(model, cfg):
    inp = synth.synth_inputs(cfg.cross_attention_dim, 0, 3, S_SD, 21)
    model.masks = [x.cuda() for x in inp["masks"]]
    tfd = synth.font_sizes()
    tfd.update(synth.color_dict(inp["masks"], S_SD, 0.5))
    return model.produce_latents(inp["ctx"].cuda(), height=S_SD * 8, width=S_SD * 8, num_inference_steps=5,
                                 guidance_scale=8.5, latents=inp["latents"].clone(), use_guidance=True,
                                 text_format_dict=tfd, inject_selfattn=0.3, inject_background=0.5).clone()


def _sd_model(unet):
    from rtti_b200.region_diffusion import RegionDiffusion
    return RegionDiffusion(device="cuda", unet=unet, vae=synth.TinyVAE("cuda"))


@pytest.mark.gpu
def test_lora_sd_produce_latents_is_bit_identical_to_premerged_weights():
    """RegionDiffusion.produce_latents (tiny SD1.5-shaped UNet: conv proj_in / proj_out) with a LoRA in diffusers'
    naming on every target, against pre-merged weights, and after set_lora_scale against a fresh model at that scale."""
    cfg, unet = _sd_unet()
    targets = lora.unet_targets(unet)
    lsd = ls.kohya_dict(ls.lora_factors(targets, 8, 4), {n: ls.diffusers_stem(n) for n in targets}, ALPHA)
    model = _sd_model(unet)
    base = _sd_run(model, cfg)
    model.load_lora_weights(lsd, scale=0.7)
    got = _sd_run(model, cfg)
    assert torch.equal(got, _sd_run(_sd_model(_premerged(_sd_unet, lsd, 0.7)), cfg))
    assert not torch.equal(got, base)
    model.set_lora_scale(0.3)
    fresh = _sd_model(_sd_unet()[1])
    fresh.load_lora_weights(lsd, scale=0.3)
    assert torch.equal(_sd_run(model, cfg), _sd_run(fresh, cfg))
    model.unload_lora_weights()
    assert torch.equal(_sd_run(model, cfg), base)


@pytest.mark.gpu
def test_lora_rich_loop_two_gpus():
    """The rich-text loop with a LoRA on two GPUs against one (tests/multigpu_lora_check.py)."""
    import os
    import subprocess
    import sys
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
                        "--master-addr", "127.0.0.1", "--master-port", "29551",
                        os.path.join(root, "tests", "multigpu_lora_check.py")],
                       capture_output=True, text=True, timeout=900)
    print(r.stdout[-2000:], r.stderr[-2000:])
    assert r.returncode == 0 and "MULTIGPU_LORA_CHECK PASS" in r.stdout
