"""CPU: the oracle against the UNMODIFIED reference on inputs other than the golden fixtures of test_oracle_golden.py.
The reference's side of every comparison was recorded from the reference itself by oracle/gen_golden.py
(reference_checks): tests/golden/reference_checks.npz and tests/golden/richtext_reference.json."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import unet_oracle as uo

UNET_TIMESTEPS = (torch.tensor(999), torch.tensor(37.0, dtype=torch.float64))


@pytest.fixture(scope="module")
def ref(golden_dir):
    return np.load(os.path.join(golden_dir, "reference_checks.npz"), allow_pickle=False)


def unet_inputs(cfg, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(2, 4, 16, 16, generator=g)
    ctx = torch.randn(2, 77, cfg.cross_attention_dim, generator=g)
    added = None
    if cfg.addition_embed_type:
        pooled = cfg.projection_class_embeddings_input_dim - 6 * cfg.addition_time_embed_dim
        added = {"text_embeds": torch.randn(2, pooled, generator=g), "time_ids": torch.tensor([[128.0, 128, 0, 0, 128, 128]] * 2)}
    return x, ctx, added


@pytest.mark.parametrize("cfg_fn,seed", [(uo.tiny_sd_config, 3), (uo.tiny_xl_config, 4)])
def test_unet_forward_bit_exact(ref, cfg_fn, seed):
    name = cfg_fn.__name__[:-len("_config")]   # tiny_sd / tiny_xl
    cfg = cfg_fn()
    sd = uo.make_state_dict(cfg, seed)
    x, ctx, added = unet_inputs(cfg, seed)
    with torch.no_grad():
        for i, t in enumerate(UNET_TIMESTEPS):
            yo = uo.unet_forward(sd, cfg, x, t, ctx, added)
            assert torch.equal(torch.from_numpy(ref[f"unet_{name}_t{i}"]), yo)


def test_full_size_parameter_inventories(ref):
    for name, cfg, nparams in (("sd15", uo.sd15_config(), 859.5e6), ("sdxl", uo.sdxl_config(), 2567.5e6)):
        shapes = {str(k): tuple(int(d) for d in s if d >= 0) for k, s in zip(ref[f"inv_{name}_names"], ref[f"inv_{name}_shapes"])}
        mine = {k: tuple(v) for k, v in uo.param_shapes(cfg).items()}
        assert shapes == mine
        assert abs(sum(torch.Size(s).numel() for s in mine.values()) - nparams) < 0.1e6


def attention_weights():
    return {"word_pos": torch.LongTensor([1, 4, 4]), "font_size": torch.FloatTensor([3.0, -2.0, 0.25])}


def test_attention_fontsize_and_injection(ref):
    sd = {"a." + k[len("attn_w_"):]: torch.from_numpy(ref[k]) for k in ref.files if k.startswith("attn_w_")}
    hs, ctx = torch.from_numpy(ref["attn_hs"]), torch.from_numpy(ref["attn_ctx"])
    aw = attention_weights()

    class C(uo.AttnControl):
        def pre_attn(self, name):
            return None, aw

        def post_attn(self, name, pavg, p):
            self.out = (pavg, p)

    c = C()
    with torch.no_grad():
        o = uo.attention(sd, "a", 2, hs, ctx, c)
    o_ref, pavg_ref, p_ref = (torch.from_numpy(ref[k]) for k in ("attn_out", "attn_pavg", "attn_p"))
    assert torch.allclose(o, o_ref, atol=1e-6) and torch.allclose(c.out[0], pavg_ref, atol=1e-7)
    assert torch.allclose(c.out[1], p_ref, atol=1e-7)


# --------------------------------------------------------------------------- host-side text preparation (SURVEY 8f.4)
class _Tok:
    def _tokenize(self, text):
        return text.lower().replace(",", " ,").split()


class _Model:
    tokenizer = _Tok()


_DELTAS = [
    {"ops": [{"insert": "a church "}, {"attributes": {"color": "#fd6c9e"}, "insert": "garden"},
             {"insert": " with "}, {"attributes": {"font": "slabo"}, "insert": "mountains"},
             {"attributes": {"size": "60px"}, "insert": " snowy"}, {"attributes": {"link": "a red sun"}, "insert": " sky"},
             {"insert": "\n"}]},
    {"ops": [{"attributes": {"font": "mirza"}, "insert": "a lake"}, {"attributes": {"font": "mirza"}, "insert": " at dawn"},
             {"insert": ", "}, {"attributes": {"color": "#00ff00", "size": "18px", "strike": True}, "insert": "reeds"},
             {"insert": " and a "}, {"attributes": {"color": "#a52a2a"}, "insert": "boat"}, {"insert": "\n"}]},
    {"ops": [{"insert": "a plain prompt without attributes\n"}]},
]


def same(a, b):
    if torch.is_tensor(a) or torch.is_tensor(b):
        return torch.is_tensor(a) and torch.is_tensor(b) and a.shape == b.shape and torch.allclose(a.float().cpu(), b.float().cpu())
    if isinstance(a, (list, tuple)):
        return isinstance(b, (list, tuple)) and len(a) == len(b) and all(same(x, y) for x, y in zip(a, b))
    return a == b


@pytest.mark.parametrize("delta", _DELTAS)
def test_richtext_utils_match_the_reference_functions(golden_dir, delta):
    """rtti_b200.richtext_utils against utils/richtext_utils.py of the unmodified reference on the same Quill deltas:
    parse_json :74-136, get_region_diffusion_input :139-185, get_attention_control_input :188-209,
    get_gradient_guidance_input :212-234 — identical prompts, token ids, font sizes and target colours."""
    from oracle.gen_golden import from_json
    from rtti_b200 import richtext_utils as ru
    with open(os.path.join(golden_dir, "richtext_reference.json")) as f:
        rec = from_json(json.load(f)[_DELTAS.index(delta)])
    out_r = rec["parse_json"]
    out_p = ru.parse_json(delta, device="cpu")
    assert len(out_r) == len(out_p) == 9
    for j, (a, b) in enumerate(zip(out_r, out_p)):
        assert same(a, b), f"parse_json output {j}: {a!r} vs {b!r}"
    base, styles, notes, note_t, cspans, cnames, crgbs, sizes, use_grad = out_p
    pr, idr, btr = rec["region"]
    pp, idp, btp = ru.get_region_diffusion_input(_Model(), base, styles, notes, note_t, cspans, cnames)
    assert pr == pp and btr == btp and same(idr, idp)
    tr = rec["control"]
    tp = ru.get_attention_control_input(_Model(), btp, sizes, device="cpu")
    assert set(tr) == set(tp) and all(same(tr[k], tp[k]) for k in tr)
    tr2, cr = rec["gradient"]
    tp2, cp = ru.get_gradient_guidance_input(_Model(), btp, cspans, out_p[6], dict(tp), color_guidance_weight=0.5)
    assert same(cr, cp) and set(tr2) == set(tp2)
    for k in tr2:
        assert same(tr2[k], tp2[k]), k


XL_LIVE_CASES = [
    # n_prompts, steps, inject_selfattn, inject_background, use_guidance, with_fs, seed
    (4, 3, 0.4, 0.0, False, True, 71),      # more regions, self-attention / feature injection on the first step only
    (2, 3, 0.0, 0.4, True, False, 72),      # configs[3]-like: background injection only (the joint-stepping quirk), colour guidance
]
XL_S = 128   # the reference asserts a 64-wide injected feature map (sdxl.py:1090): 1024^2 images only


def xl_reference_loop(ns, n_prompts, steps, inject_selfattn, inject_background, use_guidance, with_fs, seed):
    """RegionDiffusionXL.sample(run_rich_text=True) of the reference (models/region_diffusion_sdxl.py:772-878)."""
    from oracle import gen_golden as gg
    cfg = uo.tiny_xl_config()
    inp = gg.synth_inputs(cfg, n_prompts, XL_S, seed)
    ctx, te = inp["ctx"], inp["text_embeds"]
    m = gg.make_xl_sampler(ns, cfg, 5, (ctx[1:], ctx[:1], te[1:], te[:1]))
    m.masks = inp["masks"]
    tfd = gg.text_format(1, XL_S, seed, with_fs=with_fs)
    if use_guidance:
        tfd.update(gg.color_dict(inp["masks"], XL_S, weight=0.7))
    return m.sample(["p"] * n_prompts, height=XL_S * 8, width=XL_S * 8, num_inference_steps=steps, guidance_scale=6.0,
                    negative_prompt=[""], latents=inp["latents"].clone(), output_type="latent", use_guidance=use_guidance,
                    inject_selfattn=inject_selfattn, inject_background=inject_background, text_format_dict=dict(tfd),
                    run_rich_text=True).images.detach()


@pytest.mark.parametrize("n_prompts,steps,inject_selfattn,inject_background,use_guidance,with_fs,seed", XL_LIVE_CASES)
def test_xl_rich_loop_live_reference_other_settings(ref, n_prompts, steps, inject_selfattn, inject_background, use_guidance,
                                                    with_fs, seed):
    """The reference's rich-text XL loop against the oracle's rich_text_loop at settings the golden loop fixtures do
    not cover: other region counts, step counts, injection windows, with / without font sizes and colour guidance."""
    from oracle import sampler_oracle as sam, schedulers_oracle as so
    from oracle.gen_golden import synth_inputs, text_format, color_dict
    from tests import synth
    i = XL_LIVE_CASES.index((n_prompts, steps, inject_selfattn, inject_background, use_guidance, with_fs, seed))
    cfg = uo.tiny_xl_config()
    inp = synth_inputs(cfg, n_prompts, XL_S, seed)
    ctx, te = inp["ctx"], inp["text_embeds"]
    tfd = text_format(1, XL_S, seed, with_fs=with_fs)
    if use_guidance:
        tfd.update(color_dict(inp["masks"], XL_S, weight=0.7))
    sd = uo.make_state_dict(cfg, 5)
    sch = so.EulerDiscreteSchedulerOracle()
    sch.set_timesteps(steps)
    added = {"text_embeds": te, "time_ids": inp["time_ids"]}
    lat = sam.rich_text_loop(sam.make_unet_fn(sd, cfg), sch, ctx, inp["masks"], inp["latents"].clone() * sch.init_noise_sigma,
                             steps, 6.0, xl=True, added_cond=added, use_guidance=use_guidance, text_format_dict=dict(tfd),
                             inject_selfattn=inject_selfattn, inject_background=inject_background,
                             vae_decode=synth.TinyVAE() if use_guidance else None, scaling_factor=0.13025)
    out = torch.from_numpy(ref[f"xl_live_{i}"])
    assert torch.isfinite(out).all()
    torch.testing.assert_close(lat, out, atol=5e-4, rtol=1e-4)
