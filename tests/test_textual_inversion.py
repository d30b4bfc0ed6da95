"""Textual-inversion embeddings (rtti_b200/textual_inversion.py) on the tiny on-disk CLIP fixture of test_loading.py
(20-token BPE vocabulary, hidden size 32, two tokenizer / encoder pairs).

The restatement every encoding is checked against: the encoder as it was before loading, given the prompt with the
token written as n placeholder words, and the learned vectors put at those positions by hand (a forward hook on the
token-embedding table). On the CPU in fp32; on the GPU in fp16, through both samplers, where the same embeddings must
give the same latents bit for bit."""
import pytest
import torch

from oracle import unet_oracle as uo
from rtti_b200 import loading
from rtti_b200 import richtext_utils as ru
from rtti_b200 import textual_inversion as ti
from rtti_b200.region_diffusion import RegionDiffusion
from rtti_b200.region_diffusion_sdxl import RegionDiffusionXL
from rtti_b200.unet import UNet2DConditionModel, UNetConfig
from tests import lora_synth as ls
from tests import synth

safetensors = pytest.importorskip("safetensors.torch")

TOK = "<tok>"
N = 3
PH = "b"    # placeholder word of the restatement: one token ("b</w>") that the test prompts do not otherwise use
PROMPTS = ["a <tok> red cat", "cat a red"]
NEGATIVE = ["<tok> a cat"]


@pytest.fixture(scope="module")
def clip_root(tmp_path_factory):
    from tests.test_loading import _tiny_clip_dir
    root = tmp_path_factory.mktemp("clip")
    _tiny_clip_dir(str(root))
    return str(root)


def _encoders(root, xl, device="cpu", fp32=True):
    enc = loading.ClipTextEncoders(root, device, xl=xl)
    if fp32:
        enc.text_encoder.float()
        if xl:
            enc.text_encoder_2.float()
    return enc


def _meta_unet(cfg):
    with torch.device("meta"):
        return UNet2DConditionModel(UNetConfig.from_dict(cfg.__dict__))


def _model(root, xl, fp32=True):
    enc = _encoders(root, xl, fp32=fp32)
    if xl:
        return RegionDiffusionXL(device="cpu", unet=_meta_unet(uo.tiny_xl_config()), vae=None, text_encoders=enc)
    return RegionDiffusion(device="cpu", unet=_meta_unet(uo.tiny_sd_config()), vae=None, text_encoder=enc)


def _vecs(xl, n=N, seed=0, widths=None):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(n, w, generator=g) for w in (widths or ((32, 32) if xl else (32,)))]


def _pairs(enc, xl):
    return [(enc.tokenizer, enc.text_encoder)] + ([(enc.tokenizer_2, enc.text_encoder_2)] if xl else [])


class _Placed:
    """Forward hooks on the token-embedding tables of `enc` (no embedding loaded) that write the learned vectors over
    the runs of N placeholder tokens, one hook per encoder with its own vectors."""

    def __init__(self, enc, xl, vecs):
        self.handles = []
        for (tok, model), vec in zip(_pairs(enc, xl), vecs):
            ph = tok.convert_tokens_to_ids(PH + "</w>")

            def hook(mod, inp, out, ph=ph, vec=vec):
                out = out.clone()
                for b in range(out.shape[0]):
                    at = (inp[0][b] == ph).nonzero().flatten()
                    assert len(at) % N == 0
                    out[b, at] = vec.to(out.device, out.dtype).repeat(len(at) // N, 1)
                return out
            self.handles.append(model.get_input_embeddings().register_forward_hook(hook))

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        for h in self.handles:
            h.remove()


def _restate(prompts):
    return [p.replace(TOK, " ".join([PH] * N)) for p in prompts]


def _restated_encode(ref, xl, vecs, prompts, negative, device="cpu"):
    with _Placed(ref, xl, vecs):
        if xl:
            return ref.encode(_restate(prompts), _restate(negative), device)
        return ref.encode_pair(_restate(prompts), _restate(negative), device)


def _write(fmt, tmp_path, vecs):
    """(source, token argument) of one embedding in the format `fmt`."""
    v = vecs[0]
    if fmt == "diffusers_bin":
        torch.save({TOK: v}, tmp_path / "learned_embeds.bin")
        return str(tmp_path / "learned_embeds.bin"), None
    if fmt == "diffusers_safetensors":
        safetensors.save_file({TOK: v}, str(tmp_path / "any.safetensors"))
        return str(tmp_path / "any.safetensors"), None
    if fmt == "diffusers_dir":
        (tmp_path / "concept").mkdir()
        safetensors.save_file({TOK: v}, str(tmp_path / "concept" / "learned_embeds.safetensors"))
        return str(tmp_path / "concept"), None
    if fmt == "dir_weight_name":
        (tmp_path / "concept").mkdir()
        torch.save({TOK: v}, tmp_path / "concept" / "cat.bin")
        safetensors.save_file({"<other>": v * 0}, str(tmp_path / "concept" / "learned_embeds.safetensors"))
        return str(tmp_path / "concept"), None
    if fmt == "state_dict":
        return {"<other>": v}, TOK          # the token argument wins over the stored one
    if fmt == "a1111_pt":
        torch.save({"string_to_token": {"*": 265}, "string_to_param": {"*": v}, "name": TOK, "step": 500,
                    "sd_checkpoint": None, "sd_checkpoint_name": None}, tmp_path / "concept.pt")
        return str(tmp_path / "concept.pt"), None
    if fmt == "a1111_emb_params":
        safetensors.save_file({"emb_params": v}, str(tmp_path / f"{TOK}.safetensors"))   # token: the file name
        return str(tmp_path / f"{TOK}.safetensors"), None
    if fmt == "sdxl_safetensors":
        safetensors.save_file({"clip_l": vecs[0], "clip_g": vecs[1]}, str(tmp_path / "sdxl.safetensors"))
        return str(tmp_path / "sdxl.safetensors"), TOK
    if fmt == "sdxl_dict":
        return {"clip_l": vecs[0], "clip_g": vecs[1]}, TOK
    raise AssertionError(fmt)


# ---------------------------------------------------------------------------------------------------- CPU: encoding
@pytest.mark.parametrize("fmt", ["diffusers_bin", "diffusers_safetensors", "diffusers_dir", "dir_weight_name", "state_dict",
                                 "a1111_pt", "a1111_emb_params"])
def test_sd15_encoding_equals_the_restatement(clip_root, tmp_path, fmt):
    vecs = _vecs(False)
    model = _model(clip_root, xl=False)
    ref = _encoders(clip_root, xl=False)
    before = model.get_text_embeds(PROMPTS, NEGATIVE)
    src, token = _write(fmt, tmp_path, vecs)
    model.load_textual_inversion(src, token=token, **({"weight_name": "cat.bin"} if fmt == "dir_weight_name" else {}))
    got = model.get_text_embeds(PROMPTS, NEGATIVE)
    want = _restated_encode(ref, False, vecs, PROMPTS, NEGATIVE)
    assert got.dtype == torch.float32 and torch.equal(got, want)
    # rows [uncond, prompt 0, prompt 1]: the one without the token is untouched, the others changed
    assert torch.equal(got[2], before[2]) and not torch.equal(got[1], before[1]) and not torch.equal(got[0], before[0])


@pytest.mark.parametrize("legacy_eos", [False, True])
@pytest.mark.parametrize("fmt", ["sdxl_safetensors", "sdxl_dict"])
def test_sdxl_encoding_equals_the_restatement(clip_root, tmp_path, fmt, legacy_eos):
    """Penultimate states of both encoders and the pooled output of the second. legacy_eos: the configuration of the
    released SDXL encoders (eos_token_id = 2) pools at the largest token id; the added ids are larger than EOS, and the
    pooled output must stay at the EOS position."""
    vecs = _vecs(True)
    model = _model(clip_root, xl=True)
    ref = _encoders(clip_root, xl=True)
    if legacy_eos:
        for e in (model.text_encoders, ref):
            e.text_encoder.text_model.eos_token_id = e.text_encoder_2.text_model.eos_token_id = 2
    before = model.encode_prompt(PROMPTS, NEGATIVE)
    src, token = _write(fmt, tmp_path, vecs)
    model.load_textual_inversion(src, token=token)
    got = model.encode_prompt(PROMPTS, NEGATIVE)
    want = _restated_encode(ref, True, vecs, PROMPTS, NEGATIVE)
    for g, w, b, what in zip(got, want, before, ("prompt_embeds", "negative", "pooled", "negative pooled")):
        assert g.dtype == torch.float32 and torch.equal(g, w), what
        assert not torch.equal(g[0], b[0]), what
    assert torch.equal(got[0][1], before[0][1]) and torch.equal(got[2][1], before[2][1])
    model.unload_textual_inversion()
    assert all(torch.equal(a, b) for a, b in zip(model.encode_prompt(PROMPTS, NEGATIVE), before))


def test_multi_vector_token_is_n_consecutive_ids(clip_root):
    model = _model(clip_root, xl=True)
    tok = model.tokenizer
    n0 = len(tok)
    vecs = _vecs(True)
    model.load_textual_inversion({"clip_l": vecs[0], "clip_g": vecs[1]}, token=TOK)
    model.load_textual_inversion({"clip_l": vecs[0][0], "clip_g": vecs[1][0]}, token="<one>")   # [d]: one token
    assert len(tok) == n0 + N + 1 and len(model.tokenizer_2) == n0 + N + 1
    seen = []
    hooks = [e.get_input_embeddings().register_forward_pre_hook(lambda m, a: seen.append(a[0].clone()))
             for e in (model.text_encoders.text_encoder, model.text_encoders.text_encoder_2)]
    model.encode_prompt(["a <tok> cat <one>"], ["<tok>"])
    for h in hooks:
        h.remove()
    assert len(seen) == 4    # prompt and negative prompt, both encoders
    ids = list(range(n0, n0 + N))
    bos, eos = tok.bos_token_id, tok.eos_token_id
    a, cat = tok.convert_tokens_to_ids(["a</w>", "cat</w>"])
    for got in seen[:2]:
        assert got[0, :8].tolist() == [bos, a] + ids + [cat, n0 + N, eos]
    for got in seen[2:]:
        assert got[0, :5].tolist() == [bos] + ids + [eos]
    assert ti.expand_prompt(tok, "a <tok>cat <one>") == "a <tok> <tok>_1 <tok>_2cat <one>"
    assert ti.tokenize(tok, "a <tok>cat <one>") == ["a</w>", "<tok>", "<tok>_1", "<tok>_2", "cat</w>", "<one>"]


# ---------------------------------------------------------------------------------------------------- CPU: rich text
def _delta(word, attrs):
    span = {"insert": word, "attributes": attrs} if attrs else {"insert": word}
    return {"ops": [{"insert": "a "}, span, {"insert": " "}, {"insert": "cat", "attributes": {"color": "#0000ff"}},
                    {"insert": " a "}, {"insert": "bed", "attributes": {"size": "60px"}}, {"insert": "\n"}]}


def _rich(model, delta):
    base, styles, notes, note_t, cspans, cnames, crgbs, sizes, _ = ru.parse_json(delta, device="cpu")
    prompts, ids, base_tokens = ru.get_region_diffusion_input(model, base, styles, notes, note_t, cspans, cnames)
    tfd = ru.get_attention_control_input(model, base_tokens, sizes, device="cpu")
    tfd, cids = ru.get_gradient_guidance_input(model, base_tokens, cspans, crgbs, tfd)
    return prompts, ids, base_tokens, tfd["word_pos"], tfd["font_size"], cids


def _expected(attr, word_pos):
    """Region ids, word_pos, font sizes and colour ids of _delta for positions {span: 1-based positions}."""
    p, n = word_pos, max(i for v in word_pos.values() for i in v)
    rest = lambda groups: [sorted(set(range(1, n + 1)) - {i for g in groups for i in g})]
    regions = {"link": [p["w"], p["cat"]], "color": [p["w"], p["cat"]], "font": [p["w"], p["cat"]],
               "size": [p["cat"]]}[attr]
    colours = [p["w"], p["cat"]] if attr == "color" else [p["cat"]]
    pos, fs = list(p["bed"]), [20.0] * 3
    if attr == "size":
        pos, fs = p["w"] + pos, [10.0] * len(p["w"]) + fs
    return regions + rest(regions), pos, fs, colours + rest(colours)


ATTRS = {"link": {"link": "a <tok> cat"}, "color": {"color": "#ff0000"}, "font": {"font": "slabo"},
         "size": {"size": "30px"}}


@pytest.mark.parametrize("attr", list(ATTRS))
def test_rich_text_positions_cover_the_vectors_and_shift_later_spans(clip_root, attr):
    """Base prompt "a <tok> cat a bed" with the span over <tok> coloured, footnoted, styled or resized, "cat" coloured and
    "bed" resized: <tok> covers positions 2-4 and every later span moves by N - 1 = 2. The same prompt with an ordinary
    word ("red") in place of <tok> gives the same lists and tensors with and without an embedding loaded."""
    model = _model(clip_root, xl=False)
    plain = _delta("red", ATTRS[attr])
    today = _rich(model, plain)
    model.load_textual_inversion({TOK: _vecs(False)[0]})
    model.load_textual_inversion({"<one>": torch.randn(32)})   # loaded, unused
    after = _rich(model, plain)
    for a, b in zip(today, after):
        if torch.is_tensor(a):
            assert a.dtype == b.dtype and torch.equal(a, b)
        else:
            assert len(a) == len(b) and all(torch.equal(x, y) if torch.is_tensor(x) else x == y for x, y in zip(a, b))
    want = _expected(attr, {"w": [2], "cat": [3], "bed": [5, 6, 7]})
    assert [i.tolist() for i in today[1]] == want[0] and today[3].tolist() == want[1]
    assert today[4].tolist() == want[2] and [i.tolist() for i in today[5]] == want[3]

    prompts, ids, base_tokens, word_pos, font_size, cids = _rich(model, _delta(TOK, ATTRS[attr]))
    assert base_tokens == ["a</w>", "<tok>", "<tok>_1", "<tok>_2", "cat</w>", "a</w>", "b", "e", "d</w>"]
    want = _expected(attr, {"w": [2, 3, 4], "cat": [5], "bed": [7, 8, 9]})
    assert [i.tolist() for i in ids] == want[0]
    assert word_pos.tolist() == want[1] and font_size.tolist() == want[2]
    assert [i.tolist() for i in cids] == want[3]
    assert prompts[-1] == "a <tok> cat a bed" and any(TOK in p for p in prompts[:-1]) == (attr != "size")


# ---------------------------------------------------------------------------------------------------- CPU: errors
def test_errors_name_the_problem_and_change_nothing(clip_root, tmp_path):
    sd, xl = _model(clip_root, xl=False), _model(clip_root, xl=True)
    n0 = len(sd.tokenizer)
    with pytest.raises(ValueError, match=r"hidden size 32.*\[n, 48\]"):
        sd.load_textual_inversion({TOK: torch.randn(N, 48)})
    with pytest.raises(ValueError, match=r"clip_l \[n, 32\] and clip_g \[n, 32\].*one \[n, 32\]"):   # SD1.5 file into SDXL
        xl.load_textual_inversion({TOK: torch.randn(N, 32)})
    with pytest.raises(ValueError, match=r"clip_g \[n, 48\]"):
        xl.load_textual_inversion({"clip_l": torch.randn(N, 32), "clip_g": torch.randn(N, 48)}, token=TOK)
    with pytest.raises(ValueError, match=r"one \[n, 32\] embedding.*clip_l \[n, 32\] and clip_g"):   # SDXL file into SD1.5
        sd.load_textual_inversion({"clip_l": torch.randn(N, 32), "clip_g": torch.randn(N, 32)}, token=TOK)
    with pytest.raises(ValueError, match="unknown format"):
        sd.load_textual_inversion({"a": torch.randn(32), "b": torch.randn(32)})
    torch.save([torch.randn(32)], tmp_path / "list.pt")
    with pytest.raises(ValueError, match="not a state dict"):
        sd.load_textual_inversion(str(tmp_path / "list.pt"), token=TOK)
    (tmp_path / "empty").mkdir()
    with pytest.raises(ValueError, match="none of.*weight_name"):
        sd.load_textual_inversion(str(tmp_path / "empty"), token=TOK)
    with pytest.raises(ValueError, match="not a local file or directory"):
        sd.load_textual_inversion("sd-concepts-library/cat-toy")
    with pytest.raises(ValueError, match="not a path or a state dict"):
        sd.load_textual_inversion(3)
    with pytest.raises(ValueError, match="no token"):
        xl.load_textual_inversion({"clip_l": torch.randn(N, 32), "clip_g": torch.randn(N, 32)})
    with pytest.raises(ValueError, match="'ca' is already in the tokenizer's vocabulary"):
        sd.load_textual_inversion({"ca": torch.randn(32)})
    assert len(sd.tokenizer) == n0 and len(xl.tokenizer) == n0 and len(xl.tokenizer_2) == n0
    assert sd.text_encoder.text_encoder.get_input_embeddings().num_embeddings == n0
    sd.load_textual_inversion({TOK: torch.randn(N, 32)})
    with pytest.raises(ValueError, match="already loaded"):
        sd.load_textual_inversion({TOK: torch.randn(2, 32)})
    with pytest.raises(ValueError, match="'<tok>_1' is already in"):   # a name taken by the vectors of <tok>
        sd.load_textual_inversion({"<tok>_1": torch.randn(32)})
    with pytest.raises(ValueError, match="'<x>_1' is already in"):     # the same clash inside one call
        sd.load_textual_inversion([{"<x>": torch.randn(2, 32)}, {"<x>_1": torch.randn(32)}])
    assert len(sd.tokenizer) == n0 + N


# ---------------------------------------------------------------------------------------------------- CPU: unload
@pytest.mark.parametrize("fp32", [True, False])
def test_unload_restores_vocabulary_and_tables_bit_for_bit(clip_root, fp32):
    model = _model(clip_root, xl=True, fp32=fp32)
    te = model.text_encoders
    state = [(len(t), t.tokenize("a <tok> cat"), e.get_input_embeddings().weight.clone(), e.config.vocab_size)
             for t, e in _pairs(te, True)]
    before = model.encode_prompt(PROMPTS, NEGATIVE)
    rng = torch.random.get_rng_state()
    vecs = _vecs(True)
    model.load_textual_inversion([{"clip_l": vecs[0], "clip_g": vecs[1]}, {"clip_l": vecs[0][0], "clip_g": vecs[1][0]}],
                                 token=[TOK, "<one>"])
    assert torch.equal(torch.random.get_rng_state(), rng), "loading drew from the global random stream"
    for (t, e), v in zip(_pairs(te, True), vecs):
        w = e.get_input_embeddings().weight
        assert w.dtype == (torch.float32 if fp32 else torch.float16)
        assert torch.equal(w[-N - 1:-1], v.to(w.dtype)) and torch.equal(w[-1], v[0].to(w.dtype))
    model.unload_textual_inversion()
    for (t, e), (n, toks, w, vs) in zip(_pairs(te, True), state):
        assert len(t) == n and t.tokenize("a <tok> cat") == toks and e.config.vocab_size == vs
        got = e.get_input_embeddings().weight
        assert got.shape == w.shape and got.dtype == w.dtype and torch.equal(got, w)
    assert all(torch.equal(a, b) for a, b in zip(model.encode_prompt(PROMPTS, NEGATIVE), before))
    model.unload_textual_inversion()    # no-op
    model.load_textual_inversion({"clip_l": vecs[0], "clip_g": vecs[1]}, token=TOK)   # the token is free again


# ---------------------------------------------------------------------------------------------------- CPU: LoRA
def _te_lora(model):
    from rtti_b200 import lora
    encs = (model.text_encoders.text_encoder, model.text_encoders.text_encoder_2)
    sd = {}
    for i, e in enumerate(encs):
        t = lora.clip_targets(e)
        sd.update(ls.kohya_dict(ls.lora_factors(t, 2, i + 1), {n: f"lora_te{i + 1}_" + n.replace(".", "_") for n in t}, 3.0))
    return sd


def _te_weights(model):
    return {f"{i}.{k}": v.clone() for i, e in enumerate((model.text_encoders.text_encoder, model.text_encoders.text_encoder_2))
            for k, v in e.state_dict().items()}


def test_lora_and_textual_inversion_are_independent(clip_root):
    vecs = _vecs(True)
    emb = {"clip_l": vecs[0], "clip_g": vecs[1]}
    a, b = _model(clip_root, xl=True), _model(clip_root, xl=True)
    lsd = _te_lora(a)
    w0 = _te_weights(a)
    a.load_lora_weights(lsd, scale=0.7)
    lora_only = _te_weights(a)
    a.load_textual_inversion(emb, token=TOK)
    b.load_textual_inversion(emb, token=TOK)
    b.load_lora_weights(lsd, scale=0.7)
    wa, wb = _te_weights(a), _te_weights(b)
    assert wa.keys() == wb.keys() and all(torch.equal(wa[k], wb[k]) for k in wa), "the load order changed the weights"
    ea, eb = a.encode_prompt(PROMPTS, NEGATIVE), b.encode_prompt(PROMPTS, NEGATIVE)
    assert all(torch.equal(x, y) for x, y in zip(ea, eb))
    emb_keys = [k for k in wa if "token_embedding" in k]
    # re-merging the LoRA leaves the added rows alone
    b.set_lora_scale(0.2)
    b.set_lora_scale(0.7)
    assert all(torch.equal(_te_weights(b)[k], wa[k]) for k in wa)
    # unloading the embedding keeps the merged LoRA
    a.unload_textual_inversion()
    wa = _te_weights(a)
    assert all(torch.equal(wa[k], lora_only[k]) for k in wa)
    # unloading the LoRA keeps the embedding
    b.unload_lora_weights()
    wb = _te_weights(b)
    assert all(torch.equal(wb[k], w0[k]) for k in w0 if k not in emb_keys)
    ti_only = _model(clip_root, xl=True)
    ti_only.load_textual_inversion(emb, token=TOK)
    assert all(torch.equal(x, y) for x, y in zip(b.encode_prompt(PROMPTS, NEGATIVE), ti_only.encode_prompt(PROMPTS, NEGATIVE)))
    a.unload_lora_weights()
    assert all(torch.equal(_te_weights(a)[k], w0[k]) for k in w0)


# ---------------------------------------------------------------------------------------------------- GPU: samplers
S_XL, S_SD = 64, 32
RICH = {"ops": [{"insert": "a "}, {"insert": TOK, "attributes": {"link": "a <tok> red cat"}}, {"insert": " "},
                {"insert": "cat", "attributes": {"color": "#0000ff"}}, {"insert": " a "},
                {"insert": "bed", "attributes": {"size": "60px"}}, {"insert": "\n"}]}


def _cuda_unet(cfg, seed):
    unet = UNet2DConditionModel(UNetConfig.from_dict(cfg.__dict__))
    unet.load_state_dict(uo.make_state_dict(cfg, seed))
    return unet.finalize("cuda")


def _rich_inputs(model, latent, seed):
    """Region prompts, masks and font sizes of RICH for `model`."""
    base, styles, notes, note_t, cspans, cnames, _, sizes, _ = ru.parse_json(RICH, device="cuda")
    prompts, _, base_tokens = ru.get_region_diffusion_input(model, base, styles, notes, note_t, cspans, cnames)
    tfd = ru.get_attention_control_input(model, base_tokens, sizes, device="cuda")
    assert tfd["word_pos"].tolist() == [7, 8, 9] and len(prompts) == 3
    model.masks = [m.cuda() for m in synth.synth_inputs(8, 0, len(prompts), latent, seed)["masks"]]
    return prompts, tfd


@pytest.mark.gpu
def test_xl_sampler_with_embedding_equals_the_restated_prompt_embeds(clip_root):
    """RegionDiffusionXL with fp16 tiny encoders (penultimate width 32 + 32, pooled 24) and a tiny SDXL-shaped UNet
    of that cross-attention and pooled width: the plain and rich-text passes from prompts with a 3-vector token equal
    the same passes given the restated embeddings, bit for bit."""
    import dataclasses
    cfg = dataclasses.replace(uo.tiny_xl_config(), cross_attention_dim=64, projection_class_embeddings_input_dim=24 + 6 * 32)
    enc = _encoders(clip_root, xl=True, device="cuda", fp32=False)
    ref = _encoders(clip_root, xl=True, device="cuda", fp32=False)
    model = RegionDiffusionXL(device="cuda", unet=_cuda_unet(cfg, 2), vae=None, text_encoders=enc)
    vecs = _vecs(True)
    model.load_textual_inversion({"clip_l": vecs[0], "clip_g": vecs[1]}, token=TOK)
    vecs = [v.half() for v in vecs]
    lat = synth.synth_inputs(8, 0, 1, S_XL, 5)["latents"]
    common = dict(height=S_XL * 8, width=S_XL * 8, num_inference_steps=3, guidance_scale=7.5, output_type="latent")

    def embeds(prompts, negative):
        got = model.encode_prompt(prompts, negative)
        want = _restated_encode(ref, True, vecs, prompts, negative, "cuda")
        assert all(torch.equal(a, b) for a, b in zip(got, want)), "encoded prompt differs from the restatement"
        return dict(zip(("prompt_embeds", "negative_prompt_embeds", "pooled_prompt_embeds",
                         "negative_pooled_prompt_embeds"), want))

    plain = model.sample(["a <tok> red cat"], negative_prompt=NEGATIVE, latents=lat.clone(), **common).images.clone()
    plain_ref = model.sample(latents=lat.clone(), **embeds(["a <tok> red cat"], NEGATIVE), **common).images
    assert torch.equal(plain, plain_ref), "plain pass"
    prompts, tfd = _rich_inputs(model, S_XL, 6)
    kw = dict(run_rich_text=True, text_format_dict=tfd, inject_selfattn=0.5, inject_background=0.3, **common)
    rich = model.sample(prompts, negative_prompt=NEGATIVE, latents=lat.clone(), **kw).images.clone()
    rich_ref = model.sample(latents=lat.clone(), **embeds(prompts, NEGATIVE), **kw).images
    assert torch.equal(rich, rich_ref), "rich-text pass"
    model.unload_textual_inversion()
    assert not torch.equal(model.sample(["a <tok> red cat"], negative_prompt=NEGATIVE, latents=lat.clone(),
                                        **common).images, plain)


@pytest.mark.gpu
def test_sd_sampler_with_embedding_equals_the_restated_text_embeddings(clip_root):
    """RegionDiffusion with an fp16 tiny encoder (width 32) and a tiny SD1.5-shaped UNet of that cross-attention
    width: produce_attn_maps (plain) and prompt_to_img (rich text) from prompts with a 3-vector token equal the same
    calls given the restated text embeddings, bit for bit."""
    import dataclasses
    cfg = dataclasses.replace(uo.tiny_sd_config(), cross_attention_dim=32)
    enc = _encoders(clip_root, xl=False, device="cuda", fp32=False)
    ref = _encoders(clip_root, xl=False, device="cuda", fp32=False)
    model = RegionDiffusion(device="cuda", unet=_cuda_unet(cfg, 1), vae=synth.TinyVAE("cuda"), text_encoder=enc)
    vecs = _vecs(False)
    model.load_textual_inversion({TOK: vecs[0]})
    vecs = [v.half() for v in vecs]
    lat = synth.synth_inputs(8, 0, 1, S_SD, 7)["latents"]
    common = dict(height=S_SD * 8, width=S_SD * 8, num_inference_steps=4, guidance_scale=7.5)

    def embeds(prompts, negative):
        got = model.get_text_embeds(prompts, negative)
        want = _restated_encode(ref, False, vecs, prompts, negative, "cuda")
        assert torch.equal(got, want), "encoded prompt differs from the restatement"
        return want

    plain = model.produce_attn_maps(["a <tok> red cat"], NEGATIVE, latents=lat.clone(), decode=False, **common).clone()
    plain_ref = model.produce_attn_maps(None, text_embeddings=embeds(["a <tok> red cat"], NEGATIVE), latents=lat.clone(),
                                        decode=False, **common)
    assert torch.equal(plain, plain_ref), "plain pass"
    prompts, tfd = _rich_inputs(model, S_SD, 8)
    kw = dict(text_format_dict=tfd, inject_selfattn=0.3, inject_background=0.5, **common)
    rich = model.prompt_to_img(prompts, NEGATIVE, latents=lat.clone(), **kw)
    rich_ref = model.prompt_to_img(prompts, NEGATIVE, latents=lat.clone(), text_embeddings=embeds(prompts, NEGATIVE), **kw)
    assert (rich == rich_ref).all(), "rich-text pass"
    latents = model.produce_latents(model.get_text_embeds(prompts, NEGATIVE), latents=lat.clone(), **kw)
    latents_ref = model.produce_latents(embeds(prompts, NEGATIVE), latents=lat.clone(), **kw)
    assert torch.equal(latents, latents_ref), "rich-text pass latents"
