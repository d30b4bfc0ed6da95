"""CPU: checkpoints in the diffusers on-disk layout load into the rtti_b200 modules (rtti_b200/loading.py) — the drop-in claim
for real weights (the reference downloads them from the hub: models/region_diffusion.py:24-33, region_diffusion_sdxl.py:105-120)."""
import json
import os

import pytest
import torch

from oracle import unet_oracle as uo
from rtti_b200 import loading
from rtti_b200.vae import AutoencoderKLDecoder, VAEConfig

safetensors = pytest.importorskip("safetensors.torch")


def test_unet_directory_roundtrip(tmp_path):
    cfg = uo.tiny_xl_config()
    sd = {k: v.contiguous() for k, v in uo.make_state_dict(cfg, 3).items()}     # reference (= diffusers) parameter names
    folder = tmp_path / "unet"
    folder.mkdir()
    (folder / "config.json").write_text(json.dumps(cfg.__dict__))
    safetensors.save_file(sd, str(folder / "diffusion_pytorch_model.safetensors"))
    unet = loading.load_unet(str(folder), "cpu")
    got = dict(unet.named_parameters())
    assert len(got) > 50
    # tensors that finalize() does not fold into others survive the trip exactly up to its fp16 cast
    for name in ("conv_in.weight", "time_embedding.linear_1.weight", "mid_block.resnets.0.norm1.weight",
                 "down_blocks.1.attentions.0.transformer_blocks.0.attn2.to_out.0.weight"):
        assert torch.equal(got[name].float(), sd[name].half().float()), name
    del sd["conv_out.bias"]
    safetensors.save_file(sd, str(folder / "diffusion_pytorch_model.safetensors"))
    with pytest.raises(RuntimeError, match="missing"):
        loading.load_unet(str(folder), "cpu")


def test_vae_directory_with_pre_0_18_attention_names(tmp_path):
    cfg = VAEConfig(block_out_channels=(32, 32, 64, 64))
    ref = AutoencoderKLDecoder(cfg).init_synthetic(seed=1)
    sd = {}
    for k, v in ref.state_dict().items():
        for new, old in (("to_q", "query"), ("to_k", "key"), ("to_v", "value"), ("to_out.0", "proj_attn")):
            k = k.replace(f".attentions.0.{new}.", f".attentions.0.{old}.")
        sd[k] = v.contiguous()
    sd["encoder.conv_in.weight"] = torch.zeros(4, 3, 3, 3)      # encoder tensors are ignored
    folder = tmp_path / "vae"
    folder.mkdir()
    (folder / "config.json").write_text(json.dumps({"block_out_channels": [32, 32, 64, 64], "scaling_factor": 0.13025}))
    safetensors.save_file(sd, str(folder / "diffusion_pytorch_model.safetensors"))
    vae = loading.load_vae(str(folder), "cpu", 0.18215)
    assert vae.config.scaling_factor == 0.13025
    for (k, a), (_, b) in zip(sorted(vae.state_dict().items()), sorted(ref.state_dict().items())):
        assert torch.equal(a.float(), b.float()), k


def test_missing_directory_message():
    with pytest.raises(FileNotFoundError, match="no network access"):
        loading.load_sdxl_components("/nonexistent/sdxl", "cpu")


def _tiny_clip_dir(root):
    """Tokenizer(s) + text encoder(s) in the diffusers on-disk layout with a 20-token BPE vocabulary and random 3-layer
    CLIP text models (the real ones need the hub)."""
    transformers = pytest.importorskip("transformers")
    from transformers import CLIPTextConfig, CLIPTextModel, CLIPTextModelWithProjection, CLIPTokenizer

    def make_tok(path):
        os.makedirs(path)
        chars = list("abcdret")
        vocab = {}
        for t in chars + [c + "</w>" for c in chars] + ["re", "red</w>", "ca", "cat</w>", "<|startoftext|>", "<|endoftext|>"]:
            vocab.setdefault(t, len(vocab))
        json.dump(vocab, open(os.path.join(path, "vocab.json"), "w"))
        open(os.path.join(path, "merges.txt"), "w").write("#version: 0.2\nr e\nre d</w>\nc a\nca t</w>\n")
        tok = CLIPTokenizer(os.path.join(path, "vocab.json"), os.path.join(path, "merges.txt"), model_max_length=77)
        tok.save_pretrained(path)
        return tok

    tok = make_tok(os.path.join(root, "tokenizer"))
    make_tok(os.path.join(root, "tokenizer_2"))
    torch.manual_seed(0)
    cfg = CLIPTextConfig(vocab_size=len(tok), hidden_size=32, intermediate_size=64, num_hidden_layers=3, num_attention_heads=2,
                         max_position_embeddings=77, projection_dim=24, bos_token_id=tok.bos_token_id, eos_token_id=tok.eos_token_id)
    CLIPTextModel(cfg).save_pretrained(os.path.join(root, "text_encoder"))
    CLIPTextModelWithProjection(cfg).save_pretrained(os.path.join(root, "text_encoder_2"))
    return transformers


def test_clip_text_encoders_follow_the_reference_encode_prompt(tmp_path):
    """loading.ClipTextEncoders against the steps of the reference's encode_prompt (models/region_diffusion_sdxl.py:326-440):
    per encoder `hidden_states[-2]`, concatenated along the channel axis; pooled = output [0] of the SECOND encoder (the
    projected text embedding); negative_prompt=None + force_zeros_for_empty_prompt -> zero negative / negative-pooled
    embeddings (:368-373), an explicit '' is encoded. SD1.5: last hidden state, [uncond, cond...] (region_diffusion.py:47-67)."""
    _tiny_clip_dir(str(tmp_path))
    enc = loading.ClipTextEncoders(str(tmp_path), "cpu", xl=True)
    prompts = ["a red cat", "a cat"]
    pe, ne, pp, npool = enc.encode(prompts, None, "cpu")
    assert pe.shape == (2, 77, 64) and ne.shape == (1, 77, 64) and pp.shape == (2, 24) and npool.shape == (1, 24)
    assert float(ne.abs().max()) == 0.0 and float(npool.abs().max()) == 0.0
    with torch.no_grad():
        want, pooled = [], None
        for tok, model in ((enc.tokenizer, enc.text_encoder), (enc.tokenizer_2, enc.text_encoder_2)):
            ids = tok(prompts, padding="max_length", max_length=tok.model_max_length, truncation=True, return_tensors="pt").input_ids
            out = model(ids, output_hidden_states=True)
            pooled = out[0]
            want.append(out.hidden_states[-2])
        assert torch.equal(pe, torch.cat(want, -1)) and torch.equal(pp, pooled) and pooled.shape[-1] == 24
    pe2, ne2, _, npool2 = enc.encode(prompts[:1], [""], "cpu")
    assert float(ne2.abs().max()) > 0 and float(npool2.abs().max()) > 0 and torch.equal(pe2, pe[:1])
    _, ne3, _, _ = enc.encode(prompts[:1], None, "cpu", force_zeros_for_empty_prompt=False)
    assert torch.equal(ne3, ne2)
    sd = loading.ClipTextEncoders(str(tmp_path), "cpu", xl=False)
    both = sd.encode_pair(prompts, [""], "cpu")
    assert both.shape == (3, 77, 32)
    with torch.no_grad():
        ids = sd.tokenizer([""], padding="max_length", max_length=77, truncation=True, return_tensors="pt").input_ids
        assert torch.equal(both[:1], sd.text_encoder(ids)[0])
