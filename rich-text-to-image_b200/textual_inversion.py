"""Textual-inversion embeddings added to the CLIP tokenizers and token-embedding tables.

An embedding of n vectors becomes n new tokens `tok`, `tok_1` ... `tok_{n-1}` (diffusers' multi-vector convention) and
n new rows of the text encoder's token-embedding table, written in the encoder's dtype. A prompt is expanded before it
is tokenized: every `tok` in it becomes "tok tok_1 ... tok_{n-1}". Only the prompt embeddings change, so a denoising
step runs the same kernels at the same speed. The tokens are added with `normalized=False`, so they match the prompt
text case for case.

Formats (a local file, a local directory, a state dict, or a list of them):
  * diffusers `learned_embeds.bin` / `.safetensors`: {token: [d] or [n, d]};
  * A1111 `.pt`: {"string_to_param": {"*": [n, d]}, "name": ...}, and the bare {"emb_params": [n, d]} `.safetensors`;
  * SDXL: {"clip_l": [n, 768], "clip_g": [n, 1280]}, into `text_encoder` and `text_encoder_2`.
The token is, in order: the `token` argument, the token or `name` stored in the file, the file name without suffix.

The rich-text helpers (richtext_utils.py) find token positions with `tokenize` below, which gives the expanded sequence
the text encoder sees, so spans after a multi-vector token keep their true positions.
"""
import copy
import os
import re

import torch

_DIR_NAMES = ("learned_embeds.safetensors", "learned_embeds.bin")


def _vector_tokens(tokenizer):
    """Every added, non-special token of `tokenizer` -> the tokens its vectors occupy ([tok, tok_1, ...]).
    Empty for a tokenizer without added tokens, which then tokenizes exactly as before."""
    added = getattr(tokenizer, "added_tokens_encoder", None)
    if not added:
        return {}
    special = set(tokenizer.all_special_tokens)
    added = [t for t in added if t not in special]
    names = set(added)
    out = {}
    for t in added:
        seq = [t]
        while f"{t}_{len(seq)}" in names:
            seq.append(f"{t}_{len(seq)}")
        out[t] = seq
    return out


def _pattern(groups):
    # longest first: at one position `tok_1` wins over `tok`, as in the tokenizer's own added-token split
    return re.compile("|".join(re.escape(t) for t in sorted(groups, key=len, reverse=True)))


def expand_prompt(tokenizer, text):
    """`text` with every multi-vector token `tok` written out as "tok tok_1 ... tok_{n-1}" (diffusers'
    maybe_convert_prompt); unchanged when the tokenizer has no added tokens."""
    groups = _vector_tokens(tokenizer)
    if not groups:
        return text
    return _pattern(groups).sub(lambda m: " ".join(groups[m.group()]), text)


def tokenize(tokenizer, text):
    """The BPE tokens of `text` without BOS / EOS, as the text encoder sees them: each added token kept whole and
    expanded to its n tokens, the text between them split by the tokenizer's BPE (`_tokenize` where the tokenizer has
    it, else `tokenize`)."""
    bpe = tokenizer._tokenize if hasattr(tokenizer, "_tokenize") else tokenizer.tokenize
    groups = _vector_tokens(tokenizer)
    if not groups:
        return bpe(text)
    out, pos = [], 0
    for m in _pattern(groups).finditer(text):
        out += bpe(text[pos:m.start()]) + groups[m.group()]
        pos = m.end()
    return out + bpe(text[pos:])


def _read(source, weight_name):
    """(state dict, file name without suffix or None) of one source."""
    if isinstance(source, dict):
        return source, None
    if not isinstance(source, (str, os.PathLike)):
        raise ValueError(f"textual inversion: {type(source).__name__} is not a path or a state dict")
    path = os.fspath(source)
    if os.path.isdir(path):
        names = [weight_name] if weight_name else _DIR_NAMES
        found = [os.path.join(path, n) for n in names if os.path.isfile(os.path.join(path, n))]
        if not found:
            raise ValueError(f"textual inversion: the directory {path!r} holds none of {list(names)}; pass weight_name=")
        path = found[0]
    elif not os.path.isfile(path):
        raise ValueError(f"textual inversion: {path!r} is not a local file or directory. Hub downloads are not "
                         "supported: download the embedding once and pass its path")
    if path.endswith(".safetensors"):
        from safetensors.torch import load_file
        sd = load_file(path)
    else:
        sd = torch.load(path, map_location="cpu", weights_only=True)
    if not isinstance(sd, dict):
        raise ValueError(f"textual inversion: {path!r} holds a {type(sd).__name__}, not a state dict")
    return sd, os.path.splitext(os.path.basename(path))[0]


def _parse(sd, token, stem):
    """(token, [n, d] fp32 tensors: one per text encoder) of one state dict."""
    keys = sorted(sd)
    name = None
    if "clip_l" in sd or "clip_g" in sd:
        if keys != ["clip_g", "clip_l"]:
            raise ValueError(f"textual inversion: an SDXL embedding holds clip_l and clip_g; got keys {keys}")
        vecs = [sd["clip_l"], sd["clip_g"]]
    elif "string_to_param" in sd:
        vecs = [dict(sd["string_to_param"]).get("*")]
        name = sd.get("name")
    elif keys == ["emb_params"]:
        vecs = [sd["emb_params"]]
    elif len(sd) == 1:
        name, v = next(iter(sd.items()))
        vecs = [v]
    else:
        raise ValueError(f"textual inversion: unknown format with keys {keys[:8]}; expected {{token: tensor}} "
                         "(diffusers), string_to_param / emb_params (A1111) or clip_l / clip_g (SDXL)")
    token = token or name or stem
    if not isinstance(token, str) or not token:
        raise ValueError("textual inversion: the embedding names no token; pass token=")
    out = []
    for v in vecs:
        if not torch.is_tensor(v) or v.dim() not in (1, 2) or not v.is_floating_point() or v.numel() == 0:
            raise ValueError(f"textual inversion {token!r}: expected a float tensor [d] or [n, d], got "
                             f"{tuple(v.shape) if torch.is_tensor(v) else type(v).__name__}")
        out.append(v.detach().reshape(-1, v.shape[-1]).float())
    return token, out


def _describe(widths):
    if len(widths) == 2:
        return f"clip_l [n, {widths[0]}] and clip_g [n, {widths[1]}]"
    return f"one [n, {widths[0]}] embedding"


def _check_widths(token, vecs, encoders):
    widths = [e.get_input_embeddings().weight.shape[1] for e in encoders]
    got = [v.shape[1] for v in vecs]
    if got != widths:
        raise ValueError(f"textual inversion {token!r}: the text encoders of this model need {_describe(widths)} "
                         f"(hidden size {', '.join(map(str, widths))}); the embedding holds {_describe(got)}")
    if len({v.shape[0] for v in vecs}) != 1:
        raise ValueError(f"textual inversion {token!r}: clip_l and clip_g hold {[v.shape[0] for v in vecs]} vectors")


def _resize(encoder, rows):
    """resize_token_embeddings without touching the caller's random streams (it initialises the new rows)."""
    dev = encoder.get_input_embeddings().weight.device
    with torch.random.fork_rng(devices=[dev] if dev.type == "cuda" else []):
        encoder.resize_token_embeddings(rows, mean_resizing=False)


class TextualInversionLoaderMixin:
    """load_textual_inversion / unload_textual_inversion of the samplers. The sampler gives its (tokenizer, text
    encoder) pairs, in the order clip_l, clip_g, through `_textual_inversion_components()`."""

    _ti_tokens = None   # the token of every embedding loaded
    _ti_saved = None    # per pair: (tokenizer, its state before the first load, encoder, table rows, eos_token_id)

    def _textual_inversion_components(self):
        raise NotImplementedError

    def load_textual_inversion(self, pretrained_model_name_or_path, token=None, weight_name=None):
        """Add textual-inversion embeddings to the tokenizers and text encoders. `pretrained_model_name_or_path`: a local
        file, a local directory (its file `weight_name`, else learned_embeds.safetensors or learned_embeds.bin),
        a state dict, or a list of them; `token`: one token, or a list with one per embedding. Raises ValueError for a
        source that is not local, an unknown format, an embedding whose width does not fit a text encoder, or a token
        that is already in the vocabulary or already loaded; nothing is changed then."""
        pairs = self._textual_inversion_components()
        if not pairs:
            raise RuntimeError("no text encoder loaded: textual inversion needs the tokenizer and the text encoder")
        sources = list(pretrained_model_name_or_path) if isinstance(pretrained_model_name_or_path, (list, tuple)) \
            else [pretrained_model_name_or_path]
        tokens = list(token) if isinstance(token, (list, tuple)) else [token] * len(sources)
        if len(tokens) != len(sources) or (isinstance(token, str) and len(sources) > 1):
            raise ValueError(f"textual inversion: {len(sources)} embeddings need {len(sources)} tokens, got {token!r}")
        loaded = set(self._ti_tokens or ())
        new, pending = [], set()
        for src, tok in zip(sources, tokens):
            sd, stem = _read(src, weight_name)
            tok, vecs = _parse(sd, tok, stem)
            _check_widths(tok, vecs, [e for _, e in pairs])
            names = [tok] + [f"{tok}_{i}" for i in range(1, vecs[0].shape[0])]
            if tok in loaded:
                raise ValueError(f"textual inversion: the token {tok!r} is already loaded; call "
                                 "unload_textual_inversion() first or choose another token")
            for tokenizer, _ in pairs:
                vocab = tokenizer.get_vocab()
                clash = [n for n in names if n in vocab or n in pending]
                if clash:
                    raise ValueError(f"textual inversion: the token {clash[0]!r} is already in the tokenizer's "
                                     "vocabulary; choose another token")
            loaded.add(tok)
            pending.update(names)
            new.append((names, vecs))
        self._add(pairs, new)
        self._ti_tokens = loaded

    @torch.no_grad()
    def _add(self, pairs, new):
        from transformers import AddedToken
        if self._ti_saved is None:
            self._ti_saved = [(tz, copy.deepcopy(tz.__dict__), enc, enc.get_input_embeddings().num_embeddings,
                               enc.text_model.eos_token_id) for tz, enc in pairs]
        for j, (tz, enc) in enumerate(pairs):
            # eos_token_id == 2 is the legacy CLIP config, which pools at the largest token id: with added ids past EOS
            # that would be an added token. Pooling at the first EOS picks the same position for every other prompt.
            if enc.text_model.eos_token_id == 2:
                enc.text_model.eos_token_id = tz.eos_token_id
            for names, vecs in new:
                tz.add_tokens([AddedToken(n, normalized=False) for n in names])
                ids = tz.convert_tokens_to_ids(names)
                emb = enc.get_input_embeddings()
                if max(ids) >= emb.num_embeddings:
                    _resize(enc, max(emb.num_embeddings, len(tz)))
                    emb = enc.get_input_embeddings()
                emb.weight[ids] = vecs[j].to(emb.weight.device, emb.weight.dtype)

    def unload_textual_inversion(self):
        """Remove every loaded embedding: the tokenizers, token-embedding tables and pooling rule return to their state
        before the first load, bit for bit. A merged LoRA stays merged. No-op when none is loaded."""
        if self._ti_saved is None:
            return
        for tz, state, enc, rows, eos in self._ti_saved:
            # transformers has no call that removes added tokens: the tokenizer's own state is put back in place, so
            # every reference to this tokenizer object sees the original vocabulary
            tz.__dict__.clear()
            tz.__dict__.update(state)
            _resize(enc, rows)
            enc.text_model.eos_token_id = eos
        self._ti_saved = self._ti_tokens = None
