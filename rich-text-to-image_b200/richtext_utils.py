"""Rich-text (Quill delta JSON) -> region prompts / token ids / format dict.

Host-side preparation around the hot path; same function names, argument meaning and return values as the
reference's utils/richtext_utils.py (parse_json :74-136, get_region_diffusion_input :139-185,
get_attention_control_input :188-209, get_gradient_guidance_input :212-234, hex_to_rgb :30-44,
find_nearest_color :47-56, font2style :59-71, seed_everything :22-27), but device-agnostic: tensors are
created on `device` (default: CUDA when available) instead of hard-coded `.cuda()`.
"""
import os
import random

import numpy as np
import torch

from .textual_inversion import tokenize

COLORS = {
    "brown": (165, 42, 42), "red": (255, 0, 0), "pink": (253, 108, 158), "orange": (255, 165, 0),
    "yellow": (255, 255, 0), "purple": (128, 0, 128), "green": (0, 128, 0), "blue": (0, 0, 255),
    "white": (255, 255, 255), "gray": (128, 128, 128), "black": (0, 0, 0),
}

FONT_STYLES = {
    "mirza": "Claud Monet, impressionism, oil on canvas",
    "roboto": "Ukiyoe",
    "cursive": "Cyber Punk, futuristic, blade runner, william gibson, trending on artstation hq",
    "sofia": "Pop Art, masterpiece, andy warhol",
    "slabo": "Vincent Van Gogh",
    "inconsolata": "Pixel Art, 8 bits, 16 bits",
    "ubuntu": "Rembrandt",
    "Monoton": "neon art, colorful light, highly details, octane render",
    "Akronim": "Abstract Cubism, Pablo Picasso",
}


def _default_device():
    return torch.device("cuda" if torch.cuda.is_available() else "cpu")


def seed_everything(seed):
    random.seed(seed)
    os.environ["PYTHONHASHSEED"] = str(seed)
    np.random.seed(seed)
    torch.manual_seed(seed)
    if torch.cuda.is_available():
        torch.cuda.manual_seed(seed)


def find_nearest_color(rgb):
    """Name of the palette colour closest (L2 in [0,1]^3) to `rgb` ([1,3,1,1] tensor in [0,1] or 0-255 triple)."""
    if isinstance(rgb, (list, tuple)):
        rgb = torch.tensor(rgb, dtype=torch.float32)[None, :, None, None] / 255.0
    v = rgb.detach().float().cpu().reshape(3)
    names = list(COLORS)
    palette = torch.tensor([COLORS[n] for n in names], dtype=torch.float32) / 255.0
    return names[int(torch.argmin((palette - v).norm(dim=1)))]


def hex_to_rgb(hex_string, return_nearest_color=False, device=None):
    h = hex_string.lstrip("#")
    rgb = torch.tensor([int(h[i:i + 2], 16) for i in (0, 2, 4)], dtype=torch.float32)[None, :, None, None] / 255.0
    out = rgb.to(device or _default_device())
    if return_nearest_color:
        return out, find_nearest_color(rgb)
    return out


def font2style(font):
    return FONT_STYLES[font]


def _font_size_of(attrs):
    if "size" not in attrs:
        return 1
    px = float(attrs["size"][:-2]) / 3.0
    return -px if "strike" in attrs else px


def parse_json(json_str, device=None):
    """Quill delta -> (base prompt, style prompts, footnote prompts, footnote target spans, colour spans,
    colour names, colour RGBs, [(span, font size)], use_grad_guidance)."""
    base = ""
    styles, footnotes, footnote_targets = [], [], []
    color_spans, color_rgbs, color_names, sizes = [], [], [], []
    last_style, use_grad = None, False
    for op in json_str["ops"]:
        text = op["insert"].rstrip("\n")
        base += text
        if text == " ":
            continue
        attrs = op.get("attributes")
        if not attrs:
            continue
        if "font" in attrs:
            style = font2style(attrs["font"])
            if style == last_style:  # adjacent spans of one style merge into one region prompt
                head = styles[-1].split("in the style of")[0]
                styles[-1] = f"{head} {text} in the style of {style}"
            else:
                styles.append(f"{text} in the style of {style}")
            last_style = style
        else:
            last_style = None
        if "link" in attrs:
            footnotes.append(attrs["link"])
            footnote_targets.append(text)
        size = _font_size_of(attrs)
        if "color" in attrs:
            use_grad = True
            rgb, name = hex_to_rgb(attrs["color"], True, device=device)
            # the reference compares against `prev_color_rgb`, which it never updates (richtext_utils.py:84,124):
            # consecutive spans of one colour therefore stay separate regions; kept.
            color_rgbs.append(rgb)
            color_names.append(name)
            color_spans.append(text)
        if size != 1:
            sizes.append([text, size])
    return base, styles, footnotes, footnote_targets, color_spans, color_names, color_rgbs, sizes, use_grad


def _positions(tokenizer, base_tokens, text):
    """1-based index in the base prompt of the FIRST occurrence of each BPE token of `text`. A textual-inversion
    token of n vectors is n tokens here, as in the encoded prompt."""
    return [base_tokens.index(tok) + 1 for tok in tokenize(tokenizer, text)]


def _with_rest(groups, n_tokens):
    taken = {i for g in groups for i in g}
    groups = groups + [[i for i in range(1, n_tokens + 1) if i not in taken]]
    return [torch.LongTensor(g) for g in groups]


def get_region_diffusion_input(model, base_text_prompt, style_text_prompts, footnote_text_prompts,
                               footnote_target_tokens, color_text_prompts, color_names):
    """Algorithm 1 of the paper: region prompts [styles..., footnotes..., colours..., base] and the
    1-based token ids each region is anchored on (last entry: all remaining tokens)."""
    tok = model.tokenizer
    base_tokens = tokenize(tok, base_text_prompt)
    prompts, ids = [], []
    for p in style_text_prompts:
        prompts.append(p)
        ids.append(_positions(tok, base_tokens, p.split("in the style of")[0]))
    for note, target in zip(footnote_text_prompts, footnote_target_tokens):
        prompts.append(note)
        ids.append(_positions(tok, base_tokens, target))
    for span, name in zip(color_text_prompts, color_names):
        prompts.append(name + " " + span)
        ids.append(_positions(tok, base_tokens, span))
    prompts.append(base_text_prompt)
    return prompts, _with_rest(ids, len(base_tokens)), base_tokens


def get_attention_control_input(model, base_tokens, size_text_prompts_and_sizes, device=None):
    pos, sizes = [], []
    for text, size in size_text_prompts_and_sizes:
        for p in _positions(model.tokenizer, base_tokens, text):
            pos.append(p)
            sizes.append(size)
    if not pos:
        return {"word_pos": None, "font_size": None}
    device = device or _default_device()
    return {"word_pos": torch.LongTensor(pos).to(device), "font_size": torch.FloatTensor(sizes).to(device)}


def get_gradient_guidance_input(model, base_tokens, color_text_prompts, color_rgbs, text_format_dict,
                                guidance_start_step=999, color_guidance_weight=1):
    ids = [_positions(model.tokenizer, base_tokens, span) for span in color_text_prompts]
    text_format_dict["target_RGB"] = color_rgbs
    text_format_dict["guidance_start_step"] = guidance_start_step
    text_format_dict["color_guidance_weight"] = color_guidance_weight
    return text_format_dict, _with_rest(ids, len(base_tokens))
