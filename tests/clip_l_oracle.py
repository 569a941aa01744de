"""TEST INFRASTRUCTURE ONLY -- CPU fp32 oracle for the OpenAI CLIP ViT-L/14 text model as VideoCrafter's FrozenCLIPEmbedder
drives it (videocrafter/lvdm/models/modules/condition_modules.py:15-40: transformers' CLIPTextModel, `last_hidden_state`
of `self.transformer(input_ids=tokens)`, no attention mask).

Restated with transformers' parameter names (relative to the CLIPTextModel):
    x = token_embedding(tokens) + position_embedding(arange(L))
    x = x + out_proj(attn(layer_norm1(x)))       q, k, v: separate projections with bias; q scaled by d^-0.5; causal mask
    x = x + fc2(quick_gelu(fc1(layer_norm2(x))))  quick_gelu(x) = x * sigmoid(1.702 x)
for every encoder layer, then final_layer_norm (eps 1e-5 everywhere).  Kept apart from oracle/clip_oracle.py (the OpenCLIP
ViT-H-14 tower).  Pinned by tests/test_clip_l.py against tests/golden/clip_l.pt, which scripts/make_golden_clip_l.py writes
from the reference's own FrozenCLIPEmbedder class, and against a live transformers CLIPTextModel when one is installed.
"""
from dataclasses import dataclass
from typing import Dict, Tuple

import torch
import torch.nn.functional as F


@dataclass
class ClipLConfig:
    width: int = 768
    heads: int = 12
    layers: int = 12
    context: int = 77
    vocab: int = 49408


NARROW = ClipLConfig(width=128, heads=2, layers=3, context=77, vocab=300)


def clip_l_param_specs(cfg: ClipLConfig) -> Dict[str, Tuple[int, ...]]:
    W = cfg.width
    s = {'text_model.embeddings.token_embedding.weight': (cfg.vocab, W),
         'text_model.embeddings.position_embedding.weight': (cfg.context, W)}
    for i in range(cfg.layers):
        p = f'text_model.encoder.layers.{i}'
        for n in ('q_proj', 'k_proj', 'v_proj', 'out_proj'):
            s.update({f'{p}.self_attn.{n}.weight': (W, W), f'{p}.self_attn.{n}.bias': (W,)})
        s.update({p + '.layer_norm1.weight': (W,), p + '.layer_norm1.bias': (W,), p + '.layer_norm2.weight': (W,),
                  p + '.layer_norm2.bias': (W,), p + '.mlp.fc1.weight': (4 * W, W), p + '.mlp.fc1.bias': (4 * W,),
                  p + '.mlp.fc2.weight': (W, 4 * W), p + '.mlp.fc2.bias': (W,)})
    s.update({'text_model.final_layer_norm.weight': (W,), 'text_model.final_layer_norm.bias': (W,)})
    return s


@torch.no_grad()
def clip_l_text_forward(Wt: Dict[str, torch.Tensor], cfg: ClipLConfig, tokens):
    """tokens [B, context] int -> last_hidden_state [B, context, width]."""
    x = F.embedding(tokens.long(), Wt['text_model.embeddings.token_embedding.weight'])
    x = x + Wt['text_model.embeddings.position_embedding.weight'][:tokens.shape[1]]
    B, L, W = x.shape
    H, d = cfg.heads, W // cfg.heads
    mask = torch.full((L, L), float('-inf'), dtype=x.dtype, device=x.device).triu_(1)
    for i in range(cfg.layers):
        p = f'text_model.encoder.layers.{i}'
        h = F.layer_norm(x, (W,), Wt[p + '.layer_norm1.weight'], Wt[p + '.layer_norm1.bias'], 1e-5)
        q, k, v = (F.linear(h, Wt[f'{p}.self_attn.{n}.weight'], Wt[f'{p}.self_attn.{n}.bias']).reshape(B, L, H, d).permute(0, 2, 1, 3)
                   for n in ('q_proj', 'k_proj', 'v_proj'))
        a = torch.softmax((q * (d ** -0.5)) @ k.transpose(-1, -2) + mask, dim=-1) @ v
        a = a.permute(0, 2, 1, 3).reshape(B, L, W)
        x = x + F.linear(a, Wt[p + '.self_attn.out_proj.weight'], Wt[p + '.self_attn.out_proj.bias'])
        h = F.layer_norm(x, (W,), Wt[p + '.layer_norm2.weight'], Wt[p + '.layer_norm2.bias'], 1e-5)
        h = F.linear(h, Wt[p + '.mlp.fc1.weight'], Wt[p + '.mlp.fc1.bias'])
        h = h * torch.sigmoid(1.702 * h)
        x = x + F.linear(h, Wt[p + '.mlp.fc2.weight'], Wt[p + '.mlp.fc2.bias'])
    return F.layer_norm(x, (W,), Wt['text_model.final_layer_norm.weight'], Wt['text_model.final_layer_norm.bias'], 1e-5)


def layout_digest(state_dict):
    """sha256 of a state dict's {key: shape} in canonical (sorted JSON) form: equal digests <=> equal layouts."""
    import hashlib
    import json
    return hashlib.sha256(json.dumps(sorted((k, list(v.shape)) for k, v in state_dict.items())).encode()).hexdigest()


# VideoCrafter LatentDiffusion at a tiny size whose text encoder is the NARROW tower: the keyword arguments of
# t2v_b200.videocrafter.LatentDiffusion; scripts/make_golden_clip_l.py builds the reference class with the same sizes
# (the rest of base_t2v/model_config.yaml unchanged) and stores its state-dict layout.
TINY_LDM = dict(unet_config=dict(model_channels=64, context_dim=NARROW.width, temporal_length=4), image_size=[8, 8], video_length=4)


# A tiny BPE vocabulary in the CLIP tokenizer's file format, for building a transformers CLIPTokenizer offline.  Every
# lowercase letter and two-letter word piece is a token; the last two ids are <|startoftext|> / <|endoftext|>, as in the
# OpenAI vocabulary (49406 / 49407 of 49408).
def synthetic_vocab(vocab=300):
    import string
    toks = ['!', ',', '.']
    toks += list(string.ascii_lowercase) + [c + '</w>' for c in string.ascii_lowercase]
    merges = []
    for a in 'aeiost':
        for b in 'nrt':
            merges.append((a, b + '</w>'))
            toks.append(a + b + '</w>')
    toks = toks[:vocab - 2]
    toks += [f'<unused{i}>' for i in range(vocab - 2 - len(toks))]
    toks += ['<|startoftext|>', '<|endoftext|>']
    return {t: i for i, t in enumerate(toks)}, merges


def write_synthetic_tokenizer(directory, vocab=300):
    """vocab.json + merges.txt for `CLIPTokenizer(vocab_file, merges_file)` (pad token: <|endoftext|>)."""
    import json
    import os
    enc, merges = synthetic_vocab(vocab)
    vf, mf = os.path.join(directory, 'vocab.json'), os.path.join(directory, 'merges.txt')
    with open(vf, 'w') as f:
        json.dump(enc, f)
    with open(mf, 'w') as f:
        f.write('#version: 0.2\n' + ''.join(f'{a} {b}\n' for a, b in merges))
    return vf, mf


class WordTokenizer(object):
    """A plain `.encode(str) -> list[int]` tokenizer (the shape of open_clip's SimpleTokenizer): one id per character of
    each lowercase word, ids from the synthetic vocabulary; used where no transformers tokenizer is at hand."""

    def __init__(self, vocab=300):
        self.encoder = synthetic_vocab(vocab)[0]

    def encode(self, text):
        out = []
        for w in text.lower().split():
            w = ''.join(c for c in w if c in 'abcdefghijklmnopqrstuvwxyz')
            out += [self.encoder[c] for c in w[:-1]] + [self.encoder[w[-1] + '</w>']] if w else []
        return out
