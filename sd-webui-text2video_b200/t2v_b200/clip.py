"""`FrozenOpenCLIPEmbedder` -- the text conditioning step in front of the denoising loop (reference:
scripts/modelscope/clip_hardcode.py:59-422), with the OpenCLIP ViT-H-14 text transformer on the GPU-native library.

Kept from the reference: the class name, `.model` holding open_clip's parameter tree (`model.token_embedding`,
`model.positional_embedding`, `model.transformer.resblocks[i].{ln_1, attn, ln_2, mlp.c_fc, mlp.c_proj}`, `model.ln_final`,
so `load_state_dict` of the text side of open_clip_pytorch_model.bin works and the Stable-LoRA code finds
`clip_encoder.model.transformer`, lora_webui.py:187), `layer='penultimate'`, 75-token prompt chunks framed by
<start_of_text> / <end_of_text>, padding after the first end token, per-token emphasis multipliers with the mean restored
(`process_tokens` :397-422), `encode(text) -> [B, 77 * chunks, 1024]`.

Not here: the BPE vocabulary (open_clip ships it; there is no copy offline) -- pass `tokenizer` (anything with
`.encode(str) -> list[int]`; `open_clip.tokenizer._tokenizer` when the package is installed) -- and the webui's prompt-attention
syntax parser (`modules.prompt_parser`, used when importable; otherwise every token has weight 1).

`FrozenCLIPEmbedder` is VideoCrafter's text conditioning (videocrafter/lvdm/models/modules/condition_modules.py:15-40): the
OpenAI CLIP ViT-L/14 text model with transformers' parameter names, on the same library tower (arch 1).
"""
import math
import os

import torch
import torch.nn as nn

from . import _lib
from .modules import _NativeModule, _Holder


class _InProj(nn.Module):
    """Parameter holder with nn.MultiheadAttention's names (in_proj_weight / in_proj_bias / out_proj)."""

    def __init__(self, width):
        super().__init__()
        self.in_proj_weight = nn.Parameter(torch.zeros(3 * width, width))
        self.in_proj_bias = nn.Parameter(torch.zeros(3 * width))
        self.out_proj = nn.Linear(width, width)


class _NativeTextTower(_NativeModule):
    """A CLIP text transformer whose arithmetic runs in libt2v_b200.so (csrc/clip.cu); subclasses build the parameter tree,
    which may hold checkpoint tensors the library does not use (they are not shipped)."""

    def _create(self, width, heads, layers, layers_run, context, vocab, arch):
        self.width, self.heads, self.layers, self.layers_run, self.context, self.vocab = width, heads, layers, layers_run, context, vocab
        self._open('clip', _lib.ClipConfigC(width, heads, layers_run, context, vocab, arch))

    @torch.no_grad()
    def encode_tokens(self, tokens, out_dtype=torch.float32):
        """tokens [B, context] integer tensor -> ln_final(transformer(...)) [B, context, width]."""
        self.sync_weights()
        tokens = tokens.to('cuda', torch.int32).contiguous()
        B, L = tokens.shape
        if L != self.context:
            raise ValueError(f'expected {self.context} tokens per chunk, got {L}')
        out = torch.empty((B, L, self.width), device='cuda', dtype=out_dtype)
        _lib.check(_lib.lib().t2v_clip_encode(self._handle, _lib.ptr(tokens), _lib.ptr(out), int(out_dtype == torch.float32), B,
                                              _lib.stream_ptr()), 'clip_encode')
        return out


class _TextTower(_NativeTextTower):
    """`model` of the embedder: open_clip's text-side module tree; arithmetic in libt2v_b200.so (csrc/clip.cu)."""

    def __init__(self, width=1024, heads=16, layers=24, layers_run=23, context=77, vocab=49408):
        super().__init__()
        self._create(width, heads, layers, layers_run, context, vocab, arch=0)
        self.token_embedding = nn.Embedding(vocab, width)
        self.positional_embedding = nn.Parameter(torch.zeros(context, width))
        self.transformer = _Holder()
        blocks = []
        for _ in range(layers):                      # all 24 blocks exist (checkpoint keys); only the first layers_run are shipped
            b = _Holder()
            b.ln_1 = nn.LayerNorm(width)
            b.attn = _InProj(width)
            b.ln_2 = nn.LayerNorm(width)
            b.mlp = _Holder()
            b.mlp.c_fc = nn.Linear(width, 4 * width)
            b.mlp.c_proj = nn.Linear(4 * width, width)
            blocks.append(b)
        self.transformer.resblocks = nn.ModuleList(blocks)
        self.ln_final = nn.LayerNorm(width)
        self.text_projection = nn.Parameter(torch.zeros(width, width))      # in the checkpoint, unused on this path
        self.logit_scale = nn.Parameter(torch.zeros(()))


class _HFEmbeddings(_Holder):
    """`text_model.embeddings` of transformers' CLIPTextModel.  Older transformers releases saved the `position_ids`
    buffer (arange(77)) in checkpoints; it carries no weight, so a state dict that has it loads and the entry is dropped."""

    def __init__(self, vocab, context, width):
        super().__init__()
        self.token_embedding = nn.Embedding(vocab, width)
        self.position_embedding = nn.Embedding(context, width)

    def _load_from_state_dict(self, state_dict, prefix, *a, **kw):
        state_dict.pop(prefix + 'position_ids', None)
        super()._load_from_state_dict(state_dict, prefix, *a, **kw)


class _CLIPTextModel(_NativeTextTower):
    """`transformer` of FrozenCLIPEmbedder: transformers' CLIPTextModel module tree (`text_model.embeddings`,
    `text_model.encoder.layers[i].{layer_norm1, self_attn.{q,k,v,out}_proj, layer_norm2, mlp.fc1, mlp.fc2}`,
    `text_model.final_layer_norm`); arithmetic in libt2v_b200.so (csrc/clip.cu, arch 1)."""

    def __init__(self, width=768, heads=12, layers=12, context=77, vocab=49408):
        super().__init__()
        self._create(width, heads, layers, layers, context, vocab, arch=1)
        tm = _Holder()
        tm.embeddings = _HFEmbeddings(vocab, context, width)
        blocks = []
        for _ in range(layers):
            b = _Holder()
            b.self_attn = _Holder()
            for n in ('k_proj', 'v_proj', 'q_proj', 'out_proj'):
                setattr(b.self_attn, n, nn.Linear(width, width))
            b.layer_norm1 = nn.LayerNorm(width)
            b.mlp = _Holder()
            b.mlp.fc1 = nn.Linear(width, 4 * width)
            b.mlp.fc2 = nn.Linear(4 * width, width)
            b.layer_norm2 = nn.LayerNorm(width)
            blocks.append(b)
        tm.encoder = _Holder()
        tm.encoder.layers = nn.ModuleList(blocks)
        tm.final_layer_norm = nn.LayerNorm(width)
        self.text_model = tm

    def forward(self, input_ids):
        """input_ids [B, context] -> last_hidden_state [B, context, width] fp32 (no attention mask: causal only)."""
        return self.encode_tokens(input_ids)


class PromptChunk(object):
    def __init__(self):
        self.tokens, self.multipliers = [], []


class FrozenOpenCLIPEmbedder(nn.Module):
    LAYERS = ['last', 'penultimate']

    def __init__(self, arch='ViT-H-14', version=None, device='cuda', max_length=77, freeze=True, layer='penultimate', tokenizer=None,
                 width=1024, heads=16, layers=24, vocab=49408):
        super().__init__()
        assert layer in self.LAYERS
        self.layer, self.layer_idx = layer, (0 if layer == 'last' else 1)
        self.model = _TextTower(width, heads, layers, layers - self.layer_idx, max_length, vocab)
        self.device, self.max_length, self.chunk_length = device, max_length, 75
        if tokenizer is None:
            try:
                import open_clip                                         # type: ignore
                tokenizer = open_clip.tokenizer._tokenizer
            except Exception:
                tokenizer = None
        self.tokenizer = tokenizer
        enc = getattr(tokenizer, 'encoder', None) or {}
        self.id_start = enc.get('<start_of_text>', 49406)
        self.id_end = enc.get('<end_of_text>', 49407)
        self.comma_token = enc.get(',</w>', 267)
        self.id_pad = 0
        if version is not None:
            sd = torch.load(version, map_location='cpu')
            self.model.load_state_dict({k: v for k, v in sd.items() if not k.startswith('visual.')}, strict=False)

    # ---- prompt -> chunks of 75 tokens (clip_hardcode.py:146-260, without textual-inversion embeddings)
    def _parse(self, line):
        try:
            from modules import prompt_parser                            # type: ignore
            return prompt_parser.parse_prompt_attention(line)
        except Exception:
            return [[line, 1.0]]

    def tokenize_line(self, line):
        if self.tokenizer is None:
            raise RuntimeError('FrozenOpenCLIPEmbedder needs a BPE tokenizer (open_clip is not installed): pass tokenizer=...')
        parsed = self._parse(line)
        chunks, chunk, token_count = [], PromptChunk(), 0

        def next_chunk():
            nonlocal chunk, token_count
            token_count += len(chunk.tokens)
            pad = self.chunk_length - len(chunk.tokens)
            if pad > 0:
                chunk.tokens += [self.id_end] * pad
                chunk.multipliers += [1.0] * pad
            chunk.tokens = [self.id_start] + chunk.tokens + [self.id_end]
            chunk.multipliers = [1.0] + chunk.multipliers + [1.0]
            chunks.append(chunk)
            chunk = PromptChunk()
        for text, weight in parsed:
            if text == 'BREAK' and weight == -1:
                next_chunk()
                continue
            for tok in self.tokenizer.encode(text):
                if len(chunk.tokens) == self.chunk_length:
                    next_chunk()
                chunk.tokens.append(tok)
                chunk.multipliers.append(weight)
        if len(chunk.tokens) > 0 or len(chunks) == 0:
            next_chunk()
        return chunks, token_count

    def empty_chunk(self):
        c = PromptChunk()
        c.tokens = [self.id_start] + [self.id_end] * (self.chunk_length + 1)
        c.multipliers = [1.0] * (self.chunk_length + 2)
        return c

    def get_target_prompt_token_count(self, token_count):
        return math.ceil(max(token_count, 1) / self.chunk_length) * self.chunk_length

    # ---- transformer
    def encode_with_transformer(self, tokens):
        return self.model.encode_tokens(tokens)

    def process_tokens(self, remade_batch_tokens, batch_multipliers):
        tokens = torch.as_tensor(remade_batch_tokens).clone()
        if self.id_end != self.id_pad:                                   # :408-411: everything after the first end token is padding
            for b in range(tokens.shape[0]):
                idx = list(remade_batch_tokens[b]).index(self.id_end)
                tokens[b, idx + 1:] = self.id_pad
        z = self.encode_with_transformer(tokens)
        m = torch.as_tensor(batch_multipliers, dtype=z.dtype, device=z.device)
        original_mean = z.mean()
        z = z * m.reshape(m.shape + (1,)).expand(z.shape)
        return z * (original_mean / z.mean())

    def forward(self, texts):
        batch_chunks = [self.tokenize_line(t)[0] for t in texts]
        chunk_count = max(len(c) for c in batch_chunks)
        zs = []
        for i in range(chunk_count):
            batch = [chunks[i] if i < len(chunks) else self.empty_chunk() for chunks in batch_chunks]
            zs.append(self.process_tokens([c.tokens for c in batch], [c.multipliers for c in batch]))
        return torch.hstack(zs)

    def encode(self, text):
        return self(text)

    def get_learned_conditioning(self, text):
        return self.encode(text)


def _is_hf_tokenizer(tok):
    return any(c.__module__.startswith('transformers.') for c in type(tok).__mro__)


class FrozenCLIPEmbedder(nn.Module):
    """VideoCrafter's text conditioning (videocrafter/lvdm/models/modules/condition_modules.py:15-40): the OpenAI CLIP
    ViT-L/14 text model, `forward(list of str) -> last_hidden_state [B, 77, 768]` fp32, on the library (csrc/clip.cu, arch 1).

    `transformer` holds transformers' CLIPTextModel parameter tree, so the `cond_stage_model.transformer.text_model.*` keys
    of a VideoCrafter `model.ckpt` load into it.  Prompts are framed as the reference's `tokenizer(text, truncation=True,
    max_length=77, padding='max_length')`: <|startoftext|>, at most 75 BPE ids, <|endoftext|>, then <|endoftext|> (the
    ViT-L/14 tokenizer's pad token) up to 77.

    tokenizer: a transformers CLIPTokenizer (called exactly as the reference calls it), or any object with
    `.encode(str) -> list of int` over the OpenAI CLIP BPE vocabulary (e.g. open_clip's SimpleTokenizer; the framing is
    then done here).  `version` names the model; when it is a local directory (a Hugging Face snapshot of
    openai/clip-vit-large-patch14) the tokenizer and the text weights are read from it.  Nothing is downloaded."""
    ID_START, ID_END = 49406, 49407

    def __init__(self, version='openai/clip-vit-large-patch14', device='cuda', max_length=77, tokenizer=None, width=768, heads=12,
                 layers=12, vocab=49408):
        super().__init__()
        self.transformer = _CLIPTextModel(width, heads, layers, max_length, vocab)
        self.version, self.device, self.max_length = version, device, max_length
        local = isinstance(version, str) and os.path.isdir(version)
        if tokenizer is None and local:
            from transformers import CLIPTokenizer                      # type: ignore
            tokenizer = CLIPTokenizer.from_pretrained(version, local_files_only=True)
        self.tokenizer = tokenizer
        if local:
            self.transformer.load_state_dict(_text_weights(version), strict=True)
        self.freeze()

    def freeze(self):
        self.transformer = self.transformer.eval()
        for param in self.parameters():
            param.requires_grad = False

    # read from the tokenizer when used, so a tokenizer attached after construction frames prompts with its own ids
    @property
    def id_start(self):
        enc = getattr(self.tokenizer, 'encoder', None) or {}
        return enc.get('<|startoftext|>', enc.get('<start_of_text>', self.ID_START))

    @property
    def id_end(self):
        enc = getattr(self.tokenizer, 'encoder', None) or {}
        return enc.get('<|endoftext|>', enc.get('<end_of_text>', self.ID_END))

    def tokenize(self, text):
        """list of str (or one str) -> input_ids [B, max_length] int64 on the CPU."""
        texts = [text] if isinstance(text, str) else list(text)
        tok = self.tokenizer
        if tok is None:
            raise RuntimeError('FrozenCLIPEmbedder needs the CLIP BPE tokenizer to encode strings: pass tokenizer= (a '
                               'transformers CLIPTokenizer, or an object with .encode(str) -> list of int such as open_clip\'s '
                               'SimpleTokenizer), or version= a local openai/clip-vit-large-patch14 snapshot directory')
        if _is_hf_tokenizer(tok):
            be = tok(texts, truncation=True, max_length=self.max_length, return_length=True, return_overflowing_tokens=False,
                     padding='max_length', return_tensors='pt')
            return be['input_ids']
        rows = []
        for t in texts:
            ids = [self.id_start] + list(tok.encode(t))[:self.max_length - 2] + [self.id_end]
            rows.append(ids + [self.id_end] * (self.max_length - len(ids)))
        return torch.tensor(rows, dtype=torch.long)

    def encode_with_transformer(self, tokens):
        """Already tokenised input [B, max_length] -> last_hidden_state [B, max_length, width] fp32 on the GPU."""
        return self.transformer.encode_tokens(torch.as_tensor(tokens))

    def forward(self, text):
        return self.encode_with_transformer(self.tokenize(text))

    def encode(self, text):
        return self(text)


def _text_weights(directory):
    """`text_model.*` tensors of a local Hugging Face CLIP snapshot (model.safetensors or pytorch_model.bin)."""
    st = os.path.join(directory, 'model.safetensors')
    if os.path.exists(st):
        from safetensors.torch import load_file                           # type: ignore
        sd = load_file(st)
    else:
        sd = torch.load(os.path.join(directory, 'pytorch_model.bin'), map_location='cpu')
    return {k: v for k, v in sd.items() if k.startswith('text_model.') and not k.endswith('.position_ids')}
