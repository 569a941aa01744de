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
"""
import ctypes as C
import math

import torch
import torch.nn as nn

from . import _lib
from .modules import _NativeModule, _param_table, _Holder


class _InProj(nn.Module):
    """Parameter holder with nn.MultiheadAttention's names (in_proj_weight / in_proj_bias / out_proj)."""

    def __init__(self, width):
        super().__init__()
        self.in_proj_weight = nn.Parameter(torch.zeros(3 * width, width))
        self.in_proj_bias = nn.Parameter(torch.zeros(3 * width))
        self.out_proj = nn.Linear(width, width)


class _TextTower(_NativeModule):
    """`model` of the embedder: open_clip's text-side module tree; arithmetic in libt2v_b200.so (csrc/clip.cu)."""
    _set_fn = 't2v_clip_set_param'

    def __init__(self, width=1024, heads=16, layers=24, layers_run=23, context=77, vocab=49408):
        super().__init__()
        cfg = _lib.ClipConfigC(width, heads, layers_run, context, vocab)
        self.width, self.heads, self.layers, self.layers_run, self.context, self.vocab = width, heads, layers, layers_run, context, vocab
        h = C.c_void_p()
        _lib.check(_lib.load_library().t2v_clip_create(C.byref(cfg), C.byref(h)), 'clip_create')
        object.__setattr__(self, '_handle', h)
        self._native_names = set(_param_table('t2v_clip_param_info', h))
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
        self._init_native()

    def __del__(self):
        h = self.__dict__.get('_handle')
        if h:
            try:
                _lib.load_library().t2v_clip_destroy(h)
            except Exception:
                pass

    def named_parameters(self, *a, **kw):
        for name, p in super().named_parameters(*a, **kw):
            if name in self._native_names:
                yield name, p

    def state_dict(self, *a, **kw):
        return nn.Module.state_dict(self, *a, **kw)

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
