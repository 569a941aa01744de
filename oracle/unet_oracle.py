"""TEST INFRASTRUCTURE ONLY -- CPU oracle for the ModelScope `UNetSD` denoiser.

A functional restatement (plain torch ops on a flat {name: tensor} weight dict; no
nn.Module tree) of the reference forward pass, every function citing the reference
lines it follows (paths relative to /root/reference/scripts/modelscope/t2v_model.py
unless noted).  It is the checker for the CUDA path; only tests/, bench.py's
cpu_baseline / --impl reference leg and __graft_entry__.smoke() may import it.

PARITY PINNING: the reference ships no tests or golden vectors ("parity unpinned" by
the reference itself).  This restatement is pinned instead against the reference's own
modules executed in-process on CPU (oracle/make_golden.py, tests/test_oracle_vs_reference.py)
and against the committed fixtures in tests/golden/ that script produced.

Everything runs in whatever dtype/device the weights are in (fp32 CPU for the gate;
tests may also run it on CUDA under fp16 autocast to reproduce the reference's GPU
numerics contract, SURVEY.md appendix B).
"""
from dataclasses import dataclass, field
from typing import Dict, List, Tuple
import math

import torch
import torch.nn.functional as F


@dataclass
class UNetConfig:
    """Hyper-parameters consumed at t2v_pipeline.py:76-94 (public damo-vilab values)."""
    in_dim: int = 4
    dim: int = 320
    context_dim: int = 1024
    out_dim: int = 4
    dim_mult: Tuple[int, ...] = (1, 2, 4, 4)
    num_heads: int = 8            # only used by the stem TemporalTransformer (:171-179)
    head_dim: int = 64
    num_res_blocks: int = 2
    attn_scales: Tuple[float, ...] = (1.0, 0.5, 0.25)

    @property
    def embed_dim(self):
        return self.dim * 4       # :120


# -------------------------------------------------------------------------------------
# module-tree enumeration (names == reference state_dict keys, SURVEY.md appendix D)
# -------------------------------------------------------------------------------------
@dataclass
class Block:
    kind: str                     # 'stem' | 'res' | 'st' | 'tt' | 'down' | 'up'
    prefix: str
    cin: int = 0
    cout: int = 0
    heads: int = 0
    inner: int = 0


def enumerate_blocks(cfg: UNetConfig):
    """Walks UNetSD.__init__ (:148-323) and returns (input_blocks, middle, output_blocks)
    as lists of lists of Block."""
    dim, hd = cfg.dim, cfg.head_dim
    enc_dims = [dim * u for u in (1,) + tuple(cfg.dim_mult)]
    dec_dims = [dim * u for u in (cfg.dim_mult[-1],) + tuple(cfg.dim_mult[::-1])]
    shortcut = []
    scale = 1.0
    inputs: List[List[Block]] = []
    # :167-181 stem conv + temporal transformer with `num_heads` heads
    inputs.append([Block('stem', 'input_blocks.0.0', cfg.in_dim, dim),
                   Block('tt', 'input_blocks.0.1', dim, dim, cfg.num_heads, cfg.num_heads * hd)])
    shortcut.append(dim)
    for i, (cin, cout) in enumerate(zip(enc_dims[:-1], enc_dims[1:])):
        for j in range(cfg.num_res_blocks):
            n = len(inputs)
            blk = [Block('res', f'input_blocks.{n}.0', cin, cout)]
            if scale in cfg.attn_scales:
                blk.append(Block('st', f'input_blocks.{n}.1', cout, cout, cout // hd, cout))
                blk.append(Block('tt', f'input_blocks.{n}.2', cout, cout, cout // hd, cout))
            cin = cout
            inputs.append(blk)
            shortcut.append(cout)
            if i != len(cfg.dim_mult) - 1 and j == cfg.num_res_blocks - 1:
                n = len(inputs)
                inputs.append([Block('down', f'input_blocks.{n}', cout, cout)])   # bare module (:229)
                shortcut.append(cout)
                scale /= 2.0
    c = enc_dims[-1]
    middle = [Block('res', 'middle_block.0', c, c),
              Block('st', 'middle_block.1', c, c, c // hd, c),
              Block('tt', 'middle_block.2', c, c, c // hd, c),
              Block('res', 'middle_block.3', c, c)]
    outputs: List[List[Block]] = []
    for i, (cin, cout) in enumerate(zip(dec_dims[:-1], dec_dims[1:])):
        for j in range(cfg.num_res_blocks + 1):
            n = len(outputs)
            blk = [Block('res', f'output_blocks.{n}.0', cin + shortcut.pop(), cout)]
            k = 1
            if scale in cfg.attn_scales:
                blk.append(Block('st', f'output_blocks.{n}.1', cout, cout, cout // hd, cout))
                blk.append(Block('tt', f'output_blocks.{n}.2', cout, cout, cout // hd, cout))
                k = 3
            cin = cout
            if i != len(cfg.dim_mult) - 1 and j == cfg.num_res_blocks:
                blk.append(Block('up', f'output_blocks.{n}.{k}', cout, cout))
                scale *= 2.0
            outputs.append(blk)
    return inputs, middle, outputs


def param_specs(cfg: UNetConfig) -> Dict[str, Tuple[int, ...]]:
    """name -> shape for every UNetSD parameter (1480 tensors at the public config)."""
    specs: Dict[str, Tuple[int, ...]] = {}
    E = cfg.embed_dim

    def lin(p, o, i, bias=True):
        specs[p + '.weight'] = (o, i)
        if bias:
            specs[p + '.bias'] = (o,)

    def norm(p, c):
        specs[p + '.weight'] = (c,)
        specs[p + '.bias'] = (c,)

    def conv(p, o, i, *k):
        specs[p + '.weight'] = (o, i) + tuple(k)
        specs[p + '.bias'] = (o,)

    def transformer_block(p, inner, ctx):
        for a, cd in (('attn1', inner), ('attn2', ctx)):
            lin(f'{p}.{a}.to_q', inner, inner, False)
            lin(f'{p}.{a}.to_k', inner, cd, False)
            lin(f'{p}.{a}.to_v', inner, cd, False)
            lin(f'{p}.{a}.to_out.0', inner, inner)
        lin(f'{p}.ff.net.0.proj', inner * 8, inner)
        lin(f'{p}.ff.net.2', inner, inner * 4)
        for n in ('norm1', 'norm2', 'norm3'):
            norm(f'{p}.{n}', inner)

    lin('time_embed.0', E, cfg.dim)
    lin('time_embed.2', E, E)
    ins, mid, outs = enumerate_blocks(cfg)
    for b in [x for blk in ins for x in blk] + mid + [x for blk in outs for x in blk]:
        p = b.prefix
        if b.kind == 'stem':
            conv(p, b.cout, b.cin, 3, 3)
        elif b.kind == 'res':
            norm(p + '.in_layers.0', b.cin)
            conv(p + '.in_layers.2', b.cout, b.cin, 3, 3)
            lin(p + '.emb_layers.1', b.cout, E)
            norm(p + '.out_layers.0', b.cout)
            conv(p + '.out_layers.3', b.cout, b.cout, 3, 3)
            if b.cin != b.cout:
                conv(p + '.skip_connection', b.cout, b.cin, 1, 1)
            # attribute really is spelled `temopral_conv` (:968); conv1 has no Dropout slot
            for name, ci in (('conv1', 2), ('conv2', 3), ('conv3', 3), ('conv4', 3)):
                norm(f'{p}.temopral_conv.{name}.0', b.cout)
                conv(f'{p}.temopral_conv.{name}.{ci}', b.cout, b.cout, 3, 1, 1)
        elif b.kind == 'st':
            norm(p + '.norm', b.cin)
            lin(p + '.proj_in', b.inner, b.cin)
            transformer_block(p + '.transformer_blocks.0', b.inner, cfg.context_dim)
            lin(p + '.proj_out', b.cin, b.inner)
        elif b.kind == 'tt':
            norm(p + '.norm', b.cin)
            conv(p + '.proj_in', b.inner, b.cin, 1)
            transformer_block(p + '.transformer_blocks.0', b.inner, b.inner)   # only_self_att (:684-685)
            conv(p + '.proj_out', b.cin, b.inner, 1)
        elif b.kind == 'down':
            conv(p + '.op', b.cout, b.cin, 3, 3)
        elif b.kind == 'up':
            conv(p + '.conv', b.cout, b.cin, 3, 3)
    norm('out.0', cfg.dim)
    conv('out.2', cfg.out_dim, cfg.dim, 3, 3)
    return specs


# -------------------------------------------------------------------------------------
# forward
# -------------------------------------------------------------------------------------
def sinusoidal_embedding(t, dim):
    """:504-515  [cos | sin](t * 10000^(-i/half))."""
    half = dim // 2
    t = t.float()
    freqs = torch.pow(10000, -torch.arange(half).to(t).div(half))
    s = torch.outer(t, freqs)
    e = torch.cat([torch.cos(s), torch.sin(s)], dim=1)
    if dim % 2:
        e = torch.cat([e, torch.zeros_like(e[:, :1])], dim=1)
    return e


# Which branch of CrossAttention.forward (:556-582) is restated: 'math' = the einsum + softmax fallback (:570-580; the CPU
# gate), 'sdpa' = F.scaled_dot_product_attention on (b h) n d tensors (:566-569; the backend the reference takes without
# xformers installed).  bench.py's GPU comparator and the autocast parity tests set 'sdpa'.
ATTN_IMPL = 'math'


def _attention(W, p, x, ctx, heads):
    """CrossAttention.forward :540-584 (softmax(q k^T d^-1/2) v, then to_out)."""
    q = F.linear(x, W[p + '.to_q.weight'])
    ctx = x if ctx is None else ctx
    k = F.linear(ctx, W[p + '.to_k.weight'])
    v = F.linear(ctx, W[p + '.to_v.weight'])
    B, N, C = q.shape
    d = C // heads

    def split(t):
        return t.reshape(t.shape[0], t.shape[1], heads, d).permute(0, 2, 1, 3)

    q, k, v = split(q), split(k), split(v)
    if ATTN_IMPL == 'sdpa':
        o = F.scaled_dot_product_attention(q.reshape(-1, q.shape[2], d), k.reshape(-1, k.shape[2], d),
                                           v.reshape(-1, v.shape[2], d), dropout_p=0.0).reshape(B, heads, N, d)
    else:
        sim = torch.matmul(q, k.transpose(-1, -2)) * (d ** -0.5)
        o = torch.matmul(sim.softmax(dim=-1), v)
    o = o.permute(0, 2, 1, 3).reshape(B, N, C)
    return F.linear(o, W[p + '.to_out.0.weight'], W[p + '.to_out.0.bias'])


def _transformer_block(W, p, x, ctx, heads):
    """BasicTransformerBlock.forward :803-809 + GEGLU :819-821 + FeedForward :845."""
    def ln(n, t):
        return F.layer_norm(t, (t.shape[-1],), W[f'{p}.{n}.weight'], W[f'{p}.{n}.bias'], 1e-5)

    x = _attention(W, p + '.attn1', ln('norm1', x), None, heads) + x
    x = _attention(W, p + '.attn2', ln('norm2', x), ctx, heads) + x
    h = F.linear(ln('norm3', x), W[p + '.ff.net.0.proj.weight'], W[p + '.ff.net.0.proj.bias'])
    a, gate = h.chunk(2, dim=-1)
    h = a * F.gelu(gate)
    h = F.linear(h, W[p + '.ff.net.2.weight'], W[p + '.ff.net.2.bias'])
    return h + x


def _spatial_transformer(W, b: Block, x, ctx):
    """SpatialTransformer.forward :639-658 with use_linear=True.  x: [(b f), C, h, w]."""
    n, c, h, w = x.shape
    y = F.group_norm(x, 32, W[b.prefix + '.norm.weight'], W[b.prefix + '.norm.bias'], 1e-6)
    y = y.permute(0, 2, 3, 1).reshape(n, h * w, c)
    y = F.linear(y, W[b.prefix + '.proj_in.weight'], W[b.prefix + '.proj_in.bias'])
    y = _transformer_block(W, b.prefix + '.transformer_blocks.0', y, ctx, b.heads)
    y = F.linear(y, W[b.prefix + '.proj_out.weight'], W[b.prefix + '.proj_out.bias'])
    y = y.reshape(n, h, w, c).permute(0, 3, 1, 2)
    return y + x


def _temporal_transformer(W, b: Block, x, batch):
    """TemporalTransformer.forward :716-767 (use_linear False, only_self_att True).
    x: [(b f), C, h, w]; GroupNorm is 5-D, i.e. statistics over all frames (:724)."""
    n, c, h, w = x.shape
    f = n // batch
    x5 = x.reshape(batch, f, c, h, w).permute(0, 2, 1, 3, 4)              # b c f h w (:479)
    y = F.group_norm(x5, 32, W[b.prefix + '.norm.weight'], W[b.prefix + '.norm.bias'], 1e-6)
    y = y.permute(0, 3, 4, 2, 1).reshape(batch * h * w, f, c)                # (b h w) f c
    y = F.linear(y, W[b.prefix + '.proj_in.weight'][:, :, 0], W[b.prefix + '.proj_in.bias'])   # Conv1d k=1
    y = _transformer_block(W, b.prefix + '.transformer_blocks.0', y, None, b.heads)
    y = F.linear(y, W[b.prefix + '.proj_out.weight'][:, :, 0], W[b.prefix + '.proj_out.bias'])
    y = y.reshape(batch, h, w, f, c).permute(0, 4, 3, 1, 2)                  # b c f h w
    y = y + x5
    return y.permute(0, 2, 1, 3, 4).reshape(n, c, h, w)


def _temporal_conv(W, p, x, batch):
    """TemporalConvBlock_v2.forward :1218-1229: 4 x [GN32(5-D) -> SiLU -> Conv3d (3,1,1)] + identity."""
    n, c, h, w = x.shape
    f = n // batch
    x5 = x.reshape(batch, f, c, h, w).permute(0, 2, 1, 3, 4)
    y = x5
    for name, ci in (('conv1', 2), ('conv2', 3), ('conv3', 3), ('conv4', 3)):
        y = F.group_norm(y, 32, W[f'{p}.{name}.0.weight'], W[f'{p}.{name}.0.bias'], 1e-5)
        y = F.silu(y)
        y = F.conv3d(y, W[f'{p}.{name}.{ci}.weight'], W[f'{p}.{name}.{ci}.bias'], padding=(1, 0, 0))
    y = x5 + y
    return y.permute(0, 2, 1, 3, 4).reshape(n, c, h, w)


def _res_block(W, b: Block, x, e, batch):
    """ResBlock._forward :983-1009 (use_scale_shift_norm False, no up/down)."""
    p = b.prefix
    h = F.group_norm(x, 32, W[p + '.in_layers.0.weight'], W[p + '.in_layers.0.bias'], 1e-5)
    h = F.conv2d(F.silu(h), W[p + '.in_layers.2.weight'], W[p + '.in_layers.2.bias'], padding=1)
    emb = F.linear(F.silu(e), W[p + '.emb_layers.1.weight'], W[p + '.emb_layers.1.bias']).type(h.dtype)
    h = h + emb[:, :, None, None]
    h = F.group_norm(h, 32, W[p + '.out_layers.0.weight'], W[p + '.out_layers.0.bias'], 1e-5)
    h = F.conv2d(F.silu(h), W[p + '.out_layers.3.weight'], W[p + '.out_layers.3.bias'], padding=1)
    if b.cin != b.cout:
        x = F.conv2d(x, W[p + '.skip_connection.weight'], W[p + '.skip_connection.bias'])
    h = x + h
    return _temporal_conv(W, p + '.temopral_conv', h, batch)


def _run_block(W, blk: List[Block], x, e, ctx, batch, taps=None):
    for b in blk:
        if b.kind == 'stem':
            x = F.conv2d(x, W[b.prefix + '.weight'], W[b.prefix + '.bias'], padding=1)
        elif b.kind == 'res':
            x = _res_block(W, b, x, e, batch)
        elif b.kind == 'st':
            x = _spatial_transformer(W, b, x, ctx)
        elif b.kind == 'tt':
            x = _temporal_transformer(W, b, x, batch)
        elif b.kind == 'down':
            x = F.conv2d(x, W[b.prefix + '.op.weight'], W[b.prefix + '.op.bias'], stride=2, padding=1)   # :1034-1039
        elif b.kind == 'up':
            x = F.interpolate(x, scale_factor=2, mode='nearest')                                      # :880
            x = F.conv2d(x, W[b.prefix + '.conv.weight'], W[b.prefix + '.conv.bias'], padding=1)
        if taps is not None:
            taps[b.prefix] = x
    return x


@torch.no_grad()
def unet_forward(W: Dict[str, torch.Tensor], cfg: UNetConfig, x, t, y, taps=None):
    """UNetSD.forward :386-459.  x [B,4,F,h,w], t [B], y [B,L,context_dim] -> eps [B,out,F,h,w].
    `taps` (optional dict) receives every sub-module's output in (b f) c h w layout."""
    ins, mid, outs = enumerate_blocks(cfg)
    B, _, Fr, h, w = x.shape
    wdt = W['time_embed.0.weight'].dtype
    e = sinusoidal_embedding(t, cfg.dim).to(wdt)
    e = F.linear(e, W['time_embed.0.weight'], W['time_embed.0.bias'])
    e = F.linear(F.silu(e), W['time_embed.2.weight'], W['time_embed.2.bias'])
    e = e.repeat_interleave(Fr, dim=0)                       # :425
    ctx = y.to(wdt).repeat_interleave(Fr, dim=0)             # :426
    x = x.to(wdt).permute(0, 2, 1, 3, 4).reshape(B * Fr, -1, h, w)   # :429
    xs = []
    for blk in ins:
        x = _run_block(W, blk, x, e, ctx, B, taps)
        xs.append(x)
    x = _run_block(W, mid, x, e, ctx, B, taps)
    for blk in outs:
        x = torch.cat([x, xs.pop()], dim=1)                  # :444
        x = _run_block(W, blk, x, e, ctx, B, taps)
    x = F.group_norm(x, 32, W['out.0.weight'], W['out.0.bias'], 1e-5)
    x = F.conv2d(F.silu(x), W['out.2.weight'], W['out.2.bias'], padding=1)
    return x.reshape(B, Fr, -1, h, w).permute(0, 2, 1, 3, 4).contiguous()


# -------------------------------------------------------------------------------------
# deterministic synthetic weights (no checkpoint can be downloaded here)
# -------------------------------------------------------------------------------------
def make_weights(specs: Dict[str, Tuple[int, ...]], seed: int = 0, dtype=torch.float32,
                 gain: float = 1.0) -> Dict[str, torch.Tensor]:
    """Seeded synthetic parameters with NO all-zero tensor (the reference zero-initialises every
    residual branch -- t2v_model.py:326,:631-636,:708-713,:955-956,:1214-1216 -- which would make
    parity vacuous, SURVEY.md section 4).  One CPU generator, keys in sorted order, so the same
    (specs, seed) gives bit-identical tensors on any host with this torch build."""
    g = torch.Generator(device='cpu').manual_seed(seed)
    out = {}
    for name in sorted(specs):
        shape = specs[name]
        if len(shape) == 1:
            is_norm_w = name.endswith('.weight')
            v = torch.randn(shape, generator=g) * (0.1 if is_norm_w else 0.05)
            if is_norm_w:
                v += 1.0
        else:
            fan_in = 1
            for s in shape[1:]:
                fan_in *= s
            v = torch.randn(shape, generator=g) * (gain / math.sqrt(fan_in))
        out[name] = v.to(dtype)
    return out
