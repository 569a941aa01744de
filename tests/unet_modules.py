"""Module-by-module restatement of how the UNet plan builder (csrc/unet.cu `build()`) wires its modules, for ModelScope's
UNetSD and VideoCrafter's UNetModel (test infrastructure; imports the oracles as the checkers only).

Given the per-module taps of one forward (the library's `read_tap`, or an oracle's `taps=` dict), `module_inputs` yields
every module in forward order with the input the forward fed it, so each module can be re-run on its own through the
oracle (`run_module`) and compared with its tap.  Every tensor here is in the taps' layout [(b f), C, h, w].

`slice_names` / `slice_mean_squares` cut a tap into the pieces a wiring mistake tends to confine itself to: one (sample,
frame), one of the 32 GroupNorm channel groups, the border ring of one frame (where the 3x3 convs read their zero padding)
and its interior."""
from dataclasses import dataclass

import torch
import torch.nn.functional as F

from oracle import unet_oracle as UO, vc_oracle as VC

MS, VCR = 'modelscope', 'videocrafter'


@dataclass
class Head:
    """The output head (GroupNorm -> SiLU -> conv `out.2`), checked against the `out` tap."""
    kind: str = 'head'
    prefix: str = 'out'


HEAD = Head()


def arch_of(cfg):
    return MS if isinstance(cfg, UO.UNetConfig) else VCR


def blocks(cfg):
    """(input blocks, middle, output blocks) as the oracle enumerates them: lists of lists of blocks, middle a list."""
    if arch_of(cfg) == MS:
        return UO.enumerate_blocks(cfg)
    L = VC.vc_enumerate(cfg)
    return L.input_blocks, L.middle, L.output_blocks


def tap_names(cfg):
    """Every tap `build()` records for this config, in forward order: one per module under its reference name, then `out`."""
    ins, mid, outs = blocks(cfg)
    return [b.prefix for blk in ins for b in blk] + [b.prefix for b in mid] + [b.prefix for blk in outs for b in blk] + ['out']


def feature_block(i):
    """Input blocks after which VideoCrafter adds an adapter feature (openaimodel3d.py:658)."""
    return (i + 1) % 3 == 0


def module_inputs(cfg, taps, latent, feats=None):
    """Yields (module, input) in forward order; the head comes last as HEAD.

    `latent` [B, C, F, h, w]: the stem reads it rounded to fp16, as the library ingests it.  `feats` (VideoCrafter): the
    adapter features as staged, [fb, C, F, h_i, w_i] each, sample j reading feature sample j % fb.  The tap of a feature
    block is taken before the add; the next module and the skip connection see fp16(tap + feature), added in fp32 like
    `feature_add`.  The first module of each output block reads cat([previous output, skip]), the skips popped last in,
    first out.  Inputs have the taps' dtype."""
    ins, mid, outs = blocks(cfg)
    B, _, Fr, h, w = latent.shape
    t0 = next(iter(taps.values()))
    dt = t0.dtype
    x = latent.to(t0.device).half().to(dt).permute(0, 2, 1, 3, 4).reshape(B * Fr, -1, h, w)
    skips, nf = [], 0
    for i, blk in enumerate(ins):
        for b in blk:
            yield b, x
            x = taps[b.prefix]
        if feats is not None and feature_block(i):
            f = feats[nf]
            nf += 1
            f = f.repeat(B // f.shape[0], 1, 1, 1, 1).permute(0, 2, 1, 3, 4).reshape(x.shape)
            acc = torch.float32 if dt == torch.float16 else dt
            x = (x.to(acc) + f.to(device=x.device, dtype=acc)).to(dt)
        skips.append(x)
    if feats is not None and nf != len(feats):
        raise ValueError(f'{len(feats)} adapter features for {nf} injection points')
    for b in mid:
        yield b, x
        x = taps[b.prefix]
    for blk in outs:
        x = torch.cat([x, skips.pop()], dim=1)
        for b in blk:
            yield b, x
            x = taps[b.prefix]
    yield HEAD, x


def time_embedding(cfg, W, t):
    """[B, 4 dim] time embedding as the oracle's forward computes it: the sinusoid in fp32 (t2v_model.py:504-515;
    VideoCrafter util.py:142-162), then time_embed's Linear -> SiLU -> Linear in W's dtype."""
    w0 = W['time_embed.0.weight']
    if arch_of(cfg) == MS:
        e = UO.sinusoidal_embedding(t, cfg.dim)
    else:
        e = VC.vc_timestep_embedding(t, cfg.model_channels)
    e = F.linear(e.to(device=w0.device, dtype=w0.dtype), w0, W['time_embed.0.bias'])
    return F.linear(F.silu(e), W['time_embed.2.weight'], W['time_embed.2.bias'])


def feature_shapes(cfg, fb, Fr, h, w):
    """[fb, C, F, h_i, w_i] of each adapter feature of a [., ., F, h, w] latent: one per input block with (id + 1) % 3 == 0,
    at that block's output width and resolution."""
    ins, _, _ = blocks(cfg)
    out = []
    for i, blk in enumerate(ins):
        if blk[0].kind == 'down':
            h, w = (h + 1) // 2, (w + 1) // 2
        if feature_block(i):
            out.append((fb, blk[-1].cout, Fr, h, w))
    return out


def structured_inputs(cfg, B, Fr, h, w, L, Bc=None, seed=0):
    """(latent [B, C, F, h, w], t [B], prompts [Bc, L, context_dim]), fp16-representable, built so that a module reading
    the wrong sample, frame or prompt is off by O(1): timesteps spread from 999 down to 1, frame f of the latent scaled by
    1 + f mod 3, sample j offset by j / 2, and a different random prompt per sample (per prompt of a shared batch)."""
    g = torch.Generator().manual_seed(seed)
    cin = cfg.in_dim if arch_of(cfg) == MS else cfg.in_channels
    x = torch.randn(B, cin, Fr, h, w, generator=g)
    x = x * (1 + torch.arange(Fr) % 3).view(1, 1, Fr, 1, 1).float() + 0.5 * torch.arange(B).view(B, 1, 1, 1, 1).float()
    t = torch.linspace(999, 1, B).round() if B > 1 else torch.tensor([999.0])
    y = torch.randn(Bc or B, L, cfg.context_dim, generator=g)
    return x.half().float(), t, y.half().float()


def _to5(x, B):
    n, c, h, w = x.shape
    return x.reshape(B, n // B, c, h, w).permute(0, 2, 1, 3, 4).contiguous()


def _from5(x):
    b, c, f, h, w = x.shape
    return x.permute(0, 2, 1, 3, 4).reshape(b * f, c, h, w)


def run_module(cfg, W, b, x, emb, ctx, B):
    """The oracle's module `b` on x [(b f), C, h, w] -> its output in the same layout.  emb [B, E] and ctx [B, L, C] hold
    one row per sample; ModelScope's forward repeats both per frame (t2v_model.py:425-426), VideoCrafter's takes them per
    sample."""
    Fr = x.shape[0] // B
    if arch_of(cfg) == MS:
        if b is HEAD:       # t2v_model.py:321-323
            y = F.group_norm(x, 32, W['out.0.weight'], W['out.0.bias'], 1e-5)
            return F.conv2d(F.silu(y), W['out.2.weight'], W['out.2.bias'], padding=1)
        return UO._run_block(W, [b], x, emb.repeat_interleave(Fr, dim=0), ctx.repeat_interleave(Fr, dim=0), B)
    h = _to5(x, B)
    if b is HEAD:           # openaimodel3d.py:669
        h = F.conv3d(F.silu(VC._gn(W, 'out.0', h, 1e-5)), W['out.2.weight'], W['out.2.bias'], padding=(0, 1, 1))
    else:
        h = VC._run(W, [b], h, emb, ctx, cfg)
    return _from5(h)


def module_weights(W, b):
    """The names of W module `b` reads (the head: out.0 / out.2)."""
    if b is HEAD:
        return [k for k in W if k.startswith('out.')]
    return [k for k in W if k.startswith(b.prefix + '.')]


def _ring(h, w, device):
    ring = torch.zeros(h, w, dtype=torch.bool, device=device)
    ring[0], ring[-1], ring[:, 0], ring[:, -1] = True, True, True, True
    return ring


def slice_names(shape, B):
    """Names of the slices of a tap of `shape` [(b f), C, h, w] from a B-sample forward, in slice_mean_squares' order:
    each (sample, frame); each of the 32 channel groups (each channel when C < 32: the head); the border ring (first and
    last row and column) of each frame; the interior of each frame, when it has one."""
    n, C, h, w = shape
    frames = [(j, f) for j in range(B) for f in range(n // B)]
    names = [f'sample {j} frame {f}' for j, f in frames]
    names += [f'channel group {i}' for i in range(min(32, C))]
    names += [f'border of sample {j} frame {f}' for j, f in frames]
    if h > 2 and w > 2:
        names += [f'interior of sample {j} frame {f}' for j, f in frames]
    return names


def slice_mean_squares(t, B):
    """Mean of t**2 over every slice of slice_names(t.shape, B), in fp64."""
    n, C, h, w = t.shape
    g = min(32, C)
    assert C % g == 0, C
    t2 = t.double().pow(2)
    px = t2.mean(1)
    ring = _ring(h, w, t.device)
    parts = [t2.mean((1, 2, 3)), t2.reshape(n, g, C // g, h, w).mean((0, 2, 3, 4)), px[:, ring].mean(1)]
    if h > 2 and w > 2:
        parts.append(px[:, ~ring].mean(1))
    return torch.cat(parts)
