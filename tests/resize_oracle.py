"""CPU restatement of Pillow's Image.resize((W, H), Image.LANCZOS) for uint8 RGB frames (libImaging/Resample.c) and of the
reference's normalisation (process_modelscope.py:115-137): the checker of t2v_frames_resize.  Needs neither Pillow nor a GPU;
the tables are numpy, the integer passes torch CPU ops (threaded, so a 250-frame clip takes seconds).

Tables in double: scale = in / out, filterscale = max(scale, 1), support = 3 * filterscale; output pixel xx reads input
pixels [first, first + taps) with first = max(int(center - support + 0.5), 0), center = (xx + 0.5) * scale, weight
lanczos((x + first - center + 0.5) * (1 / filterscale)), normalised by the sum and rounded half away from zero to int32 with
22 fractional bits.  The horizontal pass runs first over the rows the vertical pass reads, into uint8; each pass is
(2^21 + sum(pixel * k)) >> 22 clipped to [0, 255]; a pass whose size does not change is skipped."""
import math

import numpy as np
import torch

PRECISION_BITS = 22


def _sinc(x):
    if x == 0.0:
        return 1.0
    x *= math.pi
    return math.sin(x) / x


def lanczos(x):
    return _sinc(x) * _sinc(x / 3.0) if -3.0 <= x < 3.0 else 0.0


def coeffs(in_size, out_size):
    """Pillow's tables: bounds int32 [out, 2] (first input pixel, taps used), k int32 [out, ksize]."""
    scale = in_size / out_size
    fs = max(scale, 1.0)
    support = 3.0 * fs
    ss = 1.0 / fs
    ksize = int(math.ceil(support)) * 2 + 1
    bounds = np.zeros((out_size, 2), dtype=np.int32)
    k = np.zeros((out_size, ksize), dtype=np.int32)
    for xx in range(out_size):
        center = (xx + 0.5) * scale
        xmin = max(int(center - support + 0.5), 0)
        n = min(int(center + support + 0.5), in_size) - xmin
        w = [lanczos((x + xmin - center + 0.5) * ss) for x in range(n)]
        ww = sum(w)
        for x in range(n):
            v = (w[x] / ww if ww != 0.0 else w[x]) * (1 << PRECISION_BITS)
            k[xx, x] = int(-0.5 + v) if v < 0 else int(0.5 + v)
        bounds[xx] = (xmin, n)
    return bounds, k


def _pass(a, dim, bounds, k):
    """Resample uint8 `a` (a CPU tensor) along `dim` with the tables, in int32 as Pillow accumulates."""
    idx = torch.from_numpy(np.clip(bounds[:, :1] + np.arange(k.shape[1])[None, :], 0, a.shape[dim] - 1))   # k is 0 past taps
    kk = torch.from_numpy(k)
    shape = [1] * a.dim()
    shape[dim] = -1
    acc = torch.full((), 1 << (PRECISION_BITS - 1), dtype=torch.int32)
    for j in range(k.shape[1]):
        acc = acc + a.index_select(dim, idx[:, j]).to(torch.int32) * kk[:, j].view(shape)
    return (acc >> PRECISION_BITS).clamp_(0, 255).to(torch.uint8)


def resize(frames, width, height):
    """uint8 [..., H0, W0, 3] -> uint8 [..., height, width, 3], Pillow's LANCZOS resize of every frame."""
    a = torch.from_numpy(np.ascontiguousarray(frames))
    h0, w0 = a.shape[-3], a.shape[-2]
    bv, kv = coeffs(h0, height)
    if width != w0:
        y0, y1 = int(bv[0, 0]), int(bv[-1, 0] + bv[-1, 1])
        bh, kh = coeffs(w0, width)
        a = _pass(a[..., y0:y1, :, :], a.dim() - 2, bh, kh)
        bv = bv - np.array([y0, 0], dtype=np.int32)
    if height != h0:
        a = _pass(a, a.dim() - 3, bv, kv)
    return a.contiguous().numpy()


def normalise(u8):
    """The reference's x / 255 then 2 * x - 1 in float32, op by op: uint8 [..., H, W, 3] -> float32 [..., 3, H, W]."""
    x = u8.astype(np.float32) / np.float32(255)
    x = np.float32(2) * x - np.float32(1)
    return np.ascontiguousarray(np.moveaxis(x, -1, -3))
