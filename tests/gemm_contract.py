"""The implicit-GEMM engine's contract (csrc/gemm_tc.cuh, gemm_tc.cu, kernels.cuh), restated in fp64 torch, and generators of
operands on which that contract has exactly one correct bit pattern per output element.

Contract, per output element (row r, column n), with acc = sum_tap sum_k A[r + tap, k] W[tap, n, k]:
  fp16 output         fp16(acc * alpha + bias_row(r)[n] + residual[r, n])         one RN rounding, the sum in fp32
  GEMM_OUT_F32        fp32(acc * alpha + bias_row(r)[n])
  GEGLU (H columns)   fp16(fp16(value) * G), value = acc_v + b_v, gate = fp16(acc_g + b_g), G within 1 fp16 ulp of
                      fp16(gelu_erf_exact(gate)) (the kernel's gelu_erf uses rcp.approx / ex2.approx)
  split-K             fp16(sum_s part_s + bias_row(r)[n] + residual[r, n])
bias_row(r) = r // bias_rows with a per-sample bias (bias_rows > 0), else the single bias row.

Exact operands.  A holds small integers, W / bias / residual integers times a power-of-two grid g (GEGLU gate rows a finer
grid).  Every product, every partial sum in any order and every epilogue intermediate is then a multiple of g whose magnitude
is at most sum|a w| + |bias| + |res|, and the generators keep that below 2^BITS g with BITS = 16: 8 bits below fp32's 24,
so an accumulator that aligns addends with a few bits of truncation inside an MMA still sums exactly.  `premise_bits`
measures it on the data and the tests assert it.  The outputs themselves need up to ~15 significant bits, so the final fp16
rounding is not trivial (and some outputs are exact ties).

Also here: the tap geometry of conv_taps_2d / conv_taps_temporal (zero padding per frame / per sample), gemm_plan's row-box
planner, and pack_geglu_weight's tile interleave."""
import math

import numpy as np
import torch

BITS = 16                  # bits above the grid that any exact-mode intermediate may need
GRID = 2.0 ** -6           # W / bias / residual grid (value columns)
GATE_GRID = 2.0 ** -12     # GEGLU gate rows: gates of a few units, where GELU is not trivial
SUM_TARGET = 2.0 ** 14     # aimed-at sum |a w| per output, in grid units
EPI_MAX = 2048             # |bias|, |residual| in grid units: integers up to 2^11 are exact in fp16
A_LO, A_HI = -2, 6         # activations: integers, mean 2 (so outputs are mostly far from 0 and need > 11 bits)


# ---------------------------------------------------------------------------------------------------- exact operands
def gen(seed):
    return torch.Generator().manual_seed(seed)


def _ints(g, shape, lo, hi):
    return torch.randint(lo, hi + 1, tuple(shape), generator=g).double()


def exact_a(g, rows, K, k_eff):
    """fp16 [rows, K] of integers in [A_LO, A_HI]; entries zeroed at random where k_eff is so large that even the smallest
    weights would push sum |a w| past SUM_TARGET."""
    a = torch.randint(A_LO, A_HI + 1, (rows, K), generator=g, dtype=torch.int16)
    keep = min(1.0, SUM_TARGET / (1.8 * k_eff))
    if keep < 1.0:
        a = a * (torch.rand((rows, K), generator=g) < keep)
    return a.half()


def weight_range(k_eff):
    """wm of exact_w: weights are o_n + U[-wm, wm] integers (o_n per output column in [-wm, wm]), |w| <= 2 wm < 2^11 / grid
    so fp16 holds them."""
    return min(1023, max(1, int(SUM_TARGET / (1.8 * k_eff))))


def exact_w(g, taps, N, K, k_eff, grid=GRID):
    """fp16 [taps, N, K]: per output column an offset o_n and integer noise, both in [-wm, wm], times the grid.  Columns
    with o_n = 0 have outputs near zero, the others large ones of either sign."""
    wm = weight_range(k_eff)
    off = _ints(g, (1, N, 1), -wm, wm)
    w = off + _ints(g, (taps, N, K), -wm, wm)
    return (w * grid).half()


def exact_vec(g, shape, grid=GRID, lim=EPI_MAX):
    """fp16 bias / residual: integers in [-lim, lim] times the grid."""
    return (_ints(g, shape, -lim, lim) * grid).half()


def tap_operands(seed, dims, taps, K, N, *, bias=None, bias_rows=0, residual=False, k_valid=None, batches=0):
    """CPU exact operands of one GEMM over the row grid dims: a [rows, K] (columns from k_valid on zero, as a channel pad),
    w [taps (or batches), N, K], bias None / 'row' ([N]) / 'sample' ([rows // bias_rows, N]), residual [rows, N]."""
    g = gen(seed)
    rows = math.prod(dims)
    k_eff = len(taps) * (k_valid or K)
    a = exact_a(g, rows, K, k_eff)
    w = exact_w(g, batches or len(taps), N, K, k_eff)
    if k_valid is not None:
        a[:, k_valid:] = 0
        w[:, :, k_valid:] = 0
    c = dict(a=a, w=w, dims=list(dims), taps=taps, rows=rows, N=N, K=K, bias_rows=bias_rows if bias == 'sample' else 0,
             bias=None, res=None)
    if bias == 'row':
        c['bias'] = exact_vec(g, (N,))
    elif bias == 'sample':
        c['bias'] = exact_vec(g, (-(-rows // bias_rows), N))
    if residual:
        c['res'] = exact_vec(g, (rows, N))
    return c


def geglu_operands(seed, rows, K, H):
    """CPU exact operands of a GEGLU GEMM: a, w [2H, K] (value rows on GRID, gate rows on GATE_GRID), b [2H]."""
    g = gen(seed)
    a = exact_a(g, rows, K, K)
    wv, wg = exact_w(g, 1, H, K, K)[0], exact_w(g, 1, H, K, K, grid=GATE_GRID)[0]
    bv, bg = exact_vec(g, (H,)), exact_vec(g, (H,), grid=GATE_GRID)
    return dict(a=a, w=torch.cat([wv, wg]), b=torch.cat([bv, bg]), rows=rows, K=K, H=H)


def geglu_accumulators(c):
    """fp64 (value, gate, sum |terms|, grid per packed-order-free column [2H]) of geglu_operands' case (on its device)."""
    H = c['H']
    ad, wd, bd = c['a'].double(), c['w'].double(), c['b'].double()
    value = ad @ wd[:H].t() + bd[:H]
    gate = ad @ wd[H:].t() + bd[H:]
    absum = ad.abs() @ wd.abs().t() + bd.abs()
    grid = torch.tensor([GRID] * H + [GATE_GRID] * H, dtype=torch.float64, device=absum.device)
    return value, gate, absum, grid


def tap_contract(c, f32=False, alpha=1.0):
    """(contract output, sum |a w| + |bias| + |res|) of tap_operands' case, fp64 on its tensors' device.  A batched case
    (w has one slice per outermost-dim index, one tap [0, ..]) contracts each slice with its own rows."""
    a, w = c['a'], c['w']
    if w.shape[0] != len(c['taps']):                 # batched B
        nb = w.shape[0]
        ab = a.double().view(nb, -1, a.shape[1])
        acc = (ab @ w.double().transpose(1, 2)).reshape(c['rows'], -1)
        absum = (ab.abs() @ w.double().abs().transpose(1, 2)).reshape(c['rows'], -1)
    else:
        acc = implicit_gemm64(a, c['dims'], c['taps'], w)
        absum = implicit_gemm64(a, c['dims'], c['taps'], w, absolute=True)
    acc, absum = acc * alpha, absum * alpha
    brow = bias_rows_of(c['bias'], c['rows'], c['bias_rows']) if c['bias'] is not None else None
    if brow is not None:
        absum = absum + brow.abs()
    if c['res'] is not None:
        absum = absum + c['res'].double().abs()
    ref = epilogue_f32(acc, bias=brow) if f32 else epilogue_f16(acc, bias=brow, residual=c['res'])
    return ref, absum


# The variant matrix of tests/test_gemm_exact_gpu.py: one linear problem per epilogue kind.  9000 rows (70 x 128 + 40) and
# N = 456 are ragged at every tile width, K = 200 leaves a partial last K chunk, and at BN 224 / 256 the 142 tiles take more
# than one wave of 132 SMs (the TMA-store variant).  The B-stationary variant needs many M-tiles per N-tile: 12800 x 320.
MATRIX_KINDS = ['plain', 'bias', 'residual', 'in_place', 'ps_bias', 'f32', 'unaligned', 'unaligned_f32', 'batched', 'splitk',
                'geglu']
M_ROWS, M_K, M_N = 9000, 200, 456
BS_ROWS, BS_N = 12800, 320
PS_ROWS = 300                          # per-sample bias: 128-row tiles straddle the samples
BATCH_S, BATCH_NB, BATCH_ALPHA = 300, 3, 0.125
GEGLU_H = 512


def matrix_operands(kind, bs=False):
    """CPU exact operands of the variant matrix's kind (geglu_operands' dict for 'geglu', else tap_operands')."""
    seed = 100 + MATRIX_KINDS.index(kind) + (50 if bs else 0)
    rows, N = (BS_ROWS, BS_N) if bs else (M_ROWS, M_N)
    if kind == 'geglu':
        return geglu_operands(seed, rows, M_K, GEGLU_H)
    if kind == 'batched':
        return tap_operands(seed, [BATCH_S, BATCH_NB], [[0, 0]], M_K, N, batches=BATCH_NB)
    bias = 'sample' if kind == 'ps_bias' else (None if kind == 'plain' else 'row')
    residual = kind in ('residual', 'in_place', 'unaligned', 'splitk')
    return tap_operands(seed, [rows], [[0]], M_K, N, bias=bias, bias_rows=PS_ROWS, residual=residual)


def to(c, device):
    """The case dict with its tensors on device."""
    return {k: (v.to(device) if torch.is_tensor(v) else v) for k, v in c.items()}


def on_grid(t, grid):
    """Every element of t is an integer multiple of grid (fp64 check)."""
    q = t.double() / grid
    return bool((q == torch.round(q)).all())


def premise_bits(absum, grid):
    """log2 of the largest sum |a w| + |bias| + |res| (fp64, any shape) in units of grid (a scalar or a per-column tensor)."""
    m = (absum / grid).max().item()
    return math.log2(m) if m > 0 else 0.0


def inexact_fraction(v):
    """Share of the fp64 values v that fp16 cannot hold (the output rounding has work to do), and the count of exact ties
    (v halfway between two fp16 neighbours)."""
    v = v.double().flatten()
    hh = v.float().half()                            # one rounding: v is exact in fp32 on exact operands
    h = hh.double()
    miss = v != h
    o = _ordered(hh.view(torch.int16))
    other = _from_ordered(torch.where(v > h, o + 1, o - 1)).view(torch.float16).double()
    ties = miss & ((v - h).abs() == (other - v).abs())
    return miss.double().mean().item(), int(ties.sum().item())


# ---------------------------------------------------------------------------------------------------- geometry
def _shift(x, off):
    """x [d_{nd-1}, ..., d0, K]: y[.., i_d, ..] = x[.., i_d + off_d, ..], zero where that falls outside the dim."""
    nd = x.dim() - 1
    for d, o in enumerate(off):
        if o == 0:
            continue
        ax = nd - 1 - d
        n = x.shape[ax]
        y = torch.zeros_like(x)
        if abs(o) < n:
            if o > 0:
                y.narrow(ax, 0, n - o).copy_(x.narrow(ax, o, n - o))
            else:
                y.narrow(ax, -o, n + o).copy_(x.narrow(ax, 0, n + o))
        x = y
    return x


def implicit_gemm64(a, dims, taps, w, outer=None, absolute=False):
    """fp64 acc[row, n] = sum_tap sum_k a[row + tap, k] w[tap, n, k] (the GEMM's tap contraction, gemm_tc.cuh) on a's device.
    a [rows, >= K] over the row grid dims (d0 fastest), taps [[off_d0, off_d1, ...]], w [taps, >= N, K].  outer = (o0, o1):
    only the rows whose outermost-dim index lies in [o0, o1) (a block, with the halo its taps read).  absolute: sum |a w|."""
    K = w.shape[-1]
    nd = len(dims)
    x = a[:, :K].double().reshape(*reversed(dims), K)
    o0, o1 = (0, dims[-1]) if outer is None else outer
    h = max(abs(t[nd - 1]) for t in taps)
    lo, hi = max(0, o0 - h), min(dims[-1], o1 + h)
    x = x.narrow(0, lo, hi - lo)
    if absolute:
        x = x.abs()
    out = 0
    for t, off in enumerate(taps):
        wt = w[t].double()
        out = out + _shift(x, off).reshape(-1, K) @ (wt.abs() if absolute else wt).t()
    per = math.prod(dims[:-1])
    return out[(o0 - lo) * per:(o1 - lo) * per]


def conv_taps_2d():
    """ops.conv_taps_2d: tap ky * 3 + kx reads row offset (kx - 1, ky - 1, 0) over dims (w, h, frames)."""
    return [[kx - 1, ky - 1, 0] for ky in range(3) for kx in range(3)]


def conv_taps_temporal():
    """ops.conv_taps_temporal: tap kt reads (0, kt - 1, 0) over dims (pixels, frames, samples)."""
    return [[0, kt - 1, 0] for kt in range(3)]


def row_boxes(dims, b_batch_dim=-1, block_m=128):
    """gemm_plan's row box: box[d] fills from the fastest dim and grows into the next only once the current one is covered;
    a batched B's dim (and the dims above it) get box 1.  Returns (box, tiles per dim)."""
    box, remaining = [], block_m
    for ext in dims:
        b = max(1, min(ext, remaining))
        box.append(b)
        remaining = remaining // b if b >= ext else 1
    if b_batch_dim >= 0:
        for d in range(b_batch_dim, len(dims)):
            box[d] = 1
    return box, [-(-e // b) for e, b in zip(dims, box)]


def tile_first_rows(dims, b_batch_dim=-1):
    """Global row of the first row (box origin) of the tile each row belongs to."""
    box, _ = row_boxes(dims, b_batch_dim)
    idx = torch.arange(math.prod(dims))
    first = torch.zeros_like(idx)
    mul = 1
    for ext, b in zip(dims, box):
        c = (idx // mul) % ext
        first += (c - c % b) * mul
        mul *= ext
    return first


def geglu_rows(H, bn):
    """pack_geglu_weight's interleave: packed row p holds source row tile * bn/2 + j (value) for j = p % bn < bn/2, else
    H + tile * bn/2 + (j - bn/2) (gate), tile = p // bn."""
    p = torch.arange(2 * H)
    tile, j, hb = p // bn, p % bn, bn // 2
    return torch.where(j < hb, tile * hb + j, H + tile * hb + (j - hb))


# ---------------------------------------------------------------------------------------------------- epilogues
def bias_rows_of(bias, rows, bias_rows):
    """The fp64 bias row each output row adds: [rows, N] (per sample: row r // bias_rows), or [N]."""
    b = bias.double()
    if bias_rows > 0:
        return b[torch.arange(rows, device=b.device) // bias_rows]
    return b


def f32_exact(v):
    """v (fp64) as the fp32 value it must equal; asserts fp32 holds it (the exact-mode premise)."""
    f = v.float()
    assert torch.equal(f.double(), v), 'exact-mode premise broken: an intermediate is not exact in fp32'
    return f


def epilogue_f16(acc, alpha=1.0, bias=None, residual=None):
    """fp16(acc * alpha + bias + residual): one rounding of the fp32 sum (exact in fp32 on exact operands)."""
    v = acc * alpha
    if bias is not None:
        v = v + bias
    f32_exact(v)
    if residual is not None:
        v = v + residual.double()
    return f32_exact(v).half()


def epilogue_f32(acc, alpha=1.0, bias=None):
    v = acc * alpha
    if bias is not None:
        v = v + bias
    return f32_exact(v)


def double_rounded_f16(acc, bias, residual):
    """A plausible wrong epilogue: fp16(fp16(acc + bias) + residual)."""
    return (f32_exact(acc + bias).half().float() + residual.float()).half()


def gelu64(x):
    """Exact erf-form GELU x * Phi(x) in fp64."""
    x = x.double()
    return x * 0.5 * torch.special.erfc(-x / math.sqrt(2.0))


def gelu_tanh64(x):
    """The tanh-form GELU (F.gelu(approximate='tanh')), the wrong one for this model, in fp64."""
    x = x.double()
    return 0.5 * x * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (x + 0.044715 * x ** 3)))


def _f16_table(fn):
    """fp16 result of fn (fp64) for every fp16 bit pattern, rounded once (numpy's float64 -> float16), as int16 bits [65536]."""
    allh = torch.arange(65536, dtype=torch.int32).to(torch.int16).view(torch.float16)
    v = fn(allh.double()).numpy().astype(np.float16)
    return torch.from_numpy(v.view(np.int16).copy())


_GELU16 = {}


def gelu16_table(form='erf'):
    if form not in _GELU16:
        _GELU16[form] = _f16_table(gelu64 if form == 'erf' else gelu_tanh64)
    return _GELU16[form]


def _ordered(b):
    """fp16 bits (int16) -> an integer order (-0 and +0 both 0), so neighbours are +-1."""
    b = b.int()
    return torch.where(b < 0, -(b & 0x7FFF), b)


def _from_ordered(o):
    return torch.where(o < 0, (-o) | 0x8000, o).to(torch.int16)


def geglu_candidates(value, gate, form='erf'):
    """Outputs the GEGLU contract allows for value / gate accumulators (fp64, exact): fp16(fp16(value) * G) for the G
    within 1 fp16 ulp of fp16(gelu(fp16(gate))).  Returns int16 bits [4, ...] (the fourth covers -0 / +0 at G = 0)."""
    xh = f32_exact(value).half()
    gh = f32_exact(gate).half()
    table = gelu16_table(form).to(gh.device)
    g0 = table[gh.view(torch.int16).long() & 0xFFFF]
    o = _ordered(g0)
    cands = [_from_ordered(o - 1), g0, _from_ordered(o + 1), g0 ^ torch.tensor(-32768, dtype=torch.int16, device=g0.device)]
    outs = [(xh.float() * c.view(torch.float16).float()).half().view(torch.int16) for c in cands]
    return torch.stack(outs)


def geglu_matches(out, value, gate, form='erf'):
    """Boolean mask: out (fp16) is one of the contract's candidates."""
    ob = out.view(torch.int16)
    return (geglu_candidates(value, gate, form) == ob.unsqueeze(0)).any(0)


def fp16_ulp(v):
    """Spacing of fp16 at |v| (fp64): 2^-24 below the normal range, else 2^(floor(log2 |v|) - 10)."""
    e = torch.floor(torch.log2(v.abs().clamp_min(2.0 ** -14)))
    return torch.pow(2.0, e - 10)


def accumulation_bound(out, ref, absum, k_eff):
    """Per-element gate of the random-operand GEMMs: 1/2 ulp16 + k_eff 2^-24 absum (test_vae_resolution_gpu.py's bound)."""
    return 0.5 * fp16_ulp(torch.maximum(out.double().abs(), ref.abs())) + k_eff * 2.0 ** -24 * absum
