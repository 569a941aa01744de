"""GPU: the implicit-GEMM engine (csrc/gemm_tc.cu) against the contract restated in tests/gemm_contract.py.

A. Exact operands (small-integer activations, weights / bias / residual on a power-of-two grid; gemm_contract's module doc):
   the accumulator is exact in any K order, tile width or split, so every output element has one correct bit pattern, and
   the outputs are compared as integer bit patterns.  Outputs start out filled with a NaN sentinel and carry guard columns
   (ldo > N) and guard rows; a write outside [rows, N] fails.  Covered: every epilogue kind ops.gemm / ops.gemm_splitk reach
   (plain, bias, bias + residual, residual in place, per-sample bias on tiles that straddle samples, fp32 output, GEGLU,
   batched B with alpha and ragged rows per batch, unaligned ldo / ldr, split-K) at every tile width, a two-CTA cluster,
   the B-stationary variant and the slab epilogue; the row boxes of the model's latent and pixel sizes (conv3x3, the
   temporal conv across frame and sample edges); K and N edges (K = 8, 72, the up path's concat widths; N = 3 / 4 / 8 in a
   16-row weight allocation, ragged N); the stride-2 downsample (im2col_s2 + GEMM) against a strided conv.
B. Gaussian fp16 operands at some of the same layer shapes, every element against fp64 within
   1/2 ulp16 + K_eff 2^-24 (sum|a w| + |bias| + |res|), K_eff = taps K + 2.  `pytest -s` prints the worst ratio per case.
C. The weight packers bit for bit: pack_conv_weight (fp16 and fp32 sources, rounding / tie / overflow patterns, zero
   padding to n_alloc / k_alloc, 9 and 3 taps) and pack_geglu_weight's tile interleave, including its refusal of
   2H % bn != 0."""
import math

import pytest
import torch
import torch.nn.functional as F

import gemm_contract as GC

pytestmark = pytest.mark.gpu
dev = 'cuda'
S16, S32 = 0x7E5A, 0x7FA5A5A5          # sentinel NaN payloads no GEMM produces
GUARD_ROWS = 3
WIDTHS = [16, 64, 128, 160, 192, 224, 256]
CG2_WIDTHS = [64, 128, 160, 256]
SLAB_WIDTHS = [64, 128, 160, 192, 224, 256]
GEGLU_WIDTHS = [64, 128, 256]


@pytest.fixture(scope='module')
def ops():
    from t2v_b200 import ops as o
    return o


def num_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ---------------------------------------------------------------------------------------------------- buffers
def sentinel_buffer(rows, N, dtype, ldo=None, unaligned=False):
    """A NaN-sentinel buffer of rows + GUARD_ROWS rows of pitch ldo (default: N rounded up to 8, plus 8 guard columns) and a
    [rows, N] view of it.  unaligned: odd pitch and a start 2 or 4 bytes past a 16-byte boundary (element-wise stores)."""
    if ldo is None:
        if unaligned:
            ldo = N + 3 if (N + 3) % 2 else N + 5
        else:
            ldo = -(-N // 8) * 8 + 8
    off = 1 if unaligned else 0
    flat = torch.empty((rows + GUARD_ROWS) * ldo + off + 8, dtype=dtype, device=dev)
    flat.view(torch.int16 if dtype == torch.float16 else torch.int32).fill_(S16 if dtype == torch.float16 else S32)
    return flat, flat.as_strided((rows, N), (ldo, 1), off)


def matrix_view(t, ldr=None, unaligned=False):
    """A copy of the dense [rows, N] t in a buffer of pitch ldr (unaligned: odd, 2 bytes past a 16-byte boundary)."""
    rows, N = t.shape
    _, v = sentinel_buffer(rows, N, t.dtype, ldo=ldr, unaligned=unaligned)
    v.copy_(t)
    return v


def assert_out(flat, view, ref, what):
    """view equals ref bit for bit, and every element of flat outside view still holds the sentinel."""
    it = torch.int16 if ref.dtype == torch.float16 else torch.int32
    ob, rb = view.view(it), ref.to(dev).view(it)
    bad = (ob != rb).nonzero()
    if bad.numel():
        r, c = bad[0].tolist()
        raise AssertionError(f'{what}: {bad.shape[0]} of {ob.numel()} elements differ; first at row {r} col {c} (M-tile of 128 '
                             f'rows {r // 128}): {view[r, c].item()!r}, contract {ref[r, c].item()!r}')
    inside = torch.zeros(flat.numel(), dtype=torch.bool, device=dev)
    ldo, off = view.stride(0), view.storage_offset()
    inside.as_strided(view.shape, view.stride(), off).fill_(True)
    s = S16 if ref.dtype == torch.float16 else S32
    touched = (flat.view(it) != s) & ~inside
    if touched.any():
        p = touched.nonzero()[0].item() - off
        raise AssertionError(f'{what}: {int(touched.sum())} elements outside the output were written; first at row {p // ldo} '
                             f'col {p % ldo} (N {view.shape[1]}, ldo {ldo})')


def check_premise(name, absum, grid):
    """The exact-mode premise on the case's data: sum |a w| + |bias| + |res| below 2^BITS grid units (printed with -s)."""
    bits = GC.premise_bits(absum, grid)
    print(f'exact operands {name}: {bits:.2f} bits above the grid')
    assert bits <= GC.BITS, f'{name}: exact-mode operands need {bits:.2f} bits'
    return bits


# ---------------------------------------------------------------------------------------------------- A. variant matrix
KINDS = GC.MATRIX_KINDS
SPLITS = 4


def bs_width(tiles_m, N, K, ntaps, sms):
    """gemm_bs_bn's choice when the B-stationary variant is forced (0: not eligible), restated so the BS cases can assert it
    runs."""
    kt = ntaps * -(-K // 64)
    for c in (160, 128, 64):
        tn = -(-N // c)
        if N <= 16 or N / (tn * c) < 0.9 or kt * c * 64 * 2 > (216 - 64) * 1024 or tn > sms:
            continue
        if tiles_m < 3 * (sms // tn):
            continue
        return c
    return 0


def variants(kind):
    """(name, force_bn, force_cg, flags) of each variant the kind meets: every tile width, a two-CTA cluster, the
    B-stationary variant and the slab epilogue, where the kind allows them (cluster and slab widths rotate over the kinds)."""
    i = KINDS.index(kind)
    if kind == 'geglu':
        return [(f'bn{b}', b, 1, 0) for b in GEGLU_WIDTHS] + [('cg2', GEGLU_WIDTHS[i % 3], 2, 0), ('slab', 128, 1, 'slab')]
    v = [(f'bn{b}', b, 1, 0) for b in WIDTHS]
    if kind != 'batched':                          # a cluster shares one B tile: never across B batches
        v.append(('cg2', CG2_WIDTHS[i % 4], 2, 0))
    if kind not in ('batched', 'splitk'):
        v.append(('bs', 0, 0, 'bs'))
    if kind not in ('f32', 'unaligned', 'unaligned_f32', 'splitk'):        # those store through the slabs anyway
        v.append(('slab', SLAB_WIDTHS[i % 6], 1, 'slab'))
    return v


MATRIX = [(k, v) for k in KINDS for v in variants(k)]
_CASES = {}


def matrix_case(kind, bs):
    """The kind's operands on the GPU, the contract's output (fp64 reference on the GPU) and its premise, once per module."""
    key = (kind, bs)
    if key not in _CASES:
        c = GC.to(GC.matrix_operands(kind, bs), dev)
        name = kind + ('-bs' if bs else '')
        if kind == 'geglu':
            c['value'], c['gate'], absum, grid = GC.geglu_accumulators(c)
            check_premise(name, absum, grid)
        else:
            alpha = GC.BATCH_ALPHA if kind == 'batched' else 1.0
            c['ref'], absum = GC.tap_contract(c, f32=kind in ('f32', 'unaligned_f32'), alpha=alpha)
            check_premise(name, absum, GC.GRID * alpha)         # acc * alpha lives on the grid g * alpha
        _CASES[key] = c
    return _CASES[key]


@pytest.mark.parametrize('kind,variant', MATRIX, ids=[f'{k}-{v[0]}' for k, v in MATRIX])
def test_exact_variant_matrix(ops, kind, variant):
    name, bn, cg, fl = variant
    bs = fl == 'bs'
    c = matrix_case(kind, bs)
    rows, N = c['rows'], c.get('N', 0)
    flags = {0: 0, 'bs': ops.GEMM_FORCE_BS, 'slab': ops.GEMM_SLAB_OUT}[fl]
    if bs:
        bn_bs = bs_width(-(-rows // 128), N, c['K'], 1, num_sms())
        assert bn_bs, 'the B-stationary case must be eligible'
    what = f'{kind} {name} (BN {bn or "auto"}, CG {cg or "auto"})'
    if kind == 'geglu':
        H = c['H']
        wp, bp = ops.pack_geglu_weight(c['w'], c['b'], bn)
        flat, out = sentinel_buffer(rows, H, torch.float16, ldo=H + 16)      # GEGLU stores need ldo % 16 == 0
        ops.gemm(c['a'], wp, 2 * H, bias=bp, flags=ops.GEMM_GEGLU | flags, out=out, force_bn=bn, force_cg=cg)
        ok = GC.geglu_matches(out, c['value'], c['gate'])
        if not ok.all():
            r, col = (~ok).nonzero()[0].tolist()
            raise AssertionError(f'{what}: {int((~ok).sum())} outputs outside the GEGLU contract; first at row {r} col {col}: '
                                 f'{out[r, col].item()!r} (value {c["value"][r, col].item()}, gate {c["gate"][r, col].item()})')
        assert_out(flat, out, out.clone(), what)           # the guards
        return
    f32 = kind in ('f32', 'unaligned_f32')
    unaligned = kind in ('unaligned', 'unaligned_f32')
    flat, out = sentinel_buffer(rows, N, torch.float32 if f32 else torch.float16, unaligned=unaligned)
    res = c['res']
    if kind == 'in_place':
        out.copy_(res)
        res = out
    elif kind == 'unaligned' and res is not None:
        res = matrix_view(res, unaligned=True)
    kw = dict(bias=c['bias'], bias_rows=c['bias_rows'], bias_stride=N if c['bias_rows'] else 0, residual=res, out=out,
              force_bn=bn, force_cg=cg)
    if kind == 'batched':
        ops.gemm(c['a'], c['w'], N, dims=c['dims'], taps=c['taps'], b_batch_dim=1, alpha=GC.BATCH_ALPHA, flags=flags, **kw)
    elif kind == 'splitk':
        scratch = torch.full((SPLITS, rows, N), float('nan'), device=dev)
        _, used = ops.gemm_splitk(c['a'], c['w'], N, SPLITS, scratch=scratch, flags=flags, **kw)
        assert used == SPLITS
    else:
        ops.gemm(c['a'], c['w'], N, flags=flags | (ops.GEMM_OUT_F32 if f32 else 0), **kw)
    assert_out(flat, out, c['ref'], what)


# ---------------------------------------------------------------------------------------------------- A. conv geometry
def conv_case(seed, dims, taps, K, N, *, bias='row', bias_rows=0, residual=True, k_valid=None):
    """gemm_contract.tap_operands' case on the GPU (bias and residual by default) with its contract output and premise."""
    c = GC.to(GC.tap_operands(seed, dims, taps, K, N, bias=bias, bias_rows=bias_rows, residual=residual, k_valid=k_valid), dev)
    c['ref'], absum = GC.tap_contract(c)
    check_premise(f'tap GEMM {dims} K {K} N {N}', absum, GC.GRID)
    return c


def run_conv(ops, c, what, ldo=None, n_alloc=None, **kw):
    N = c['N']
    flat, out = sentinel_buffer(c['rows'], N, torch.float16, ldo=ldo)
    w = c['w']
    if n_alloc is not None:
        w = torch.zeros((w.shape[0], n_alloc, w.shape[2]), device=dev, dtype=torch.float16)
        w[:, :N] = c['w']
    ops.gemm(c['a'], w, N, dims=c['dims'], taps=c['taps'], bias=c['bias'], bias_rows=c['bias_rows'],
             bias_stride=N if c['bias_rows'] else 0, residual=c['res'], out=out, **kw)
    assert_out(flat, out, c['ref'], what)


# (h, w, frames, K, N): the model's latent and pixel sizes and the row box gemm_plan gives them (test_gemm_contract_cpu.py
# checks the boxes)
GEOMETRY = [
    ('320x576-l0', 40, 72, 4, 64, 64),        # [72, 1, 1]
    ('320x576-l1', 20, 36, 4, 64, 64),        # [36, 3, 1], the last box has 2 of 3 rows
    ('320x576-l2', 10, 18, 4, 64, 64),        # [18, 7, 1]
    ('320x576-l3', 5, 9, 5, 64, 64),          # [9, 5, 2]: boxes span frames
    ('576x1024-l2', 18, 32, 2, 64, 64),       # [32, 4, 1], ragged in h
    ('576x1024-l3', 9, 16, 2, 64, 64),        # [16, 8, 1], ragged in h
    ('vc512x320-l3', 5, 8, 16, 64, 64),       # [8, 5, 3], ragged over B * F frames
    ('256-l0', 32, 32, 4, 64, 64),            # [32, 4, 1]
    ('256-l1', 16, 16, 4, 64, 64),            # [16, 8, 1]
    ('256-l2', 8, 8, 4, 64, 64),              # [8, 8, 2]
    ('256-l3', 4, 4, 16, 64, 64),             # [4, 4, 8]
    ('vae-576x1024-1f', 576, 1024, 1, 128, 128),   # [128, 1, 1]
    ('vae-576x1024-2f', 576, 1024, 2, 64, 64),
]


@pytest.mark.parametrize('name,h,w,nf,K,N', GEOMETRY, ids=[gm[0] for gm in GEOMETRY])
def test_exact_conv3x3_geometry(ops, name, h, w, nf, K, N):
    """3x3 conv (bias + residual) at the row boxes of the model's sizes, with the automatic plan and the slab epilogue."""
    c = conv_case(200 + GEOMETRY.index((name, h, w, nf, K, N)), [w, h, nf], GC.conv_taps_2d(), K, N)
    run_conv(ops, c, f'{name} auto')
    run_conv(ops, c, f'{name} slab', flags=ops.GEMM_SLAB_OUT)


@pytest.mark.parametrize('variant', [(0, 0, 0), (64, 1, 0), (128, 2, 0), (160, 1, 'slab'), (256, 1, 0)],
                         ids=['auto', 'bn64', 'cg2-bn128', 'slab-bn160', 'bn256'])
def test_exact_conv3x3_per_sample_bias(ops, variant):
    """The ResBlock's conv1 with its per-sample time-embedding bias (bias_rows = F h w): at 320x576 level 3 the [9, 5, 2]
    boxes span frames, so with F = 5 one box holds the last frame of sample 0 and the first of sample 1."""
    bn, cg, fl = variant
    h, w, Fr, B = 5, 9, 5, 2
    c = conv_case(300, [w, h, Fr * B], GC.conv_taps_2d(), 320, 320, bias='sample', bias_rows=Fr * h * w,
                  residual=False)
    run_conv(ops, c, f'conv1 per-sample bias {variant}', force_bn=bn, force_cg=cg,
             flags=ops.GEMM_SLAB_OUT if fl == 'slab' else 0)


TEMPORAL = [(9, 1), (9, 2), (9, 5), (9, 16), (9, 24), (40, 16), (3, 24)]


@pytest.mark.parametrize('P,Fr', TEMPORAL, ids=[f'P{p}-F{f}' for p, f in TEMPORAL])
def test_exact_temporal_conv(ops, P, Fr):
    """(3,1,1) temporal conv, dims [P, F, B = 2]: taps read the previous and next frame, zero past each sample's first and
    last frame.  P = 9 boxes span up to 14 frames, so one box holds both samples' edge frames."""
    c = conv_case(400 + P * 31 + Fr, [P, Fr, 2], GC.conv_taps_temporal(), 64, 64)
    run_conv(ops, c, f'temporal P {P} F {Fr} auto')
    run_conv(ops, c, f'temporal P {P} F {Fr} slab', flags=ops.GEMM_SLAB_OUT)


EDGES = [
    # name, (h, w, frames), K, k_valid, N, n_alloc, ldo
    ('conv_in-unet', (40, 72, 2), 8, 4, 320, None, None),       # 4 channels padded to K = 8
    ('conv_in-vae-enc', (64, 96, 1), 8, 3, 128, None, None),    # RGB padded to K = 8
    ('up-concat-2560', (5, 9, 2), 2560, None, 1280, None, None),
    ('up-concat-1920', (10, 18, 2), 1920, None, 640, None, None),
    ('up-concat-960', (20, 36, 2), 960, None, 320, None, None),
    ('conv_out-vae-N3', (64, 96, 1), 128, None, 3, 16, 8),      # N = 3 in 16 weight rows, output pitch 8
    ('conv_out-unet-N4', (40, 72, 2), 320, None, 4, 16, 8),
    ('moments-N8', (16, 24, 1), 512, None, 8, 16, 8),
    ('ragged-N200', (10, 18, 2), 64, None, 200, None, None),
]


@pytest.mark.parametrize('name,hwf,K,k_valid,N,n_alloc,ldo', EDGES, ids=[e[0] for e in EDGES])
def test_exact_conv3x3_k_n_edges(ops, name, hwf, K, k_valid, N, n_alloc, ldo):
    h, w, nf = hwf
    c = conv_case(500 + [e[0] for e in EDGES].index(name), [w, h, nf], GC.conv_taps_2d(), K, N, k_valid=k_valid)
    run_conv(ops, c, name, ldo=ldo, n_alloc=n_alloc)
    run_conv(ops, c, f'{name} slab', ldo=ldo, n_alloc=n_alloc, flags=ops.GEMM_SLAB_OUT)


def test_exact_linear_k72(ops):
    g = GC.gen(600)
    rows, K, N = 1000, 72, 200
    a, w, b, r = GC.exact_a(g, rows, K, K), GC.exact_w(g, 1, N, K, K), GC.exact_vec(g, (N,)), GC.exact_vec(g, (rows, N))
    a, w, b, r = a.to(dev), w.to(dev), b.to(dev), r.to(dev)
    check_premise('linear K 72', a.double().abs() @ w[0].double().abs().t() + b.double().abs() + r.double().abs(), GC.GRID)
    ref = GC.epilogue_f16(a.double() @ w[0].double().t(), bias=b.double(), residual=r)
    for bn in (0, 16, 224):
        flat, out = sentinel_buffer(rows, N, torch.float16)
        ops.gemm(a, w, N, bias=b, residual=r, out=out, force_bn=bn)
        assert_out(flat, out, ref, f'linear K 72 BN {bn}')


@pytest.mark.parametrize('pad_lo,h,w,C,N', [(1, 40, 72, 64, 64), (1, 9, 15, 64, 128), (0, 64, 96, 128, 128),
                                            (0, 37, 50, 128, 64)])
def test_exact_stride2_downsample(ops, pad_lo, h, w, C, N):
    """The stride-2 downsample as the model runs it: im2col_s2 (pad_lo 1: padding 1 as the UNet's and the adapter's
    Downsample; 0: the VAE's (0, 1, 0, 1) pad) feeding a GEMM with the tap-major weight, against a strided fp64 conv."""
    g = GC.gen(700 + h + C)
    nf, k_eff = 2, 9 * C
    x = GC.exact_a(g, nf * h * w, C, k_eff).view(nf, h, w, C).to(dev)
    wt = GC.exact_w(g, 1, N, 9 * C, k_eff)[0].view(N, 3, 3, C).permute(0, 3, 1, 2).contiguous().to(dev)     # [N, C, ky, kx]
    b = GC.exact_vec(g, (N,)).to(dev)
    xd = x.permute(0, 3, 1, 2).double()
    xp = F.pad(xd, (1, 1, 1, 1) if pad_lo else (0, 1, 0, 1))
    acc = F.conv2d(xp, wt.double(), stride=2).permute(0, 2, 3, 1).reshape(-1, N)
    absum = F.conv2d(xp.abs(), wt.double().abs(), stride=2).permute(0, 2, 3, 1).reshape(-1, N) + b.double().abs()
    check_premise(f'stride2 pad_lo {pad_lo} {h}x{w}', absum, GC.GRID)
    ref = GC.epilogue_f16(acc, bias=b.double())
    col = ops.im2col_s2(x, pad_lo=pad_lo)
    wp = wt.permute(0, 2, 3, 1).reshape(1, N, 9 * C).contiguous()          # column tap * C + c, tap = ky * 3 + kx
    flat, out = sentinel_buffer(col.shape[0] * col.shape[1] * col.shape[2], N, torch.float16)
    ops.gemm(col.view(-1, 9 * C), wp, N, bias=b, out=out)
    assert_out(flat, out, ref, f'stride-2 pad_lo {pad_lo}')


# ---------------------------------------------------------------------------------------------------- B. random operands
RANDOM = [
    # name, kind, dims, K, N, bias, residual
    ('linear-l0-proj', 'linear', [9216], 320, 320, True, True),
    ('conv3x3-320x576-l1', 'conv', [36, 20, 16], 640, 640, True, False),
    ('conv3x3-up-concat-2560', 'conv', [9, 5, 16], 2560, 1280, True, True),
    ('temporal-320x576-l0', 'temporal', [2880, 16, 2], 320, 320, True, True),
    ('vae-conv3x3-576x1024', 'conv', [1024, 576, 1], 128, 128, True, True),
    ('conv_out-N4', 'conv', [72, 40, 4], 320, 4, True, False),
    ('batched-scores', 'batched', [1024, 4], 64, 1024, False, False),
    ('splitk-conv3x3-l3', 'splitk', [9, 5, 8], 1280, 1280, True, True),
]


@pytest.mark.parametrize('name,kind,dims,K,N,bias,res', RANDOM, ids=[r[0] for r in RANDOM])
def test_random_vs_fp64(ops, name, kind, dims, K, N, bias, res):
    """Gaussian fp16 operands (weights of std (taps K)^-1/2, as a trained layer's), every element against fp64 within
    1/2 ulp16 + K_eff 2^-24 (sum|a w| + |bias| + |res|), K_eff = taps K + 2: an element near zero is held to its own scale."""
    torch.manual_seed(800 + RANDOM.index((name, kind, dims, K, N, bias, res)))
    taps = {'linear': [[0]], 'conv': GC.conv_taps_2d(), 'splitk': GC.conv_taps_2d(), 'temporal': GC.conv_taps_temporal(),
            'batched': [[0, 0]]}[kind]
    rows = math.prod(dims)
    nb = dims[-1] if kind == 'batched' else len(taps)
    k_eff = len(taps) * K + 2
    a = torch.randn(rows, K, device=dev).half()
    w = (torch.randn(nb, N, K, device=dev) * (len(taps) * K) ** -0.5).half()
    b = torch.randn(N, device=dev).half() if bias else None
    r = torch.randn(rows, N, device=dev).half() if res else None
    n_alloc = max(N, 16)
    wp = torch.zeros(nb, n_alloc, K, device=dev, dtype=torch.float16)
    wp[:, :N] = w
    alpha = K ** -0.5 if kind == 'batched' else 1.0
    if kind == 'splitk':
        out, _ = ops.gemm_splitk(a, wp, N, 4, dims=dims, taps=taps, n_alloc=n_alloc, bias=b, residual=r)
    else:
        out = ops.gemm(a, wp, N, dims=dims, taps=taps, n_alloc=n_alloc, bias=b, residual=r, alpha=alpha,
                       b_batch_dim=1 if kind == 'batched' else -1)
    assert torch.isfinite(out).all()
    worst = 0.0
    per = rows // dims[-1]
    step = max(1, dims[-1] // 4) if kind != 'batched' else 1
    for o0 in range(0, dims[-1], step):
        o1 = min(dims[-1], o0 + step)
        sl = slice(o0 * per, o1 * per)
        if kind == 'batched':
            ab = a[sl].double()
            acc, absum = ab @ w[o0].double().t() * alpha, ab.abs() @ w[o0].double().abs().t() * alpha
        else:
            acc = GC.implicit_gemm64(a, dims, taps, w, outer=(o0, o1))
            absum = GC.implicit_gemm64(a, dims, taps, w, outer=(o0, o1), absolute=True)
        if b is not None:
            acc, absum = acc + b.double(), absum + b.double().abs()
        if r is not None:
            acc, absum = acc + r[sl].double(), absum + r[sl].double().abs()
        o = out[sl].double()
        ratio = ((o - acc).abs() / GC.accumulation_bound(o, acc, absum, k_eff)).max().item()
        worst = max(worst, ratio)
    print(f'random {name}: worst |out - ref| / bound {worst:.3f}')
    assert worst <= 1.0, f'{name}: {worst:.3f} x the bound'


# ---------------------------------------------------------------------------------------------------- C. packers
def f32_patterns(n, g):
    """fp32 values that round, tie (to even, both directions), overflow to +-inf, or fall to fp16 subnormals and zero,
    interleaved with ordinary Gaussian values."""
    special = torch.tensor([
        1.0 + 2.0 ** -11, 1.0 + 3 * 2.0 ** -11, 1.0 + 2.0 ** -11 + 2.0 ** -20, -(1.0 + 2.0 ** -11), 2.0 ** -25,
        3 * 2.0 ** -25, 2.0 ** -24 * 1.5, 2.0 ** -26, 65504.0, 65519.0, 65520.0, -65520.0, 1e6, -1e-30, 0.1, 1.0 / 3,
        2.0 ** -14 - 2.0 ** -25, 6e-5, -0.0], dtype=torch.float32)
    v = torch.randn(n, generator=g) * 3
    v[::3] = special[torch.arange(0, n, 3) // 3 % special.numel()]
    return v


def pack_direct(ops, w, n_alloc, k_alloc):
    """t2v_op_pack_conv_weight into a sentinel buffer with guards (ops.pack_conv_weight allocates its own)."""
    from t2v_b200 import _lib
    cout, cin = w.shape[:2]
    taps = math.prod(w.shape[2:])
    n = taps * n_alloc * k_alloc
    buf = torch.empty(n + 16, dtype=torch.float16, device=dev)
    buf.view(torch.int16).fill_(S16)
    rc = _lib.lib().t2v_op_pack_conv_weight(_lib.ptr(w), int(w.dtype == torch.float32), _lib.ptr(buf), cout, cin, taps,
                                            n_alloc, k_alloc, _lib.stream_ptr())
    _lib.check(rc, 'pack_conv_weight')
    return buf


@pytest.mark.parametrize('src', ['f16', 'f32'])
@pytest.mark.parametrize('shape,n_alloc,k_alloc', [((3, 128, 3, 3), 16, 128), ((320, 4, 3, 3), 320, 8), ((4, 320, 3, 3), 16, 320),
                                                   ((64, 64, 3, 1, 1), 64, 64), ((40, 24, 3, 1, 1), 48, 32),
                                                   ((320, 320, 3, 3), 320, 320)])
def test_pack_conv_weight(ops, src, shape, n_alloc, k_alloc):
    """[Cout, Cin, taps] -> [taps, n_alloc, k_alloc] fp16, rounded once (RN-even, overflow to inf), padding exactly +0."""
    g = torch.Generator().manual_seed(900 + sum(shape) + n_alloc + k_alloc)
    n = math.prod(shape)
    w = f32_patterns(n, g).view(shape) if src == 'f32' else (torch.randn(shape, generator=g) * 2).half()
    buf = pack_direct(ops, w.to(dev), n_alloc, k_alloc)
    cout, cin = shape[:2]
    taps = math.prod(shape[2:])
    ref = torch.zeros((taps, n_alloc, k_alloc), dtype=torch.float16)
    ref[:, :cout, :cin] = w.reshape(cout, cin, taps).permute(2, 0, 1).half()
    out = buf[:-16].view(taps, n_alloc, k_alloc).cpu()
    bad = (out.view(torch.int16) != ref.view(torch.int16)).nonzero()
    assert bad.numel() == 0, f'{bad.shape[0]} elements differ, first at {bad[0].tolist()}'
    assert (buf[-16:].view(torch.int16) == S16).all(), 'write past the packed weight'
    if src == 'f32':
        assert torch.isinf(ref.float()).any() and (ref.float() == 1.0).any()      # the patterns reached overflow and ties


@pytest.mark.parametrize('src', ['f16', 'f32'])
@pytest.mark.parametrize('bn', GEGLU_WIDTHS)
def test_pack_geglu_weight(ops, src, bn):
    """Packed row p = source row gemm_contract.geglu_rows(H, bn)[p], weight and bias, bit for bit."""
    H, K = 640, 72
    g = torch.Generator().manual_seed(950 + bn)
    w = f32_patterns(2 * H * K, g).view(2 * H, K)
    b = f32_patterns(2 * H, g)
    if src == 'f16':
        w, b = w.half(), b.half()
    wp, bp = ops.pack_geglu_weight(w.to(dev), b.to(dev), bn)
    rows = GC.geglu_rows(H, bn)
    assert torch.equal(wp[0].cpu().view(torch.int16), w[rows].half().view(torch.int16))
    assert torch.equal(bp.cpu().view(torch.int16), b[rows].half().view(torch.int16))


def test_pack_geglu_weight_refuses_ragged_tiles(ops):
    """2H % bn != 0 would leave a tile with value columns and no gates: refused, nothing written."""
    from t2v_b200 import _lib
    H, K, bn = 96, 64, 128
    w = torch.randn(2 * H, K, device=dev).half()
    b = torch.randn(2 * H, device=dev).half()
    wd = torch.empty(2 * H * K, dtype=torch.float16, device=dev)
    bd = torch.empty(2 * H, dtype=torch.float16, device=dev)
    wd.view(torch.int16).fill_(S16)
    bd.view(torch.int16).fill_(S16)
    rc = _lib.lib().t2v_op_pack_geglu_weight(_lib.ptr(w), _lib.ptr(b), 0, _lib.ptr(wd), _lib.ptr(bd), H, K, bn, _lib.stream_ptr())
    torch.cuda.synchronize()
    assert rc != 0
    assert (wd.view(torch.int16) == S16).all() and (bd.view(torch.int16) == S16).all()
    with pytest.raises(RuntimeError, match='pack_geglu_weight'):
        ops.pack_geglu_weight(w, b, bn)
