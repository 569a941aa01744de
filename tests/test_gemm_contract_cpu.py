"""CPU: tests/gemm_contract.py, the restated GEMM contract that tests/test_gemm_exact_gpu.py holds the kernels to.

* The tap geometry (implicit_gemm64 with conv_taps_2d / conv_taps_temporal) against naive per-element loops on tiny grids,
  with padding at every border and at frame and sample boundaries, and against fp64 torch convolutions.
* gemm_plan's row boxes at the model's latent and pixel sizes, and the GEGLU tile interleave against a naive loop.
* The exact operands the GPU tests use: the premise (every intermediate within 2^BITS grid units, so exact in fp32), a final
  fp16 rounding with work to do (inexact outputs and exact ties), and data that tells the contract from plausible wrong ones:
  a double rounding fp16(fp16(acc + bias) + res), the tanh-form GELU, a per-sample bias taken from a tile's first row."""
import math

import pytest
import torch
import torch.nn.functional as F

import gemm_contract as GC


def naive_taps(a, dims, taps, w):
    """acc[row, n] by explicit loops: row -> grid coordinates (d0 fastest), shifted by the tap, zero outside the grid."""
    rows, N, K = a.shape[0], w.shape[1], w.shape[2]
    out = torch.zeros(rows, N, dtype=torch.float64)
    for r in range(rows):
        coord, rr = [], r
        for e in dims:
            coord.append(rr % e)
            rr //= e
        for t, off in enumerate(taps):
            src = [c + o for c, o in zip(coord, off)]
            if any(s < 0 or s >= e for s, e in zip(src, dims)):
                continue
            sr = 0
            for s, e in reversed(list(zip(src, dims))):
                sr = sr * e + s
            for n in range(N):
                out[r, n] += sum(float(a[sr, k]) * float(w[t, n, k]) for k in range(K))
    return out


@pytest.mark.parametrize('dims,taps', [([4, 3, 3], GC.conv_taps_2d()), ([1, 1, 2], GC.conv_taps_2d()),
                                       ([5, 2, 1], GC.conv_taps_2d()), ([2, 3, 2], GC.conv_taps_temporal()),
                                       ([3, 1, 3], GC.conv_taps_temporal()),
                                       ([3, 4, 1], GC.conv_taps_temporal()), ([6], [[0]]), ([3, 2], [[0, 0]])])
def test_implicit_gemm_matches_loops(dims, taps):
    g = torch.Generator().manual_seed(sum(dims) + len(taps))
    rows, K, N = math.prod(dims), 3, 2
    a = torch.randint(-3, 4, (rows, K), generator=g).double()
    w = torch.randint(-3, 4, (len(taps), N, K), generator=g).double()
    ref = naive_taps(a, dims, taps, w)
    assert torch.equal(GC.implicit_gemm64(a, dims, taps, w), ref)
    assert torch.equal(GC.implicit_gemm64(a, dims, taps, w, absolute=True), naive_taps(a.abs(), dims, taps, w.abs()))
    per = rows // dims[-1]
    for o0 in range(dims[-1]):              # one outermost index at a time, with the halo its taps read
        assert torch.equal(GC.implicit_gemm64(a, dims, taps, w, outer=(o0, o0 + 1)), ref[o0 * per:(o0 + 1) * per])


def test_conv_taps_match_torch_convolutions():
    """conv_taps_2d with w[ky * 3 + kx] = weight[:, :, ky, kx] is Conv2d(padding 1) per frame; conv_taps_temporal with
    w[kt] = weight[:, :, kt] is Conv3d((3, 1, 1), padding (1, 0, 0)) per sample, zero past each sample's end frames."""
    g = torch.Generator().manual_seed(1)
    nf, h, w_, C, N = 3, 5, 7, 4, 6
    x = torch.randn(nf, h, w_, C, generator=g, dtype=torch.float64)
    wt = torch.randn(N, C, 3, 3, generator=g, dtype=torch.float64)
    ours = GC.implicit_gemm64(x.reshape(-1, C), [w_, h, nf], GC.conv_taps_2d(), wt.permute(2, 3, 0, 1).reshape(9, N, C))
    ref = F.conv2d(x.permute(0, 3, 1, 2), wt, padding=1).permute(0, 2, 3, 1).reshape(-1, N)
    assert torch.allclose(ours, ref, rtol=0, atol=1e-12)
    B, Fr, P = 2, 4, 5
    x = torch.randn(B, Fr, P, C, generator=g, dtype=torch.float64)
    wt = torch.randn(N, C, 3, 1, 1, generator=g, dtype=torch.float64)
    ours = GC.implicit_gemm64(x.reshape(-1, C), [P, Fr, B], GC.conv_taps_temporal(), wt[:, :, :, 0, 0].permute(2, 0, 1))
    x5 = x.permute(0, 3, 1, 2).reshape(B, C, Fr, P, 1)
    ref = F.conv3d(x5, wt, padding=(1, 0, 0)).reshape(B, N, Fr, P).permute(0, 2, 3, 1).reshape(-1, N)
    assert torch.allclose(ours, ref, rtol=0, atol=1e-12)


@pytest.mark.parametrize('dims,box', [
    ([72, 40, 4], [72, 1, 1]), ([36, 20, 4], [36, 3, 1]), ([18, 10, 4], [18, 7, 1]), ([9, 5, 5], [9, 5, 2]),
    ([32, 18, 2], [32, 4, 1]), ([16, 9, 2], [16, 8, 1]), ([8, 5, 16], [8, 5, 3]), ([32, 32, 4], [32, 4, 1]),
    ([16, 16, 4], [16, 8, 1]), ([8, 8, 4], [8, 8, 2]), ([4, 4, 16], [4, 4, 8]), ([1024, 576, 2], [128, 1, 1]),
    ([9, 5, 2], [9, 5, 2]), ([9, 24, 2], [9, 14, 1]), ([9, 1, 2], [9, 1, 2]), ([40, 16, 2], [40, 3, 1]),
    ([3, 24, 2], [3, 24, 1]), ([300, 3], [128, 1])])
def test_row_boxes(dims, box):
    """The boxes test_gemm_exact_gpu.py's geometry cases rely on (the 320x576, 576x1024, VideoCrafter 512x320 and 256^2
    latent levels, the VAE at 576x1024 pixels, the temporal conv's [P, F, 2] grids)."""
    assert GC.row_boxes(dims)[0] == box


def test_row_boxes_batched_and_first_rows():
    box, tiles = GC.row_boxes([300, 3], b_batch_dim=1)
    assert box == [128, 1] and tiles == [3, 3]
    box, _ = GC.row_boxes([9, 5, 4], b_batch_dim=2)
    assert box == [9, 5, 1]
    first = GC.tile_first_rows([9, 5, 4])               # box [9, 5, 2]: frames 0-1 and 2-3 share tiles
    assert first[45 * 1 + 7].item() == 0 and first[45 * 3 + 1].item() == 90
    assert torch.equal(GC.tile_first_rows([300]), torch.arange(300) // 128 * 128)


@pytest.mark.parametrize('H,bn', [(256, 64), (640, 128), (512, 256), (64, 128)])
def test_geglu_rows(H, bn):
    rows = GC.geglu_rows(H, bn)
    hb = bn // 2
    expect = []
    for tile in range(2 * H // bn):
        expect += [tile * hb + j for j in range(hb)] + [H + tile * hb + j for j in range(hb)]
    assert rows.tolist() == expect
    assert sorted(expect) == list(range(2 * H))


def test_gelu_table_against_math_erf():
    """The exact-GELU fp16 table the GEGLU gate uses, spot-checked against math.erf in Python floats."""
    table = GC.gelu16_table('erf')
    xs = torch.tensor([-7.5, -3.0, -1.25, -0.5, -0.001, 0.0, 0.3, 1.0, 2.5, 6.0], dtype=torch.float16)
    for x in xs.tolist():
        exact = x * 0.5 * (1.0 + math.erf(x / math.sqrt(2.0)))
        got = table[torch.tensor([x], dtype=torch.float16).view(torch.int16).long() & 0xFFFF].view(torch.float16).item()
        assert abs(got - exact) <= 0.5 * GC.fp16_ulp(torch.tensor(exact)).item() + 1e-12, (x, got, exact)


# ------------------------------------------------------------------------------------------------ the GPU tests' data
@pytest.fixture(scope='module')
def matrix():
    """The variant matrix's operands and contract outputs (fp64 on the CPU)."""
    out = {}
    for kind in GC.MATRIX_KINDS:
        c = GC.matrix_operands(kind)
        if kind == 'geglu':
            c['value'], c['gate'], c['absum'], c['grid'] = GC.geglu_accumulators(c)
        else:
            alpha = GC.BATCH_ALPHA if kind == 'batched' else 1.0
            c['ref'], c['absum'] = GC.tap_contract(c, f32=kind in ('f32', 'unaligned_f32'), alpha=alpha)
            c['grid'] = GC.GRID * alpha
        out[kind] = c
    return out


def test_operands_are_fp16_and_on_grid(matrix):
    for kind, c in matrix.items():
        assert torch.equal(c['a'].double(), torch.round(c['a'].double())), kind
        if kind == 'geglu':
            H = c['H']
            assert GC.on_grid(c['w'][:H], GC.GRID) and GC.on_grid(c['w'][H:], GC.GATE_GRID)
            assert GC.on_grid(c['b'][:H], GC.GRID) and GC.on_grid(c['b'][H:], GC.GATE_GRID)
            continue
        for t in (c['w'], c['bias'], c['res']):
            if t is not None:
                assert torch.isfinite(t).all() and GC.on_grid(t, GC.GRID), kind


def test_premise(matrix):
    """Every intermediate of every kind within 2^BITS grid units (fp32 holds it with 8 bits to spare)."""
    for kind, c in matrix.items():
        bits = GC.premise_bits(c['absum'], c['grid'])
        assert bits <= GC.BITS, (kind, bits)


@pytest.mark.parametrize('kind', ['plain', 'bias', 'residual', 'ps_bias', 'batched', 'splitk'])
def test_final_rounding_has_work(matrix, kind):
    """Most outputs need more than fp16's 11 significant bits, and some are exact ties."""
    frac, ties = GC.inexact_fraction(_exact_sum(matrix[kind]))
    assert frac > 0.5 and ties > 100, (kind, frac, ties)


def _exact_sum(c):
    """acc * alpha + bias + res in fp64 (before the fp16 rounding)."""
    a, w = c['a'].double(), c['w'].double()
    if w.shape[0] != len(c['taps']):
        nb = w.shape[0]
        return (a.view(nb, -1, a.shape[1]) @ w.transpose(1, 2)).reshape(c['rows'], -1) * GC.BATCH_ALPHA
    v = GC.implicit_gemm64(a, c['dims'], c['taps'], w)
    if c['bias'] is not None:
        v = v + GC.bias_rows_of(c['bias'], c['rows'], c['bias_rows'])
    if c['res'] is not None:
        v = v + c['res'].double()
    return v


def test_double_rounding_is_told_apart(matrix):
    c = matrix['residual']
    acc = GC.implicit_gemm64(c['a'], c['dims'], c['taps'], c['w'])
    wrong = GC.double_rounded_f16(acc, c['bias'].double(), c['res'])
    n = (wrong.view(torch.int16) != c['ref'].view(torch.int16)).sum().item()
    assert n > 1000, n


def test_tanh_gelu_is_told_apart(matrix):
    c = matrix['geglu']
    xh = c['value'].float().half()
    gh = c['gate'].float().half()
    g_tanh = GC.gelu16_table('tanh')[gh.view(torch.int16).long() & 0xFFFF].view(torch.float16)
    wrong = (xh.float() * g_tanh.float()).half()
    bad = ~GC.geglu_matches(wrong, c['value'], c['gate'])
    assert bad.sum().item() > 100, bad.sum().item()
    right = GC.geglu_matches((xh.float() * GC.gelu16_table('erf')[gh.view(torch.int16).long() & 0xFFFF]
                              .view(torch.float16).float()).half(), c['value'], c['gate'])
    assert right.all()
    # the gates cover GELU's curved range, not only its linear and zero tails
    gf = gh.float()
    assert ((gf > -3) & (gf < 3)).float().mean().item() > 0.3


def per_sample_from_tile_start(c, dims):
    """A plausible wrong per-sample bias: the row of the sample holding the tile's first row, for every row of the tile."""
    first = GC.tile_first_rows(dims)
    acc = GC.implicit_gemm64(c['a'], c['dims'], c['taps'], c['w'])
    return GC.epilogue_f16(acc, bias=c['bias'].double()[first // c['bias_rows']], residual=c['res'])


def test_tile_start_bias_is_told_apart(matrix):
    c = matrix['ps_bias']
    wrong = per_sample_from_tile_start(c, c['dims'])
    assert (wrong.view(torch.int16) != c['ref'].view(torch.int16)).sum().item() > 1000
    # the 3x3 conv case of test_gemm_exact_gpu.py: [9, 5, 2] boxes over F = 5 frames of 2 samples
    h, w, Fr, B = 5, 9, 5, 2
    cc = GC.tap_operands(300, [w, h, Fr * B], GC.conv_taps_2d(), 320, 320, bias='sample', bias_rows=Fr * h * w)
    ref, absum = GC.tap_contract(cc)
    assert GC.premise_bits(absum, GC.GRID) <= GC.BITS
    wrong = per_sample_from_tile_start(cc, cc['dims'])
    assert (wrong.view(torch.int16) != ref.view(torch.int16)).sum().item() > 100


def test_exact_ties_and_overflow_helpers():
    v = torch.tensor([1.0 + 2.0 ** -11, 1.0 + 3 * 2.0 ** -11, 1.0 + 2.0 ** -12, 2048.0 + 1.0, 3.0], dtype=torch.float64)
    frac, ties = GC.inexact_fraction(v)
    assert ties == 3 and frac == pytest.approx(4 / 5)
    with pytest.raises(AssertionError):
        GC.f32_exact(torch.tensor([1.0 + 2.0 ** -30], dtype=torch.float64))
