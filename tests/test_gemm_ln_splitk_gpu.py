"""GPU: the two GEMM paths that ops.gemm does not reach, checked at op level against fp64 references of the same operation
on the same fp16 inputs, plus the four small launchers the model uses around them.

* LayerNorm fold (ops.ln_linear = the launchers of ln_linear in runtime.cu): the fold kernel's folded weight, column sums and
  fp32 bias; the row statistics; the fused output at the model's shapes; its independence of the tile width; and how its
  error grows with |mean| / std of a row (the epilogue subtracts mean * colsum from the accumulator in fp32).
* Split-K (ops.gemm_splitk = the path Builder::gemm takes for contractions that cannot fill the GPU): fp32 partials per
  split and the fix-up pass, at the split schedule's edges (normalised split counts, a short last split, splits that start
  in the middle of a tap), with the scratch filled with NaN so a partial the GEMM did not write cannot go unnoticed.
* upsample2x, im2col_s2, time_sinusoid, small_linear.

Gate for GEMM outputs: max |out - ref| <= 2e-3 * max |ref|, as tests/test_ops_gpu.py."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
dev = 'cuda'
EPS = 1e-5
U32 = 2.0 ** -24          # unit roundoff of fp32
GATE = 2e-3


@pytest.fixture(scope='module')
def ops():
    from t2v_b200 import ops as o
    return o


def rand(*shape, scale=1.0, gen=None):
    return (torch.randn(*shape, device=dev, generator=gen) * scale).half()


def maxerr(out, ref):
    return (out.double() - ref.double()).abs().max().item()


def rel(out, ref):
    return maxerr(out, ref) / ref.double().abs().max().item()


def ulp16(v):
    """fp16 spacing at |v| (subnormal spacing below 2^-14)."""
    e = torch.floor(torch.log2(v.double().abs().clamp_min(2.0 ** -14)))
    return torch.pow(2.0, e - 10)


def ln_params(K, N, seed, bias=True):
    g = torch.Generator(device=dev).manual_seed(seed)
    w = rand(N, K, scale=K ** -0.5, gen=g)
    b = rand(N, gen=g) if bias else None
    gamma = (1 + 0.2 * torch.randn(K, device=dev, generator=g)).half()
    beta = (0.2 * torch.randn(K, device=dev, generator=g)).half()
    return w, b, gamma, beta


def ln_ref64(x, w, b, gamma, beta, residual=None):
    """Linear(LayerNorm(x)) in fp64 (biased variance, eps 1e-5)."""
    xd = x.double()
    y = F.layer_norm(xd, (x.shape[1],), gamma.double(), beta.double(), EPS) @ w.double().t()
    if b is not None:
        y = y + b.double()
    if residual is not None:
        y = y + residual.double()
    return y


def geglu_ref64(h):
    xa, gate = h.chunk(2, dim=-1)
    return xa * F.gelu(gate)


# ------------------------------------------------------------------------------------------------- LayerNorm fold
@pytest.mark.parametrize('K,N', [(320, 960), (768, 2304), (1280, 1280), (72, 200)])
def test_fold_intermediates(ops, K, N):
    """w_folded = fp16(w * gamma) bit for bit; colsum = sum of the *folded fp16* weights; bias32 = w @ beta + bias.
    Both sums are fp32 over K terms in the kernel's order (32 lanes of K / 32 terms, then a 5-level shuffle tree), so
    their error is at most (K / 32 + 5) * 2^-24 * sum |terms|."""
    w, b, gamma, beta = ln_params(K, N, seed=10)
    x = rand(130, K)
    _, wf, colsum, bias32, _ = ops.ln_linear(x, w, b, gamma, beta)
    assert torch.equal(wf, (w.float() * gamma.float()).half())
    depth = math.ceil(K / 32) + 5
    ref_cs = wf.double().sum(1)
    tol_cs = depth * U32 * wf.double().abs().sum(1)
    assert ((colsum.double() - ref_cs).abs() <= tol_cs).all(), (colsum.double() - ref_cs).abs().max().item()
    # the same bound cannot be met by the sum of the unrounded products w * gamma: the gate tells the two apart
    unrounded = (w.double() * gamma.double()).sum(1)
    assert ((unrounded - ref_cs).abs() > tol_cs).any()
    prod = w.double() * beta.double()
    ref_b = prod.sum(1) + b.double()
    tol_b = (depth + 1) * U32 * (prod.abs().sum(1) + b.double().abs())
    assert ((bias32.double() - ref_b).abs() <= tol_b).all(), (bias32.double() - ref_b).abs().max().item()


def rowstat_ref(x):
    xd = x.double()
    mean = xd.mean(1)
    var = ((xd - mean[:, None]) ** 2).mean(1)
    return mean, 1.0 / torch.sqrt(var + EPS)


@pytest.mark.parametrize('rows,C,pitch', [(1000, 64, 64), (1000, 320, 320), (777, 640, 640), (1000, 768, 768),
                                          (1000, 1024, 1024), (500, 1280, 1280), (300, 2048, 2048), (1000, 320, 1000),
                                          (24576, 320, 320), (24576 + 77, 1024, 1024)])
def test_rowstats(ops, rows, C, pitch):
    """(mean, rstd) per row vs fp64.  C = 1024 runs the 5-vector kernel with padding lanes; pitch > C reads x as a column
    slice of a wider matrix; 24576 rows > 132 SMs * 8 blocks * 16 rows run the grid-stride loop and rows whose pair
    partner is absent.  Rows have different means and scales, so a row's statistics taken from another row are caught."""
    g = torch.Generator(device=dev).manual_seed(rows + C)
    base = torch.randn(rows, pitch, device=dev, generator=g)
    loc = torch.randn(rows, 1, device=dev, generator=g) * 2
    scale = torch.rand(rows, 1, device=dev, generator=g) * 3 + 0.2
    xw = (base * scale + loc).half()
    x = xw[:, :C]
    w, b, gamma, beta = ln_params(C, 64, seed=11)
    _, _, _, _, rs = ops.ln_linear(x, w, b, gamma, beta)
    mean, rstd = rowstat_ref(x)
    # mean: a lane adds its 8 * ceil(C / 256) values pairwise (two roundings per pair), then a 5-level shuffle tree and the
    # scaling by 1 / C; rstd: two-pass fp32 variance, relative error of the same order
    tol_m = (8 * math.ceil(C / 256) + 7) * U32 * x.double().abs().mean(1)
    assert ((rs[:, 0].double() - mean).abs() <= tol_m).all(), (rs[:, 0].double() - mean).abs().max().item()
    relr = ((rs[:, 1].double() - rstd).abs() / rstd).max().item()
    assert relr < 1e-5, relr


LN_CASES = [
    # rows, K, N, geglu, residual                      model layer
    (1024, 320, 960, False, False),                  # level-0 transformer q|k|v
    (1000, 640, 1920, False, False),                 # level-1 q|k|v, ragged rows
    (300, 1280, 3840, False, False),                 # level-2 q|k|v, ragged rows
    (2048, 640, 640, False, False),                  # cross-attention to_q
    (154, 768, 2304, False, False),                  # ViT-L/14 q|k|v, 77 * 2 rows
    (231, 1024, 3072, False, False),                 # OpenCLIP ViT-H q|k|v, 77 * 3 rows
    (154, 768, 3072, False, False),                  # ViT-L/14 fc1
    (1000, 320, 2560, True, False),                  # LN + GEGLU feed-forward, 2H = 2560
    (129, 72, 200, False, False),                    # ragged N: zero-filled column operands past N
    (1000, 320, 320, False, True),                   # with a residual
]


@pytest.mark.parametrize('rows,K,N,geglu,res', LN_CASES)
def test_ln_linear_vs_fp64(ops, rows, K, N, geglu, res):
    """Fused output vs fp64 Linear(LayerNorm(x)), and not worse than the library's unfused path (ops.layernorm, which
    rounds the normalised rows to fp16, then ops.gemm) on the same inputs."""
    torch.manual_seed(rows + K + N)
    x = (torch.randn(rows, K, device=dev) * 2 + 0.5).half()
    w, b, gamma, beta = ln_params(K, N, seed=rows + N)
    r = rand(rows, N // 2 if geglu else N) if res else None
    if geglu:
        bn = 128
        wp, bp = ops.pack_geglu_weight(w, b, bn)
        out = ops.ln_linear(x, wp, bp, gamma, beta, flags=ops.GEMM_GEGLU, force_bn=bn)[0]
        ref = geglu_ref64(ln_ref64(x, w, b, gamma, beta))
        unfused = ops.gemm(ops.layernorm(x, gamma, beta), wp, N, bias=bp, flags=ops.GEMM_GEGLU, force_bn=bn)
    else:
        out = ops.ln_linear(x, w, b, gamma, beta, residual=r)[0]
        ref = ln_ref64(x, w, b, gamma, beta, r)
        unfused = ops.gemm(ops.layernorm(x, gamma, beta), w.view(1, N, K), N, bias=b, residual=r)
    e_fused, e_unfused = rel(out, ref), rel(unfused, ref)
    print(f'ln_linear rows {rows} K {K} N {N} geglu {geglu} res {res}: fused {e_fused:.3e} unfused {e_unfused:.3e}')
    assert e_fused < GATE
    assert e_fused <= 1.25 * e_unfused, (e_fused, e_unfused)


WIDTHS = [16, 128, 160, 192, 224, 256]
CG2_WIDTHS = [64, 128, 160, 256]


@pytest.mark.parametrize('rows,K,N,res', [(1000, 320, 960, False), (129, 72, 200, True), (154, 768, 2304, False)])
def test_ln_linear_widths(ops, rows, K, N, res):
    """Every tile width keeps each element's K order and epilogue arithmetic: equal to the BN = 64 output bit for bit."""
    torch.manual_seed(20)
    x = (torch.randn(rows, K, device=dev) + 1).half()
    w, b, gamma, beta = ln_params(K, N, seed=21)
    r = rand(rows, N) if res else None
    ref = ops.ln_linear(x, w, b, gamma, beta, residual=r, force_bn=64)[0]
    for bn, cg in [(bn, 1) for bn in WIDTHS] + [(bn, 2) for bn in CG2_WIDTHS]:
        out = ops.ln_linear(x, w, b, gamma, beta, residual=r, force_bn=bn, force_cg=cg)[0]
        assert torch.equal(out, ref), f'BN {bn} CG {cg}: max |diff| {maxerr(out, ref)}'


def test_ln_geglu_widths(ops):
    """LN + GEGLU: the weights are packed per tile width; every width and cluster shape gives the BN = 64 output."""
    torch.manual_seed(22)
    K, H, rows = 320, 640, 1000
    x = (torch.randn(rows, K, device=dev) + 1).half()
    w, b, gamma, beta = ln_params(K, 2 * H, seed=23)

    def run(bn, cg):
        wp, bp = ops.pack_geglu_weight(w, b, bn)
        return ops.ln_linear(x, wp, bp, gamma, beta, flags=ops.GEMM_GEGLU, force_bn=bn, force_cg=cg)[0]
    ref = run(64, 1)
    for bn, cg in [(128, 1), (256, 1), (64, 2), (128, 2), (256, 2)]:
        out = run(bn, cg)
        assert torch.equal(out, ref), f'BN {bn} CG {cg}: max |diff| {maxerr(out, ref)}'


# Measured on H100 SXM (80 GB HBM3, 700 W): the largest (err - plain gate) / (2^-24 K |mean| rstd max|W'|) over the rows
# of test_ln_conditioning is 0.0 at K = 320 and 0.13 at K = 1280 (the test prints it with -s); without subtracting the plain
# gate, err / (2^-24 K |mean| rstd max|W'|) peaks at 3.9 / 1.7 on the |mean| / std = 100 rows.
C_COND = 1.0


@pytest.mark.parametrize('K,N', [(320, 960), (1280, 1280)])
def test_ln_conditioning(ops, K, N):
    """Rows with |mean| / std in {0, 1, 10, 100}, and constant rows (variance 0: rstd = 1 / sqrt(eps) ~ 316, the output is
    exactly W @ beta + bias).  The fold computes acc - mean * colsum in fp32 from two sums of size ~ K |mean| max|W'|, so a
    row's error may grow as 2^-24 K |mean| rstd max|W'|; each row must stay within C_COND times that plus the plain gate.
    A wrong mean or colsum is an O(1) error at every ratio."""
    torch.manual_seed(30)
    per = 128
    parts, means = [], []
    for ratio in (0.0, 1.0, 10.0, 100.0):
        z = torch.randn(per, K, device=dev)
        z = (z - z.mean(1, keepdim=True)) / z.std(1, keepdim=True)
        sign = torch.where(torch.rand(per, 1, device=dev) < 0.5, -1.0, 1.0)
        parts.append(z + ratio * sign)
        means.append(torch.full((per,), ratio))
    const = torch.tensor([3.0, -0.5, 40.0, 1.0], device=dev)[:, None].expand(4, K)
    parts.append(const)
    x = torch.cat(parts).half()
    w, b, gamma, beta = ln_params(K, N, seed=31)
    out, wf, _, _, rs = ops.ln_linear(x, w, b, gamma, beta)
    ref = ln_ref64(x, w, b, gamma, beta)
    mean, rstd = rowstat_ref(x)
    err = (out.double() - ref).abs().max(1).values
    scale = U32 * K * mean.abs() * rstd * wf.double().abs().max()
    plain = GATE * ref.abs().max()
    c_meas = ((err - plain).clamp_min(0) / scale.clamp_min(1e-30)).max().item()
    c_raw = (err / scale.clamp_min(1e-30))
    nconst = const.shape[0]
    rows_rel = err / ref.abs().max(1).values
    print(f'conditioning K {K}: c over the plain gate {c_meas:.3f}; err / scale per ratio '
          + ', '.join(f'{r}: {c_raw[i * per:(i + 1) * per].max().item():.3f}' for i, r in enumerate((0, 1, 10, 100)))
          + f'; constant rows err / max|ref| {[round(v, 6) for v in rows_rel[-nconst:].tolist()]}'
          + f', rstd {rs[-nconst:, 1].tolist()}')
    assert (err <= C_COND * scale + plain).all(), (err / (C_COND * scale + plain)).max().item()
    # the constant rows: exactly W @ beta + bias in fp64
    cref = w.double() @ beta.double() + b.double()
    assert torch.allclose(ref[-nconst:], cref.expand(nconst, N), rtol=0, atol=1e-9)


# ------------------------------------------------------------------------------------------------------- split-K
def kt_of(K, ntaps):
    return ntaps * ((K + 63) // 64)


def effective_splits(kt, S):
    kps = -(-kt // S)
    return -(-kt // kps)


def nan_scratch(S, rows, N):
    return torch.full((S, rows, N), float('nan'), device=dev)


def conv2d_ref64(x, wt, b, NF, h, w):
    y = F.conv2d(x.permute(0, 3, 1, 2).double(), wt.double(), None, padding=1).permute(0, 2, 3, 1).reshape(NF * h * w, -1)
    return y


def temporal_ref64(x, wt, B, Fr, P):
    C = x.shape[-1]
    x5 = x.view(B, Fr, P, C).permute(0, 3, 1, 2).reshape(B, C, Fr, P, 1).double()
    y = F.conv3d(x5, wt.double(), None, padding=(1, 0, 0))
    return y.reshape(B, -1, Fr, P).permute(0, 2, 3, 1).reshape(B * Fr * P, -1)


def splitk_case(ops, kind, seed):
    """(kwargs of gemm / gemm_splitk, fp64 contraction without bias / residual, rows, N)."""
    g = torch.Generator(device=dev).manual_seed(seed)
    if kind[0] == 'linear':
        _, M, K, N = kind
        a = rand(M, K, gen=g)
        w = rand(N, K, scale=K ** -0.5, gen=g)
        return dict(a=a, w_packed=w.view(1, N, K), N=N), a.double() @ w.double().t(), M, N
    if kind[0] == 'conv3x3':
        _, NF, h, w_, K, N = kind
        x = rand(NF, h, w_, K, gen=g)
        wt = rand(N, K, 3, 3, scale=(9 * K) ** -0.5, gen=g)
        return (dict(a=x.view(-1, K), w_packed=ops.pack_conv_weight(wt), N=N, dims=[w_, h, NF], taps=ops.conv_taps_2d()),
                conv2d_ref64(x, wt, None, NF, h, w_), NF * h * w_, N)
    _, B, Fr, P, K, N = kind
    x = rand(B, Fr, P, K, gen=g)
    wt = rand(N, K, 3, 1, 1, scale=(3 * K) ** -0.5, gen=g)
    return (dict(a=x.view(-1, K), w_packed=ops.pack_conv_weight(wt), N=N, dims=[P, Fr, B], taps=ops.conv_taps_temporal()),
            temporal_ref64(x, wt, B, Fr, P), B * Fr * P, N)


SPLITK_CASES = [
    # kind, requested S, per-sample bias rows (0: one bias row), residual
    (('linear', 768, 1280, 320), 4, 0, True),            # plain rows, kt = 20
    (('linear', 3072, 640, 640), 2, 0, True),            # S = 2
    (('linear', 200, 1920, 256), 7, 100, True),          # kt = 30, S 7 -> 6
    (('conv3x3', 6, 4, 4, 640, 640), 8, 48, True),       # 4x4 frames, kt = 90, S = 8: 8 splits of 12 (last 6), mid-tap starts
    (('conv3x3', 3, 8, 8, 1280, 640), 8, 0, True),       # 8x8, kt = 180, S = 8: seven splits of 23, then 19
    (('conv3x3', 2, 8, 8, 640, 320), 4, 64, False),      # kt = 90, S = 4: splits of 23 (last 21) start mid-tap
    (('conv3x3', 5, 4, 4, 320, 320), 4, 16, True),       # NF = 5 at 4x4: 80-row boxes that do not fill 128 rows
    (('temporal', 2, 4, 16, 1280, 640), 8, 64, True),    # 3 temporal taps, kt = 60, S = 8: splits of 8 (last 4)
    (('temporal', 2, 4, 16, 640, 640), 7, 0, True),      # kt = 30, S 7 -> 6: splits of 5 start in the middle of a tap
]


def splitk_operands(case, rows, N, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    _, _, bias_rows, res = case
    if bias_rows:
        bias = rand(rows // bias_rows, N, gen=g)
        bref = bias.double().repeat_interleave(bias_rows, 0)
    else:
        bias = rand(N, gen=g)
        bref = bias.double()
    r = rand(rows, N, gen=g) if res else None
    return dict(bias=bias, bias_rows=bias_rows, bias_stride=N if bias_rows else 0, residual=r), bref


@pytest.mark.parametrize('case', SPLITK_CASES, ids=lambda c: f'{c[0][0]}-S{c[1]}-{"x".join(map(str, c[0][1:]))}')
def test_splitk_vs_fp64(ops, case):
    """Output vs fp64 with bias (per sample where bias_rows > 0) and residual applied by the fix-up pass; the scratch is NaN
    before the call, sized for the requested S, so a partial the GEMM did not write (or a reduce over more splits than
    ran) shows.  The effective split count is the schedule's; the output agrees with the unsplit GEMM within the gate."""
    kind, S, _, _ = case
    kw, acc, rows, N = splitk_case(ops, kind, seed=40)
    extra, bref = splitk_operands(case, rows, N, seed=41)
    ref = acc + bref + (extra['residual'].double() if extra['residual'] is not None else 0)
    kt = kt_of(kw['a'].shape[1], len(kw.get('taps', [[0]])))
    out, used = ops.gemm_splitk(splits=S, scratch=nan_scratch(S, rows, N), **kw, **extra)
    assert used == effective_splits(kt, S)
    assert torch.isfinite(out).all()
    assert rel(out, ref) < GATE, rel(out, ref)
    whole = ops.gemm(**kw, **extra)
    assert rel(whole, ref) < GATE
    assert maxerr(out, whole) <= GATE * ref.abs().max().item()


@pytest.mark.parametrize('kt_K,ntaps,S,expect', [(1920, 1, 7, 6), (640, 3, 7, 6), (1280, 9, 8, 8), (640, 9, 7, 7),
                                                   (1280, 1, 8, 7), (576, 1, 4, 3), (128, 1, 8, 2), (64, 3, 8, 3),
                                                   (1280, 3, 2, 2), (4480, 1, 8, 8)])
def test_splitk_schedule(ops, kt_K, ntaps, S, expect):
    """The split count the op reports is the schedule's (ceil(kt / S) iterations per split, empty splits dropped)."""
    kt = kt_of(kt_K, ntaps)
    assert effective_splits(kt, S) == expect
    rows, N = 256, 64
    g = torch.Generator(device=dev).manual_seed(50)
    if ntaps == 1:
        kw = dict(a=rand(rows, kt_K, gen=g), w_packed=rand(1, N, kt_K, scale=kt_K ** -0.5, gen=g), N=N)
        ref = kw['a'].double() @ kw['w_packed'][0].double().t()
    else:
        taps = ops.conv_taps_2d()[:ntaps] if ntaps != 3 else ops.conv_taps_temporal()
        dims = [16, 4, 4] if ntaps == 3 else [8, 8, 4]
        kw = dict(a=rand(rows, kt_K, gen=g), w_packed=rand(ntaps, N, kt_K, scale=(ntaps * kt_K) ** -0.5, gen=g), N=N,
                  dims=dims, taps=taps)
        ref = ops.gemm(**kw).double()
    out, used = ops.gemm_splitk(splits=S, scratch=nan_scratch(S, rows, N), **kw)
    assert used == expect
    assert torch.isfinite(out).all()
    assert rel(out, ref) < GATE


@pytest.mark.parametrize('case', [SPLITK_CASES[3], SPLITK_CASES[4], SPLITK_CASES[7], SPLITK_CASES[0]],
                         ids=lambda c: f'{c[0][0]}-S{c[1]}')
def test_splitk_invariants(ops, case):
    """At a fixed S the output is bit-identical across tile widths and cluster shapes (each element's K order and the
    fix-up's split order do not depend on them) and from one run to the next."""
    kind, S, _, _ = case
    kw, _, rows, N = splitk_case(ops, kind, seed=60)
    extra, _ = splitk_operands(case, rows, N, seed=61)
    first, _ = ops.gemm_splitk(splits=S, scratch=nan_scratch(S, rows, N), force_bn=64, **kw, **extra)
    again, _ = ops.gemm_splitk(splits=S, scratch=nan_scratch(S, rows, N), force_bn=64, **kw, **extra)
    assert torch.equal(first, again)
    for bn in (64, 128, 160, 256):
        for cg in (1, 2):
            out, _ = ops.gemm_splitk(splits=S, scratch=nan_scratch(S, rows, N), force_bn=bn, force_cg=cg, **kw, **extra)
            assert torch.equal(out, first), f'BN {bn} CG {cg}: max |diff| {maxerr(out, first)}'


def test_splitk_rejections(ops):
    """Each problem split-K cannot take is refused with an error before anything runs: the output and the scratch keep
    their sentinel contents."""
    M, K, N, S = 300, 256, 64, 2
    a = rand(M, K)
    w = rand(1, N, K, scale=K ** -0.5)
    cases = {
        'geglu': dict(a=a, w_packed=w, N=N, flags=ops.GEMM_GEGLU),
        'fp32 output': dict(a=a, w_packed=w, N=N, flags=ops.GEMM_OUT_F32),
        'batched B': dict(a=rand(3 * 100, 64), w_packed=rand(3, N, 64), N=N, K=64, dims=[100, 3], taps=[[0, 0]],
                          b_batch_dim=1),
        'alpha': dict(a=a, w_packed=w, N=N, alpha=0.5),
        'N % 8': dict(a=a, w_packed=rand(1, 60, K), N=60),
        'scratch': dict(a=a, w_packed=w, N=N, scratch_elems=S * M * N - 1),
    }
    for name, kw in cases.items():
        n = kw['N']
        small = kw.pop('scratch_elems', None)
        scratch = torch.full((S * M * N,), 7.0, device=dev)
        if small is not None:
            scratch = scratch[:small]
        out = torch.full((M, n), 5.0, device=dev, dtype=torch.float16)
        with pytest.raises(RuntimeError, match='op_gemm_splitk'):
            ops.gemm_splitk(splits=S, scratch=scratch, out=out, **kw)
        torch.cuda.synchronize()
        assert (out == 5.0).all(), name
        assert (scratch == 7.0).all(), name


# ------------------------------------------------------------------------------------- upsample / im2col / sinusoid / small linear
@pytest.mark.parametrize('nf,h,w,C', [(3, 5, 7, 64), (2, 8, 8, 320), (1, 1, 3, 8)])
def test_upsample2x(ops, nf, h, w, C):
    x = rand(nf, h, w, C)
    assert torch.equal(ops.upsample2x(x), x.repeat_interleave(2, 1).repeat_interleave(2, 2))


@pytest.mark.parametrize('nf,h,w,C', [(2, 7, 9, 16), (3, 8, 8, 64), (1, 5, 3, 320), (2, 1, 1, 8)])
def test_im2col_s2(ops, nf, h, w, C):
    """Stride-2 3x3 gather with padding 1 = F.unfold(k=3, stride=2, padding=1), reordered tap-major (column tap * C + c)."""
    x = rand(nf, h, w, C)
    ho, wo = (h + 1) // 2, (w + 1) // 2
    u = F.unfold(x.permute(0, 3, 1, 2).float(), 3, padding=1, stride=2)                  # [nf, C * 9, ho * wo]
    ref = u.view(nf, C, 9, ho * wo).permute(0, 3, 2, 1).reshape(nf, ho, wo, 9 * C).half()
    assert torch.equal(ops.im2col_s2(x), ref)


@pytest.mark.parametrize('dim', [320, 321, 7])
def test_time_sinusoid(ops, dim):
    """[cos(t f_k) | sin(t f_k)], f_k = 10000^(-k / half), half = dim // 2, vs fp64; odd dim leaves the last column 0.
    Gate: 1 fp16 ulp of the fp64 value plus the fp32 rounding of the argument t f_k, which the fp32 reference
    (torch.pow, outer product) makes too: the exponent k / half, powf and the product move t f_k by up to ~14 * 2^-24
    relative, allowed as |t f_k| * 2^-19."""
    t = torch.tensor([0.0, 1.0, 17.0, 250.0, 500.0, 981.0, 999.0], device=dev)
    out = ops.time_sinusoid(t, dim)
    half = dim // 2
    k = torch.arange(half, device=dev, dtype=torch.float64)
    arg = t.double()[:, None] * torch.pow(10000.0, -k / half)[None]
    ref = torch.cat([torch.cos(arg), torch.sin(arg)], 1)
    err = (out[:, :2 * half].double() - ref).abs()
    tol = ulp16(ref) + arg.abs().repeat(1, 2) * 2.0 ** -19
    strict = (err / ulp16(ref)).max().item()
    print(f'time_sinusoid dim {dim}: max err / ulp16(ref) {strict:.3f}')
    assert (err <= tol).all(), (err / tol).max().item()
    if dim % 2:
        assert (out[:, -1] == 0).all()


@pytest.mark.parametrize('B,N,K', [(3, 100, 320), (2, 1280, 1280), (1, 37, 512)])
@pytest.mark.parametrize('silu,addend', [(False, False), (True, False), (True, True), (False, True)])
def test_small_linear(ops, B, N, K, silu, addend):
    """y = fp16(fp16(act(x) @ w^T + bias) + addend) with act = fp16(SiLU(x)) when silu, fp32 accumulation (K > 256: each
    lane walks K more than once; N not a multiple of 8).  Reference in fp64 with the same fp16 rounding points; allowed:
    one fp16 ulp at each of the two roundings, one of the SiLU's per term, plus the fp32 sum's (K / 32 + 6) * 2^-24 *
    sum |terms| (a lane adds K / 32 products, then a 5-level shuffle tree and the bias)."""
    torch.manual_seed(B * N + K)
    x = rand(B, K, scale=2)
    w = rand(N, K, scale=K ** -0.5)
    b = rand(N)
    ad = rand(N) if addend else None
    act = F.silu(x.double()).half().double() if silu else x.double()
    lin64 = act @ w.double().t() + b.double()
    lin = lin64.half().double()
    ref = lin + ad.double() if addend else lin
    y = ops.small_linear(x, w, b, ad, silu_in=silu)
    terms = act.abs() @ w.double().abs().t() + b.double().abs()
    tol = ulp16(lin64) + (ulp16(ref) if addend else 0) + (K / 32 + 6) * U32 * terms
    if silu:
        tol = tol + ulp16(act.abs().max()) * w.double().abs().sum(1)
    err = (y.double() - ref).abs()
    assert (err <= tol).all(), (err / tol).max().item()
