"""GPU: the GEMM output does not depend on the tile width.  Every width keeps each element's K order and its epilogue
arithmetic, so the output at each forced width (and with two-CTA clusters) must equal the BN = 64 output bit for bit.  The
cases cover each epilogue kind ops.gemm reaches: plain, residual, fp32 output, per-sample bias, GEGLU, batched B with
alpha, multi-dimensional row boxes with ragged (out-of-range) rows, ragged N, and unaligned rows (odd ldo / ldr), which
store element by element.  The LayerNorm fold and split-K, which ops.gemm does not reach, have their own op-level tests
(fp64 references, tile-width independence) in test_gemm_ln_splitk_gpu.py."""
import pytest
import torch

pytestmark = pytest.mark.gpu
dev = 'cuda'
WIDTHS = [16, 64, 128, 160, 192, 224, 256]
CG2_WIDTHS = [64, 128, 160, 256]


@pytest.fixture(scope='module')
def ops():
    from t2v_b200 import ops as o
    return o


def widths(cg2=True):
    return [(bn, 1) for bn in WIDTHS if bn != 64] + ([(bn, 2) for bn in CG2_WIDTHS] if cg2 else [])


def check_widths(run, cases):
    ref = run(64, 1)
    for bn, cg in cases:
        out = run(bn, cg)
        assert torch.equal(out, ref), f'BN {bn} CG {cg}: max |diff| {(out.float() - ref.float()).abs().max().item()}'


def rand(*shape, scale=1.0):
    return (torch.randn(*shape, device=dev) * scale).half()


@pytest.mark.parametrize('M,K,N,bias,res', [(1000, 320, 320, True, False), (129, 72, 200, True, True), (1, 64, 64, True, True),
                                            (4096, 640, 640, False, True), (300, 320, 1920, True, True)])
def test_linear_widths(ops, M, K, N, bias, res):
    torch.manual_seed(0)
    a, w = rand(M, K), rand(1, N, K, scale=K ** -0.5)
    b = rand(N) if bias else None
    r = rand(M, N) if res else None
    check_widths(lambda bn, cg: ops.gemm(a, w, N, bias=b, residual=r, force_bn=bn, force_cg=cg), widths())


@pytest.mark.parametrize('M,N', [(1000, 320), (77, 200)])
def test_fp32_output_widths(ops, M, N):
    torch.manual_seed(1)
    a, w, b = rand(M, 320), rand(1, N, 320, scale=320 ** -0.5), rand(N)
    check_widths(lambda bn, cg: ops.gemm(a, w, N, bias=b, flags=ops.GEMM_OUT_F32, force_bn=bn, force_cg=cg), widths())


def test_per_sample_bias_widths(ops):
    torch.manual_seed(2)
    a, w, b = rand(3 * 700, 320), rand(1, 320, 320, scale=320 ** -0.5), rand(3, 320)
    check_widths(lambda bn, cg: ops.gemm(a, w, 320, bias=b, bias_rows=700, bias_stride=320, force_bn=bn, force_cg=cg),
                 widths())


@pytest.mark.parametrize('M,K,H', [(300, 64, 256), (1024, 320, 640)])
def test_geglu_widths(ops, M, K, H):
    torch.manual_seed(3)
    a, w, b = rand(M, K), rand(2 * H, K, scale=K ** -0.5), rand(2 * H)

    def run(bn, cg):
        wp, bp = ops.pack_geglu_weight(w, b, bn)
        return ops.gemm(a, wp, 2 * H, bias=bp, flags=ops.GEMM_GEGLU, force_bn=bn, force_cg=cg)
    check_widths(run, [(128, 1), (256, 1), (64, 2), (128, 2), (256, 2)])


def test_batched_alpha_widths(ops):
    torch.manual_seed(4)
    q, k = rand(3, 300, 64), rand(3, 256, 64)
    check_widths(lambda bn, cg: ops.gemm(q.view(-1, 64), k, 256, dims=[300, 3], taps=[[0, 0]], n_alloc=256, b_batch_dim=1,
                                         alpha=0.125, force_bn=bn, force_cg=cg), widths(cg2=False))


@pytest.mark.parametrize('NF,h,w,Cin,Cout', [(2, 6, 200, 64, 96), (3, 9, 16, 64, 320), (2, 5, 5, 128, 64)])
def test_conv3x3_row_boxes_widths(ops, NF, h, w, Cin, Cout):
    """nd = 3 row boxes; w = 200 and h = 9 leave boxes that reach past the grid (rows with no output)."""
    torch.manual_seed(5)
    x = rand(NF, h, w, Cin)
    wp = ops.pack_conv_weight(rand(Cout, Cin, 3, 3, scale=(9 * Cin) ** -0.5))
    b, r = rand(Cout), rand(NF * h * w, Cout)
    check_widths(lambda bn, cg: ops.gemm(x.view(-1, Cin), wp, Cout, dims=[w, h, NF], taps=ops.conv_taps_2d(), bias=b,
                                         residual=r, force_bn=bn, force_cg=cg), widths())


@pytest.mark.parametrize('out_f32', [False, True])
def test_unaligned_rows_widths(ops, out_f32):
    """Odd output and residual pitches: nothing is 16-byte aligned, every element is stored on its own."""
    torch.manual_seed(6)
    M, K, N = 333, 128, 200
    a, w, b = rand(M, K), rand(1, N, K, scale=K ** -0.5), rand(N)
    r = None if out_f32 else rand(M, N + 3)[:, 1:N + 1]
    dt = torch.float32 if out_f32 else torch.float16

    def run(bn, cg):
        buf = torch.zeros(M, N + 1, device=dev, dtype=dt)
        ops.gemm(a, w, N, bias=b, residual=r, ldr=N + 3 if r is not None else None, out=buf[:, 1:], ldo=N + 1,
                 flags=ops.GEMM_OUT_F32 if out_f32 else 0, force_bn=bn, force_cg=cg)
        return buf
    check_widths(run, widths())
