"""GPU: the TMA-store epilogue (fp16 tiles written to a shared output tile and stored by TMA, residual loaded by TMA into
the same tile) computes exactly what the per-warp slab epilogue computes.  ops.GEMM_SLAB_OUT forces the slab path on
problems that would take the TMA path; the two outputs must match bit for bit, for each epilogue kind, at several tile
widths (including the 16-column tiles and the 5- and 7-chunk widths 160 / 224), with row boxes whose tiles cut the problem
edge, ragged N, and an in-place residual (out is residual).  At BN 224 / 256 a launch of one wave (tiles <= SMs) takes the
variant without the output tile, so the 20000-row case is the one that exercises TMA stores at those widths."""
import pytest
import torch

pytestmark = pytest.mark.gpu
dev = 'cuda'


@pytest.fixture(scope='module')
def ops():
    from t2v_b200 import ops as o
    return o


def rand(*shape, scale=1.0):
    return (torch.randn(*shape, device=dev) * scale).half()


def check_paths(ops, run, widths):
    for bn in widths:
        tma, slab = run(bn, 0), run(bn, ops.GEMM_SLAB_OUT)
        assert torch.equal(tma, slab), f'BN {bn}: max |diff| {(tma.float() - slab.float()).abs().max().item()}'


@pytest.mark.parametrize('M,K,N,res', [(1000, 320, 320, False), (1000, 320, 960, True), (129, 72, 200, True),
                                       (300, 128, 16, True), (517, 64, 1000, False),
                                       (20000, 64, 512, True)])
def test_linear_tma_vs_slab(ops, M, K, N, res):
    torch.manual_seed(10)
    a, w, b = rand(M, K), rand(1, N, K, scale=K ** -0.5), rand(N)
    r = rand(M, N) if res else None
    widths = [16] if N <= 16 else [64, 128, 160, 192, 224, 256]
    check_paths(ops, lambda bn, fl: ops.gemm(a, w, N, bias=b, residual=r, flags=fl, force_bn=bn), widths)


def test_in_place_residual_tma_vs_slab(ops):
    torch.manual_seed(11)
    M, K, N = 700, 320, 320
    a, w, b, x = rand(M, K), rand(1, N, K, scale=K ** -0.5), rand(N), rand(M, N)

    def run(bn, fl):
        y = x.clone()
        ops.gemm(a, w, N, bias=b, residual=y, out=y, flags=fl, force_bn=bn)
        return y
    check_paths(ops, run, [64, 160, 256])


def test_per_sample_bias_tma_vs_slab(ops):
    torch.manual_seed(12)
    a, w, b = rand(3 * 700, 320), rand(1, 320, 320, scale=320 ** -0.5), rand(3, 320)
    check_paths(ops, lambda bn, fl: ops.gemm(a, w, 320, bias=b, bias_rows=700, bias_stride=320, flags=fl, force_bn=bn),
                [64, 160])


@pytest.mark.parametrize('M,K,H', [(300, 64, 256), (1024, 320, 640)])
def test_geglu_tma_vs_slab(ops, M, K, H):
    torch.manual_seed(13)
    a, w, b = rand(M, K), rand(2 * H, K, scale=K ** -0.5), rand(2 * H)

    def run(bn, fl):
        wp, bp = ops.pack_geglu_weight(w, b, bn)
        return ops.gemm(a, wp, 2 * H, bias=bp, flags=ops.GEMM_GEGLU | fl, force_bn=bn)
    check_paths(ops, run, [64, 128, 256])


@pytest.mark.parametrize('NF,h,w,Cin,Cout', [(2, 6, 200, 64, 96), (3, 9, 16, 64, 320), (2, 5, 5, 128, 64)])
def test_conv3x3_row_boxes_tma_vs_slab(ops, NF, h, w, Cin, Cout):
    """nd = 3 row boxes; w = 200 and h = 9 leave boxes that reach past the grid, clipped by the output tensor map."""
    torch.manual_seed(14)
    x = rand(NF, h, w, Cin)
    wp = ops.pack_conv_weight(rand(Cout, Cin, 3, 3, scale=(9 * Cin) ** -0.5))
    b, r = rand(Cout), rand(NF * h * w, Cout)
    check_paths(ops, lambda bn, fl: ops.gemm(x.view(-1, Cin), wp, Cout, dims=[w, h, NF], taps=ops.conv_taps_2d(), bias=b,
                                             residual=r, flags=fl, force_bn=bn), [64, 128, 160, 256])


def test_two_cta_tma_vs_slab(ops):
    """CG = 2 with an odd number of M-tiles (3): the cluster's tail CTA has no tile to store."""
    torch.manual_seed(15)
    M, K, N = 2 * 128 + 5, 320, 640
    a, w, b, r = rand(M, K), rand(1, N, K, scale=K ** -0.5), rand(N), rand(M, N)
    for bn in (64, 128, 160, 256):
        tma = ops.gemm(a, w, N, bias=b, residual=r, force_bn=bn, force_cg=2)
        slab = ops.gemm(a, w, N, bias=b, residual=r, flags=ops.GEMM_SLAB_OUT, force_bn=bn, force_cg=2)
        assert torch.equal(tma, slab), f'BN {bn} CG 2'
