"""GPU: every kernel-level entry point against a plain torch fp32 reference of the same op on the same fp16-rounded
inputs (fp64 for the convolutions: cuDNN runs fp32 convolutions in TF32 by default, whose error is near the gate).
Tolerance: max |err| <= 2e-3 * max|ref|  (fp16 output rounding is 4.9e-4 relative; accumulation is fp32)."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
dev = 'cuda'


def rel(a, b):
    return ((a.float() - b.float()).abs().max() / (b.float().abs().max() + 1e-6)).item()


@pytest.fixture(scope='module')
def ops():
    from t2v_b200 import ops as o
    torch.manual_seed(0)
    return o


@pytest.mark.parametrize('cg', [1, 2])
@pytest.mark.parametrize('M,K,N,bn,bias,res', [
    (128, 64, 64, 64, True, False), (256, 128, 128, 128, False, False), (1000, 320, 320, 0, True, False),
    (1000, 320, 320, 160, True, True), (4096, 512, 256, 256, True, False), (24576, 320, 2560, 0, True, False),
    (384, 1280, 1280, 0, True, True), (77, 1024, 640, 0, False, False), (512, 320, 4, 16, True, False),
    (1, 64, 64, 0, True, False), (129, 72, 200, 0, True, True)])
def test_linear(ops, M, K, N, bn, bias, res, cg):
    if cg == 2 and (bn == 16 or N <= 16):
        pytest.skip('two-CTA clusters need BN >= 64')
    a = torch.randn(M, K, device=dev).half()
    w = (torch.randn(N, K, device=dev) / K ** 0.5).half()
    b = torch.randn(N, device=dev).half() if bias else None
    r = torch.randn(M, N, device=dev).half() if res else None
    n_alloc = max(N, 16)
    wp = torch.zeros(1, n_alloc, K, device=dev, dtype=torch.half)
    wp[0, :N] = w
    out = ops.gemm(a, wp, N, n_alloc=n_alloc, bias=b, residual=r, force_bn=bn, force_cg=cg)
    ref = a.float() @ w.float().t()
    if bias:
        ref = ref + b.float()
    if res:
        ref = ref + r.float()
    assert rel(out, ref) < 2e-3


@pytest.mark.parametrize('NF,h,w,Cin,Cout', [(2, 16, 16, 64, 64), (3, 32, 32, 320, 320), (4, 8, 8, 128, 256),
                                             (4, 4, 4, 256, 128), (5, 2, 2, 64, 64), (2, 16, 8, 64, 128),
                                             (2, 18, 32, 64, 64), (2, 9, 16, 64, 64), (3, 16, 16, 8, 64),
                                             (3, 16, 16, 320, 4), (1, 1, 1, 64, 64), (2, 6, 200, 64, 64)])
@pytest.mark.parametrize('cg', [1, 2])
def test_conv3x3_implicit_gemm(ops, NF, h, w, Cin, Cout, cg):
    if cg == 2 and Cout < 64:
        pytest.skip('two-CTA clusters need BN >= 64')
    x = torch.randn(NF, h, w, Cin, device=dev).half()
    wt = (torch.randn(Cout, Cin, 3, 3, device=dev) / (9 * Cin) ** 0.5).half()
    b = torch.randn(Cout, device=dev).half()
    n_alloc = max(Cout, 16)
    wp = ops.pack_conv_weight(wt, n_alloc=n_alloc)
    out = ops.gemm(x.view(-1, Cin), wp, Cout, dims=[w, h, NF], taps=ops.conv_taps_2d(), n_alloc=n_alloc, bias=b, force_cg=cg)
    ref = F.conv2d(x.permute(0, 3, 1, 2).double(), wt.double(), b.double(), padding=1).permute(0, 2, 3, 1).reshape(-1, Cout)
    assert rel(out, ref) < 2e-3


@pytest.mark.parametrize('B,Fr,P,C', [(1, 24, 256, 320), (2, 4, 16, 128), (2, 5, 4, 64), (1, 3, 128, 64), (2, 1, 64, 64)])
@pytest.mark.parametrize('cg', [1, 2])
def test_temporal_conv(ops, B, Fr, P, C, cg):
    x = torch.randn(B, Fr, P, C, device=dev).half()
    wt = (torch.randn(C, C, 3, 1, 1, device=dev) / (3 * C) ** 0.5).half()
    b = torch.randn(C, device=dev).half()
    out = ops.gemm(x.view(-1, C), ops.pack_conv_weight(wt), C, dims=[P, Fr, B], taps=ops.conv_taps_temporal(), bias=b,
                   residual=x.view(-1, C), force_cg=cg)
    x5 = x.permute(0, 3, 1, 2).reshape(B, C, Fr, P, 1).double()
    ref = (F.conv3d(x5, wt.double(), b.double(), padding=(1, 0, 0)) + x5).reshape(B, C, Fr, P).permute(0, 2, 3, 1).reshape(-1, C)
    assert rel(out, ref) < 2e-3


@pytest.mark.parametrize('M,K,H,bn', [(1024, 320, 1280, 256), (512, 64, 256, 128), (300, 64, 256, 64)])
@pytest.mark.parametrize('cg', [1, 2])
def test_geglu_epilogue(ops, M, K, H, bn, cg):
    a = torch.randn(M, K, device=dev).half()
    w = (torch.randn(2 * H, K, device=dev) / K ** 0.5).half()
    b = torch.randn(2 * H, device=dev).half()
    wp, bp = ops.pack_geglu_weight(w, b, bn)
    out = ops.gemm(a, wp, 2 * H, bias=bp, flags=ops.GEMM_GEGLU, force_bn=bn, force_cg=cg)
    hh = (a.float() @ w.float().t() + b.float()).half()
    xa, gate = hh.chunk(2, dim=-1)
    ref = xa * F.gelu(gate)
    assert rel(out, ref) < 4e-3


@pytest.mark.parametrize('M,K,N,bias,res', [(24576, 320, 320, True, True), (24576, 320, 960, False, False), (20000, 320, 512, True, False),
                                            (70000, 64, 64, True, True), (30000, 640, 640, True, True), (19000, 320, 1920, True, False),
                                            (148 * 3 * 128 // 2 + 5, 320, 320, True, True)])
def test_linear_b_stationary_variant(ops, M, K, N, bias, res):
    """The B-stationary GEMM variant (weight slice of the N-tile resident in shared memory, A-only ring) against torch and
    against the streaming variant: the K order inside the tensor core is the same, so the two must agree bit for bit."""
    a = torch.randn(M, K, device=dev).half()
    w = (torch.randn(N, K, device=dev) / K ** 0.5).half()
    b = torch.randn(N, device=dev).half() if bias else None
    r = torch.randn(M, N, device=dev).half() if res else None
    wp = w.view(1, N, K).contiguous()
    out = ops.gemm(a, wp, N, bias=b, residual=r, flags=ops.GEMM_FORCE_BS)
    plain = ops.gemm(a, wp, N, bias=b, residual=r, flags=ops.GEMM_NO_BS)
    ref = a.float() @ w.float().t()
    if bias:
        ref = ref + b.float()
    if res:
        ref = ref + r.float()
    assert rel(out, ref) < 2e-3
    assert torch.equal(out, plain)


@pytest.mark.parametrize('M,K,H', [(24576, 320, 1280), (9000, 320, 1280), (40000, 64, 256)])
def test_geglu_b_stationary_variant(ops, M, K, H):
    a = torch.randn(M, K, device=dev).half()
    w = (torch.randn(2 * H, K, device=dev) / K ** 0.5).half()
    b = torch.randn(2 * H, device=dev).half()
    wp, bp = ops.pack_geglu_weight(w, b, 128)
    out = ops.gemm(a, wp, 2 * H, bias=bp, flags=ops.GEMM_GEGLU | ops.GEMM_FORCE_BS, force_bn=128)
    plain = ops.gemm(a, wp, 2 * H, bias=bp, flags=ops.GEMM_GEGLU | ops.GEMM_NO_BS, force_bn=128)
    hh = (a.float() @ w.float().t() + b.float()).half()
    xa, gate = hh.chunk(2, dim=-1)
    assert rel(out, xa * F.gelu(gate)) < 4e-3
    assert torch.equal(out, plain)


def test_temporal_conv_b_stationary_variant(ops):
    """3-tap temporal conv (tap = frame offset, zero padding by TMA out-of-bounds fill) through the resident-weight variant."""
    B, Fr, P, C = 2, 24, 1024, 64
    x = torch.randn(B, Fr, P, C, device=dev).half()
    wt = (torch.randn(C, C, 3, 1, 1, device=dev) / (3 * C) ** 0.5).half()
    wp = ops.pack_conv_weight(wt)
    taps = ops.conv_taps_temporal()
    out = ops.gemm(x.view(-1, C), wp, C, dims=[P, Fr, B], taps=taps, flags=ops.GEMM_FORCE_BS)
    plain = ops.gemm(x.view(-1, C), wp, C, dims=[P, Fr, B], taps=taps, flags=ops.GEMM_NO_BS)
    xr = x.double().permute(0, 3, 1, 2).reshape(B, C, Fr, P, 1)
    ref = F.conv3d(xr, wt.double(), padding=(1, 0, 0)).reshape(B, C, Fr, P).permute(0, 2, 3, 1).reshape(-1, C)
    assert rel(out, ref) < 2e-3
    assert torch.equal(out, plain)


def test_batched_gemm_and_per_sample_bias(ops):
    q = torch.randn(3, 256, 512, device=dev).half()
    k = torch.randn(3, 256, 512, device=dev).half()
    out = ops.gemm(q.view(-1, 512), k, 256, dims=[256, 3], taps=[[0, 0]], n_alloc=256, b_batch_dim=1, alpha=512 ** -0.5)
    assert rel(out, torch.bmm(q.float(), k.float().transpose(1, 2)).reshape(-1, 256) * 512 ** -0.5) < 2e-3
    a = torch.randn(2 * 640, 320, device=dev).half()
    w = (torch.randn(320, 320, device=dev) / 320 ** 0.5).half()
    b = torch.randn(2, 320, device=dev).half()
    out = ops.gemm(a, w.view(1, 320, 320), 320, bias=b, bias_rows=640, bias_stride=320)
    ref = (a.float() @ w.float().t()).view(2, 640, 320) + b.float()[:, None, :]
    assert rel(out, ref.view(-1, 320)) < 2e-3


@pytest.mark.parametrize('n_inst,rows,C,silu,eps', [(3, 128, 64, True, 1e-5), (24, 1024, 320, True, 1e-5),
                                                   (2, 24 * 64, 640, False, 1e-6), (1, 4 * 256, 960, True, 1e-5),
                                                   (5, 4, 2560, True, 1e-5), (2, 1, 256, True, 1e-5)])
def test_groupnorm_back_to_back_shapes(ops, n_inst, rows, C, silu, eps):
    """Different (instances, rows) shapes share one workspace: run two shapes back to back (regression: the completion
    counters must stay at a fixed, zeroed location)."""
    for (ni, rr) in ((n_inst, rows), (max(1, n_inst // 2), rows * 2 if n_inst > 1 else rows)):
        x = (torch.randn(ni * rr, C, device=dev) * 2 + 0.5).half()
        g = (1 + 0.1 * torch.randn(C, device=dev)).half()
        b = (0.1 * torch.randn(C, device=dev)).half()
        y = ops.groupnorm(x, g, b, rr, eps, silu)
        xr = x.float().view(ni, rr, C).permute(0, 2, 1)           # [inst, C, rows]
        ref = F.group_norm(xr, 32, g.float(), b.float(), eps)
        if silu:
            ref = F.silu(ref)
        ref = ref.permute(0, 2, 1).reshape(-1, C)
        assert rel(y, ref) < 2e-3


@pytest.mark.parametrize('n_inst,rows,C', [(48, 256, 640), (2, 6144, 640), (48, 1024, 320), (2, 24576, 320), (48, 16, 1280),
                                          (300, 16, 128), (24, 4096, 128), (7, 333, 1920), (2, 100, 2560)])
def test_groupnorm_single_launch_paths(ops, n_inst, rows, C):
    """The single-launch kernel (statistics -> per-instance barrier -> apply) in its regimes: slice cached in shared memory
    (one CTA per SM), second pass from L2 (two CTAs per SM), one CTA per instance, and the two-kernel fallback when the
    instances outnumber the co-resident CTAs; replayed back to back (the barrier's generation counter is reused)."""
    x = (torch.randn(n_inst * rows, C, device=dev) * 1.5 - 0.25).half()
    g = (1 + 0.1 * torch.randn(C, device=dev)).half()
    b = (0.1 * torch.randn(C, device=dev)).half()
    ref = F.silu(F.group_norm(x.float().view(n_inst, rows, C).permute(0, 2, 1), 32, g.float(), b.float(), 1e-5))
    ref = ref.permute(0, 2, 1).reshape(-1, C)
    first = ops.groupnorm(x, g, b, rows, 1e-5, True)
    assert rel(first, ref) < 2e-3
    for _ in range(20):
        assert torch.equal(ops.groupnorm(x, g, b, rows, 1e-5, True), first)       # deterministic fold order, barrier reusable


@pytest.mark.parametrize('rows,C', [(1000, 64), (24576, 320), (77, 1280), (5, 512)])
def test_layernorm(ops, rows, C):
    x = (torch.randn(rows, C, device=dev) * 3 + 1).half()
    g = (1 + 0.1 * torch.randn(C, device=dev)).half()
    b = (0.1 * torch.randn(C, device=dev)).half()
    y = ops.layernorm(x, g, b)
    assert rel(y, F.layer_norm(x.float(), (C,), g.float(), b.float(), 1e-5)) < 2e-3


@pytest.mark.parametrize('batch,heads,sq,skv', [(3, 5, 128, 128), (2, 10, 1024, 1024), (4, 2, 24, 24), (3, 4, 256, 77),
                                               (2, 1, 100, 77), (2, 2, 16, 16), (1, 1, 130, 130)])
def test_attention_dense_layout(ops, batch, heads, sq, skv):
    C = heads * 64
    q = torch.randn(batch, sq, C, device=dev).half()
    k = torch.randn(batch, skv, C, device=dev).half()
    v = torch.randn(batch, skv, C, device=dev).half()
    o = torch.empty_like(q)
    ops.attention(q, k, v, o, sq * C, C, skv * C, C, skv * C, C, sq * C, C, batch, heads, sq, skv)

    def sp(t):
        return t.float().view(t.shape[0], t.shape[1], heads, 64).permute(0, 2, 1, 3)
    ref = F.scaled_dot_product_attention(sp(q), sp(k), sp(v)).permute(0, 2, 1, 3).reshape(batch, sq, C)
    assert rel(o, ref) < 3e-3


@pytest.mark.parametrize('batch,heads,S', [(2, 5, 1024), (3, 2, 320), (1, 2, 9216), (2, 3, 256), (1, 1, 1000)])
def test_attention_tcgen05_fused_qkv(ops, batch, heads, S):
    """Long spatial sequences take the wgmma kernel (csrc/attention_tc.cu): Q, K, V are column slices of the fused
    [tokens, 3C] matrix, the head is a tensor-map column offset, ragged tails (S % 128 != 0) are TMA zero fill + masking."""
    C = heads * 64
    qkv = torch.randn(batch * S, 3 * C, device=dev).half()
    o = torch.zeros(batch * S, C, device=dev, dtype=torch.half)
    ld = 3 * C
    ops.attention(qkv, qkv[:, C:], qkv[:, 2 * C:], o, S * ld, ld, S * ld, ld, S * ld, ld, S * C, C, batch, heads, S, S)
    t = qkv.float().view(batch, S, 3, heads, 64).permute(2, 0, 3, 1, 4)      # [3, batch, heads, S, 64]
    ref = F.scaled_dot_product_attention(t[0], t[1], t[2]).permute(0, 2, 1, 3).reshape(batch * S, C)
    assert rel(o, ref) < 3e-3
    assert (o.float() - ref).abs().max() < 2e-2


def test_attention_tcgen05_shared_kv_and_peaked_scores(ops):
    """kv_batch_div (frames sharing K/V), skv != sq with a ragged last key tile, and scores large enough that the running
    max actually moves between key tiles (exercises the exp2 rescale of the running output).  Kept under its original name:
    the kernel is the wgmma one in csrc/attention_tc.cu."""
    batch, heads, sq, skv, div = 4, 2, 384, 200, 2
    C = heads * 64
    q = (torch.randn(batch, sq, C, device=dev) * 3).half()
    k = (torch.randn(batch // div, skv, C, device=dev) * 3).half()
    k[:, 150:] *= 2          # later keys dominate: max rises in the second tile
    v = torch.randn(batch // div, skv, C, device=dev).half()
    o = torch.zeros_like(q)
    ops.attention(q, k, v, o, sq * C, C, skv * C, C, skv * C, C, sq * C, C, batch, heads, sq, skv, kv_batch_div=div)

    def sp(t):
        return t.float().view(t.shape[0], t.shape[1], heads, 64).permute(0, 2, 1, 3)
    kk = k.repeat_interleave(div, 0)
    vv = v.repeat_interleave(div, 0)
    ref = F.scaled_dot_product_attention(sp(q), sp(kk), sp(vv)).permute(0, 2, 1, 3).reshape(batch, sq, C)
    assert rel(o, ref) < 3e-3


@pytest.mark.parametrize('hd', [8, 16, 32, 40, 80, 160])
@pytest.mark.parametrize('S,skv', [(256, 256), (100, 77), (1024, 1024)])
def test_attention_other_head_dims(ops, hd, S, skv):
    """VideoCrafter heads (C/8 = 40 / 80 / 160, and the tiny-config widths): spatial self- and CLIP cross-attention."""
    batch, heads = 3, 8
    if S == 1024 and hd not in (40, 160):
        pytest.skip('large case only for the production widths')
    C = heads * hd
    q = torch.randn(batch, S, C, device=dev).half()
    k = torch.randn(batch, skv, C, device=dev).half()
    v = torch.randn(batch, skv, C, device=dev).half()
    o = torch.zeros_like(q)
    ops.attention_hd(q, k, v, o, S * C, C, skv * C, C, skv * C, C, S * C, C, batch, heads, hd, S, skv)

    def sp(t):
        return t.float().view(t.shape[0], t.shape[1], heads, hd).permute(0, 2, 1, 3)
    ref = F.scaled_dot_product_attention(sp(q), sp(k), sp(v)).permute(0, 2, 1, 3).reshape(batch, S, C)
    assert rel(o, ref) < 3e-3


@pytest.mark.parametrize('hd,T,L', [(40, 16, 16), (80, 16, 16), (160, 16, 16), (8, 4, 4), (32, 4, 4), (16, 7, 9), (40, 12, 16),
                                     (40, 24, 16), (80, 32, 16), (160, 24, 16), (16, 7, 3), (8, 20, 4), (64, 17, 16)])
def test_attention_relative_position_temporal(ops, hd, T, L):
    """TemporalCrossAttention with RelativePosition tables (videocrafter attention_temporal.py:107-144) on the token
    matrix [(b, f, p), 3C]: sequences run along frames for every pixel, no rearrange copies."""
    B, P, heads = 2, 24, 8
    C = heads * hd
    qkv = torch.randn(B * T * P, 3 * C, device=dev).half()
    tk = (torch.randn(2 * L + 1, hd, device=dev) * 0.5).half()
    tv = (torch.randn(2 * L + 1, hd, device=dev) * 0.5).half()
    o = torch.zeros(B * T * P, C, device=dev, dtype=torch.half)
    ld = 3 * C
    ops.attention_relpos(qkv, qkv[:, C:], qkv[:, 2 * C:], o, tk, tv, B * P, P, T * P * ld, ld, P * ld, T * P * C, C, P * C,
                         heads, hd, T, L)
    t = qkv.float().view(B, T, P, 3, heads, hd).permute(3, 0, 2, 4, 1, 5)       # [3, B, P, heads, T, hd]
    q, k, v = t[0], t[1], t[2]
    idx = (torch.arange(T, device=dev)[None, :] - torch.arange(T, device=dev)[:, None]).clamp(-L, L) + L
    k2, v2 = tk.float()[idx], tv.float()[idx]                                       # [T, T, hd]
    scale = hd ** -0.5
    sim = (torch.einsum('bphtd,bphsd->bphts', q, k) + torch.einsum('bphtd,tsd->bphts', q, k2)) * scale
    attn = sim.softmax(-1)
    out = torch.einsum('bphts,bphsd->bphtd', attn, v) + torch.einsum('bphts,tsd->bphtd', attn, v2)
    ref = out.permute(0, 3, 1, 2, 4).reshape(B * T * P, C)                          # [(b, t, p), (h d)]
    assert rel(o, ref) < 3e-3


def test_attention_temporal_strides_on_token_matrix(ops):
    """Sequences along frames for every pixel of a [(f, p), 3C] fused qkv matrix -- no rearrange copies."""
    Fr, P, heads = 24, 64, 5
    C = heads * 64
    qkv = torch.randn(Fr * P, 3 * C, device=dev).half()
    o = torch.empty(Fr * P, C, device=dev, dtype=torch.half)
    ld = 3 * C
    ops.attention(qkv, qkv[:, C:], qkv[:, 2 * C:], o, ld, P * ld, ld, P * ld, ld, P * ld, C, P * C, P, heads, Fr, Fr)
    t = qkv.float().view(Fr, P, 3, heads, 64).permute(2, 1, 3, 0, 4)     # [3, P, heads, F, 64]
    ref = F.scaled_dot_product_attention(t[0], t[1], t[2]).permute(2, 0, 1, 3).reshape(Fr * P, C)
    assert rel(o, ref) < 3e-3
