"""The LoRA merge kernels (csrc/elementwise.cu lora_merge_kernel, lora_apply_kernel) at op level, and the in-place re-pack
every library handle runs after a hot merge, restore or clear.

Op level, through t2v_op_lora_merge / t2v_op_lora_apply (ops.lora_merge_ / ops.lora_apply_):
  exact operands  factors on a dyadic grid where every partial sum of the product is representable (fp16 for the Stable-LoRA
                  merge, fp32 for VideoCrafter's), so no summation order, TF32 or reduced-precision reduction can change the
                  product and only the rounding points remain: they must match the reference's torch ops bit for bit
                  (stable_lora/stable_utils/lora_processor.py:50-96 under autocast; videocrafter lora.py:650-666);
  Gaussian        per element against the fp64 product within a derived bound; against torch on the GPU within one fp16
                  step wherever the fp32 accumulation error bound is below a quarter ulp, and within one step plus both
                  accumulation errors elsewhere (mismatch counts and the worst step count are printed).
Handles: handle A hot-merges; handle B is shipped the weight ops.lora_merge_ / ops.lora_apply_ computed on a copy of the
base, i.e. the same kernel on the same inputs and so the same bits.  A's output must equal B's bit for bit: a packed variant
the merge left stale (fused q|k|v and k|v, LayerNorm fold, GEGLU interleave, tap-major, padded and K-major conv packs)
differs.  The CPU test checks that the weights named below exist with the layouts they are chosen for."""
import contextlib
import math
import zlib

import numpy as np
import pytest
import torch

from oracle import clip_oracle as CO, unet_oracle as UO, vae_oracle as VO, vc_oracle as VC
import adapter_oracle as AO
import clip_l_oracle as CL
from parity_util import report

S16 = 0x7E5A                # NaN sentinel past the written elements
ALPHA = 0.7                 # handle merges: a non-dyadic scale


@contextlib.contextmanager
def _no_tf32():
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        yield
    finally:
        torch.backends.cuda.matmul.allow_tf32 = old


@contextlib.contextmanager
def _fp32_sums():
    old = torch.backends.cuda.matmul.allow_fp16_reduced_precision_reduction
    torch.backends.cuda.matmul.allow_fp16_reduced_precision_reduction = False
    try:
        yield
    finally:
        torch.backends.cuda.matmul.allow_fp16_reduced_precision_reduction = old


def _ulp16(x):
    """fp16 ulp of |x| (float64 array); 2^-24 below the normal range."""
    return 2.0 ** (np.floor(np.log2(np.maximum(np.abs(x), 2.0 ** -14))) - 10)


def _guarded(w):
    """A copy of w in a buffer with a NaN-sentinel tail past its elements: (buffer, n)."""
    n = w.numel()
    buf = torch.empty(n + 64, dtype=torch.float16, device='cuda')
    buf.view(torch.int16)[n:] = S16
    buf[:n] = w.reshape(-1).cuda()
    return buf, n


def _tail_intact(buf, n):
    return bool((buf.view(torch.int16)[n:] == S16).all())


def _grid(shape, step_exp, kmax, g):
    return torch.randint(-kmax, kmax + 1, shape, generator=g).float() * 2.0 ** step_exp


def _bits(t):
    return t.contiguous().view(torch.int16)


# ------------------------------------------------------------------------------------------------ op level, exact operands
# (weight shape, rank, temporal_mean)
MERGE_SHAPES = [((64, 40), 4, False),               # Linear
                ((24, 37), 3, False),               # cols not a multiple of 8
                ((1, 96), 13, False),               # out = 1
                ((32, 16, 3, 3), 13, False),        # Conv2d 3x3
                ((48, 48, 1), 1, False),            # Conv1d k=1
                ((40, 24, 3, 1, 1), 4, True),       # Conv3d (3,1,1): the product averaged over the second kernel axis
                ((96, 72), 64, False),              # rank 64, on a coarser grid
                ((320, 320, 3, 3), 4, False)]       # 921600 elements > 132 * 16 * 256: the grid-stride loop wraps


def _ref_merge(w, A, B, alpha, temporal):
    """process_lora_weight(weight, lora_B @ lora_A, alpha) as lora_{linear,conv}_forward run it under autocast."""
    with torch.autocast('cuda'):
        lw = B @ A
        if temporal:
            lw = lw.view(w.shape[0], w.shape[1], 3, 3, 1).mean(dim=-2, keepdim=True)
        new = w.clone()
        new += lw.to(w.dtype).view(w.shape) * alpha
    return new


@pytest.mark.gpu
@pytest.mark.parametrize('shape,rank,temporal', MERGE_SHAPES, ids=lambda v: str(v).replace(' ', ''))
def test_merge_exact_operands_bit_for_bit(ops, shape, rank, temporal):
    g = torch.Generator().manual_seed(sum(shape) * 31 + rank)
    out, cols = shape[0], math.prod(shape[1:])
    kmax = 4 if rank > 16 else 8
    A = _grid((rank, cols * 3 if temporal else cols), -6, kmax, g).half().cuda()
    B = _grid((out, rank), -4, kmax, g).half().cuda()
    # every partial sum is a multiple of 2^-10 below 2 in magnitude: an fp16 number, whatever the order of the sum
    assert rank * B.abs().max().item() * A.abs().max().item() < 2
    w = (torch.randn(shape, generator=g) * 0.5).half().cuda()
    for alpha in (1.0, 0.75, -1.3, 0.0):
        buf, n = _guarded(w)
        ops.lora_merge_(buf, A, B, alpha, temporal, out=out, cols=cols)
        ref = _ref_merge(w, A, B, alpha, temporal)
        assert torch.equal(_bits(buf[:n]), _bits(ref.reshape(-1))), (alpha, int((buf[:n] != ref.reshape(-1)).sum()))
        assert _tail_intact(buf, n)
        assert alpha == 0.0 or not torch.equal(ref, w)


APPLY_SHAPES = [((64, 40), 4), ((24, 37), 3), ((1, 96), 13), ((32, 16, 3, 3), 13), ((48, 48, 1, 1), 1), ((96, 72), 64),
                ((320, 320, 3, 3), 4)]


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', ['f16', 'f32'])
@pytest.mark.parametrize('shape,rank', APPLY_SHAPES, ids=lambda v: str(v).replace(' ', ''))
def test_apply_exact_operands_bit_for_bit(ops, shape, rank, dtype):
    g = torch.Generator().manual_seed(sum(shape) * 37 + rank)
    out, cols = shape[0], math.prod(shape[1:])
    if dtype == 'f16':
        kmax = 4 if rank > 16 else 8
        up, down = _grid((out, rank), -4, kmax, g).half(), _grid((rank, cols), -6, kmax, g).half()
    else:
        # up = +-m 2^-16 with m odd in (2048, 4096): 12 significant bits, no fp16 number; every partial sum is a multiple of
        # 2^-22 below 2^2 in magnitude, exact in fp32
        m = 2049 + 2 * torch.randint(0, 1024, (out, rank), generator=g)
        up = (m * (2 * torch.randint(0, 2, (out, rank), generator=g) - 1)).float() * 2.0 ** -16
        down = _grid((rank, cols), -6, 8, g)
        assert not (up.half().float() == up).any()
    assert rank * up.float().abs().max().item() * down.float().abs().max().item() < 2
    up, down = up.cuda(), down.cuda()
    with _no_tf32():
        prod = torch.mm(up.float(), down.float())
    assert torch.equal(prod.cpu(), (up.double().cpu() @ down.double().cpu()).float())        # the product is exact
    w = (torch.randn(shape, generator=g) * 0.5).half().cuda()
    for alpha in (1.0, 0.75, -1.3):                  # -1.3: the reference's `remove`
        buf, n = _guarded(w)
        ops.lora_apply_(buf, up, down, alpha, out=out, cols=cols)
        ref = w.clone()
        ref += alpha * prod.view(w.shape)            # lora.py:656-666 on an fp16 weight
        assert torch.equal(_bits(buf[:n]), _bits(ref.reshape(-1))), (alpha, int((buf[:n] != ref.reshape(-1)).sum()))
        assert _tail_intact(buf, n)


@pytest.mark.gpu
def test_op_entry_points_refuse_bad_arguments(ops):
    from t2v_b200 import _lib
    l = _lib.lib()
    w = torch.randn(8, 16, device='cuda').half()
    before = w.clone()
    A, B = torch.ones(2, 16, device='cuda').half(), torch.ones(8, 2, device='cuda').half()
    s = _lib.stream_ptr()
    p = _lib.ptr
    for out, cols, rank in ((8, 16, 0), (0, 16, 2), (8, 0, 2), (8, 16, -1)):
        assert l.t2v_op_lora_merge(p(w), p(A), p(B), out, cols, rank, 1.0, 0, s) == -1
        assert l.t2v_op_lora_apply(p(w), p(B), p(A), 0, out, cols, rank, 1.0, s) == -1
    assert l.t2v_op_lora_apply(p(w), p(B), p(A), 2, 8, 16, 2, 1.0, s) == -1
    assert b'dtype' in l.t2v_last_error()
    torch.cuda.synchronize()
    assert torch.equal(w, before)


# ------------------------------------------------------------------------------------------------ op level, Gaussian operands
GAUSS_MERGE = [((160, 300), 13, False), ((128, 192), 64, False), ((64, 40, 3, 1, 1), 4, True), ((33, 50), 1, False)]


@pytest.mark.gpu
@pytest.mark.parametrize('shape,rank,temporal', GAUSS_MERGE, ids=lambda v: str(v).replace(' ', ''))
def test_merge_gaussian_against_fp64(ops, shape, rank, temporal):
    g = torch.Generator().manual_seed(sum(shape) + 7 * rank)
    out, cols = shape[0], math.prod(shape[1:])
    acols = cols * 3 if temporal else cols
    A = (torch.randn(rank, acols, generator=g) / math.sqrt(acols)).half()
    B = torch.randn(out, rank, generator=g).half()
    An, Bn = A.double().numpy(), B.double().numpy()
    P, S = Bn @ An, np.abs(Bn) @ np.abs(An)
    e = 1.01 * rank * 2.0 ** -24 * S                 # the fp32 accumulation's error bound
    Ac, Bc = A.cuda(), B.cuda()
    # the product alone: w = 0, alpha = 1
    w0 = torch.zeros(shape, dtype=torch.float16, device='cuda')
    ops.lora_merge_(w0, Ac, Bc, 1.0, temporal)
    d = w0.double().cpu().numpy().reshape(out, cols)
    if temporal:
        # each of the three products rounded to fp16, summed and divided in fp32, rounded to fp16
        Pq, eq = P.reshape(out, cols, 3), e.reshape(out, cols, 3)
        M = Pq.mean(-1)
        bound = 0.5 * _ulp16(M) + (0.5 * _ulp16(Pq) + eq).sum(-1) / 3 + 2.0 ** -23 * (np.abs(Pq) + eq).sum(-1)
    else:
        M, bound = P, 0.5 * _ulp16(P) + e
    ratio = (np.abs(d - M) / bound).max()
    # torch's autocast product, with fp32 sums (cuBLAS may otherwise reduce fp16 products in fp16): both it and the kernel
    # lie within their fp32 accumulation error of P, so they differ by at most one fp16 step plus both errors, and by at
    # most one fp16 step wherever that error is below half an fp16 ulp
    with _fp32_sums(), torch.autocast('cuda'):
        tp = Bc @ Ac
        if temporal:
            tp = tp.view(out, cols // 3, 3, 3, 1).mean(dim=-2, keepdim=True)
    tp = tp.to(torch.float16).double().cpu().numpy().reshape(out, cols)
    ulp = _ulp16(np.maximum(np.abs(tp), np.abs(d)))
    eo = bound - 0.5 * _ulp16(M)                       # the error bound before the final rounding
    ulps = np.abs(tp - d) / ulp
    report(f'lora_merge_gauss_{shape}_r{rank}', worst_err_over_bound=float(ratio), torch_mismatches=int((tp != d).sum()),
           of=d.size, torch_max_ulp=float(ulps.max()), torch_over_1ulp=int((ulps > 1).sum()))
    assert ratio <= 1.0, ratio
    assert (np.abs(tp - d) <= ulp + 2 * eo).all()
    assert (ulps[2 * eo < 0.5 * ulp] <= 1).all()
    if temporal:
        return
    # w != 0 and a non-dyadic alpha: the reference's rounding chain fp16(w + fp16(fp16(P) * alpha)) in fp32 ops on the fp64
    # product; where P +- e straddles fp16 rounding points, any value of the chain over that interval (the chain is monotone
    # in its product, so those lie between its values at the two ends)
    alpha = -0.7
    w = (torch.randn(shape, generator=g) * 0.3).half()
    wk = w.cuda()
    ops.lora_merge_(wk, Ac, Bc, alpha, False)
    got = wk.cpu().numpy()
    w32 = w.numpy().astype(np.float32)

    def chain(d16):
        s = (d16.astype(np.float32) * np.float32(alpha)).astype(np.float16)
        return (w32 + s.astype(np.float32)).astype(np.float16)
    lo, hi = (P - e).astype(np.float16), (P + e).astype(np.float16)
    c_lo, c_hi = chain(lo), chain(hi)
    ok = (got >= np.minimum(c_lo, c_hi)) & (got <= np.maximum(c_lo, c_hi))
    report(f'lora_merge_chain_{shape}_r{rank}', straddling=int((lo != hi).sum()), failing=int((~ok).sum()))
    assert ok.all()
    # the same chain in torch's fp16 ops on the kernel's own product: bit for bit
    ref = w.cuda()
    ref += w0 * alpha
    assert torch.equal(_bits(wk), _bits(ref))
    full = w.cuda()
    full += torch.from_numpy(tp).half().cuda().view(shape) * alpha
    report(f'lora_merge_vs_torch_{shape}_r{rank}', mismatches=int((full != wk).sum()), of=wk.numel())


GAUSS_APPLY = [((160, 300), 13), ((128, 192), 64), ((33, 50), 1), ((64, 32, 3, 3), 4)]


@pytest.mark.gpu
@pytest.mark.parametrize('shape,rank', GAUSS_APPLY, ids=lambda v: str(v).replace(' ', ''))
def test_apply_gaussian_against_fp64(ops, shape, rank):
    g = torch.Generator().manual_seed(sum(shape) + 11 * rank)
    out, cols = shape[0], math.prod(shape[1:])
    up = torch.randn(out, rank, generator=g)                   # fp32 factors
    down = torch.randn(rank, cols, generator=g) / math.sqrt(cols)
    Un, Dn = up.double().numpy(), down.double().numpy()
    P, S = Un @ Dn, np.abs(Un) @ np.abs(Dn)
    e = 1.01 * rank * 2.0 ** -24 * S
    uc, dc = up.cuda(), down.cuda()
    with _no_tf32():
        tprod = torch.mm(uc, dc)
    worst = {}
    for alpha, scale in ((1.0, 0.0), (-0.7, 0.3)):
        w = (torch.randn(shape, generator=g) * scale).half()
        wk = w.cuda()
        ops.lora_apply_(wk, uc, dc, alpha)
        got = wk.double().cpu().numpy().reshape(out, cols)
        wn = w.double().numpy().reshape(out, cols)
        a32 = float(np.float32(alpha))
        v = wn + a32 * P
        # 1/2 ulp of the final rounding, plus the accumulation error and the fp32 roundings of alpha * acc and of the sum
        ap = abs(a32) * (np.abs(P) + e)
        bound = 0.5 * _ulp16(v) + abs(a32) * e + 1.01 * 2.0 ** -24 * (ap + np.abs(wn) + ap)
        ratio = (np.abs(got - v) / bound).max()
        ref = w.cuda()
        ref += alpha * tprod.view(shape)
        r = ref.double().cpu().numpy().reshape(out, cols)
        ulp = _ulp16(np.maximum(np.abs(r), np.abs(got)))
        ulps = np.abs(r - got) / ulp
        # torch and the kernel each lie within |alpha| e plus the fp32 roundings of v: one fp16 step plus both apart
        slack = 2 * (abs(a32) * e + 1.01 * 2.0 ** -24 * (2 * ap + np.abs(wn)))
        report(f'lora_apply_gauss_{shape}_r{rank}_a{alpha}', worst_err_over_bound=float(ratio),
               torch_mismatches=int((r != got).sum()), of=got.size, torch_max_ulp=float(ulps.max()),
               torch_over_1ulp=int((ulps > 1).sum()))
        worst[alpha] = (ratio, bool((np.abs(r - got) <= ulp + slack).all()), bool((ulps[slack < 0.5 * ulp] <= 1).all()))
    for alpha, (ratio, near, one_ulp) in worst.items():
        assert ratio <= 1.0 and near and one_ulp, (alpha, ratio, near, one_ulp)


# ------------------------------------------------------------------------------------------------ handles
def _unet_inputs(s, ctx_dim, L):
    B, Fr, h, w = s
    g = torch.Generator().manual_seed(B * 1000 + Fr * 100 + h + w)
    x = torch.randn(B, 4, Fr, h, w, generator=g)
    y = torch.randn(B, L, ctx_dim, generator=g)
    t = torch.randint(0, 1000, (B,), generator=g)
    return x.cuda(), t.cuda(), y.cuda()


def _run_unet_sd(m, s):
    return m(*_unet_inputs(s, 1024, 77)).clone()


def _run_unet_vc(m, s):
    x, t, y = _unet_inputs(s, 48, 9)
    return m(x, t, context=y).clone()


def _run_tower(m, B):
    tok = torch.randint(0, 300, (B, 77), generator=torch.Generator().manual_seed(B))
    return m.encode_tokens(tok).clone()


def _run_vae(m, F):
    g = torch.Generator().manual_seed(F)
    z = torch.randn(F, 4, 8, 8, generator=g).cuda()
    x = (torch.rand(F, 3, 64, 64, generator=g) * 2 - 1).cuda()
    return torch.cat([m.decode(z).flatten(), m.encode(x).mean.flatten()])


def _run_adapter(m, s):
    N, H, W = s
    x = torch.rand((N, 1, H, W), generator=torch.Generator().manual_seed(N * H + W)).cuda()
    return torch.cat([f.reshape(-1) for f in m(x)])


def _unet_plan_state(L):
    return lambda m, s: (m.num_launches(), m.plan_info(*s, L=L)[2])


def _vae_plan_state(m, F):
    return (m.cached_plans(False)[0], m.cached_plans(True)[0])


def _sd():
    from t2v_b200.modules import UNetSD
    return UNetSD(dim=64)


def _vc():
    from t2v_b200.modules import UNetModel
    return UNetModel(model_channels=64, context_dim=48, temporal_length=4)


def _open_clip():
    from t2v_b200.clip import FrozenOpenCLIPEmbedder
    return FrozenOpenCLIPEmbedder(width=128, heads=2, layers=4, vocab=300).model


def _clip_l():
    from t2v_b200.clip import FrozenCLIPEmbedder
    return FrozenCLIPEmbedder(width=128, heads=2, layers=3, vocab=300).transformer


def _vae():
    from t2v_b200.modules import AutoencoderKL
    from t2v_b200.pipeline import VAE_DDCONFIG
    return AutoencoderKL(VAE_DDCONFIG, 4)


def _adapter(cfg):
    def make():
        from t2v_b200.adapter import Adapter
        return Adapter(**cfg)
    return make


ST = 'input_blocks.1.1.transformer_blocks.0.'
UNET_SD_SINGLES = [  # name -> the packed variant it feeds
    (ST + 'attn1.to_q.weight', 'q of the fused q|k|v, LayerNorm-folded'),
    (ST + 'attn1.to_k.weight', 'k of the fused q|k|v, LayerNorm-folded'),
    (ST + 'attn1.to_v.weight', 'v of the fused q|k|v, LayerNorm-folded'),
    (ST + 'attn2.to_q.weight', 'LayerNorm fold over a raw weight'),
    (ST + 'attn2.to_k.weight', 'k of the cross-attention k|v'),
    (ST + 'attn2.to_v.weight', 'v of the cross-attention k|v'),
    (ST + 'ff.net.0.proj.weight', 'GEGLU interleave, then the fold'),
    ('input_blocks.0.1.transformer_blocks.0.attn2.to_v.weight', 'temporal transformer q|k|v'),
    ('input_blocks.1.0.in_layers.2.weight', '3x3 conv, tap-major'),
    ('out.2.weight', '3x3 conv, padded to 16 outputs'),
    ('input_blocks.1.0.temopral_conv.conv1.2.weight', 'temporal conv, 3 taps'),
    ('input_blocks.3.op.weight', 'stride-2 conv, K-major'),
    ('input_blocks.0.1.proj_in.weight', 'raw Conv1d k=1'),
    ('input_blocks.4.0.skip_connection.weight', 'raw 1x1 conv'),
    ('middle_block.1.proj_out.weight', 'raw Linear'),
]
UNET_VC_SINGLES = [
    (ST + 'attn1.to_q.weight', 'q of the fused q|k|v, LayerNorm-folded'),
    (ST + 'attn1.to_k.weight', 'k of the fused q|k|v, LayerNorm-folded'),
    (ST + 'attn1.to_v.weight', 'v of the fused q|k|v, LayerNorm-folded'),
    (ST + 'attn1_tmp.to_k.weight', 'relative-position temporal q|k|v'),
    (ST + 'attn2.to_q.weight', 'LayerNorm fold over a raw weight'),
    (ST + 'attn2.to_k.weight', 'k of the cross-attention k|v'),
    (ST + 'attn2.to_v.weight', 'v of the cross-attention k|v'),
    (ST + 'ff.net.0.proj.weight', 'GEGLU interleave, then the fold'),
    ('input_blocks.1.0.in_layers.2.weight', '(1,3,3) conv, tap-major'),
    ('out.2.weight', '(1,3,3) conv, padded to 16 outputs'),
    ('input_blocks.3.0.op.weight', 'stride-2 conv, K-major'),
    ('input_blocks.1.1.proj_in.weight', 'raw 1x1x1 conv'),
    ('time_embed.0.weight', 'raw Linear of the time embedding'),
]
OPEN_CLIP_SINGLES = [
    ('transformer.resblocks.0.attn.in_proj_weight', 'LayerNorm fold over the raw in_proj'),
    ('transformer.resblocks.1.mlp.c_fc.weight', 'LayerNorm fold over a raw weight'),
    ('transformer.resblocks.0.attn.out_proj.weight', 'raw Linear'),
    ('transformer.resblocks.2.mlp.c_proj.weight', 'raw Linear'),
]
CLIP_L_SINGLES = [
    ('text_model.encoder.layers.0.self_attn.q_proj.weight', 'q of the fused q|k|v, LayerNorm-folded'),
    ('text_model.encoder.layers.1.self_attn.k_proj.weight', 'k of the fused q|k|v, LayerNorm-folded'),
    ('text_model.encoder.layers.2.self_attn.v_proj.weight', 'v of the fused q|k|v, LayerNorm-folded'),
    ('text_model.encoder.layers.1.mlp.fc1.weight', 'LayerNorm fold over a raw weight'),
    ('text_model.encoder.layers.0.mlp.fc2.weight', 'raw Linear'),
]
VAE_SINGLES = [
    ('decoder.mid.block_1.conv1.weight', '3x3 conv, tap-major'),
    ('decoder.conv_out.weight', '3x3 conv, padded to 16 outputs'),
    ('post_quant_conv.weight', 'padded 1-tap pack'),
    ('quant_conv.weight', 'padded 1-tap pack (encoder)'),
    ('encoder.down.0.downsample.conv.weight', 'stride-2 conv, K-major'),
    ('encoder.conv_in.weight', '3x3 conv of the encoder'),
    ('decoder.mid.attn_1.q.weight', 'raw 1x1 conv'),
    ('encoder.down.1.block.0.nin_shortcut.weight', 'raw 1x1 conv (encoder)'),
]
ADAPTER_A_SINGLES = [
    ('conv_in.weight', '3x3 conv, tap-major'),
    ('body.0.block1.weight', '3x3 conv, tap-major'),
    ('body.0.block2.weight', '1x1 conv'),
    ('body.2.in_conv.weight', '1x1 conv'),
]
ADAPTER_B_SINGLES = [
    ('body.3.down_opt.op.weight', 'stride-2 conv, K-major'),
    ('body.3.in_conv.weight', '3x3 conv, tap-major'),
    ('body.0.block2.weight', '3x3 conv, tap-major'),
]


class Handle(object):
    def __init__(self, ctor, specs, seed, shapes, run, singles, kind='apply', plan_state=None):
        self.ctor, self.specs, self.seed, self.shapes, self.run = ctor, specs, seed, shapes, run
        self.singles, self.kind, self.plan_state = [n for n, _ in singles], kind, plan_state
        self._W = None

    def weights(self):
        """The full state dict every instance loads (tensors the library does not run keep one fixed value too)."""
        if self._W is None:
            m = self.ctor()
            W = {k: v.detach().clone() for k, v in m.state_dict().items()}
            W.update(UO.make_weights(self.specs(), seed=self.seed))
            self._W = W
        return self._W

    def make(self, changes=None):
        m = self.ctor().half()
        m.load_state_dict({**self.weights(), **(changes or {})}, strict=True)
        return m.cuda().eval()

    def state(self, m, s):
        return self.plan_state(m, s) if self.plan_state else None


SD_SHAPES = [(1, 3, 8, 8), (1, 2, 8, 16), (2, 2, 8, 8), (1, 2, 16, 8), (1, 4, 8, 16), (1, 1, 16, 16)]   # > the bound of 4
HANDLES = {
    'unet_sd_merge': Handle(_sd, lambda: UO.param_specs(UO.UNetConfig(dim=64)), 1, SD_SHAPES, _run_unet_sd, UNET_SD_SINGLES,
                            'merge', _unet_plan_state(77)),
    'unet_sd_apply': Handle(_sd, lambda: UO.param_specs(UO.UNetConfig(dim=64)), 1, SD_SHAPES, _run_unet_sd, UNET_SD_SINGLES,
                            'apply', _unet_plan_state(77)),
    'unet_vc': Handle(_vc, lambda: VC.vc_param_specs(VC.VCConfig(model_channels=64, context_dim=48, temporal_length=4)), 4,
                      SD_SHAPES, _run_unet_vc, UNET_VC_SINGLES, 'apply', _unet_plan_state(9)),
    'clip_open': Handle(_open_clip, lambda: CO.clip_param_specs(CO.ClipConfig(width=128, heads=2, layers=4, layers_run=3,
                                                                              context=77, vocab=300)),
                        4, [2, 3], _run_tower, OPEN_CLIP_SINGLES),
    'clip_l': Handle(_clip_l, lambda: CL.clip_l_param_specs(CL.NARROW), 5, [2, 3], _run_tower, CLIP_L_SINGLES),
    'vae': Handle(_vae, lambda: {**VO.decoder_param_specs(VO.VAEConfig()), **VO.encoder_param_specs(VO.VAEConfig())}, 3,
                  [2, 3], _run_vae, VAE_SINGLES, plan_state=_vae_plan_state),
    'adapter_A': Handle(_adapter(AO.NARROW_A), lambda: AO.adapter_param_specs(**AO.NARROW_A), 21, [(1, 64, 64), (2, 64, 128)],
                        _run_adapter, ADAPTER_A_SINGLES),
    'adapter_B': Handle(_adapter(AO.NARROW_B), lambda: AO.adapter_param_specs(**AO.NARROW_B), 22, [(1, 64, 64), (2, 64, 128)],
                        _run_adapter, ADAPTER_B_SINGLES),
}


def _temporal(shape):
    return len(shape) == 5 and tuple(shape[2:]) == (3, 1, 1)


def _factors(h, m, name, salt=0, rank=4):
    """Distinct seeded LoRA factors for one weight; the product is about half the weight's own scale."""
    p = m.get_parameter(name)
    out, cols = p.shape[0], p.numel() // p.shape[0]
    seed = zlib.crc32(name.encode()) + 7919 * salt
    g = torch.Generator(device='cuda').manual_seed(seed)
    if h.kind == 'merge':
        t = _temporal(p.shape)
        ac = cols * 3 if t else cols
        A = (torch.randn(rank, ac, generator=g, device='cuda') / math.sqrt(ac)).half()
        B = (torch.randn(out, rank, generator=g, device='cuda') * (0.5 / math.sqrt(rank))).half()
        return ('merge', A, B, t)
    dt = torch.float32 if seed % 2 else torch.float16              # both factor types of lora_apply
    up = (torch.randn(out, rank, generator=g, device='cuda') * (0.5 / math.sqrt(rank))).to(dt)
    down = (torch.randn(rank, cols, generator=g, device='cuda') / math.sqrt(cols)).to(dt)
    return ('apply', up, down)


def _merge_into(m, name, f):
    if f[0] == 'merge':
        m.lora_merge(name, f[1], f[2], ALPHA, temporal_mean=f[3])
    else:
        m.lora_apply(name, f[1], f[2], ALPHA)


def _merged(base, f):
    """The merged weight the handle must hold: the same kernel on a copy of the base, through the op entry points."""
    from t2v_b200 import ops
    w = base.detach().clone()
    if f[0] == 'merge':
        return ops.lora_merge_(w, f[1], f[2], ALPHA, f[3])
    return ops.lora_apply_(w, f[1], f[2], ALPHA)


def _captured(h, m, s):
    """Runs shape s twice (the second run captures the plan's CUDA graph); returns the output and the plan state."""
    out = h.run(m, s)
    assert torch.equal(h.run(m, s), out)
    return out, h.state(m, s)


@pytest.fixture
def ops():
    from t2v_b200 import ops
    return ops


def _handle(key):
    return HANDLES[key]


@pytest.mark.parametrize('key', sorted(HANDLES))
def test_handle_weight_names_exist(key):
    """CPU: every weight the handle cases merge alone exists in the library's parameter table with the layout it stands for."""
    h = _handle(key)
    m = h.ctor()
    shapes = {n: tuple(m.get_parameter(n).shape) for n in m._native_names}
    for n in h.singles:
        assert n in shapes, n
        assert len(shapes[n]) >= 2, n
    assert sum(_temporal(shapes[n]) for n in h.singles) == (1 if key.startswith('unet_sd') else 0)
    assert set(h.specs()) <= set(m.state_dict())


@pytest.mark.gpu
@pytest.mark.parametrize('key', sorted(HANDLES))
def test_single_merges_repack_bit_for_bit(key):
    """Each weight of h.singles merged alone into a captured plan: A equals B (shipped that merged weight) bit for bit, the
    plan is not rebuilt, and lora_restore gives the base output back."""
    h = _handle(key)
    A, B = h.make(), h.make()
    s0 = h.shapes[0]
    base, st = _captured(h, A, s0)
    for name in h.singles:
        f = _factors(h, A, name)
        _merge_into(A, name, f)
        assert A.lora_merged() == 1, name
        assert h.state(A, s0) == st, name
        hot = h.run(A, s0)
        assert h.state(A, s0) == st, name
        B.load_state_dict({**h.weights(), name: _merged(A.get_parameter(name), f)}, strict=True)
        shipped = h.run(B, s0)
        assert not torch.equal(shipped, base), name                  # the merge changes the output
        assert torch.equal(hot, shipped), (name, (hot.float() - shipped.float()).abs().max().item())
        A.lora_restore(name)
        assert A.lora_merged() == 0
        assert torch.equal(h.run(A, s0), base), name


@pytest.mark.gpu
@pytest.mark.parametrize('key', sorted(HANDLES))
def test_every_weight_merged_then_restore_one_then_clear(key):
    h = _handle(key)
    A = h.make()
    s0 = h.shapes[0]
    base, st = _captured(h, A, s0)
    names = sorted(n for n in A._native_names if A.get_parameter(n).dim() >= 2)
    merged = {}
    for n in names:
        f = _factors(h, A, n, salt=1)
        _merge_into(A, n, f)
        merged[n] = _merged(A.get_parameter(n), f)
    assert A.lora_merged() == len(names)
    hot = h.run(A, s0)
    assert h.state(A, s0) == st
    assert torch.equal(hot, h.run(h.make(merged), s0))
    one = h.singles[0]
    A.lora_restore(one)
    assert A.lora_merged() == len(names) - 1
    rest = {k: v for k, v in merged.items() if k != one}
    assert torch.equal(h.run(A, s0), h.run(h.make(rest), s0))
    A.lora_clear()
    assert A.lora_merged() == 0
    assert torch.equal(h.run(A, s0), base)
    assert h.state(A, s0) == st


@pytest.mark.gpu
@pytest.mark.parametrize('key', sorted(HANDLES))
def test_merge_before_the_first_forward(key):
    h = _handle(key)
    A, B = h.make(), h.make()
    s0 = h.shapes[0]
    base, _ = _captured(h, B, s0)
    names = h.singles[:2]
    changes = {}
    for n in names:
        f = _factors(h, A, n, salt=2)
        _merge_into(A, n, f)                           # no plan exists yet: the first build packs the merged weights
        changes[n] = _merged(A.get_parameter(n), f)
    hot, _ = _captured(h, A, s0)
    B.load_state_dict({**h.weights(), **changes}, strict=True)
    assert torch.equal(hot, h.run(B, s0))
    A.lora_clear()
    assert torch.equal(h.run(A, s0), base)


@pytest.mark.gpu
@pytest.mark.parametrize('key', sorted(HANDLES))
def test_merge_then_a_new_shape_then_clear(key):
    h = _handle(key)
    A, B = h.make(), h.make()
    s0, s1 = h.shapes[0], h.shapes[1]
    base0, _ = _captured(h, A, s0)
    base1 = h.run(B, s1)
    name = h.singles[-1]
    f = _factors(h, A, name, salt=3)
    _merge_into(A, name, f)
    hot1 = h.run(A, s1)                                # a plan built after the merge
    B.load_state_dict({**h.weights(), name: _merged(A.get_parameter(name), f)}, strict=True)
    assert torch.equal(hot1, h.run(B, s1))
    assert torch.equal(h.run(A, s0), h.run(B, s0))
    A.lora_clear()
    assert torch.equal(h.run(A, s0), base0)
    assert torch.equal(h.run(A, s1), base1)


@pytest.mark.gpu
@pytest.mark.parametrize('key', ['unet_sd_merge', 'unet_vc'])
def test_merge_survives_plan_eviction(key):
    """More shapes than the UNet's plan cache holds (4) after a merge: the first shape's plan is rebuilt and carries it."""
    h = _handle(key)
    A, B = h.make(), h.make()
    s0 = h.shapes[0]
    _captured(h, A, s0)
    name = h.singles[0]
    f = _factors(h, A, name, salt=4)
    _merge_into(A, name, f)
    for s in h.shapes[1:]:
        h.run(A, s)
    assert not A.plan_info(*s0, L=77 if key == 'unet_sd_merge' else 9)[2]          # evicted
    hot = h.run(A, s0)
    B.load_state_dict({**h.weights(), name: _merged(A.get_parameter(name), f)}, strict=True)
    assert torch.equal(hot, h.run(B, s0))


@pytest.mark.gpu
@pytest.mark.parametrize('key', sorted(HANDLES))
def test_reshipped_weight_drops_its_merge(key):
    """A merged weight re-shipped through load_state_dict: its merge is dropped, the output is that of the new weights, and a
    later lora_clear keeps them (restores only the weights still merged)."""
    h = _handle(key)
    A = h.make()
    s0 = h.shapes[0]
    _captured(h, A, s0)
    name, other = h.singles[0], h.singles[1]
    f, fo = _factors(h, A, name, salt=5), _factors(h, A, other, salt=5)
    _merge_into(A, name, f)
    _merge_into(A, other, fo)
    merged_other = _merged(A.get_parameter(other), fo)
    assert A.lora_merged() == 2
    new = (A.get_parameter(name).detach().float() * -0.5).half()
    A.load_state_dict({name: new}, strict=False)
    out = h.run(A, s0)
    assert A.lora_merged() == 1
    assert torch.equal(out, h.run(h.make({name: new, other: merged_other}), s0))
    A.lora_clear()
    assert A.lora_merged() == 0
    assert torch.equal(h.run(A, s0), h.run(h.make({name: new}), s0))


@pytest.mark.gpu
@pytest.mark.parametrize('key', sorted(HANDLES))
def test_refused_merges_leave_the_handle_untouched(key):
    from t2v_b200 import _lib
    h = _handle(key)
    A = h.make()
    s0 = h.shapes[0]
    base, st = _captured(h, A, s0)
    l, s, p = _lib.lib(), _lib.stream_ptr(), _lib.ptr
    kind = A._kind
    bias = sorted(n for n in A._native_names if A.get_parameter(n).dim() == 1)[0]
    name = h.singles[0]
    f = _factors(h, A, name)
    up, down = (f[2], f[1]) if f[0] == 'merge' else (f[1], f[2])
    dt = int(up.dtype == torch.float32)
    apply = getattr(l, f't2v_{kind}_lora_apply')
    handle = A._handle
    assert apply(handle, b'no.such.weight', p(up), p(down), dt, 4, 1.0, s) != 0
    assert apply(handle, bias.encode(), p(up), p(down), dt, 4, 1.0, s) != 0
    assert apply(handle, name.encode(), p(up), p(down), dt, 0, 1.0, s) != 0
    assert apply(handle, name.encode(), p(up), p(down), 2, 4, 1.0, s) != 0
    if kind == 'unet':
        conv = next(n for n in h.singles if not _temporal(A.get_parameter(n).shape))
        fc = _factors(HANDLES['unet_sd_merge'], A, conv)
        assert l.t2v_unet_lora_merge(handle, conv.encode(), p(fc[1]), p(fc[2]), 4, 1.0, 1, s) != 0     # temporal_mean, not (3,1,1)
        assert l.t2v_unet_lora_merge(handle, b'no.such.weight', p(fc[1]), p(fc[2]), 4, 1.0, 0, s) != 0
        assert l.t2v_unet_lora_merge(handle, bias.encode(), p(fc[1]), p(fc[2]), 4, 1.0, 0, s) != 0
        assert l.t2v_unet_lora_merge(handle, conv.encode(), p(fc[1]), p(fc[2]), 0, 1.0, 0, s) != 0
    assert A.lora_merged() == 0
    assert torch.equal(h.run(A, s0), base)
    assert h.state(A, s0) == st
