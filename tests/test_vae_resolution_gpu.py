"""GPU: the VAE at the resolutions the pipeline runs -- 256^2 (32 x 32 latent), 576 x 1024 (72 x 128, ZeroScope) and the
UI's largest 1024^2 (128 x 128) -- against fp64 references.  At these shapes the mid-block attention's per-frame S x S
scores reach S = 16384 columns, its P.V GEMM accumulates over K = S, and the level-0 GroupNorms normalise a million rows
per instance: all past what the toy-size fixtures reach.

1. The attention block's pieces (vae.cu attn_block: batched score GEMM, softmax_rows, transpose_batched, P.V GEMM) at
   production S, each against an fp64 restatement on the same fp16 operands, rounded where the kernels' contracts round:
   GEMMs within 1/2 fp16 ulp of the result + K 2^-24 sum|a b| (fp32 accumulation) and 2e-3 max|ref|; softmax within
   1 fp16 ulp; the transpose bit for bit; the composed block against fp64 attention on the same q, k, v.  Scores past
   65504 overflow as the reference's fp16 bmm does, and the rows holding +inf come out NaN, as torch.softmax gives.
2. GroupNorm at the VAE's largest instances (576 x 1024 and 1024^2 rows, C 128 / 256), fused phase 0, against fp64 under
   test_norm_gpu.py's bound.
3. The decoder and encoder block by block (the library's taps) and whole, against oracle/vae_oracle.py run in fp64 on the
   GPU.  Gate (DESIGN.md section 5): relative RMS err(ours) <= 1.5 x err(the same oracle under torch.autocast(fp16), the
   reference's own GPU arithmetic), and absolute caps on relative RMS and max error; the uint8 frames within a few LSB.

Weights: seeded `make_weights`, with the tensors that write the residual stream (conv_in, every ResnetBlock's conv2,
the shortcut and resampling biases, the attention's proj_out) scaled by STREAM_GAIN = 1/32, then rounded to fp16.  Scaling
those is exact and moves the whole stream by the gain; at gain 1 the stream's group variance is ~27, where no GroupNorm
eps below ~0.1 changes anything visible.  At 1/32 the variance is ~0.03 (values still far from fp16's subnormals), so a
wrong eps (1e-3 instead of 1e-6 moves rstd by ~2 %) shows at norm_out.  `pytest -s` prints every error next to its gate."""
import contextlib

import numpy as np
import pytest
import torch

from oracle import unet_oracle as UO, vae_oracle as VO

pytestmark = pytest.mark.gpu
dev = 'cuda'
U16, U32 = 2.0 ** -11, 2.0 ** -24
C_ATT = 512                          # the mid block's width: single head, d = C
SCALE = 1.0 / 0.18215                # the pipeline's latent scale (t2v_pipeline.py:348)
STREAM_GAIN = 1.0 / 32
RMS_CAP, MAX_CAP = 4e-3, 6e-3        # the VAE gates of test_vc_lora_gpu.py
AUTOCAST_K = 1.5


@pytest.fixture(scope='module')
def ops():
    from t2v_b200 import ops as o
    return o


def gen(seed):
    return torch.Generator(device=dev).manual_seed(seed)


def fp16_ulp(v):
    """Spacing of fp16 at |v| (fp64 tensor): 2^-24 below the normal range, else 2^(floor(log2|v|) - 10)."""
    e = torch.floor(torch.log2(v.abs().clamp_min(2.0 ** -14)))
    return torch.pow(2.0, e - 10)


# ------------------------------------------------------------------------------------------------ 1. attention pieces
def gemm_ratio(out, ref, absprod, K):
    """Worst |out - ref| / (1/2 ulp16 + K 2^-24 sum|a b|) and max |out - ref|, out finite."""
    out = out.double()
    assert torch.isfinite(out).all(), 'non-finite GEMM output'
    err = (out - ref).abs()
    bound = 0.5 * fp16_ulp(torch.maximum(out.abs(), ref.abs())) + K * U32 * absprod
    return (err / bound).max().item(), err.max().item()


def softmax_ulps(p, ref):
    """Worst |p - ref| in fp16 ulps of the fp64 softmax."""
    return ((p.double() - ref).abs() / fp16_ulp(ref)).max().item()


def qkv(S, frames, sd, seed):
    g = gen(seed)
    q = (torch.randn(frames * S, C_ATT, device=dev, generator=g) * sd).half()
    k = (torch.randn(frames * S, C_ATT, device=dev, generator=g) * sd).half()
    v = torch.randn(frames * S, C_ATT, device=dev, generator=g).half()
    return q, k, v


def attn_chain(ops, q, k, v, S, frames):
    """vae.cu attn_block from q, k, v: the kernels' intermediates (scores, P, V^T) and the output."""
    sc = ops.gemm(q, k.view(frames, S, C_ATT), S, dims=[S, frames], taps=[[0, 0]], n_alloc=S, b_batch_dim=1)
    p = ops.softmax_rows(sc, C_ATT ** -0.5)
    vt = ops.transpose_batched(v.view(frames, S, C_ATT))
    o = ops.gemm(p, vt, C_ATT, dims=[S, frames], taps=[[0, 0]], n_alloc=C_ATT, b_batch_dim=1)
    return sc, p, vt, o


def row_blocks(S, frames, step=2048):
    """(frame, row slice of that frame, the same rows of the [frames * S, ...] matrices): fp64 references a block at a time."""
    for f in range(frames):
        for r0 in range(0, S, step):
            r1 = min(S, r0 + step)
            yield f, slice(r0, r1), slice(f * S + r0, f * S + r1)


@pytest.mark.parametrize('S,frames', [(1024, 3), (9216, 2), (16384, 1), (72 * 127, 2)])
def test_attn_block_pieces_at_production_S(ops, S, frames):
    """q, k of std 1.6: scores of std ~58 (max a few hundred, inside fp16), logits of std ~2.6, so each softmax row is
    led by a few tens of keys and P.V sums many small products.  Gates: score and P.V GEMMs 1 x their bound and 2e-3
    max|ref|; softmax 1 fp16 ulp; transpose bit for bit; the block vs fp64 attention 4e-3 relative RMS, 1e-2 max."""
    q, k, v = qkv(S, frames, 1.6, S + frames)
    sc, p, vt, o = attn_chain(ops, q, k, v, S, frames)
    assert torch.equal(vt, v.view(frames, S, C_ATT).transpose(1, 2))
    q64, k64, v64 = (t.double().view(frames, S, C_ATT) for t in (q, k, v))
    scale = float(np.float32(C_ATT ** -0.5))
    g_sc = g_pv = ulps = 0.0
    m_sc = m_pv = r_sc = r_pv = 0.0
    se = sr = me = mr = 0.0
    for f, rs, rows in row_blocks(S, frames):
        ref = q64[f, rs] @ k64[f].t()
        a, m = gemm_ratio(sc[rows], ref, q64[f, rs].abs() @ k64[f].abs().t(), C_ATT)
        g_sc, m_sc, r_sc = max(g_sc, a), max(m_sc, m), max(r_sc, ref.abs().max().item())
        att = torch.softmax(ref * C_ATT ** -0.5, dim=-1) @ v64[f]            # fp64 attention on the same q, k, v
        ulps = max(ulps, softmax_ulps(p[rows], torch.softmax((sc[rows].float() * scale).half().double(), dim=-1)))
        p64 = p[rows].double()
        ref = p64 @ v64[f]
        a, m = gemm_ratio(o[rows], ref, p64 @ v64[f].abs(), S)
        g_pv, m_pv, r_pv = max(g_pv, a), max(m_pv, m), max(r_pv, ref.abs().max().item())
        d = o[rows].double() - att
        se, sr = se + d.pow(2).sum().item(), sr + att.pow(2).sum().item()
        me, mr = max(me, d.abs().max().item()), max(mr, att.abs().max().item())
    rms, mx = (se / sr) ** 0.5, me / mr
    print(f'\n[S{S} x{frames}] scores |err|/bound {g_sc:.3f}, max err/max|ref| {m_sc / r_sc:.2e}; softmax {ulps:.3f} ulp; '
          f'P.V |err|/bound {g_pv:.3f}, max err/max|ref| {m_pv / r_pv:.2e}; block vs fp64 attention rms {rms:.2e} max {mx:.2e}',
          end='')
    assert g_sc <= 1.0 and m_sc <= 2e-3 * r_sc, ('scores', g_sc, m_sc / r_sc)
    assert ulps <= 1.0, ('softmax', ulps)
    assert g_pv <= 1.0 and m_pv <= 2e-3 * r_pv, ('P.V', g_pv, m_pv / r_pv)
    assert rms <= 4e-3 and mx <= 1e-2, ('attention', rms, mx)


def test_attn_block_score_overflow_matches_fp16_bmm(ops):
    """q, k of std 30: scores of std ~2e4, ~0.1 % of them past fp16's range.  The reference's fp16 bmm gives +-inf there;
    so must the score GEMM (either is allowed within 1e-3 of the threshold, where the fp32 sum order decides).  A row
    holding +inf softmaxes to NaN in torch (inf - inf); the kernel must give NaN in exactly those rows, and P.V carries
    the NaN to exactly those output rows.  The other rows keep the 1-ulp softmax gate."""
    S, frames = 1024, 2
    q, k, v = qkv(S, frames, 30.0, 7)
    sc, p, vt, o = attn_chain(ops, q, k, v, S, frames)
    q64, k64 = (t.double().view(frames, S, C_ATT) for t in (q, k))
    ref = torch.bmm(q64, k64.transpose(1, 2)).view(-1, S)
    over, under = ref.abs() >= 65520 * (1 + 1e-3), ref.abs() < 65520 * (1 - 1e-3)
    reduced = torch.backends.cuda.matmul.allow_fp16_reduced_precision_reduction
    torch.backends.cuda.matmul.allow_fp16_reduced_precision_reduction = False      # fp32 sums, as autocast's bmm on H100
    try:
        torch_sc = torch.bmm(q.view(frames, S, C_ATT), k.view(frames, S, C_ATT).transpose(1, 2)).view(-1, S)
    finally:
        torch.backends.cuda.matmul.allow_fp16_reduced_precision_reduction = reduced
    for name, s in (('ours', sc), ('torch fp16 bmm', torch_sc)):
        assert torch.equal(torch.isinf(s[over]), torch.ones_like(s[over], dtype=torch.bool)), name
        assert torch.equal(torch.sign(s[over]).double(), torch.sign(ref[over])), name
        assert torch.isfinite(s[under]).all(), name
    n_over = int(over.sum())
    assert n_over > 100, n_over
    pinf_rows = torch.isposinf(sc).any(dim=1)
    scale = float(np.float32(C_ATT ** -0.5))
    torch_p = torch.softmax((sc.float() * scale).half().float(), dim=-1)
    assert torch.equal(torch.isnan(torch_p).all(dim=1), pinf_rows)
    assert torch.equal(torch.isnan(p).all(dim=1), pinf_rows) and not torch.isnan(p[~pinf_rows]).any()
    ok = ~pinf_rows
    ulps = softmax_ulps(p[ok], torch.softmax((sc[ok].float() * scale).half().double(), dim=-1))
    assert ulps <= 1.0, ulps
    assert torch.equal(torch.isnan(o).all(dim=1), pinf_rows) and torch.isfinite(o[ok]).all()
    print(f'\n[score overflow] {n_over} scores past fp16, {int(pinf_rows.sum())} of {frames * S} rows hold +inf; other rows '
          f'softmax {ulps:.3f} ulp', end='')
    assert 0 < int(pinf_rows.sum()) < frames * S


# ------------------------------------------------------------------------------------------------ 2. GroupNorm
@pytest.mark.parametrize('R,n,C,silu,offset', [
    (576 * 1024, 2, 128, True, 0.0),        # decoder norm_out / level-0 ResnetBlocks at 576 x 1024
    (576 * 1024, 1, 256, False, 0.0),       # level-0 ResnetBlock norm1 of up.0.block.0 (256 in)
    (1024 * 1024, 1, 128, True, 0.0),       # norm_out at 1024^2
    (1024 * 1024, 1, 256, True, 100.0),     # a common offset of 100 std at 1024^2
    (1024 * 1024, 2, 128, False, 10.0),
])
def test_groupnorm_at_vae_instance_sizes(ops, R, n, C, silu, offset):
    """Phase 0 (the model's path) against fp64 under test_norm_gpu.py's fused bound, applied in slices of rows."""
    from t2v_b200 import _lib
    import test_norm_gpu as N
    sms = _lib.lib().t2v_num_sms()
    g = gen(R + C + n)
    z = torch.randn(n, R, C, device=dev, generator=g)
    if offset:
        sign = torch.randint(0, 2, (n, 1, 32, 1), device=dev, generator=g) * 2 - 1
        x = (z.view(n, R, 32, C // 32) + sign * offset).half().view(-1, C)
    else:
        loc = torch.randn(n, 1, C, device=dev, generator=g) * 2
        x = (z * (torch.rand(n, 1, C, device=dev, generator=g) * 2 + 0.3) + loc).half().view(-1, C)
    del z
    gamma, beta = N.affine(C, seed=C)
    kind, _, rpc = N.gn_plan(R, n, C, sms)
    y = ops.groupnorm(x, gamma, beta, R, 1e-6, silu)
    mean, rstd, dmean, drel = N.gn_stats64(x, n, R, C, 1e-6, rpc)
    cpg, slope = C // 32, (1.1 if silu else 1.0)
    worst = 0.0
    step = 1 << 17
    for i in range(n):
        for r0 in range(0, R, step):
            rows = slice(i * R + r0, i * R + min(R, r0 + step))
            xs = x[rows]
            ref, u, ab = N.gn_apply64(xs, 1, xs.shape[0], C, mean[i:i + 1], rstd[i:i + 1], gamma, beta, silu)
            carried = slope * (gamma.double().abs() * (rstd[i] * dmean[i]).repeat_interleave(cpg)
                               + (u - beta.double()).abs() * drel[i].repeat_interleave(cpg))
            out = y[rows].double()
            assert torch.isfinite(out).all()
            worst = max(worst, ((out - ref).abs() / (N.GATE_K * (ab + carried + N.out_round(ref)))).max().item())
    print(f'\n[groupnorm R{R} n{n} C{C} {kind} offset {offset}] worst |err| / gate = {worst:.3f}', end='')
    assert worst <= 1.0


# ------------------------------------------------------------------------------------------------ 3. decoder / encoder
def stream_gain(W, s):
    """W with the tensors that write the residual stream scaled by s (see the module docstring)."""
    def writes_stream(k):
        return (k.startswith(('decoder.conv_in.', 'encoder.conv_in.')) or '.conv2.' in k or '.attn_1.proj_out.' in k
                or (k.endswith('.bias') and ('.nin_shortcut.' in k or 'sample.conv.' in k)))
    return {k: v * s if writes_stream(k) else v for k, v in W.items()}


@pytest.fixture(scope='module')
def weights():
    cfg = VO.VAEConfig()
    W = {**UO.make_weights(VO.decoder_param_specs(cfg), seed=3), **UO.make_weights(VO.encoder_param_specs(cfg), seed=4)}
    return {k: v.half() for k, v in stream_gain(W, STREAM_GAIN).items()}


def make_ae(W, taps):
    from t2v_b200.modules import AutoencoderKL
    from t2v_b200.pipeline import VAE_DDCONFIG
    m = AutoencoderKL(VAE_DDCONFIG, 4, None).half()
    m.load_state_dict(W, strict=True)
    m = m.cuda().eval()
    if taps:
        m.enable_taps(True)
    return m


@pytest.fixture(scope='module')
def ae(weights):
    return make_ae(weights, taps=True)


# The oracle's block outputs under the library's tap names.  vae_decode records 'mid' (= mid.block_2) and 'up<lvl>'
# itself; the others are caught by wrapping the layer functions it calls: a ResnetBlock's input is the previous block's
# output (conv_in, the encoder's level outputs after their downsample conv), and norm_out is the GroupNorm + swish.
ENTRY_OF = {'decoder.mid.block_1': 'decoder.conv_in', 'encoder.down.0.block.0': 'encoder.conv_in',
            'encoder.down.1.block.0': 'encoder.down.0', 'encoder.down.2.block.0': 'encoder.down.1',
            'encoder.down.3.block.0': 'encoder.down.2', 'encoder.mid.block_1': 'encoder.down.3'}


@contextlib.contextmanager
def oracle_taps(sink):
    resnet, attn, gn = VO._resnet, VO._attn, VO._gn

    def _resnet(W, p, x):
        if p in ENTRY_OF:
            sink(ENTRY_OF[p], x)
        y = resnet(W, p, x)
        if '.mid.' in p:
            sink(p, y)
        return y

    def _attn(W, p, x):
        y = attn(W, p, x)
        sink(p, y)
        return y

    def _gn(W, p, x):
        y = gn(W, p, x)
        if p.endswith('.norm_out'):
            sink(p, VO._swish(y))
        return y

    VO._resnet, VO._attn, VO._gn = _resnet, _attn, _gn
    try:
        yield
    finally:
        VO._resnet, VO._attn, VO._gn = resnet, attn, gn


class DecodeTaps(dict):
    """vae_decode's own `taps` argument: 'up<lvl>' forwarded to the sink as 'decoder.up.<lvl>'."""

    def __init__(self, sink):
        super().__init__()
        self.sink = sink

    def __setitem__(self, k, v):
        if k.startswith('up'):
            self.sink(f'decoder.up.{k[2:]}', v)


def errs(a, r):
    """(relative RMS, max |a - r| / max |r|) in fp64, over slices of channels to bound the temporaries."""
    se = sr = me = mr = 0.0
    for i in range(0, r.shape[1], 32):
        d = a[:, i:i + 32].double() - r[:, i:i + 32].double()
        rr = r[:, i:i + 32].double()
        se += d.pow(2).sum().item()
        sr += rr.pow(2).sum().item()
        me = max(me, d.abs().max().item())
        mr = max(mr, rr.abs().max().item())
    return (se / sr) ** 0.5, me / mr


def gate(name, ours, auto, rms_cap=RMS_CAP, max_cap=MAX_CAP):
    """err(ours) <= 1.5 err(autocast) in relative RMS, and the absolute caps; returns a report line."""
    line = (f'{name:28s} ours rms {ours[0]:.2e} max {ours[1]:.2e} | autocast rms {auto[0]:.2e} max {auto[1]:.2e} | '
            f'gate rms <= {min(AUTOCAST_K * auto[0], rms_cap):.2e}, max <= {max_cap:.0e}')
    print('\n' + line, end='')
    ok = ours[0] <= AUTOCAST_K * auto[0] and ours[0] <= rms_cap and ours[1] <= max_cap
    return None if ok else line


def run_oracles(fn, W, x, ae=None):
    """fn(W, x) = the oracle in fp64 and under autocast(fp16) on the GPU.  Returns (fp64 output, autocast output,
    failing tap lines); with `ae`, every tap of the library's last plan is gated against the fp64 oracle's."""
    Wg = {k: v.to(dev) for k, v in W.items()}
    auto_taps = {}
    with torch.autocast('cuda', dtype=torch.float16), oracle_taps(auto_taps.__setitem__):
        auto = fn({k: v.float() for k, v in Wg.items()}, x.float(), DecodeTaps(auto_taps.__setitem__)).float()
    fails = []

    def check(name, ref):
        if ae is None:
            return
        line = gate(f'tap {name}', errs(ae.read_tap(name), ref), errs(auto_taps.pop(name), ref))
        if line:
            fails.append(line)

    with oracle_taps(check):
        ref = fn({k: v.double() for k, v in Wg.items()}, x.double(), DecodeTaps(check))
    return ref, auto, fails


def decode_fn(W, z, taps):
    return VO.vae_decode(W, VO.VAEConfig(), z, taps=taps)


def encode_fn(W, x, taps):
    return VO.vae_encode_moments(W, VO.VAEConfig(), x)


def latent(frames, h, w, seed):
    """A sampler latent [1, 4, F, h, w] (CPU) and what the decoder sees: fp16(z / 0.18215) per frame, [F, 4, h, w]."""
    z = torch.randn(1, 4, frames, h, w, generator=torch.Generator().manual_seed(seed))
    return z, (z * float(np.float32(SCALE))).half()[0].permute(1, 0, 2, 3).contiguous()


_OUT = {}        # (frames, h, w) -> (fp64 output, autocast output) of the oracles, shared with the chunked test


@pytest.mark.parametrize('frames,h,w', [(2, 32, 32), (2, 72, 128), (1, 128, 128)])
def test_decode_block_by_block_vs_fp64_oracle(ae, weights, frames, h, w):
    z, zin = latent(frames, h, w, seed=frames * 1000 + h)
    out = ae.decode_video(z.cuda(), SCALE, as_uint8=False)
    assert ae.last_chunking() == (frames, 1)
    ref, auto, fails = run_oracles(decode_fn, weights, zin.to(dev), ae)
    _OUT[(frames, h, w)] = (ref.float(), auto)
    line = gate(f'decode {frames}x{8 * h}x{8 * w}', errs(out, ref), errs(auto, ref))
    assert not fails and not line, fails + [line]
    u8 = ae.decode_video(z.cuda(), SCALE, as_uint8=True).cpu()
    ref_u8 = torch.from_numpy(VO.tensor2vid_u8(ref.float().cpu()[None].permute(0, 2, 1, 3, 4)))
    diff = (u8.int() - ref_u8.int()).abs()
    print(f'\n[uint8 {frames}x{8 * h}x{8 * w}] max {diff.max().item()} LSB (gate 3), mean {diff.float().mean():.3f} (gate 0.5)',
          end='')
    assert u8.shape == ref_u8.shape and diff.max() <= 3 and diff.float().mean() < 0.5


def test_chunked_decode_576x1024_vs_fp64_oracle(weights):
    """The 576 x 1024 decode forced into two one-frame chunks by a budget between the one- and two-frame plans, against the
    same oracle and gates as the whole-clip decode (a handle without taps: the production plans)."""
    frames, h, w = 2, 72, 128
    z, zin = latent(frames, h, w, seed=frames * 1000 + h)
    m = make_ae(weights, taps=False)
    one, two = m.plan_bytes(1, h, w), m.plan_bytes(2, h, w)
    m.memory_budget = (one + two) // 2
    try:
        out = m.decode_video(z.cuda(), SCALE, as_uint8=False)
        assert m.last_chunking() == (1, 2)
    finally:
        m.memory_budget = 0
    if (frames, h, w) not in _OUT:
        ref, auto, _ = run_oracles(decode_fn, weights, zin.to(dev))
        _OUT[(frames, h, w)] = (ref.float(), auto)
    ref, auto = _OUT[(frames, h, w)]
    line = gate('decode 2x576x1024 chunked', errs(out, ref), errs(auto, ref))
    assert not line, line


def test_encode_576x1024_block_by_block_vs_fp64_oracle(ae, weights):
    """vid2vid's encode of one 576 x 1024 frame: the stride-2 im2col + GEMM downsamples (K = 9 C) at w = 1024 and 512, the
    mid attention at S = 72 x 128.  The moments' mean under the decoder's gates; the logvar under the 1.5 x rule and the
    2e-2 relative RMS of test_model_gpu.py's encode check."""
    x = torch.rand((1, 3, 576, 1024), generator=torch.Generator().manual_seed(17)) * 2 - 1
    mom = ae.encode(x.cuda()).parameters
    assert ae.last_chunking(encode=True) == (1, 1)
    ref, auto, fails = run_oracles(encode_fn, weights, x.half().to(dev), ae)
    fails.append(gate('encode mean', errs(mom[:, :4], ref[:, :4]), errs(auto[:, :4], ref[:, :4])))
    fails.append(gate('encode logvar', errs(mom[:, 4:], ref[:, 4:]), errs(auto[:, 4:], ref[:, 4:]), rms_cap=2e-2,
                      max_cap=float('inf')))
    fails = [f for f in fails if f]
    assert not fails, fails
