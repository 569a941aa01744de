"""GPU: the glue kernels of csrc/elementwise.cu (layout ingest / egress, stride-2 gather, pooling, pixel unshuffle, ReLU, feature
add, concat, transpose, frame conversion, fp16 conversion, row softmax, sampler updates) against plain references of the same
operation on the CPU.

Most of these kernels have an exact contract (kernels.cuh, include/t2v_b200.h): a copy, one fp16 rounding of an fp32 value, or a
fixed op order in fp32 / fp64.  Those are checked bit for bit (float outputs compared as integer bit patterns) against a torch
restatement in the kernel's own op order.  Outputs start out filled with a sentinel (a NaN payload no kernel produces, or two
different byte values for uint8) and carry guard elements past their end, so an element the kernel skips or a write past a row
or the buffer fails.  Every kernel also runs one shape whose element count exceeds the 132 * 16 * 256 threads of its grid, so the
grid-stride loop wraps.  softmax_rows (__expf) and lincomb (fmaf chain) are gated at one ulp of an fp64 reference."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
dev = 'cuda'
WRAP = 132 * 16 * 256          # threads of a capped grid_for grid: larger problems take more than one grid-stride pass

_INT = {torch.float16: torch.int16, torch.float32: torch.int32, torch.float64: torch.int64, torch.uint8: torch.uint8}
_SENTINEL = {torch.float16: 0x7E5A, torch.float32: 0x7FA5A5A5, torch.float64: 0x7FF5A5A5A5A5A5A5, torch.uint8: 0xA5}


@pytest.fixture(scope='module')
def ops():
    from t2v_b200 import ops as o
    return o


@pytest.fixture(scope='module')
def lib():
    from t2v_b200 import _lib
    return _lib


def gen(seed):
    return torch.Generator().manual_seed(seed)


def sentinel(n, dtype, value=None):
    """A flat CUDA buffer of n elements holding the sentinel bit pattern."""
    t = torch.empty(n, dtype=dtype, device=dev)
    t.view(_INT[dtype]).fill_(_SENTINEL[dtype] if value is None else value)
    return t


def bits(t):
    return t.detach().cpu().contiguous().view(_INT[t.dtype])


def assert_bits(out, ref, what=''):
    """out (any device) equals ref bit for bit."""
    assert out.shape == ref.shape and out.dtype == ref.dtype, (what, out.shape, ref.shape, out.dtype, ref.dtype)
    ob, rb = bits(out), bits(ref)
    bad = (ob != rb).nonzero()
    assert bad.numel() == 0, f'{what}: {bad.shape[0]} of {ob.numel()} elements differ, first at {bad[0].tolist()}: ' \
                             f'{out.cpu()[tuple(bad[0])].item()!r} vs {ref.cpu()[tuple(bad[0])].item()!r}'


def halves(shape, g, scale=1.0):
    return (torch.randn(shape, generator=g) * scale).half()


def all_halves():
    """Every fp16 bit pattern, once."""
    return torch.arange(65536, dtype=torch.int32).to(torch.int16).view(torch.float16)


# ------------------------------------------------------------------------------------------------ ingest / egress
@pytest.mark.parametrize('B,Cc,Fr,h,w,cpad,ld,frame0,nframes,src,scale', [
    (2, 4, 3, 5, 7, 8, 8, 0, None, torch.float32, 1 / 0.18215),       # whole latent, odd h and w, pad columns
    (3, 4, 3, 5, 7, 8, 16, 2, 5, torch.float16, 1.0),                  # starts and ends mid-sample, ld > cpad
    (3, 4, 3, 5, 7, 8, 16, 4, 4, torch.float32, 1 / 0.18215),          # starts mid-sample, crosses two boundaries
    (2, 3, 4, 1, 1, 8, 24, 3, 3, torch.float32, 1.0),                  # h * w = 1, C = 3
    (1, 4, 5, 9, 3, 16, 16, 1, 3, torch.float16, 5.4899),              # scale != 1 on fp16, inner frames of one sample
    (2, 8, 2, 3, 1, 8, 8, 0, None, torch.float16, 1.0),                # C = cpad
    (2, 4, 16, 64, 64, 8, 8, 0, None, torch.float32, 1 / 0.18215),     # grid-stride wrap
    (2, 4, 24, 40, 72, 8, 16, 7, 30, torch.float16, 0.5),              # wrap, mid-sample range
])
def test_ingest_latent(ops, B, Cc, Fr, h, w, cpad, ld, frame0, nframes, src, scale):
    scale = float(np.float32(scale))          # the kernel takes an fp32 scale
    g = gen(1)
    x = torch.randn(B, Cc, Fr, h, w, generator=g).to(src)
    nframes = B * Fr - frame0 if nframes is None else nframes
    rows = nframes * h * w
    assert rows * cpad > WRAP or rows * cpad < 4096
    buf = sentinel((rows + 3) * ld, torch.float16)
    tok = buf[:rows * ld].view(rows, ld)
    ops.ingest_latent(x.to(dev), tok, cpad, frame0, nframes, scale)
    frames = x.permute(0, 2, 3, 4, 1).reshape(B * Fr, h * w, Cc)[frame0:frame0 + nframes].reshape(rows, Cc)
    ref = sentinel((rows + 3) * ld, torch.float16).cpu()
    r2 = ref[:rows * ld].view(rows, ld)
    r2[:, :Cc] = (frames.float() * scale).half()
    r2[:, Cc:cpad] = 0
    assert_bits(buf, ref, 'ingest')


@pytest.mark.parametrize('B,Cc,Fr,h,w,ld,dst', [
    (2, 4, 3, 5, 7, 8, torch.float32), (2, 4, 3, 5, 7, 8, torch.float16), (1, 4, 5, 1, 1, 8, torch.float16),
    (3, 3, 2, 9, 3, 16, torch.float32), (2, 4, 24, 48, 61, 8, torch.float32), (2, 4, 24, 48, 61, 16, torch.float16)])
def test_egress_latent(ops, B, Cc, Fr, h, w, ld, dst):
    n = B * Cc * Fr * h * w
    assert n > WRAP or n < 4096
    tok = halves((B * Fr * h * w, ld), gen(2))
    buf = sentinel(n + 5, dst)
    ops.egress_latent(tok.to(dev), buf[:n].view(B, Cc, Fr, h, w))
    ref = sentinel(n + 5, dst).cpu()
    ref[:n] = tok[:, :Cc].reshape(B, Fr, h, w, Cc).permute(0, 4, 1, 2, 3).reshape(-1).to(dst)
    assert_bits(buf, ref, 'egress')


def test_ingest_egress_round_trip(ops):
    """egress(ingest(x)) of an fp16 latent with scale 1 is x itself, -0 and subnormals included."""
    x = all_halves()
    x = x[~torch.isnan(x)]
    x = x[torch.randperm(x.numel(), generator=gen(18))[:2 * 4 * 3 * 5 * 77]].view(2, 4, 3, 5, 77)
    tok = sentinel(2 * 3 * 5 * 77 * 8, torch.float16).view(-1, 8)
    ops.ingest_latent(x.to(dev), tok, 8)
    out = sentinel(x.numel(), torch.float16).view(x.shape)
    ops.egress_latent(tok, out)
    assert_bits(out, x, 'round trip')


# ------------------------------------------------------------------------------------------------ im2col_s2
def im2col_ref(x, pad_lo):
    nf, h, w, Cc = x.shape
    xn = x.permute(0, 3, 1, 2).float()
    if pad_lo == 0:
        xn = F.pad(xn, (0, 1, 0, 1))           # ldm Downsample: pad right and bottom by one, then a padding-0 conv
    ho, wo = ((h + 1) // 2, (w + 1) // 2) if pad_lo else (h // 2, w // 2)
    cols = F.unfold(xn, 3, padding=pad_lo, stride=2)                 # [nf, C * 9, ho * wo], row c * 9 + tap
    return cols.view(nf, Cc, 9, ho * wo).permute(0, 3, 2, 1).reshape(nf, ho, wo, 9 * Cc).half()


@pytest.mark.parametrize('pad_lo', [0, 1])
@pytest.mark.parametrize('nf,h,w,Cc', [(2, 7, 9, 8), (3, 8, 6, 16), (2, 2, 2, 8), (1, 2, 5, 24), (2, 5, 2, 8),
                                       (2, 1, 6, 8), (2, 7, 1, 16), (1, 1, 1, 8), (3, 3, 3, 8), (8, 64, 63, 64),
                                       (8, 65, 64, 64)])
def test_im2col_s2(ops, nf, h, w, Cc, pad_lo):
    x = halves((nf, h, w, Cc), gen(3))
    ho, wo = ((h + 1) // 2, (w + 1) // 2) if pad_lo else (h // 2, w // 2)
    n = nf * ho * wo * 9 * Cc
    assert n // 8 > WRAP or n < 65536
    buf = sentinel(n + 8, torch.float16)
    ops.im2col_s2(x.to(dev), pad_lo=pad_lo, out=buf[:n].view(nf, ho, wo, 9 * Cc))
    ref = sentinel(n + 8, torch.float16).cpu()
    if n:                                      # pad_lo = 0 with h or w = 1: no output (the reference's conv would refuse it)
        ref[:n] = im2col_ref(x, pad_lo).reshape(-1)
    assert_bits(buf, ref, f'im2col pad_lo={pad_lo}')


# ------------------------------------------------------------------------------------------------ avgpool2x2
def avgpool_ref(x):
    """The kernel's op order: fp32 ((((0 + x00) + x01) + x10) + x11) * 0.25, one fp16 rounding."""
    nf, h, w, Cc = x.shape
    ho, wo = h // 2, w // 2
    xf = x.float()[:, :2 * ho, :2 * wo]
    acc = torch.zeros(nf, ho, wo, Cc)
    for dy, dx in ((0, 0), (0, 1), (1, 0), (1, 1)):
        acc = acc + xf[:, dy::2, dx::2]
    return (acc * 0.25).half()


@pytest.mark.parametrize('nf,h,w,Cc', [(2, 5, 7, 8), (3, 8, 6, 16), (2, 2, 2, 8), (1, 3, 3, 24), (4, 33, 17, 24),
                                       (3, 1, 4, 16), (1, 9, 1, 8), (16, 96, 97, 128)])
def test_avgpool2x2(ops, nf, h, w, Cc):
    x = halves((nf, h, w, Cc), gen(4), 3.0)
    n = nf * (h // 2) * (w // 2) * Cc
    assert n // 8 > WRAP or n < 65536
    buf = sentinel(n + 8, torch.float16)
    ops.avgpool2x2(x.to(dev), out=buf[:n].view(nf, h // 2, w // 2, Cc))
    ref = sentinel(n + 8, torch.float16).cpu()
    ref[:n] = avgpool_ref(x).reshape(-1)
    assert_bits(buf, ref, 'avgpool')


def test_avgpool2x2_sums_in_fp32_near_fp16_max(ops):
    """Taps near 65504: an fp16 running sum would overflow to inf, the kernel's fp32 sum must not; mixed signs cancel."""
    g = gen(5)
    mag = 60000 + torch.rand(4, 10, 12, 32, generator=g) * 5504
    sign = torch.where(torch.rand(mag.shape, generator=g) < 0.2, -1.0, 1.0)
    x = (mag * sign).half()
    x[0, :2, :2] = 65504                      # four maximal taps: exactly 65504 again
    y = ops.avgpool2x2(x.to(dev))
    ref = avgpool_ref(x)
    assert torch.isfinite(ref.float()).all()
    assert_bits(y, ref, 'avgpool near 65504')
    assert (y[0, 0, 0].cpu().float() == 65504).all()


# ------------------------------------------------------------------------------------------------ pixel_unshuffle
@pytest.mark.parametrize('N,Cc,H,W,src', [(2, 1, 16, 24, torch.float32), (3, 3, 8, 8, torch.float16), (1, 3, 40, 64, torch.float32),
                                          (2, 1, 8, 48, torch.float16), (8, 3, 512, 512, torch.float32),
                                          (4, 1, 1024, 1088, torch.float16)])
def test_pixel_unshuffle(ops, N, Cc, H, W, src):
    x = torch.randn(N, Cc, H, W, generator=gen(6)).to(src)
    n = N * Cc * H * W
    assert n // 8 > WRAP or n < 65536
    buf = sentinel(n + 8, torch.float16)
    ops.pixel_unshuffle(x.to(dev), out=buf[:n].view(-1, 64 * Cc))
    ref = sentinel(n + 8, torch.float16).cpu()
    ref[:n] = F.pixel_unshuffle(x.float(), 8).permute(0, 2, 3, 1).half().reshape(-1)
    assert_bits(buf, ref, 'pixel_unshuffle')


# ------------------------------------------------------------------------------------------------ relu
def test_relu_every_fp16_pattern(ops):
    """nn.ReLU on all 65536 fp16 bit patterns: the same values as torch.relu (+-0, +-inf, subnormals), NaN stays NaN
    (torch.relu propagates it; a plain max(x, 0) would give 0).  The kernel returns +0 for -0, torch.relu returns -0:
    equal values, different sign bit."""
    x = all_halves().view(-1, 8)
    y = ops.relu_(x.clone().to(dev)).cpu()
    ref = torch.relu(x)
    nan = torch.isnan(ref)
    assert torch.equal(torch.isnan(y), nan), 'NaN inputs must stay NaN'
    assert torch.equal(y[~nan], ref[~nan])
    nz = ~nan & (ref != 0)
    assert torch.equal(bits(y)[nz], bits(ref)[nz])
    zero = ~nan & (ref == 0)
    assert (bits(y)[zero] == 0).all(), 'every input <= 0 (including -0) gives +0'


@pytest.mark.parametrize('rows,Cc', [(1, 8), (37, 24), (100000, 48)])
def test_relu_dense(ops, rows, Cc):
    x = halves((rows, Cc), gen(7), 2.0)
    assert rows * Cc // 8 > WRAP or rows * Cc < 65536
    buf = sentinel(rows * Cc + 8, torch.float16)
    buf[:rows * Cc] = x.reshape(-1).to(dev)
    ops.relu_(buf[:rows * Cc].view(rows, Cc))
    ref = sentinel(rows * Cc + 8, torch.float16).cpu()
    ref[:rows * Cc] = torch.where(x > 0, x, torch.zeros_like(x)).reshape(-1)      # +0 for every input <= 0, as the kernel
    assert_bits(buf, ref, 'relu')


# ------------------------------------------------------------------------------------------------ feature_add
@pytest.mark.parametrize('samples,rps,fs,Cc,ldx', [
    (4, 13, 2, 16, 24),       # CFG halves: samples 0, 2 read feature sample 0, samples 1, 3 read 1; rps not a multiple of 8
    (3, 7, 1, 8, 8),          # one feature sample broadcast over the batch
    (6, 5, 3, 24, 32),
    (2, 1, 2, 8, 16),
    (5, 9, 5, 40, 40),        # one feature sample per sample
    (2, 40000, 1, 64, 72),    # grid-stride wrap
])
def test_feature_add(ops, samples, rps, fs, Cc, ldx):
    g = gen(8)
    rows = samples * rps
    assert rows * Cc // 8 > WRAP or rows * Cc < 65536
    x = halves((rows, Cc), g)
    f = halves((fs * rps, Cc), g)
    buf = sentinel((rows + 2) * ldx, torch.float16)
    xv = buf[:rows * ldx].view(rows, ldx)
    xv[:, :Cc] = x.to(dev)
    ops.feature_add_(xv[:, :Cc], f.to(dev), rps, fs)
    r = torch.arange(rows)
    idx = (r // rps % fs) * rps + r % rps
    ref = sentinel((rows + 2) * ldx, torch.float16).cpu()
    ref[:rows * ldx].view(rows, ldx)[:, :Cc] = (x.float() + f[idx].float()).half()
    assert_bits(buf, ref, 'feature_add')


# ------------------------------------------------------------------------------------------------ concat_cols
@pytest.mark.parametrize('rows,Ca,Cb,lda,ldb,ldo', [(37, 8, 24, 16, 40, 40), (5, 24, 8, 24, 8, 48), (1, 8, 8, 8, 8, 16),
                                                    (300, 40, 56, 48, 64, 104), (50000, 72, 40, 80, 40, 120)])
def test_concat_cols(ops, rows, Ca, Cb, lda, ldb, ldo):
    g = gen(9)
    assert rows * (Ca + Cb) // 8 > WRAP or rows < 1000
    a = halves((rows, lda), g)
    b = halves((rows, ldb), g)
    buf = sentinel((rows + 2) * ldo, torch.float16)
    ops.concat_cols(a.to(dev)[:, :Ca], b.to(dev)[:, :Cb], buf[:rows * ldo].view(rows, ldo))
    ref = sentinel((rows + 2) * ldo, torch.float16).cpu()
    r2 = ref[:rows * ldo].view(rows, ldo)
    r2[:, :Ca] = a[:, :Ca]
    r2[:, Ca:Ca + Cb] = b[:, :Cb]
    assert_bits(buf, ref, 'concat')


# ------------------------------------------------------------------------------------------------ transpose_batched
@pytest.mark.parametrize('nb,R,Cc', [(3, 1, 1), (2, 33, 31), (1, 32, 64), (5, 1, 77), (4, 100, 1), (2, 1000, 333),
                                     (3, 31, 32)])
def test_transpose_batched(ops, nb, R, Cc):
    x = halves((nb, R, Cc), gen(10))
    n = nb * R * Cc
    buf = sentinel(n + 8, torch.float16)
    ops.transpose_batched(x.to(dev), out=buf[:n].view(nb, Cc, R))
    ref = sentinel(n + 8, torch.float16).cpu()
    ref[:n] = x.transpose(1, 2).reshape(-1)
    assert_bits(buf, ref, 'transpose')


# ------------------------------------------------------------------------------------------------ frames_to_u8 / _f32
def frames_tok(ld, extra_pixels=0):
    """[65536 + extra, ld] fp16 with every fp16 pattern in each of the RGB columns (rotated per column); other columns
    random."""
    p = torch.arange(65536, dtype=torch.int32)
    cols = [p, (p + 21845) % 65536, 65535 - p]
    tok = halves((65536 + extra_pixels, ld), gen(11))
    for c in range(3):
        tok[:65536, c] = cols[c].to(torch.int16).view(torch.float16)
    return tok


def u8_ref(v):
    """numpy's tensor2vid arithmetic in fp32: (v * 0.5 + 0.5).clip(0, 1) * 255, astype(uint8) truncating."""
    return ((v.float() * 0.5 + 0.5).clamp(0, 1) * 255).to(torch.uint8)


@pytest.mark.parametrize('ld,extra', [(8, 0), (5, 0), (16, 200000)])
def test_frames_to_u8(ops, ld, extra):
    """Every fp16 value of the RGB columns (ld > 3: the other columns are not read).  NaN gives 0: the kernel's
    fmaxf(NaN, 0) picks 0, where numpy's cast of NaN is undefined."""
    tok = frames_tok(ld, extra)
    px = tok.shape[0]
    assert px * 3 > WRAP or extra == 0
    v = tok[:, :3]
    nan = torch.isnan(v)
    ref = u8_ref(v)
    ref[nan] = 0
    for fill in (0x5A, 0xA5):                 # two fills: an element the kernel skips cannot match the reference twice
        buf = sentinel(px * 3 + 16, torch.uint8, fill)
        ops.frames_to_u8(tok.to(dev), out=buf[:px * 3].view(px, 3))
        out = buf.cpu()
        assert (out[px * 3:] == fill).all(), 'write past the end'
        assert_bits(out[:px * 3].view(px, 3), ref, 'frames_to_u8')
    assert (ref[~nan][v[~nan] >= 1] == 255).all() and (ref[~nan][v[~nan] <= -1] == 0).all()


@pytest.mark.parametrize('n,H,W,ld', [(1, 256, 256, 8), (4, 3, 5, 6), (4, 320, 512, 16)])
def test_frames_to_f32(ops, n, H, W, ld):
    """tok [n*H*W, ld] -> [n, 3, H, W] fp32, exact; a NaN stays NaN."""
    px = n * H * W
    tok = frames_tok(ld, px - 65536) if px >= 65536 else halves((px, ld), gen(12))
    assert px * 3 > WRAP or px <= 65536
    buf = sentinel(px * 3 + 8, torch.float32)
    ops.frames_to_f32(tok.to(dev), n, H, W, out=buf[:px * 3].view(n, 3, H, W))
    out = buf.cpu()
    assert (bits(out[px * 3:]) == _SENTINEL[torch.float32]).all(), 'write past the end'
    ref = tok[:, :3].float().view(n, H, W, 3).permute(0, 3, 1, 2).reshape(-1)
    nan = torch.isnan(ref)
    assert torch.equal(torch.isnan(out[:px * 3]), nan)
    assert torch.equal(bits(out[:px * 3])[~nan], bits(ref)[~nan])


# ------------------------------------------------------------------------------------------------ convert_to_f16
def f32_sweep():
    """fp32 bit patterns where a conversion to fp16 goes wrong: a strided sweep of all 2^32 patterns, dense windows at the
    fp16 underflow boundary (2^-25), the subnormal / normal boundary (2^-14), the overflow threshold (65520 = 65504 + half
    an ulp), and every tie between two adjacent finite fp16 values with its fp32 neighbours; both signs, +-inf, NaNs."""
    parts = [torch.arange(0, 2 ** 32, 4099, dtype=torch.int64)]
    for centre in (2.0 ** -25, 2.0 ** -24, 2.0 ** -14, 65504.0, 65520.0):
        c = int(np.array(centre, dtype=np.float32).view(np.int32))
        parts.append(torch.arange(c - 40000, c + 40000, dtype=torch.int64))
    h = torch.arange(0, 0x7BFF, dtype=torch.int32).to(torch.int16).view(torch.float16).double()
        # every fp16 value below 65504, as fp64
    nxt = torch.arange(1, 0x7C00, dtype=torch.int32).to(torch.int16).view(torch.float16).double()
    mid = ((h + nxt) / 2).float()                                     # exact in fp32 (12 significant bits)
    mb = mid.view(torch.int32).to(torch.int64)
    parts += [mb - 1, mb, mb + 1]
    pos = torch.cat(parts) & 0x7FFFFFFF
    allb = torch.cat([pos, pos | 0x80000000, torch.tensor([0x7F800000, 0xFF800000, 0x7FC00000, 0x7F800001, 0xFFC01234])])
    return (allb & 0xFFFFFFFF).to(torch.int64).numpy().astype(np.uint32).view(np.float32)


def test_convert_to_f16_fp32_patterns(ops):
    x = torch.from_numpy(f32_sweep().copy())
    n = x.numel()
    assert n > WRAP
    buf = sentinel(n + 8, torch.float16)
    ops.convert_to_f16(x.to(dev), out=buf[:n])
    out = buf.cpu()
    assert (bits(out[n:]) == _SENTINEL[torch.float16]).all()
    ref = x.half()
    nan = torch.isnan(ref)
    assert torch.equal(torch.isnan(out[:n]), nan)
    assert_bits(out[:n][~nan], ref[~nan], 'convert fp32 -> fp16')
    assert out[:n][x == 65520.0].isinf().all() and (out[:n][(x > 65504) & (x < 65520)] == 65504).all()


def test_convert_to_f16_copies_fp16(ops):
    x = all_halves()
    assert_bits(ops.convert_to_f16(x.to(dev)), x, 'convert fp16 copy')


# ------------------------------------------------------------------------------------------------ softmax_rows
def fp16_ulp(v):
    """Spacing of fp16 at |v| (fp64 tensor): 2^-24 below the normal range, else 2^(floor(log2|v|) - 10)."""
    e = torch.floor(torch.log2(v.abs().clamp_min(2.0 ** -14)))
    return torch.pow(2.0, e - 10)


def softmax_logits(kind, rows, cols, g):
    if kind == 'randn':
        return torch.randn(rows, cols, generator=g) * 4
    if kind == 'equal':
        return torch.full((rows, cols), 1.5) + torch.arange(rows)[:, None] * 0.25
    if kind == 'dominant':
        x = torch.randn(rows, cols, generator=g)
        x[torch.arange(rows), torch.randint(0, cols, (rows,), generator=g)] = 40.0
        return x
    return torch.rand(rows, cols, generator=g) * 60 - 50          # 'spread': exp arguments down to -60


@pytest.mark.parametrize('kind', ['randn', 'equal', 'dominant', 'spread'])
@pytest.mark.parametrize('rows,cols,scale', [(13, 1, 1.0), (9, 7, 0.125), (5, 31, 1.0), (8, 32, 0.7), (3, 33, 1.0),
                                             (1003, 1000, 512 ** -0.5), (45, 4096, 512 ** -0.5)])
def test_softmax_rows(ops, rows, cols, scale, kind):
    """Gate: 1 fp16 ulp of fp64 softmax(fp16(x * scale)).  The kernel rounds the scaled logits to fp16 (as the reference's
    fp16 `w_ * c^-0.5`), exponentiates with __expf in fp32 and rounds the output once."""
    scale = float(np.float32(scale))
    x = (softmax_logits(kind, rows, cols, gen(13)) / scale).half()
    buf = sentinel((rows + 1) * cols, torch.float16)
    ops.softmax_rows(x.to(dev), scale, out=buf[:rows * cols].view(rows, cols))
    out = buf.cpu()
    assert (bits(out[rows * cols:]) == _SENTINEL[torch.float16]).all()
    y = out[:rows * cols].view(rows, cols)
    ref = torch.softmax((x.float() * scale).half().double(), dim=1)
    err = ((y.double() - ref).abs() / fp16_ulp(ref)).max().item()
    print(f'softmax {kind} rows {rows} cols {cols}: max error {err:.3f} fp16 ulp')
    assert err <= 1.0
    if kind == 'equal' or cols == 1:
        want = torch.tensor(float(np.float32(1) / np.float32(cols))).half()
        assert (bits(y) == bits(want)).all(), 'equal logits give fp16(fp32(1 / cols))'


# ------------------------------------------------------------------------------------------------ lincomb
def fp32_ulp(v):
    a = np.abs(v).astype(np.float32)
    return np.spacing(np.maximum(a, np.float32(2.0 ** -126))).astype(np.float64)


@pytest.mark.parametrize('n_src', range(1, 9))
@pytest.mark.parametrize('n', [1000, 600001])
def test_lincomb(lib, n_src, n):
    """out = fmaf chain over the sources in order; gate: 1 fp32 ulp of the fp64 restatement (each step exact in fp64,
    rounded to fp32).  The sources nearly cancel, so a different summation order is visible."""
    g = gen(14 + n_src)
    base = torch.randn(n, generator=g)
    srcs = [base * (1 + 1e-3 * i) + 1e-3 * torch.randn(n, generator=g) for i in range(n_src)]
    coefs = np.array([(-1) ** i * (2.0 + 0.37 * i) for i in range(n_src)], dtype=np.float32)
    out = sentinel(n + 8, torch.float32)
    dsrc = [s.to(dev) for s in srcs]
    ptrs = (C.c_void_p * n_src)(*[s.data_ptr() for s in dsrc])
    cf = (C.c_float * n_src)(*coefs.tolist())
    l = lib.lib()
    lib.check(l.t2v_lincomb(lib.ptr(out), ptrs, cf, n_src, n, lib.stream_ptr()), 'lincomb')
    o = out.cpu()
    assert (bits(o[n:]) == _SENTINEL[torch.float32]).all()
    acc = np.zeros(n, dtype=np.float32)
    for s, c in zip(srcs, coefs):
        acc = (np.float64(c) * s.numpy().astype(np.float64) + acc.astype(np.float64)).astype(np.float32)
    err = (np.abs(o[:n].numpy().astype(np.float64) - acc) / fp32_ulp(acc)).max()
    print(f'lincomb n_src {n_src} n {n}: max error {err:.3f} fp32 ulp')
    assert err <= 1.0


# ------------------------------------------------------------------------------------------------ latent_blend
@pytest.mark.parametrize('with_mask', [False, True])
@pytest.mark.parametrize('BC,Fr,hw,img_frames', [(3, 5, 7, 1), (3, 5, 7, 5), (2, 1, 33, 1), (8, 24, 4096, 1), (8, 24, 4096, 24)])
def test_latent_blend(lib, BC, Fr, hw, img_frames, with_mask):
    """img * (1 - w[f]) + noise * w[f] in numpy float64, bit for bit."""
    rng = np.random.default_rng(15)
    img = rng.standard_normal((BC, img_frames, hw)).astype(np.float32)
    noise = rng.standard_normal((BC, Fr, hw))
    w = rng.random(Fr)
    w[0] = 0.0
    n = BC * Fr * hw
    out = sentinel(n + 4, torch.float64)
    mask = sentinel(n + 4, torch.float64) if with_mask else None
    di, dn, dw = (torch.from_numpy(a).to(dev) for a in (img, noise, w))
    l = lib.lib()
    lib.check(l.t2v_latent_blend(lib.ptr(di), img_frames, lib.ptr(dn), lib.ptr(dw), lib.ptr(out), lib.ptr(mask), BC, Fr, hw,
                                 lib.stream_ptr()), 'latent_blend')
    wb = w[None, :, None]
    ref = img.astype(np.float64) * (1 - wb) + noise * wb
    o = out.cpu()
    assert_bits(o[:n], torch.from_numpy(ref.reshape(-1)), 'latent_blend')
    assert (bits(o[n:]) == _SENTINEL[torch.float64]).all()
    if with_mask:
        m = mask.cpu()
        assert_bits(m[:n], torch.from_numpy(np.broadcast_to(wb, (BC, Fr, hw)).reshape(-1).copy()), 'latent_blend mask')
        assert (bits(m[n:]) == _SENTINEL[torch.float64]).all()


# ------------------------------------------------------------------------------------------------ ddim_step / cfg_x0
def cfg_ref(c, u, g, fp16):
    """The kernel's cfg_combine on fp32 tensors: u + g (c - u), op by op in fp16 when fp16 (whatever eps' dtype)."""
    if fp16:
        d = (c - u).half().float()
        s = (g * d).half().float()
        return (u + s).half().float()
    return u + g * (c - u)


def ddim_ref(x, ec, eu, gch, g, mode, a, noise, fp16):
    """tests/test_samplers_host_cpu.py::_TorchKernels.t2v_ddim_step in fp32 torch ops (no contraction)."""
    a0, a1, a2, a3, a4 = a
    c = ec.float()
    e = c.clone()
    if eu is not None:
        e[:, :gch] = cfg_ref(c, eu.float(), g, fp16)[:, :gch]
    nz = a4 * noise if (noise is not None and a4 != 0.0) else 0.0
    if mode == 0:
        ax = a0 * x
        x0 = ax - a1 * e
        eps = (ax - x0) / a1
        return a2 * x0 + a3 * eps + nz
    x0 = (x - a0 * e) / a1
    return a2 * x0 + a3 * e + nz


def f32(*v):
    return tuple(float(np.float32(t)) for t in v)


DDIM_COEFS = {0: f32(1.0270127, 0.2304173, 0.9738153, 0.2273596, 0.0),
              1: f32(0.2304173, 0.9738153, 0.9815229, 0.1913546, 0.0)}


def sampler_inputs(shape, eps_dtype, seed):
    g = gen(seed)
    x = torch.randn(shape, generator=g)
    ec = (torch.randn(shape, generator=g) * 0.8).to(eps_dtype)
    eu = (torch.randn(shape, generator=g) * 0.8).to(eps_dtype)
    noise = torch.randn(shape, generator=g)
    return x, ec, eu, noise


@pytest.mark.parametrize('noise_kind', ['noise', 'none'])
@pytest.mark.parametrize('cfg_fp16', [0, 1])
@pytest.mark.parametrize('gch', [0, 2, 'C'])
@pytest.mark.parametrize('eps_dtype', [torch.float16, torch.float32])
@pytest.mark.parametrize('mode', [0, 1])
@pytest.mark.parametrize('shape', [(3, 4, 3, 7, 9), (2, 4, 25, 48, 61)], ids=['small', 'wrap'])
def test_ddim_step(lib, shape, mode, eps_dtype, gch, cfg_fp16, noise_kind):
    """t2v_ddim_step bit for bit: mode 0 (DDIM_Gaussian) and 1 (ldm DDIM), eps fp16 / fp32, guided channels none / some / all,
    fp16 or fp32 CFG, noise with a4 != 0 or a4 = 0 without noise; n is not a multiple of 256 and B > 1."""
    Cc = shape[1]
    gch = Cc if gch == 'C' else gch
    x, ec, eu, noise = sampler_inputs(shape, eps_dtype, 16)
    a = DDIM_COEFS[mode]
    if noise_kind == 'noise':
        a = a[:4] + f32(0.0473)
    else:
        noise = None
    g = 17.0 if mode == 0 else 7.5
    n = x.numel()
    assert n % 256 and (n > WRAP or n < 4096)
    out = sentinel(n + 4, torch.float32)
    d = [t.to(dev) if t is not None else None for t in (x, ec, eu, noise)]
    l = lib.lib()
    rc = l.t2v_ddim_step(lib.ptr(d[0]), lib.ptr(d[1]), lib.ptr(d[2]), int(eps_dtype == torch.float32), lib.ptr(out), n,
                         n // (shape[0] * Cc), Cc, gch, g, mode, *a, lib.ptr(d[3]), cfg_fp16, lib.stream_ptr())
    lib.check(rc, 'ddim_step')
    o = out.cpu()
    assert (bits(o[n:]) == _SENTINEL[torch.float32]).all()
    assert_bits(o[:n].view(shape), ddim_ref(x, ec, eu, gch, g, mode, a, noise, cfg_fp16), 'ddim_step')


@pytest.mark.parametrize('uncond', [True, False])
@pytest.mark.parametrize('cfg_fp16', [0, 1])
@pytest.mark.parametrize('eps_dtype', [torch.float16, torch.float32])
@pytest.mark.parametrize('shape', [(3, 4, 3, 7, 9), (2, 4, 25, 48, 61)], ids=['small', 'wrap'])
def test_cfg_x0(lib, shape, eps_dtype, cfg_fp16, uncond):
    """t2v_cfg_x0 bit for bit: x0 = (x - sigma * cfg(eps)) / alpha in fp32."""
    x, ec, eu, _ = sampler_inputs(shape, eps_dtype, 17)
    eu = eu if uncond else None
    alpha, sigma = f32(0.8123457, 0.5832164)
    g = 9.0
    n = x.numel()
    out = sentinel(n + 4, torch.float32)
    d = [t.to(dev) if t is not None else None for t in (x, ec, eu)]
    l = lib.lib()
    rc = l.t2v_cfg_x0(lib.ptr(d[0]), lib.ptr(d[1]), lib.ptr(d[2]), int(eps_dtype == torch.float32), lib.ptr(out), n, g, alpha,
                      sigma, cfg_fp16, lib.stream_ptr())
    lib.check(rc, 'cfg_x0')
    e = cfg_ref(ec.float(), eu.float(), g, cfg_fp16) if uncond else ec.float()
    o = out.cpu()
    assert (bits(o[n:]) == _SENTINEL[torch.float32]).all()
    assert_bits(o[:n].view(shape), (x - sigma * e) / alpha, 'cfg_x0')


# ------------------------------------------------------------------------------------------------ argument checks
def test_entry_points_reject_what_their_launchers_refuse(lib):
    """-1 without launching (the output keeps its sentinel), and t2v_last_error names the entry point."""
    l = lib.lib()
    s = lib.stream_ptr()
    x = torch.zeros(4096, dtype=torch.float16, device=dev)
    P = lib.ptr
    calls = {
        'op_im2col_s2': [lambda o: l.t2v_op_im2col_s2(P(x), P(o), 1, 4, 4, 12, 1, s),
                         lambda o: l.t2v_op_im2col_s2(P(x), P(o), 1, 4, 4, 8, 2, s)],
        'op_avgpool2x2': [lambda o: l.t2v_op_avgpool2x2(P(x), P(o), 1, 4, 4, 12, s)],
        'op_pixel_unshuffle': [lambda o: l.t2v_op_pixel_unshuffle(P(x), 0, P(o), 1, 1, 12, 8, s),
                               lambda o: l.t2v_op_pixel_unshuffle(P(x), 0, P(o), 1, 1, 8, 20, s)],
        'op_relu': [lambda o: l.t2v_op_relu(P(o), 4, 12, s)],
        'op_feature_add': [lambda o: l.t2v_op_feature_add(P(o), 16, P(x), 12, 4, 2, 1, s),
                           lambda o: l.t2v_op_feature_add(P(o), 12, P(x), 8, 4, 2, 1, s),
                           lambda o: l.t2v_op_feature_add(P(o), 16, P(x), 8, 4, 0, 1, s),
                           lambda o: l.t2v_op_feature_add(P(o), 16, P(x), 8, 4, 2, 0, s)],
        'op_concat_cols': [lambda o: l.t2v_op_concat_cols(P(x), 16, 12, P(x), 16, 8, P(o), 32, 4, s),
                           lambda o: l.t2v_op_concat_cols(P(x), 16, 8, P(x), 16, 4, P(o), 32, 4, s),
                           lambda o: l.t2v_op_concat_cols(P(x), 12, 8, P(x), 16, 8, P(o), 32, 4, s),
                           lambda o: l.t2v_op_concat_cols(P(x), 16, 8, P(x), 20, 8, P(o), 32, 4, s),
                           lambda o: l.t2v_op_concat_cols(P(x), 16, 8, P(x), 16, 8, P(o), 36, 4, s)],
    }
    for name, fns in calls.items():
        for i, fn in enumerate(fns):
            o = sentinel(4096, torch.float16)
            assert fn(o) == -1, (name, i)
            assert l.t2v_last_error().decode().startswith(name + ':'), (name, i, l.t2v_last_error())
            torch.cuda.synchronize()
            assert (bits(o) == _SENTINEL[torch.float16]).all(), (name, i)
