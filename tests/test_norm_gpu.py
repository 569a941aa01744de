"""GPU: GroupNorm(+SiLU) in every launch regime and LayerNorm against fp64 references of the same operation on the same
fp16 operands, at the shapes, channel and row geometries, conditionings and views where the kernels can go wrong.

GroupNorm paths (groupnorm_silu in csrc/norm.cu; gn_plan below restates its choice from t2v_num_sms()):
  1 cached   gn_fused_kernel, the CTA's row slice kept in shared memory (one CTA per SM)
  2 lean     gn_fused_kernel, two CTAs per SM, second pass from L2
  3 single   gn_fused_kernel with one CTA per instance: no barrier
  4 two/1    gn_stats_kernel + gn_apply_kernel, one chunk per instance (more instances than two CTAs per SM)
  5 two/n    gn_stats_kernel + gn_apply_kernel, many chunks per instance: phase 1 (statistics only, the chunking of the
             frame-sharded plans) and phase 2 (apply only, caller statistics)
Which kernels ran is read from torch.profiler, in a process of its own.

References: two-pass mean and population variance in fp64 per (instance, group), then the affine and SiLU in fp64.
u16 = 2^-11, u32 = 2^-24.  Every gate is GATE_K = 2 times the bound below; `pytest -s` prints the worst |err| / gate.

Statistics (phase 1).  The kernels sum d = x - K in fp32, K the group's pivot (its first channel in the instance's first
row): per thread a chain of n_t = ceil(rows per CTA / RL) terms per channel (RL = 320 / (C / 8) rows per pass), then RL
row lanes, then cpg = C / 32 channels, one rounding of d itself; the chunk fold and the moments are in double.  With
n = n_t + RL + cpg + 2, N elements per group, A1 = sum |d|, A2 = sum d^2 (fp64, from the data):
  |dS| <= n u32 A1,  |dQ| <= (n + 1) u32 A2
  |dmean| <= |dS| / N + u32 |mean|                       (the fp32 mean)
  |drstd| / rstd <= (|dQ| / N + 2 |mean - K| |dS| / N) / (2 (var + eps)) + 2 u32
A1 / N and A2 / N are of the size of std and var + (mean - K)^2, so in units of std and as a relative error the gate does
not grow with mean / std (a raw sum of x^2 would lose var to cancellation once |mean| / std ~ 100).
Apply (phase 2, exact statistics rounded to fp32, the reference using those fp32 values).  d = x - mean, a = rstd gamma,
u = fma(d, a, beta): one rounding each, |du| <= u32 (2 |d a| + |u|).  SiLU u * rcp.approx(1 + ex2.approx(-u log2 e)): slope
at most 1.1, evaluation error <= u32 (|u| + 8) |silu(u)|.  Output rounding u16 |ref| + 2^-25 (2^-25 absolute below 2^-14).
Fused / phase 0.  The apply bound at the exact statistics plus the statistics error carried through:
  slope (|gamma| rstd |dmean| + |u - beta| |drstd| / rstd).
LayerNorm (layernorm_kernel: one warp per row, fp32 sums over 8 ceil(C / 256) values per lane and a 5-level shuffle tree,
two-pass variance, rsqrtf, y = (x - mean) rstd gamma + beta): with n = 8 ceil(C / 256) + 8,
  |dmean| <= n u32 sum |x| / C + u32 |mean|,  |dvar| <= n u32 sum (x - mean)^2 / C + dmean^2 + 2 u32 (var + eps),
  |drstd| / rstd <= |dvar| / (2 (var + eps)) + 2^-22 (rsqrtf),
  |dy| <= 3 u32 |d rstd gamma| + u32 |y| + |gamma| rstd |dmean| + |d rstd gamma| |drstd| / rstd + u16 |ref| + 2^-25.

Views put NaN in the pad columns of x and around the output view (pad columns, rows past it) inside the allocation; a
mis-bounded read shows up as a non-finite output, a mis-bounded write as a changed pad."""
import json
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
dev = 'cuda'
U16, U32 = 2.0 ** -11, 2.0 ** -24
GATE_K = 2.0
NAN16 = 0x7E00


@pytest.fixture(scope='module')
def ops():
    from t2v_b200 import ops as o
    return o


@pytest.fixture(scope='module')
def sms():
    from t2v_b200 import _lib
    return _lib.lib().t2v_num_sms()


def gen(seed):
    return torch.Generator(device=dev).manual_seed(seed)


def cdiv(a, b):
    return -(-a // b)


# ------------------------------------------------------------------------------------------------ GroupNorm plan + refs
def gn_plan(R, n, C, sms, phase=0):
    """groupnorm_silu's launch choice: ('cached' | 'lean' | 'single', cpi, rows per CTA) or ('two', chunks, rows per chunk)."""
    RL = 320 // (C // 8)
    if phase == 0:
        fixed = (2 * RL * C + 2 * C) * 4 + 8 * 32 * 2 * 8 + 32 * 8
        cap = 200 * 1024 - fixed
        cpi = cache = 0
        if n <= sms and cdiv(R * C * 2, cap) <= sms // n:
            cpi, cache = sms // n, 1
        if not cache and n <= 2 * sms:
            cpi = 2 * sms // n
        if cpi > 0:
            cpi = max(1, min(cpi, cdiv(R, RL)))
            rpc = cdiv(R, cpi)
            cpi = cdiv(R, rpc)
            if cache and fixed + rpc * C * 2 > 226 * 1024:
                cache = 0
            return ('single' if cpi == 1 else 'cached' if cache else 'lean'), cpi, rpc
    chunks = max(1, cdiv(2 * sms, n))
    rpc = max(8, cdiv(R, chunks))
    rpc = cdiv(rpc, 8) * 8
    return 'two', cdiv(R, rpc), rpc


def gn_stats64(x, n, R, C, eps, rpc):
    """fp64 (mean, rstd) [n, 32] and the statistics bound (dmean, drel) of the kernels for CTAs of rpc rows."""
    cpg = C // 32
    RL = 320 // (C // 8)
    xd = x.double().view(n, R, 32, cpg)
    mean = xd.mean(dim=(1, 3))
    var = ((xd - mean[:, None, :, None]) ** 2).mean(dim=(1, 3))
    rstd = 1.0 / torch.sqrt(var + eps)
    K = xd[:, 0, :, 0]
    d = xd - K[:, None, :, None]
    N = R * cpg
    A1 = d.abs().sum(dim=(1, 3))
    A2 = (d * d).sum(dim=(1, 3))
    nc = cdiv(rpc, RL) + RL + cpg + 2
    dS = nc * U32 * A1
    dQ = (nc + 1) * U32 * A2
    dmean = dS / N + U32 * mean.abs()
    drel = (dQ / N + 2 * (mean - K).abs() * dS / N) / (2 * (var + eps)) + 2 * U32
    return mean, rstd, dmean, drel


def silu64(u):
    return u / (1 + torch.exp(-u))


def gn_apply64(x, n, R, C, mean, rstd, gamma, beta, silu):
    """fp64 output [n*R, C], the pre-activation u, and the apply bound for per-group (mean, rstd) [n, 32]."""
    cpg = C // 32
    xd = x.double().view(n, R, C)
    m = mean.repeat_interleave(cpg, dim=1)[:, None, :]
    r = rstd.repeat_interleave(cpg, dim=1)[:, None, :]
    g, b = gamma.double()[None, None, :], beta.double()[None, None, :]
    da = (xd - m) * r * g
    u = da + b
    bound = U32 * (2 * da.abs() + u.abs())
    out = u
    if silu:
        out = silu64(u)
        bound = 1.1 * bound + U32 * (u.abs() + 8) * out.abs()
    return out.view(-1, C), u.view(-1, C), bound.view(-1, C)


def out_round(ref):
    return U16 * ref.abs() + 2.0 ** -25


def check(name, out, ref, bound):
    """|out - ref| <= GATE_K bound everywhere, out finite; prints the worst ratio."""
    out = out.double()
    assert torch.isfinite(out).all(), f'{name}: non-finite output'
    ratio = ((out - ref).abs() / (GATE_K * bound)).max().item()
    print(f'\n[{name}] worst |err| / gate = {ratio:.3f}', end='')
    assert ratio <= 1.0, f'{name}: worst |err| / gate = {ratio:.3f}'
    return ratio


def check_stats(name, st, mean, rstd, dmean, drel):
    """phase-1 statistics [n, 32, 2] vs fp64: mean within the dmean gate, rstd within the relative gate."""
    st = st.double()
    rm = ((st[..., 0] - mean).abs() / (GATE_K * dmean + 1e-300)).max().item()
    rr = (((st[..., 1] - rstd).abs() / rstd) / (GATE_K * drel)).max().item()
    print(f'\n[{name} stats] worst |dmean| / gate = {rm:.3f}, |drstd/rstd| / gate = {rr:.3f}', end='')
    assert rm <= 1.0 and rr <= 1.0, f'{name}: statistics |err| / gate = {rm:.3f} (mean), {rr:.3f} (rstd)'


def launched(fn):
    """GroupNorm kernels that `fn` launched, from torch.profiler's CUDA activity."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return {k for e in prof.events() for k in ('gn_fused_kernel', 'gn_stats_kernel', 'gn_apply_kernel') if k in e.name}


def regime_kernels():
    """{regime: (kernels of phase 0, kernels of phase 1)} for every regime of regime_shapes, printed as JSON."""
    from t2v_b200 import _lib, ops
    res = {}
    for i, (name, R, n, C, _) in enumerate(regime_shapes(_lib.lib().t2v_num_sms())):
        x = gn_input(n, R, C, seed=i)
        gamma, beta = affine(C, seed=100 + i)
        res[name] = [sorted(launched(lambda: ops.groupnorm(x, gamma, beta, R, 1e-5, True, phase=p))) for p in (0, 1)]
    print(json.dumps(res))


@pytest.fixture(scope='module')
def routes():
    """regime_kernels() in a process of its own: a profiler session in a process that has already run other GPU test
    modules has come back without the library's kernels, so the routing is read where no earlier test has run."""
    here = os.path.dirname(os.path.abspath(__file__))
    path = os.pathsep.join([here] + [p for p in sys.path if p])
    r = subprocess.run([sys.executable, '-s', '-c', 'import test_norm_gpu as t; t.regime_kernels()'], capture_output=True,
                       text=True, timeout=300, env=dict(os.environ, PYTHONPATH=path))
    assert r.returncode == 0, r.stderr[-3000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


def affine(C, seed):
    g = gen(seed)
    gamma = (1 + 0.5 * torch.randn(C, device=dev, generator=g)).half()
    beta = (0.5 * torch.randn(C, device=dev, generator=g)).half()
    return gamma, beta


def gn_input(n, R, C, seed, ratio=None, std=1.0):
    """[n*R, C] fp16.  Default: per-channel offsets and scales (channel means differ within a group).  ratio: every group
    of every instance has |mean| / std = ratio (random sign), std `std` per element."""
    g = gen(seed)
    z = torch.randn(n, R, C, device=dev, generator=g)
    if ratio is None:
        loc = torch.randn(n, 1, C, device=dev, generator=g) * 2
        sc = torch.rand(n, 1, C, device=dev, generator=g) * 2 + 0.3
        return (z * sc + loc).half().view(-1, C)
    sign = torch.randint(0, 2, (n, 1, 32, 1), device=dev, generator=g) * 2 - 1
    x = z.view(n, R, 32, C // 32) * std + sign * ratio * std
    return x.half().view(-1, C)


def run_gn(ops, name, x, n, R, C, gamma, beta, eps, silu, sms, *, out=None, expect=None):
    """phase 0 vs the fused gate, phase 1 vs the statistics gate, phase 2 fed exact statistics vs the apply gate."""
    kind, _, rpc = gn_plan(R, n, C, sms)
    if expect is not None:
        assert kind == expect, f'{name}: planned {kind}, wanted {expect}'
    mean, rstd, dmean, drel = gn_stats64(x, n, R, C, eps, rpc)
    ref, u, ab = gn_apply64(x, n, R, C, mean, rstd, gamma, beta, silu)
    cpg = C // 32
    slope = 1.1 if silu else 1.0
    carried = slope * (gamma.double().abs()[None, :] * (rstd * dmean).repeat_interleave(cpg, 1).repeat_interleave(R, 0)
                       + (u - beta.double()[None, :]).abs() * drel.repeat_interleave(cpg, 1).repeat_interleave(R, 0))
    y = ops.groupnorm(x, gamma, beta, R, eps, silu, out=out)
    check(f'{name} fused', y, ref, ab + carried + out_round(ref))
    # phase 1: the two-kernel chunking
    _, nch, rpc1 = gn_plan(R, n, C, sms, phase=1)
    st = ops.groupnorm(x, gamma, beta, R, eps, silu, phase=1)
    m1, r1, dm1, dr1 = gn_stats64(x, n, R, C, eps, rpc1)
    check_stats(f'{name} ({nch} chunks)', st, m1, r1, dm1, dr1)
    # phase 2: exact statistics, rounded to fp32
    ex = torch.stack([mean, rstd], dim=-1).float().contiguous()
    ref2, _, ab2 = gn_apply64(x, n, R, C, ex[..., 0].double(), ex[..., 1].double(), gamma, beta, silu)
    y2 = ops.groupnorm(x, gamma, beta, R, eps, silu, phase=2, stats=ex, out=out)
    check(f'{name} apply', y2, ref2, ab2 + out_round(ref2))
    return kind


# ------------------------------------------------------------------------------------------------ 1. every path
def regime_shapes(sms):
    """(name, R, n, C, expected kind) landing in each regime for this GPU's SM count."""
    fixed = (2 * 8 * 320 + 2 * 320) * 4 + 8 * 32 * 2 * 8 + 32 * 8
    lean_rows = cdiv((sms // 4 + 1) * (200 * 1024 - fixed), 640) + 13
    return [
        ('cached', 4096, 2, 320, 'cached'),
        ('lean', lean_rows, 4, 320, 'lean'),
        ('lean_many_inst', 700, sms // 2 + 3, 128, 'lean'),
        ('single_cta', 200, 2 * sms - 3, 128, 'single'),
        ('single_cta_short_inst', 2, 3, 1280, 'single'),          # rows_per_inst <= RL = 2: max_useful = 1
        ('capped_cpi', 50, 3, 640, 'cached'),                      # max_useful = 13 CTAs, not sms // 3
        ('two_one_chunk', 300, 2 * sms + 7, 64, 'two'),
        ('rows_per_inst_1', 1, 2 * sms + 40, 320, 'two'),
    ]


@pytest.mark.parametrize('idx', range(8))
def test_groupnorm_paths(ops, sms, routes, idx):
    name, R, n, C, kind = regime_shapes(sms)[idx]
    x = gn_input(n, R, C, seed=idx)
    gamma, beta = affine(C, seed=100 + idx)
    silu = idx % 2 == 0
    run_gn(ops, name, x, n, R, C, gamma, beta, 1e-5, silu, sms, expect=kind)
    ran, ran1 = routes[name]
    assert ran == (['gn_fused_kernel'] if kind != 'two' else ['gn_apply_kernel', 'gn_stats_kernel']), ran
    assert ran1 == ['gn_stats_kernel'], ran1
    if kind == 'cached':
        _, nch, _ = gn_plan(R, n, C, sms, phase=1)
        assert nch > 1                                             # path 5: the chunk fold over many CTAs


# ------------------------------------------------------------------------------------------------ 2. channel geometry
@pytest.mark.parametrize('C', [32, 64, 96, 160, 320, 640, 960, 1280, 1920, 2048, 2560])
def test_groupnorm_channel_geometry(ops, sms, C):
    """C = 32: one channel per group (RL = 80); 96 / 160 / 320: groups straddle 8-channel vectors, 96 leaves 8 idle threads;
    1920 / 2048: 64 idle threads; 2560: every thread.  333 rows per instance: not a multiple of RL nor of 4 RL."""
    n, R = 3, 333
    x = gn_input(n, R, C, seed=C)
    gamma, beta = affine(C, seed=C + 1)
    run_gn(ops, f'C{C}', x, n, R, C, gamma, beta, 1e-6, C % 64 == 0, sms)


# ------------------------------------------------------------------------------------------------ 3. conditioning
COND_SHAPES = {'vae': (4096, 2, 128), 'unet5d': (16384, 2, 320)}


@pytest.mark.parametrize('ratio', [0, 1, 10, 100, 300])
@pytest.mark.parametrize('shape', ['vae', 'unet5d'])
def test_groupnorm_offset_conditioning(ops, sms, shape, ratio):
    """Groups with |mean| / std = ratio: the statistics must keep their accuracy relative to std."""
    R, n, C = COND_SHAPES[shape]
    x = gn_input(n, R, C, seed=ratio + 7, ratio=ratio, std=0.05 if ratio >= 100 else 1.0)
    gamma, beta = affine(C, seed=3)
    run_gn(ops, f'{shape} m/s={ratio}', x, n, R, C, gamma, beta, 1e-6, True, sms)


def special_input(case, n, R, C, seed):
    g = gen(seed)
    if case == 'mixed_channels':             # channel means spread by 50 std within each group, around a common offset
        loc = torch.randn(1, 1, C, device=dev, generator=g) * 50 + 200
        return (torch.randn(n, R, C, device=dev, generator=g) + loc).half().view(-1, C)
    if case == 'near_constant':              # std 1e-3 around means of 1 to 40 (fp16 quantises most of it away)
        m = torch.rand(n, 1, 32, 1, device=dev, generator=g) * 39 + 1
        return (m + 1e-3 * torch.randn(n, R, 32, C // 32, device=dev, generator=g)).half().view(-1, C)
    if case == 'constant':                   # every group exactly constant
        m = (torch.rand(n, 1, 32, 1, device=dev, generator=g) * 80 - 40).half().float()
        return m.expand(n, R, 32, C // 32).half().reshape(-1, C)
    if case == 'large':                      # |x| up to 3e4
        m = (torch.rand(n, 1, 32, 1, device=dev, generator=g) * 2 - 1) * 2.5e4
        return (m + 2000 * torch.randn(n, R, 32, C // 32, device=dev, generator=g)).clamp(-3e4, 3e4).half().view(-1, C)
    raise ValueError(case)


@pytest.mark.parametrize('case', ['mixed_channels', 'near_constant', 'constant', 'large'])
@pytest.mark.parametrize('shape', ['vae', 'unet5d'])
def test_groupnorm_special_conditioning(ops, sms, shape, case):
    R, n, C = COND_SHAPES[shape]
    x = special_input(case, n, R, C, seed=11)
    gamma, beta = affine(C, seed=5)
    for silu in (False, True):
        run_gn(ops, f'{shape} {case} silu={silu}', x, n, R, C, gamma, beta, 1e-6, silu, sms)
    if case == 'constant':                   # exactly beta / SiLU(beta), within the output rounding
        for silu in (False, True):
            y = ops.groupnorm(x, gamma, beta, R, 1e-6, silu).double()
            ref = beta.double().expand_as(y)
            ref = silu64(ref) if silu else ref
            tol = out_round(ref) + (U32 * (ref.abs() + 8) * ref.abs() if silu else 0)
            assert ((y - ref).abs() <= tol).all(), ((y - ref).abs() - tol).max().item()


# ------------------------------------------------------------------------------------------------ 4. production shapes
# (rows_per_inst, instances, C, eps, silu)  source
PRODUCTION = [
    # ModelScope, 24 frames at 256^2 (latent 32 x 32), CFG batch 2 (bench.py)
    (1024, 48, 320, 1e-5, True),     # unet.cu:560/563 resblock in_layers.0 / out_layers.0, level 0, per frame
    (256, 48, 640, 1e-5, True),      # unet.cu:560 level 1
    (64, 48, 1280, 1e-5, True),      # unet.cu:560 level 2
    (16, 48, 1280, 1e-5, True),      # unet.cu:560 level 3
    (24576, 2, 320, 1e-5, True),     # unet.cu:590 temporal_conv GroupNorms, 5-D, level 0
    (6144, 2, 640, 1e-5, True),      # unet.cu:590 level 1
    (1024, 48, 320, 1e-6, False),    # unet.cu:533 SpatialTransformer norm
    (24576, 2, 320, 1e-6, False),    # unet.cu:533 TemporalTransformer norm (5-D)
    (1024, 48, 320, 1e-5, True),     # unet.cu:960 out.0
    # VAE decode of the same clip, per frame (vae.cu:135/138 resblocks, vae.cu:157 attention norm, vae.cu:254 norm_out)
    (1024, 2, 512, 1e-6, True),      # mid block at 32 x 32
    (1024, 2, 512, 1e-6, False),     # mid attention norm
    (16384, 2, 512, 1e-6, True),     # up block at 128 x 128
    (65536, 1, 256, 1e-6, True),     # up block at 256 x 256
    (65536, 1, 128, 1e-6, True),     # norm_out at 256 x 256
    # VideoCrafter test configuration (model_channels 64, 8 x 8 latent, 4 frames, CFG batch 2; the adapter runs the same
    # per-frame resblock norms at its widths)
    (64, 8, 64, 1e-5, True),         # unet.cu:560 per frame
    (256, 2, 64, 1e-5, True),        # unet.cu:632/635 5-D resblock norms
    (256, 2, 128, 1e-6, False),      # unet.cu:660 temporal transformer norm
    (16, 8, 128, 1e-5, True),        # level 1 per frame
]


@pytest.mark.parametrize('R,n,C,eps,silu', PRODUCTION)
def test_groupnorm_production_shapes(ops, sms, R, n, C, eps, silu):
    x = gn_input(n, R, C, seed=R + C)
    gamma, beta = affine(C, seed=R)
    run_gn(ops, f'R{R} n{n} C{C}', x, n, R, C, gamma, beta, eps, silu, sms)


# ------------------------------------------------------------------------------------------------ 5. views and traps
def nan_view(rows, C, pad_rows, pad_cols, fill=None):
    buf = torch.full((rows + pad_rows, C + pad_cols), float('nan'), device=dev, dtype=torch.half)
    if fill is not None:
        buf[:rows, :C] = fill
    return buf, buf[:rows, :C]


def pads_untouched(buf, rows, C):
    bits = buf.view(torch.int16)
    return bool((bits[:, C:] == NAN16).all()) and bool((bits[rows:] == NAN16).all())


@pytest.mark.parametrize('idx', [0, 1, 2, 6])
def test_groupnorm_strided_views_with_nan_pads(ops, sms, idx):
    """x a column slice (ldx = C + 24) with NaN pads, y a view (ldy = C + 8) of a NaN buffer with 5 rows past it."""
    name, R, n, C, _ = regime_shapes(sms)[idx]
    data = gn_input(n, R, C, seed=idx + 50)
    xb, x = nan_view(n * R, C, 0, 24, data)
    yb, y = nan_view(n * R, C, 5, 8)
    gamma, beta = affine(C, seed=idx)
    run_gn(ops, f'{name} strided', x, n, R, C, gamma, beta, 1e-5, True, sms, out=y)
    assert pads_untouched(yb, n * R, C)


# ------------------------------------------------------------------------------------------------ 6. workspace reuse
def test_groupnorm_workspace_reuse_and_determinism(ops, sms):
    """Alternate regimes in one process (the chunk counters clean themselves, the barrier's generation word is reused),
    then one shape 20 times: bitwise-equal outputs."""
    shapes = [regime_shapes(sms)[i] for i in (0, 6, 1, 3, 6, 0)]
    firsts = {}
    for k, (name, R, n, C, _) in enumerate(shapes):
        x = gn_input(n, R, C, seed=len(name))
        gamma, beta = affine(C, seed=1)
        y = ops.groupnorm(x, gamma, beta, R, 1e-5, True)
        st = ops.groupnorm(x, gamma, beta, R, 1e-5, True, phase=1)
        if name in firsts:
            assert torch.equal(y, firsts[name][0]) and torch.equal(st, firsts[name][1]), name
        else:
            firsts[name] = (y, st)
            mean, rstd, _, _ = gn_stats64(x, n, R, C, 1e-5, R)
            assert ((st[..., 1].double() - rstd).abs() / rstd).max().item() < 1e-4, name
    name, R, n, C, _ = shapes[2]
    x = gn_input(n, R, C, seed=len(name))
    gamma, beta = affine(C, seed=1)
    first = ops.groupnorm(x, gamma, beta, R, 1e-5, True)
    for _ in range(20):
        assert torch.equal(ops.groupnorm(x, gamma, beta, R, 1e-5, True), first)


# ------------------------------------------------------------------------------------------------ 7. LayerNorm
def ln_ref64(x, gamma, beta, eps):
    xd = x.double()
    C = x.shape[1]
    mean = xd.mean(1, keepdim=True)
    d = xd - mean
    var = (d * d).mean(1, keepdim=True)
    rstd = 1.0 / torch.sqrt(var + eps)
    g, b = gamma.double()[None, :], beta.double()[None, :]
    drs = d * rstd * g
    y = drs + b
    n = 8 * cdiv(C, 256) + 8
    dmean = n * U32 * xd.abs().sum(1, keepdim=True) / C + U32 * mean.abs()
    dvar = n * U32 * (d * d).sum(1, keepdim=True) / C + dmean ** 2 + 2 * U32 * (var + eps)
    drel = dvar / (2 * (var + eps)) + 2.0 ** -22
    bound = 3 * U32 * drs.abs() + U32 * y.abs() + g.abs() * rstd * dmean + drs.abs() * drel + out_round(y)
    return y, bound


def ln_input(rows, C, seed, ratio=None):
    g = gen(seed)
    z = torch.randn(rows, C, device=dev, generator=g)
    if ratio is None:                                     # rows with different means and scales
        return (z * (torch.rand(rows, 1, device=dev, generator=g) * 3 + 0.2)
                + torch.randn(rows, 1, device=dev, generator=g) * 2).half()
    sign = torch.randint(0, 2, (rows, 1), device=dev, generator=g) * 2 - 1
    std = 0.05 if ratio >= 100 else 1.0
    return (z * std + sign * ratio * std).half()


@pytest.mark.parametrize('C', [8, 64, 248, 256, 320, 640, 768, 1024, 1280, 2048])
def test_layernorm_vs_fp64(ops, C):
    """C = 8 / 248: partial lanes; 2048: all 8 vectors per lane.  157 rows: the last block has idle warps.  Also a strided
    view with NaN pads around both operands."""
    rows = 157
    gamma, beta = affine(C, seed=C)
    x = ln_input(rows, C, seed=C)
    ref, bound = ln_ref64(x, gamma, beta, 1e-5)
    check(f'ln C{C}', ops.layernorm(x, gamma, beta), ref, bound)
    xb, xv = nan_view(rows, C, 0, 16, x)
    yb, yv = nan_view(rows, C, 3, 8)
    ops.layernorm(xv, gamma, beta, out=yv)
    check(f'ln C{C} strided', yv, ref, bound)
    assert pads_untouched(yb, rows, C)


@pytest.mark.parametrize('ratio', [0, 1, 10, 100, 'constant'])
@pytest.mark.parametrize('C', [320, 1024])
def test_layernorm_conditioning(ops, C, ratio):
    rows = 203
    gamma, beta = affine(C, seed=9)
    if ratio == 'constant':
        x = ((torch.rand(rows, 1, device=dev, generator=gen(2)) * 80 - 40).half().float().expand(rows, C)).half().contiguous()
    else:
        x = ln_input(rows, C, seed=C + 1, ratio=ratio)
    ref, bound = ln_ref64(x, gamma, beta, 1e-5)
    y = ops.layernorm(x, gamma, beta)
    check(f'ln C{C} m/s={ratio}', y, ref, bound)
    if ratio == 'constant':
        assert torch.equal(y, beta.expand(rows, C))
