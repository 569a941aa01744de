"""GPU: every attention route at op level against fp64 references of the same operation on the same fp16 operands, at the
shapes, tile edges and batch mappings where the kernels can go wrong.

Routes (attention() in csrc/attention.cu picks the first four by head_dim -> attention_tc_eligible -> sq, skv <= 32):
  tc       attention_tc_kernel          wgmma + TMA, 128-query CTAs, 128-key tiles (head 64, sq >= 256, skv >= 128, b_inner 1)
  warp64   attention_kernel<64>         warp MMA, 64 x 64 tiles (everything else with head 64 ...)
  warp32   attention_kernel<32>         ... 32 x 32 tiles when sq, skv <= 32 (ModelScope temporal attention)
  hd       attention_hd_kernel<HD>      head widths 8 / 16 / 32 / 40 / 80 / 160, 64 x 64 tiles
  relpos   attention_relpos_kernel<HD, RT>   VideoCrafter temporal attention with relative-position tables, T <= RT
  clip     clip_attention_kernel        causal CLIP text-tower attention, L <= 128, P kept in fp32

Gate: per element, |out - ref| <= GATE_K (= 2) x bound, with the bound taken from the kernels' stated numerics
(tests/attention_ref.py computes the fp64 terms; u16 = 2^-11, u32 = 2^-24, u32t = 2^-23 for fp32 sums inside the tensor
cores, which may truncate):
  * Scores: fp16 operands, exact fp16 products, fp32 sums over hd terms: |ds_j| <= hd u32t sum_d |q_d k_jd|.  The kernels
    compute p_j = exp2(s_j scale log2e - m scale log2e) (relpos, clip: __expf of scale s_j - m): the argument's roundings add
    about u32t (|scale s_j| + |scale m|), the exp approximation about 2 u32t.  So every p_j carries a relative error
    E <= scale hd u32t max_j sum_d |q_d k_jd| + 2 u32t max_j |scale s_j| + 2 u32t.  A relative error e_j on p_j moves
    o = sum p_j v_j / sum p_j by sum_j p_j e_j (v_j - o), so by at most E (sum_j p_j |v_j| + |o|): the score error scales
    into the output as scale x ds times the spread of V.
  * P.V: the unnormalised P (flash kernels) or the normalised P (relpos) is rounded to fp16 before the MMA: u16 sum_j p_j |v_j|
    for normal fp16 values, and an absolute 2^-25 for each p_j below 2^-14 (the term `tiny`).  The clip kernel keeps P in
    fp32 (no u16 term).  The relpos kernel rounds the clamped end columns (lo / hi sums) to fp16 once more: u16 sum_j p_j
    |Rv_j|.
  * Accumulation: P.V adds one fp32 rounding per 16-key MMA step and two per key tile (rescale): n_acc u32t sum_j p_j |v_j|;
    the row sum l is summed by each thread over skv / 4 terms then shuffled: n_l u32 |o| (flash_counts).  clip: n_acc = L.
  * The final store rounds to fp16: u16 |ref| (2^-25 absolute below 2^-14).
  bound = (u16 + n_l u32) |ref| + 2^-25 + E (pv + |ref|) + (u16 [P rounded] + n_acc u32t) pv + 2^-25 tiny (+ u16 pv_tab)
  with pv = sum_j p_j |v_j| from the fp64 reference probabilities.  With K = 0 every p_j is exactly 1 (E = 0, no P rounding
  on the flash kernels): the uniform tests run with that near-exact gate.
`pytest -s` prints the worst |err| / gate of every case.

Operands are laid out as the model lays them out (fused [tokens, 3C] matrices, cross-attention K/V shared by the frames of a
sample, the ModelScope temporal two-level batch); the pad tests put NaN or dominant trap keys just outside every input view
(8 pad rows per batch, 8 pad columns) and NaN around the output view, inside the allocation, so a mis-bounded read or write
shows up as a failed assertion.  Which kernel ran is read from torch.profiler."""
import math
import re

import pytest
import torch

from attention_ref import attention64, flash_counts, gate, gather

pytestmark = pytest.mark.gpu
dev = 'cuda'
NAN16 = 0x7E00


@pytest.fixture(scope='module')
def ops():
    from t2v_b200 import ops as o
    return o


def gen(seed):
    return torch.Generator(device=dev).manual_seed(seed)


def check(name, out, r, g, extra=''):
    """|out - ref| <= gate everywhere, out finite; prints the worst ratio."""
    out = out.double()
    assert torch.isfinite(out).all(), f'{name}: non-finite output'
    ratio = ((out - r.out).abs() / g).max().item()
    print(f'\n[{name}{extra}] worst |err| / gate = {ratio:.3f}', end='')
    assert ratio <= 1.0, f'{name}{extra}: worst |err| / gate = {ratio:.3f}'
    return ratio


# ------------------------------------------------------------------------------------------------ AttnParams routes
class Attn:
    """One t2v_op_attention / t2v_op_attention_hd call on separately allocated Q, K, V, O:
    Q [batch, sq + pr, ld], K / V [ceil(batch / div), skv + pr, ld], O [batch, sq + po, C + pc] with ld = heads hd + pc.
    pad=True: pr = 8 pad rows per batch and pc = 8 pad columns of NaN, po = 3 NaN pad rows of O; O starts all NaN."""

    def __init__(self, *, hd, batch, heads, sq, skv, div=1, scale=None, pad=False, seed=0, qscale=1.0):
        self.hd, self.batch, self.heads, self.sq, self.skv, self.div = hd, batch, heads, sq, skv, div
        self.scale = hd ** -0.5 if scale is None else scale
        self.kvb = -(-batch // div)
        C = heads * hd
        pr, pc = (8, 8) if pad else (0, 0)
        self.ld = C + pc
        g = gen(seed)
        nan = float('nan')

        def alloc(nb, S, rows_pad, cols, fill_scale):
            t = torch.full((nb, S + rows_pad, cols), nan, device=dev, dtype=torch.half)
            t[:, :S, :C] = (torch.randn(nb, S, C, device=dev, generator=g) * fill_scale).half()
            return t
        self.qb = alloc(batch, sq, pr, self.ld, qscale)
        self.kb = alloc(self.kvb, skv, pr, self.ld, 1.0)
        self.vb = alloc(self.kvb, skv, pr, self.ld, 1.0)
        self.ob = torch.full((batch, sq + (3 if pad else 0), C + pc), nan, device=dev, dtype=torch.half)
        self.q = self.qb[:, :sq, :C].unflatten(-1, (heads, hd))         # [batch, sq, heads, hd] views
        self.k = self.kb[:, :skv, :C].unflatten(-1, (heads, hd))
        self.v = self.vb[:, :skv, :C].unflatten(-1, (heads, hd))

    def run(self, ops, scale=None):
        scale = self.scale if scale is None else scale
        C = self.heads * self.hd
        a = (self.qb, self.kb, self.vb, self.ob, self.qb.stride(0), self.ld, self.kb.stride(0), self.ld, self.kb.stride(0), self.ld,
             self.ob.stride(0), self.ob.stride(1), self.batch, self.heads)
        if self.hd == 64:
            ops.attention(*a, self.sq, self.skv, kv_batch_div=self.div, scale=scale)
        else:
            ops.attention_hd(*a, self.hd, self.sq, self.skv, kv_batch_div=self.div, scale=scale)
        return self.ob[:, :self.sq, :C].unflatten(-1, (self.heads, self.hd))

    def ref(self, scale=None):
        scale = self.scale if scale is None else scale
        kv = torch.arange(self.batch, device=dev) // self.div
        q = gather(self.qb, self.sq, self.heads, self.hd, self.qb.stride(0), self.ld, torch.arange(self.batch))
        k = gather(self.kb, self.skv, self.heads, self.hd, self.kb.stride(0), self.ld, kv)
        v = gather(self.vb, self.skv, self.heads, self.hd, self.vb.stride(0), self.ld, kv)
        return attention64(q, k, v, scale)

    def tile(self):
        if self.hd != 64:
            return 64
        if self.sq >= 256 and self.skv >= 128:
            return 128
        return 32 if (self.sq <= 32 and self.skv <= 32) else 64

    def gate(self, r, scale=None, **kw):
        n_acc, n_l = flash_counts(self.skv, self.tile())
        return gate(r, hd=self.hd, scale=self.scale if scale is None else scale, n_acc=n_acc, n_l=n_l, **kw)

    def expect(self, ops, name, scale=None, **kw):
        out = self.run(ops, scale)
        r = self.ref(scale)
        check(name, out, r, self.gate(r, scale, **kw))
        return out, r


def peak(q, k, jstar, lead, scale, kv_of=None):
    """Every query of (batch b, head h) gets +4 in dimension h % hd; key jstar(bk, h) of K batch bk gets a value there that
    puts its scaled score `lead` above the typical score.  Returns the table of j* [K batches, heads]."""
    nb, heads, hd = k.shape[0], k.shape[2], k.shape[3]
    js = torch.zeros(nb, heads, dtype=torch.long)
    for h in range(heads):
        d0 = h % hd
        q[:, :, h, d0] = 4.0
        for bk in range(nb):
            j = jstar(bk, h)
            js[bk, h] = j
            k[bk, j, h, d0] = (lead + 2.0) / (4.0 * scale)
    return js


def assert_follows_peak(out, v, js, div, rows=None):
    """out[b, :, h] == v[b // div, j*(b // div, h), h] to fp16 rounding and the lead's residue."""
    for b in range(out.shape[0]):
        for h in range(out.shape[2]):
            want = v[b // div, js[b // div, h], h].double()
            got = out[b, :, h].double() if rows is None else out[b, rows, h].double()
            err = (got - want).abs().max().item()
            assert err <= 4 * 2.0 ** -11 * want.abs().max().item() + 1e-3, f'batch {b} head {h}: output is not v[j*] ({err})'


# ---------------------------------------------------------------- 1. random inputs over the tile / routing edges
TC_SQ, TC_SKV = [256, 257, 383, 1000, 4096, 9216], [128, 129, 200, 255, 256, 1000]


@pytest.mark.parametrize('sq', TC_SQ)
@pytest.mark.parametrize('skv', TC_SKV)
def test_tc_random(ops, sq, skv):
    batch, heads = (1, 2) if sq == 9216 else (2, 2)
    Attn(hd=64, batch=batch, heads=heads, sq=sq, skv=skv, seed=sq * 7 + skv).expect(ops, f'tc sq={sq} skv={skv}')


@pytest.mark.parametrize('batch,div,sq,skv', [(5, 2, 256, 128), (7, 3, 383, 200), (4, 3, 1000, 1000), (5, 2, 257, 129)])
def test_tc_kv_batch_div(ops, batch, div, sq, skv):
    """Frames sharing K / V (kv_batch_div), batch not a multiple of it: the last K/V batch serves fewer frames."""
    Attn(hd=64, batch=batch, heads=3, sq=sq, skv=skv, div=div, seed=batch * 31 + div).expect(ops, f'tc div={div} batch={batch}')


@pytest.mark.parametrize('sq', [33, 64, 65, 100, 255])
@pytest.mark.parametrize('skv', [1, 2, 31, 33, 64, 65, 77, 127])
def test_warp64_random(ops, sq, skv):
    Attn(hd=64, batch=3, heads=2, sq=sq, skv=skv, div=3 if skv == 77 else 1, seed=sq * 131 + skv).expect(
        ops, f'warp64 sq={sq} skv={skv}')


@pytest.mark.parametrize('sq', [1, 2, 7, 16, 24, 31, 32])
@pytest.mark.parametrize('skv', [1, 2, 7, 16, 24, 31, 32])
def test_warp32_random(ops, sq, skv):
    Attn(hd=64, batch=4, heads=2, sq=sq, skv=skv, seed=sq * 37 + skv).expect(ops, f'warp32 sq={sq} skv={skv}')


HDS = [8, 16, 32, 40, 80, 160]
HD_S = [1, 63, 64, 65, 77, 200]


@pytest.mark.parametrize('hd', HDS)
@pytest.mark.parametrize('sq', HD_S)
@pytest.mark.parametrize('skv', HD_S)
def test_hd_random(ops, hd, sq, skv):
    """kv_batch_div 1 and F = 3 (6 frames of 2 samples reading their sample's K / V)."""
    for div in (1, 3):
        Attn(hd=hd, batch=6, heads=2, sq=sq, skv=skv, div=div, seed=hd * 1000 + sq * 7 + skv).expect(
            ops, f'hd{hd} sq={sq} skv={skv} div={div}')


@pytest.mark.parametrize('scale', [0.05, 0.3])
@pytest.mark.parametrize('route,hd,sq,skv', [('tc', 64, 300, 200), ('warp64', 64, 100, 77), ('warp32', 64, 24, 24),
                                             ('hd40', 40, 100, 77), ('hd160', 160, 65, 130)])
def test_nondefault_scale(ops, route, hd, sq, skv, scale):
    Attn(hd=hd, batch=2, heads=2, sq=sq, skv=skv, scale=scale, seed=int(scale * 100) + sq).expect(ops, f'{route} scale={scale}')


# ---------------------------------------------------------------- 2. peaked scores: the online-softmax rescale runs
PEAK_CASES = {        # route: (hd, sq, skv, positions of j*: first tile, last row of a tile, first row of the next, ragged last)
    'tc': (64, 300, 300, [3, 127, 128, 299]),
    'warp64': (64, 100, 150, [3, 63, 64, 149]),
    'warp32': (64, 24, 31, [0, 15, 16, 30]),
    'hd40': (40, 100, 150, [3, 63, 64, 149]),
    'hd80': (80, 65, 150, [3, 63, 64, 149]),
    'hd160': (160, 65, 150, [3, 63, 64, 149]),
    'hd8': (8, 65, 150, [3, 63, 64, 149]),
}


@pytest.mark.parametrize('route', list(PEAK_CASES))
@pytest.mark.parametrize('div', [1, 2])
def test_peaked_scores(ops, route, div):
    """Lead ~30: the output is v[j*] of the query's own (K batch, head); j* moves with both, over every tile edge."""
    hd, sq, skv, pos = PEAK_CASES[route]
    a = Attn(hd=hd, batch=8 // (3 - div), heads=3, sq=sq, skv=skv, div=div, seed=11, qscale=0.5)
    js = peak(a.q, a.k, lambda b, h: pos[(3 * b + h) % len(pos)], 30.0, a.scale)
    out, _ = a.expect(ops, f'peak30 {route} div={div}')
    assert_follows_peak(out, a.v, js, div)


@pytest.mark.parametrize('route', list(PEAK_CASES))
def test_late_moderate_peak(ops, route):
    """Lead ~6 with j* in the last tiles: the earlier tiles hold real probability mass that the late maximum rescales."""
    hd, sq, skv, pos = PEAK_CASES[route]
    a = Attn(hd=hd, batch=3, heads=3, sq=sq, skv=skv, seed=12, qscale=0.5)
    late = pos[-2:]
    peak(a.q, a.k, lambda b, h: late[(b + h) % 2], 6.0, a.scale)
    a.expect(ops, f'peak6 {route}')


# ---------------------------------------------------------------- 3. uniform attention (K = 0)
UNIFORM = [('tc', 64, 257, 200), ('warp64', 64, 100, 77), ('warp32', 64, 7, 31), ('hd40', 40, 65, 130), ('hd8', 8, 1, 65),
           ('hd160', 160, 77, 1)]


@pytest.mark.parametrize('route,hd,sq,skv', UNIFORM)
def test_uniform_attention(ops, route, hd, sq, skv):
    """Every row is the mean of exactly the valid V rows of its own (K batch, head): a wrong denominator, a pad key counted
    as valid or a wrong K / V batch fails the near-exact gate."""
    a = Attn(hd=hd, batch=6, heads=2, sq=sq, skv=skv, div=3, pad=True, seed=13)
    a.k.zero_()
    out = a.run(ops)
    r = a.ref()
    check(f'uniform {route}', out, r, a.gate(r, p_round=False, exact_scores=True))


# ---------------------------------------------------------------- 4 / 5. traps outside the input views, writes inside the output view
ROUTES = [('tc', 64, 300, 200), ('warp64', 64, 100, 77), ('warp32', 64, 24, 31), ('hd40', 40, 100, 77), ('hd80', 80, 65, 65),
          ('hd160', 160, 64, 200), ('hd16', 16, 200, 63)]


def assert_output_pads_untouched(a):
    """Pad rows / columns of O are still the NaN they were filled with, bit for bit."""
    bits = a.ob.view(torch.int16)
    C = a.heads * a.hd
    assert (bits[:, a.sq:] == NAN16).all(), 'a kernel wrote past the last query row of a batch'
    assert (bits[:, :, C:] == NAN16).all(), 'a kernel wrote into the pad columns'


@pytest.mark.parametrize('route,hd,sq,skv', ROUTES)
def test_nan_pads(ops, route, hd, sq, skv):
    """NaN in every pad row and pad column of Q, K, V and around O: the output is finite, passes the gate, and O's pads
    are untouched."""
    a = Attn(hd=hd, batch=5, heads=2, sq=sq, skv=skv, div=2, pad=True, seed=14)
    a.expect(ops, f'nan pads {route}')
    assert_output_pads_untouched(a)


@pytest.mark.parametrize('route,hd,sq,skv', ROUTES)
def test_trap_key_past_skv(ops, route, hd, sq, skv):
    """K row skv (inside the batch stride) would dominate every score and the V row behind it is 1e4: nothing moves."""
    a = Attn(hd=hd, batch=4, heads=2, sq=sq, skv=skv, div=2, pad=True, seed=15, qscale=0.5)
    C = a.heads * hd
    for h in range(a.heads):
        a.q[:, :, h, h % hd] = 4.0
        a.kb[:, skv, h * hd + h % hd] = 40.0 / (4.0 * a.scale)
    a.kb[:, skv:, :C].nan_to_num_(0.0)
    a.vb[:, skv, :C] = 1e4
    a.expect(ops, f'trap {route}')
    assert_output_pads_untouched(a)


# ---------------------------------------------------------------- 6. the ModelScope temporal two-level batch
class Temporal:
    """qkv [(b, f, p), 3C] as the UNet's temporal transformer holds it: batch = B * P sequences, b_inner = P."""

    def __init__(self, *, B, P, F, heads, seed):
        self.B, self.P, self.F, self.heads = B, P, F, heads
        self.C = heads * 64
        self.ld = 3 * self.C
        self.qkv = (torch.randn(B * F * P, self.ld, device=dev, generator=gen(seed))).half()
        self.o = torch.full((B * F * P, self.C), float('nan'), device=dev, dtype=torch.half)

    def views(self):           # [B * P, F, heads, 64] views of q / k / v in the kernels' batch order (b, p)
        t = self.qkv.view(self.B, self.F, self.P, 3, self.heads, 64)
        return [t[:, :, :, i].permute(0, 2, 1, 3, 4).reshape(self.B * self.P, self.F, self.heads, 64) for i in range(3)]

    def run(self, ops):
        B, P, F, C, ld = self.B, self.P, self.F, self.C, self.ld
        q = self.qkv
        ops.attention_hd(q, q[:, C:], q[:, 2 * C:], self.o, F * P * ld, P * ld, F * P * ld, P * ld, F * P * ld, P * ld, F * P * C,
                         P * C, B * P, self.heads, 64, F, F, scale=0.125, b_inner=P, q_bsi=ld, k_bsi=ld, v_bsi=ld, o_bsi=C)
        return self.o.view(B, F, P, self.heads, 64).permute(0, 2, 1, 3, 4).reshape(B * P, F, self.heads, 64)

    def ref(self):
        B, P, F, ld = self.B, self.P, self.F, self.ld
        bm = torch.arange(B * P)
        q, k, v = (gather(self.qkv[:, i * self.C:], F, self.heads, 64, F * P * ld, P * ld, bm, b_inner=P, bsi=ld) for i in range(3))
        return attention64(q, k, v, 0.125)

    def gate(self, r):
        n_acc, n_l = flash_counts(self.F, 32 if self.F <= 32 else 64)
        return gate(r, hd=64, scale=0.125, n_acc=n_acc, n_l=n_l)


@pytest.mark.parametrize('P', [24, 64])
@pytest.mark.parametrize('F', [1, 2, 16, 24, 32, 33, 40, 125])
def test_temporal_two_level_batch(ops, P, F):
    t = Temporal(B=2, P=P, F=F, heads=2, seed=P * 1000 + F)
    out = t.run(ops)
    r = t.ref()
    check(f'temporal P={P} F={F}', out, r, t.gate(r))


@pytest.mark.parametrize('P', [24, 64])
@pytest.mark.parametrize('F', [16, 33, 125])
def test_temporal_two_level_batch_peaked(ops, P, F):
    """j* depends on (b, p): a wrong outer / inner batch mapping reads another pixel's V."""
    t = Temporal(B=2, P=P, F=F, heads=2, seed=P + F)
    q, k, v = t.views()                         # copies (the (b, p) order is not a view); written back below
    q.mul_(0.5)
    pos = sorted({p for p in (0, 3, F // 2, 31, 32, 63, 64, F - 1) if p < F})
    js = peak(q, k, lambda s, h: pos[(s * 5 + h) % len(pos)], 30.0, 0.125)
    qkv = t.qkv.view(t.B, t.F, t.P, 3, t.heads, 64)
    for i, x in enumerate((q, k, v)):
        qkv[:, :, :, i] = x.view(t.B, t.P, t.F, t.heads, 64).permute(0, 2, 1, 3, 4)
    out = t.run(ops)
    r = t.ref()
    check(f'temporal peak P={P} F={F}', out, r, t.gate(r))
    assert_follows_peak(out, v, js, 1)


# ---------------------------------------------------------------- relative-position temporal attention
class Relpos:
    """VideoCrafter temporal attention on qkv [(b, t, p), ld], ld = 3C (+ 8 NaN pad columns), sequences (b, p) along t;
    pad=True: one NaN frame past T per sample and 48-row tables with NaN past row 2L."""

    def __init__(self, *, hd, T, L, heads=2, B=2, P=3, pad=False, seed=0):
        self.hd, self.T, self.L, self.heads, self.B, self.P = hd, T, L, heads, B, P
        self.C = heads * hd
        self.ld = 3 * self.C + (8 if pad else 0)
        self.Tb = T + (1 if pad else 0)
        g = gen(seed)
        nan = float('nan')
        self.qkv = torch.full((B, self.Tb, P, self.ld), nan, device=dev, dtype=torch.half)
        self.qkv[:, :T, :, :3 * self.C] = torch.randn(B, T, P, 3 * self.C, device=dev, generator=g).half()
        rows = 48 if pad else 2 * L + 1
        self.tk = torch.full((rows, hd), nan, device=dev, dtype=torch.half)
        self.tv = torch.full((rows, hd), nan, device=dev, dtype=torch.half)
        self.tk[:2 * L + 1] = (torch.randn(2 * L + 1, hd, device=dev, generator=g) * 0.5).half()
        self.tv[:2 * L + 1] = (torch.randn(2 * L + 1, hd, device=dev, generator=g) * 0.5).half()
        self.o = torch.full((B, self.Tb, P, self.C + (8 if pad else 0)), nan, device=dev, dtype=torch.half)
        self.scale = hd ** -0.5

    def run(self, ops):
        C, ld, P, Tb = self.C, self.ld, self.P, self.Tb
        q = self.qkv.view(-1, ld)
        lo = self.o.shape[-1]
        ops.attention_relpos(q, q[:, C:], q[:, 2 * C:], self.o, self.tk, self.tv, self.B * P, P, Tb * P * ld, ld, P * ld,
                             Tb * P * lo, lo, P * lo, self.heads, self.hd, self.T, self.L)
        return self.o[:, :self.T, :, :C].permute(0, 2, 1, 3).reshape(self.B * P, self.T, self.heads, self.hd)

    def ref(self):
        P, ld = self.P, self.ld
        bm = torch.arange(self.B * P)
        q, k, v = (gather(self.qkv.view(-1, ld)[:, i * self.C:], self.T, self.heads, self.hd, self.Tb * P * ld, P * ld, bm,
                          b_inner=P, bsi=ld) for i in range(3))
        return attention64(q, k, v, self.scale, rk=self.tk[:2 * self.L + 1], rv=self.tv[:2 * self.L + 1], max_rel=self.L)

    def gate(self, r, **kw):
        return gate(r, hd=self.hd, scale=self.scale, n_acc=(self.T + 48) / 16 + 4, n_l=self.T / 4 + 4, tab_round=True, **kw)


RELPOS_HD = [8, 16, 32, 40, 64, 80, 160]
RELPOS_TL = sorted({(T, L) for T in (1, 2, 15, 16, 17, 31, 32) for L in (1, T - 1, T, 23) if 1 <= L <= 23})   # 2L+1 <= 48


@pytest.mark.parametrize('hd', RELPOS_HD)
@pytest.mark.parametrize('T,L', RELPOS_TL)
def test_relpos_random(ops, hd, T, L):
    a = Relpos(hd=hd, T=T, L=L, seed=hd * 100 + T * 3 + L)
    out = a.run(ops)
    r = a.ref()
    check(f'relpos hd={hd} T={T} L={L}', out, r, a.gate(r))


@pytest.mark.parametrize('hd', [40, 64, 160])
@pytest.mark.parametrize('T,L', [(16, 23), (17, 7), (32, 16), (1, 1), (5, 2)])
def test_relpos_nan_pads(ops, hd, T, L):
    """NaN in table rows 2L+1 .. 47, in the frame past T and in the pad columns; O's pads stay NaN."""
    a = Relpos(hd=hd, T=T, L=L, pad=True, seed=hd + T + L)
    out = a.run(ops)
    r = a.ref()
    check(f'relpos pads hd={hd} T={T} L={L}', out, r, a.gate(r))
    bits = a.o.view(torch.int16)
    assert (bits[:, T:] == NAN16).all() and (bits[..., a.C:] == NAN16).all(), 'relpos wrote outside its output view'


@pytest.mark.parametrize('hd', [40, 80])
@pytest.mark.parametrize('T', [16, 24])
def test_relpos_uniform(ops, hd, T):
    """K = 0 and both tables 0: every frame is the mean of its sequence's T value rows."""
    a = Relpos(hd=hd, T=T, L=16, seed=T)
    a.qkv[..., a.C:2 * a.C] = 0
    a.tk.zero_()
    a.tv.zero_()
    out = a.run(ops)
    r = a.ref()
    check(f'relpos uniform hd={hd} T={T}', out, r, a.gate(r))


# ---------------------------------------------------------------- CLIP causal attention
def clip_case(ops, B, L, heads, seed, qkv=None):
    W = heads * 64
    if qkv is None:
        qkv = torch.randn(B * L, 3 * W, device=dev, generator=gen(seed)).half()
    ob = torch.full((B * L + 3, W), float('nan'), device=dev, dtype=torch.half)
    ops.clip_attention(qkv, L, heads, o=ob[:B * L])
    assert (ob[B * L:].view(torch.int16) == NAN16).all(), 'clip attention wrote past its output'
    return qkv, ob[:B * L]


def clip_ref(qkv, B, L, heads):
    W = heads * 64
    bm = torch.arange(B)
    q, k, v = (gather(qkv[:, i * W:], L, heads, 64, L * 3 * W, 3 * W, bm) for i in range(3))
    return attention64(q, k, v, 0.125, causal=True)


@pytest.mark.parametrize('L', [1, 31, 32, 33, 77, 128])
@pytest.mark.parametrize('heads', [12, 16, 20])
@pytest.mark.parametrize('B', [1, 3])
def test_clip_random(ops, L, heads, B):
    qkv, o = clip_case(ops, B, L, heads, seed=L * 100 + heads + B)
    r = clip_ref(qkv, B, L, heads)
    check(f'clip B={B} L={L} heads={heads}', o.view(B, L, heads, 64), r, gate(r, hd=64, scale=0.125, n_acc=L, n_l=8, p_round=False))


@pytest.mark.parametrize('L', [2, 33, 77, 128])
def test_clip_causality(ops, L):
    """A key at position L - 1 that dominates every score leaves rows 0 .. L - 2 bit-identical; row L - 1 follows it."""
    B, heads = 2, 12
    W = heads * 64
    plain = torch.randn(B, L, 3 * W, device=dev, generator=gen(L)).half()
    plain[:, :, :W] *= 0.5
    plain[:, :, 0:W:64] = 4.0                       # every query has +4 in component 0 of every head
    trap = plain.clone()
    trap[:, L - 1, W:2 * W:64] = 100.0              # key L - 1 leads every score it enters by ~50
    _, o_plain = clip_case(ops, B, L, heads, 0, qkv=plain.view(B * L, 3 * W))
    _, o_trap = clip_case(ops, B, L, heads, 0, qkv=trap.view(B * L, 3 * W))
    o_plain, o_trap = o_plain.view(B, L, W), o_trap.view(B, L, W)
    assert torch.equal(o_trap[:, :L - 1].view(torch.int16), o_plain[:, :L - 1].view(torch.int16)), 'a query saw a future key'
    v_last = trap[:, L - 1, 2 * W:].double()
    err = (o_trap[:, L - 1].double() - v_last).abs().max().item()
    assert err <= 4 * 2.0 ** -11 * v_last.abs().max().item(), f'row L - 1 does not follow its dominant key ({err})'


def test_clip_uniform(ops):
    """K = 0: row t is the mean of V rows 0 .. t."""
    B, L, heads = 2, 77, 16
    W = heads * 64
    qkv = torch.randn(B * L, 3 * W, device=dev, generator=gen(5)).half()
    qkv[:, W:2 * W] = 0
    _, o = clip_case(ops, B, L, heads, seed=0, qkv=qkv)
    r = clip_ref(qkv, B, L, heads)
    check('clip uniform', o.view(B, L, heads, 64), r, gate(r, hd=64, scale=0.125, n_acc=L, n_l=8, p_round=False))


# ---------------------------------------------------------------- 8. routing, read from the profiler
def launched(fn):
    """Kernel routes that `fn` launched, from torch.profiler's CUDA activity (a run of its own, nothing is timed)."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    names = {e.name for e in prof.events() if 'attention' in e.name}
    routes = set()
    for n in names:
        if 'attention_tc_kernel' in n:
            routes.add('tc')
        elif 'clip_attention_kernel' in n:
            routes.add('clip')
        elif 'attention_relpos_kernel' in n:
            m = re.search(r'attention_relpos_kernel(?:<(\d+), ?(\d+)>|ILi(\d+)ELi(\d+)E)', n)
            routes.add('relpos%s_%s' % ((m.group(1), m.group(2)) if m.group(1) else (m.group(3), m.group(4))))
        elif 'attention_hd_kernel' in n:
            m = re.search(r'attention_hd_kernel(?:<(\d+)>|ILi(\d+)E)', n)
            routes.add('hd' + (m.group(1) or m.group(2)))
        elif 'attention_kernel' in n:
            m = re.search(r'attention_kernel(?:<(\d+)>|ILi(\d+)E)', n)
            routes.add('warp' + (m.group(1) or m.group(2)))
    return routes


def fused_self(ops, heads, S, batch, hd=64):
    C = heads * hd
    ld = 3 * C
    qkv = torch.randn(batch * S, ld, device=dev, generator=gen(S)).half()
    o = torch.empty(batch * S, C, device=dev, dtype=torch.half)
    a = (qkv, qkv[:, C:], qkv[:, 2 * C:], o, S * ld, ld, S * ld, ld, S * ld, ld, S * C, C, batch, heads)
    return lambda: ops.attention(*a, S, S) if hd == 64 else ops.attention_hd(*a, hd, S, S)


def cross(ops, heads, S, F, B=2, hd=64, L=77):
    """Spatial cross-attention: B samples of F frames, K / V of the prompt [(b, l), 2C] shared by a sample's frames."""
    C = heads * hd
    q = torch.randn(B * F * S, C, device=dev, generator=gen(S)).half()
    kv = torch.randn(B * L, 2 * C, device=dev, generator=gen(L)).half()
    o = torch.empty_like(q)
    a = (q, kv, kv[:, C:], o, S * C, C, L * 2 * C, 2 * C, L * 2 * C, 2 * C, S * C, C, B * F, heads)
    if hd == 64:
        return lambda: ops.attention(*a, S, L, kv_batch_div=F)
    return lambda: ops.attention_hd(*a, hd, S, L, kv_batch_div=F)


def temporal(ops, heads, P, F, B=2):
    t = Temporal(B=B, P=P, F=F, heads=heads, seed=1)
    return lambda: t.run(ops)


def relpos_call(ops, hd, T, P, heads=8, L=16):
    a = Relpos(hd=hd, T=T, L=L, heads=heads, B=1, P=P, seed=2)
    return lambda: a.run(ops)


def clip_call(ops, B, heads, L=77):
    qkv = torch.randn(B * L, 3 * heads * 64, device=dev, generator=gen(3)).half()
    return lambda: ops.clip_attention(qkv, L, heads)


def sized(ops, sq, skv, b_inner=1):
    """Dense head-64 call at (sq, skv); b_inner > 1 through t2v_op_attention_hd."""
    C = 64
    q = torch.randn(2 * sq, C, device=dev, generator=gen(7)).half()
    k = torch.randn(2 * skv, C, device=dev, generator=gen(8)).half()
    o = torch.empty_like(q)
    if b_inner == 1:
        return lambda: ops.attention(q, k, k, o, sq * C, C, skv * C, C, skv * C, C, sq * C, C, 2, 1, sq, skv)
    # batch (outer, inner) = (b // 2, b % 2) with outer stride 0: the two inner batches are the two halves
    return lambda: ops.attention_hd(q, k, k, o, 0, C, 0, C, 0, C, 0, C, 2, 1, 64, sq, skv, b_inner=2,
                                    q_bsi=sq * C, k_bsi=skv * C, v_bsi=skv * C, o_bsi=sq * C)


ROUTING = [
    ('sq 255 -> warp64', lambda o: sized(o, 255, 256), 'warp64'),
    ('sq 256 -> tc', lambda o: sized(o, 256, 256), 'tc'),
    ('skv 127 -> warp64', lambda o: sized(o, 256, 127), 'warp64'),
    ('skv 128 -> tc', lambda o: sized(o, 256, 128), 'tc'),
    ('32 x 32 -> warp32', lambda o: sized(o, 32, 32), 'warp32'),
    ('33 x 33 -> warp64', lambda o: sized(o, 33, 33), 'warp64'),
    ('b_inner 2 at S 1024 -> warp64', lambda o: sized(o, 1024, 1024, b_inner=2), 'warp64'),
    ('ModelScope spatial 32x32', lambda o: fused_self(o, 5, 1024, 2), 'tc'),
    ('ModelScope spatial 16x16', lambda o: fused_self(o, 10, 256, 2), 'tc'),
    ('ModelScope spatial 8x8', lambda o: fused_self(o, 20, 64, 2), 'warp64'),
    ('ModelScope cross 32x32', lambda o: cross(o, 5, 1024, 16), 'warp64'),
    ('ModelScope cross 8x8', lambda o: cross(o, 20, 64, 16), 'warp64'),
    ('ModelScope temporal F=16', lambda o: temporal(o, 5, 1024, 16), 'warp32'),
    ('ModelScope temporal F=125', lambda o: temporal(o, 20, 64, 125), 'warp64'),
    ('VideoCrafter spatial 40', lambda o: fused_self(o, 8, 1280, 2, hd=40), 'hd40'),
    ('VideoCrafter spatial 160', lambda o: fused_self(o, 8, 80, 2, hd=160), 'hd160'),
    ('VideoCrafter cross 80', lambda o: cross(o, 8, 320, 16, hd=80), 'hd80'),
    ('VideoCrafter temporal 40 T=16', lambda o: relpos_call(o, 40, 16, 1280), 'relpos40_16'),
    ('VideoCrafter temporal 160 T=24', lambda o: relpos_call(o, 160, 24, 80), 'relpos160_32'),
    ('CLIP ViT-H text tower', lambda o: clip_call(o, 2, 16), 'clip'),
    ('CLIP ViT-L text tower', lambda o: clip_call(o, 2, 12), 'clip'),
]


@pytest.mark.parametrize('what,make,route', ROUTING, ids=[r[0] for r in ROUTING])
def test_routing(ops, what, make, route):
    fn = make(ops)
    fn()                                # module load / shared-memory attribute outside the profiled run
    assert launched(fn) == {route}, f'{what}: expected {route}'


# ---------------------------------------------------------------- 9. determinism
DETERMINISM = [('tc', lambda o: fused_self(o, 5, 1024, 2)), ('warp64', lambda o: cross(o, 5, 256, 4)),
               ('warp32', lambda o: temporal(o, 5, 64, 16)), ('hd40', lambda o: cross(o, 8, 320, 4, hd=40)),
               ('relpos', lambda o: relpos_call(o, 80, 16, 64)), ('clip', lambda o: clip_call(o, 2, 16))]


@pytest.mark.parametrize('route,make', DETERMINISM, ids=[d[0] for d in DETERMINISM])
def test_deterministic(ops, route, make):
    """No atomics anywhere: two identical calls return identical bits."""
    fn = make(ops)
    a = fn().clone()
    b = fn()
    assert torch.equal(a.view(torch.int16), b.view(torch.int16))
