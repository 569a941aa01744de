"""CPU: the attention entry points refuse operands their kernels cannot load, before any launch.

The warp-MMA and any-head-dim kernels load Q, K, V (and the relative-position tables) with 16-byte cp.async and store O
as __half2, so t2v_op_attention / _hd / _relpos return -1 when a pointer or stride breaks that, instead of launching a
kernel that would fault.  t2v_op_clip_attention returns -1 for shapes the CLIP kernel does not take.

The pointers here are fake integers and t2v_init is never called: a rejected call never touches them.  Without a device,
a call that gets past the checks fails later at its launch with a different code (-2, or -4 where a shared-memory
attribute is set first), so each -1 below is the argument check and nothing else.  The module is skipped on a machine
with a GPU: no misaligned call is ever launched on a device."""
import ctypes as C

import pytest
import torch

from t2v_b200 import _lib

pytestmark = pytest.mark.skipif(torch.cuda.is_available(), reason='argument checks run on CPU only: never launch a misaligned call')

BASE = 0x10000000          # fake, 256-byte aligned device addresses
Q, K, V, O, TK, TV = (C.c_void_p(BASE + i * 0x1000000) for i in range(6))


@pytest.fixture(scope='module')
def lib():
    return _lib.load_library()


def shifted(p, nbytes):
    return C.c_void_p(p.value + nbytes)


# ---------------------------------------------------------------- t2v_op_attention / t2v_op_attention_hd (AttnParams)
def attn_args(heads=2, hd=64, sq=256, skv=256, **over):
    """A dense fused-QKV self-attention call (3 frames), every operand aligned; `over` replaces single arguments."""
    C_ = heads * hd
    ld = 3 * C_
    a = dict(q=Q, k=K, v=V, o=O, q_bs=sq * ld, q_ss=ld, k_bs=skv * ld, k_ss=ld, v_bs=skv * ld, v_ss=ld, o_bs=sq * C_, o_ss=C_,
             batch=3, heads=heads, sq=sq, skv=skv, kv_batch_div=1, scale=hd ** -0.5, b_inner=1, q_bsi=0, k_bsi=0, v_bsi=0,
             o_bsi=0)
    a.update(over)
    return a


def call_attention(lib, a):
    return lib.t2v_op_attention(a['q'], a['k'], a['v'], a['o'], a['q_bs'], a['q_ss'], a['k_bs'], a['k_ss'], a['v_bs'], a['v_ss'],
                                a['o_bs'], a['o_ss'], a['batch'], a['heads'], a['sq'], a['skv'], a['kv_batch_div'], a['scale'],
                                None)


def call_attention_hd(lib, a, hd):
    return lib.t2v_op_attention_hd(a['q'], a['k'], a['v'], a['o'], a['q_bs'], a['q_ss'], a['k_bs'], a['k_ss'], a['v_bs'],
                                   a['v_ss'], a['o_bs'], a['o_ss'], a['batch'], a['heads'], hd, a['sq'], a['skv'],
                                   a['kv_batch_div'], a['scale'], a['b_inner'], a['q_bsi'], a['k_bsi'], a['v_bsi'], a['o_bsi'],
                                   None)


MISALIGNED = [
    ('q', lambda a: shifted(a['q'], 8)), ('k', lambda a: shifted(a['k'], 2)), ('v', lambda a: shifted(a['v'], 4)),
    ('o', lambda a: shifted(a['o'], 2)),
    ('q_ss', lambda a: a['q_ss'] + 4), ('k_ss', lambda a: a['k_ss'] + 2), ('v_ss', lambda a: a['v_ss'] + 1),
    ('q_bs', lambda a: a['q_bs'] + 4), ('k_bs', lambda a: a['k_bs'] + 6), ('v_bs', lambda a: a['v_bs'] + 4),
    ('o_ss', lambda a: a['o_ss'] + 1), ('o_bs', lambda a: a['o_bs'] + 1),
]
# (sq, skv) reaching each head-64 kernel with aligned operands: wgmma (misaligned calls fall off it), warp MMA 64 and 32
SHAPES64 = [(256, 256), (100, 77), (24, 24)]


@pytest.mark.parametrize('field,bad', MISALIGNED, ids=[m[0] for m in MISALIGNED])
@pytest.mark.parametrize('sq,skv', SHAPES64)
def test_attention_rejects_misaligned(lib, field, bad, sq, skv):
    a = attn_args(sq=sq, skv=skv)
    a[field] = bad(a)
    assert call_attention(lib, a) == -1
    assert b'attention' in lib.t2v_last_error()


@pytest.mark.parametrize('hd', [8, 16, 32, 40, 80, 160, 64])
@pytest.mark.parametrize('field,bad', MISALIGNED, ids=[m[0] for m in MISALIGNED])
def test_attention_hd_rejects_misaligned(lib, field, bad, hd):
    a = attn_args(hd=hd, sq=100, skv=77)
    a[field] = bad(a)
    assert call_attention_hd(lib, a, hd) == -1


@pytest.mark.parametrize('hd', [40, 64])
@pytest.mark.parametrize('field', ['q_bsi', 'k_bsi', 'v_bsi', 'o_bsi'])
def test_attention_hd_rejects_misaligned_inner_batch_stride(lib, field, hd):
    """The two-level (ModelScope temporal) layout: [(b, f, p), 3C], b_inner = P; an odd inner stride is refused."""
    Fr, P = 16, 24
    C_ = 2 * hd
    ld = 3 * C_
    a = attn_args(hd=hd, sq=Fr, skv=Fr, batch=2 * P, b_inner=P, q_bs=Fr * P * ld, k_bs=Fr * P * ld, v_bs=Fr * P * ld,
                  o_bs=Fr * P * C_, q_bsi=ld, k_bsi=ld, v_bsi=ld, o_bsi=C_, q_ss=P * ld, k_ss=P * ld, v_ss=P * ld, o_ss=P * C_)
    a[field] += 1 if field == 'o_bsi' else 4
    assert call_attention_hd(lib, a, hd) == -1


@pytest.mark.parametrize('sq,skv', SHAPES64)
def test_aligned_calls_get_past_the_check(lib, sq, skv):
    """Control: the same calls with every operand aligned (and zero broadcast strides) are not refused by the argument
    check; with no device they fail at the launch with another code."""
    a = attn_args(sq=sq, skv=skv, k_bs=0, v_bs=0)
    assert call_attention(lib, a) not in (0, -1)
    assert call_attention_hd(lib, attn_args(hd=40, sq=sq, skv=skv), 40) not in (0, -1)


# ---------------------------------------------------------------- t2v_op_attention_relpos
def relpos_args(hd=40, T=16, L=16, **over):
    heads, B, P = 8, 2, 24
    C_ = heads * hd
    ld = 3 * C_
    a = dict(q=Q, k=K, v=V, o=O, tk=TK, tv=TV, n_seq=B * P, seq_inner=P, bs_outer=T * P * ld, bs_inner=ld, ss=P * ld,
             o_bs_outer=T * P * C_, o_bs_inner=C_, o_ss=P * C_, heads=heads, hd=hd, T=T, L=L, scale=hd ** -0.5)
    a.update(over)
    return a


def call_relpos(lib, a):
    return lib.t2v_op_attention_relpos(a['q'], a['k'], a['v'], a['o'], a['tk'], a['tv'], a['n_seq'], a['seq_inner'],
                                       a['bs_outer'], a['bs_inner'], a['ss'], a['o_bs_outer'], a['o_bs_inner'], a['o_ss'],
                                       a['heads'], a['hd'], a['T'], a['L'], a['scale'], None)


RELPOS_BAD = [
    ('q', lambda a: shifted(a['q'], 8)), ('k', lambda a: shifted(a['k'], 4)), ('v', lambda a: shifted(a['v'], 2)),
    ('o', lambda a: shifted(a['o'], 2)), ('tk', lambda a: shifted(a['tk'], 8)), ('tv', lambda a: shifted(a['tv'], 2)),
    ('bs_outer', lambda a: a['bs_outer'] + 4), ('bs_inner', lambda a: a['bs_inner'] + 2), ('ss', lambda a: a['ss'] + 1),
    ('o_bs_outer', lambda a: a['o_bs_outer'] + 1), ('o_bs_inner', lambda a: a['o_bs_inner'] + 1),
    ('o_ss', lambda a: a['o_ss'] + 1),
]


@pytest.mark.parametrize('hd,T', [(40, 16), (80, 32), (64, 17), (8, 1)])
@pytest.mark.parametrize('field,bad', RELPOS_BAD, ids=[m[0] for m in RELPOS_BAD])
def test_attention_relpos_rejects_misaligned(lib, field, bad, hd, T):
    a = relpos_args(hd=hd, T=T)
    a[field] = bad(a)
    assert call_relpos(lib, a) == -1
    assert b'attention_relpos' in lib.t2v_last_error()


def test_attention_relpos_aligned_call_gets_past_the_check(lib):
    assert call_relpos(lib, relpos_args()) not in (0, -1)


# ---------------------------------------------------------------- t2v_op_clip_attention
@pytest.mark.parametrize('B,L,W,heads', [(2, 129, 1024, 16), (2, 77, 1024, 8), (2, 77, 1000, 16), (1, 0, 768, 12),
                                         (0, 77, 768, 12)])
def test_clip_attention_rejects_bad_shapes(lib, B, L, W, heads):
    assert lib.t2v_op_clip_attention(Q, O, B, L, W, heads, None) == -1


def test_clip_attention_rejects_misaligned_qkv(lib):
    assert lib.t2v_op_clip_attention(shifted(Q, 2), O, 2, 77, 1024, 16, None) == -1


def test_clip_attention_valid_shape_gets_past_the_check(lib):
    assert lib.t2v_op_clip_attention(Q, O, 2, 77, 1024, 16, None) not in (0, -1)
