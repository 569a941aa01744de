"""CPU: the GroupNorm and LayerNorm entry points refuse arguments their kernels cannot take, before any allocation or launch.

Both kernels load and store x, y, gamma and beta as 16-byte vectors, so an unaligned pointer or a row pitch that is not a
multiple of 8 is refused with -1; so are shapes that would divide by zero on the host (rows_per_inst <= 0, no whole
instance, C = 0) or exceed the grid (more than 65535 GroupNorm instances).

The pointers here are fake integers and t2v_init is never called: a rejected call never touches them.  Without a device, a
GroupNorm call that gets past the checks fails at its workspace allocation with -5, and a LayerNorm call at its launch with
-2, so each -1 below is the argument check and nothing else.  The module is skipped on a machine with a GPU: no bad call is
ever launched on a device."""
import ctypes as C

import pytest
import torch

from t2v_b200 import _lib

pytestmark = pytest.mark.skipif(torch.cuda.is_available(), reason='argument checks run on CPU only: never launch a bad call')

BASE = 0x10000000          # fake, 256-byte aligned device addresses
X, Y, G, B, S = (C.c_void_p(BASE + i * 0x1000000) for i in range(5))


@pytest.fixture(scope='module')
def lib():
    return _lib.load_library()


def shifted(p, nbytes):
    return C.c_void_p(p.value + nbytes)


def gn_args(**over):
    """A valid GroupNorm call: 2 instances of 256 rows, C = 320, dense."""
    a = dict(x=X, ldx=320, y=Y, ldy=320, rows=512, C=320, rpi=256, g=G, b=B, eps=1e-5, silu=1, phase=0, stats=None)
    a.update(over)
    return a


def call_gn(lib, a):
    return lib.t2v_op_groupnorm(a['x'], a['ldx'], a['y'], a['ldy'], a['rows'], a['C'], a['rpi'], a['g'], a['b'], a['eps'],
                                a['silu'], a['phase'], a['stats'], None)


GN_BAD = [
    # host division by zero before the checks existed (the process died with SIGFPE)
    ('rows_per_inst=0', dict(rpi=0)), ('rows_per_inst<0', dict(rpi=-4)), ('empty x', dict(rows=0)),
    ('rows<rows_per_inst', dict(rows=100, rpi=256)), ('C=0', dict(C=0, ldx=0, ldy=0)),
    # shapes the kernels do not take
    ('C=48', dict(C=48)), ('C=2592', dict(C=2592, ldx=2592, ldy=2592)), ('C<0', dict(C=-32)),
    ('partial instance', dict(rows=513)),
    ('65536 instances', dict(rows=65536, rpi=1)), ('131073 instances', dict(rows=131073, rpi=1)),
    # 16-byte vector accesses
    ('x+2', dict(x=shifted(X, 2))), ('x+8', dict(x=shifted(X, 8))), ('y+4', dict(y=shifted(Y, 4))),
    ('gamma+2', dict(g=shifted(G, 2))), ('beta+8', dict(b=shifted(B, 8))),
    ('ldx%8', dict(ldx=324)), ('ldy%8', dict(ldy=322)), ('ldx<C', dict(ldx=312)), ('ldy<C', dict(ldy=0)),
    # phases
    ('phase 3', dict(phase=3)), ('phase -1', dict(phase=-1)), ('phase 1 without stats', dict(phase=1)),
    ('phase 2 without stats', dict(phase=2)),
]


@pytest.mark.parametrize('over', [c[1] for c in GN_BAD], ids=[c[0] for c in GN_BAD])
def test_groupnorm_rejects_bad_arguments(lib, over):
    assert call_gn(lib, gn_args(**over)) == -1
    assert b'groupnorm' in lib.t2v_last_error()


@pytest.mark.parametrize('over', [{}, dict(rows=65535, rpi=1, C=32, ldx=32, ldy=32), dict(ldx=328, ldy=640),
                                  dict(phase=1, stats=S), dict(phase=2, stats=S), dict(C=2560, ldx=2560, ldy=2560, rows=1, rpi=1)],
                         ids=['dense', '65535 instances', 'strided', 'phase 1', 'phase 2', 'C=2560 one row'])
def test_groupnorm_valid_call_gets_past_the_check(lib, over):
    """Control: valid calls reach the workspace allocation, which fails without a device with its own code."""
    assert call_gn(lib, gn_args(**over)) == -5
    assert b'workspace' in lib.t2v_last_error()


def ln_args(**over):
    a = dict(x=X, ldx=768, y=Y, ldy=768, rows=154, C=768, g=G, b=B, eps=1e-5)
    a.update(over)
    return a


def call_ln(lib, a):
    return lib.t2v_op_layernorm(a['x'], a['ldx'], a['y'], a['ldy'], a['rows'], a['C'], a['g'], a['b'], a['eps'], None)


LN_BAD = [
    ('C=0', dict(C=0)), ('C=12', dict(C=12)), ('C=2056', dict(C=2056, ldx=2056, ldy=2056)), ('rows=0', dict(rows=0)),
    ('rows<0', dict(rows=-1)),
    ('x+2', dict(x=shifted(X, 2))), ('y+8', dict(y=shifted(Y, 8))), ('gamma+4', dict(g=shifted(G, 4))),
    ('beta+2', dict(b=shifted(B, 2))), ('ldx%8', dict(ldx=772)), ('ldy%8', dict(ldy=770)), ('ldx<C', dict(ldx=760)),
]


@pytest.mark.parametrize('over', [c[1] for c in LN_BAD], ids=[c[0] for c in LN_BAD])
def test_layernorm_rejects_bad_arguments(lib, over):
    assert call_ln(lib, ln_args(**over)) == -1
    assert b'layernorm' in lib.t2v_last_error()


@pytest.mark.parametrize('over', [{}, dict(ldx=1024, ldy=776), dict(C=8, ldx=8, ldy=8, rows=1)], ids=['dense', 'strided', 'C=8'])
def test_layernorm_valid_call_gets_past_the_check(lib, over):
    assert call_ln(lib, ln_args(**over)) not in (0, -1)
