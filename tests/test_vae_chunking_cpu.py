"""CPU: the VAE's plan-size model (t2v_vae_plan_bytes, the host-only dry pass) and the frame-chunk policy built on it
(t2v_vae_plan_chunks), for the decoder and the encoder of the ModelScope VAE config, without a GPU."""
import ctypes as C

import pytest

from t2v_b200 import _lib

MB = 1 << 20
SIZES = [8, 32]                 # latent sizes; the encoder takes the image, 8x as large
FRAMES = list(range(1, 13))


@pytest.fixture(scope='module')
def ae():
    from t2v_b200.modules import AutoencoderKL
    from t2v_b200.pipeline import VAE_DDCONFIG
    return AutoencoderKL(VAE_DDCONFIG, 4, None)


def _hw(s, encode):
    return (s * 8, s * 8) if encode else (s, s)


def _raw(ae, encode, frames, h, w):
    arena, gn = C.c_size_t(0), C.c_size_t(0)
    rc = _lib.load_library().t2v_vae_plan_bytes(ae._handle, int(encode), frames, h, w, C.byref(arena), C.byref(gn))
    assert rc == 0, _lib.load_library().t2v_last_error()
    return arena.value, gn.value


@pytest.mark.parametrize('encode', [False, True])
@pytest.mark.parametrize('s', SIZES)
def test_plan_bytes_without_device_and_matches_mirror(ae, encode, s):
    h, w = _hw(s, encode)
    for f in (1, 5, 96):
        arena, gn = _raw(ae, encode, f, h, w)
        assert arena > MB and 0 < gn < arena
        assert ae.plan_bytes(f, h, w, encode=encode) == arena + gn


@pytest.mark.parametrize('encode', [False, True])
def test_plan_bytes_monotone_and_affine_in_frames(ae, encode):
    # 32 x 32: the activations set the peak, which grows by the same bytes per frame (least-squares line within 64 KB).
    # 8 x 8: a split-K GEMM's fp32 partials (up to 8 splits, chosen by tile count, so the split count changes with the frame
    # count) are as large as the activations there, so the peak dips by up to 4 MB between some frame counts and sits
    # within 8 MB of the line (measured: 6.0 MB decoder, 4.2 MB encoder).
    import numpy as np
    for s, dip, affine_tol in ((32, 0, 64 << 10), (8, 4 * MB, 8 * MB)):
        h, w = _hw(s, encode)
        b = [ae.plan_bytes(f, h, w, encode=encode) for f in FRAMES]
        for f in range(len(b) - 1):
            assert b[f + 1] >= b[f] - dip, (s, FRAMES[f], b)
        line = np.polyval(np.polyfit(FRAMES, np.array(b, dtype=np.float64), 1), FRAMES)
        assert np.abs(np.array(b) - line).max() <= affine_tol, (s, b)
        if s == 32:
            assert all(b[f + 1] > b[f] for f in range(len(b) - 1))


def _policy(ae, frames, h, w, budget, encode):
    """The chunk policy restated: the largest n whose plan fits (plan bytes are monotone at the sizes this is used at)."""
    fits = [n for n in range(1, frames + 1) if ae.plan_bytes(n, h, w, encode=encode) <= budget]
    n = max(fits)
    return n, -(-frames // n)


@pytest.mark.parametrize('encode', [False, True])
def test_chunk_policy_from_plan_bytes(ae, encode):
    h, w = _hw(32, encode)
    b = {n: ae.plan_bytes(n, h, w, encode=encode) for n in range(1, 8)}
    # F = 7: fits whole, chunks of 3 + a tail of 1, chunks of 2 + a tail of 1, chunks of 1
    assert ae.plan_chunks(7, h, w, b[7], encode=encode) == (7, 1)
    assert ae.plan_chunks(7, h, w, b[7] - 1, encode=encode) == (6, 2)
    assert ae.plan_chunks(7, h, w, b[3], encode=encode) == (3, 3)
    assert ae.plan_chunks(7, h, w, b[3] - 1, encode=encode) == (2, 4)
    assert ae.plan_chunks(7, h, w, b[1], encode=encode) == (1, 7)
    for budget in (b[1] + 1, (b[2] + b[3]) // 2, b[5] + MB, b[6] - MB):
        assert ae.plan_chunks(7, h, w, budget, encode=encode) == _policy(ae, 7, h, w, budget, encode)


def test_chunk_policy_at_zeroscope_xl_size(ae):
    # 96 frames of 72 x 128 latents (576 x 1024) do not fit the 80 GB card as one plan; 24 frames do
    whole, f24 = ae.plan_bytes(96, 72, 128), ae.plan_bytes(24, 72, 128)
    assert whole > 80 * 10 ** 9 * 0.9 and f24 < 40 * 10 ** 9
    n, k = ae.plan_chunks(96, 72, 128, 40 << 30)
    assert ae.plan_bytes(n, 72, 128) <= 40 << 30 < ae.plan_bytes(n + 1, 72, 128)
    assert k == -(-96 // n)


@pytest.mark.parametrize('encode', [False, True])
def test_chunk_policy_result_fits_where_plan_bytes_dip(ae, encode):
    # at 8 x 8 plan bytes are not monotone over 1-4 frames: the bisection still returns a chunk that fits whose successor does not
    h, w = _hw(8, encode)
    b = {n: ae.plan_bytes(n, h, w, encode=encode) for n in range(1, 10)}
    for budget in sorted(set(b.values())):
        if budget >= b[9]:
            continue
        n, k = ae.plan_chunks(9, h, w, budget, encode=encode)
        assert b[n] <= budget < b[n + 1] and k == -(-9 // n), (budget, n, b)


@pytest.mark.parametrize('encode', [False, True])
def test_budget_below_one_frame_is_a_clear_error(ae, encode):
    h, w = _hw(8, encode)
    one = ae.plan_bytes(1, h, w, encode=encode)
    with pytest.raises(RuntimeError) as e:
        ae.plan_chunks(5, h, w, one - 1, encode=encode)
    msg = str(e.value)
    assert 'one-frame plan needs' in msg and f'{h} x {w}' in msg and f'{one / MB:.1f} MB' in msg and 'memory budget' in msg


def test_memory_budget_property(ae):
    assert ae.memory_budget == 0
    ae.memory_budget = 3 << 30
    assert ae.memory_budget == 3 << 30
    ae.memory_budget = 0
    assert ae.memory_budget == 0
    with pytest.raises(ValueError):
        ae.memory_budget = -1
    assert ae.last_chunking() == (0, 0) and ae.cached_plans() == (0, 0)
