"""CPU: VideoCrafter's per-step DDIM outputs and webui state.

  * t2v_ddim_step_ex refuses a cfg_variant outside 0..2, a variant 1 / 2 with fp16 CFG, x0_out outside mode 1 and an x0_out
    that overlaps any operand, with -1 and a t2v_last_error message, before any launch.  The pointers are fake integers and
    t2v_init is never called; these checks run only without a GPU, so none of these calls can reach a device.
  * The restatement tests/vc_ddim_outputs_oracle.py reproduces every case of tests/golden/vc_ddim_outputs.pt, which
    scripts/make_golden_vc_ddim_outputs.py wrote from the reference's own DDIMSampler.
  * The mirror's process_videocrafter handles the webui's Skip and Interrupt between batches (process_videocrafter.py:59-69)."""
import ctypes as C
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import unet_oracle as UO, vc_oracle as VC

import vc_ddim_outputs_oracle as DO

N = 4 * 4 * 8 * 8
BASE = 0x10000000
X, EC, EU, XO, NZ = (BASE + i * 0x1000000 for i in range(5))
COEFS = (0.9, 0.4, 0.95, 0.3, 0.1)


@pytest.fixture(scope='module')
def gold(gold_dir):
    return torch.load(os.path.join(gold_dir, 'vc_ddim_outputs.pt'))


# ---------------------------------------------------------------------------------------------------------- C ABI
no_gpu = pytest.mark.skipif(torch.cuda.is_available(), reason='argument checks with fake pointers run on CPU only')


def _call(x0_out, variant=0, mode=1, cfg_fp16=0, eps_is_f32=0, noise=NZ, n=N):
    from t2v_b200 import _lib
    l = _lib.load_library()
    p = C.c_void_p
    return l.t2v_ddim_step_ex(p(X), p(EC), p(EU), eps_is_f32, p(XO), n, n // 16, 4, 4, 7.5, mode, *COEFS, p(noise), cfg_fp16,
                              variant, p(x0_out), None), l.t2v_last_error().decode()


@no_gpu
@pytest.mark.parametrize('variant', [-1, 3, 7])
def test_ex_rejects_an_unknown_variant(variant):
    rc, msg = _call(None, variant=variant)
    assert rc == -1 and 'cfg_variant' in msg and str(variant) in msg


@no_gpu
def test_ex_rejects_fp16_cfg_with_variants_1_and_2_and_x0_outside_mode_1():
    for v in (1, 2):
        rc, msg = _call(None, variant=v, cfg_fp16=1)
        assert rc == -1 and 'cfg_fp16' in msg
    rc, msg = _call(BASE + 0x8000000, mode=0)
    assert rc == -1 and 'mode 1' in msg


@no_gpu
@pytest.mark.parametrize('eps_is_f32', [0, 1])
@pytest.mark.parametrize('target,elem', [(X, 4), (XO, 4), (EC, None), (EU, None), (NZ, 4)])
def test_ex_rejects_an_x0_out_that_overlaps_an_operand(target, elem, eps_is_f32):
    elem = elem or (4 if eps_is_f32 else 2)
    last = target + N * elem - 4                  # x0_out's first element on the operand's last 4 bytes
    for x0 in (target, target + 4, last, target - N * 4 + 4):
        rc, msg = _call(x0, eps_is_f32=eps_is_f32)
        assert rc == -1 and 'overlaps' in msg, hex(x0 - target)


# ---------------------------------------------------------------------------------------------------------- restatement
def _rel(a, b):
    return ((a - b).abs().max() / b.abs().max()).item()


@pytest.mark.parametrize('key', DO.CASES)
def test_restatement_matches_the_reference(gold, key):
    cfg = VC.VCConfig(**gold['unet_cfg'])
    W = UO.make_weights(VC.vc_param_specs(cfg), seed=gold['seeds']['unet'])
    img, inter, x0s, steps, forwards = DO.run_case(gold, key, lambda a, b, d: VC.vc_unet_forward(W, cfg, a, b, d),
                                                   gold['c'], gold['uc'])
    ref = gold[key]
    assert steps == ref['sampling_steps'] and forwards == ref['unet_calls'] and (img is None) == ref['interrupted']
    assert len(x0s) == len(ref['x0s']) and all(_rel(a, b) < 1e-5 for a, b in zip(x0s, ref['x0s']))
    if img is not None:
        assert _rel(img, ref['img']) < 1e-5
        for lst in ('x_inter', 'pred_x0'):
            assert len(inter[lst]) == len(ref[lst]) and all(_rel(a, b) < 1e-5 for a, b in zip(inter[lst], ref[lst]))


def test_fixture_pins_the_reference_contract(gold):
    S, stop = gold['S'], gold['stop_at']
    assert gold['a_None']['sampling_steps'] == list(range(S))
    assert gold['d_interrupt']['interrupted'] and gold['d_interrupt']['unet_calls'] == 2 * (stop + 1)
    assert gold['e_skip']['sampling_steps'] == list(range(stop + 1)) and not gold['e_skip']['interrupted']
    # log_every_t = 2 over S = 5 logs indices 4 (the first step), 2 and 0: x_T plus three entries; the skip run stops after
    # index 2, so it logged x_T plus two
    assert len(gold['a_None']['x_inter']) == 4 and len(gold['e_skip']['x_inter']) == 3
    assert all(torch.equal(a, b) for a, b in zip(gold['a_None']['x0s'][:stop + 1], gold['e_skip']['x0s']))
    # the x0 passed to img_callback is the one logged, and the mask does not reach it: case b's first x0 is case a's
    assert torch.equal(gold['a_None']['pred_x0'][1], gold['a_None']['x0s'][0])
    assert torch.equal(gold['b_mask']['x0s'][0], gold['a_None']['x0s'][0])
    assert not torch.equal(gold['a_cfg_ours']['img'], gold['a_None']['img'])
    assert gold['unknown_uc_type_raises']


# ---------------------------------------------------------------------------------------------------------- process_videocrafter
def test_process_videocrafter_skip_and_interrupt_between_batches(monkeypatch):
    from t2v_b200 import videocrafter as V, samplers as S
    log = []

    def fake_sample(model, prompt, n_prompt, n_samples, batch_size, **kw):
        log.append((S.state.job_no, S.state.job, S.state.skipped))
        return np.zeros((n_samples, 1, 1, 1, 1), dtype=np.float32)

    def encoder(clip, a):
        if len(log) == 1:
            S.state.skipped = True                  # Skip pressed during batch 1: batch 2 starts with the flag cleared
        if len(log) == 2:
            S.state.interrupted = True              # Interrupt during batch 2: batch 3 never starts
        return len(log)
    monkeypatch.setattr(V, 'sample_text2video', fake_sample)
    monkeypatch.setattr(V, 'video_encoder', encoder)
    monkeypatch.setattr(V, 'model_cache', None)
    monkeypatch.setattr(S, 'state', SimpleNamespace(interrupted=False, skipped=False, job='', job_no=0, job_count=0))
    out = V.process_videocrafter({'seed': 3, 'batch_count': 3}, model=SimpleNamespace(num_timesteps=1000))
    assert out == [1, 2] and S.state.job_count == 3
    assert log == [(1, 'Batch 1 out of 3', False), (2, 'Batch 2 out of 3', False)]
    assert S.state.job_no == 3 and S.state.interrupted
