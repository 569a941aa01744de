"""GPU: VideoCrafter's per-step DDIM outputs on the library.

  * op level: t2v_ddim_step_ex's x_{t-1} and x0 bit for bit against torch's fp32 ops for every cfg_variant (uc_type), eta 0 and
    > 0, fp16 and fp32 eps, at ragged sizes; variant 0 without x0 bit for bit against t2v_ddim_step;
  * model level: the tiny VideoCrafter model's `DDIMSampler.sample` (img_callback, intermediates, uc_type, mask,
    postprocess_fn, webui Interrupt / Skip / progress) against the CPU restatement tests/vc_ddim_outputs_oracle.py, which
    tests/test_vc_ddim_outputs_cpu.py pins to the reference, on the gates tests/test_vc_masked_gpu.py uses for this model;
  * process_videocrafter with batch_count 3: Skip moves to the next batch, Interrupt stops the run."""
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import unet_oracle as UO, vae_oracle as VO, vc_oracle as VC

import vc_ddim_outputs_oracle as DO
from parity_util import report

pytestmark = pytest.mark.gpu

GATE = 5e-3                      # max |d| / max |ref| of tests/test_vc_masked_gpu.py's sampler cases
COEFS = tuple(float(np.float32(v)) for v in (0.9, 0.4, 0.95, 0.3, 0.1))     # fp32 values, as the sampler passes


@pytest.fixture(scope='module')
def gold(gold_dir):
    return torch.load(os.path.join(gold_dir, 'vc_ddim_outputs.pt'))


@pytest.fixture()
def state(monkeypatch):
    from t2v_b200 import samplers as S
    st = SimpleNamespace(interrupted=False, skipped=False, sampling_step=0, sampling_steps=0, job='', job_no=0, job_count=0)
    monkeypatch.setattr(S, 'state', st)
    return st


# ---------------------------------------------------------------------------------------------------------- kernel
def _torch_step(x, ec, eu, g, variant, a, noise):
    """p_sample_ddim in torch's fp32 ops (ddim.py:233-277), every channel guided.  Run on the CPU: torch's CUDA division by a
    Python scalar multiplies by the reciprocal, where the reference divides by a tensor."""
    c = ec.float()
    if eu is None:
        e = c
    else:
        u = eu.float()
        e = [u + g * (c - u), c + g * (c - u), c + g * (u - c)][variant]
    x0 = (x - a[0] * e) / a[1]
    xn = a[2] * x0 + a[3] * e
    xn = xn + a[4] * noise if a[4] != 0.0 else xn + 0.0
    return xn, x0


def _bits(t):
    return t.contiguous().view(torch.int32)


@pytest.mark.parametrize('shape', [(1, 4, 3, 7, 9), (3, 4, 5, 11, 13)])
@pytest.mark.parametrize('eps_dtype', [torch.float16, torch.float32])
@pytest.mark.parametrize('eta', [0.0, 0.5])
@pytest.mark.parametrize('variant', [0, 1, 2])
def test_step_ex_is_bit_identical_to_torch(shape, eps_dtype, eta, variant):
    from t2v_b200 import samplers as S
    g = torch.Generator('cuda').manual_seed(7)
    x = torch.randn(shape, device='cuda', generator=g)
    ec = torch.randn(shape, device='cuda', generator=g).to(eps_dtype)
    eu = torch.randn(shape, device='cuda', generator=g).to(eps_dtype)
    noise = torch.randn(shape, device='cuda', generator=g)
    a = COEFS[:4] + ((COEFS[4] if eta > 0 else 0.0),)
    out, x0 = S._step_kernel_ex(x, ec, eu, 7.5, shape[1], 1, a, noise, cfg_fp16=False, cfg_variant=variant, want_x0=True)
    ref, ref_x0 = _torch_step(x.cpu(), ec.cpu(), eu.cpu(), 7.5, variant, a, noise.cpu())
    assert torch.equal(_bits(out.cpu()), _bits(ref)) and torch.equal(_bits(x0.cpu()), _bits(ref_x0))
    plain, none = S._step_kernel_ex(x, ec, eu, 7.5, shape[1], 1, a, noise, cfg_fp16=False, cfg_variant=variant)
    assert none is None and torch.equal(_bits(plain), _bits(out))          # the x0 store changes nothing else
    if variant == 0:
        old = S._step_kernel(x, ec, eu, 7.5, shape[1], 1, a, noise, cfg_fp16=False)
        assert torch.equal(_bits(plain), _bits(old))
    # unguided: no CFG whatever the variant
    u, u0 = S._step_kernel_ex(x, ec, None, 1.0, shape[1], 1, a, noise, cfg_fp16=False, cfg_variant=variant, want_x0=True)
    ref_u, ref_u0 = _torch_step(x.cpu(), ec.cpu(), None, 1.0, 0, a, noise.cpu())
    assert torch.equal(_bits(u.cpu()), _bits(ref_u)) and torch.equal(_bits(u0.cpu()), _bits(ref_u0))


@pytest.mark.parametrize('mode,cfg_fp16,gch', [(0, 0, 2), (0, 1, 2), (1, 1, 4), (1, 0, 3)])
def test_step_ex_variant_0_without_x0_is_t2v_ddim_step(mode, cfg_fp16, gch):
    """Every mode / CFG rounding of the old entry point, through the new one."""
    from t2v_b200 import samplers as S
    g = torch.Generator('cuda').manual_seed(11)
    shape = (2, 4, 3, 5, 7)
    x, noise = torch.randn(shape, device='cuda', generator=g), torch.randn(shape, device='cuda', generator=g)
    ec, eu = (torch.randn(shape, device='cuda', generator=g).half() for _ in range(2))
    old = S._step_kernel(x, ec, eu, 9.0, gch, mode, COEFS, noise, cfg_fp16=bool(cfg_fp16))
    new, _ = S._step_kernel_ex(x, ec, eu, 9.0, gch, mode, COEFS, noise, cfg_fp16=bool(cfg_fp16))
    assert torch.equal(_bits(new), _bits(old))


def test_step_ex_rejects_bad_arguments_before_launch():
    from t2v_b200 import _lib
    l = _lib.lib()
    x = torch.randn(2, 4, 3, 5, 7, device='cuda')
    ec = torch.randn_like(x).half()
    out = torch.full_like(x, 7.0)
    n = x.numel()

    def call(x0, variant=0, mode=1, cfg_fp16=0):
        rc = l.t2v_ddim_step_ex(_lib.ptr(x), _lib.ptr(ec), None, 0, _lib.ptr(out), n, n // 8, 4, 4, 7.5, mode, *COEFS[:4], 0.0,
                                None, cfg_fp16, variant, _lib.ptr(x0), _lib.stream_ptr())
        return rc, l.t2v_last_error().decode()
    assert call(None, variant=3)[0] == -1 and 'cfg_variant' in call(None, variant=3)[1]
    assert call(None, variant=1, cfg_fp16=1)[0] == -1
    assert call(torch.empty_like(x), mode=0)[0] == -1
    for x0 in (x, out, x[1:], ec.flatten()[2:].view(torch.float32)):
        rc, msg = call(x0)
        assert rc == -1 and 'overlaps' in msg
    torch.cuda.synchronize()
    assert (out == 7.0).all()                     # nothing was launched


# ---------------------------------------------------------------------------------------------------------- model level
@pytest.fixture(scope='module')
def ldm(gold):
    from t2v_b200.videocrafter import LatentDiffusion
    cfg = VC.VCConfig(**gold['unet_cfg'])
    W = UO.make_weights(VC.vc_param_specs(cfg), seed=gold['seeds']['unet'])
    m = LatentDiffusion(unet_config=dict(gold['unet_cfg']), image_size=[8, 8], video_length=4)
    m.model.half()
    m.first_stage_model.half()
    m.model.diffusion_model.load_state_dict(W, strict=True)
    m.first_stage_model.load_state_dict({**UO.make_weights(VO.decoder_param_specs(VO.VAEConfig()), seed=gold['seeds']['vae_dec']),
                                         **UO.make_weights(VO.encoder_param_specs(VO.VAEConfig()), seed=gold['seeds']['vae_enc'])},
                                        strict=True)                    # process_videocrafter decodes
    return m.cuda().eval(), cfg, {k: v.half().float() for k, v in W.items()}


def _mirror(m, gold, key, state, monkeypatch, q_seed=1234, **extra):
    """The library's run of fixture case `key`: (img or None, intermediates, x0s, steps, forwards, q tape)."""
    from t2v_b200.videocrafter import DDIMSampler
    from t2v_b200 import samplers as S
    stop = {'d_interrupt': 'interrupted', 'e_skip': 'skipped'}.get(key)
    spec = dict(S=gold['S'], eta=gold['eta'], scale=gold['scale'])
    kw = {}
    if key.startswith('a_'):
        kw['uc_type'] = gold['uc_types'][[str(u) for u in gold['uc_types']].index(key[2:])]
    elif key == 'b_mask':
        kw.update(mask=gold['mask'], x0=gold['x0'].cuda())
    elif key == 'c_post':
        spec, kw['postprocess_fn'] = gold['cases']['post'], DO.postprocess
    elif key == 'f_unguided':
        spec = gold['cases']['unguided']
    kw.update(extra)
    forwards = [0]
    apply_model = m.apply_model

    def counting(x, *a, **k):
        forwards[0] += x.shape[0]                  # cond and uncond run as one B = 2 forward: two evaluations
        return apply_model(x, *a, **k)
    monkeypatch.setattr(m, 'apply_model', counting)
    steps, x0s = [], []

    def cb(i):
        steps.append(state.sampling_step)
        if stop is not None and i == gold['stop_at']:
            setattr(state, stop, True)
    smp = DDIMSampler(m)
    smp.noise_gen.manual_seed(gold['seeds']['noise'])
    torch.cuda.manual_seed(q_seed)
    try:
        img, inter = smp.sample(S=spec['S'], batch_size=1, shape=gold['shape'][1:], conditioning=gold['c'].half().float().cuda(),
                                unconditional_conditioning=gold['uc'].half().float().cuda(),
                                unconditional_guidance_scale=spec['scale'], eta=spec['eta'], verbose=False, x_T=gold['x_T'].cuda(),
                                callback=cb, img_callback=lambda x, i: x0s.append(x), log_every_t=gold['log_every_t'], **kw)
    except S.InterruptedException:
        img, inter = None, None
    finally:
        monkeypatch.setattr(m, 'apply_model', apply_model)
    tape = None
    if 'mask' in kw:
        torch.cuda.manual_seed(q_seed)
        tape = [torch.randn_like(gold['x0'].cuda()).cpu() for _ in range(spec['S'])]
    return img, inter, x0s, steps, forwards[0], tape


def _rel(a, b):
    return float((a.cpu() - b).abs().max() / b.abs().max())


@pytest.mark.parametrize('key', DO.CASES)
def test_sampler_outputs_vs_restatement(ldm, gold, state, monkeypatch, key):
    m, cfg, Wh = ldm
    img, inter, x0s, steps, forwards, tape = _mirror(m, gold, key, state, monkeypatch)
    ref = gold[key]
    assert steps == ref['sampling_steps'] and forwards == ref['unet_calls'] and (img is None) == ref['interrupted']
    assert state.sampling_steps == {'c_post': 4, 'f_unguided': 4}.get(key, gold['S'])        # the progress bar's total
    rs = DO.run_case(gold, key, lambda a, b, d: VC.vc_unet_forward(Wh, cfg, a, b, d), gold['c'].half().float(),
                     gold['uc'].half().float(), q_tape=tape)                    # tape: the library's q_sample draws
    assert len(x0s) == len(rs[2]) == len(ref['x0s'])
    errs = [_rel(a, b) for a, b in zip(x0s, rs[2])]
    assert len({t.data_ptr() for t in x0s}) == len(x0s) and all(t.dtype == torch.float32 and t.is_cuda for t in x0s)
    if img is not None:
        errs.append(_rel(img, rs[0]))
        assert torch.equal(inter['x_inter'][-1], img)
        assert len(inter['pred_x0']) == len(rs[1]['pred_x0']) and len(inter['x_inter']) == len(rs[1]['x_inter'])
        logged = [i for i in range(len(x0s)) if any(p is x0s[i] for p in inter['pred_x0'])]
        assert len(logged) == len(inter['pred_x0']) - 1              # every logged x0 is the one img_callback got
        errs += [_rel(a, b) for a, b in zip(inter['x_inter'][1:], rs[1]['x_inter'][1:])]
    report(f'vc_ddim_outputs:{key}', max=max(errs))
    assert max(errs) < GATE, errs


def test_x0_is_only_written_when_asked(ldm, gold, state, monkeypatch):
    """No img_callback: x0 only on the logged steps; log_every_t = 100 over 5 steps logs the first and the last."""
    from t2v_b200 import samplers as S, videocrafter as V
    m = ldm[0]
    asked = []
    orig = S._step_kernel_ex
    monkeypatch.setattr(V, '_step_kernel_ex', lambda *a, **k: asked.append(k['want_x0']) or orig(*a, **k))
    smp = V.DDIMSampler(m)
    out, inter = smp.sample(S=5, batch_size=1, shape=gold['shape'][1:], conditioning=gold['c'].half().float().cuda(),
                            unconditional_conditioning=gold['uc'].half().float().cuda(), unconditional_guidance_scale=7.5,
                            eta=0.0, x_T=gold['x_T'].cuda(), log_every_t=100)
    assert asked == [True, False, False, False, True] and len(inter['pred_x0']) == 3


def test_uc_type_errors_and_unguided_runs(ldm, gold, state, monkeypatch):
    m = ldm[0]
    base = _mirror(m, gold, 'f_unguided', state, monkeypatch)[0]
    for u in ('cfg_ours', 'not a uc_type'):
        assert torch.equal(_mirror(m, gold, 'f_unguided', state, monkeypatch, uc_type=u)[0], base)
    with pytest.raises(NotImplementedError):
        _mirror(m, gold, 'a_None', state, monkeypatch, uc_type='not a uc_type')


# ---------------------------------------------------------------------------------------------------------- webui batch loop
def _process(m, monkeypatch, on_forward):
    from t2v_b200 import videocrafter as vcm
    g = torch.Generator('cpu').manual_seed(2)
    c, uc = torch.randn(1, 9, 48, generator=g).half().float(), torch.randn(1, 9, 48, generator=g).half().float()
    x_T = torch.randn((1, 4, 4, 8, 8), generator=torch.Generator('cpu').manual_seed(9)).cuda()
    calls = [0]
    apply_model = m.apply_model

    def counting(*a, **k):
        calls[0] += 1
        on_forward(calls[0])
        return apply_model(*a, **k)
    monkeypatch.setattr(m, 'apply_model', counting)
    monkeypatch.setattr(vcm, 'video_encoder', None)
    try:
        out = vcm.process_videocrafter(dict(prompt_embeds=c.cuda(), n_prompt_embeds=uc.cuda(), steps=4, frames=4, seed=3,
                                            cfg_scale=4.0, eta=0.0, batch_count=3, x_T=x_T), model=m)
    finally:
        monkeypatch.setattr(m, 'apply_model', apply_model)
    return out, calls[0]


def test_process_videocrafter_skip_and_interrupt(ldm, state, monkeypatch):
    from t2v_b200 import samplers as S
    m = ldm[0]
    plain, n = _process(m, monkeypatch, lambda k: None)
    assert len(plain) == 3 and n == 12 and state.job_count == 3 and state.job == 'Batch 3 out of 3'

    def skip(k):
        if k == 2:
            state.skipped = True                  # during batch 1's second step: it ends after that step
    out, n = _process(m, monkeypatch, skip)
    assert n == 2 + 4 + 4 and len(out) == 3 and not state.skipped
    assert not np.array_equal(out[0], plain[0]) and np.array_equal(out[1], plain[1]) and np.array_equal(out[2], plain[2])

    def interrupt(k):
        if k == 6:
            state.interrupted = True              # during batch 2's second step: the next step raises
    with pytest.raises(S.InterruptedException):
        _process(m, monkeypatch, interrupt)
    assert state.job_no == 2 and state.sampling_step == 2
