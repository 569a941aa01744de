"""TEST INFRASTRUCTURE ONLY -- CPU fp32 restatement of VideoCrafter's DDIM loop with its per-step outputs and webui state
(videocrafter/lvdm/samplers/ddim.py:135-206, p_sample_ddim :208-279):

  * `state.sampling_steps = total`, then per step `state.sampling_step = i` and InterruptedException on `state.interrupted`;
  * `img = postprocess_fn(img, ts)` before the step;
  * the guidance formula of `uc_type` (None / 'cfg_original' / 'cfg_ours', NotImplementedError otherwise) on a guided step;
  * pred_x0 = (x - sqrt(1 - a_t) e_t) / sqrt(a_t) and the update, then the mask blend (tests/vc_masked_oracle.py's q_sample);
  * `callback(i)`, `img_callback(pred_x0, i)`, the intermediates append every `log_every_t` steps and at the last step, and
    `break` on `state.skipped`.

`state` is any object with the webui's flags; `interrupt` is the exception class to raise.  Pinned by
tests/test_vc_ddim_outputs_cpu.py against tests/golden/vc_ddim_outputs.pt, which scripts/make_golden_vc_ddim_outputs.py writes
from the reference's own DDIMSampler.
"""
from types import SimpleNamespace

import numpy as np
import torch

from oracle.samplers_oracle import ddim_schedule, linear_sd_betas

import vc_masked_oracle as MO


@torch.no_grad()
def vc_ddim_sample_outputs(model, betas, x_T, S, cond, uncond, guide_scale, state, interrupt, eta=0.0, noise_gen=None,
                           mask=None, x0=None, q_tape=None, callback=None, img_callback=None, log_every_t=100,
                           postprocess_fn=None, uc_type=None):
    """`model(x, t, c)` = apply_model.  Returns (img, intermediates) as ddim_sampling does."""
    acp = torch.cumprod(1 - betas, dim=0)
    ts, alphas, alphas_prev, sigmas = ddim_schedule(acp, S, eta)
    sqrt_1m = np.sqrt(1.0 - alphas)
    bufs = MO.schedule_buffers(betas)
    img = x_T
    b = img.shape[0]
    size = (b,) + (1,) * (img.dim() - 1)
    total = ts.shape[0]
    noise_gen = torch.Generator(device='cpu') if noise_gen is None else noise_gen
    tape = iter(q_tape or [])
    intermediates = {'x_inter': [img], 'pred_x0': [img]}
    state.sampling_steps = total
    for i, step in enumerate(np.flip(ts)):
        state.sampling_step = i
        if state.interrupted:
            raise interrupt
        index = total - i - 1
        t = torch.full((b,), int(step), dtype=torch.long)
        if postprocess_fn is not None:
            img = postprocess_fn(img, t)
        if uncond is None or guide_scale == 1.0:
            e_t = model(img, t, cond)
        else:
            e_c = model(img, t, cond)
            e_u = model(img, t, uncond)
            if uc_type is None:
                e_t = e_u + guide_scale * (e_c - e_u)
            elif uc_type == 'cfg_original':
                e_t = e_c + guide_scale * (e_c - e_u)
            elif uc_type == 'cfg_ours':
                e_t = e_c + guide_scale * (e_u - e_c)
            else:
                raise NotImplementedError
        a_t = torch.full(size, float(alphas[index]))
        a_prev = torch.full(size, float(alphas_prev[index]))
        sigma_t = torch.full(size, float(sigmas[index]))
        s1m = torch.full(size, float(sqrt_1m[index]))
        pred_x0 = (img - s1m * e_t) / a_t.sqrt()
        dir_xt = (1.0 - a_prev - sigma_t ** 2).sqrt() * e_t
        noise = sigma_t * torch.randn(img.shape, generator=noise_gen) * 1.0
        img = a_prev.sqrt() * pred_x0 + dir_xt + noise
        if mask is not None:
            tq = torch.tensor([int(step) - 1] * x0.shape[0], dtype=torch.long)
            img = MO.q_sample(bufs, x0, tq, next(tape)) * mask + (1. - mask) * img
        if callback is not None:
            callback(i)
        if img_callback is not None:
            img_callback(pred_x0, i)
        if index % log_every_t == 0 or index == total - 1:
            intermediates['x_inter'].append(img)
            intermediates['pred_x0'].append(pred_x0)
        if state.skipped:
            break
    return img, intermediates


def postprocess(img, ts):
    """The fixture's deterministic `postprocess_fn`: a timestep-dependent affine map of the latent."""
    return img * (1.0 - ts.float().view(-1, *([1] * (img.dim() - 1))) * 1e-4) + 0.01


# ------------------------------------------------------------------------------------------- the fixture's cases
CASES = ['a_None', 'a_cfg_original', 'a_cfg_ours', 'b_mask', 'c_post', 'd_interrupt', 'e_skip', 'f_unguided']


def _state():
    return SimpleNamespace(interrupted=False, skipped=False, sampling_step=0, sampling_steps=0)


class _Interrupted(BaseException):
    pass


def run_case(gold, key, model, c, uc, state=None, **extra):
    """Runs the restatement on case `key` of tests/golden/vc_ddim_outputs.pt with `model`; returns (img or None,
    intermediates, img_callback's x0s, state.sampling_step at each callback, denoiser evaluations).  `q_tape=` replaces the
    mask's q_sample draws (by default replayed from the CPU seed, as the reference drew them)."""
    state = _state() if state is None else state
    stop = {'d_interrupt': 'interrupted', 'e_skip': 'skipped'}.get(key)
    spec = dict(S=gold['S'], eta=gold['eta'], scale=gold['scale'])
    kw = {}
    if key.startswith('a_'):
        kw['uc_type'] = gold['uc_types'][[str(u) for u in gold['uc_types']].index(key[2:])]
    elif key == 'b_mask':
        kw.update(mask=gold['mask'], x0=gold['x0'])
    elif key == 'c_post':
        spec, kw['postprocess_fn'] = gold['cases']['post'], postprocess
    elif key == 'f_unguided':
        spec = gold['cases']['unguided']
    kw.update(extra)
    tape = kw.pop('q_tape', None)
    steps, x0s, forwards = [], [], [0]

    def net(a, b, d):
        forwards[0] += a.shape[0]
        return model(a, b, d)

    def cb(i):
        steps.append(state.sampling_step)
        if stop is not None and i == gold['stop_at']:
            setattr(state, stop, True)
    if 'mask' in kw and tape is None:
        torch.manual_seed(gold['seeds']['q'])
        tape = [torch.randn_like(gold['x0']) for _ in range(spec['S'])]
    try:
        img, inter = vc_ddim_sample_outputs(net, linear_sd_betas(), gold['x_T'], spec['S'], c, uc, spec['scale'], state,
                                            _Interrupted, eta=spec['eta'],
                                            noise_gen=torch.Generator('cpu').manual_seed(gold['seeds']['noise']),
                                            q_tape=tape, callback=cb, img_callback=lambda x, i: x0s.append(x),
                                            log_every_t=gold['log_every_t'], **kw)
    except _Interrupted:
        img, inter = None, None
    return img, inter, x0s, steps, forwards[0]
