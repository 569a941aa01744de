"""Writes tests/golden/vc_ddim_outputs.pt from VideoCrafter's own `DDIMSampler` (lvdm/samplers/ddim.py) and `LatentDiffusion`,
run on CPU fp32 through oracle/ref_shim.py, and checks the restatement tests/vc_ddim_outputs_oracle.py against them.  The model,
weights, conditionings, x_T, x0 and frame mask are those of scripts/make_golden_vc_masked.py (UNet model_channels 64,
context_dim 48, temporal_length 4; 4 frames x 8x8 latents; seeded weights the tests regenerate).

Cases (the sampler's noise_gen seeded, the global generator seeded before each run for the mask's q_sample draws):
  a. uc_type None / 'cfg_original' / 'cfg_ours', S 5, eta 0.5, scale 7.5, log_every_t 2: every img_callback x0, both
     intermediates lists, the final latent and the state.sampling_step seen by each callback;
  b. the frame mask (first 2 of 4 frames known) with img_callback, S 5, eta 0.5, scale 7.5: x0 is taken before the blend;
  c. a deterministic postprocess_fn (vc_ddim_outputs_oracle.postprocess), S 4, eta 0.5, scale 3.0;
  d. state.interrupted set by `callback` at step 2 of case a (None): InterruptedException, and the UNet calls made;
  e. state.skipped set by `callback` at step 2 of case a (None): the early result, the intermediates and the steps run;
  f. an unguided run (scale 1.0) with uc_type 'cfg_ours' and with an unknown uc_type, against uc_type None; and the
     NotImplementedError an unknown uc_type raises on a guided run.
The fixture holds inputs, outputs and seeds only.

    python scripts/make_golden_vc_ddim_outputs.py
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
import make_golden_vc_masked as VM                            # noqa: E402  (puts tests/ and the repository on sys.path)
from oracle import vc_oracle as VC                            # noqa: E402
from oracle import samplers_oracle as SO                      # noqa: E402
import vc_ddim_outputs_oracle as DO                           # noqa: E402

S, ETA, SCALE, LOG_EVERY = 5, 0.5, 7.5, 2
UC_TYPES = [None, 'cfg_original', 'cfg_ours']
CASES = {'post': dict(S=4, eta=0.5, scale=3.0), 'unguided': dict(S=4, eta=0.5, scale=1.0)}
STOP_AT = 2


def _rel(a, b):
    return ((a - b).abs().max() / b.abs().max().clamp_min(1e-30)).item()


def _check(name, got, want):
    err = _rel(got, want)
    assert err < 1e-5, (name, err)
    return err


def main():
    VM._install()
    from videocrafter.lvdm.samplers.ddim import DDIMSampler
    from modules.shared import state
    from modules.sd_samplers_common import InterruptedException
    DDIMSampler.register_buffer = lambda self, name, attr: setattr(self, name, attr)    # ddim.py:22-26 hard-codes "cuda"
    m, Wu, _ = VM.reference_model()
    cfg = VC.VCConfig(**VM.UNET_CFG)
    betas = SO.linear_sd_betas()
    c, uc, x_T, x0, _ = VM.inputs()
    frames = VM.masks()['frames']
    net = lambda a, b, d: VC.vc_unet_forward(Wu, cfg, a, b, d)                 # noqa: E731
    unet_calls = [0]
    apply_model = m.apply_model

    def counting(*a, **k):
        unet_calls[0] += 1
        return apply_model(*a, **k)
    m.apply_model = counting

    def reset():
        state.interrupted = state.skipped = False
        state.sampling_step = state.sampling_steps = 0
        unet_calls[0] = 0

    def run(sampler_fn, s, eta, scale, stop=None, **kw):
        """Runs sampler_fn (the reference's sample or the restatement) with a callback that records state.sampling_step and
        sets `stop` ('interrupted' / 'skipped') at step STOP_AT; returns (img, intermediates, x0s, steps, error)."""
        reset()
        steps, x0s = [], []

        def cb(i):
            steps.append(state.sampling_step)
            if stop is not None and i == STOP_AT:
                setattr(state, stop, True)
        torch.manual_seed(VM.SEEDS['q'])
        try:
            img, inter = sampler_fn(s, eta, scale, cb, lambda x, i: x0s.append(x), **kw)
        except InterruptedException:
            img, inter = None, None
        return img, inter, x0s, steps

    def ref(s, eta, scale, cb, icb, **kw):
        smp = DDIMSampler(m)
        smp.noise_gen.manual_seed(VM.SEEDS['noise'])
        return smp.sample(S=s, batch_size=1, shape=VM.SHAPE[1:], conditioning=c, x_T=x_T, verbose=False, eta=eta,
                          unconditional_guidance_scale=scale, unconditional_conditioning=uc, callback=cb, img_callback=icb,
                          log_every_t=LOG_EVERY, **kw)

    def restated(s, eta, scale, cb, icb, mask=None, x0=None, **kw):
        tape = None
        if mask is not None:
            torch.manual_seed(VM.SEEDS['q'])
            tape = [torch.randn_like(x0) for _ in range(s)]
        return DO.vc_ddim_sample_outputs(net, betas, x_T, s, c, uc, scale, state, InterruptedException, eta=eta,
                                         noise_gen=torch.Generator('cpu').manual_seed(VM.SEEDS['noise']), mask=mask, x0=x0,
                                         q_tape=tape, callback=cb, img_callback=icb, log_every_t=LOG_EVERY, **kw)

    out = {'seeds': VM.SEEDS, 'unet_cfg': VM.UNET_CFG, 'shape': VM.SHAPE, 'c': c, 'uc': uc, 'x_T': x_T, 'x0': x0, 'mask': frames,
           'S': S, 'eta': ETA, 'scale': SCALE, 'log_every_t': LOG_EVERY, 'stop_at': STOP_AT, 'cases': CASES, 'uc_types': UC_TYPES}

    def record(key, s, eta, scale, stop=None, **kw):
        r = run(ref, s, eta, scale, stop, **kw)
        calls = unet_calls[0]
        o = run(restated, s, eta, scale, stop, **kw)
        assert r[3] == o[3] and len(r[2]) == len(o[2]), key
        errs = [_check(key + ':x0', a, b) for a, b in zip(r[2], o[2])]
        if r[0] is not None:
            errs.append(_check(key + ':img', r[0], o[0]))
            for lst in ('x_inter', 'pred_x0'):
                assert len(r[1][lst]) == len(o[1][lst])
                errs += [_check(key + ':' + lst, a, b) for a, b in zip(r[1][lst], o[1][lst])]
        else:
            assert o[0] is None, key
        print(f'[{key}] {len(r[3])} steps, {calls} UNet calls, raised: {r[0] is None}; restatement max rel. err. {max(errs):.2e}')
        out[key] = {'img': r[0], 'x0s': r[2], 'sampling_steps': r[3], 'unet_calls': calls, 'interrupted': r[0] is None,
                    'x_inter': None if r[1] is None else r[1]['x_inter'], 'pred_x0': None if r[1] is None else r[1]['pred_x0']}

    for u in UC_TYPES:
        record(f'a_{u}', S, ETA, SCALE, uc_type=u)
    record('b_mask', S, ETA, SCALE, mask=frames, x0=x0)
    record('c_post', CASES['post']['S'], CASES['post']['eta'], CASES['post']['scale'], postprocess_fn=DO.postprocess)
    record('d_interrupt', S, ETA, SCALE, stop='interrupted')
    record('e_skip', S, ETA, SCALE, stop='skipped')
    u = CASES['unguided']
    record('f_unguided', u['S'], u['eta'], u['scale'])
    for name, kind in (('cfg_ours', 'cfg_ours'), ('bogus', 'not a uc_type')):
        r = run(ref, u['S'], u['eta'], u['scale'], uc_type=kind)
        assert torch.equal(r[0], out['f_unguided']['img']), name            # an unguided run never reads uc_type
    try:
        run(ref, 2, ETA, SCALE, uc_type='not a uc_type')
        raise AssertionError('a guided run with an unknown uc_type did not raise')
    except NotImplementedError:
        out['unknown_uc_type_raises'] = True
    reset()
    path = os.path.join(VM.ROOT, 'tests', 'golden', 'vc_ddim_outputs.pt')
    torch.save(out, path)
    print(f'wrote {path} ({os.path.getsize(path) / 1e3:.0f} kB)')


if __name__ == '__main__':
    main()
