"""Writes tests/golden/vc_masked.pt from VideoCrafter's own `DDIMSampler` (lvdm/samplers/ddim.py) and `LatentDiffusion`
(lvdm/models/ddpm3d.py), imported through oracle/ref_shim.py and run on CPU fp32 (pytorch_lightning stood in by nn.Module), and
checks the restatement tests/vc_masked_oracle.py against them.  The model is the tiny configuration of
tests/test_videocrafter_gpu.py (UNet model_channels 64, context_dim 48, temporal_length 4; latents of 4 frames x 8x8) with the
full base_t2v VAE; weights are seeded (oracle.unet_oracle.make_weights; the tests regenerate them from the seeds).

Cases (CFG with seeded [1, 9, 48] conditionings, x_T given, the sampler's noise_gen seeded, the global generator seeded
before each run so that the q_sample draws, torch.randn_like(x0) once per step, can be replayed):
  a. frame mask [1,1,4,1,1], the first 2 of 4 frames known, eta 0, S 5, scale 7.5;
  b. region mask [1,1,1,8,8] (the left half known), eta 0.5, S 4, scale 3.0;
  c. timesteps=6 of S 10 from x_T = model.q_sample(x0, t_start), t_start the last step of the prefix, no mask, eta 1.0;
  d. encode_first_stage_2DAE of a seeded [1,3,3,64,64] clip with encode_bs=2 (two chunks of posterior noise);
  e. the number of UNet calls (through `callback`) of sample(S, timesteps=k) for every 1 <= k <= S <= 100 (None where the
     reference's make_schedule raises IndexError: S = 3, 9, 27, 36, 37 put DDIM timestep 1000 past the 1000-entry schedule).
The fixture holds inputs, outputs, shapes and seeds only.

    python scripts/make_golden_vc_masked.py
"""
import os
import sys
import types

import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'tests'))
sys.path.insert(0, ROOT)
from oracle import ref_shim                                   # noqa: E402
from oracle import unet_oracle as UO                          # noqa: E402
from oracle import vae_oracle as VO                           # noqa: E402
from oracle import vc_oracle as VC                            # noqa: E402
from oracle import samplers_oracle as SO                      # noqa: E402
import vc_masked_oracle as MO                                 # noqa: E402
from oracle.make_golden import _SchedModel                    # noqa: E402

SEEDS = {'unet': 4, 'vae_dec': 3, 'vae_enc': 5, 'ctx': 2, 'x_T': 5, 'x0': 7, 'noise': 11, 'q': 13, 'video': 17, 'post': 19, 'q_start': 23}
UNET_CFG = dict(model_channels=64, context_dim=48, temporal_length=4)
SHAPE = (1, 4, 4, 8, 8)
CASES = {'a': dict(S=5, eta=0.0, scale=7.5, mask='frames'), 'b': dict(S=4, eta=0.5, scale=3.0, mask='region'),
         'c': dict(S=10, eta=1.0, scale=7.5, timesteps=6)}
VIDEO_SHAPE, ENCODE_BS = (1, 3, 3, 64, 64), 2


def _install():
    ref_shim.install()
    if 'pytorch_lightning' not in sys.modules:          # ddpm3d imports it; LightningModule is only a base class here
        pl = types.ModuleType('pytorch_lightning')
        pl.LightningModule = nn.Module
        ut = types.ModuleType('pytorch_lightning.utilities')
        ut.rank_zero_only = lambda f: f
        pl.utilities = ut
        sys.modules['pytorch_lightning'], sys.modules['pytorch_lightning.utilities'] = pl, ut


def masks():
    frames = torch.zeros(1, 1, 4, 1, 1)
    frames[:, :, :2] = 1.0
    region = torch.zeros(1, 1, 1, 8, 8)
    region[..., :4] = 1.0
    return {'frames': frames, 'region': region}


def inputs():
    g = torch.Generator('cpu').manual_seed(SEEDS['ctx'])
    c, uc = torch.randn(1, 9, 48, generator=g), torch.randn(1, 9, 48, generator=g)
    x_T = torch.randn(SHAPE, generator=torch.Generator('cpu').manual_seed(SEEDS['x_T']))
    x0 = torch.randn(SHAPE, generator=torch.Generator('cpu').manual_seed(SEEDS['x0']))
    video = torch.rand(VIDEO_SHAPE, generator=torch.Generator('cpu').manual_seed(SEEDS['video'])) * 2 - 1
    return c, uc, x_T, x0, video


def weights():
    Wu = UO.make_weights(VC.vc_param_specs(VC.VCConfig(**UNET_CFG)), seed=SEEDS['unet'])
    Wv = {**UO.make_weights(VO.decoder_param_specs(VO.VAEConfig()), seed=SEEDS['vae_dec']),
          **UO.make_weights(VO.encoder_param_specs(VO.VAEConfig()), seed=SEEDS['vae_enc'])}
    return Wu, Wv


def reference_model():
    from videocrafter.lvdm.models import ddpm3d
    m = ddpm3d.LatentDiffusion(
        unet_config=dict(target='lvdm.models.modules.openaimodel3d.UNetModel', params=dict(
            image_size=32, in_channels=4, out_channels=4, model_channels=64, attention_resolutions=[4, 2, 1], num_res_blocks=2,
            channel_mult=[1, 2, 4, 4], num_heads=8, transformer_depth=1, context_dim=48, use_checkpoint=False, legacy=False,
            kernel_size_t=1, padding_t=0, temporal_length=4, use_relative_position=True)),
        first_stage_config=dict(target='lvdm.models.autoencoder.AutoencoderKL', params=dict(
            embed_dim=4, monitor='val/rec_loss', lossconfig=dict(target='torch.nn.Identity'), ddconfig=dict(
                double_z=True, z_channels=4, resolution=256, in_channels=3, out_ch=3, ch=128, ch_mult=[1, 2, 4, 4],
                num_res_blocks=2, attn_resolutions=[], dropout=0.0))),
        cond_stage_config=None, linear_start=0.00085, linear_end=0.012, num_timesteps_cond=1, log_every_t=200, timesteps=1000,
        first_stage_key='video', cond_stage_key='caption', image_size=[8, 8], video_length=4, channels=4,
        cond_stage_trainable=False, conditioning_key='crossattn', scale_by_std=False, scale_factor=0.18215)
    m.device = torch.device('cpu')           # a LightningModule property the sampler reads
    Wu, Wv = weights()
    res = m.load_state_dict({**{'model.diffusion_model.' + k: v for k, v in Wu.items()},
                             **{'first_stage_model.' + k: v for k, v in Wv.items()}}, strict=False)
    assert not res.unexpected_keys and all(not k.startswith(('model.', 'first_stage_model.')) for k in res.missing_keys), res
    return m.eval(), Wu, Wv


def main():
    _install()
    from videocrafter.lvdm.samplers.ddim import DDIMSampler
    DDIMSampler.register_buffer = lambda self, name, attr: setattr(self, name, attr)    # ddim.py:22-26 hard-codes "cuda"
    m, Wu, Wv = reference_model()
    cfg = VC.VCConfig(**UNET_CFG)
    betas = SO.linear_sd_betas()
    bufs = MO.schedule_buffers(betas)
    assert torch.equal(bufs[0], m.sqrt_alphas_cumprod) and torch.equal(bufs[1], m.sqrt_one_minus_alphas_cumprod)
    c, uc, x_T, x0, video = inputs()
    M = masks()
    out = {'seeds': SEEDS, 'unet_cfg': UNET_CFG, 'shape': SHAPE, 'cases': CASES, 'video_shape': VIDEO_SHAPE,
           'encode_bs': ENCODE_BS, 'masks': M, 'c': c, 'uc': uc, 'x_T': x_T, 'x0': x0}
    net = lambda a, b, d: VC.vc_unet_forward(Wu, cfg, a, b, d)                 # noqa: E731
    for name, case in CASES.items():
        smp = DDIMSampler(m)
        smp.noise_gen.manual_seed(SEEDS['noise'])
        kw = {}
        start = x_T
        if 'mask' in case:
            kw = dict(mask=M[case['mask']], x0=x0)
        else:
            smp.make_schedule(case['S'], ddim_eta=case['eta'], verbose=False)
            t_start = int(MO.ddim_prefix(smp.ddim_timesteps, case['timesteps'])[-1])
            torch.manual_seed(SEEDS['q_start'])
            start = m.q_sample(x0, torch.tensor([t_start]))
            out['t_start'], out['x_T_c'] = t_start, start
            kw = dict(timesteps=case['timesteps'])
        calls = []
        torch.manual_seed(SEEDS['q'])
        with torch.no_grad():
            r, _ = smp.sample(S=case['S'], batch_size=1, shape=SHAPE[1:], conditioning=c, x_T=start, verbose=False, eta=case['eta'],
                              unconditional_guidance_scale=case['scale'], unconditional_conditioning=uc,
                              callback=calls.append, **kw)
        torch.manual_seed(SEEDS['q'])
        tape = [torch.randn_like(x0) for _ in calls] if 'mask' in case else None
        o = MO.vc_ddim_sample_masked(net, betas, start, case['S'], c, uc, case['scale'], eta=case['eta'],
                                     noise_gen=torch.Generator('cpu').manual_seed(SEEDS['noise']),
                                     mask=kw.get('mask'), x0=x0, q_tape=tape, timesteps=case.get('timesteps'))
        err = (r - o).abs().max().item()
        print(f'[{name}] {len(calls)} steps, absmax {r.abs().max().item():.3f}; restatement-vs-reference max|d| = {err:.3e}')
        assert err < 1e-5 * max(1.0, r.abs().max().item())
        out['out_' + name], out['steps_' + name] = r, len(calls)

    torch.manual_seed(SEEDS['post'])
    with torch.no_grad():
        z = m.encode_first_stage_2DAE(video, encode_bs=ENCODE_BS)
    n = VIDEO_SHAPE[0] * VIDEO_SHAPE[2]
    tape = MO.posterior_tape(SEEDS['post'], n, ENCODE_BS, (4, VIDEO_SHAPE[3] // 8, VIDEO_SHAPE[4] // 8))
    o = MO.encode_first_stage_2DAE(Wv, video, ENCODE_BS, tape)
    err = (z - o).abs().max().item()
    print(f'[encode] {tuple(z.shape)}, absmax {z.abs().max().item():.3f}; restatement-vs-reference max|d| = {err:.3e}')
    assert err < 1e-5 * max(1.0, z.abs().max().item())
    out['z'] = z.contiguous()                # the clip is regenerated from its seed

    class _Zero(_SchedModel):                 # the step count does not depend on the network
        def apply_model(self, xx, tt, cc, **kw):
            return torch.zeros_like(xx)
    steps = {}
    for S in range(1, 101):
        smp = DDIMSampler(_Zero(betas))
        for k in range(1, S + 1):
            calls = []
            try:
                smp.sample(S=S, batch_size=1, shape=(1, 1, 1, 1), conditioning=None, x_T=torch.zeros(1, 1, 1, 1, 1),
                           verbose=False, callback=calls.append, timesteps=k)
            except IndexError:                 # 999 in range(0, 1000, 1000 // S): ddim timestep 1000 is out of the schedule
                calls = None
            steps[(k, S)] = None if calls is None else len(calls)
    bad = sorted({S for (k, S), v in steps.items() if v is None})
    print(f'[timesteps] {len(steps)} (k, S) pairs; (6, 10): {steps[(6, 10)]}, (15, 22): {steps[(15, 22)]}, '
          f'(15, 21): {steps[(15, 21)]}; S whose schedule raises IndexError: {bad}')
    out['prefix_steps'] = steps
    path = os.path.join(ROOT, 'tests', 'golden', 'vc_masked.pt')
    torch.save(out, path)
    print(f'wrote {path} ({os.path.getsize(path) / 1e3:.0f} kB)')


if __name__ == '__main__':
    main()
