"""CPU: VideoCrafter's masked / truncated DDIM and encode_first_stage_2DAE.  The restatement tests/vc_masked_oracle.py is pinned
to tests/golden/vc_masked.pt, which the reference's own DDIMSampler / LatentDiffusion wrote (scripts/make_golden_vc_masked.py),
and the mirror's `timesteps=k` prefix (t2v_b200/videocrafter.py DDIMSampler.timestep_prefix) is checked against the step
counts the reference ran for every 1 <= k <= S <= 100."""
import os
from types import SimpleNamespace

import pytest
import torch

from oracle import unet_oracle as UO, vae_oracle as VO, vc_oracle as VC, samplers_oracle as SO

import vc_masked_oracle as MO


@pytest.fixture(scope='module')
def gold(gold_dir):
    return torch.load(os.path.join(gold_dir, 'vc_masked.pt'))


def _rel(a, b):
    return ((a - b).abs().max() / b.abs().max()).item()


@pytest.mark.parametrize('case', ['a', 'b', 'c'])
def test_restatement_matches_the_reference(gold, case):
    cfg = VC.VCConfig(**gold['unet_cfg'])
    W = UO.make_weights(VC.vc_param_specs(cfg), seed=gold['seeds']['unet'])
    spec = gold['cases'][case]
    mask = gold['masks'][spec['mask']] if 'mask' in spec else None
    x_T = gold['x_T'] if mask is not None else gold['x_T_c']
    calls = []
    torch.manual_seed(gold['seeds']['q'])
    tape = [torch.randn_like(gold['x0']) for _ in range(gold['steps_' + case])] if mask is not None else None
    out = MO.vc_ddim_sample_masked(lambda a, b, d: VC.vc_unet_forward(W, cfg, a, b, d), SO.linear_sd_betas(), x_T, spec['S'],
                                   gold['c'], gold['uc'], spec['scale'], eta=spec['eta'],
                                   noise_gen=torch.Generator('cpu').manual_seed(gold['seeds']['noise']), mask=mask, x0=gold['x0'],
                                   q_tape=tape, timesteps=spec.get('timesteps'), callback=calls.append)
    assert len(calls) == gold['steps_' + case]
    assert _rel(out, gold['out_' + case]) < 1e-5


def test_q_sample_start_matches_the_reference(gold):
    torch.manual_seed(gold['seeds']['q_start'])
    bufs = MO.schedule_buffers(SO.linear_sd_betas())
    x = MO.q_sample(bufs, gold['x0'], torch.tensor([gold['t_start']]), torch.randn_like(gold['x0']))
    assert torch.equal(x, gold['x_T_c'])


def test_encode_first_stage_2DAE_restatement_matches_the_reference(gold):
    W = {**UO.make_weights(VO.decoder_param_specs(VO.VAEConfig()), seed=gold['seeds']['vae_dec']),
         **UO.make_weights(VO.encoder_param_specs(VO.VAEConfig()), seed=gold['seeds']['vae_enc'])}
    b, _, t, H, Wd = gold['video_shape']
    video = torch.rand(gold['video_shape'], generator=torch.Generator('cpu').manual_seed(gold['seeds']['video'])) * 2 - 1
    tape = MO.posterior_tape(gold['seeds']['post'], b * t, gold['encode_bs'], (4, H // 8, Wd // 8))
    assert [n.shape[0] for n in tape] == [2, 1]
    z = MO.encode_first_stage_2DAE(W, video, gold['encode_bs'], tape)
    assert z.shape == gold['z'].shape and _rel(z, gold['z']) < 1e-5


def test_mirror_timestep_prefix_matches_the_reference_for_every_k_and_S(gold):
    from t2v_b200.videocrafter import DDIMSampler
    acp = torch.cumprod(1 - SO.linear_sd_betas(), 0).float()
    smp = DDIMSampler(SimpleNamespace(num_timesteps=1000, alphas_cumprod=acp))
    steps = gold['prefix_steps']
    assert len(steps) == 5050
    for S in range(1, 101):
        if steps[(1, S)] is None:                # the reference's schedule indexes past the table at this S: so does the mirror
            with pytest.raises(IndexError):
                smp.make_schedule(S)
            continue
        smp.make_schedule(S)
        for k in range(1, S + 1):
            assert smp.timestep_prefix(k).shape[0] == steps[(k, S)], (k, S)
            assert smp.timestep_prefix(k).shape[0] == MO.ddim_prefix(smp.ddim_timesteps, k).shape[0]
    # the prefix is taken over the n DDIM timesteps (n > S when S does not divide 1000), in float64: S = 22 has n = 23, so
    # k = S runs S - 1 steps; k / n * n can round below k, e.g. (15, 21) runs 13 steps, not 14
    assert (steps[(6, 10)], steps[(15, 22)], steps[(22, 22)], steps[(15, 21)]) == (5, 14, 21, 13)
    assert all(steps[(1, S)] in (0, None) for S in range(1, 101))
    assert sum(1 for (k, S), v in steps.items() if v is not None and v == k - 2) > 0


def test_mirror_q_sample_coefficients_are_the_reference_buffers_in_fp32():
    """register_schedule's fp32 values, also after .half() (load_model), which rounds the module's own buffers."""
    from t2v_b200.videocrafter import LatentDiffusion
    m = LatentDiffusion(unet_config=dict(model_channels=64, context_dim=48, temporal_length=4), image_size=[8, 8], video_length=4)
    ref = MO.schedule_buffers(SO.linear_sd_betas())
    assert torch.equal(m.sqrt_alphas_cumprod, ref[0]) and torch.equal(m.sqrt_one_minus_alphas_cumprod, ref[1])
    m = m.half()
    assert m.sqrt_alphas_cumprod.dtype == torch.float16
    got = m.q_coefficients('cpu')
    assert got[0].dtype == torch.float32 and torch.equal(got[0], ref[0]) and torch.equal(got[1], ref[1])
