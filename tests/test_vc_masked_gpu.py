"""GPU: VideoCrafter's masked / truncated DDIM on the library -- the t2v_q_sample_blend kernel bit for bit against torch's fp32
ops, `DDIMSampler.sample(mask=, x0=, timesteps=)` / `LatentDiffusion.q_sample` / `encode_first_stage_2DAE` against the CPU
restatement tests/vc_masked_oracle.py (pinned to the reference by tests/test_vc_masked_cpu.py), replaying the library's
q_sample draws from the re-seeded CUDA generator."""
import os

import pytest
import torch

from oracle import unet_oracle as UO, vae_oracle as VO, vc_oracle as VC, samplers_oracle as SO

import vc_masked_oracle as MO
from parity_util import errs, report

pytestmark = pytest.mark.gpu

RMS_GATE, MAX_GATE = 4e-3, 6e-3          # the VAE encode gates of tests/test_model_gpu.py


@pytest.fixture(scope='module')
def gold(gold_dir):
    return torch.load(os.path.join(gold_dir, 'vc_masked.pt'))


@pytest.fixture(scope='module')
def ldm(gold):
    from t2v_b200.videocrafter import LatentDiffusion
    cfg = VC.VCConfig(**gold['unet_cfg'])
    W = UO.make_weights(VC.vc_param_specs(cfg), seed=gold['seeds']['unet'])
    Wv = {**UO.make_weights(VO.decoder_param_specs(VO.VAEConfig()), seed=gold['seeds']['vae_dec']),
          **UO.make_weights(VO.encoder_param_specs(VO.VAEConfig()), seed=gold['seeds']['vae_enc'])}
    m = LatentDiffusion(unet_config=dict(gold['unet_cfg']), image_size=[8, 8], video_length=4)
    m.model.half()                 # fp16 networks; the schedule buffers stay fp32 as in the reference's model (its load_model
    m.first_stage_model.half()     # does not call .half()), so the DDIM coefficients are the restatement's
    m.model.diffusion_model.load_state_dict(W, strict=True)
    m.first_stage_model.load_state_dict(Wv, strict=True)
    return m.cuda().eval(), cfg, {k: v.half().float() for k, v in W.items()}, {k: v.half().float() for k, v in Wv.items()}


def _bufs(device='cuda'):
    return [b.to(device) for b in MO.schedule_buffers(SO.linear_sd_betas())]


# ---------------------------------------------------------------------------------------------------------- kernel
def test_q_sample_kernel_is_bit_identical_to_torch_with_per_sample_t():
    from t2v_b200 import ops
    g = torch.Generator('cuda').manual_seed(3)
    x0 = torch.randn(3, 4, 5, 7, 9, device='cuda', generator=g)                    # 3780 elements: ragged vs the 256 block
    noise = torch.randn(3, 4, 5, 7, 9, device='cuda', generator=g)
    sa, sm = _bufs()
    t = torch.tensor([0, 517, 999], device='cuda')
    a, s = sa[t], sm[t]
    ref = a.view(3, 1, 1, 1, 1) * x0 + s.view(3, 1, 1, 1, 1) * noise
    assert torch.equal(ops.q_sample_blend(x0, noise, a, s), ref)
    # noise of batch 1 broadcast over the batch, and a non-contiguous x0 (a transposed view)
    xt = torch.randn(3, 4, 9, 7, 5, device='cuda', generator=g).transpose(2, 4)
    n1 = noise[:1]
    assert torch.equal(ops.q_sample_blend(xt, n1, a, s), a.view(3, 1, 1, 1, 1) * xt + s.view(3, 1, 1, 1, 1) * n1)


@pytest.mark.parametrize('mask_kind', ['frames', 'region', 'full', 'batch', 'soft'])
def test_blend_kernel_is_bit_identical_to_torch(mask_kind):
    from t2v_b200 import ops
    g = torch.Generator('cuda').manual_seed(5)
    B, C, T, h, w = 2, 4, 5, 7, 9
    img = torch.randn(B, C, T, h, w, device='cuda', generator=g)
    x0 = torch.randn(1, C, T, h, w, device='cuda', generator=g)                    # batch 1 against the batch-2 latent
    noise = torch.randn_like(x0)
    mask = {'frames': (torch.arange(T, device='cuda') < 2).float().view(1, 1, T, 1, 1),
            'region': (torch.rand(1, 1, 1, h, w, device='cuda', generator=g) > 0.5).float(),
            'full': (torch.rand(B, C, T, h, w, device='cuda', generator=g) > 0.5).float(),
            'batch': torch.tensor([1.0, 0.0], device='cuda').view(B, 1, 1, 1, 1),
            'soft': torch.rand(1, C, T, h, w, device='cuda', generator=g)}[mask_kind]
    sa, sm = _bufs()
    t = torch.tensor([400], device='cuda')
    known = sa[t].view(1, 1, 1, 1, 1) * x0 + sm[t].view(1, 1, 1, 1, 1) * noise        # q_sample(x0, t) as ddim.py:193-194
    ref = known * mask + (1. - mask) * img
    out = ops.q_sample_blend(x0, noise, sa[t].expand(B), sm[t].expand(B), mask=mask, img=img)
    assert torch.equal(out, ref)
    ops.q_sample_blend(x0, noise, sa[t].expand(B), sm[t].expand(B), mask=mask, img=img, out=img)      # in place
    assert torch.equal(img, ref)


def test_blend_entry_point_rejects_bad_arguments():
    from t2v_b200 import ops
    x = torch.zeros(1, 4, 2, 8, 8, device='cuda')
    a = torch.ones(1, device='cuda')
    with pytest.raises(RuntimeError, match='mask and img'):
        ops.q_sample_blend(x, x, a, a, mask=torch.ones_like(x))                     # a mask without the latent it blends into
    with pytest.raises(ValueError):
        ops.q_sample_blend(x, x, torch.ones(2, device='cuda'), a)                    # one coefficient per sample
    with pytest.raises(RuntimeError):
        ops.q_sample_blend(x, x, a, a, mask=torch.ones(1, 1, 3, 1, 1, device='cuda'), img=x)   # mask does not broadcast


# ---------------------------------------------------------------------------------------------------------- sampler
def _run(m, gold, S, eta, scale, seed, **kw):
    from t2v_b200.videocrafter import DDIMSampler
    smp = DDIMSampler(m)
    smp.noise_gen.manual_seed(gold['seeds']['noise'])
    calls = []
    torch.cuda.manual_seed(seed)
    out, inter = smp.sample(S=S, batch_size=1, shape=gold['shape'][1:], conditioning=gold['c'].half().float().cuda(),
                            unconditional_conditioning=gold['uc'].half().float().cuda(), unconditional_guidance_scale=scale,
                            eta=eta, verbose=False, callback=calls.append, **kw)
    return out, inter, len(calls)


def _tape(x0, n, seed):
    """The library's q_sample draws: torch.randn_like(x0) on the device, once per step, from the re-seeded generator."""
    torch.cuda.manual_seed(seed)
    return [torch.randn_like(x0) for _ in range(n)]


@pytest.mark.parametrize('case', ['a', 'b', 'c'])
def test_masked_and_truncated_ddim_vs_restatement(ldm, gold, case):
    m, cfg, Wh, _ = ldm
    spec = gold['cases'][case]
    x0 = gold['x0'].cuda()
    mask = gold['masks'][spec['mask']] if 'mask' in spec else None
    kw = dict(mask=mask, x0=x0) if mask is not None else dict(timesteps=spec['timesteps'])
    x_T = gold['x_T'] if mask is not None else gold['x_T_c']
    out, inter, n = _run(m, gold, spec['S'], spec['eta'], spec['scale'], 1234, x_T=x_T.cuda(), **kw)
    assert n == gold['steps_' + case] and torch.equal(inter['x_inter'][-1], out)      # logged after the blend
    tape = _tape(x0, n, 1234) if mask is not None else None
    ref = MO.vc_ddim_sample_masked(lambda a, b, d: VC.vc_unet_forward(Wh, cfg, a, b, d), SO.linear_sd_betas(), x_T, spec['S'],
                                   gold['c'].half().float(), gold['uc'].half().float(), spec['scale'], eta=spec['eta'],
                                   noise_gen=torch.Generator('cpu').manual_seed(gold['seeds']['noise']), mask=mask,
                                   x0=gold['x0'], q_tape=[t.cpu() for t in tape] if tape else None,
                                   timesteps=spec.get('timesteps'))
    err = (out.cpu() - ref).abs().max() / ref.abs().max()
    report(f'vc_masked_ddim:{case}', max=float(err))
    assert err < 5e-3, err
    if mask is not None:                          # the last blend runs at t = 0: the known region is q_sample(x0, 0), bit for bit
        bufs = MO.schedule_buffers(SO.linear_sd_betas())
        known = MO.q_sample(bufs, gold['x0'], torch.tensor([0]), tape[-1].cpu())
        sel = mask.expand_as(ref) == 1
        assert torch.equal(out.cpu()[sel], known[sel])


def test_mask_invariances(ldm, gold):
    m = ldm[0]
    x0, x_T = gold['x0'].cuda(), gold['x_T'].cuda()
    plain, _, _ = _run(m, gold, 4, 0.5, 3.0, 7, x_T=x_T)
    zero, _, _ = _run(m, gold, 4, 0.5, 3.0, 7, x_T=x_T, mask=torch.zeros(1, 1, 4, 1, 1), x0=x0)
    assert torch.equal(zero, plain)
    one, _, n = _run(m, gold, 4, 0.5, 3.0, 7, x_T=x_T, mask=torch.ones(1, 1, 1, 1, 1, dtype=torch.float16), x0=x0)
    assert torch.equal(one, m.q_sample(x0, torch.tensor([0]), noise=_tape(x0, n, 7)[-1]))


@pytest.mark.parametrize('k,S', [(6, 10), (15, 22)])
def test_timesteps_runs_the_reference_prefix(ldm, gold, k, S):
    m = ldm[0]
    _, _, n = _run(m, gold, S, 0.0, 1.0, 0, x_T=gold['x_T'].cuda(), timesteps=k)
    assert n == gold['prefix_steps'][(k, S)]


def test_errors_are_loud(ldm, gold, monkeypatch):
    from t2v_b200 import distributed as dist
    m = ldm[0]
    with pytest.raises(AssertionError):
        _run(m, gold, 2, 0.0, 3.0, 0, x_T=gold['x_T'].cuda(), mask=torch.ones(1, 1, 4, 1, 1))       # mask without x0
    monkeypatch.setattr(dist, 'cfg_split_enabled', lambda: True)
    with pytest.raises(NotImplementedError):
        _run(m, gold, 2, 0.0, 3.0, 0, x_T=gold['x_T'].cuda(), mask=torch.ones(1, 1, 4, 1, 1), x0=gold['x0'].cuda())


# ---------------------------------------------------------------------------------------------------------- encode
def _video(gold, shape=None):
    shape = gold['video_shape'] if shape is None else shape
    return torch.rand(shape, generator=torch.Generator('cpu').manual_seed(gold['seeds']['video'])) * 2 - 1


def test_encode_first_stage_2DAE_vs_restatement(ldm, gold):
    m, _, _, Wvh = ldm
    video = _video(gold)
    b, _, t, H, W = video.shape
    torch.manual_seed(gold['seeds']['post'])
    z = m.encode_first_stage_2DAE(video.cuda(), encode_bs=gold['encode_bs'])
    assert z.shape == (b, 4, t, H // 8, W // 8)
    tape = MO.posterior_tape(gold['seeds']['post'], b * t, gold['encode_bs'], (4, H // 8, W // 8))
    ref = MO.encode_first_stage_2DAE(Wvh, video, gold['encode_bs'], tape)
    e = errs(z, ref)
    report('vc_encode_first_stage_2DAE', max=e[0], rms=e[1])
    assert e[1] < RMS_GATE and e[0] < MAX_GATE, e
    torch.manual_seed(gold['seeds']['post'])
    assert torch.equal(m.encode_first_stage_2DAE(video.cuda(), encode_bs=gold['encode_bs']), z)     # same CPU seed, same latent
    # encode_bs changes only the posterior draws, exactly as the per-chunk tapes differ.  (torch's CPU normal generator gives
    # the same numbers for chunked and whole draws when a frame's latent holds a multiple of 16 elements, as here.)
    post = m.first_stage_model.encode(video.cuda().permute(0, 2, 1, 3, 4).reshape(b * t, 3, H, W))
    zs, tapes = [], []
    for bs in (1, 16):
        torch.manual_seed(gold['seeds']['post'])
        zs.append(m.encode_first_stage_2DAE(video.cuda(), encode_bs=bs))
        tapes.append(torch.cat(MO.posterior_tape(gold['seeds']['post'], b * t, bs, (4, H // 8, W // 8))).cuda())
        want = 0.18215 * ((post.mean + post.std * tapes[-1]) + 0.0)
        assert torch.equal(zs[-1], want.reshape(b, t, 4, H // 8, W // 8).permute(0, 2, 1, 3, 4))
    assert torch.equal(zs[0], zs[1]) == torch.equal(tapes[0], tapes[1])


# ---------------------------------------------------------------------------------------------------------- end to end
@pytest.mark.parametrize('with_adapter', [False, True])
def test_continuation_end_to_end(ldm, gold, gold_dir, with_adapter):
    """encode a clip, continue it with its first two frames known (optionally guided by adapter features), decode it."""
    m = ldm[0]
    video = _video(gold, (1, 3, 4, 64, 64))
    torch.manual_seed(3)
    z = m.encode_first_stage_2DAE(video.cuda())
    assert z.shape == (1, 4, 4, 8, 8)
    frames_mask = torch.zeros(1, 1, 4, 1, 1)
    frames_mask[:, :, :2] = 1.0
    kw = {}
    if with_adapter:
        kw['features_adapter'] = [f.cuda() for f in torch.load(os.path.join(gold_dir, 'adapter.pt'))['features_A']]
    x_T = torch.randn(1, 4, 4, 8, 8, generator=torch.Generator('cpu').manual_seed(9)).cuda()
    out, _, n = _run(m, gold, 5, 1.0, 7.5, 21, x_T=x_T, mask=frames_mask, x0=z, **kw)
    known = m.q_sample(z, torch.tensor([0]), noise=_tape(z, n, 21)[-1])
    assert torch.equal(out[:, :, :2], known[:, :, :2]) and torch.isfinite(out).all()
    dec = m.decode_first_stage(out, return_cpu=False)
    assert dec.shape == (1, 3, 4, 64, 64) and torch.isfinite(dec).all()
