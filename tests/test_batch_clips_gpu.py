"""GPU: batched ModelScope clips (`infer(batch_size=n)`, tiny seeded UNetSD, full-size VAE decoder) against the same seeds
run one at a time, for every sampler and for eta > 0 on shared per-clip noise tapes; the shared-context forward (Bc = 2 prompts
for B samples) against the context repeated to B; the Bc = B entry on the parent's plan; budget-sized groups.

Batched and single runs differ only by reduction orders that depend on the batch (GEMM split-K count, GroupNorm statistics
grid; DESIGN.md section 2).  On this seeded tiny model one forward of a sample in a B = 6 batch already differs from its B = 2
forward by 2.4e-3 max-relative (H100), and classifier-free guidance at scale 6 multiplies eps differences by 6: the runs below
measured 4.1e-3 to 7.9e-3 on the final latent and up to 3 LSB on the frames.  Gates: 1e-2 and 3 LSB.  A sample reading the
wrong prompt would be off by ~0.3 (the cond / uncond eps differ by 0.57 at a maximum of 1.9).  The shared-context forward
itself is checked against the repeated context on the same batch, where nothing but the K/V rows changes: bit for bit."""
import numpy as np
import pytest
import torch

from oracle import unet_oracle as UO, vae_oracle as VO

from parity_util import report  # noqa: E402

pytestmark = pytest.mark.gpu

F_, SIZE = 3, 64


@pytest.fixture(scope='module')
def pipe():
    from t2v_b200.pipeline import TextToVideoSynthesis
    W = UO.make_weights(UO.param_specs(UO.UNetConfig(dim=64)), seed=1)
    Wv = UO.make_weights(VO.decoder_param_specs(VO.VAEConfig()), seed=3)
    return TextToVideoSynthesis(None, model_cfg={'unet_dim': 64}, unet_state=W, vae_state=Wv)


def conds():
    g = torch.Generator().manual_seed(2)
    return torch.randn(1, 77, 1024, generator=g).half(), torch.randn(1, 77, 1024, generator=g).half()


def run(p, sampler, steps, seed, eta=0.0, batch_size=1, frames=F_):
    c, uc = conds()
    return p.infer(c, uc, steps, frames, seed, 6.0, SIZE, SIZE, eta, 'GPU (half precision)', torch.device('cuda'), None, 0, 0.0, None,
                   False, sampler, batch_size=batch_size)


def check_clip(tag, frames_b, latent_b, frames_s, latent_s, frames=F_):
    err = float((latent_b - latent_s).abs().max() / latent_s.abs().max())
    lsb = max(int(np.abs(a.astype(int) - b.astype(int)).max()) for a, b in zip(frames_b, frames_s))
    report(tag, max=err, lsb=lsb)
    assert latent_b.shape == latent_s.shape and len(frames_b) == len(frames_s) == frames
    assert err <= 1e-2, err
    assert lsb <= 3, lsb


SAMPLERS = [('DDIM_Gaussian', 6), ('DDIM', 5), ('UniPC', 5)]


@pytest.mark.parametrize('sampler,steps', SAMPLERS)
def test_batch_matches_single_runs(pipe, sampler, steps):
    videos, latents, infos = run(pipe, sampler, steps, 40, batch_size=3)
    assert len(videos) == len(latents) == len(infos) == 3 and pipe.last_batch_groups == [3]
    for i in range(3):
        frames, latent, info = run(pipe, sampler, steps, 40 + i)
        assert f'seed: {40 + i}' in infos[i] and infos[i] == info
        check_clip(f'batch_clips:{sampler}:clip{i}', videos[i], latents[i], frames, latent)
    assert not torch.equal(latents[0], latents[1])


@pytest.mark.parametrize('sampler', ['DDIM_Gaussian', 'DDIM'])
def test_batch_matches_single_runs_eta_positive(pipe, sampler, monkeypatch):
    """eta > 0: the per-step noise of clip i is the same tape in the batched and in the single run (fed through the samplers'
    one noise hook, distributed.step_noise: the batch draws one clip-sized tensor per clip, in clip order)."""
    from t2v_b200 import distributed as D
    S, n = 4, 3
    tapes = [[torch.randn((1, 4, F_, 8, 8), generator=torch.Generator().manual_seed(900 + 10 * i + s)) for s in range(S)]
             for i in range(n)]

    def feed(clips):
        step = {'s': 0}

        def noise(like):
            out = torch.cat([tapes[i][step['s']] for i in clips]).to(device=like.device, dtype=like.dtype)
            step['s'] += 1
            assert out.shape == like.shape
            return out
        monkeypatch.setattr(D, 'step_noise', noise)
    feed(range(n))
    videos, latents, _ = run(pipe, sampler, S, 70, eta=0.8, batch_size=n)
    for i in range(n):
        feed([i])
        frames, latent, _ = run(pipe, sampler, S, 70 + i, eta=0.8)
        check_clip(f'batch_clips:{sampler}_eta0.8:clip{i}', videos[i], latents[i], frames, latent)


def test_shared_context_matches_repeated_context(pipe):
    """B = 6 samples over Bc = 2 prompts (t2v_unet_forward_ctx) vs the prompts repeated to B (t2v_unet_forward): the same eps
    bit for bit, same launch count, and the shared plan's K/V GEMMs project 2 * L rows where the repeated one projects
    6 * L (flop of the launch lists, exactly the difference)."""
    net = pipe.sd_model
    c, uc = conds()
    n = 3
    x = torch.randn((n, 4, F_, 8, 8), generator=torch.Generator().manual_seed(5)).cuda()
    xb = torch.cat([x, x])
    t = torch.full((2 * n,), 421.0, device='cuda')
    y = torch.cat([c, uc]).cuda()
    shared = net(xb, t, y)
    launches_shared = net.num_launches()
    repeated = net(xb, t, y.repeat_interleave(n, dim=0))
    launches_repeated = net.num_launches()
    err = float((shared.float() - repeated.float()).abs().max() / repeated.float().abs().max())
    report('batch_clips:shared_vs_repeated_context', max=err)
    assert torch.equal(shared, repeated), err                      # only the K/V GEMMs' row count differs; each row is the same
    assert launches_shared == launches_repeated
    _, fl_shared, cached_shared = net.plan_info(2 * n, F_, 8, 8, 77, ctx_batch=2)
    _, fl_rep, cached_rep = net.plan_info(2 * n, F_, 8, 8, 77)
    assert cached_shared and cached_rep
    kv = [p.shape[0] for k, p in net.named_parameters() if k.endswith('attn2.to_k.weight') and p.shape[1] == net.context_dim]
    assert fl_rep - fl_shared == pytest.approx(sum(2.0 * (2 * n - 2) * 77 * 2 * C_ * net.context_dim for C_ in kv), rel=1e-9)


def test_full_context_batch_keeps_the_parent_plan(pipe):
    """t2v_unet_forward_ctx with ctx_B = B is t2v_unet_forward: the same plan (key), launch count and bits."""
    from t2v_b200 import _lib
    net = pipe.sd_model
    B, F, h, w, L = 4, 2, 8, 8, 77
    x = torch.randn((B, 4, F, h, w), generator=torch.Generator().manual_seed(6)).cuda()
    t = torch.full((B,), 300.0, device='cuda')
    y = torch.randn((B, L, 1024), generator=torch.Generator().manual_seed(7)).half().cuda()
    assert not net.plan_info(B, F, h, w, L)[2]
    ref = net(x, t, y)
    launches = net.num_launches()
    assert net.plan_info(B, F, h, w, L)[2] and not net.plan_info(B, F, h, w, L, ctx_batch=2)[2]
    out = torch.empty_like(ref)
    rc = _lib.lib().t2v_unet_forward_ctx(net._handle, _lib.ptr(x), 1, _lib.ptr(t), _lib.ptr(y), B, _lib.ptr(out), 0, B, F, h, w, L,
                                         _lib.stream_ptr())
    _lib.check(rc, 'unet_forward_ctx')
    assert net.num_launches() == launches and torch.equal(out, ref)
    assert not net.plan_info(B, F, h, w, L, ctx_batch=2)[2]          # no other plan was built
    for bad in (0, 3):
        rc = _lib.lib().t2v_unet_forward_ctx(net._handle, _lib.ptr(x), 1, _lib.ptr(t), _lib.ptr(y), bad, _lib.ptr(out), 0, B, F, h,
                                             w, L, _lib.stream_ptr())
        assert rc != 0 and b'does not divide' in _lib.load_library().t2v_last_error()


def test_small_budget_runs_two_groups(pipe):
    """A budget that holds the B = 4 plan but not the B = 6 or B = 8 one: 4 clips run as two groups of 2, each clip still
    matching its single run.  (4 frames: no earlier test cached a plan of this shape, and a cached plan needs no budget.)"""
    net = pipe.sd_model
    F4 = 4
    need = {k: net.plan_info(2 * k, F4, 8, 8, 77, ctx_batch=2) for k in (2, 3, 4)}
    assert not any(cached for _, _, cached in need.values())
    assert need[2][0] < need[3][0] < need[4][0]
    pipe.batch_memory_budget = need[2][0]
    try:
        videos, latents, _ = run(pipe, 'DDIM_Gaussian', 4, 90, batch_size=4, frames=F4)
        assert pipe.last_batch_groups == [2, 2]
    finally:
        pipe.batch_memory_budget = 0
    for i in range(4):
        frames, latent, _ = run(pipe, 'DDIM_Gaussian', 4, 90 + i, frames=F4)
        check_clip(f'batch_clips:budget_groups:clip{i}', videos[i], latents[i], frames, latent, frames=F4)


def test_process_modelscope_batch_size(pipe):
    from t2v_b200 import process_modelscope as pm
    pm.pipe = pipe
    c, uc = conds()
    base = {'prompt_embeds': c, 'n_prompt_embeds': uc, 'steps': 4, 'frames': F_, 'seed': 5, 'cfg_scale': 4.0, 'width': SIZE,
            'height': SIZE, 'batch_count': 3, 'sampler': 'DDIM', 'return_frames': True}
    try:
        batched = pm.process_modelscope(dict(base, batch_size=2))
        seq = pm.process_modelscope(base)
    finally:
        pm.pipe = None
    assert len(batched) == len(seq) == 3
    for a, b in zip(batched, seq):
        assert len(a) == F_ and max(int(np.abs(x.astype(int) - y.astype(int)).max()) for x, y in zip(a, b)) <= 3


def with_encoder(p):
    Wenc = UO.make_weights(VO.encoder_param_specs(VO.VAEConfig()), seed=5)
    p.autoencoder.load_state_dict(Wenc, strict=False)
    p.autoencoder.cuda()


def max_lsb(a, b):
    return max(int(np.abs(x.astype(int) - y.astype(int)).max()) for x, y in zip(a, b))


def test_img2vid_batch_blends_one_start_latent_per_clip(pipe):
    """img2vid: the blended start latent is the clip's x_T, so a batch takes one per clip.  infer() with the three blends
    stacked matches three single runs on them; process_modelscope blends one per clip from numpy's generator in clip order,
    like the sequential loop, so the clips of a batch differ."""
    from t2v_b200 import process_modelscope as pm
    with_encoder(pipe)
    c, uc = conds()
    img = torch.rand((3, SIZE, SIZE), generator=torch.Generator().manual_seed(8)) * 2 - 1
    blends = [pm.inpainting_latents(pipe, img, F_, SIZE, SIZE, 2, '0:(t/max_i_f), "max_i_f":(1)', 21, 'GPU (half precision)',
                                    np.random.RandomState(300 + i).normal(size=(1, 4, F_, 8, 8))) for i in range(3)]
    lat, mask = torch.cat([b[0] for b in blends]), torch.cat([b[1] for b in blends])
    # guidance 3: at guidance 6 the same comparison measured 7.5e-3 on the latent (the residue of every other test) but 5 LSB
    # on the frames, which decode from image-derived latents; at 3: 3.2e-3 to 3.4e-3 and 3 LSB
    args = (c, uc, 4, F_, 21, 3.0, SIZE, SIZE, 0.0, 'GPU (half precision)', torch.device('cuda'))
    videos, latents, _ = pipe.infer(*args, lat, 0, 1, mask, False, 'DDIM_Gaussian', batch_size=3)
    for i in range(3):
        frames, latent, _ = pipe.infer(*args[:4], 21 + i, *args[5:], blends[i][0], 0, 1, blends[i][1], False, 'DDIM_Gaussian')
        check_clip(f'batch_clips:img2vid:clip{i}', videos[i], latents[i], frames, latent)
    pm.pipe = pipe
    base = dict(prompt_embeds=c, n_prompt_embeds=uc, steps=4, frames=F_, seed=21, cfg_scale=6.0, width=SIZE, height=SIZE,
                sampler='DDIM_Gaussian', return_frames=True, batch_count=2, batch_size=2, inpainting_frames=2,
                inpainting_image_tensor=img)
    try:
        out = pm.process_modelscope(base)
    finally:
        pm.pipe = None
    assert len(out) == 2 and max_lsb(out[0], out[1]) > 3


@pytest.mark.parametrize('sampler', ['DDIM_Gaussian', 'DDIM', 'UniPC'])
def test_vid2vid_batch_matches_sequential(pipe, sampler):
    """vid2vid: the encoded video is shared, each clip noises it with its own x_T (encode_latent), so the clips of a batch
    differ and each matches its sequential run."""
    from t2v_b200 import process_modelscope as pm
    with_encoder(pipe)
    pm.pipe = pipe
    c, uc = conds()
    vid = torch.rand((1, 3, F_, SIZE, SIZE), generator=torch.Generator().manual_seed(4)) * 2 - 1
    base = dict(prompt_embeds=c, n_prompt_embeds=uc, steps=8, frames=F_, seed=11, cfg_scale=6.0, width=SIZE, height=SIZE,
                sampler=sampler, return_frames=True, batch_count=2, do_vid2vid=True, vid2vid_frames_tensor=vid, strength=0.5)
    try:
        batched = pm.process_modelscope(dict(base, batch_size=2))
        seq = pm.process_modelscope(base)
    finally:
        pm.pipe = None
    assert max_lsb(batched[0], batched[1]) > 3
    for i, (a, b) in enumerate(zip(batched, seq)):
        lsb = max_lsb(a, b)
        report(f'batch_clips:vid2vid_{sampler}:clip{i}', lsb=lsb)
        assert len(a) == F_ and lsb <= 3, lsb


@pytest.fixture(scope='module')
def ldm():
    from oracle import vc_oracle as VC
    from t2v_b200.videocrafter import LatentDiffusion
    W = UO.make_weights(VC.vc_param_specs(VC.VCConfig(model_channels=64, context_dim=48, temporal_length=4)), seed=4)
    Wv = UO.make_weights(VO.decoder_param_specs(VO.VAEConfig()), seed=3)
    m = LatentDiffusion(unet_config=dict(model_channels=64, context_dim=48, temporal_length=4), image_size=[8, 8],
                        video_length=4).half()
    m.model.diffusion_model.load_state_dict(W, strict=True)
    m.first_stage_model.load_state_dict(Wv, strict=False)
    return m.cuda().eval()


def vc_conds():
    g = torch.Generator().manual_seed(2)
    return torch.randn(1, 9, 48, generator=g).half().cuda(), torch.randn(1, 9, 48, generator=g).half().cuda()


def test_videocrafter_shared_context_matches_repeated(ldm):
    """VideoCrafter's UNetModel (arch 1) on the shared-context forward: the DDIM sampler's batched pair of 2 clips with one
    prompt pair ([x; x] over [c; uc], Bc = 2 of B = 4) equals the same run with the prompts repeated per clip, bit for bit,
    and process_videocrafter(batch_size=2) returns two different clips."""
    from t2v_b200 import videocrafter as vcm
    c, uc = vc_conds()
    x_T = torch.randn((2, 4, 4, 8, 8), generator=torch.Generator().manual_seed(6)).cuda()
    smp = vcm.DDIMSampler(ldm)
    kw = dict(S=4, batch_size=2, shape=(4, 4, 8, 8), x_T=x_T, eta=0.0, unconditional_guidance_scale=5.0, verbose=False)
    shared, _ = smp.sample(conditioning=c, unconditional_conditioning=uc, **kw)
    repeated, _ = smp.sample(conditioning=c.repeat(2, 1, 1), unconditional_conditioning=uc.repeat(2, 1, 1), **kw)
    report('batch_clips:vc_shared_vs_repeated_context',
           max=float((shared.float() - repeated.float()).abs().max() / repeated.float().abs().max()))
    assert torch.equal(shared, repeated)
    out = vcm.process_videocrafter(dict(prompt_embeds=c, n_prompt_embeds=uc, steps=4, frames=4, seed=3, cfg_scale=5.0, eta=0.0,
                                        batch_count=1, batch_size=2), model=ldm)
    assert len(out) == 2 and out[0].shape == (1, 3, 4, 64, 64) and not np.array_equal(out[0], out[1])
