"""GPU: frame-chunked VAE decode and encode.  An explicit memory budget between the one-frame and the whole-clip plan bytes
forces the library to split a small clip; the result must match the whole-clip call.  Every op is per frame, but two
reduction orders depend on the frame count of a plan -- the GroupNorm statistics grid (chunks per instance =
ceil(2 * SMs / frames)) and the GEMM split-K count (chosen from the tile count) -- so a chunk's fp32 sums may round
differently in the last bit: uint8 frames agree within 1 LSB, fp32 outputs within F32_BOUND (DESIGN.md section 2)."""
import numpy as np
import pytest
import torch

from oracle import unet_oracle as UO, vae_oracle as VO, vc_oracle as VC

from parity_util import report  # noqa: E402

pytestmark = pytest.mark.gpu

# max |chunked - whole| of the fp32 decode ([-1, 1]) and of the encoder's moments: one uint8 step of [-1, 1] (2 / 255).
# Measured on an H100 at these shapes: decode 3.9e-3 (B = 1, F = 5) and 4.9e-3 (B = 2, F = 3), moments 2.9e-3 (N = 7) --
# last-bit fp16 differences from the frame-count-dependent reduction orders, carried through the following layers.
F32_BOUND = 2.0 / 255


@pytest.fixture
def ae():
    # one handle per test: a cached whole-clip plan is always replayed whatever the budget, so each test forces its
    # chunked call before the whole-clip call at that shape
    from t2v_b200.modules import AutoencoderKL
    from t2v_b200.pipeline import VAE_DDCONFIG
    cfg = VO.VAEConfig()
    W = {**UO.make_weights(VO.decoder_param_specs(cfg), seed=3), **UO.make_weights(VO.encoder_param_specs(cfg), seed=4)}
    m = AutoencoderKL(VAE_DDCONFIG, 4, None).half()
    m.load_state_dict(W, strict=True)
    return m.cuda().eval()


def _latent(B, F, h=16, w=16, seed=0):
    return torch.randn(B, 4, F, h, w, generator=torch.Generator().manual_seed(seed)).cuda()


def _same(name, got, ref, u8):
    d = (got.float() - ref.float()).abs().max().item()
    report(f'vae_chunked:{name}', max_abs=d, equal=bool(torch.equal(got, ref)))
    assert d <= (1.0 if u8 else F32_BOUND), (name, d)


def _chunked(ae, budget, fn, encode=False):
    ae.memory_budget = budget
    try:
        return fn(), ae.last_chunking(encode), ae.cached_plans(encode)
    finally:
        ae.memory_budget = 0


@pytest.mark.parametrize('B,F,n,u8', [(1, 5, 2, True), (1, 5, 2, False), (2, 3, 2, True), (2, 3, 2, False)])
def test_chunked_decode_matches_whole_clip(ae, B, F, n, u8):
    # (1, 5): chunks of 2 + a tail of 1; (2, 3): the second chunk holds frame 2 of sample 0 and frame 0 of sample 1
    z = _latent(B, F, seed=B * 10 + F)
    budget = ae.plan_bytes(n, 16, 16)
    assert ae.plan_bytes(1, 16, 16) < budget < ae.plan_bytes(n + 1, 16, 16)
    out, split, (cached, _) = _chunked(ae, budget, lambda: ae.decode_video(z, as_uint8=u8))
    assert split == (n, -(-B * F // n))
    assert cached == 0                          # a chunked call leaves no plan behind (they are sized to the free memory)
    out = out.clone()
    ref = ae.decode_video(z, as_uint8=u8)
    assert ae.last_chunking() == (B * F, 1) and ae.cached_plans()[0] == 1
    assert out.shape == ref.shape
    _same(f'decode_B{B}F{F}_{"u8" if u8 else "f32"}', out, ref, u8)
    ae.memory_budget = budget
    assert torch.equal(ae.decode_video(z, as_uint8=u8), ref) and ae.last_chunking() == (B * F, 1)    # cached: whole clip
    ae.memory_budget = 0


def test_chunked_encode_matches_whole_clip(ae):
    x = (torch.rand((7, 3, 128, 128), generator=torch.Generator().manual_seed(3)) * 2 - 1).cuda()
    budget = ae.plan_bytes(3, 128, 128, encode=True)
    out, split, (cached, _) = _chunked(ae, budget, lambda: ae.encode(x).parameters, encode=True)
    assert split == (3, 3) and cached == 0
    out = out.clone()
    ref = ae.encode(x).parameters
    assert ae.last_chunking(encode=True) == (7, 1)
    _same('encode_N7', out, ref, False)


def test_budget_below_one_frame_raises_before_allocating(ae):
    torch.cuda.synchronize()
    z = _latent(1, 3, 24, 24, seed=5)                                  # a shape no plan exists for yet
    one = ae.plan_bytes(1, 24, 24)
    before = ae.cached_plans()
    ae.memory_budget = one - 1
    try:
        with pytest.raises(RuntimeError) as e:
            ae.decode_video(z)
    finally:
        ae.memory_budget = 0
    msg = str(e.value)
    assert 'one-frame plan needs' in msg and '24 x 24' in msg and f'{one / 2 ** 20:.1f} MB' in msg and 'memory budget' in msg
    after = ae.cached_plans()
    assert after[0] <= before[0] and after[1] <= before[1]             # nothing was built


def _pipe():
    from t2v_b200.pipeline import TextToVideoSynthesis
    cfg = VO.VAEConfig()
    W = UO.make_weights(UO.param_specs(UO.UNetConfig(dim=64)), seed=1)
    Wv = {**UO.make_weights(VO.decoder_param_specs(cfg), seed=3), **UO.make_weights(VO.encoder_param_specs(cfg), seed=5)}
    return TextToVideoSynthesis(None, model_cfg={'unet_dim': 64}, unet_state=W, vae_state=Wv)


def test_infer_and_process_modelscope_with_a_forced_budget():
    from t2v_b200 import process_modelscope as pm
    p = _pipe()
    g = torch.Generator().manual_seed(2)
    c, uc = torch.randn(1, 77, 1024, generator=g).half(), torch.randn(1, 77, 1024, generator=g).half()
    args = (c, uc, 3, 5, 123, 7.5, 128, 128, 0.0, 'GPU (half precision)', torch.device('cuda'), None, 0, 0.0, None, False,
            'DDIM_Gaussian')
    ae = p.autoencoder
    ae.memory_budget = ae.plan_bytes(2, 16, 16)
    try:
        frames2, latent2, _ = p.infer(*args)
        assert ae.last_chunking() == (2, 3)
        pm.pipe = p
        base = dict(prompt_embeds=c, n_prompt_embeds=uc, steps=8, frames=5, seed=11, cfg_scale=5.0, width=128, height=128,
                    sampler='DDIM', return_frames=True)
        vid = torch.rand((1, 3, 5, 128, 128), generator=torch.Generator().manual_seed(4)) * 2 - 1
        forced = pm.process_modelscope(dict(base, do_vid2vid=True, vid2vid_frames_tensor=vid, strength=0.5))
        assert ae.last_chunking(encode=True)[1] > 1
    finally:
        ae.memory_budget = 0
    frames, latent, _ = p.infer(*args)
    assert ae.last_chunking() == (5, 1)
    whole = pm.process_modelscope(dict(base, do_vid2vid=True, vid2vid_frames_tensor=vid, strength=0.5))
    assert ae.last_chunking(encode=True) == (5, 1)
    pm.pipe = None
    assert torch.equal(latent, latent2)
    d = max(np.abs(a.astype(np.int16) - b.astype(np.int16)).max() for a, b in zip(frames, frames2))
    report('vae_chunked:infer_u8', max_abs=int(d))
    assert d <= 1
    # vid2vid: the input video is encoded in chunks too; its latent feeds a sampler, so allow the fp32 moment difference to
    # show up in the frames, but no more than a few LSB
    d2 = max(np.abs(a.astype(np.int16) - b.astype(np.int16)).max() for a, b in zip(forced[0], whole[0]))
    report('vae_chunked:process_modelscope_vid2vid_u8', max_abs=int(d2))
    assert d2 <= 4


def test_videocrafter_decode_and_encode_with_a_forced_budget():
    from t2v_b200 import videocrafter as vcm
    from t2v_b200.videocrafter import LatentDiffusion
    cfg = VO.VAEConfig()
    m = LatentDiffusion(unet_config=dict(model_channels=64, context_dim=48, temporal_length=4), image_size=[16, 16],
                        video_length=4).half()
    m.model.diffusion_model.load_state_dict(UO.make_weights(VC.vc_param_specs(VC.VCConfig(model_channels=64, context_dim=48,
                                                                                            temporal_length=4)), seed=4), strict=True)
    m.first_stage_model.load_state_dict({**UO.make_weights(VO.decoder_param_specs(cfg), seed=3),
                                         **UO.make_weights(VO.encoder_param_specs(cfg), seed=4)}, strict=True)
    m = m.cuda().eval()
    ae = m.first_stage_model
    g = torch.Generator('cpu').manual_seed(2)
    c, uc = torch.randn(1, 9, 48, generator=g).half().float().cuda(), torch.randn(1, 9, 48, generator=g).half().float().cuda()
    x_T = torch.randn((1, 4, 4, 16, 16), generator=torch.Generator('cpu').manual_seed(9)).cuda()
    run = lambda: vcm.sample_text2video(m, c, uc, 1, 1, ddim_steps=4, eta=0.0, cfg_scale=4.0, num_frames=4, x_T=x_T)
    lat = torch.randn((1, 4, 4, 16, 16), generator=torch.Generator('cpu').manual_seed(1)).cuda()
    video = (torch.rand((1, 3, 5, 128, 128), generator=torch.Generator().manual_seed(6)) * 2 - 1).cuda()
    ae.memory_budget = ae.plan_bytes(2, 16, 16)
    try:
        vids2 = run()
        assert ae.last_chunking() == (2, 2)
        dec2 = m.decode_first_stage(lat, return_cpu=False).clone()
        assert ae.last_chunking() == (2, 2)
        ae.memory_budget = ae.plan_bytes(2, 128, 128, encode=True)
        torch.manual_seed(0)
        z2 = m.encode_first_stage_2DAE(video, encode_bs=2)
        assert ae.last_chunking(encode=True) == (2, 3)
    finally:
        ae.memory_budget = 0
    vids = run()
    dec = m.decode_first_stage(lat, return_cpu=False)
    assert ae.last_chunking() == (4, 1)
    torch.manual_seed(0)
    z = m.encode_first_stage_2DAE(video, encode_bs=2)
    assert ae.last_chunking(encode=True) == (5, 1)
    d = np.abs(np.asarray(vids, dtype=np.float64) - np.asarray(vids2, dtype=np.float64)).max()
    report('vae_chunked:vc_sample_text2video', max_abs=float(d))
    assert d <= 1.0
    _same('vc_decode_first_stage', dec2, dec, False)
    # same CPU seed: the posterior noise is drawn per encode_bs chunk as before, so only the moments can differ
    d = (z2 - z).abs().max().item() / z.abs().max().item()
    report('vae_chunked:vc_encode_first_stage_2DAE', max_rel=d)
    assert d <= F32_BOUND
