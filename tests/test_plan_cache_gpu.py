"""GPU: every library handle keeps its plans in one bounded cache (csrc/runtime.cuh PlanCache): more shapes than the bound
evict and rebuild plans, a grown GroupNorm workspace drops them, and handles live side by side.  None of that may change a
result: every comparison here is bit for bit."""
import gc

import pytest
import torch

from oracle import clip_oracle as CO, unet_oracle as UO, vae_oracle as VO, vc_oracle as VC
import adapter_oracle as AO

pytestmark = pytest.mark.gpu

UNET_SHAPES = [(1, 2, 8, 8), (1, 3, 8, 8), (2, 2, 8, 8), (1, 2, 16, 8), (1, 4, 8, 16), (1, 1, 16, 16)]    # > the UNet bound of 4


def _unet_sd():
    from t2v_b200.modules import UNetSD
    net = UNetSD(dim=64).half()
    net.load_state_dict(UO.make_weights(UO.param_specs(UO.UNetConfig(dim=64)), seed=1), strict=True)
    return net.cuda().eval()


def _unet_inputs(B, Fr, h, w):
    g = torch.Generator().manual_seed(B * 1000 + Fr * 100 + h + w)
    x = torch.randn(B, 4, Fr, h, w, generator=g)
    y = torch.randn(B, 77, 1024, generator=g)
    t = torch.randint(0, 1000, (B,), generator=g)
    return x.cuda(), t.cuda(), y.cuda()


def _vae():
    from t2v_b200.modules import AutoencoderKL
    from t2v_b200.pipeline import VAE_DDCONFIG
    cfg = VO.VAEConfig()
    W = {**UO.make_weights(VO.decoder_param_specs(cfg), seed=3), **UO.make_weights(VO.encoder_param_specs(cfg), seed=4)}
    ae = AutoencoderKL(VAE_DDCONFIG, 4, None).half()
    ae.load_state_dict(W, strict=True)
    return ae.cuda().eval()


def _latent(frames, h=8, w=8):
    return torch.randn(frames, 4, h, w, generator=torch.Generator().manual_seed(frames * 100 + h)).cuda()


def _cycled_twice(shapes, run):
    """Runs every shape twice over, in the same order; the second round must reproduce the first bit for bit."""
    first = [run(s).clone() for s in shapes]
    for s, ref in zip(shapes, first):
        assert torch.equal(run(s), ref), s


def test_unet_evicts_and_rebuilds_plans_without_changing_results():
    net = _unet_sd()
    _cycled_twice(UNET_SHAPES, lambda s: net(*_unet_inputs(*s)))


def test_feature_plan_between_plain_forwards():
    from t2v_b200.modules import UNetModel
    kw = dict(model_channels=64, context_dim=48, temporal_length=4)
    m = UNetModel(**kw).half()
    m.load_state_dict(UO.make_weights(VC.vc_param_specs(VC.VCConfig(**kw)), seed=4), strict=True)
    m = m.cuda().eval()
    g = torch.Generator().manual_seed(7)
    x = torch.randn(1, 4, 3, 8, 8, generator=g).cuda()
    ctx = torch.randn(1, 9, 48, generator=g).cuda()
    t = torch.tensor([500]).cuda()
    plain = m(x, t, context=ctx).clone()
    feats = [torch.randn((1,) + s, generator=g).half().cuda() for s in m.feature_shapes(3, 8, 8)]
    with_feats = m(x, t, context=ctx, features_adapter=feats)
    assert not torch.equal(with_feats, plain)
    assert torch.equal(m(x, t, context=ctx), plain)


def test_vae_evicts_and_survives_workspace_growth():
    ae = _vae()
    frames = [1, 2, 3, 4]                                       # > the decoder bound of 3
    decode = lambda f: ae.decode(_latent(f))
    first = [decode(f).clone() for f in frames]
    for f, ref in zip(frames, first):
        assert torch.equal(decode(f), ref), f
    # 12 frames need a larger GroupNorm workspace than any decode above: growing it drops the decoder's plans too
    x = torch.rand((12, 3, 64, 64), generator=torch.Generator().manual_seed(9)).cuda() * 2 - 1
    assert torch.isfinite(ae.encode(x).mean).all()
    for f, ref in zip(frames, first):
        assert torch.equal(decode(f), ref), f


def test_text_tower_evicts_and_rebuilds_plans():
    from t2v_b200.clip import FrozenOpenCLIPEmbedder
    cfg = CO.ClipConfig(width=128, heads=2, layers=4, layers_run=3, context=77, vocab=300)
    e = FrozenOpenCLIPEmbedder(width=cfg.width, heads=cfg.heads, layers=cfg.layers, vocab=cfg.vocab)
    sd = e.model.state_dict()
    sd.update(UO.make_weights(CO.clip_param_specs(cfg), seed=4))
    e.model.load_state_dict(sd)
    e.model.half().cuda()
    tokens = lambda B: torch.randint(0, cfg.vocab, (B, cfg.context), generator=torch.Generator().manual_seed(B))
    _cycled_twice([1, 2, 3, 4, 5], lambda B: e.encode_with_transformer(tokens(B)))       # > the text-tower bound of 4


def test_adapter_evicts_and_rebuilds_plans():
    from t2v_b200.adapter import Adapter
    a = Adapter(**AO.NARROW_A).half()
    a.load_state_dict(UO.make_weights(AO.adapter_param_specs(**AO.NARROW_A), seed=21), strict=True)
    a = a.cuda()
    sizes = [(1, 64, 64), (2, 64, 64), (1, 128, 64), (3, 64, 128), (1, 128, 128)]      # > the adapter bound of 4

    def run(s):
        N, H, W = s
        x = torch.rand((N, 1, H, W), generator=torch.Generator().manual_seed(N * H + W)).cuda()
        return torch.cat([f.reshape(-1) for f in a(x)])
    _cycled_twice(sizes, run)


def test_two_unet_handles_live_side_by_side():
    a = _unet_sd()
    small = _unet_inputs(1, 2, 8, 8)
    ref = a(*small).clone()
    b = _unet_sd()
    b(*_unet_inputs(2, 4, 16, 16))                              # a larger shape: grows b's workspace, drops b's plans
    del b
    gc.collect()
    assert torch.equal(a(*small), ref)


def test_two_vae_handles_live_side_by_side():
    a = _vae()
    ref = a.decode(_latent(2)).clone()
    b = _vae()
    b.decode(_latent(6, 16, 16))                                # a larger shape: grows b's workspace, drops b's plans
    del b
    gc.collect()
    assert torch.equal(a.decode(_latent(2)), ref)
