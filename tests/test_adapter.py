"""CPU: VideoCrafter's depth adapter path.  The restatement (tests/adapter_oracle.py) against the reference's own classes
(tests/golden/adapter.pt, written by scripts/make_golden_adapter.py); the library's parameter tables against the reference
Adapter's; T2VAdapterDepth's layout and depth preprocessing; the errors raised before anything reaches the GPU."""
import os

import pytest
import torch

from oracle import unet_oracle as UO, vc_oracle as VC, samplers_oracle as SO
import adapter_oracle as AO


@pytest.fixture(scope='module')
def gold(gold_dir):
    return torch.load(os.path.join(gold_dir, 'adapter.pt'))


def _frames(g):
    d = g['depth']                                                       # b c t h w
    b, c, t, h, w = d.shape
    return d.permute(0, 2, 1, 3, 4).reshape(b * t, c, h, w), b, t


@pytest.mark.parametrize('name', ['A', 'B'])
def test_oracle_adapter_matches_reference(gold, name):
    cfg = gold['configs'][name]
    W = UO.make_weights(AO.adapter_param_specs(**cfg), seed=gold['seeds'][name])
    x, b, t = _frames(gold)
    out = AO.to_video_features(AO.adapter_forward(W, x, **cfg), b, t)
    ref = gold['features_' + name]
    assert [tuple(f.shape) for f in out] == [tuple(f.shape) for f in ref]
    for o, r in zip(out, ref):
        assert torch.allclose(o, r, rtol=0, atol=1e-5), (o - r).abs().max()


def _unet_setup(gold):
    cfg = VC.VCConfig(**gold['unet_cfg'])
    W = UO.make_weights(VC.vc_param_specs(cfg), seed=gold['seeds']['unet'])
    B, _, T, h, w = gold['shape']
    x = torch.randn(gold['shape'], generator=torch.Generator().manual_seed(gold['seeds']['x']))
    ctx = torch.randn((B, gold['L'], cfg.context_dim), generator=torch.Generator().manual_seed(gold['seeds']['ctx']))
    return cfg, W, x, ctx


def test_oracle_unet_with_and_without_features_matches_reference(gold):
    cfg, W, x, ctx = _unet_setup(gold)
    e0 = AO.vc_unet_forward(W, cfg, x, gold['t'], ctx)
    e1 = AO.vc_unet_forward(W, cfg, x, gold['t'], ctx, gold['features_A'])
    assert torch.allclose(e0, gold['eps'], rtol=0, atol=1e-5)
    assert torch.allclose(e1, gold['eps_features'], rtol=0, atol=1e-5)
    assert torch.equal(e0, VC.vc_unet_forward(W, cfg, x, gold['t'], ctx))        # no features: vc_oracle's forward
    assert (e1 - e0).abs().max() > 0.1 * e1.abs().max()                           # the features matter


@pytest.mark.parametrize('eta', [0.0, 0.5])
def test_oracle_ddim_trajectory_matches_reference(gold, eta):
    cfg, W, _, _ = _unet_setup(gold)
    o = AO.vc_ddim_sample(W, cfg, SO.linear_sd_betas(), gold['x_T'], 4, gold['c'], gold['uc'], 5.0, eta,
                          torch.Generator('cpu').manual_seed(gold['seeds']['noise']), gold['features_A'])
    r = gold[f'ddim_eta{eta}']
    assert (o - r).abs().max() <= 1e-5 * max(1.0, r.abs().max().item())


def _meta_adapter(**cfg):
    from t2v_b200.adapter import Adapter
    with torch.device('meta'):
        return Adapter(**cfg)


@pytest.mark.parametrize('which', ['depth', 'sk'])
def test_adapter_state_dict_matches_reference_tables(gold, which):
    cfg = AO.DEPTH if which == 'depth' else dict(AO.DEFAULTS, sk=True)
    sd = _meta_adapter(**cfg).state_dict()
    ref = gold['table_' + which]
    assert {k: tuple(v.shape) for k, v in sd.items()} == ref
    assert {k: tuple(v) for k, v in AO.adapter_param_specs(**cfg).items()} == ref
    assert len(ref) == (38 if which == 'depth' else 60)


def test_adapter_rejects_configs_the_reference_cannot_run():
    from t2v_b200.adapter import Adapter
    with pytest.raises(ValueError, match='sk=False'):
        Adapter()                                             # the class defaults: sk=False with widths 320 -> 640
    with pytest.raises(ValueError, match='multiple of 64'):
        Adapter(channels=[64, 64], cin=32, sk=True)
    a = _meta_adapter(channels=[64, 64, 64], nums_rb=2, ksize=3, sk=False, use_conv=True)          # sk=False, equal widths: runs
    assert 'body.0.skep.weight' in a.state_dict() and 'body.2.down_opt.op.weight' in a.state_dict()


def test_adapter_level_sizes_and_empty_levels():
    a = _meta_adapter(**AO.NARROW_A)
    assert a.feature_sizes(64, 64) == [(8, 8), (4, 4), (2, 2), (1, 1)]
    assert a.feature_sizes(96, 64) == [(12, 8), (6, 4), (3, 2), (1, 1)]
    for H, W in ((80, 48), (72, 40)):                         # 10x6 -> 5x3 -> 2x1 -> 1x0, 9x5 -> 4x2 -> 2x1 -> 1x0
        with pytest.raises(ValueError, match='level 3 .* would be empty'):
            a.feature_sizes(H, W)
    with pytest.raises(ValueError, match='multiple of 8'):
        a.feature_sizes(60, 64)
    assert _meta_adapter(**AO.NARROW_B).feature_sizes(80, 48) == [(10, 6), (5, 3), (3, 2), (2, 1)]     # stride-2 convs round up


def _tiny_unet():
    from t2v_b200.modules import UNetModel
    return UNetModel(model_channels=64, context_dim=48, temporal_length=4)


def test_unet_feature_shapes_and_mismatches_are_loud():
    """A 10x6 latent: the UNet's levels are 10x6, 5x3, 3x2, 2x1; an average-pooling adapter gives 5x3 -> 2x1 at levels 1, 2,
    which must be an error rather than a misaligned add."""
    net = _tiny_unet()
    assert net.feature_shapes(4, 10, 6) == [(64, 4, 10, 6), (128, 4, 5, 3), (256, 4, 3, 2), (256, 4, 2, 1)]
    x, t, ctx = torch.randn(2, 4, 4, 10, 6), torch.tensor([5, 5]), torch.randn(2, 9, 48)
    pooled = [torch.zeros(1, c, 4, h, w) for c, (h, w) in zip((64, 128, 256, 256), ((10, 6), (5, 3), (2, 1), (1, 0)))]
    with pytest.raises(ValueError, match='does not match'):
        net(x, t, context=ctx, features_adapter=pooled)
    good = [torch.zeros(1, *s) for s in net.feature_shapes(4, 10, 6)]
    with pytest.raises(ValueError, match='got 3 feature maps'):
        net(x, t, context=ctx, features_adapter=good[:3])
    with pytest.raises(ValueError, match='does not broadcast'):
        net(torch.randn(3, 4, 4, 10, 6), torch.tensor([5] * 3), context=torch.randn(3, 9, 48),
            features_adapter=[f.expand(2, -1, -1, -1, -1) for f in good])
    with pytest.raises(NotImplementedError):
        net(x, t, context=ctx, time_emb_replace=torch.zeros(2, 256))


def _t2v_adapter_depth(**kw):
    from t2v_b200.videocrafter import T2VAdapterDepth
    return T2VAdapterDepth(dict(target='lvdm.models.modules.midas.api.MiDaSInference', params=dict(model_type='dpt_hybrid')),
                           dict(target='lvdm.models.modules.adapter.Adapter', cond_name='depth', params=AO.NARROW_A),
                           unet_config=dict(model_channels=64, context_dim=48, temporal_length=4), image_size=[8, 8],
                           video_length=4, **kw)


def test_t2v_adapter_depth_layout_and_depth_preprocessing(gold):
    m = _t2v_adapter_depth(depth_stage_model=AO.StubDepth())
    assert m.condtype == 'depth'
    sd = m.state_dict()
    adapter_keys = {k[len('adapter.'):] for k in sd if k.startswith('adapter.')}
    assert adapter_keys == set(AO.adapter_param_specs(**AO.NARROW_A))
    assert 'model.diffusion_model.input_blocks.0.0.weight' in sd and 'alphas_cumprod' in sd
    d = m.get_batch_depth(gold['video'], tuple(gold['video'].shape[-2:]))
    assert torch.equal(d, gold['batch_depth'])
    assert torch.equal(m.get_batch_depth(gold['video'], tuple(gold['video'].shape[-2:]), encode_bs=2), gold['batch_depth'])


def test_t2v_adapter_depth_without_a_depth_model_says_what_to_pass():
    with pytest.raises(RuntimeError, match='MiDaS.*depth_stage_model'):
        _t2v_adapter_depth()


def test_load_model_checkpoint_loads_the_adapter_strictly(tmp_path):
    from t2v_b200.videocrafter import load_model_checkpoint
    m = _t2v_adapter_depth(depth_stage_model=AO.StubDepth())
    W = UO.make_weights(AO.adapter_param_specs(**AO.NARROW_A), seed=5)
    main = {k: v for k, v in m.state_dict().items() if not k.startswith('adapter.')}
    torch.save({'state_dict': main}, tmp_path / 'model.ckpt')
    torch.save(W, tmp_path / 'adapter.pth')
    load_model_checkpoint(m, str(tmp_path / 'model.ckpt'), str(tmp_path / 'adapter.pth'))
    assert torch.equal(m.adapter.state_dict()['body.3.block2.weight'], W['body.3.block2.weight'])
    assert m.adapter._dirty                                   # the next encode ships the new weights
    torch.save({k: v for k, v in W.items() if k != 'conv_in.bias'}, tmp_path / 'bad.pth')
    with pytest.raises(RuntimeError, match='conv_in.bias'):
        load_model_checkpoint(m, str(tmp_path / 'model.ckpt'), str(tmp_path / 'bad.pth'))
