"""GPU: VideoCrafter's depth adapter on the library -- the Adapter network (csrc/adapter.cu), the UNet plan variant that adds
its features (csrc/unet.cu), the sampler and `adapter_guided_synthesis` -- against the CPU restatement
(tests/adapter_oracle.py) and the reference fixture (tests/golden/adapter.pt)."""
import ctypes as C
import os

import pytest
import torch

from oracle import unet_oracle as UO, vae_oracle as VO, vc_oracle as VC
import adapter_oracle as AO
from parity_util import report

pytestmark = pytest.mark.gpu

UNET_KW = dict(model_channels=64, context_dim=48, temporal_length=4)
CFG = VC.VCConfig(**UNET_KW)
GATE = 5e-3                       # the VideoCrafter UNet gate of tests/test_videocrafter_gpu.py


@pytest.fixture(scope='module')
def gold(gold_dir):
    return torch.load(os.path.join(gold_dir, 'adapter.pt'))


def _half(W):
    return {k: v.half().float() for k, v in W.items()}


def _adapter(cfg, seed):
    from t2v_b200.adapter import Adapter
    W = UO.make_weights(AO.adapter_param_specs(**cfg), seed=seed)
    a = Adapter(**cfg).half()
    a.load_state_dict(W, strict=True)
    return a.cuda(), W


def _rel(out, ref):
    out, ref = out.float().cpu(), ref.float().cpu()
    return ((out - ref).pow(2).mean().sqrt() / ref.pow(2).mean().sqrt()).item(), ((out - ref).abs().max() / ref.abs().max()).item()


@pytest.mark.parametrize('name', ['A', 'B', 'depth'])
def test_adapter_features_vs_oracle_and_graph_replay(gold, name):
    cfg = {'A': AO.NARROW_A, 'B': AO.NARROW_B, 'depth': AO.DEPTH}[name]
    a, W = _adapter(cfg, {'A': 21, 'B': 22, 'depth': 23}[name])
    d = gold['depth']
    x = d.permute(0, 2, 1, 3, 4).reshape(-1, 1, 64, 64)
    first = [f.clone() for f in a(x.cuda())]
    second = a(x.cuda())
    ref = AO.adapter_forward(_half(W), x.half().float(), **cfg)
    worst = (0.0, 0.0)
    for i, (o, r) in enumerate(zip(first, ref)):
        assert o.shape == r.shape and o.dtype == torch.float16
        assert o.permute(0, 2, 3, 1).is_contiguous()                          # channels-last view of the library output
        rms, mx = _rel(o, r)
        worst = (max(worst[0], rms), max(worst[1], mx))
        assert torch.equal(o, second[i])                                       # the graph replay is bit-identical
    report(f'adapter_{name}', rel_rms=worst[0], max_rel=worst[1])
    assert worst[0] < 3e-3 and worst[1] < 1e-2, worst
    if name == 'A':                                                            # and the oracle is the reference's output
        rms, mx = _rel(AO.to_video_features(ref, 1, 4)[3], gold['features_A'][3])
        assert mx < 1e-2


def test_adapter_encode_errors():
    a, _ = _adapter(AO.NARROW_A, 21)
    l = __import__('t2v_b200._lib', fromlist=['lib']).lib()
    x = torch.zeros(1, 1, 60, 64, device='cuda')
    outs = (C.c_void_p * 4)(*[0, 0, 0, 0])
    assert l.t2v_adapter_encode(a._handle, C.c_void_p(x.data_ptr()), 1, outs, 1, 60, 64, None) != 0
    assert b'multiple' in l.t2v_last_error()
    assert l.t2v_adapter_encode(a._handle, C.c_void_p(x.data_ptr()), 1, outs, 1, 80, 48, None) != 0
    assert b'empty' in l.t2v_last_error()


@pytest.fixture(scope='module')
def net():
    from t2v_b200.modules import UNetModel
    W = UO.make_weights(VC.vc_param_specs(CFG), seed=4)
    m = UNetModel(**UNET_KW).half()
    m.load_state_dict(W, strict=True)
    return m.cuda().eval(), W


def _inputs(gold):
    B, _, T, h, w = gold['shape']
    x = torch.randn(gold['shape'], generator=torch.Generator().manual_seed(gold['seeds']['x']))
    ctx = torch.randn((B, gold['L'], 48), generator=torch.Generator().manual_seed(gold['seeds']['ctx']))
    return x.cuda(), gold['t'].cuda(), ctx.cuda()


def test_unet_with_features_vs_reference_and_oracle(gold, net):
    m, W = net
    x, t, ctx = _inputs(gold)
    feats = [f.cuda() for f in gold['features_A']]
    e1 = m(x, t, context=ctx, features_adapter=feats).float().cpu()
    e0 = m(x, t, context=ctx).float().cpu()
    _, err_ref = _rel(e1, gold['eps_features'])
    orc = AO.vc_unet_forward(_half(W), CFG, x.cpu(), t.cpu(), ctx.cpu().half().float(), [f.half().float() for f in gold['features_A']])
    _, err_orc = _rel(e1, orc)
    moved = ((e1 - e0).abs().max() / e1.abs().max()).item()
    report('vc_unet_features', vs_reference=err_ref, vs_oracle=err_orc, moved=moved)
    assert err_ref < GATE and err_orc < GATE, (err_ref, err_orc)
    assert moved > 20 * GATE                                                   # the comparison is not vacuous
    e1b = m(x, t, context=ctx, features_adapter=feats).float().cpu()           # graph replay of the feature plan
    assert torch.equal(e1, e1b)


def test_zero_features_equal_no_features(gold, net):
    m, _ = net
    x, t, ctx = _inputs(gold)
    ref = m(x, t, context=ctx)
    zeros = [torch.zeros((1,) + s, device='cuda', dtype=torch.float16) for s in m.feature_shapes(*x.shape[2:])]
    assert torch.equal(m(x, t, context=ctx, features_adapter=zeros), ref)


def test_feature_plan_leaves_the_default_plan_alone_and_restages(gold, net):
    from t2v_b200.modules import UNetModel
    m, W = net
    x, t, ctx = _inputs(gold)
    fresh = UNetModel(**UNET_KW).half()
    fresh.load_state_dict(W, strict=True)
    fresh = fresh.cuda().eval()
    want = fresh(x, t, context=ctx)
    f1 = [f.cuda() for f in gold['features_A']]
    a = m(x, t, context=ctx, features_adapter=f1).clone()
    assert torch.equal(m(x, t, context=ctx), want)                            # no features after features: the default plan
    f2 = [f.clone() * 0.5 for f in f1]
    b = m(x, t, context=ctx, features_adapter=f2)
    assert not torch.equal(a, b)                                               # new feature tensors are staged, not stale ones
    for f in f1:
        f.mul_(0.5)                                                            # in place: the channels-last copy is refreshed
    assert torch.equal(m(x, t, context=ctx, features_adapter=f1), b)


def test_batched_cfg_pair_with_features_equals_single_runs(gold, net):
    m, _ = net
    x, t, ctx = _inputs(gold)
    uc = torch.randn_like(ctx)
    feats = [f.cuda() for f in gold['features_A']]
    pair = m(torch.cat([x, x]), torch.cat([t, t]), context=torch.cat([ctx, uc]), features_adapter=feats, features_adapter_tiled=True)
    c1 = m(x, t, context=ctx, features_adapter=feats)
    u1 = m(x, t, context=uc, features_adapter=feats)
    _, ec = _rel(pair[:1], c1)
    _, eu = _rel(pair[1:], u1)
    report('vc_unet_features_pair', cond=ec, uncond=eu)
    assert ec < 1e-3 and eu < 1e-3
    bcast = m(torch.cat([x, x]), torch.cat([t, t]), context=torch.cat([ctx, uc]), features_adapter=feats)      # batch 1 broadcast
    assert torch.equal(bcast, pair)


def test_library_rejects_bad_feature_calls(net):
    from t2v_b200 import _lib
    from t2v_b200.modules import UNetSD
    m, _ = net
    l = _lib.lib()
    x = torch.zeros(2, 4, 4, 8, 8, device='cuda')
    t = torch.zeros(2, device='cuda')
    ctx = torch.zeros(2, 9, 48, device='cuda', dtype=torch.float16)
    out = torch.empty(2, 4, 4, 8, 8, device='cuda', dtype=torch.float16)
    f = [torch.zeros((1,) + s, device='cuda', dtype=torch.float16) for s in m.feature_shapes(4, 8, 8)]
    ptrs = (C.c_void_p * 4)(*[v.data_ptr() for v in f])
    P = _lib.ptr

    def call(handle, n, fb, B=2):
        return l.t2v_unet_forward_adapter(handle, P(x), 1, P(t), P(ctx), ptrs, n, fb, P(out), 0, B, 4, 8, 8, 9, None)
    assert call(m._handle, 3, 1) != 0 and b'4 input blocks' in l.t2v_last_error()
    assert call(m._handle, 4, 3) != 0 and b'does not divide' in l.t2v_last_error()
    sd = UNetSD(dim=64)
    assert call(sd._handle, 4, 1) != 0 and b'arch 1' in l.t2v_last_error()


@pytest.fixture(scope='module')
def ldm():
    from t2v_b200.videocrafter import T2VAdapterDepth
    W = UO.make_weights(VC.vc_param_specs(CFG), seed=4)
    Wa = UO.make_weights(AO.adapter_param_specs(**AO.NARROW_A), seed=21)
    Wv = UO.make_weights(VO.decoder_param_specs(VO.VAEConfig()), seed=3)
    m = T2VAdapterDepth(None, dict(params=AO.NARROW_A, cond_name='depth'), unet_config=UNET_KW, image_size=[8, 8], video_length=4,
                        depth_stage_model=AO.StubDepth()).half()
    m.model.diffusion_model.load_state_dict(W, strict=True)
    m.adapter.load_state_dict(Wa, strict=True)
    m.first_stage_model.load_state_dict(Wv, strict=False)
    return m.cuda().eval()


@pytest.mark.parametrize('eta', [0.0, 0.5])
def test_ddim_trajectory_with_features_vs_reference(gold, ldm, eta):
    from t2v_b200.videocrafter import DDIMSampler
    depth = gold['depth'].cuda()
    feats = ldm.get_adapter_features(depth)
    smp = DDIMSampler(ldm)
    smp.noise_gen.manual_seed(gold['seeds']['noise'])
    out, _ = smp.sample(S=4, batch_size=1, shape=(4, 4, 8, 8), conditioning=gold['c'].cuda(), x_T=gold['x_T'].cuda(), eta=eta,
                        unconditional_guidance_scale=5.0, unconditional_conditioning=gold['uc'].cuda(), verbose=False,
                        features_adapter=feats, temporal_length=4, conditional_guidance_scale_temporal=None)
    ref = gold[f'ddim_eta{eta}']
    err = ((out.cpu() - ref).abs().max() / ref.abs().max()).item()
    report(f'vc_ddim_features_eta{eta}', max=err)
    assert err < GATE, err


def test_adapter_guided_synthesis_shapes(ldm):
    from t2v_b200.videocrafter import adapter_guided_synthesis
    g = torch.Generator().manual_seed(8)
    c, uc = torch.randn(1, 9, 48, generator=g), torch.randn(1, 9, 48, generator=g)
    ldm.cond_stage_model = lambda prompts: (uc if prompts == [''] else c).cuda()
    video = (torch.rand(1, 3, 4, 64, 64, generator=g) * 2 - 1).cuda()
    x_T = torch.randn(1, 4, 4, 8, 8, generator=g).cuda()
    samples, extra = adapter_guided_synthesis(ldm, 'a prompt', video, [1, 4, 4, 8, 8], n_samples=2, ddim_steps=4, ddim_eta=0.0,
                                              unconditional_guidance_scale=4.0, x_T=x_T)
    assert samples.shape == (1, 2, 3, 4, 64, 64) and extra.shape == (1, 1, 4, 64, 64)
    assert torch.equal(samples[:, 0], samples[:, 1])                           # eta 0, same x_T: deterministic
    assert extra.min() >= -1 - 1e-6 and extra.max() <= 1 + 1e-6
