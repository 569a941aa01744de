"""GPU parity at BASELINE.json's own configurations, through the C ABI.

Three yardsticks per case (all printed as `[parity] {...}` lines; T2V_PARITY_REPORT=<file> records them):
  1. the REFERENCE's fp32 CPU output committed in tests/golden (written by oracle/make_golden.py from the unmodified
     reference modules) -- relative RMS and max error of our fp16 path against it, gated by the constants below (the
     values measured on H100 are listed beside them and in DESIGN.md section 5);
  2. the reference's GPU numerics contract: the same torch ops under fp16 autocast + SDPA on the same GPU
     (parity_util.AutocastOracle).  Gate: err(ours, fp32 fixture) <= 1.5 x err(autocast path, fp32 fixture) -- i.e. we are
     at least as close to the fp32 truth as the reference's own fp16 path is (up to the stated slack);
  3. BASELINE.json's element-wise gate rtol 1e-3 / atol 1e-4: the pass rate is REPORTED for both paths (no fp16 path meets
     it end to end against fp32 -- the autocast numbers printed beside ours are the evidence).
"""
import os

import pytest
import torch

from oracle import unet_oracle as UO, samplers_oracle as SO, vc_oracle as VC
from oracle.make_golden import synth_inputs
from parity_util import AutocastOracle, errs, first_update, on_fixture_frames, pass_rate, report

pytestmark = pytest.mark.gpu

SLACK = 1.5
# relative-RMS error of eps vs the reference's fp32 output, measured on H100 (T2V_PARITY_REPORT): tiny 2.45e-3, cfg1 2.88e-3,
# cfg2 2.85e-3, cfg3 slice 2.68e-3, 125 frames 2.99e-3, VC cfg5 2.07e-3
GATE_RMS = {'unet_tiny': 4.0e-3, 'unet_cfg1': 4.4e-3, 'unet_cfg2': 4.3e-3, 'unet_cfg3_slice': 4.0e-3, 'unet_f125': 4.5e-3,
            'vc_unet_cfg5': 3.1e-3}
# max |err| / max |ref|, measured on H100 2.4e-3 / 3.4e-3 / 2.7e-3 / 2.9e-3 / 3.7e-3 / 2.2e-3
GATE_MAX = {'unet_tiny': 3.6e-3, 'unet_cfg1': 4.4e-3, 'unet_cfg2': 4.7e-3, 'unet_cfg3_slice': 4.1e-3, 'unet_f125': 5.3e-3,
            'vc_unet_cfg5': 3.3e-3}
# latent after ONE scheduler update vs the reference sampler's, measured on H100 (cfg1 / cfg2): DDIM_Gaussian 1.75e-3 rms /
# 2.8e-3 max, DDIM 2.4e-3 / 2.8e-3; UniPC (the latent handed to the 5th model call: corrector of update 1 + predictor of update 2, i.e.
# differences of x0-predictions at sigma/alpha ~ 15) 7.2e-3 / 8.5e-3.  Its scheduler arithmetic is pinned on the CPU
# (tests/test_samplers_host_cpu.py: product host algebra == oracle to 1e-7 with fp16 eps); the rest is fp16 rounding noise of the
# denoiser re-rolled by the UniPC update (scripts/diag_unipc.py: a 3.5e-8 change of x moves the fp16 eps by 2.4e-3)
GATE_STEP = {'ddim_gaussian_x1': (2.7e-3, 4.5e-3), 'ddim_x1': (3.8e-3, 4.7e-3), 'unipc_x1': (1.07e-2, 1.03e-2)}


def _full_net(wseed=0):
    from t2v_b200.modules import UNetSD
    cfg = UO.UNetConfig()
    W = UO.make_weights(UO.param_specs(cfg), seed=wseed)
    with torch.device('cuda'):
        net = UNetSD()
    net = net.half()
    net.load_state_dict(W, strict=True)
    net = net.cuda().eval()
    betas = SO.linear_sd_betas()
    net.register_schedule(given_betas=betas.numpy())
    return cfg, W, net, betas


@pytest.fixture(scope='module')
def full():
    cfg, W, net, betas = _full_net()
    ac = AutocastOracle(W, cfg)
    yield cfg, W, net, betas, ac
    del net, ac
    torch.cuda.empty_cache()


def _gate_forward(name, ours, autocast, ref):
    e, a = errs(ours, ref), errs(autocast, ref)
    report(name, ours_max=e[0], ours_rms=e[1], autocast_max=a[0], autocast_rms=a[1],
           ours_pass_1e3=pass_rate(ours, ref), autocast_pass_1e3=pass_rate(autocast, ref),
           ours_vs_autocast_rms=errs(ours, autocast)[1])
    assert e[1] <= SLACK * a[1], f'{name}: rel-RMS {e[1]:.3e} vs the autocast path {a[1]:.3e}'
    key = name.split(':')[0]
    assert e[1] <= GATE_RMS[key] and e[0] <= GATE_MAX[key], (name, e)


def _sampler(name, model, betas):
    from t2v_b200 import samplers
    entry = [s for s in samplers.available_samplers if s.name == name][0]
    return entry.init_sampler(model, betas=betas, device=torch.device('cuda'))


def _gate_step(case, g, net, betas, ac):
    """One update of each scheduler from x_T on the full model: the latent after the first update against the one the
    REFERENCE sampler classes produced (fixture), with the autocast path's own step error as the yardstick."""
    F, h, w = g['F'], g['h'], g['w']
    x, c, uc = synth_inputs(F, h, w)
    xg, cg, ucg = x.cuda(), c.cuda(), uc.cuda()
    kw = dict(conditioning=cg, unconditional_conditioning=ucg, unconditional_guidance_scale=17.0, x_T=xg, shape=tuple(x.shape),
              eta=0.0, batch_size=1)
    acm = lambda a, b, d: ac(a, b, d)       # noqa: E731
    runs = {
        'ddim_gaussian_x1': ('DDIM_Gaussian', 50, 3, lambda m: SO.ddim_gaussian_sample(m, betas, xg, 50, cg, ucg, 17.0)),
        'ddim_x1': ('DDIM', 50, 3, lambda m: SO.ddim_sample(m, betas, xg, 50, cg, ucg, 17.0)),
        'unipc_x1': ('UniPC', 30, 5, None),
    }
    for key, (sname, S, stop_at, oracle_run) in runs.items():
        if key not in g:
            continue
        ours = on_fixture_frames(first_update(lambda m: _sampler(sname, m, betas).sample(S=S, **kw), net, stop_at), g)
        e = errs(ours, g[key])
        rec = dict(ours_max=e[0], ours_rms=e[1], ours_pass_1e3=pass_rate(ours, g[key]))
        if oracle_run is not None:
            auto = on_fixture_frames(first_update(oracle_run, acm, stop_at), g)
            a = errs(auto, g[key])
            rec.update(autocast_max=a[0], autocast_rms=a[1], autocast_pass_1e3=pass_rate(auto, g[key]))
        report(f'{case}:{key}', **rec)
        if oracle_run is not None:
            assert e[1] <= SLACK * a[1] + 1e-6, (key, e, a)
        assert e[1] <= GATE_STEP[key][0] and e[0] <= GATE_STEP[key][1], (key, e)
    # the batched cond+uncond forward the samplers use in production (one B = 2 call) gives the same update
    smp = _sampler('DDIM_Gaussian', net, betas)
    from t2v_b200 import samplers as S_
    seen = {}
    orig = S_._step_kernel

    class Stop(Exception):
        pass

    def spy(*a, **k):
        seen['x1'] = orig(*a, **k)
        raise Stop()
    S_._step_kernel = spy
    try:
        smp.sample(S=50, **kw)
    except Stop:
        pass
    finally:
        S_._step_kernel = orig
    eb = errs(on_fixture_frames(seen['x1'], g), g['ddim_gaussian_x1'])
    report(f'{case}:ddim_gaussian_x1:batched_B2', ours_max=eb[0], ours_rms=eb[1])
    assert eb[1] <= GATE_STEP['ddim_gaussian_x1'][0] and eb[0] <= GATE_STEP['ddim_gaussian_x1'][1], eb


def test_config1_forward_and_single_step(full, gold_dir):
    """BASELINE config 1 (the stated parity gate): ModelScope UNetSD, 4 frames x 128^2, one step of every scheduler."""
    cfg, W, net, betas, ac = full
    g = torch.load(os.path.join(gold_dir, 'unet_cfg1.pt'))
    x, c, uc = synth_inputs(g['F'], g['h'], g['w'])
    t = torch.tensor([g['t']])
    for tag, ctx, key in (('cond', c, 'eps_cond'), ('uncond', uc, 'eps_uncond')):
        _gate_forward(f'unet_cfg1:{tag}', net(x.cuda(), t.cuda(), ctx.cuda()), ac(x, t, ctx), g[key])
    _gate_step('unet_cfg1', g, net, betas, ac)


def test_config2_forward_and_single_step(full, gold_dir):
    """BASELINE config 2's shape -- 24 frames x 256^2, the shape every bench number is quoted on (different tile counts,
    split-K decisions, attention_tc at S = 1024 than config 1).  The fixture keeps a fixed subset of the 24 frames; the
    network still runs all of them."""
    cfg, W, net, betas, ac = full
    g = torch.load(os.path.join(gold_dir, 'unet_cfg2.pt'))
    x, c, uc = synth_inputs(g['F'], g['h'], g['w'])
    t = torch.tensor([g['t']])
    outs = {}
    for tag, ctx, key in (('cond', c, 'eps_cond'), ('uncond', uc, 'eps_uncond')):
        outs[tag] = on_fixture_frames(net(x.cuda(), t.cuda(), ctx.cuda()), g)
        _gate_forward(f'unet_cfg2:{tag}', outs[tag], on_fixture_frames(ac(x, t, ctx), g), g[key])
    # the production B = 2 forward (cond + uncond in one call) against the two B = 1 forwards
    both = on_fixture_frames(net(x.cuda().expand(2, -1, -1, -1, -1), t.cuda().expand(2), torch.cat([c, uc]).cuda()), g)
    eb = errs(both[0:1], g['eps_cond']), errs(both[1:2], g['eps_uncond'])
    report('unet_cfg2:B2', cond_rms=eb[0][1], uncond_rms=eb[1][1], b2_vs_b1_rms=errs(both[0:1], outs['cond'])[1])
    assert max(eb[0][1], eb[1][1]) <= GATE_RMS['unet_cfg2']
    _gate_step('unet_cfg2', g, net, betas, ac)


def test_config3_sequence_length_slice(full, gold_dir):
    """Config 3's spatial sequence length (576 x 1024 -> S = 9216 tokens per frame, attention_tc's long-sequence regime)
    through the full model on 2 frames."""
    cfg, W, net, betas, ac = full
    g = torch.load(os.path.join(gold_dir, 'unet_cfg3_slice.pt'))
    x, c, uc = synth_inputs(g['F'], g['h'], g['w'])
    _gate_forward('unet_cfg3_slice', net(x.cuda(), g['t'].cuda(), c.cuda()), ac(x, g['t'], c), g['eps'])


def test_config4_frame_count_narrow_net(gold_dir):
    """Config 4's frame count (125) through temporal conv / temporal attention / 5-D GroupNorm on the dim-64 net, B = 2."""
    from t2v_b200.modules import UNetSD
    g = torch.load(os.path.join(gold_dir, 'unet_f125.pt'))
    cfg = UO.UNetConfig(dim=64)
    W = UO.make_weights(UO.param_specs(cfg), seed=g['wseed'])
    net = UNetSD(dim=64).half()
    net.load_state_dict(W, strict=True)
    net = net.cuda().eval()
    x, c, uc = synth_inputs(g['F'], g['h'], g['w'])
    x = torch.cat([x, x.flip(2) * 0.5], 0)
    ctx = torch.cat([c, uc], 0)
    _gate_forward('unet_f125', net(x.cuda(), g['t'].cuda(), ctx.cuda()), AutocastOracle(W, cfg)(x, g['t'], ctx), g['eps'])


def test_config5_videocrafter_shape(gold_dir):
    """Config 5's per-GPU shape: VideoCrafter UNetModel (958.9 M params), 16 frames x 256^2."""
    from t2v_b200.modules import UNetModel
    g = torch.load(os.path.join(gold_dir, 'vc_unet_cfg5.pt'))
    cfg = VC.VCConfig(**g['cfg'])
    W = UO.make_weights(VC.vc_param_specs(cfg), seed=g['wseed'])
    with torch.device('cuda'):
        net = UNetModel(model_channels=cfg.model_channels, context_dim=cfg.context_dim, temporal_length=cfg.temporal_length)
    net = net.half()
    net.load_state_dict(W, strict=True)
    net = net.cuda().eval()
    B = g['shape'][0]
    x = torch.randn(g['shape'], generator=torch.Generator('cpu').manual_seed(g['x_seed']))
    ctx = torch.randn((B, g['L'], cfg.context_dim), generator=torch.Generator('cpu').manual_seed(g['ctx_seed']))
    ours = net(x.cuda(), g['t'].cuda(), context=ctx.cuda())
    # scripts/videocrafter never enables autocast or .half(): the reference's own GPU path for this model is fp32 (einsum
    # attention, attention_temporal.py:167-190).  BASELINE config 5 asks for fp16, so the yardstick is the same op sequence
    # under fp16 autocast -- what the reference would compute if it were switched to half precision.
    ac = AutocastOracle(W, cfg, forward=VC.vc_unet_forward, attn_impl='math')
    _gate_forward('vc_unet_cfg5', ours, ac(x, g['t'], ctx), g['out'])


def test_tiny_block_taps_vs_autocast(gold_dir):
    """Per-module taps of the dim-64 net: our activation error against the reference fp32 taps vs the autocast path's."""
    from t2v_b200.modules import UNetSD
    g = torch.load(os.path.join(gold_dir, 'unet_tiny.pt'))
    cfg = UO.UNetConfig(dim=64)
    W = UO.make_weights(UO.param_specs(cfg), seed=g['wseed'])
    net = UNetSD(dim=64).half()
    net.load_state_dict(W, strict=True)
    net = net.cuda().eval()
    x, c, uc = synth_inputs(g['F'], g['h'], g['w'])
    t = torch.tensor([g['t']])
    net.enable_taps(True)
    out = net(x.cuda(), t.cuda(), c.cuda())
    taps = {}
    auto = AutocastOracle(W, cfg)(x, t, c, taps=taps)
    worst = 0.0
    for k, v in g.items():
        if not k.startswith('tap:'):
            continue
        e = errs(net.read_tap(k[4:], tuple(v.shape)), v)
        a = errs(taps[k[4:]], v)
        report('unet_tiny:' + k, ours_rms=e[1], autocast_rms=a[1])
        # single modules early in the net sit at the fp16 rounding floor where the ratio is noisy: absolute floor 1e-3
        assert e[1] <= max(SLACK * a[1], 1e-3), (k, e, a)
        worst = max(worst, e[1])
    net.enable_taps(False)
    _gate_forward('unet_tiny', out, auto, g['eps_cond'])
