"""GPU: every module of the ModelScope and VideoCrafter UNets in isolation, on the input the library fed it, against the
oracle's module in fp64, per (sample, frame), channel group and frame border.

The whole-forward gates (test_model_gpu.py, test_parity_gpu.py) take one relative RMS over the whole eps, so an error
confined to one sample or frame of a B = 2, F = 5 forward moves them by about sqrt(1/10) of its size.  Here each module
is re-run by the oracle from the library's own tap of the module before it (unet_modules.py restates the wiring; its
premise is test_unet_modules_cpu.py), so a module's error is its own, and it is measured per slice:

  rel-RMS(ours - fp64) <= 1.5 x rel-RMS(autocast - fp64) + 2^-11 on every slice, and per module
  max|ours - fp64| <= 1.5 x max|autocast - fp64| + 2^-11 x max|fp64|.

fp64 = the oracle module in fp64 on the fp16-rounded weights; autocast = the same module under fp16 autocast on the fp16
weights, ModelScope's attention through SDPA and VideoCrafter's through its einsums (each reference's own GPU
arithmetic).  1.5 is the factor of the whole-forward gates (DESIGN.md section 5); 2^-11 is one fp16 rounding of the output.
The inputs are structured so that reading another sample's embedding, prompt or frames is an O(1) error: timesteps 999 ..
1, a different prompt per sample, a per-frame latent scale and a per-sample offset.  `-s` prints each config's table."""
import gc
import os

import pytest
import torch

import unet_modules as UM
from oracle import unet_oracle as UO, vc_oracle as VC
from parity_util import report

pytestmark = pytest.mark.gpu

FACTOR, FLOOR = 1.5, 2.0 ** -11

# model: (config, weight seed, prompt length)
MODELS = {
    'ms64': (lambda: UO.UNetConfig(dim=64), 1, 77),
    'ms320': (lambda: UO.UNetConfig(), 0, 77),
    'vc64': (lambda: VC.VCConfig(model_channels=64, context_dim=48, temporal_length=4), 5, 9),
    'vc320': (lambda: VC.VCConfig(**torch.load(os.path.join(os.path.dirname(__file__), 'golden', 'vc_unet_full.pt'))['cfg']), 0, 77),
}
# config: model, B, Bc (prompts; B when absent), F, h, w, fb (adapter feature batch; no features when absent)
CONFIGS = {
    'A': dict(model='ms64', B=2, F=5, h=16, w=24),              # attention_tc at level 0 (S = 384), odd F
    'B': dict(model='ms64', B=4, Bc=2, F=3, h=8, w=8),          # shared prompts: t2v_unet_forward_ctx, kv_batch_div = F B / Bc
    'C1': dict(model='ms64', B=1, F=1, h=8, w=8),               # temporal modules on one frame
    'C33': dict(model='ms64', B=1, F=33, h=8, w=8),             # temporal attention past the 32-frame route edge
    'D': dict(model='ms320', B=2, F=3, h=32, w=32),             # production widths: heads 5/10/20, K up to 2560
    'E': dict(model='vc64', B=2, F=9, h=16, w=16),              # relative positions clamped (F > temporal_length + 1)
    'F': dict(model='vc64', B=2, F=4, h=16, w=16, fb=1),        # adapter features added before the skip push
    'G': dict(model='vc320', B=2, F=16, h=32, w=32),            # the benchmark's per-GPU VideoCrafter shape
}


def _build(key):
    from t2v_b200.modules import UNetSD, UNetModel
    make_cfg, seed, L = MODELS[key]
    cfg = make_cfg()
    if UM.arch_of(cfg) == UM.MS:
        W = UO.make_weights(UO.param_specs(cfg), seed=seed)
        net = UNetSD(dim=cfg.dim).half()
    else:
        W = UO.make_weights(VC.vc_param_specs(cfg), seed=seed)
        net = UNetModel(model_channels=cfg.model_channels, context_dim=cfg.context_dim, temporal_length=cfg.temporal_length).half()
    net.load_state_dict(W, strict=True)
    W16 = {k: v.half().cuda() for k, v in W.items()}
    return cfg, L, net.cuda().eval(), W16


@pytest.fixture(scope='module')
def models():
    """One model alive at a time (the full ModelScope net is 2.8 GB in fp16 and twice held: ours and the yardstick's)."""
    held = {}

    def get(key):
        if key not in held:
            held.clear()
            gc.collect()
            torch.cuda.empty_cache()
            held[key] = _build(key)
        return held[key]
    yield get
    held.clear()


def _forward(net, cfg, x, t, y, feats):
    if UM.arch_of(cfg) == UM.MS:
        return net(x.cuda(), t.cuda(), y.cuda()).clone()
    return net(x.cuda(), t.cuda(), context=y.cuda(), features_adapter=feats, features_adapter_tiled=True).clone()


_conv2d, _conv3d = torch.nn.functional.conv2d, torch.nn.functional.conv3d


def _conv3d_by_frames(x, w, b=None, stride=1, padding=0):
    """F.conv3d as a sum of per-frame conv2d over the kernel's frame taps: torch has no CUDA fp64 conv3d."""
    st, sh, sw = (stride,) * 3 if isinstance(stride, int) else stride
    pt, ph, pw = (padding,) * 3 if isinstance(padding, int) else padding
    N, C, T = x.shape[:3]
    kt = w.shape[2]
    xp = torch.nn.functional.pad(x, (0, 0, 0, 0, pt, pt))
    To = (T + 2 * pt - kt) // st + 1
    y = 0
    for i in range(kt):
        xi = xp[:, :, i:i + st * (To - 1) + 1:st].permute(0, 2, 1, 3, 4).reshape(N * To, C, *x.shape[3:])
        y = y + _conv2d(xi, w[:, :, i], None, (sh, sw), (ph, pw))
    y = y.reshape(N, To, *y.shape[1:]).permute(0, 2, 1, 3, 4)
    return y if b is None else y + b.view(1, -1, 1, 1, 1)


def _oracle(cfg, W, b, x, emb, ctx, B):
    """The oracle's module: fp64 (attention as softmax(q k^T) v, conv3d by frames) or, on fp16 x under autocast, the
    reference's GPU arithmetic (ModelScope's attention through SDPA)."""
    f64 = x.dtype == torch.float64
    old = UO.ATTN_IMPL
    UO.ATTN_IMPL = 'math' if f64 else 'sdpa'
    if f64:
        torch.nn.functional.conv3d = _conv3d_by_frames
    try:
        return UM.run_module(cfg, W, b, x, emb, ctx, B)
    finally:
        UO.ATTN_IMPL = old
        torch.nn.functional.conv3d = _conv3d


def _check_module(cfg, W16, b, xin, ours, emb, ctx, B):
    """(gate ratio, worst slice, our rel-RMS there, autocast's there, max-gate ratio); a ratio > 1 fails."""
    W64 = {k: W16[k].double() for k in UM.module_weights(W16, b)}
    ref = _oracle(cfg, W64, b, xin.double(), emb[0], ctx[0], B)
    with torch.autocast('cuda', dtype=torch.float16):
        ac = _oracle(cfg, {k: W16[k] for k in W64}, b, xin, emb[1], ctx[1], B)
    assert ours.shape == ref.shape == ac.shape, (b.prefix, ours.shape, ref.shape, ac.shape)
    d_ours, d_ac = ours.double() - ref, ac.double() - ref
    ms_ref = UM.slice_mean_squares(ref, B)
    rel_ours = (UM.slice_mean_squares(d_ours, B) / ms_ref).sqrt()
    rel_ac = (UM.slice_mean_squares(d_ac, B) / ms_ref).sqrt()
    ratio = rel_ours / (FACTOR * rel_ac + FLOOR)
    k = int(ratio.argmax())
    max_ratio = d_ours.abs().max().item() / (FACTOR * d_ac.abs().max().item() + FLOOR * ref.abs().max().item())
    name = UM.slice_names(ref.shape, B)[k]
    return ratio[k].item(), name, rel_ours[k].item(), rel_ac[k].item(), max_ratio


@pytest.mark.parametrize('name', list(CONFIGS))
def test_every_module_vs_fp64_per_slice(models, name):
    c = CONFIGS[name]
    cfg, L, net, W16 = models(c['model'])
    B, Fr, h, w = c['B'], c['F'], c['h'], c['w']
    Bc = c.get('Bc', B)
    x, t, y = UM.structured_inputs(cfg, B, Fr, h, w, L, Bc, seed=len(name) * 100 + ord(name[0]))
    feats = None
    if 'fb' in c:
        g = torch.Generator().manual_seed(11)
        feats = [torch.randn(s, generator=g).half().cuda() for s in UM.feature_shapes(cfg, c['fb'], Fr, h, w)]

    # one forward with taps (no arena reuse, no graph); the same forward on the production plan must be bit-identical
    net.enable_taps(True)
    try:
        eps = _forward(net, cfg, x, t, y, feats)
        taps = {n: net.read_tap_auto(n) for n in UM.tap_names(cfg)}
    finally:
        net.enable_taps(False)
    assert torch.equal(taps['out'], eps.permute(0, 2, 1, 3, 4).reshape(B * Fr, -1, h, w))
    for _ in range(2):                   # plan build + first run, then graph replay
        assert torch.equal(_forward(net, cfg, x, t, y, feats), eps)

    ctx = y.repeat_interleave(B // Bc, dim=0).cuda()           # sample j reads prompt j // (B / Bc)
    emb64 = UM.time_embedding(cfg, {k: v.double() for k, v in W16.items() if k.startswith('time_embed.')}, t.cuda())
    with torch.autocast('cuda', dtype=torch.float16):
        emb16 = UM.time_embedding(cfg, W16, t.cuda())
    rows, failed = [], []
    with torch.no_grad():
        for b, xin in UM.module_inputs(cfg, taps, x, feats):
            r = _check_module(cfg, W16, b, xin, taps[b.prefix], (emb64, emb16), (ctx.double(), ctx.half()), B)
            rows.append((b.prefix,) + r)
            if (r[0] > 1.0 or r[4] > 1.0) and not failed:
                failed.append(rows[-1])
    print(f'\n[{name}] {"module":44s} {"worst slice":30s} {"ours":>9s} {"autocast":>9s} {"gate":>6s} {"max gate":>8s}')
    for m, ratio, sl, eo, ea, mr in rows:
        print(f'[{name}] {m:44s} {sl:30s} {eo:9.2e} {ea:9.2e} {ratio:6.3f} {mr:8.3f}')
    worst = max(rows, key=lambda r: r[1])
    report(f'unet_modules:{name}', modules=len(rows), worst_module=worst[0], worst_slice=worst[2], worst_gate_ratio=worst[1],
           ours_rel_rms=worst[3], autocast_rel_rms=worst[4], worst_max_gate_ratio=max(r[5] for r in rows))
    assert len(rows) == len(UM.tap_names(cfg))
    if failed:
        m, ratio, sl, eo, ea, mr = failed[0]
        pytest.fail(f'config {name}: first failing module {m}: worst slice {sl}: ours {eo:.3e} vs autocast {ea:.3e} '
                    f'(slice gate ratio {ratio:.2f}, max gate ratio {mr:.2f})')
