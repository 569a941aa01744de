"""Writes tests/golden/adapter.pt from VideoCrafter's own classes (imported through oracle/ref_shim.py), run on CPU fp32, and
checks the restatement tests/adapter_oracle.py against them:

  1. `Adapter` (videocrafter/lvdm/models/modules/adapter.py) features at two narrow configs on seeded 64x64 depth frames
     (levels 8, 4, 2, 1), through `T2VAdapterDepth.get_adapter_features` (ddpm3d.py:1470-1484):
       A: channels [64, 128, 256, 256], nums_rb 2, ksize 1, sk, average pooling      (the depth config's structure)
       B: the same widths, nums_rb 3, ksize 3, sk, stride-2 conv downsampling
  2. the state-dict key / shape tables of the full-width depth config and of Adapter(sk=True);
  3. `UNetModel` (openaimodel3d.py) eps with and without `features_adapter` at the tiny config of tests/test_videocrafter_gpu.py
     (model_channels 64, context_dim 48, temporal_length 4; 4 frames of 8x8), the features being config A's;
  4. `DDIMSampler` (lvdm/samplers/ddim.py) trajectories with those features: S = 4, CFG scale 5, eta 0 and 0.5, given x_T,
     the sampler's noise_gen seeded;
  5. `T2VAdapterDepth.get_batch_depth` on the fixed stub depth model tests/adapter_oracle.py defines.

Weights are regenerated from seeds (oracle.unet_oracle.make_weights); the fixture holds inputs and outputs only.

    python scripts/make_golden_adapter.py
"""
import os
import sys
import types
from types import SimpleNamespace

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'tests'))
sys.path.insert(0, ROOT)
from oracle import ref_shim                                   # noqa: E402
from oracle import unet_oracle as UO                          # noqa: E402
from oracle import vc_oracle as VC                            # noqa: E402
from oracle import samplers_oracle as SO                      # noqa: E402
from oracle.make_golden import build_ref_vc_unet, _SchedModel  # noqa: E402
import adapter_oracle as AO                                   # noqa: E402

SEEDS = {'A': 21, 'B': 22, 'unet': 4, 'depth_in': 31, 'x': 123, 'ctx': 2, 'x_T': 5, 'noise': 11, 'video': 41}
UNET_CFG = dict(model_channels=64, context_dim=48, temporal_length=4)
B, T, HL, WL, L = 1, 4, 8, 8, 9


def _install():
    ref_shim.install()
    if 'pytorch_lightning' not in sys.modules:          # ddpm3d imports it; LightningModule is only a base class here
        pl = types.ModuleType('pytorch_lightning')
        pl.LightningModule = torch.nn.Module
        ut = types.ModuleType('pytorch_lightning.utilities')
        ut.rank_zero_only = lambda f: f
        pl.utilities = ut
        sys.modules['pytorch_lightning'], sys.modules['pytorch_lightning.utilities'] = pl, ut


def ref_adapter(cfg, seed):
    from videocrafter.lvdm.models.modules.adapter import Adapter
    a = Adapter(**cfg).eval()
    specs = AO.adapter_param_specs(**cfg)
    sd = a.state_dict()
    assert set(sd) == set(specs) and all(tuple(sd[k].shape) == specs[k] for k in sd)
    W = UO.make_weights(specs, seed=seed)
    a.load_state_dict(W, strict=True)
    return a, W


def table(cfg):
    from videocrafter.lvdm.models.modules.adapter import Adapter
    with torch.device('meta'):
        a = Adapter(**cfg)
    return {k: tuple(v.shape) for k, v in a.state_dict().items()}


def main():
    _install()
    from videocrafter.lvdm.models.ddpm3d import T2VAdapterDepth
    from videocrafter.lvdm.samplers.ddim import DDIMSampler
    DDIMSampler.register_buffer = lambda self, name, attr: setattr(self, name, attr)    # ddim.py:22-26 hard-codes "cuda"
    out = {'seeds': SEEDS, 'configs': {'A': AO.NARROW_A, 'B': AO.NARROW_B}, 'unet_cfg': UNET_CFG, 'shape': (B, 4, T, HL, WL), 'L': L}
    depth = torch.rand((B, 1, T, 64, 64), generator=torch.Generator().manual_seed(SEEDS['depth_in'])) * 2 - 1     # b c t h w
    out['depth'] = depth
    feats_A = None
    for name in ('A', 'B'):
        cfg = out['configs'][name]
        a, W = ref_adapter(cfg, SEEDS[name])
        with torch.no_grad():
            ref = T2VAdapterDepth.get_adapter_features(SimpleNamespace(adapter=a), depth)          # 4 x [b, c, t, h, w]
        o = AO.to_video_features(AO.adapter_forward(W, depth.permute(0, 2, 1, 3, 4).reshape(B * T, 1, 64, 64), **cfg), B, T)
        err = max((x - y).abs().max().item() for x, y in zip(o, ref))
        print(f'[adapter {name}] shapes {[tuple(f.shape) for f in ref]}; oracle-vs-reference max|d| = {err:.3e}')
        assert err < 1e-5
        out['features_' + name] = [f.clone() for f in ref]
        if name == 'A':
            feats_A = ref
    out['table_depth'] = table(AO.DEPTH)
    out['table_sk'] = table(dict(sk=True))
    print(f"[tables] depth: {len(out['table_depth'])} tensors, Adapter(sk=True): {len(out['table_sk'])} tensors")

    vcfg = VC.VCConfig(**UNET_CFG)
    net = build_ref_vc_unet(vcfg)
    Wu = UO.make_weights(VC.vc_param_specs(vcfg), seed=SEEDS['unet'])
    net.load_state_dict(Wu, strict=True)
    x = torch.randn((B, 4, T, HL, WL), generator=torch.Generator().manual_seed(SEEDS['x']))
    ctx = torch.randn((B, L, 48), generator=torch.Generator().manual_seed(SEEDS['ctx']))
    t = torch.tensor([981])
    with torch.no_grad():
        e0 = net(x, t, context=ctx)
        e1 = net(x, t, context=ctx, features_adapter=feats_A)
    o0 = AO.vc_unet_forward(Wu, vcfg, x, t, ctx)
    o1 = AO.vc_unet_forward(Wu, vcfg, x, t, ctx, feats_A)
    err = max((o0 - e0).abs().max().item(), (o1 - e1).abs().max().item())
    print(f'[unet] eps absmax {e0.abs().max().item():.3f} / with features {e1.abs().max().item():.3f}, moved by '
          f'{(e1 - e0).abs().max().item():.3f}; oracle-vs-reference max|d| = {err:.3e}')
    assert err < 1e-5 * max(1.0, e1.abs().max().item())
    out.update(eps=e0, eps_features=e1, t=t)

    betas = SO.linear_sd_betas()

    class _LDM(_SchedModel):
        def apply_model(self, xx, tt, c, **kw):
            return net(xx, tt, context=c, **kw)
    c = torch.randn((B, L, 48), generator=torch.Generator().manual_seed(SEEDS['ctx'] + 100))
    uc = torch.randn((B, L, 48), generator=torch.Generator().manual_seed(SEEDS['ctx'] + 101))
    x_T = torch.randn((B, 4, T, HL, WL), generator=torch.Generator().manual_seed(SEEDS['x_T']))
    out.update(c=c, uc=uc, x_T=x_T)
    for eta in (0.0, 0.5):
        smp = DDIMSampler(_LDM(betas))
        smp.noise_gen.manual_seed(SEEDS['noise'])
        with torch.no_grad():
            r, _ = smp.sample(S=4, batch_size=B, shape=(4, T, HL, WL), conditioning=c, x_T=x_T, verbose=False,
                              unconditional_guidance_scale=5.0, unconditional_conditioning=uc, eta=eta, temporal_length=T,
                              conditional_guidance_scale_temporal=None, features_adapter=feats_A)
        o = AO.vc_ddim_sample(Wu, vcfg, betas, x_T, 4, c, uc, 5.0, eta, torch.Generator('cpu').manual_seed(SEEDS['noise']), feats_A)
        print(f'[ddim] eta={eta}: oracle-vs-reference max|d| = {(r - o).abs().max().item():.3e} (absmax {r.abs().max().item():.3f})')
        assert (r - o).abs().max().item() < 1e-5 * max(1.0, r.abs().max().item())
        out[f'ddim_eta{eta}'] = r

    video = torch.rand((1, 3, 2, 40, 48), generator=torch.Generator().manual_seed(SEEDS['video'])) * 2 - 1
    stub = AO.StubDepth()
    ns = SimpleNamespace(depth_stage_model=stub)
    ns.prepare_midas_input = lambda v: T2VAdapterDepth.prepare_midas_input(ns, v)
    d = T2VAdapterDepth.get_batch_depth(ns, video, (40, 48))
    o = AO.get_batch_depth(stub, video, (40, 48))
    print(f'[get_batch_depth] {tuple(d.shape)}; oracle-vs-reference max|d| = {(d - o).abs().max().item():.3e}')
    assert torch.equal(d, o)
    out.update(video=video, batch_depth=d)
    path = os.path.join(ROOT, 'tests', 'golden', 'adapter.pt')
    torch.save(out, path)
    print(f'wrote {path} ({os.path.getsize(path) / 1e6:.2f} MB)')


if __name__ == '__main__':
    main()
