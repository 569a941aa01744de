"""Writes tests/golden/ddim_threshold.pt from the reference's own `GaussianDiffusion` (samplers/ddim/gaussian_sampler.py,
imported through oracle/ref_shim.py) with x0 range restriction, run on CPU fp32 on the reference's UNetSD, and checks the
restatement tests/threshold_oracle.py against it.  The model is the tiny seeded UNetSD of smoke() (dim 64, weights from
oracle.unet_oracle.make_weights seed 1; latents of 3 frames x 8x8, [1, 77, 1024] conditionings), so the tests regenerate the
weights from the seed.

Cases (x_T given, the global generator seeded before each run so that the per-step draws can be replayed; the sampler carries
the inpaint hook that Txt2VideoSampler.get_sampler attaches, which draws once more per step):
  pct995   percentile 0.995, S 8, scale 17: s > 1 on every step;
  pct05    percentile 0.5, S 8, scale 5, eta 0.5: s > 1 on the early steps only, so both branches of max(s, 1) run;
  clamp5   clamp=5.0, S 8, scale 17: clamps to [-1, 1], the value is ignored;
  both     percentile 0.995 and clamp=1.0: percentile wins, the output equals pct995's.
Each case stores the final latent and the per-step s of the percentile cases (recorded from the reference's torch.quantile).

    python scripts/make_golden_ddim_threshold.py
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'tests'))
sys.path.insert(0, ROOT)
from oracle import ref_shim                                   # noqa: E402
from oracle import unet_oracle as UO                          # noqa: E402
from oracle import samplers_oracle as SO                      # noqa: E402
from oracle.make_golden import build_ref_unet                 # noqa: E402
import threshold_oracle as TO                                 # noqa: E402

SEEDS = {'unet': 1, 'x_T': 123, 'ctx': 2, 'noise': 7}
SHAPE = (1, 4, 3, 8, 8)
CASES = {'pct995': dict(S=8, scale=17.0, eta=0.0, percentile=0.995),
         'pct05': dict(S=8, scale=5.0, eta=0.5, percentile=0.5),
         'clamp5': dict(S=8, scale=17.0, eta=0.0, clamp=5.0),
         'both': dict(S=8, scale=17.0, eta=0.0, percentile=0.995, clamp=1.0)}


def inputs():
    x_T = torch.randn(SHAPE, generator=torch.Generator('cpu').manual_seed(SEEDS['x_T']))
    g = torch.Generator('cpu').manual_seed(SEEDS['ctx'])
    return x_T, torch.randn(1, 77, 1024, generator=g), torch.randn(1, 77, 1024, generator=g)


def main():
    m = ref_shim.load_modelscope()
    samplers_common = ref_shim.load_samplers()
    from samplers.ddim.gaussian_sampler import GaussianDiffusion
    cfg = UO.UNetConfig(dim=64)
    W = UO.make_weights(UO.param_specs(cfg), seed=SEEDS['unet'])
    torch.manual_seed(0)
    net = build_ref_unet(m, cfg)
    net.load_state_dict(W, strict=True)
    betas = SO.linear_sd_betas()
    x_T, c, uc = inputs()

    s_ref = []
    real_quantile = torch.quantile

    def recording_quantile(*a, **k):
        s = real_quantile(*a, **k)
        s_ref.append(s.clone())
        return s

    class Model:                      # what GaussianDiffusion reads off the webui model
        device = torch.device('cpu')

        def __call__(self, x, t, cc):
            return net(x, t, cc)

    out = {'seeds': SEEDS, 'shape': SHAPE, 'cases': CASES, 'unet_dim': 64}
    oracle = lambda a, b, d: UO.unet_forward(W, cfg, a, b, d)          # noqa: E731
    for name, case in CASES.items():
        s_ref.clear()
        torch.quantile = recording_quantile
        torch.manual_seed(SEEDS['noise'])
        try:
            with torch.no_grad():
                gd = GaussianDiffusion(Model(), betas)
                gd.inpaint_masking = samplers_common.inpaint_masking
                r = gd.sample(
                    x_T=x_T, S=case['S'], conditioning=c, unconditional_conditioning=uc, unconditional_guidance_scale=case['scale'],
                    eta=case['eta'], clamp=case.get('clamp'), percentile=case.get('percentile'))
        finally:
            torch.quantile = real_quantile
        kw = dict(eta=case['eta'], clamp=case.get('clamp'), percentile=case.get('percentile'))
        torch.manual_seed(SEEDS['noise'])
        same_net = TO.ddim_gaussian_sample_restricted(Model(), betas, x_T, case['S'], c, uc, case['scale'], **kw)
        assert torch.equal(same_net, r), (same_net - r).abs().max()        # the sampler restatement is exact
        s_trace = []
        torch.manual_seed(SEEDS['noise'])
        o = TO.ddim_gaussian_sample_restricted(oracle, betas, x_T, case['S'], c, uc, case['scale'], s_trace=s_trace, **kw)
        err = (r - o).abs().max().item()
        s = torch.stack(s_ref).reshape(-1) if s_ref else None
        print(f'[{name}] absmax {r.abs().max().item():.3f}; bit-identical on the reference UNet; on the oracle UNet max|d| = {err:.3e}'
              + (f'; s per step {[round(v, 3) for v in s.tolist()]}' if s is not None else ''))
        assert err <= 1e-4 * r.abs().max().item(), err             # the oracle UNet's fp32 re-association
        if s is not None:
            so = torch.stack(s_trace).reshape(-1)
            assert torch.allclose(s, so, rtol=1e-5, atol=0), (s, so)
        out['out_' + name] = r
        out['s_' + name] = s
    assert torch.equal(out['out_both'], out['out_pct995'])
    assert bool((out['s_pct995'] > 1).all()) and bool((out['s_pct05'] > 1).any()) and not bool((out['s_pct05'] > 1).all())
    path = os.path.join(ROOT, 'tests', 'golden', 'ddim_threshold.pt')
    torch.save(out, path)
    print(f'wrote {path} ({os.path.getsize(path) / 1e3:.0f} kB)')


if __name__ == '__main__':
    main()
