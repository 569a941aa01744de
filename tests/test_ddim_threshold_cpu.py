"""CPU: DDIM_Gaussian's x0 range restriction (`clamp=` / `percentile=`).  The restatement tests/threshold_oracle.py against the
reference's own GaussianDiffusion (tests/golden/ddim_threshold.pt, scripts/make_golden_ddim_threshold.py), its quantile against
torch.quantile bit for bit, the reference's quirks, and the host side of GaussianDiffusion.sample with the device step replaced
by the restatement."""
import ctypes as C
import os

import pytest
import torch

import threshold_oracle as TO
from oracle import unet_oracle as UO, samplers_oracle as SO
from t2v_b200 import samplers as S, _lib, distributed as D

GOLD = torch.load(os.path.join(os.path.dirname(__file__), 'golden', 'ddim_threshold.pt'))

# The fixture script finds the sampler restatement bit-identical to the reference on the reference's own UNetSD; what is left
# here is the oracle UNet's fp32 re-association, amplified by the steps (measured 9.1e-6, 1.3e-5, 8.4e-5 (clamping at scale 17
# moves elements across +-1) and 9.1e-6 of |ref|max).
GATES = {'pct995': 2e-5, 'pct05': 3e-5, 'clamp5': 2e-4, 'both': 2e-5}


def gold_inputs():
    x_T = torch.randn(GOLD['shape'], generator=torch.Generator('cpu').manual_seed(GOLD['seeds']['x_T']))
    g = torch.Generator('cpu').manual_seed(GOLD['seeds']['ctx'])
    return x_T, torch.randn(1, 77, 1024, generator=g), torch.randn(1, 77, 1024, generator=g)


@pytest.fixture(scope='module')
def tiny():
    cfg = UO.UNetConfig(dim=GOLD['unet_dim'])
    return cfg, UO.make_weights(UO.param_specs(cfg), seed=GOLD['seeds']['unet'])


@pytest.mark.parametrize('name', ['pct995', 'pct05', 'clamp5', 'both'])
def test_restatement_matches_reference_fixture(tiny, name):
    cfg, W = tiny
    case = GOLD['cases'][name]
    x_T, c, uc = gold_inputs()
    s_trace = []
    torch.manual_seed(GOLD['seeds']['noise'])
    out = TO.ddim_gaussian_sample_restricted(lambda a, b, d: UO.unet_forward(W, cfg, a, b, d), SO.linear_sd_betas(), x_T,
                                             case['S'], c, uc, case['scale'], eta=case['eta'], clamp=case.get('clamp'),
                                             percentile=case.get('percentile'), s_trace=s_trace)
    ref = GOLD['out_' + name]
    assert float((out - ref).abs().max()) <= GATES[name] * float(ref.abs().max())
    if GOLD['s_' + name] is None:
        assert s_trace == []
    else:
        assert torch.allclose(torch.stack(s_trace).reshape(-1), GOLD['s_' + name], rtol=1e-5, atol=0)


def test_fixture_covers_both_sides_of_the_threshold():
    assert bool((GOLD['s_pct995'] > 1).all())
    s = GOLD['s_pct05']
    assert bool((s > 1).any()) and bool((s <= 1).any())
    assert torch.equal(GOLD['out_both'], GOLD['out_pct995'])          # percentile wins over clamp


def _rows(kind, g):
    if kind == 'random':
        return torch.randn(3, 1000, generator=g) * 3
    if kind == 'ties':
        return torch.randint(-4, 5, (3, 777), generator=g).float() / 2
    if kind == 'all_equal':
        return torch.full((2, 513), -1.25)
    if kind == 'n1':
        return torch.randn(4, 1, generator=g)
    if kind == 'zeros':
        return torch.zeros(2, 100) * torch.tensor([[1.0], [-1.0]])          # +0 and -0
    if kind == 'nan':
        v = torch.randn(3, 257, generator=g)
        v[1, 100] = float('nan')
        return v
    raise ValueError(kind)


@pytest.mark.parametrize('kind', ['random', 'ties', 'all_equal', 'n1', 'zeros', 'nan'])
@pytest.mark.parametrize('q', [0.0, 0.3, 0.5, 0.995, 0.99951, 1.0])
def test_quantile_restatement_is_torch_quantile(kind, q):
    v = _rows(kind, torch.Generator().manual_seed(int(q * 1e5) + len(kind))).abs()
    ours = torch.cat([TO.quantile(v[i:i + 1], q) for i in range(v.shape[0])])
    ref = torch.quantile(v, q, dim=1)
    assert torch.equal(torch.isnan(ours), torch.isnan(ref))
    assert torch.equal(torch.nan_to_num(ours), torch.nan_to_num(ref))


def test_quantile_restatement_at_the_size_limit():
    v = torch.rand(1, 1 << 24, generator=torch.Generator().manual_seed(3))
    for q in (0.995, 0.5):
        assert torch.equal(TO.quantile(v, q), torch.quantile(v, q, dim=1))
    with pytest.raises(RuntimeError, match='quantile\\(\\) input tensor is too large'):
        TO.quantile(torch.zeros(1, (1 << 24) + 1), 0.5)


def test_reference_quirks():
    x0 = torch.tensor([[-7.0, -1.5, -0.25, 0.0, 0.5, 3.0]]).view(1, 1, 1, 2, 3)
    assert TO.restrict_x0(x0, clamp=5.0).reshape(-1).tolist() == [-1.0, -1.0, -0.25, 0.0, 0.5, 1.0]   # clamp's value is ignored
    assert torch.equal(TO.restrict_x0(x0, clamp=5.0, percentile=1.0), x0 / 7.0)                        # percentile wins
    assert torch.equal(TO.restrict_x0(x0 / 10, percentile=1.0), x0 / 10)                                # s below 1 is raised to 1
    for bad in (0, 1.5):
        with pytest.raises(AssertionError):
            TO.restrict_x0(x0, percentile=bad)


class _Model(object):
    device = torch.device('cpu')


def test_sampler_argument_checks():
    smp = S.GaussianDiffusion(_Model(), SO.linear_sd_betas())
    x = torch.zeros(1, 4, 2, 8, 8)
    for bad in (0, 1.5, -0.5):
        with pytest.raises(AssertionError):
            smp.sample(x_T=x, S=2, percentile=bad)
    with pytest.raises(NotImplementedError, match='condition_fn'):
        smp.sample(x_T=x, S=2, condition_fn=lambda *a, **k: 0)


def test_frame_sharded_clip_refuses_percentile(monkeypatch):
    monkeypatch.setattr(D, '_frame_shard', object())
    smp = S.GaussianDiffusion(_Model(), SO.linear_sd_betas())
    with pytest.raises(NotImplementedError, match='frame-sharded'):
        smp.sample(x_T=torch.zeros(1, 4, 2, 8, 8), S=2, percentile=0.995)


class _TorchThreshold(object):
    """t2v_ddim_step_threshold restated with threshold_oracle.threshold_step on registered tensors."""

    def __init__(self, reg):
        self.reg, self.calls = reg, []

    def t2v_abs_quantile_workspace(self, B):
        return 16448 * B

    def t2v_ddim_step_threshold(self, x, ec, eu, is32, xo, n, chan_stride, Cc, gch, g, a0, a1, a2, a3, a4, noise, fp16, B, pct,
                                s_out, ws, ws_bytes, stream):
        R = self.reg
        X = R[x.value]
        assert X.numel() == n and X.shape[0] == B and chan_stride * Cc * B == n and (pct == 0 or ws_bytes >= 16448 * B)
        self.calls.append(pct)
        kw = {'percentile': pct} if pct > 0 else {'clamp': True}
        R[xo.value].copy_(TO.threshold_step(X, R[ec.value], R[eu.value] if eu.value else None, g, gch, (a0, a1, a2, a3, a4),
                                            R[noise.value] if noise.value else None, fp16, **kw))
        return 0


@pytest.mark.parametrize('kw', [dict(percentile=0.995), dict(percentile=0.5, clamp=3.0), dict(clamp=5.0)])
def test_sampler_host_side_matches_restatement(tiny, monkeypatch, kw):
    """GaussianDiffusion.sample(clamp=, percentile=) with the device step restated: the same latent as the restated reference
    loop driven by the same fp16 denoiser, bit for bit: the host's coefficients are the reference's fp32 values."""
    cfg, W = tiny
    reg = {}

    def ptr(t):
        if t is None:
            return C.c_void_p(0)
        reg[t.data_ptr()] = t
        return C.c_void_p(t.data_ptr())
    fake = _TorchThreshold(reg)
    monkeypatch.setattr(_lib, 'lib', lambda: fake)
    monkeypatch.setattr(_lib, 'ptr', ptr)
    monkeypatch.setattr(_lib, 'stream_ptr', lambda: None)
    monkeypatch.setattr(S, '_need_cuda', lambda x: None)
    x_T, c, uc = gold_inputs()
    model = lambda a, b, d: UO.unet_forward(W, cfg, a, b, d).half()       # noqa: E731   fp16 eps, as the GPU denoiser returns

    class M(_Model):
        def __call__(self, a, b, d):
            return model(a, b, d)
    betas = SO.linear_sd_betas()
    torch.manual_seed(0)
    ours = S.GaussianDiffusion(M(), betas).sample(x_T=x_T, S=4, conditioning=c, unconditional_conditioning=uc,
                                                  unconditional_guidance_scale=9.0, **kw)
    assert fake.calls == [kw['percentile'] if 'percentile' in kw else 0.0] * 4
    torch.manual_seed(0)
    ref = TO.ddim_gaussian_sample_restricted(model, betas, x_T, 4, c, uc, 9.0, **kw)
    assert torch.equal(ours, ref)
