"""CPU: the premise of test_unet_modules_gpu.py.  unet_modules.py restates how the plan builder wires the UNet's modules
(skip pairing, adapter feature points, per-frame context and embedding, layouts); here each oracle runs end to end in fp64
with taps, and every module re-run on its own from the oracle's own taps through that restatement must give its tap bit for
bit.  The module list must also be the library's: its reference names, as the oracles and the library's parameter table
both enumerate them."""
import ctypes as C

import pytest
import torch

import adapter_oracle as AO
import unet_modules as UM
from oracle import unet_oracle as UO, vc_oracle as VC


def _f64(W):
    return {k: v.half().double() for k, v in W.items()}


def _modelscope():
    cfg = UO.UNetConfig(dim=64)
    W = _f64(UO.make_weights(UO.param_specs(cfg), seed=1))
    x, t, y = UM.structured_inputs(cfg, 2, 3, 8, 8, 77)
    taps = {}
    eps = UO.unet_forward(W, cfg, x.double(), t, y.double(), taps=taps)
    return cfg, W, x, t, y.double(), None, taps, eps


def _videocrafter():
    cfg = VC.VCConfig(model_channels=64, context_dim=48, temporal_length=4)
    W = _f64(UO.make_weights(VC.vc_param_specs(cfg), seed=5))
    x, t, y = UM.structured_inputs(cfg, 2, 4, 8, 8, 9)
    g = torch.Generator().manual_seed(7)
    feats = [torch.randn(s, generator=g).half().double() for s in UM.feature_shapes(cfg, 1, 4, 8, 8)]
    taps = {}
    eps = AO.vc_unet_forward(W, cfg, x.double(), t, y.double(), feats, taps=taps)
    # vc_oracle taps are [b, c, t, h, w]; the library's (and the helper's) layout is [(b t), c, h, w]
    taps = {k: v.permute(0, 2, 1, 3, 4).reshape(-1, *v.shape[1:2], *v.shape[3:]) for k, v in taps.items()}
    return cfg, W, x, t, y.double(), feats, taps, eps


@pytest.fixture(scope='module', params=['modelscope', 'videocrafter'])
def run(request):
    return (_modelscope if request.param == 'modelscope' else _videocrafter)()


def test_every_module_rerun_from_the_oracles_own_taps_is_bit_identical(run):
    cfg, W, x, t, y, feats, taps, eps = run
    B, Fr = x.shape[0], x.shape[2]
    taps = dict(taps, out=eps.permute(0, 2, 1, 3, 4).reshape(B * Fr, *eps.shape[1:2], *eps.shape[3:]))
    emb = UM.time_embedding(cfg, W, t)
    seen = []
    for b, xin in UM.module_inputs(cfg, taps, x, feats):
        assert xin.dtype == torch.float64
        out = UM.run_module(cfg, W, b, xin, emb, y, B)
        assert torch.equal(out, taps[b.prefix]), b.prefix
        seen.append(b.prefix)
    assert seen == UM.tap_names(cfg)
    assert sorted(seen) == sorted(taps)


def _library_modules(net):
    """Module names of the library's UNet, read from its parameter table: one characteristic parameter per module kind."""
    from t2v_b200 import _lib
    info = _lib.load_library().t2v_unet_param_info
    name, shape, ndim = C.create_string_buffer(256), (C.c_int64 * 8)(), C.c_int(0)
    names = []
    for i in range(info(net._handle, 0, name, 256, shape, C.byref(ndim))):
        info(net._handle, i, name, 256, shape, C.byref(ndim))
        names.append(name.value.decode())
    mods = {n[:-len(s)] for n in names for s in ('.in_layers.0.weight', '.norm.weight', '.op.weight', '.conv.weight')
            if n.endswith(s)}
    mods |= {m for n, m in (('input_blocks.0.0.weight', 'input_blocks.0.0'), ('out.2.weight', 'out')) if n in names}
    return mods


@pytest.mark.parametrize('arch', ['modelscope', 'modelscope_full', 'videocrafter', 'videocrafter_full'])
def test_module_list_is_the_librarys(arch):
    from t2v_b200.modules import UNetSD, UNetModel
    if arch.startswith('modelscope'):
        cfg = UO.UNetConfig() if arch.endswith('full') else UO.UNetConfig(dim=64)
        net = UNetSD(dim=cfg.dim)
    else:
        cfg = VC.VCConfig() if arch.endswith('full') else VC.VCConfig(model_channels=64, context_dim=48, temporal_length=4)
        net = UNetModel(model_channels=cfg.model_channels, context_dim=cfg.context_dim, temporal_length=cfg.temporal_length)
    names = UM.tap_names(cfg)
    assert len(names) == len(set(names))
    assert set(names) == _library_modules(net)
