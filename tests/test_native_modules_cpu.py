"""CPU: every nn.Module mirror backed by a library handle ships exactly the library's parameter table, and is flagged to reship
after a state dict is loaded or its tensors are converted through any parent module, not only through the mirror itself."""
import ctypes as C

import pytest
import torch
import torch.nn as nn

import adapter_oracle as AO
import clip_l_oracle as CL


def _library_table(m):
    """Names of t2v_{kind}_param_info of the mirror's handle, read straight from the library."""
    from t2v_b200 import _lib
    info = getattr(_lib.load_library(), f't2v_{m._kind}_param_info')
    name, shape, ndim = C.create_string_buffer(256), (C.c_int64 * 8)(), C.c_int(0)
    out = []
    for i in range(info(m._handle, 0, name, 256, shape, C.byref(ndim))):
        info(m._handle, i, name, 256, shape, C.byref(ndim))
        out.append(name.value.decode())
    return out


def _ldm_with_text_encoder():
    from t2v_b200.videocrafter import LatentDiffusion
    return LatentDiffusion(**CL.TINY_LDM, cond_stage_config=dict(
        target='lvdm.models.modules.condition_modules.FrozenCLIPEmbedder',
        params=dict(width=CL.NARROW.width, heads=CL.NARROW.heads, layers=CL.NARROW.layers, vocab=CL.NARROW.vocab)))


def _t2v_adapter_depth():
    from t2v_b200.videocrafter import T2VAdapterDepth
    return T2VAdapterDepth(None, dict(params=AO.NARROW_A), **CL.TINY_LDM, depth_stage_model=AO.StubDepth())


def _modelscope_pair():
    from t2v_b200.modules import UNetSD, AutoencoderKL
    from t2v_b200.pipeline import VAE_DDCONFIG
    parent = nn.Module()
    parent.unet, parent.vae = UNetSD(dim=64), AutoencoderKL(VAE_DDCONFIG, 4)
    return parent


def _native_children(parent):
    from t2v_b200.modules import _NativeModule
    return [m for m in parent.modules() if isinstance(m, _NativeModule)]


@pytest.mark.parametrize('make,mirrors', [(_ldm_with_text_encoder, ['UNetModel', 'AutoencoderKL', '_CLIPTextModel']),
                                          (_t2v_adapter_depth, ['UNetModel', 'AutoencoderKL', 'Adapter']),
                                          (_modelscope_pair, ['UNetSD', 'AutoencoderKL'])], ids=['ldm_clip', 'adapter_depth', 'unet_vae'])
def test_parent_load_and_conversion_mark_every_mirror_dirty(make, mirrors):
    parent = make()
    children = _native_children(parent)
    assert sorted(type(m).__name__ for m in children) == sorted(mirrors)
    for convert in (lambda: parent.load_state_dict(parent.state_dict(), strict=True), parent.half):
        for m in children:
            m._dirty = False                                # the state after a forward / decode / encode
        convert()
        assert [type(m).__name__ for m in children if not m._dirty] == []


def test_native_names_are_the_library_tables():
    from t2v_b200.modules import UNetSD, UNetModel, AutoencoderKL
    from t2v_b200.pipeline import VAE_DDCONFIG
    from t2v_b200.clip import FrozenOpenCLIPEmbedder, FrozenCLIPEmbedder
    from t2v_b200.adapter import Adapter
    with torch.device('meta'):
        mirrors = [UNetSD(dim=64), UNetModel(model_channels=64, context_dim=48, temporal_length=4), AutoencoderKL(VAE_DDCONFIG, 4),
                   FrozenCLIPEmbedder(width=128, heads=2, layers=3, vocab=300).transformer, Adapter(**AO.NARROW_A)]
        vit_h = FrozenOpenCLIPEmbedder(width=128, heads=2, layers=4, vocab=300, tokenizer=object()).model
    for m in mirrors:
        table = _library_table(m)
        assert m._native_names == set(table) == set(m.state_dict()), m._kind
    vae = mirrors[2]
    assert len(vae._native_names) == 248 and {'encoder.conv_in.weight', 'quant_conv.weight'} <= vae._native_names
    # the ViT-H tower holds open_clip's full text tree; the unused last block and the projection stay on the host
    assert vit_h._native_names == set(_library_table(vit_h))
    unshipped = set(dict(vit_h.named_parameters())) - vit_h._native_names
    assert unshipped == {k for k in vit_h.state_dict() if k.startswith('transformer.resblocks.3.')} | {'text_projection', 'logit_scale'}
