"""CPU: the host side of VideoCrafter LoRA (t2v_b200/videocrafter.py net_load_lora / net_load_lora_v2, lora.py:620-755) against
tests/golden/vc_lora.pt, which the reference's own loader wrote (scripts/make_golden_vc_lora.py): which keys reach which
library handle, under which name, with which factors and signed alpha, which keys are skipped, and that the mirror's
nn.Linear / nn.Conv2d modules sit at exactly the reference's paths (so the same keys merge and the same keys are skipped)."""
import os

import pytest
import torch
import torch.nn as nn

import clip_l_oracle as CL

TARGET = 'lvdm.models.modules.condition_modules.FrozenCLIPEmbedder'


def _gold(gold_dir):
    return torch.load(os.path.join(gold_dir, 'vc_lora.pt'))


def _meta_ldm():
    from t2v_b200.videocrafter import LatentDiffusion
    with torch.device('meta'):
        return LatentDiffusion(**CL.TINY_LDM, cond_stage_config=dict(target=TARGET, params=dict(
            width=CL.NARROW.width, heads=CL.NARROW.heads, layers=CL.NARROW.layers, vocab=CL.NARROW.vocab, max_length=77)))


def _record(m):
    """Replaces lora_apply / lora_restore of every library-backed module of `m` by recorders."""
    from t2v_b200.modules import _NativeModule
    calls = []
    for path, mod in m.named_modules():
        if isinstance(mod, _NativeModule):
            mod.lora_apply = lambda name, up, down, alpha, path=path: calls.append(
                ('apply', path, name, tuple(up.shape), tuple(down.shape), up.dtype, alpha))
            mod.lora_restore = lambda name, path=path: calls.append(('restore', path, name))
    return calls


def _missing(capsys):
    return [l.split('missing param at:', 1)[1].strip() for l in capsys.readouterr().out.splitlines() if 'missing param at:' in l]


def _owner(key):
    for prefix, handle in (('model.diffusion_model.', 'model.diffusion_model'), ('cond_stage_model.transformer.', 'cond_stage_model.transformer'),
                           ('first_stage_model.', 'first_stage_model')):
        if key.startswith(prefix):
            return handle, key[len(prefix):]
    raise AssertionError(key)


def test_mirror_linear_and_conv2d_paths_match_the_reference(gold_dir):
    m = _meta_ldm()
    mine = {(p, type(x).__name__) for p, x in m.named_modules() if type(x) in (nn.Linear, nn.Conv2d)}
    assert mine == {tuple(t) for t in _gold(gold_dir)['tree']}


def test_net_load_lora_walk(gold_dir, capsys):
    from t2v_b200 import videocrafter as vcm
    g = _gold(gold_dir)
    m = _meta_ldm()
    calls = _record(m)
    capsys.readouterr()
    vcm.net_load_lora(m, g['lora1'], alpha=g['alpha1'])
    assert _missing(capsys) == g['skipped']
    want = []
    for wk in g['merged']:                               # every weight the reference merged, in the file's order
        p = wk[:-len('.weight')]
        up, down = g['lora1'][p + '.lora_up.weight'], g['lora1'][p + '.lora_down.weight']
        handle, name = _owner(wk)
        want.append(('apply', handle, name, (up.shape[0], up.shape[1]), (down.shape[0], down.shape[1]), up.dtype, g['alpha1']))
    assert sorted(calls, key=str) == sorted(want, key=str) and len(calls) == len(g['merged'])
    assert any(c[5] == torch.float16 for c in calls) and any(c[5] == torch.float32 for c in calls)    # dtypes as stored
    vae = [c for c in calls if c[1] == 'first_stage_model']
    assert vae == [('apply', 'first_stage_model', 'decoder.up.0.block.0.nin_shortcut.weight', (128, 4), (4, 256), torch.float32,
                    g['alpha1'])]                        # 4-D factors squeezed
    calls.clear()
    vcm.net_load_lora(m, g['lora1'], alpha=g['alpha1'], remove=True)
    assert sorted(calls, key=str) == sorted([w[:6] + (-g['alpha1'],) for w in want], key=str)
    calls.clear()
    vcm.change_lora(m, inject_lora=True, lora_scale=g['alpha2'], lora_path=g['lora2'], last_time_lora=g['lora1'],
                    last_time_lora_scale=g['alpha1'])
    assert [c[6] for c in calls] == [-g['alpha1']] * len(want) + [g['alpha2']] * len(want)


def test_reference_change_lora_residue_is_below_an_fp16_ulp(gold_dir):
    """The reference's change_lora subtracts in fp32: its switched weights equal base + alpha2 * up2 @ down2 to ~1e-8, which
    is why the GPU tests build them that way, and why the library's fp16 subtraction (up to one fp16 ulp) is the deviation."""
    g = _gold(gold_dir)
    assert set(g['changed_residue']) == set(g['merged'])
    assert 0.0 < max(g['changed_residue'].values()) < 1e-6
    assert all(v.dtype == torch.float16 for v in g['merged'].values())


def test_net_load_lora_from_a_path(gold_dir, tmp_path):
    from t2v_b200 import videocrafter as vcm
    g = _gold(gold_dir)
    path = os.path.join(str(tmp_path), 'lora.ckpt')
    torch.save(g['lora1'], path)
    m = _meta_ldm()
    calls = _record(m)
    vcm.net_load_lora(m, path, alpha=0.5)
    assert len(calls) == len(g['merged']) and all(c[6] == 0.5 for c in calls)


def test_net_load_lora_v2_origin_weight_and_restore(gold_dir):
    from t2v_b200 import videocrafter as vcm
    g = _gold(gold_dir)
    m = _meta_ldm()
    calls = _record(m)
    origin = vcm.net_load_lora_v2(m, g['lora1'], alpha=g['alpha1'])
    assert sorted(origin) == g['origin_keys']
    applied = sorted((c[1], c[2]) for c in calls)
    assert sorted((_owner(k)) for k in g['merged']) == sorted((h, n) for h, n in applied)
    calls.clear()
    origin2 = vcm.change_lora_v2(m, inject_lora=True, lora_scale=g['alpha2'], lora_path=g['lora2'], last_time_lora=g['lora1'],
                                 last_time_lora_scale=g['alpha1'], origin_weight=origin)
    assert origin2 is origin and sorted(origin2) == g['origin_keys']
    n = len(g['merged'])
    assert [c[0] for c in calls] == ['restore'] * n + ['apply'] * n
    assert sorted((c[1], c[2]) for c in calls[:n]) == applied and all(c[6] == g['alpha2'] for c in calls[n:])


def test_unknown_path_raises_attribute_error():
    from t2v_b200 import videocrafter as vcm
    m = _meta_ldm()
    calls = _record(m)
    bad = {'model.diffusion_model.input_blocks.1.1.transformer_blocks.0.attn9.to_q.lora_up.weight': torch.zeros(64, 4),
           'model.diffusion_model.input_blocks.1.1.transformer_blocks.0.attn9.to_q.lora_down.weight': torch.zeros(4, 64)}
    with pytest.raises(AttributeError):
        vcm.net_load_lora(m, bad)
    with pytest.raises(AttributeError):
        vcm.net_load_lora_v2(m, bad)
    assert calls == []


def test_lora_apply_checks_shapes_before_touching_the_library():
    m = _meta_ldm()
    unet = m.model.diffusion_model
    name = 'input_blocks.1.1.transformer_blocks.0.attn1.to_q.weight'
    with pytest.raises(ValueError):
        unet.lora_apply(name, torch.zeros(64, 4, 1, 1), torch.zeros(4, 64, 1, 1), 1.0)      # unsqueezed factors
    with pytest.raises(ValueError):
        unet.lora_apply(name, torch.zeros(64, 4), torch.zeros(4, 32), 1.0)
    with pytest.raises(KeyError):
        unet.lora_apply('input_blocks.1.1.no.weight', torch.zeros(64, 4), torch.zeros(4, 64), 1.0)
