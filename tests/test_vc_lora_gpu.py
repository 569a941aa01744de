"""GPU: VideoCrafter LoRA (net_load_lora / change_lora / net_load_lora_v2 / change_lora_v2, lora.py:620-755) merged on the device
into the library's UNet, CLIP ViT-L text tower and VAE, against the weights the reference's own loader produced
(tests/golden/vc_lora.pt, scripts/make_golden_vc_lora.py) run through the fp32 oracles."""
import os

import numpy as np
import pytest
import torch

from oracle import unet_oracle as UO, vae_oracle as VO, vc_oracle as VC
import clip_l_oracle as CL
from parity_util import errs, report

pytestmark = pytest.mark.gpu
TARGET = 'lvdm.models.modules.condition_modules.FrozenCLIPEmbedder'
UCFG = VC.VCConfig(**CL.TINY_LDM['unet_config'])
PREFIX = {'unet': 'model.diffusion_model.', 'clip': 'cond_stage_model.transformer.', 'vae': 'first_stage_model.'}


@pytest.fixture(scope='module')
def gold(gold_dir):
    return torch.load(os.path.join(gold_dir, 'vc_lora.pt'))


def _cfg_kw():
    c = CL.NARROW
    return dict(width=c.width, heads=c.heads, layers=c.layers, vocab=c.vocab, max_length=c.context)


def _base_weights(s):
    """The fixture's seeded base weights per handle (fp32), as scripts/make_golden_vc_lora.py made them."""
    vc = VO.VAEConfig()
    return {'unet': UO.make_weights(VC.vc_param_specs(UCFG), seed=s['unet']),
            'clip': UO.make_weights(CL.clip_l_param_specs(CL.NARROW), seed=s['clip']),
            'vae': {**UO.make_weights(VO.decoder_param_specs(vc), seed=s['vae_dec']),
                    **UO.make_weights(VO.encoder_param_specs(vc), seed=s['vae_enc'])}}


def _build(W):
    from t2v_b200.videocrafter import LatentDiffusion
    m = LatentDiffusion(**CL.TINY_LDM, cond_stage_config=dict(target=TARGET, params=_cfg_kw()))
    m.cond_stage_model.tokenizer = CL.WordTokenizer(CL.NARROW.vocab)
    m.model.diffusion_model.load_state_dict(W['unet'], strict=True)
    m.cond_stage_model.transformer.load_state_dict(W['clip'], strict=True)
    m.first_stage_model.load_state_dict(W['vae'], strict=True)
    return m.half().cuda().eval()


def _with(W, merged):
    """W with merged weights substituted (keyed from the LatentDiffusion root), everything rounded to fp16 (what the library
    stores; the fixture's merged weights are the reference's fp32 result already rounded so)."""
    out = {}
    for kind, w in W.items():
        d = dict(w)
        for k, v in merged.items():
            if k.startswith(PREFIX[kind]):
                d[k[len(PREFIX[kind]):]] = v
        out[kind] = {k: v.half().float() for k, v in d.items()}
    return out


def _switched(W, g):
    """The reference's weights after change_lora from lora1 (alpha1) to lora2 (alpha2), keyed from the LatentDiffusion root:
    base + alpha2 * up2 @ down2 in fp32, which the reference's own result matches to g['changed_residue'] (~1e-8)."""
    out = {}
    for key in g['merged']:
        kind = next(k for k, p in PREFIX.items() if key.startswith(p))
        w = W[kind][key[len(PREFIX[kind]):]]
        p = key[:-len('.weight')]
        up, down = g['lora2'][p + '.lora_up.weight'].float(), g['lora2'][p + '.lora_down.weight'].float()
        d = up.reshape(up.shape[0], -1) @ down.reshape(down.shape[0], -1)
        out[key] = w + g['alpha2'] * d.reshape(w.shape)
    return out


@pytest.fixture(scope='module')
def base(gold):
    return _base_weights(gold['seeds'])


def _inputs():
    g = torch.Generator('cpu').manual_seed(3)
    x = torch.randn((1, 4, 4, 8, 8), generator=g)
    ctx = torch.randn((1, 12, CL.NARROW.width), generator=g).half().float()
    tok = torch.randint(0, CL.NARROW.vocab, (2, 77), generator=g)
    z = torch.randn((2, 4, 8, 8), generator=g)
    return x, torch.tensor([500]), ctx, tok, z


def _run(m, x, t, ctx, tok, z):
    eps = m.model.diffusion_model(x.cuda(), t.cuda(), context=ctx.cuda()).float().cpu()
    c = m.cond_stage_model.encode_with_transformer(tok).cpu()
    v = m.first_stage_model.decode(z.cuda()).cpu()
    return eps, c, v


def _rel(out, ref):
    rms = ((out - ref).pow(2).mean().sqrt() / ref.pow(2).mean().sqrt()).item()
    return rms, ((out - ref).abs().max() / ref.abs().max()).item()


def test_device_merge_matches_the_reference_weights(gold, base, monkeypatch):
    from t2v_b200 import _lib, videocrafter as vcm
    g = gold
    m = _build(base)
    x, t, ctx, tok, z = _inputs()
    before = _run(m, x, t, ctx, tok, z)
    unet = m.model.diffusion_model
    launches = unet.num_launches()
    shipped = []
    l = _lib.lib()
    for kind in ('unet', 'clip', 'vae'):
        fn = getattr(l, f't2v_{kind}_set_param')
        monkeypatch.setattr(l, f't2v_{kind}_set_param', lambda *a, fn=fn: shipped.append(a[1]) or fn(*a))
    vcm.net_load_lora(m, g['lora1'], alpha=g['alpha1'])
    eps, c, v = _run(m, x, t, ctx, tok, z)
    assert shipped == [] and unet.num_launches() == launches          # nothing re-shipped: same weights version, same plans
    assert (unet.lora_merged(), m.cond_stage_model.transformer.lora_merged(), m.first_stage_model.lora_merged()) == (5, 2, 1)
    Wm = _with(base, g['merged'])
    # UNet: the fp32 oracle on the reference's merged weights rounded to fp16, and a second module shipped those weights
    ref = VC.vc_unet_forward(Wm['unet'], UCFG, x, t, ctx)
    monkeypatch.undo()
    other = _build(Wm)
    e_ship = errs(other.model.diffusion_model(x.cuda(), t.cuda(), context=ctx.cuda()), ref)
    e_hot, e_before = errs(eps, ref), errs(before[0], ref)
    report('vc_lora_unet', hot_vs_oracle_max=e_hot[0], shipped_vs_oracle_max=e_ship[0], unmerged_vs_oracle_max=e_before[0])
    assert e_hot[0] < 5e-3 and e_hot[0] <= 1.5 * e_ship[0] + 5e-4, (e_hot, e_ship)
    assert e_before[0] > e_hot[0] and not torch.equal(eps, before[0]), (e_before, e_hot)    # the merge changed the function
    # CLIP ViT-L text tower (narrow)
    rms, mx = _rel(c, CL.clip_l_text_forward(Wm['clip'], CL.NARROW, tok))
    report('vc_lora_clip', rms=rms, max=mx)
    assert rms < 3e-3 and mx < 1e-2, (rms, mx)
    assert not torch.equal(c, before[1])
    # VAE decoder through the merged 1x1 nin_shortcut
    e_vae = errs(v, VO.vae_decode(Wm['vae'], VO.VAEConfig(), z))
    report('vc_lora_vae', max=e_vae[0], rms=e_vae[1])
    assert e_vae[0] < 6e-3 and e_vae[1] < 4e-3, e_vae
    assert not torch.equal(v, before[2])


def test_change_lora_v2_restores_exactly_and_v1_stays_within_the_documented_residue(gold, base):
    from t2v_b200 import videocrafter as vcm
    g = gold
    m = _build(base)
    inp = _inputs()
    never = _run(m, *inp)
    origin = vcm.change_lora_v2(m, inject_lora=True, lora_scale=g['alpha1'], lora_path=g['lora1'])
    merged = _run(m, *inp)
    origin = vcm.change_lora_v2(m, inject_lora=True, lora_scale=g['alpha2'], lora_path=g['lora2'], last_time_lora=g['lora1'],
                                last_time_lora_scale=g['alpha1'], origin_weight=origin)
    switched = _run(m, *inp)
    # v2's switch = the second LoRA merged into the base directly
    m2 = _build(base)
    vcm.net_load_lora(m2, g['lora2'], alpha=g['alpha2'])
    assert all(torch.equal(a, b) for a, b in zip(switched, _run(m2, *inp)))
    vcm.change_lora_v2(m, inject_lora=False, last_time_lora=g['lora2'], last_time_lora_scale=g['alpha2'], origin_weight=origin)
    assert all(torch.equal(a, b) for a, b in zip(_run(m, *inp), never))           # exact restore: as if never merged
    assert m.model.diffusion_model.lora_merged() == 0 and not any(torch.equal(a, b) for a, b in zip(merged, never))
    # v1: subtract then add; the subtraction happens in fp16 storage -> at most one fp16 ulp of residue per element
    vcm.net_load_lora(m, g['lora1'], alpha=g['alpha1'])
    vcm.change_lora(m, inject_lora=True, lora_scale=g['alpha2'], lora_path=g['lora2'], last_time_lora=g['lora1'],
                    last_time_lora_scale=g['alpha1'])
    eps, c, v = _run(m, *inp)
    Wc = _with(base, _switched(base, g))
    ref = VC.vc_unet_forward(Wc['unet'], UCFG, *inp[:3])
    e1, e2 = errs(eps, ref), errs(switched[0], ref)
    report('vc_lora_change_v1', v1_vs_oracle_max=e1[0], v2_vs_oracle_max=e2[0])
    assert e1[0] < 5e-3 and e1[0] <= 1.5 * e2[0] + 5e-4, (e1, e2)
    rms, mx = _rel(c, CL.clip_l_text_forward(Wc['clip'], CL.NARROW, inp[3]))
    assert rms < 3e-3 and mx < 1e-2, (rms, mx)
    # lora_clear: every handle back to the shipped weights bit for bit
    for mod in (m.model.diffusion_model, m.cond_stage_model.transformer, m.first_stage_model):
        mod.lora_clear()
    assert all(torch.equal(a, b) for a, b in zip(_run(m, *inp), never))


def test_load_model_with_inject_lora(gold, base, tmp_path):
    from t2v_b200 import videocrafter as vcm
    g = gold
    m = _build(base)
    sd = {k: v.detach().cpu() for k, v in m.state_dict().items()}
    ckpt, lora = os.path.join(str(tmp_path), 'model.ckpt'), os.path.join(str(tmp_path), 'lora.ckpt')
    torch.save({'state_dict': sd}, ckpt)
    torch.save(g['lora1'], lora)
    config = {'model': {'params': dict(CL.TINY_LDM, cond_stage_config=dict(target=TARGET, params=_cfg_kw()))}}
    a, _, _ = vcm.load_model(config, ckpt, inject_lora=True, lora_scale=g['alpha1'], lora_path=lora)
    b, _, _ = vcm.load_model(config, ckpt)
    vcm.net_load_lora(b, lora, alpha=g['alpha1'])
    for mm in (a, b):
        mm.cond_stage_model.tokenizer = CL.WordTokenizer(CL.NARROW.vocab)
    inp = _inputs()
    ra, rb = _run(a, *inp), _run(b, *inp)
    assert all(torch.equal(x, y) for x, y in zip(ra, rb))
    assert not torch.equal(ra[0], _run(m, *inp)[0])


def test_process_videocrafter_lora_keys(gold, base):
    from t2v_b200 import videocrafter as vcm
    g = gold
    m = _build(base)
    x_T = torch.randn((1, 4, 4, 8, 8), generator=torch.Generator('cpu').manual_seed(9)).cuda()
    args = dict(prompt='a cat riding a bike', n_prompt='', steps=4, frames=4, seed=3, cfg_scale=4.0, eta=0.0, batch_count=1, x_T=x_T)
    plain = vcm.process_videocrafter(dict(args), model=m)[0]
    lo = dict(args, inject_lora=True, lora_path=g['lora1'], lora_scale=g['alpha1'], lora_trigger_word=' in the style of xyz')
    with_lora = vcm.process_videocrafter(lo, model=m)[0]
    assert not np.array_equal(with_lora, plain) and m.model.diffusion_model.lora_merged() == 5
    # the trigger word is appended to the prompt: the same LoRA with the extended prompt written out gives the same frames
    again = vcm.process_videocrafter(dict(lo, prompt=args['prompt'] + ' in the style of xyz', lora_trigger_word=''), model=m)[0]
    assert np.array_equal(again, with_lora)
    no_word = vcm.process_videocrafter(dict(lo, lora_trigger_word=''), model=m)[0]
    assert not np.array_equal(no_word, with_lora)
    # another scale switches through change_lora_v2; dropping the keys restores the model exactly
    other = vcm.process_videocrafter(dict(lo, lora_scale=g['alpha2']), model=m)[0]
    assert not np.array_equal(other, with_lora)
    assert np.array_equal(vcm.process_videocrafter(dict(args), model=m)[0], plain)
    assert m.model.diffusion_model.lora_merged() == 0 and m.cond_stage_model.transformer.lora_merged() == 0
