"""VideoCrafter text conditioning: the OpenAI CLIP ViT-L/14 text model of FrozenCLIPEmbedder
(videocrafter/lvdm/models/modules/condition_modules.py:15-40) on the library (csrc/clip.cu, arch 1).

The CPU oracle (tests/clip_l_oracle.py) is pinned against tests/golden/clip_l.pt, which holds the reference class's own
output (scripts/make_golden_clip_l.py), and against a live transformers CLIPTextModel where transformers is installed.
The GPU tests compare the library tower, the tokenisation framing and VideoCrafter's string-in path with that oracle;
they do not import transformers."""
import os

import numpy as np
import pytest
import torch

from oracle import unet_oracle as UO, vae_oracle as VO, vc_oracle as VC
import clip_l_oracle as CL

FULL = CL.ClipLConfig()
NARROW = CL.NARROW
CONFIGS = {'narrow': NARROW, 'ViT-L-14': FULL}
TARGET = 'lvdm.models.modules.condition_modules.FrozenCLIPEmbedder'


def _gold(gold_dir):
    return torch.load(os.path.join(gold_dir, 'clip_l.pt'))


def _cfg_kw(cfg):
    return dict(width=cfg.width, heads=cfg.heads, layers=cfg.layers, vocab=cfg.vocab, max_length=cfg.context)


def _hf_tokenizer(tmp_path, vocab):
    transformers = pytest.importorskip('transformers')
    vf, mf = CL.write_synthetic_tokenizer(str(tmp_path), vocab)
    return transformers.CLIPTokenizer(vf, mf, pad_token='<|endoftext|>')


# ---------------------------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize('name', ['narrow', 'full'])
def test_oracle_matches_reference_golden(gold_dir, name):
    g = _gold(gold_dir)
    cfg = CL.ClipLConfig(**g[name]['cfg'])
    W = UO.make_weights(CL.clip_l_param_specs(cfg), seed=g['wseed'])
    out = CL.clip_l_text_forward(W, cfg, g[name]['input_ids'])
    ref = g[name]['last_hidden_state']
    assert out.shape == ref.shape == (len(g['prompts']), 77, cfg.width)
    assert torch.allclose(out, ref, rtol=0, atol=1e-5), (out - ref).abs().max()


def test_oracle_matches_live_transformers():
    transformers = pytest.importorskip('transformers')
    cfg = NARROW
    W = UO.make_weights(CL.clip_l_param_specs(cfg), seed=3)
    m = transformers.CLIPTextModel(transformers.CLIPTextConfig(
        vocab_size=cfg.vocab, hidden_size=cfg.width, intermediate_size=4 * cfg.width, num_hidden_layers=cfg.layers,
        num_attention_heads=cfg.heads, max_position_embeddings=cfg.context, hidden_act='quick_gelu', layer_norm_eps=1e-5))
    m.load_state_dict(W, strict=True)
    tok = torch.randint(0, cfg.vocab, (2, cfg.context), generator=torch.Generator().manual_seed(1))
    with torch.no_grad():
        ref = m.eval()(input_ids=tok).last_hidden_state
    out = CL.clip_l_text_forward(W, cfg, tok)
    assert torch.allclose(out, ref, rtol=0, atol=1e-5), (out - ref).abs().max()


def _meta_embedder(cfg, **kw):
    from t2v_b200.clip import FrozenCLIPEmbedder
    with torch.device('meta'):
        return FrozenCLIPEmbedder(**_cfg_kw(cfg), **kw)


def test_tokenisation_matches_clip_tokenizer(tmp_path):
    """Short prompt, a prompt over 75 tokens (truncated), the empty negative prompt: <|startoftext|>, <= 75 ids,
    <|endoftext|>, padded with <|endoftext|> -- through a CLIPTokenizer and through a plain `.encode` tokenizer."""
    hf = _hf_tokenizer(tmp_path, FULL.vocab)
    prompts = ['a cat riding a bike', ' '.join(['stone tower at sea'] * 12), '']
    ref = hf(prompts, truncation=True, max_length=77, padding='max_length', return_tensors='pt')['input_ids']
    assert ref[0, 0] == 49406 and ref[2, 1] == 49407 and ref[1, -1] == 49407
    e = _meta_embedder(FULL, tokenizer=hf)
    assert torch.equal(e.tokenize(prompts), ref)

    class Plain(object):
        def encode(self, text):
            return hf(text, add_special_tokens=False)['input_ids']
    p = _meta_embedder(FULL, tokenizer=Plain())
    assert (p.id_start, p.id_end) == (49406, 49407)
    assert torch.equal(p.tokenize(prompts), ref)
    assert torch.equal(p.tokenize(prompts[0]), ref[:1])


def test_plain_tokenizer_framing_and_missing_tokenizer():
    e = _meta_embedder(FULL, tokenizer=CL.WordTokenizer(FULL.vocab))
    ids = e.tokenize(['ab cd', 'abcdefghij ' * 20])
    assert ids.shape == (2, 77) and ids.dtype == torch.long
    assert ids[0, :5].tolist() == [49406, 3, 30, 5, 32] and (ids[0, 5:] == 49407).all()
    assert ids[1, 0] == 49406 and ids[1, 76] == 49407 and (ids[1, 1:76] < 300).all()
    with pytest.raises(RuntimeError, match='tokenizer'):
        _meta_embedder(FULL).tokenize(['a prompt'])


def test_state_dict_layout_matches_clip_text_model():
    transformers = pytest.importorskip('transformers')
    with torch.device('meta'):
        hf = transformers.CLIPTextModel(transformers.CLIPTextConfig(hidden_size=768, intermediate_size=3072, num_attention_heads=12,
                                                                    num_hidden_layers=12, hidden_act='quick_gelu'))
    e = _meta_embedder(FULL)
    sd = e.state_dict()
    assert set(sd) == {'transformer.' + k for k in hf.state_dict()}
    assert len(sd) == 196 and set(sd) == {'transformer.' + k for k in CL.clip_l_param_specs(FULL)}
    for k, v in hf.state_dict().items():
        assert tuple(sd['transformer.' + k].shape) == tuple(v.shape), k
    assert set(e.transformer._native_names) == set(CL.clip_l_param_specs(FULL))


def _ldm(**kw):
    from t2v_b200.videocrafter import LatentDiffusion
    return LatentDiffusion(**CL.TINY_LDM, cond_stage_config=dict(target=TARGET, params=_cfg_kw(NARROW)), **kw)


def test_latent_diffusion_builds_and_loads_the_text_encoder_strictly():
    from t2v_b200.clip import FrozenCLIPEmbedder
    m = _ldm()
    assert isinstance(m.cond_stage_model, FrozenCLIPEmbedder) and 'cond_stage_model' in dict(m.named_children())
    sd = m.state_dict()
    clip_keys = {k for k in sd if k.startswith('cond_stage_model.')}
    assert clip_keys == {'cond_stage_model.transformer.' + k for k in CL.clip_l_param_specs(NARROW)}
    W = UO.make_weights(CL.clip_l_param_specs(NARROW), seed=5)
    ckpt = dict(sd)
    ckpt.update({'cond_stage_model.transformer.' + k: v for k, v in W.items()})
    ckpt['cond_stage_model.transformer.text_model.embeddings.position_ids'] = torch.arange(77).expand(1, -1)
    m2 = _ldm()
    res = m2.load_state_dict(ckpt, strict=True)
    assert not res.missing_keys and not res.unexpected_keys
    got = m2.cond_stage_model.transformer.state_dict()
    assert all(torch.equal(got[k], W[k]) for k in W)
    with pytest.raises(RuntimeError):                      # anything else unexpected is still reported
        m2.load_state_dict(dict(ckpt, **{'cond_stage_model.transformer.text_model.extra': torch.zeros(1)}), strict=True)
    with pytest.raises(NotImplementedError):
        _ldm_target('lvdm.models.modules.condition_modules.FrozenOpenCLIPEmbedder')


def test_latent_diffusion_layout_matches_reference(gold_dir):
    """The full state-dict layout of LatentDiffusion with the text encoder equals the reference LatentDiffusion's at the same
    sizes (what a VideoCrafter model.ckpt holds), and the schedule / posterior buffers equal the reference's values."""
    ref = _gold(gold_dir)['ldm']
    sd = _ldm().state_dict()
    assert len(sd) == ref['n_keys'] and CL.layout_digest(sd) == ref['layout_sha256']
    for k, v in ref['buffers'].items():
        assert torch.equal(sd[k], v), k


def _ldm_target(target):
    from t2v_b200.videocrafter import LatentDiffusion
    return LatentDiffusion(unet_config=dict(model_channels=64, context_dim=128, temporal_length=4), image_size=[8, 8],
                           video_length=4, cond_stage_config=dict(target=target))


def test_local_snapshot_directory_loads_tokenizer_and_weights(tmp_path):
    """version = a local Hugging Face snapshot: CLIPTokenizer.from_pretrained(dir, local_files_only=True) and the
    `text_model.*` weights of the directory (vision-side keys and position_ids are skipped)."""
    transformers = pytest.importorskip('transformers')
    pytest.importorskip('safetensors')
    from safetensors.torch import save_file
    from t2v_b200.clip import FrozenCLIPEmbedder
    hf = _hf_tokenizer(tmp_path, NARROW.vocab)
    hf.save_pretrained(str(tmp_path))
    W = UO.make_weights(CL.clip_l_param_specs(NARROW), seed=6)
    sd = {k: v.contiguous() for k, v in W.items()}
    sd['text_model.embeddings.position_ids'] = torch.arange(77).unsqueeze(0)
    sd['vision_model.post_layernorm.weight'] = torch.ones(4)
    save_file(sd, os.path.join(str(tmp_path), 'model.safetensors'))
    e = FrozenCLIPEmbedder(version=str(tmp_path), **_cfg_kw(NARROW))
    assert isinstance(e.tokenizer, transformers.CLIPTokenizer)
    got = e.transformer.state_dict()
    assert all(torch.equal(got[k], W[k]) for k in W)
    prompts = ['a cat riding a bike', '']
    assert torch.equal(e.tokenize(prompts), hf(prompts, truncation=True, max_length=77, padding='max_length',
                                               return_tensors='pt')['input_ids'])


def test_clip_config_arch_field_is_last_and_zero_by_default():
    import ctypes as C
    from t2v_b200 import _lib
    assert [f[0] for f in _lib.ClipConfigC._fields_] == ['width', 'heads', 'layers_run', 'context', 'vocab', 'arch']
    assert _lib.ClipConfigC(1024, 16, 23, 77, 49408).arch == 0
    l = _lib.load_library()
    cfg = _lib.ClipConfigC(128, 2, 3, 77, 300, 2)
    h = C.c_void_p()
    assert l.t2v_clip_create(C.byref(cfg), C.byref(h)) != 0                  # unknown arch is refused


# ---------------------------------------------------------------------------------------------------------------- GPU
_EMB = {}


def _gpu_embedder(name):
    """FrozenCLIPEmbedder on the GPU with seeded fp32 weights (shipped as fp16); cached per config."""
    if name not in _EMB:
        from t2v_b200.clip import FrozenCLIPEmbedder
        cfg = CONFIGS[name]
        W = UO.make_weights(CL.clip_l_param_specs(cfg), seed=4)
        e = FrozenCLIPEmbedder(**_cfg_kw(cfg), tokenizer=CL.WordTokenizer(cfg.vocab))
        e.transformer.load_state_dict(W, strict=True)
        e.half().cuda()
        _EMB[name] = (e, {k: v.half().float() for k, v in W.items()})
    return _EMB[name]


def _rel(out, ref):
    rms = ((out - ref).pow(2).mean().sqrt() / ref.pow(2).mean().sqrt()).item()
    mx = ((out - ref).abs().max() / ref.abs().max()).item()
    return rms, mx


@pytest.mark.gpu
@pytest.mark.parametrize('B', [1, 2])
@pytest.mark.parametrize('name', ['narrow', 'ViT-L-14'])
def test_text_tower_vs_oracle(name, B):
    cfg = CONFIGS[name]
    e, Wh = _gpu_embedder(name)
    tok = torch.randint(0, cfg.vocab, (B, cfg.context), generator=torch.Generator().manual_seed(2))
    out = e.encode_with_transformer(tok).cpu()
    assert out.dtype == torch.float32 and out.shape == (B, cfg.context, cfg.width)
    ref = CL.clip_l_text_forward(Wh, cfg, tok)
    rms, mx = _rel(out, ref)
    print(f'[parity] clip ViT-L tower {name} B={B}: rel-rms {rms:.3e} max {mx:.3e}')
    assert rms < 3e-3 and mx < 1e-2, (rms, mx)
    assert torch.equal(e.encode_with_transformer(tok).cpu(), out)                 # graph replay, deterministic


@pytest.mark.gpu
def test_full_tower_vs_reference_golden(gold_dir):
    from t2v_b200.clip import FrozenCLIPEmbedder
    g = _gold(gold_dir)
    cfg = CL.ClipLConfig(**g['full']['cfg'])
    W = UO.make_weights(CL.clip_l_param_specs(cfg), seed=g['wseed'])
    e = FrozenCLIPEmbedder(**_cfg_kw(cfg))
    e.transformer.load_state_dict(W, strict=True)
    e.half().cuda()
    ref = g['full']['last_hidden_state']
    for B in (1, len(g['prompts'])):
        out = e.encode_with_transformer(g['full']['input_ids'][:B]).cpu()
        rms, mx = _rel(out, ref[:B])
        print(f'[parity] clip ViT-L tower vs reference FrozenCLIPEmbedder B={B}: rel-rms {rms:.3e} max {mx:.3e}')
        assert rms < 3e-3 and mx < 1e-2, (rms, mx)


@pytest.fixture(scope='module')
def vc_model():
    W = UO.make_weights(VC.vc_param_specs(VC.VCConfig(model_channels=64, context_dim=NARROW.width, temporal_length=4)), seed=4)
    Wv = UO.make_weights(VO.decoder_param_specs(VO.VAEConfig()), seed=3)
    Wc = UO.make_weights(CL.clip_l_param_specs(NARROW), seed=8)
    m = _ldm()
    m.cond_stage_model.tokenizer = CL.WordTokenizer(NARROW.vocab)
    m.cond_stage_model.transformer.load_state_dict(Wc, strict=True)
    m.model.diffusion_model.load_state_dict(W, strict=True)
    m.first_stage_model.load_state_dict(Wv, strict=False)
    return m.half().cuda().eval(), Wc


@pytest.mark.gpu
def test_videocrafter_encodes_strings_end_to_end(vc_model):
    from t2v_b200 import videocrafter as vcm
    m, Wc = vc_model
    prompt, n_prompt = 'a cat riding a bike', ''
    c = m.get_learned_conditioning([prompt])
    uc = m.get_learned_conditioning([n_prompt])
    assert c.shape == uc.shape == (1, 77, NARROW.width) and c.dtype == torch.float32 and c.is_cuda
    tok = m.cond_stage_model.tokenize([prompt, n_prompt])
    ref = CL.clip_l_text_forward({k: v.half().float() for k, v in Wc.items()}, NARROW, tok)
    rms, mx = _rel(torch.cat([c, uc]).cpu(), ref)
    print(f'[parity] VideoCrafter conditioning (narrow ViT-L): rel-rms {rms:.3e} max {mx:.3e}')
    assert rms < 3e-3 and mx < 1e-2, (rms, mx)
    x_T = torch.randn((1, 4, 4, 8, 8), generator=torch.Generator('cpu').manual_seed(9)).cuda()
    kw = dict(ddim_steps=4, eta=0.0, cfg_scale=4.0, num_frames=4, x_T=x_T)
    vids = vcm.sample_text2video(m, prompt, n_prompt, 1, 1, **kw)
    vids_t = vcm.sample_text2video(m, c, uc, 1, 1, **kw)
    assert vids.shape == (1, 3, 4, 64, 64) and np.array_equal(vids, vids_t)
    out = vcm.process_videocrafter(dict(prompt=prompt, n_prompt=n_prompt, steps=4, frames=4, seed=3, cfg_scale=4.0, eta=0.0,
                                        batch_count=1, x_T=x_T), model=m)
    assert len(out) == 1 and np.array_equal(out[0], vids)


@pytest.mark.gpu
def test_load_model_from_checkpoint(vc_model, tmp_path, gold_dir):
    """load_model: yaml-shaped config dict, a Lightning-style {'state_dict': ...} checkpoint with the reference
    LatentDiffusion's key set (its schedule and posterior buffers, from the fixture) and the legacy position_ids buffer,
    strict load, fp16 on the GPU; the loaded model encodes prompts as the original does."""
    from t2v_b200.videocrafter import load_model
    m = vc_model[0]
    ref = _gold(gold_dir)['ldm']
    sd = {k: v.detach().cpu() for k, v in m.state_dict().items() if '.' in k}
    sd.update(ref['buffers'])
    assert CL.layout_digest(sd) == ref['layout_sha256']                         # exactly the reference's tensors
    sd['cond_stage_model.transformer.text_model.embeddings.position_ids'] = torch.arange(77).unsqueeze(0)
    path = os.path.join(str(tmp_path), 'model.ckpt')
    torch.save({'state_dict': sd, 'global_step': 12, 'epoch': 3}, path)
    config = {'model': {'target': 'lvdm.models.ddpm3d.LatentDiffusion', 'params': {
        'image_size': CL.TINY_LDM['image_size'], 'video_length': CL.TINY_LDM['video_length'], 'conditioning_key': 'crossattn',
        'scale_factor': 0.18215, 'unet_config': {'target': 'lvdm.models.modules.openaimodel3d.UNetModel',
                                                 'params': CL.TINY_LDM['unet_config']},
        'first_stage_config': {'target': 'lvdm.models.autoencoder.AutoencoderKL', 'params': {'embed_dim': 4}},
        'cond_stage_config': {'target': TARGET, 'params': _cfg_kw(NARROW)}}}}
    m2, step, epoch = load_model(config, path)
    assert (step, epoch) == (12, 3) and not m2.training
    assert next(m2.cond_stage_model.transformer.parameters()).dtype == torch.float16
    m2.cond_stage_model.tokenizer = m.cond_stage_model.tokenizer
    assert torch.equal(m2.get_learned_conditioning(['a cat riding a bike']), m.get_learned_conditioning(['a cat riding a bike']))


@pytest.mark.gpu
def test_parent_load_after_encode_ships_the_new_weights(vc_model):
    """A state dict loaded through LatentDiffusion (copies into the tower's parameters in place) after the tower has
    already encoded is what the next encode uses."""
    m, Wc = vc_model
    before = m.get_learned_conditioning(['a cat riding a bike'])
    W2 = UO.make_weights(CL.clip_l_param_specs(NARROW), seed=9)
    base = {k: v.detach().clone() for k, v in m.state_dict().items()}
    try:
        m.load_state_dict(dict(base, **{'cond_stage_model.transformer.' + k: v for k, v in W2.items()}), strict=True)
        after = m.get_learned_conditioning(['a cat riding a bike'])
        ref = CL.clip_l_text_forward({k: v.half().float() for k, v in W2.items()}, NARROW, m.cond_stage_model.tokenize(['a cat riding a bike']))
        rms, mx = _rel(after.cpu(), ref)
        assert not torch.equal(after, before) and rms < 3e-3 and mx < 1e-2, (rms, mx)
    finally:
        m.load_state_dict(base, strict=True)
