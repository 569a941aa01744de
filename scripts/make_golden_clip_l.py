"""Writes tests/golden/clip_l.pt: VideoCrafter's FrozenCLIPEmbedder (the reference's own class,
videocrafter/lvdm/models/modules/condition_modules.py:15-40, imported through oracle/ref_shim.py) run on CPU fp32 at a narrow
and at the full ViT-L/14 text config, and checks the oracle restatement (tests/clip_l_oracle.py) against it.

Needs the reference source tree and `transformers`; nothing is downloaded.  For the duration of the call the class's
`CLIPTokenizer.from_pretrained` / `CLIPTextModel.from_pretrained` are replaced by offline constructors: a CLIPTokenizer over
a synthetic vocab.json / merges.txt in a temporary directory and a CLIPTextModel(CLIPTextConfig(..., hidden_act='quick_gelu'))
holding seeded weights (oracle.unet_oracle.make_weights).  The fixture stores prompts, the reference's input_ids and
last_hidden_state; tests regenerate the weights from the seed.

    python scripts/make_golden_clip_l.py
"""
import os
import sys
import tempfile
from types import SimpleNamespace

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'tests'))
sys.path.insert(0, ROOT)
from oracle import ref_shim                                   # noqa: E402
from oracle import unet_oracle as UO                          # noqa: E402
import clip_l_oracle as CL                                    # noqa: E402

PROMPTS = ['a cat riding a bike', '', ' '.join(['stone tower at sea'] * 12)]      # short, empty (n_prompt), > 75 tokens
WSEED = 7


def reference_run(cfg, wseed, prompts):
    import transformers
    from transformers import CLIPTextConfig, CLIPTextModel, CLIPTokenizer
    ref_shim.install()
    from videocrafter.lvdm.models.modules import condition_modules as cm
    W = UO.make_weights(CL.clip_l_param_specs(cfg), seed=wseed)
    with tempfile.TemporaryDirectory() as d:
        vf, mf = CL.write_synthetic_tokenizer(d, cfg.vocab)
        enc = CL.synthetic_vocab(cfg.vocab)[0]
        tok = CLIPTokenizer(vf, mf, pad_token='<|endoftext|>')

        def make_model(version):
            m = CLIPTextModel(CLIPTextConfig(vocab_size=cfg.vocab, hidden_size=cfg.width, intermediate_size=4 * cfg.width,
                                             num_hidden_layers=cfg.layers, num_attention_heads=cfg.heads,
                                             max_position_embeddings=cfg.context, hidden_act='quick_gelu', layer_norm_eps=1e-5,
                                             bos_token_id=enc['<|startoftext|>'], eos_token_id=enc['<|endoftext|>'],
                                             pad_token_id=enc['<|endoftext|>']))
            m.load_state_dict(W, strict=True)
            return m
        saved = cm.CLIPTokenizer, cm.CLIPTextModel
        cm.CLIPTokenizer = SimpleNamespace(from_pretrained=lambda version: tok)
        cm.CLIPTextModel = SimpleNamespace(from_pretrained=make_model)
        try:
            emb = cm.FrozenCLIPEmbedder(device='cpu', max_length=cfg.context)
        finally:
            cm.CLIPTokenizer, cm.CLIPTextModel = saved
        with torch.no_grad():
            z = emb(prompts)
            ids = emb.tokenizer(prompts, truncation=True, max_length=cfg.context, padding='max_length',
                                return_tensors='pt')['input_ids']
    o = CL.clip_l_text_forward(W, cfg, ids)
    err = (o - z).abs().max().item()
    print(f'[clip_l {cfg.width}x{cfg.layers}] oracle-vs-reference max|d| = {err:.3e} (ref absmax {z.abs().max().item():.3f})')
    assert err < 1e-5 * max(1.0, z.abs().max().item())
    return {'cfg': dict(cfg.__dict__), 'input_ids': ids.clone(), 'last_hidden_state': z.clone(), 'transformers': transformers.__version__}


def reference_ldm_layout():
    """The reference LatentDiffusion (ddpm3d.py) as base_t2v/model_config.yaml configures it, at CL.TINY_LDM's sizes with
    the NARROW text tower: what a VideoCrafter model.ckpt's state dict holds, as a layout digest, plus the top-level
    (schedule / posterior) buffers.  pytorch_lightning is not installed: LightningModule is stood in by nn.Module, which
    the constructor and state_dict only need."""
    import types
    import torch.nn as nn
    from transformers import CLIPTextConfig, CLIPTextModel
    ref_shim.install()
    if 'pytorch_lightning' not in sys.modules:
        pl = types.ModuleType('pytorch_lightning')
        pl.LightningModule = nn.Module
        ut = types.ModuleType('pytorch_lightning.utilities')
        ut.rank_zero_only = lambda f: f
        pl.utilities = ut
        sys.modules['pytorch_lightning'], sys.modules['pytorch_lightning.utilities'] = pl, ut
    from videocrafter.lvdm.models import ddpm3d
    from videocrafter.lvdm.models.modules import condition_modules as cm
    c, u = CL.NARROW, CL.TINY_LDM['unet_config']
    saved = cm.CLIPTokenizer, cm.CLIPTextModel
    cm.CLIPTokenizer = SimpleNamespace(from_pretrained=lambda version: None)
    cm.CLIPTextModel = SimpleNamespace(from_pretrained=lambda version: CLIPTextModel(CLIPTextConfig(
        vocab_size=c.vocab, hidden_size=c.width, intermediate_size=4 * c.width, num_hidden_layers=c.layers, num_attention_heads=c.heads,
        max_position_embeddings=c.context, hidden_act='quick_gelu')))
    try:
        m = ddpm3d.LatentDiffusion(
            unet_config=dict(target='lvdm.models.modules.openaimodel3d.UNetModel', params=dict(
                image_size=32, in_channels=4, out_channels=4, model_channels=u['model_channels'], attention_resolutions=[4, 2, 1],
                num_res_blocks=2, channel_mult=[1, 2, 4, 4], num_heads=8, transformer_depth=1, context_dim=u['context_dim'],
                use_checkpoint=True, legacy=False, kernel_size_t=1, padding_t=0, temporal_length=u['temporal_length'],
                use_relative_position=True)),
            first_stage_config=dict(target='lvdm.models.autoencoder.AutoencoderKL', params=dict(
                embed_dim=4, monitor='val/rec_loss', lossconfig=dict(target='torch.nn.Identity'), ddconfig=dict(
                    double_z=True, z_channels=4, resolution=256, in_channels=3, out_ch=3, ch=128, ch_mult=[1, 2, 4, 4],
                    num_res_blocks=2, attn_resolutions=[], dropout=0.0))),
            cond_stage_config=dict(target='lvdm.models.modules.condition_modules.FrozenCLIPEmbedder'),
            linear_start=0.00085, linear_end=0.012, num_timesteps_cond=1, log_every_t=200, timesteps=1000, first_stage_key='video',
            cond_stage_key='caption', image_size=CL.TINY_LDM['image_size'], video_length=CL.TINY_LDM['video_length'], channels=4,
            cond_stage_trainable=False, conditioning_key='crossattn', scale_by_std=False, scale_factor=0.18215)
    finally:
        cm.CLIPTokenizer, cm.CLIPTextModel = saved
    sd = m.state_dict()
    top = {k: v.clone() for k, v in sd.items() if '.' not in k}
    print(f'[ldm layout] {len(sd)} tensors; top-level buffers {sorted(top)}')
    return {'layout_sha256': CL.layout_digest(sd), 'n_keys': len(sd), 'buffers': top}


def main():
    out = {'wseed': WSEED, 'prompts': PROMPTS}
    out['narrow'] = reference_run(CL.NARROW, WSEED, PROMPTS)
    out['full'] = reference_run(CL.ClipLConfig(), WSEED, PROMPTS)
    out['ldm'] = reference_ldm_layout()
    path = os.path.join(ROOT, 'tests', 'golden', 'clip_l.pt')
    torch.save(out, path)
    print(f'wrote {path} ({os.path.getsize(path) / 1e6:.2f} MB)')


if __name__ == '__main__':
    main()
