"""Writes tests/golden/vc_lora.pt from VideoCrafter's own LoRA code (videocrafter/lvdm/models/modules/lora.py:620-755, imported
through oracle/ref_shim.py) applied to the reference's own `LatentDiffusion` (ddpm3d.py), built on CPU fp32 as
base_t2v/model_config.yaml configures it at the sizes of tests/clip_l_oracle.py's TINY_LDM: UNet model_channels 64, the NARROW
ViT-L text tower, the full VAE (whose channel changes give 1x1 `nin_shortcut` convs).  Weights are seeded
(oracle.unet_oracle.make_weights over the oracles' parameter tables; the tests regenerate them from the seeds).

The fixture holds:
  * `lora1` / `lora2`: seeded rank-4 LoRA dicts keyed from the LatentDiffusion root, fp32 pairs and one fp16 pair, on the
    spatial attn1.to_q (fused q|k|v, LayerNorm-folded on the library), attn2.to_k (cross-attention K), attn1_tmp.to_v
    (relative-position temporal attention), ff.net.0.proj (GEGLU), attn1.to_out.0 (a Sequential index), the text tower's
    q_proj and mlp.fc1, the VAE decoder's 1x1 nin_shortcut (4-D factors), plus an `.alpha` key and a pair on a Conv3d
    (proj_in of the spatial transformer), which the reference skips;
  * `merged`: every touched weight after `net_load_lora(model, lora1, alpha=0.7)`, rounded to fp16 (the library's storage:
    the weights the tests hand to the oracles), which keeps the fixture small;
  * `changed_residue`: per touched weight, max |W - (base + 1.3 * up2 @ down2)| in fp32 after
    `change_lora(model, True, 1.3, lora2, last_time_lora=lora1, last_time_lora_scale=0.7)` -- the reference's add-then-subtract
    residue (~1e-8, far below one fp16 ulp), so the tests build the switched weights as base + 1.3 * up2 @ down2;
  * `skipped`: the keys the reference reported as "missing param at";
  * `tree`: (path, class name) of every nn.Linear and nn.Conv2d module of the reference LatentDiffusion.

    python scripts/make_golden_vc_lora.py
"""
import contextlib
import io
import os
import sys
import tempfile
import types
from types import SimpleNamespace

import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'tests'))
sys.path.insert(0, ROOT)
from oracle import ref_shim                                   # noqa: E402
from oracle import unet_oracle as UO                          # noqa: E402
from oracle import vae_oracle as VO                           # noqa: E402
from oracle import vc_oracle as VC                            # noqa: E402
import clip_l_oracle as CL                                    # noqa: E402

SEEDS = {'unet': 4, 'clip': 8, 'vae_dec': 3, 'vae_enc': 5, 'lora1': 61, 'lora2': 62}
ALPHA1, ALPHA2, RANK = 0.7, 1.3, 4
UNET = 'model.diffusion_model.'
TB = UNET + 'input_blocks.1.1.transformer_blocks.0.'
# (module path, fp16 pair, 4-D factors)
TARGETS = [(TB + 'attn1.to_q', False, False), (TB + 'attn2.to_k', False, False), (TB + 'attn1_tmp.to_v', True, False),
           (TB + 'ff.net.0.proj', False, False), (UNET + 'input_blocks.2.1.transformer_blocks.0.attn1.to_out.0', False, False),
           ('cond_stage_model.transformer.text_model.encoder.layers.0.self_attn.q_proj', False, False),
           ('cond_stage_model.transformer.text_model.encoder.layers.2.mlp.fc1', False, False),
           ('first_stage_model.decoder.up.0.block.0.nin_shortcut', False, True),
           (UNET + 'input_blocks.1.1.proj_in', False, True)]             # a Conv3d (1,1,1) in the reference: skipped


def weights():
    """Seeded weights of the tiny LatentDiffusion, keyed from its root."""
    W = {}
    for prefix, specs, seed in ((UNET, VC.vc_param_specs(VC.VCConfig(**CL.TINY_LDM['unet_config'])), SEEDS['unet']),
                                ('cond_stage_model.transformer.', CL.clip_l_param_specs(CL.NARROW), SEEDS['clip']),
                                ('first_stage_model.', VO.decoder_param_specs(VO.VAEConfig()), SEEDS['vae_dec']),
                                ('first_stage_model.', VO.encoder_param_specs(VO.VAEConfig()), SEEDS['vae_enc'])):
        W.update({prefix + k: v for k, v in UO.make_weights(specs, seed=seed).items()})
    return W


def make_lora(shapes, seed):
    """{path.lora_up.weight, path.lora_down.weight} for every target (down listed first for every other one), + one .alpha."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for i, (path, half, conv) in enumerate(TARGETS):
        out, cols = shapes[path]
        up = torch.randn((out, RANK), generator=g) * 0.05
        down = torch.randn((RANK, cols), generator=g) * 0.05
        if conv:
            up, down = up[:, :, None, None], down[:, :, None, None]
        if half:
            up, down = up.half(), down.half()
        pair = [(path + '.lora_up.weight', up), (path + '.lora_down.weight', down)]
        for k, v in (pair[::-1] if i % 2 else pair):
            sd[k] = v
        if i == 0:
            sd[path + '.alpha'] = torch.tensor(float(RANK))
    return sd


def reference_model():
    """ddpm3d.LatentDiffusion as in scripts/make_golden_clip_l.py's layout check (pytorch_lightning stood in by nn.Module)."""
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
    m.device = torch.device('cpu')           # a LightningModule property the LoRA loader reads
    return m.eval()


def run(fn, *a, **kw):
    """fn(*a, **kw) with its prints captured; returns the keys reported as 'missing param at'."""
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        fn(*a, **kw)
    text = buf.getvalue()
    sys.stdout.write(text)
    return [line.split('missing param at:', 1)[1].strip() for line in text.splitlines() if 'missing param at:' in line]


def main():
    m = reference_model()
    from videocrafter.lvdm.models.modules import lora as L
    W = weights()
    res = m.load_state_dict(W, strict=False)
    assert not res.unexpected_keys and all('.' not in k or 'position_ids' in k for k in res.missing_keys), res
    mods = dict(m.named_modules())
    tree = sorted((p, type(mod).__name__) for p, mod in mods.items() if type(mod) in (nn.Linear, nn.Conv2d))
    shapes = {p: (mods[p].weight.shape[0], mods[p].weight[0].numel()) for p, _, _ in TARGETS}
    lora1, lora2 = make_lora(shapes, SEEDS['lora1']), make_lora(shapes, SEEDS['lora2'])
    touched = [p + '.weight' for p, _, _ in TARGETS if type(mods[p]) in (nn.Linear, nn.Conv2d)]
    base = {k: m.state_dict()[k].clone() for k in touched}
    with tempfile.TemporaryDirectory() as d:
        p1, p2 = os.path.join(d, 'lora1.ckpt'), os.path.join(d, 'lora2.ckpt')
        torch.save(lora1, p1)
        torch.save(lora2, p2)
        with torch.no_grad():
            skipped = run(L.net_load_lora, m, p1, alpha=ALPHA1)
            merged = {k: m.state_dict()[k].clone() for k in touched}
            run(L.change_lora, m, inject_lora=True, lora_scale=ALPHA2, lora_path=p2, last_time_lora=p1, last_time_lora_scale=ALPHA1)
            changed = {k: m.state_dict()[k].clone() for k in touched}
            origin = L.change_lora_v2(m, inject_lora=False, last_time_lora=p2, last_time_lora_scale=ALPHA2,
                                      origin_weight=None)
    moved = {k: (merged[k] - base[k]).abs().max().item() for k in touched}
    print(f'[net_load_lora] {len(touched)} weights merged (largest change {max(moved.values()):.3e}); skipped {skipped}')
    residue = {k: (changed[k] - (base[k] + ALPHA2 * _delta(lora2, k))).abs().max().item() for k in touched}
    print(f"[change_lora] largest residue of lora1's removal vs base + 1.3 lora2: {max(residue.values()):.3e}")
    assert max(residue.values()) < 1e-6
    print(f'[change_lora_v2] origin_weight keys {sorted(origin)[:2]} ...')
    out = {'seeds': SEEDS, 'alpha1': ALPHA1, 'alpha2': ALPHA2, 'lora1': lora1, 'lora2': lora2,
           'merged': {k: v.half() for k, v in merged.items()}, 'changed_residue': residue, 'skipped': skipped, 'tree': tree,
           'origin_keys': sorted(origin)}
    path = os.path.join(ROOT, 'tests', 'golden', 'vc_lora.pt')
    torch.save(out, path)
    print(f'wrote {path} ({os.path.getsize(path) / 1e3:.0f} kB); {len(tree)} Linear / Conv2d modules in the reference tree')


def _delta(lora, weight_key):
    p = weight_key[:-len('.weight')]
    up, down = lora[p + '.lora_up.weight'].float(), lora[p + '.lora_down.weight'].float()
    d = up.reshape(up.shape[0], -1) @ down.reshape(down.shape[0], -1)
    return d.reshape(d.shape + (1, 1)) if up.dim() == 4 else d


if __name__ == '__main__':
    main()
