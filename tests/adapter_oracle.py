"""TEST INFRASTRUCTURE ONLY -- CPU fp32 restatement of VideoCrafter's depth-adapter path.

  * `adapter_forward`     the T2I-Adapter (videocrafter/lvdm/models/modules/adapter.py:39-105): PixelUnshuffle(8), conv_in,
                          nums_rb ResnetBlocks per level (the first block of a later level downsamples: 3x3 stride-2 conv or
                          2x2 average pooling; in_conv where in_c != out_c or not sk; h = block2(relu(block1(x))); h + skep(x)
                          or h + x), one feature map per level.
  * `vc_unet_forward`     UNetModel.forward (openaimodel3d.py:632-670) WITH `features_adapter`: after input block id with
                          (id + 1) % 3 == 0, h = h + features_adapter[i] before the skip push.  Composed from
                          oracle/vc_oracle.py's enumeration and block functions; without features it is vc_oracle's forward.
  * `vc_ddim_sample`      lvdm/samplers/ddim.py with the features passed to both apply_model calls (oracle/vc_oracle.py's
                          sampler takes any model callable).
  * `get_batch_depth`     T2VAdapterDepth.get_batch_depth (ddpm3d.py:1448-1468).

Pinned by tests/test_adapter.py against tests/golden/adapter.pt, which scripts/make_golden_adapter.py writes from the
reference's own classes.
"""
from typing import Dict, List

import torch
import torch.nn.functional as F

from oracle import vc_oracle as VC

DEPTH = dict(channels=[320, 640, 1280, 1280], nums_rb=2, cin=64, ksize=1, sk=True, use_conv=False)   # VideoCrafter's depth adapter
NARROW_A = dict(channels=[64, 128, 256, 256], nums_rb=2, cin=64, ksize=1, sk=True, use_conv=False)
NARROW_B = dict(channels=[64, 128, 256, 256], nums_rb=3, cin=64, ksize=3, sk=True, use_conv=True)
DEFAULTS = dict(channels=[320, 640, 1280, 1280], nums_rb=3, cin=64, ksize=3, sk=False, use_conv=True)    # Adapter()'s defaults


def adapter_param_specs(channels, nums_rb=3, cin=64, ksize=3, sk=False, use_conv=True):
    """state_dict keys / shapes of adapter.py's Adapter."""
    S = {}

    def conv(p, o, i, k):
        S[p + '.weight'] = (o, i, k, k)
        S[p + '.bias'] = (o,)
    conv('conv_in', channels[0], cin, 3)
    for i in range(len(channels)):
        for j in range(nums_rb):
            p = f'body.{i * nums_rb + j}'
            down = i != 0 and j == 0
            in_c, out_c = (channels[i - 1] if down else channels[i]), channels[i]
            if in_c != out_c or not sk:
                conv(p + '.in_conv', out_c, in_c, ksize)
            conv(p + '.block1', out_c, out_c, 3)
            conv(p + '.block2', out_c, out_c, ksize)
            if not sk:
                conv(p + '.skep', out_c, in_c, ksize)
            if down and use_conv:
                conv(p + '.down_opt.op', in_c, in_c, 3)
    return S


def adapter_forward(W: Dict[str, torch.Tensor], x, channels, nums_rb=3, cin=64, ksize=3, sk=False, use_conv=True) -> List[torch.Tensor]:
    """x [N, cin/64, H, W] -> [N, channels[l], h_l, w_l] per level."""
    pad = ksize // 2
    x = F.pixel_unshuffle(x, 8)
    x = F.conv2d(x, W['conv_in.weight'], W['conv_in.bias'], padding=1)
    feats = []
    for i in range(len(channels)):
        for j in range(nums_rb):
            p = f'body.{i * nums_rb + j}'
            if i != 0 and j == 0:
                if use_conv:
                    x = F.conv2d(x, W[p + '.down_opt.op.weight'], W[p + '.down_opt.op.bias'], stride=2, padding=1)
                else:
                    x = F.avg_pool2d(x, kernel_size=2, stride=2)
            if p + '.in_conv.weight' in W:
                x = F.conv2d(x, W[p + '.in_conv.weight'], W[p + '.in_conv.bias'], padding=pad)
            h = F.conv2d(x, W[p + '.block1.weight'], W[p + '.block1.bias'], padding=1)
            h = F.relu(h)
            h = F.conv2d(h, W[p + '.block2.weight'], W[p + '.block2.bias'], padding=pad)
            if not sk:
                x = h + F.conv2d(x, W[p + '.skep.weight'], W[p + '.skep.bias'], padding=pad)
            else:
                x = h + x
        feats.append(x)
    return feats


def to_video_features(feats, b, t):
    """'(b t) c h w -> b c t h w' (ddpm3d.py:1483)"""
    return [f.reshape(b, t, *f.shape[1:]).permute(0, 2, 1, 3, 4) for f in feats]


def vc_unet_forward(W, cfg: VC.VCConfig, x, t, ctx, features_adapter=None, taps=None):
    """UNetModel.forward with features_adapter (openaimodel3d.py:632-670).  `taps` as in vc_oracle's forward."""
    L = VC.vc_enumerate(cfg)
    emb = VC.vc_timestep_embedding(t, cfg.model_channels)
    emb = F.linear(emb.to(W['time_embed.0.weight'].dtype), W['time_embed.0.weight'], W['time_embed.0.bias'])
    emb = F.linear(F.silu(emb), W['time_embed.2.weight'], W['time_embed.2.bias'])
    hs = []
    h = x
    adapter_idx = 0
    for idx, blk in enumerate(L.input_blocks):
        h = VC._run(W, blk, h, emb, ctx, cfg, taps)
        if (idx + 1) % 3 == 0 and features_adapter is not None:
            h = h + features_adapter[adapter_idx]
            adapter_idx += 1
        hs.append(h)
    if features_adapter is not None:
        assert len(features_adapter) == adapter_idx, 'Mismatch features adapter'
    h = VC._run(W, L.middle, h, emb, ctx, cfg, taps)
    for blk in L.output_blocks:
        h = torch.cat([h, hs.pop()], dim=1)
        h = VC._run(W, blk, h, emb, ctx, cfg, taps)
    h = F.silu(VC._gn(W, 'out.0', h, 1e-5))
    return F.conv3d(h, W['out.2.weight'], W['out.2.bias'], padding=(0, 1, 1))


def vc_ddim_sample(W, cfg, betas, x_T, S, cond, uncond, scale, eta, noise_gen, features_adapter):
    return VC.vc_ddim_sample(lambda a, b, d: vc_unet_forward(W, cfg, a, b, d, features_adapter), betas, x_T, S, cond, uncond,
                             scale, eta=eta, noise_gen=noise_gen)


class StubDepth(torch.nn.Module):
    """A fixed, smooth stand-in for the MiDaS depth model: [N, 3, 384, 384] -> [N, 1, 192, 192]."""

    def forward(self, x):
        y = F.avg_pool2d(x, 2)
        return (0.5 * y[:, 0:1] - 0.25 * y[:, 1:2] + 0.75 * y[:, 2:3]) ** 2 + 0.1 * y[:, 0:1]


def get_batch_depth(depth_model, batch_x, target_size, encode_bs=1):
    """ddpm3d.py:1448-1468"""
    b, c, t, h, w = batch_x.shape
    merge_x = batch_x.permute(0, 2, 1, 3, 4).reshape(b * t, c, h, w)
    out = []
    for x in torch.split(merge_x, encode_bs, dim=0):
        d = depth_model(F.interpolate(x, size=(384, 384), mode='bicubic'))
        d = F.interpolate(d, size=target_size, mode='bicubic', align_corners=False)
        lo, hi = torch.amin(d, dim=[1, 2, 3], keepdim=True), torch.amax(d, dim=[1, 2, 3], keepdim=True)
        out.append(2. * (d - lo) / (hi - lo + 1e-7) - 1.)
    d = torch.cat(out, 0)
    return d.reshape(b, t, *d.shape[1:]).permute(0, 2, 1, 3, 4)
