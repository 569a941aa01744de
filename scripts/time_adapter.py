"""Times VideoCrafter's depth adapter on the library, with seeded weights at the full-width depth config
(channels 320/640/1280/1280, nums_rb 2, ksize 1, sk, average pooling):

  * `Adapter` encode of a 16-frame clip at 256^2 and 512^2 (graph replay; one call per clip);
  * the VideoCrafter UNet (base_t2v config) B = 2 forward at 16 frames x 256^2 (32x32 latent) without and with adapter
    features, alternated in one run, so the cost of the feature staging copies and the four in-place adds shows directly.

CUDA events around --iters back-to-back calls after a warm-up; the card name and power limit are printed with the numbers.

    python scripts/time_adapter.py [--iters 20] [--rounds 3]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, 'sd-webui-text2video_b200'), os.path.join(ROOT, 'tests')):
    sys.path.insert(0, p)
from oracle import unet_oracle as UO, vc_oracle as VC         # noqa: E402
import adapter_oracle as AO                                   # noqa: E402


def card():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:                                    # noqa: BLE001
        return f'nvidia-smi unavailable: {e}'


def per_call_ms(fn, iters, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--rounds', type=int, default=3)
    args = ap.parse_args()
    from t2v_b200.adapter import Adapter
    from t2v_b200.modules import UNetModel
    res = {'card': card()}
    ad = Adapter(**AO.DEPTH).half()
    ad.load_state_dict(UO.make_weights(AO.adapter_param_specs(**AO.DEPTH), seed=23), strict=True)
    ad = ad.cuda()
    g = torch.Generator('cpu').manual_seed(0)
    for S in (256, 512):
        x = (torch.rand(16, 1, S, S, generator=g) * 2 - 1).cuda()
        res[f'adapter_16f_{S}_ms'] = round(per_call_ms(lambda: ad(x), args.iters), 3)
    net = UNetModel().half()
    net.load_state_dict(UO.make_weights(VC.vc_param_specs(VC.VCConfig()), seed=0), strict=True)
    net = net.cuda().eval()
    x = torch.randn(2, 4, 16, 32, 32, generator=g).cuda()
    t = torch.tensor([981, 981]).cuda()
    ctx = torch.randn(2, 77, 768, generator=g).half().cuda()
    feats = ad((torch.rand(16, 1, 256, 256, generator=g) * 2 - 1).cuda())
    feats = [f.permute(0, 2, 3, 1).reshape(1, 16, *f.shape[2:], f.shape[1]).permute(0, 4, 1, 2, 3) for f in feats]
    plain, adapted = [], []
    for _ in range(args.rounds):
        plain.append(per_call_ms(lambda: net(x, t, context=ctx), args.iters))
        adapted.append(per_call_ms(lambda: net(x, t, context=ctx, features_adapter=feats, features_adapter_tiled=True), args.iters))
    res['unet_b2_16f_256_ms'] = [round(v, 3) for v in plain]
    res['unet_b2_16f_256_features_ms'] = [round(v, 3) for v in adapted]
    res['feature_overhead_ms'] = round(min(adapted) - min(plain), 3)
    res['feature_staging_MB'] = round(sum(f.numel() for f in feats) * 2 / 1e6, 2)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
