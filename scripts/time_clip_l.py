"""Time of FrozenCLIPEmbedder.encode (VideoCrafter's CLIP ViT-L/14 text model on the library, csrc/clip.cu arch 1) for
two 77-token prompts -- the cond / uncond pair a text2video call encodes -- with seeded weights.

    python scripts/time_clip_l.py [--iters 200]

The tokenizer is a stand-in (one id per character; only the token count matters for the time).  Two numbers: the tower
alone (`encode_with_transformer` on pre-tokenised ids, graph replay + fp32 output copy) and the whole `encode` (host
tokenisation, the id upload and the tower).  CUDA events around --iters back-to-back calls after a warm-up.
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
from oracle import unet_oracle as UO                          # noqa: E402
import clip_l_oracle as CL                                    # noqa: E402


def card():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:                                    # noqa: BLE001
        return f'nvidia-smi unavailable: {e}'


def per_call_ms(fn, iters):
    for _ in range(10):
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
    ap.add_argument('--iters', type=int, default=200)
    args = ap.parse_args()
    from t2v_b200.clip import FrozenCLIPEmbedder
    cfg = CL.ClipLConfig()
    e = FrozenCLIPEmbedder(tokenizer=CL.WordTokenizer(cfg.vocab))
    e.transformer.load_state_dict(UO.make_weights(CL.clip_l_param_specs(cfg), seed=4), strict=True)
    e.half().cuda()
    prompts = ['a cat riding a bike through a field of sunflowers at dusk, cinematic lighting', '']
    tokens = e.tokenize(prompts).cuda()
    tower = per_call_ms(lambda: e.encode_with_transformer(tokens), args.iters)
    full = per_call_ms(lambda: e.encode(prompts), args.iters)
    print(json.dumps({'card': card(), 'prompts': 2, 'tokens': 77, 'tower_ms': round(tower, 4), 'encode_ms': round(full, 4),
                      'iters': args.iters}))


if __name__ == '__main__':
    main()
