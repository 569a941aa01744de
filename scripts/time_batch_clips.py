"""Batched ModelScope clips (`TextToVideoSynthesis.infer(batch_size=n)`) against one clip at a time, full-size UNetSD and VAE with
seeded weights, one GPU.  For each n: frames/s of n clips (`steps` DDIM_Gaussian steps, CFG, then the VAE decode of all n * F
frames), the B = 2n forward time per clip (CUDA events around `reps` forwards of the shared-context batch), the denoiser plan's
arena and the VAE decode plan's bytes (dry passes) and the peak device memory in use (cudaMemGetInfo, total - free, polled
while the clips run: device-wide, so it includes the caching allocator's pool and any other process on the card).  Every
shape is warmed up (plan build, graph capture) by one untimed call first.  The card name, power limit, max and current SM
clock and active clock-throttle reasons are read right after each n's last timed call and printed with its numbers; one JSON
line per measurement.

    python scripts/time_batch_clips.py [--size 256x256] [--frames 24] [--steps 50] [--ns 1,2,4,8] [--rounds 2]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, 'sd-webui-text2video_b200'), os.path.join(ROOT, 'scripts')):
    sys.path.insert(0, p)
from time_vae_chunked import PeakInUse                        # noqa: E402


def card():
    q = 'name,power.limit,clocks.max.sm,clocks.sm,clocks_throttle_reasons.active'
    try:
        return subprocess.run(['nvidia-smi', f'--query-gpu={q}', '--format=csv,noheader'], capture_output=True, text=True,
                              timeout=30).stdout.strip()
    except Exception as e:                                    # noqa: BLE001
        return f'nvidia-smi unavailable: {e}'


def emit(**kv):
    print(json.dumps(kv), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--size', default='256x256', help='HxW in pixels')
    ap.add_argument('--frames', type=int, default=24)
    ap.add_argument('--steps', type=int, default=50)
    ap.add_argument('--ns', default='1,2,4,8')
    ap.add_argument('--rounds', type=int, default=2, help='timed calls per n, alternated over the n values')
    ap.add_argument('--reps', type=int, default=10, help='forwards per forward timing')
    args = ap.parse_args()
    H, W = map(int, args.size.split('x'))
    F, ns = args.frames, [int(v) for v in args.ns.split(',')]
    from t2v_b200.pipeline import TextToVideoSynthesis
    from t2v_b200.synthetic import randomize_
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    emit(card=card())
    pipe = TextToVideoSynthesis(None, device=dev)
    randomize_(pipe.sd_model, seed=0)
    randomize_(pipe.autoencoder, seed=3)
    net = pipe.sd_model
    g = torch.Generator().manual_seed(2)
    c, uc = torch.randn(1, 77, 1024, generator=g).half(), torch.randn(1, 77, 1024, generator=g).half()

    def clips(n):
        return pipe.infer(c, uc, args.steps, F, 1, 9.0, W, H, 0.0, 'GPU (half precision)', dev, None, 0, 0.0, None, False,
                          'DDIM_Gaussian', batch_size=n)

    def forward_ms(n):
        x = torch.randn((n, 4, F, H // 8, W // 8), device=dev)
        xb = torch.cat([x, x]) if n > 1 else x.expand(2, -1, -1, -1, -1)
        t = torch.full((2 * n,), 501.0, device=dev)
        y = torch.cat([c, uc]).to(dev)
        net(xb, t, y)
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(args.reps):
            net(xb, t, y)
        b.record()
        b.synchronize()
        return a.elapsed_time(b) / args.reps

    for n in ns:
        clips(n)                                              # warm-up: plan builds, graph capture
        torch.cuda.synchronize()
    times = {n: [] for n in ns}
    peaks = {n: 0 for n in ns}
    groups, cards = {}, {}
    for _ in range(args.rounds):
        for n in ns:
            with PeakInUse() as m:
                t0 = time.perf_counter()
                clips(n)
                torch.cuda.synchronize()
                times[n].append(time.perf_counter() - t0)
            peaks[n] = max(peaks[n], m.peak)
            groups[n] = pipe.last_batch_groups if n > 1 else [1]
            cards[n] = card()
    base = None
    for n in ns:
        s = min(times[n])
        fps = n * F / s
        base = fps if base is None else base
        fwd = forward_ms(n)
        arena = net.plan_info(2 * n, F, H // 8, W // 8, 77, ctx_batch=2)[0]
        vae = pipe.autoencoder.plan_bytes(n * F, H // 8, W // 8)
        emit(what=f'{n} clip(s) of {F}f {H}x{W}, {args.steps} DDIM_Gaussian steps + decode', n=n, groups=groups[n],
             seconds=[round(v, 3) for v in times[n]], frames_per_s=round(fps, 3), vs_n1=round(fps / base, 3),
             forward_ms=round(fwd, 2), forward_ms_per_clip=round(fwd / n, 2), unet_arena_GB=round(arena / 1e9, 2),
             vae_decode_plan_GB=round(vae / 1e9, 2), device_peak_in_use_GB=round(peaks[n] / 1e9, 2), card=cards[n])


if __name__ == '__main__':
    main()
