"""Cost of DDIM_Gaussian's x0 range restriction on one GPU.

Per step, at latents [1, 4, F, H/8, W/8] for 24 f x 256^2, 125 f x 256^2, 24 f x 576x1024 and 250 f x 1024^2 (16.4 M elements):
the unrestricted step (t2v_ddim_step), the thresholded step with percentile 0.995 (x0, radix-select quantile, step), the
clamped step, and the quantile alone (t2v_abs_quantile), each captured in a CUDA graph of `reps` calls and timed with CUDA events
over graph replays; the variants alternate within each round and the best round is kept.  Then one full-size 50-step clip
(UNetSD and VAE with seeded weights, 24 f x 256^2, CFG 9, decode included) with and without percentile=0.995, alternated.
The card name, power limit and SM clocks are printed with the numbers; one JSON line per measurement.

    python scripts/time_ddim_threshold.py [--reps 50] [--rounds 5] [--clip-rounds 2]
"""
import argparse
import functools
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, 'sd-webui-text2video_b200'), os.path.join(ROOT, 'scripts')):
    sys.path.insert(0, p)
from time_batch_clips import card, emit                       # noqa: E402

SHAPES = [(24, 256, 256), (125, 256, 256), (24, 576, 1024), (250, 1024, 1024)]
COEFS = (14.2, 14.16, 0.31, 0.95, 0.0)


def step_variants(l, L, F, H, W):
    dev = torch.device('cuda')
    shape = (1, 4, F, H // 8, W // 8)
    g = torch.Generator(device=dev).manual_seed(0)
    x = torch.randn(shape, device=dev, generator=g) * 2
    ec = torch.randn(shape, device=dev, generator=g).half()
    eu = torch.randn(shape, device=dev, generator=g).half()
    out, s, q = torch.empty_like(x), torch.empty(1, device=dev), torch.empty(1, device=dev)
    ws = torch.empty(l.t2v_abs_quantile_workspace(1), dtype=torch.uint8, device=dev)
    n, cs = x.numel(), x[0, 0].numel()
    stream = L.stream_ptr

    def plain():
        L.check(l.t2v_ddim_step(L.ptr(x), L.ptr(ec), L.ptr(eu), 0, L.ptr(out), n, cs, 4, 2, 9.0, 0, *COEFS, None, 1, stream()), 's')

    def restricted(pct):
        L.check(l.t2v_ddim_step_threshold(L.ptr(x), L.ptr(ec), L.ptr(eu), 0, L.ptr(out), n, cs, 4, 2, 9.0, *COEFS, None, 1, 1, pct,
                                          L.ptr(s), L.ptr(ws), ws.numel(), stream()), 't')

    def quantile():
        L.check(l.t2v_abs_quantile(L.ptr(x), 1, n, 0.995, L.ptr(q), L.ptr(ws), ws.numel(), stream()), 'q')
    return n, {'ddim_step': plain, 'threshold_step_p0.995': functools.partial(restricted, 0.995),
               'clamp_step': functools.partial(restricted, 0.0), 'abs_quantile': quantile}


def graph_of(fn, reps):
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        fn()                                                  # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for _ in range(reps):
            fn()
    return graph


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=50, help='calls per captured graph')
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--clip-rounds', type=int, default=2)
    ap.add_argument('--no-clip', action='store_true')
    args = ap.parse_args()
    from t2v_b200 import _lib as L
    l = L.lib()
    emit(card=card())
    for F, H, W in SHAPES:
        n, fns = step_variants(l, L, F, H, W)
        graphs = {k: graph_of(f, args.reps) for k, f in fns.items()}
        best = {k: float('inf') for k in graphs}
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for _ in range(args.rounds):
            for k, gr in graphs.items():
                gr.replay()                                   # untimed replay: caches and clocks settle per variant
                a.record()
                gr.replay()
                b.record()
                b.synchronize()
                best[k] = min(best[k], a.elapsed_time(b) * 1e3 / args.reps)
        emit(what=f'per step, latent 1x4x{F}x{H // 8}x{W // 8} ({F} f x {H}x{W})', elements=n,
             us={k: round(v, 2) for k, v in best.items()},
             threshold_over_step_us=round(best['threshold_step_p0.995'] - best['ddim_step'], 2),
             quantile_GB_per_s_one_read=round(4 * n / (best['abs_quantile'] * 1e-6) / 1e9, 1), card=card())
        del graphs
        torch.cuda.empty_cache()
    if args.no_clip:
        return

    from t2v_b200.pipeline import TextToVideoSynthesis
    from t2v_b200.synthetic import randomize_
    from t2v_b200 import samplers as S
    dev = torch.device('cuda', 0)
    pipe = TextToVideoSynthesis(None, device=dev)
    randomize_(pipe.sd_model, seed=0)
    randomize_(pipe.autoencoder, seed=3)
    g = torch.Generator().manual_seed(2)
    c, uc = torch.randn(1, 77, 1024, generator=g).half(), torch.randn(1, 77, 1024, generator=g).half()
    plain_sample = S.GaussianDiffusion.sample

    def clip(pct):
        S.GaussianDiffusion.sample = plain_sample if pct is None else functools.partialmethod(plain_sample, percentile=pct)
        try:
            t0 = time.perf_counter()
            pipe.infer(c, uc, 50, 24, 1, 9.0, 256, 256, 0.0, 'GPU (half precision)', dev, None, 0, 0.0, None, False,
                       'DDIM_Gaussian')
            torch.cuda.synchronize()
            return time.perf_counter() - t0
        finally:
            S.GaussianDiffusion.sample = plain_sample
    clip(None)
    clip(0.995)                                               # warm-up: plans, graphs
    times = {'none': [], 'percentile 0.995': []}
    for _ in range(args.clip_rounds):
        times['none'].append(clip(None))
        times['percentile 0.995'].append(clip(0.995))
    emit(what='one clip of 24 f x 256x256, 50 DDIM_Gaussian steps + decode', seconds={k: [round(v, 3) for v in t]
                                                                                        for k, t in times.items()},
         percentile_cost_ms=round((min(times['percentile 0.995']) - min(times['none'])) * 1e3, 1), card=card())


if __name__ == '__main__':
    main()
