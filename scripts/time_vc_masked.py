"""Times VideoCrafter's masked DDIM (continuation from known frames) against unmasked sampling at the full base_t2v UNet
(model_channels 320, context 768) with seeded weights: 16 frames x 256^2 (latent [1, 4, 16, 32, 32]), CFG 15 (cond + uncond as
one B = 2 forward), 50 DDIM steps, eta 1.0; the masked clip keeps its first 4 frames known.

  * per-clip wall clock of `DDIMSampler.sample`, device synchronised, masked and unmasked alternated over --rounds rounds;
  * the blend (t2v_q_sample_blend at the frame mask), alone and with its per-step torch.randn_like(x0), over --iters calls:
    per call as the sampler makes it (CUDA events around back-to-back calls, which the Python wrapper's host time bounds),
    and the device time alone (the calls captured in CUDA graphs and replayed); bytes per blend are counted from the shapes.

The card name and power limit are printed with the numbers.

    python scripts/time_vc_masked.py [--rounds 3] [--iters 1000]
"""
import argparse
import json
import os
import statistics
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, 'sd-webui-text2video_b200'), os.path.join(ROOT, 'scripts')):
    sys.path.insert(0, p)
from time_adapter import card, per_call_ms                    # noqa: E402

SHAPE = (1, 4, 16, 32, 32)


def graph_us(fn, iters, per_graph=100):
    """Device microseconds per call of fn: per_graph calls captured in one CUDA graph, replayed iters / per_graph times
    between CUDA events."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(per_graph):
            fn()
    g.replay()
    torch.cuda.synchronize()
    replays = max(1, iters // per_graph)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(replays):
        g.replay()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) * 1e3 / (replays * per_graph)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--iters', type=int, default=1000)
    args = ap.parse_args()
    from t2v_b200 import ops
    from t2v_b200.synthetic import randomize_
    from t2v_b200.videocrafter import LatentDiffusion, DDIMSampler
    m = LatentDiffusion(image_size=[32, 32], video_length=16).half()
    randomize_(m.model.diffusion_model, seed=0)
    m = m.cuda().eval()
    g = torch.Generator('cpu').manual_seed(0)
    c, uc = torch.randn(1, 77, 768, generator=g).cuda(), torch.randn(1, 77, 768, generator=g).cuda()
    x_T, x0 = torch.randn(SHAPE, generator=g).cuda(), torch.randn(SHAPE, generator=g).cuda()
    mask = torch.zeros(1, 1, 16, 1, 1)
    mask[:, :, :4] = 1.0
    smp = DDIMSampler(m)

    def clip(masked):
        kw = dict(mask=mask, x0=x0) if masked else {}
        smp.noise_gen.manual_seed(0)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out, _ = smp.sample(S=50, batch_size=1, shape=SHAPE[1:], conditioning=c, unconditional_conditioning=uc,
                            unconditional_guidance_scale=15.0, eta=1.0, x_T=x_T, verbose=False, **kw)
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3, out

    res = {'card': card(), 'shape': list(SHAPE), 'steps': 50, 'cfg': 15.0, 'eta': 1.0, 'known_frames': 4}
    clip(False)
    clip(True)                                               # warm-up: plans of both paths built
    times = {'unmasked': [], 'masked': []}
    for _ in range(args.rounds):
        for name in ('unmasked', 'masked'):
            ms, out = clip(name == 'masked')
            times[name].append(ms)
            assert torch.isfinite(out).all()
    for name, v in times.items():
        res[name + '_clip_ms'] = [round(x, 1) for x in v]
        res[name + '_clip_median_ms'] = round(statistics.median(v), 1)
    res['masked_overhead_ms_per_clip'] = round(res['masked_clip_median_ms'] - res['unmasked_clip_median_ms'], 1)

    img = torch.randn(SHAPE, device='cuda')
    noise = torch.randn_like(x0)
    md = mask.cuda()
    a, s = m.sqrt_alphas_cumprod.float()[:1], m.sqrt_one_minus_alphas_cumprod.float()[:1]
    blend = lambda: ops.q_sample_blend(x0, noise, a, s, mask=md, img=img, out=img)       # noqa: E731
    step_extra = lambda: ops.q_sample_blend(x0, torch.randn_like(x0), a, s, mask=md, img=img, out=img)   # noqa: E731
    n = x0.numel()
    # as the sampler calls them (Python wrapper + launch per call: host-bound), then the device time alone (CUDA-graph replay)
    res['blend_call_us'] = round(per_call_ms(blend, args.iters, warmup=20) * 1e3, 2)
    res['randn_plus_blend_call_us'] = round(per_call_ms(step_extra, args.iters, warmup=20) * 1e3, 2)
    res['blend_kernel_us'] = round(graph_us(blend, args.iters), 2)
    res['randn_plus_blend_kernel_us'] = round(graph_us(step_extra, args.iters), 2)
    res['blend_bytes'] = 4 * (4 * n + 16)                    # x0, noise, img read; out written; the 16-entry mask
    res['blend_GB_per_s'] = round(res['blend_bytes'] / (res['blend_kernel_us'] * 1e-6) / 1e9, 1)
    res['iters'] = args.iters
    print(json.dumps(res))


if __name__ == '__main__':
    main()
