"""Times VideoCrafter's DDIM with and without an `img_callback` at the full base_t2v UNet (model_channels 320, context 768) with
seeded weights: 16 frames x 256^2 (latent [1, 4, 16, 32, 32]), CFG 15 (cond + uncond as one B = 2 forward), 50 DDIM steps,
eta 1.0.

  * per-step wall clock of `DDIMSampler.sample` (a 50-step clip, device synchronised, divided by 50), without callbacks and with
    an `img_callback` that keeps every x0, the two alternated over --rounds rounds;
  * the step kernel alone (t2v_ddim_step_ex, variant 0) without and with the x0 store, as CUDA-graph replays; the x0 store
    adds 4 bytes per latent element, counted from the shape.

The card name and power limit are printed with the numbers.

    python scripts/time_vc_ddim_outputs.py [--rounds 3] [--iters 2000]
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
from time_adapter import card                                 # noqa: E402
from time_vc_masked import graph_us                           # noqa: E402

SHAPE = (1, 4, 16, 32, 32)
STEPS = 50


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--iters', type=int, default=2000)
    args = ap.parse_args()
    from t2v_b200 import samplers as S
    from t2v_b200.synthetic import randomize_
    from t2v_b200.videocrafter import LatentDiffusion, DDIMSampler
    m = LatentDiffusion(image_size=[32, 32], video_length=16).half()
    randomize_(m.model.diffusion_model, seed=0)
    m = m.cuda().eval()
    g = torch.Generator('cpu').manual_seed(0)
    c, uc = torch.randn(1, 77, 768, generator=g).cuda(), torch.randn(1, 77, 768, generator=g).cuda()
    x_T = torch.randn(SHAPE, generator=g).cuda()
    smp = DDIMSampler(m)

    def clip(with_callback):
        kept = []
        kw = dict(img_callback=lambda x0, i: kept.append(x0)) if with_callback else {}
        smp.noise_gen.manual_seed(0)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out, _ = smp.sample(S=STEPS, batch_size=1, shape=SHAPE[1:], conditioning=c, unconditional_conditioning=uc,
                            unconditional_guidance_scale=15.0, eta=1.0, x_T=x_T, verbose=False, **kw)
        torch.cuda.synchronize()
        assert len(kept) == (STEPS if with_callback else 0)
        return (time.perf_counter() - t0) * 1e3 / STEPS, out

    res = {'card': card(), 'shape': list(SHAPE), 'steps': STEPS, 'cfg': 15.0, 'eta': 1.0}
    _, plain = clip(False)
    _, with_cb = clip(True)                                  # warm-up; the callback must not change the latent
    res['same_latent_with_img_callback'] = bool(torch.equal(plain, with_cb))
    times = {'no_callback': [], 'img_callback': []}
    for _ in range(args.rounds):
        for name in times:
            ms, out = clip(name == 'img_callback')
            times[name].append(ms)
            assert torch.isfinite(out).all()
    for name, v in times.items():
        res[name + '_step_ms'] = [round(x, 3) for x in v]
        res[name + '_step_median_ms'] = round(statistics.median(v), 3)
    res['img_callback_overhead_ms_per_step'] = round(res['img_callback_step_median_ms'] - res['no_callback_step_median_ms'], 3)

    x = torch.randn(SHAPE, device='cuda')
    ec, eu = torch.randn(SHAPE, device='cuda').half(), torch.randn(SHAPE, device='cuda').half()
    noise = torch.randn(SHAPE, device='cuda')
    a = (0.9, 0.4, 0.95, 0.3, 0.1)
    for name, want in (('step_kernel_us', False), ('step_kernel_with_x0_us', True)):
        res[name] = round(graph_us(lambda: S._step_kernel_ex(x, ec, eu, 15.0, 4, 1, a, noise, False, 0, want), args.iters), 2)
    n = x.numel()
    res['step_bytes'] = n * (4 + 2 + 2 + 4 + 4)              # x, eps_c, eps_u (fp16), noise read; x_out written
    res['x0_store_bytes'] = 4 * n
    res['iters'] = args.iters
    print(json.dumps(res))


if __name__ == '__main__':
    main()
