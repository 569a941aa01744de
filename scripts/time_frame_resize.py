"""vid2vid / img2vid frame preparation on the device (`t2v_b200.ops.frames_resize`: PIL's LANCZOS resize + x / 255 * 2 - 1, fp16
output as in the half-precision VAE mode) against PIL on one host thread.  For each shape and frame count:
  * kernel: the uint8 frames already on the device, CUDA events around `reps` calls -> ms per frame;
  * with upload: the frames in a host array, copied through the pinned staging chunks inside the call; CUDA events around
    `reps` calls, and the host clock of the same calls (each ends in a device synchronise), -> ms per frame;
  * PIL: Image.fromarray(f).resize((W, H), Image.LANCZOS) of `pil_frames` frames on this thread -> ms per frame.
Every shape is warmed up by one untimed call (coefficient tables, allocator).  The card name, power limit, max and current SM
clock and active clock-throttle reasons are read after the timings and printed with them; one JSON line per measurement.

    python scripts/time_frame_resize.py [--counts 24,250] [--reps 5] [--pil-frames 24]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, 'sd-webui-text2video_b200'), os.path.join(ROOT, 'scripts')):
    sys.path.insert(0, p)
from time_batch_clips import card, emit                       # noqa: E402

SHAPES = [((320, 576), (576, 1024)), ((1080, 1920), (576, 1024)), ((720, 1280), (256, 256))]     # (H0, W0), (H, W)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--counts', default='24,250', help='frames per call')
    ap.add_argument('--reps', type=int, default=5, help='timed calls per measurement')
    ap.add_argument('--pil-frames', type=int, default=24, help='frames resized by PIL per shape')
    args = ap.parse_args()
    from PIL import Image
    from t2v_b200 import ops
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    emit(card=card(), torch_threads=torch.get_num_threads())
    rng = np.random.default_rng(0)

    def events_ms(fn):
        fn()
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0 = time.perf_counter()
        a.record()
        for _ in range(args.reps):
            fn()
        b.record()
        b.synchronize()
        return a.elapsed_time(b) / args.reps, (time.perf_counter() - t0) * 1e3 / args.reps

    for (h0, w0), (h, w) in SHAPES:
        pil_src = rng.integers(0, 256, (args.pil_frames, h0, w0, 3), dtype=np.uint8)
        t0 = time.perf_counter()
        for f in pil_src:
            Image.fromarray(f).resize((w, h), Image.LANCZOS)
        pil_ms = (time.perf_counter() - t0) * 1e3 / args.pil_frames
        for n in [int(v) for v in args.counts.split(',')]:
            host = rng.integers(0, 256, (n, h0, w0, 3), dtype=np.uint8)
            on_dev = torch.from_numpy(host).to(dev)
            out = torch.empty((n, 3, h, w), device=dev, dtype=torch.float16)
            k_ms, _ = events_ms(lambda: ops.frames_resize(on_dev, w, h, torch.float16, out=out))
            u_ms, u_wall = events_ms(lambda: ops.frames_resize(host, w, h, torch.float16, out=out))
            emit(what=f'{n} frames {w0}x{h0} -> {w}x{h}, fp16 out', n=n, kernel_ms_per_frame=round(k_ms / n, 4),
                 with_upload_ms_per_frame=round(u_ms / n, 4), with_upload_host_ms_per_frame=round(u_wall / n, 4),
                 pil_one_thread_ms_per_frame=round(pil_ms, 3), speedup_vs_pil_with_upload=round(pil_ms * n / u_wall, 1),
                 source_MB=round(host.nbytes / 1e6, 1), card=card())
            del on_dev, out
            torch.cuda.empty_cache()


if __name__ == '__main__':
    main()
