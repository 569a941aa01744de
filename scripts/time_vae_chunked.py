"""Frame-chunked VAE at ZeroScope XL size (576 x 1024, latent 72 x 128) with the ModelScope VAE and seeded weights, one GPU:

  * the whole-clip plan bytes of a 96-frame decode and encode (AutoencoderKL.plan_bytes: shows, without trying, that
    the clip does not fit as one plan), the split the library chose (last_chunking), the device memory in use
    (cudaMemGetInfo: total - free, polled every 2 ms while the call runs; its peak), and ms per frame of the chunked
    96-frame call against the whole-clip call at 24 frames (host clock around device-synchronised calls, after a warm-up
    call at each shape);
  * one end-to-end 96-frame clip with 2 DDIM_Gaussian steps through TextToVideoSynthesis.infer with the ModelScope /
    ZeroScope UNet (seeded weights): its peak memory in use and the UNet arena (UNetSD.plan_bytes, B = 1 and 2).

The card name, power limit and clocks are printed with the numbers; one JSON line per measurement.

    python scripts/time_vae_chunked.py [--frames 96] [--reps 2]
"""
import argparse
import json
import os
import sys
import threading
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, 'sd-webui-text2video_b200'), os.path.join(ROOT, 'scripts')):
    sys.path.insert(0, p)
from time_adapter import card                                 # noqa: E402

GB = 1e9
H, W = 576, 1024
h, w = H // 8, W // 8


class PeakInUse(object):
    """Peak of total - free device memory (cudaMemGetInfo) while the block runs, polled from a thread."""

    def __enter__(self):
        self.peak, self._stop = 0, False
        self._t = threading.Thread(target=self._poll, daemon=True)
        self._t.start()
        return self

    def _poll(self):
        while not self._stop:
            free, total = torch.cuda.mem_get_info()
            self.peak = max(self.peak, total - free)
            time.sleep(0.002)

    def __exit__(self, *a):
        torch.cuda.synchronize()
        self._stop = True
        self._t.join()
        free, total = torch.cuda.mem_get_info()
        self.peak = max(self.peak, total - free)


def timed(fn, reps):
    fn()                                                      # warm-up: plan build, graph capture
    torch.cuda.synchronize()
    with PeakInUse() as m:
        t0 = time.perf_counter()
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
        ms = (time.perf_counter() - t0) * 1e3 / reps
    return ms, m.peak


def emit(**kv):
    print(json.dumps(kv), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=96)
    ap.add_argument('--reps', type=int, default=2)
    ap.add_argument('--steps', type=int, default=2)
    args = ap.parse_args()
    from t2v_b200.pipeline import TextToVideoSynthesis
    from t2v_b200.synthetic import randomize_
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    emit(card=card())
    pipe = TextToVideoSynthesis(None, device=dev)
    randomize_(pipe.sd_model, seed=0)
    randomize_(pipe.autoencoder, seed=3)
    ae, unet = pipe.autoencoder, pipe.sd_model
    F = args.frames
    emit(what='plan bytes', decode_whole_GB=ae.plan_bytes(F, h, w) / GB, decode_24_GB=ae.plan_bytes(24, h, w) / GB,
         decode_1_GB=ae.plan_bytes(1, h, w) / GB, encode_whole_GB=ae.plan_bytes(F, H, W, encode=True) / GB,
         encode_24_GB=ae.plan_bytes(24, H, W, encode=True) / GB, unet_B1_GB=unet.plan_bytes(1, F, h, w) / GB,
         unet_B2_GB=unet.plan_bytes(2, F, h, w) / GB, total_GB=torch.cuda.mem_get_info()[1] / GB)

    # end to end first, as a user would run it: the UNet's plan is built before the VAE's
    g = torch.Generator().manual_seed(2)
    c, uc = torch.randn(1, 77, 1024, generator=g).half(), torch.randn(1, 77, 1024, generator=g).half()
    torch.cuda.synchronize()
    with PeakInUse() as m:
        t0 = time.perf_counter()
        frames, _, _ = pipe.infer(c, uc, args.steps, F, 1, 17.0, W, H, 0.0, 'GPU (half precision)', dev, None, 0, 0.0, None, False,
                                  'DDIM_Gaussian')
        s = time.perf_counter() - t0
    emit(what=f'infer {F}f {H}x{W} {args.steps} steps (first call: plan builds included)', seconds=s, peak_in_use_GB=m.peak / GB,
         frames=len(frames), vae_split=ae.last_chunking(), card=card())

    z = {n: torch.randn((1, 4, n, h, w), generator=torch.Generator().manual_seed(n)).cuda() for n in (24, F)}
    x = {n: (torch.rand((n, 3, H, W), generator=torch.Generator().manual_seed(n)) * 2 - 1).half().cuda() for n in (24, F)}
    for n in (24, F):
        ms, peak = timed(lambda: ae.decode_video(z[n], as_uint8=True), args.reps)
        emit(what=f'decode {n}f', ms=ms, ms_per_frame=ms / n, split=ae.last_chunking(), peak_in_use_GB=peak / GB, card=card())
    for n in (24, F):
        ms, peak = timed(lambda: ae.encode(x[n]), args.reps)
        emit(what=f'encode {n}f', ms=ms, ms_per_frame=ms / n, split=ae.last_chunking(encode=True), peak_in_use_GB=peak / GB,
             card=card())


if __name__ == '__main__':
    main()
