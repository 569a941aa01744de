"""Shared helpers of the GPU parity tests (test infrastructure; imports the oracle as the checker only)."""
import json
import os

import torch

from oracle import unet_oracle as UO

REPORT = os.environ.get('T2V_PARITY_REPORT')        # optional: append one JSON line per measured comparison


def errs(a, b):
    """(max|a-b| / max|b|, relative RMS) in fp32 on the CPU."""
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).abs().max() / (b.abs().max() + 1e-6)).item(), \
           ((a - b).pow(2).mean().sqrt() / (b.pow(2).mean().sqrt() + 1e-9)).item()


def on_fixture_frames(t, g):
    """`t` [B, C, F, h, w] restricted to the frames a fixture stores (fixtures of large clips keep a fixed subset, `frames`)."""
    return t[:, :, g['frames']] if 'frames' in g else t


def pass_rate(a, b, rtol=1e-3, atol=1e-4):
    """Fraction of elements inside BASELINE.json's element-wise gate |a-b| <= atol + rtol*|b|."""
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).abs() <= atol + rtol * b.abs()).float().mean().item()


def report(name, **kv):
    """Prints (pytest -s / -rP shows it) and optionally records a measured comparison."""
    line = {'case': name, **{k: (round(v, 6) if isinstance(v, float) else v) for k, v in kv.items()}}
    print('[parity] ' + json.dumps(line), flush=True)
    if REPORT:
        with open(REPORT, 'a') as f:
            f.write(json.dumps(line) + '\n')


class AutocastOracle(object):
    """The reference's GPU numerics contract (SURVEY.md appendix B): the SAME torch ops as the reference module tree, fp16
    weights, under torch.autocast('cuda') (t2v_pipeline.py:271: `with amp.autocast(enabled=True)`), attention through
    F.scaled_dot_product_attention (t2v_model.py:566-569, the backend the reference takes without xformers).  It is the honest yardstick for
    "matches the reference PyTorch path": our error against the fp32 fixture is gated against THIS path's error against
    the same fixture."""

    def __init__(self, W, cfg, forward=UO.unet_forward, attn_impl='sdpa'):
        self.W = {k: v.half().cuda() for k, v in W.items()}
        self.cfg, self.fwd, self.attn_impl = cfg, forward, attn_impl

    @torch.no_grad()
    def __call__(self, x, t, y, taps=None):
        old = UO.ATTN_IMPL
        UO.ATTN_IMPL = self.attn_impl
        try:
            with torch.autocast('cuda', dtype=torch.float16):
                kw = {} if taps is None else {'taps': taps}
                return self.fwd(self.W, self.cfg, x.cuda(), torch.as_tensor(t).cuda(), y.cuda(), **kw)
        finally:
            UO.ATTN_IMPL = old


class CallRecorder(object):
    """Wraps a denoiser for the single-step gates: records the latent of every model call and aborts at call `stop_at`
    (the latent handed to the (n+1)-th evaluation is the state after the first update -- exactly how
    oracle/make_golden.py captured the reference's `*_x1` tensors).  Not a UNetSD instance, so the samplers issue the
    reference's own call sequence: cond, uncond, cond, ..."""

    class Stop(Exception):
        pass

    def __init__(self, model, stop_at):
        self._m, self.calls, self.stop_at = model, [], stop_at

    def __getattr__(self, k):
        return getattr(self._m, k)

    def __call__(self, x, t, c):
        self.calls.append(x.detach().clone())
        if len(self.calls) == self.stop_at:
            raise CallRecorder.Stop()
        return self._m(x, t, c)


def first_update(run, model, stop_at):
    rec = CallRecorder(model, stop_at)
    try:
        run(rec)
    except CallRecorder.Stop:
        pass
    return rec.calls[-1]
