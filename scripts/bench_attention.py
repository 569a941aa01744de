"""Times spatial self-attention on the fused [tokens, 3C] matrix: wgmma kernel vs the warp-MMA kernel.
usage: python scripts/bench_attention.py            (prints one line per shape)"""
import os
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(__file__), '..', 'sd-webui-text2video_b200'))
from t2v_b200 import ops  # noqa: E402

dev = 'cuda'
SHAPES = [(48, 5, 1024), (48, 10, 256), (48, 5, 9216), (48, 10, 2304), (48, 20, 576)]


def run(batch, heads, S, iters=10):
    C = heads * 64
    torch.manual_seed(0)
    qkv = torch.randn(batch * S, 3 * C, device=dev).half()
    o = torch.zeros(batch * S, C, device=dev, dtype=torch.half)
    ld = 3 * C

    def call():
        ops.attention(qkv, qkv[:, C:], qkv[:, 2 * C:], o, S * ld, ld, S * ld, ld, S * ld, ld, S * C, C, batch, heads, S, S)
    for _ in range(3):
        call()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        call()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / iters
    fl = 4.0 * batch * heads * S * S * 64
    return ms, fl / ms / 1e9, o.clone()


for shp in SHAPES:
    os.environ.pop('T2V_ATTN_WARP_MMA', None)
    ms_tc, tf_tc, o_tc = run(*shp)
    os.environ['T2V_ATTN_WARP_MMA'] = '1'
    ms_w, tf_w, o_w = run(*shp)
    os.environ.pop('T2V_ATTN_WARP_MMA', None)
    d = (o_tc.float() - o_w.float()).abs().max().item()
    print(f'batch {shp[0]} heads {shp[1]} S {shp[2]}: wgmma {ms_tc:.3f} ms {tf_tc:.0f} TF/s | warp-mma {ms_w:.3f} ms {tf_w:.0f} TF/s '
          f'| max|diff| {d:.2e}', flush=True)
