"""Times VideoCrafter LoRA on the library at the full base_t2v UNet (model_channels 320, context 768, 16 frames), seeded weights:
a rank-4 LoRA on every attention projection (to_q / to_k / to_v / to_out.0 of attn1, attn2, attn1_tmp and attn2_tmp in all 16
transformer blocks: 256 weights), keyed from the LatentDiffusion root as a VideoCrafter LoRA file is.

  * `net_load_lora_v2` merge of the LoRA (device-side merge + in-place re-pack, plans kept);
  * a `change_lora_v2` switch to a second LoRA (exact restore + merge), alternated back and forth;
  * the alternative without a device-side merge: the merged weights computed with torch, re-shipped through the parameters,
    and the plan rebuilt by the next forward (first forward: build + eager run; second: graph capture);
  * the B = 2, 16 x 256^2 forward before and after the switches (the same plan keeps running).

Wall clock around each operation with the device synchronised (they are host + device work); the card name and power limit are
printed with the numbers.

    python scripts/time_vc_lora.py [--rounds 5]
"""
import argparse
import json
import os
import statistics
import sys
import time

import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, 'sd-webui-text2video_b200'), os.path.join(ROOT, 'scripts')):
    sys.path.insert(0, p)
from time_adapter import card, per_call_ms                    # noqa: E402

PROJ = ('attn1.to_q', 'attn1.to_k', 'attn1.to_v', 'attn1.to_out.0', 'attn2.to_q', 'attn2.to_k', 'attn2.to_v', 'attn2.to_out.0',
        'attn1_tmp.to_q', 'attn1_tmp.to_k', 'attn1_tmp.to_v', 'attn1_tmp.to_out.0',
        'attn2_tmp.to_q', 'attn2_tmp.to_k', 'attn2_tmp.to_v', 'attn2_tmp.to_out.0')


def make_lora(net, seed, rank=4):
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for path, mod in net.named_modules():
        if type(mod) is nn.Linear and path.endswith(PROJ):
            key = 'model.diffusion_model.' + path
            sd[key + '.lora_up.weight'] = torch.randn((mod.weight.shape[0], rank), generator=g) * 0.02
            sd[key + '.lora_down.weight'] = torch.randn((rank, mod.weight.shape[1]), generator=g) * 0.02
    return sd


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=5)
    args = ap.parse_args()
    from t2v_b200.modules import UNetModel
    from t2v_b200.synthetic import randomize_
    from t2v_b200 import videocrafter as vcm
    root = nn.Module()
    root.model = vcm._DiffusionWrapper(randomize_(UNetModel().half().cuda().eval(), seed=0))
    net = root.model.diffusion_model
    lora1, lora2 = make_lora(net, 1), make_lora(net, 2)
    res = {'card': card(), 'lora_weights': len(lora1) // 2, 'rank': 4}
    g = torch.Generator('cpu').manual_seed(0)
    x = torch.randn(2, 4, 16, 32, 32, generator=g).cuda()
    t = torch.tensor([981, 981]).cuda()
    ctx = torch.randn(2, 77, 768, generator=g).half().cuda()
    fwd = lambda: net(x, t, context=ctx)                      # noqa: E731
    res['forward_b2_16f_256_ms_before'] = round(per_call_ms(fwd, 10), 3)
    state = {}
    res['merge_ms'] = round(timed(lambda: state.update(o=vcm.net_load_lora_v2(root, lora1, alpha=1.0))), 2)
    switches, cur = [], (lora1, lora2)
    for _ in range(args.rounds):
        switches.append(timed(lambda: state.update(o=vcm.change_lora_v2(root, True, 1.0, cur[1], cur[0], 1.0, state['o']))))
        cur = cur[::-1]
    res['change_lora_v2_switch_ms'] = [round(v, 2) for v in switches]
    res['forward_b2_16f_256_ms_after'] = round(per_call_ms(fwd, 10), 3)
    net.lora_clear()
    # the alternative: merge with torch, re-ship the touched weights, rebuild the plan at the next forward
    params = {k[len('model.diffusion_model.'):-len('.lora_up.weight')] + '.weight': k for k in lora2 if k.endswith('lora_up.weight')}
    ship, first, second = [], [], []
    for r in range(args.rounds):
        lo = (lora1, lora2)[r % 2]

        def reship():
            for name, up_key in params.items():
                p = net.get_parameter(name)
                up, down = lo[up_key].cuda(), lo[up_key.replace('lora_up', 'lora_down')].cuda()
                p.data = (p.data.float() + up @ down).half()
            net.sync_weights(force=True)
        ship.append(timed(reship))
        first.append(timed(fwd))
        second.append(timed(fwd))
    res['reship_ms'] = [round(v, 2) for v in ship]
    res['reship_first_forward_ms'] = [round(v, 2) for v in first]
    res['reship_second_forward_ms'] = [round(v, 2) for v in second]
    res['reship_total_median_ms'] = round(statistics.median(a + b + c - 2 * res['forward_b2_16f_256_ms_after']
                                                            for a, b, c in zip(ship, first, second)), 2)
    res['switch_median_ms'] = round(statistics.median(switches), 2)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
