"""Per-launch time of ops.gemm at the UNet's GEMM shapes for a 24-frame 256x256 clip (latent 32x32, B = 2: the CFG pair).

    python scripts/gemm_epilogue_ab.py [--iters N] [--out FILE]
        times every shape with the library the package loads (T2V_LIB_PATH overrides it)
    python scripts/gemm_epilogue_ab.py --ab A.so B.so [--rounds 3] [--out FILE]
        one process per library, alternating A B A B ..., then the per-shape median of each and B's gain

Times are CUDA events around --iters back-to-back launches after a warm-up.  TFLOP/s uses the algorithmic FLOPs of the
shape (2 * rows * N * K * taps), not what the tile padding computes.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

B, F, H, W = 2, 24, 32, 32
CONV3 = [[dx, dy, 0] for dy in (-1, 0, 1) for dx in (-1, 0, 1)]
TEMP3 = [[0, df, 0] for df in (-1, 0, 1)]           # dims (h*w, F, B)
# (name, family, level rows side, K, N, taps, residual, geglu)
SHAPES = [
    ('L0 proj_in 320->320', 'L0 K=320', 32, 320, 320, None, False, False),
    ('L0 qkv 320->960', 'L0 K=320', 32, 320, 960, None, False, False),
    ('L0 attn out 320->320 +res', 'L0 K=320 +res', 32, 320, 320, None, True, False),
    ('L0 GEGLU 320->2560', 'L0 GEGLU', 32, 320, 2560, None, False, True),
    ('L0 ff out 1280->320 +res', 'L0 K=1280 +res', 32, 1280, 320, None, True, False),
    ('L0 conv3x3 320->320 +res', 'L0 conv3x3 +res', 32, 320, 320, CONV3, True, False),
    ('L0 temporal conv 320 +res', 'L0 temporal +res', 32, 320, 320, TEMP3, True, False),
    ('L1 proj 640->640', 'L1 N=640', 16, 640, 640, None, False, False),
    ('L1 attn out 640->640 +res', 'L1 N=640 +res', 16, 640, 640, None, True, False),
    ('L1 qkv 640->1920', 'L1 N=1920', 16, 640, 1920, None, False, False),
    ('L1 conv3x3 640->640 +res', 'L1 conv3x3 +res', 16, 640, 640, CONV3, True, False),
    ('L2 proj 1280->1280 +res', 'L2 N=1280 +res', 8, 1280, 1280, None, True, False),
    ('L2 conv3x3 1280->1280 +res', 'L2 conv3x3 +res', 8, 1280, 1280, CONV3, True, False),
]


def gpu_info():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                              capture_output=True, text=True, timeout=60).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f'nvidia-smi unavailable: {e}'


def measure(iters):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, 'sd-webui-text2video_b200'))
    import torch
    from t2v_b200 import ops
    if not torch.cuda.is_available():
        raise SystemExit('no CUDA device: nothing to measure')
    torch.manual_seed(0)
    dev = 'cuda'
    res = {}
    for name, fam, side, K, N, taps, has_res, geglu in SHAPES:
        rows = B * F * side * side
        ntaps = len(taps) if taps else 1
        a = torch.randn(rows, K, device=dev).half()
        wp = (torch.randn(ntaps, N, K, device=dev) / (K * ntaps) ** 0.5).half()
        bias = torch.randn(N, device=dev).half()
        r = torch.randn(rows, N, device=dev).half() if has_res else None
        kw = dict(bias=bias, residual=r)
        if taps is CONV3:
            kw.update(dims=[side, side, B * F], taps=taps)
        elif taps is TEMP3:
            kw.update(dims=[side * side, F, B], taps=taps)
        if geglu:
            kw.update(flags=ops.GEMM_GEGLU, force_bn=256)     # the tile width the model packs this layer's weights for
        out = ops.gemm(a, wp, N, **kw)
        kw['out'] = out
        for _ in range(10):
            ops.gemm(a, wp, N, **kw)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            ops.gemm(a, wp, N, **kw)
        e1.record()
        torch.cuda.synchronize()
        us = e0.elapsed_time(e1) * 1e3 / iters
        flop = 2.0 * rows * N * K * ntaps
        res[name] = dict(family=fam, rows=rows, K=K, N=N, taps=ntaps, us=us, tflops=flop / us / 1e6)
        del a, wp, bias, r, out, kw
    return res


def print_table(res, title):
    print(title)
    print(f'{"shape":30s} {"rows":>7s} {"K":>5s} {"N":>5s} {"taps":>4s} {"us":>9s} {"TFLOP/s":>8s}')
    for name, v in res.items():
        print(f'{name:30s} {v["rows"]:7d} {v["K"]:5d} {v["N"]:5d} {v["taps"]:4d} {v["us"]:9.1f} {v["tflops"]:8.1f}')


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=200)
    ap.add_argument('--ab', nargs=2, metavar=('A_LIB', 'B_LIB'))
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--json', action='store_true', help='print one JSON line of results (used by --ab)')
    ap.add_argument('--out', help='also write the report to this file')
    args = ap.parse_args()
    lines = []

    def emit(s=''):
        print(s, flush=True)
        lines.append(s)

    if not args.ab:
        res = measure(args.iters)
        if args.json:
            print(json.dumps(res))
            return
        emit(f'gpu: {gpu_info()}')
        emit(f'library: {os.environ.get("T2V_LIB_PATH", "(package default)")}')
        import io, contextlib
        buf = io.StringIO()
        with contextlib.redirect_stdout(buf):
            print_table(res, f'ops.gemm per launch, {args.iters} launches per shape')
        for l in buf.getvalue().splitlines():
            emit(l)
    else:
        emit(f'gpu: {gpu_info()}')
        runs = {0: [], 1: []}
        for rnd in range(args.rounds):
            for which in (0, 1):
                env = dict(os.environ, T2V_LIB_PATH=os.path.abspath(args.ab[which]))
                p = subprocess.run([sys.executable, os.path.abspath(__file__), '--json', '--iters', str(args.iters)],
                                   env=env, capture_output=True, text=True)
                if p.returncode != 0:
                    sys.stderr.write(p.stderr[-4000:])
                    raise SystemExit(f'run {rnd} of {"AB"[which]} failed')
                runs[which].append(json.loads(p.stdout.strip().splitlines()[-1]))
        emit(f'A = {args.ab[0]}\nB = {args.ab[1]}\n{args.rounds} alternating rounds, {args.iters} launches per shape; '
             'us = median over rounds (min..max)')
        emit(f'{"shape":30s} {"A us":>18s} {"B us":>18s} {"B/A":>6s} {"A TF/s":>7s} {"B TF/s":>7s}')
        for name in runs[0][0]:
            a = [r[name]['us'] for r in runs[0]]
            b = [r[name]['us'] for r in runs[1]]
            ma, mb = statistics.median(a), statistics.median(b)
            ta, tb = runs[0][0][name]['tflops'] * runs[0][0][name]['us'] / ma, runs[0][0][name]['tflops'] * runs[0][0][name]['us'] / mb
            emit(f'{name:30s} {ma:7.1f} ({min(a):5.0f}..{max(a):5.0f}) {mb:7.1f} ({min(b):5.0f}..{max(b):5.0f}) '
                 f'{mb / ma:6.3f} {ta:7.1f} {tb:7.1f}')
    if args.out:
        with open(args.out, 'w') as f:
            f.write('\n'.join(lines) + '\n')


if __name__ == '__main__':
    main()
