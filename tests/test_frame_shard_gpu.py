"""GPU (>= 2 devices): ONE clip frame-sharded over the GPUs of the node == the same clip on one GPU.

Launches tests/shard_worker.py under torch.distributed.run (one process per GPU, NCCL for the plumbing, the activation
exchange inside the denoiser's own kernels over NVLink peer memory).  Gate: sharded vs unsharded relative RMS <= 4e-3 (the
two are independent fp16 roundings of the same function -- per-rank row counts change the GEMM tiling / split-K accumulation
order -- each ~2.3e-3 from the fp32 oracle on one H100, so they differ from each other by up to sqrt(2) x that) and the sharded path is as
close to the fp32 oracle as the unsharded one (x 1.5)."""
import json
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def run_worker(nproc, env_extra=None, timeout=900):
    env = dict(os.environ)
    env.update(env_extra or {})
    cmd = [sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', f'--nproc-per-node={nproc}', '--master-addr', '127.0.0.1',
           '--master-port', '29731', os.path.join(ROOT, 'tests', 'shard_worker.py')]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=timeout, env=env, cwd=ROOT)
    recs = [json.loads(l[6:]) for l in r.stdout.splitlines() if l.startswith('SHARD ')]
    assert r.returncode == 0 and recs, (r.stdout[-3000:], r.stderr[-3000:])
    return recs


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason='needs >= 2 GPUs')
@pytest.mark.parametrize('nproc', [2, 4, 8])
def test_sharded_clip_equals_unsharded(nproc):
    if torch.cuda.device_count() < nproc:
        pytest.skip(f'{nproc} GPUs needed')
    recs = run_worker(nproc)
    for r in recs:
        print('[shard] ' + json.dumps(r))
    for r in recs:
        if r['case'].startswith('forward'):
            assert r['sharded_vs_unsharded_rms'] <= 4e-3, r
            assert r['sharded_vs_oracle_rms'] <= 1.5 * r['unsharded_vs_oracle_rms'] + 5e-4, r
        else:
            assert r['latent_rms'] <= 1e-2 and r['u8_mean_abs_diff'] < 1.0, r
