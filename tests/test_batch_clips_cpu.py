"""CPU: host logic of batched ModelScope clips -- per-clip seeding of x_T, grouping of `batch_count` into batches and of a
batch into plan-sized groups, the errors of the frame-sharded and CFG-split modes, and the shared-context plan's K/V
projection (host dry pass: one projection per prompt row, not per sample)."""
from types import SimpleNamespace

import pytest
import torch


def test_get_noise_seeds_each_clip_like_its_own_run():
    from t2v_b200.samplers import Txt2VideoSampler
    s = Txt2VideoSampler.__new__(Txt2VideoSampler)
    s.noise_gen, s.device = torch.Generator(device='cpu'), torch.device('cpu')
    _, noise, shape = s.get_noise(3, 4, 5, 64, 48, seeds=[40, 41, 42])
    assert shape == (3, 4, 5, 8, 6) and noise.shape == shape
    for i in range(3):
        _, single, single_shape = s.get_noise(1, 4, 5, 64, 48, seed=40 + i)
        assert single_shape == (1, 4, 5, 8, 6) and torch.equal(noise[i:i + 1], single)
    lat = torch.randn(1, 4, 5, 8, 6)
    lat_b, noise_b, shape_b = s.get_noise(2, 4, 5, 64, 48, latents=lat, seeds=[7, 8])
    assert shape_b == (2, 4, 5, 8, 6) and torch.equal(lat_b, lat.expand(2, -1, -1, -1, -1))
    assert torch.equal(noise_b[1:2], s.get_noise(1, 4, 5, 64, 48, latents=lat, seed=8)[1])
    per_clip = torch.randn(2, 4, 5, 8, 6)                       # img2vid: one start latent per clip, kept as given
    lat_p, noise_p, _ = s.get_noise(2, 4, 5, 64, 48, latents=per_clip, seeds=[7, 8])
    assert torch.equal(lat_p, per_clip) and torch.equal(noise_p, noise_b)
    with pytest.raises(ValueError):
        s.get_noise(3, 4, 5, 64, 48, latents=torch.randn(2, 4, 5, 8, 6), seeds=[1, 2, 3])


def test_step_noise_draws_one_tensor_per_clip_in_clip_order():
    """Per-step noise of a batch of n clips = n clip-sized draws from the global generator, clip 0 first; batch 1 is one
    draw of its own shape, as before."""
    from t2v_b200 import distributed as D
    like = torch.empty(3, 4, 2, 3, 5)
    torch.manual_seed(5)
    got = D.step_noise(like)
    torch.manual_seed(5)
    want = torch.cat([torch.randn_like(like[:1]) for _ in range(3)])
    assert got.shape == like.shape and torch.equal(got, want)
    torch.manual_seed(5)
    one = D.step_noise(like[:1])
    torch.manual_seed(5)
    assert torch.equal(one, torch.randn_like(like[:1]))


def test_batch_count_grouped_into_batches():
    from t2v_b200.process_modelscope import batch_sizes
    assert batch_sizes(1, 1) == [(0, 1)]
    assert batch_sizes(5, 1) == [(i, 1) for i in range(5)]
    assert batch_sizes(5, 2) == [(0, 2), (2, 2), (4, 1)]
    assert batch_sizes(3, 8) == [(0, 3)]
    with pytest.raises(ValueError):
        batch_sizes(3, 0)


def test_process_modelscope_runs_batches_with_their_first_seed():
    from t2v_b200 import process_modelscope as pm
    calls = []

    class FakePipe:
        model_dir = None

        def infer(self, *args, batch_size=1):
            calls.append((args[4], batch_size))
            clips = [[f'clip{args[4] + i}'] for i in range(batch_size)]
            return (clips[0], None, '') if batch_size == 1 else (clips, None, [''] * batch_size)
    old = pm.pipe
    pm.pipe = FakePipe()
    try:
        out = pm.process_modelscope({'prompt_embeds': 1, 'n_prompt_embeds': 2, 'seed': 10, 'batch_count': 5, 'batch_size': 2,
                                     'return_frames': True})
        assert calls == [(10, 2), (12, 2), (14, 1)]
        assert out == [[f'clip{10 + i}'] for i in range(5)]           # one output per clip, in seed order
        calls.clear()
        pm.process_modelscope({'prompt_embeds': 1, 'n_prompt_embeds': 2, 'seed': 10, 'batch_count': 2, 'return_frames': True})
        assert calls == [(10, 1), (11, 1)]                              # batch_size defaults to 1: the sequential loop
    finally:
        pm.pipe = old


def test_plan_groups_policy():
    from t2v_b200.pipeline import batch_groups
    assert batch_groups(4, lambda k: True) == [4]
    assert batch_groups(4, lambda k: k <= 2) == [2, 2]
    assert batch_groups(5, lambda k: k <= 2) == [2, 2, 1]
    assert batch_groups(7, lambda k: k <= 3) == [3, 3, 1]
    assert batch_groups(3, lambda k: False) == []


def _pipe_stub(**kw):
    return SimpleNamespace(**{'frame_shard': None, **kw})


def test_batched_infer_refuses_frame_shard_and_cfg_split(monkeypatch):
    from t2v_b200 import distributed as D
    from t2v_b200.pipeline import TextToVideoSynthesis
    with pytest.raises(NotImplementedError, match='frame-sharded'):
        TextToVideoSynthesis.infer(_pipe_stub(frame_shard=object()), None, None, 3, 2, 1, 5.0, batch_size=2)
    monkeypatch.setattr(D, 'cfg_split_enabled', lambda: True)
    with pytest.raises(NotImplementedError, match='CFG-split'):
        TextToVideoSynthesis.infer(_pipe_stub(), None, None, 3, 2, 1, 5.0, batch_size=2)


def test_plan_groups_error_names_shape_bytes_and_budget():
    from t2v_b200.modules import UNetSD
    from t2v_b200.pipeline import TextToVideoSynthesis
    net = UNetSD(dim=64)
    stub = _pipe_stub(sd_model=net, batch_memory_budget=1)
    with pytest.raises(RuntimeError, match=r'batch of 3 clips of 4 x 64 x 64: .* GB, more than the memory budget of'):
        TextToVideoSynthesis.plan_groups(stub, 3, 4, 64, 64, 77)
    need = {k: net.plan_info(2 * k, 4, 8, 8, 77, ctx_batch=2)[0] for k in (1, 2, 3, 4)}
    assert need[1] < need[2] < need[4]
    stub.batch_memory_budget = need[2]
    assert TextToVideoSynthesis.plan_groups(stub, 4, 4, 64, 64, 77) == [2, 2]
    stub.batch_memory_budget = need[4]
    assert TextToVideoSynthesis.plan_groups(stub, 4, 4, 64, 64, 77) == [4]


def test_shared_context_projects_each_prompt_once():
    """The plan of B = 6 samples over Bc = 2 prompts differs from the repeated context (Bc = B) only in the cross-attention
    K/V GEMMs, which project 2 * L rows instead of 6 * L: exactly (B - Bc) * L rows fewer per spatial transformer."""
    from t2v_b200.modules import UNetSD
    net = UNetSD(dim=64)
    B, F, h, w, L = 6, 3, 8, 8, 77
    arena_rep, fl_rep, cached = net.plan_info(B, F, h, w, L)
    assert not cached and fl_rep == net.flops(B, F, h, w, L) and arena_rep == net.plan_bytes(B, F, h, w, L)
    arena_sh, fl_sh, _ = net.plan_info(B, F, h, w, L, ctx_batch=2)
    assert arena_sh <= arena_rep
    # spatial transformers: attn2.to_k maps the 1024-wide context; temporal ones (self-attention) map their own width
    kv = [p.shape[0] for n, p in net.named_parameters() if n.endswith('attn2.to_k.weight') and p.shape[1] == net.context_dim]
    assert len(kv) > 0
    saved = sum(2.0 * (B - 2) * L * (2 * C) * net.context_dim for C in kv)
    assert fl_rep - fl_sh == pytest.approx(saved, rel=1e-9)
    with pytest.raises(RuntimeError, match='does not divide'):
        net.plan_info(B, F, h, w, L, ctx_batch=4)


def test_process_videocrafter_forwards_batch_size(monkeypatch):
    import numpy as np
    from t2v_b200 import videocrafter as V
    calls = []

    def fake_sample(model, prompt, n_prompt, n_samples, batch_size, **kw):
        calls.append((n_samples, batch_size))
        return np.arange(n_samples, dtype=np.float32).reshape(n_samples, 1, 1, 1, 1)
    monkeypatch.setattr(V, 'sample_text2video', fake_sample)
    monkeypatch.setattr(V, 'video_encoder', None)
    monkeypatch.setattr(V, 'model_cache', None)          # process_videocrafter caches the model it is given
    model = SimpleNamespace(num_timesteps=1000)
    out = V.process_videocrafter({'seed': 3, 'batch_count': 2, 'batch_size': 3}, model=model)
    assert calls == [(3, 3), (3, 3)] and len(out) == 6 and [float(o[0, 0, 0, 0, 0]) for o in out] == [0, 1, 2, 0, 1, 2]
    calls.clear()
    assert len(V.process_videocrafter({'seed': 3, 'batch_count': 2}, model=model)) == 2 and calls == [(1, 1), (1, 1)]
