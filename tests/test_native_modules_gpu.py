"""GPU: a checkpoint loaded through a parent module (LatentDiffusion.load_state_dict) after the mirrors have already run is
what the next UNet forward and VAE decode use, and a reload of the same weights leaves every result bit-identical."""
import pytest
import torch

from oracle import unet_oracle as UO

pytestmark = pytest.mark.gpu


def _ldm():
    from t2v_b200.videocrafter import LatentDiffusion
    return LatentDiffusion(unet_config=dict(model_channels=64, context_dim=48, temporal_length=4), image_size=[8, 8], video_length=4)


def _weights(m, seed):
    """Seeded values for every parameter of `m` (the schedule buffers keep theirs)."""
    sd = m.state_dict()
    return dict(sd, **UO.make_weights({k: tuple(v.shape) for k, v in sd.items() if '.' in k}, seed=seed))


def _run(m):
    g = torch.Generator('cpu').manual_seed(7)
    x, ctx, z = torch.randn(2, 4, 4, 8, 8, generator=g), torch.randn(2, 9, 48, generator=g), torch.randn(1, 4, 2, 8, 8, generator=g)
    eps = m.apply_model(x.cuda(), torch.tensor([500, 20]).cuda(), ctx.cuda())
    return eps.clone(), m.decode_first_stage(z.cuda(), return_cpu=False).clone()


def test_parent_load_after_a_run_uses_the_new_weights():
    m = _ldm()
    A, B = _weights(m, 1), _weights(m, 2)
    m.load_state_dict(A, strict=True)
    m = m.half().cuda().eval()
    eps_a, frames_a = _run(m)
    m.load_state_dict(B, strict=True)
    eps_b, frames_b = _run(m)
    fresh = _ldm()
    fresh.load_state_dict(B, strict=True)
    eps_ref, frames_ref = _run(fresh.half().cuda().eval())
    assert not torch.equal(eps_a, eps_ref) and not torch.equal(frames_a, frames_ref)        # the two checkpoints differ
    assert torch.equal(eps_b, eps_ref) and torch.equal(frames_b, frames_ref)
    m.load_state_dict(m.state_dict(), strict=True)              # a no-op reload reships the same values
    eps_again, frames_again = _run(m)
    assert torch.equal(eps_again, eps_b) and torch.equal(frames_again, frames_b)
