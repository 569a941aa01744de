"""Sample-parallel sharding of clips over the GPUs of one node -- the only parallelism the reference has
(videocrafter/sample_text2video.py:174-188 + lvdm/utils/dist_utils.py:4-19): every rank owns the full weights, draws its
own noise from `seed + rank`, and ONE all-gather collects the decoded clips.  No collective touches the denoising
loop, so scaling is weak.  Backend-agnostic (NCCL over NVLink on a multi-GPU node, gloo in the CPU tests).

Opt-in second mode (T2V_CFG_SPLIT=1, even world size): the classifier-free-guidance pair of every step -- two independent
forwards, gaussian_sampler.py:161-162 / ddim/sampler.py:176-179 / ddim.py:216-217 -- is split over a PAIR of GPUs (even
rank = conditional, odd rank = unconditional) with one all-gather of the two eps tensors per step (196 KB at 24f x 256^2)
inside the pair; both ranks then apply the identical fused update, so the latent stays replicated.  This halves the
latency of ONE clip (B = 1 forward per GPU instead of B = 2) at the cost of half the clips in flight; SURVEY.md 8e.

Third mode, frame sharding (BASELINE config 4: ONE 125-frame clip over 8 GPUs, `FrameShardedClip` below): every rank keeps
only its frames of the latent through the whole sampling loop -- the scheduler updates are element-wise -- and the UNet
exchanges activations between the ranks inside its own kernels over NVLink peer memory (csrc/shard.cu; no NCCL call per
step).  NCCL is used for exactly what the north-star names: ONE all-gather of the final latent before the VAE decode (each
rank then decodes its own frames) and one all-gather of the decoded frames."""
import os

import torch
import torch.distributed as dist


def world():
    return (dist.get_rank(), dist.get_world_size()) if dist.is_available() and dist.is_initialized() else (0, 1)


def clips_for_rank(n_clips, rank, world_size):
    """Global clip indices this rank renders (round-robin, like ceil(n_samples / world) per rank)."""
    return list(range(rank, n_clips, world_size))


def clip_seed(base_seed, clip_index):
    """Global clip i always uses base_seed + i, independent of the number of ranks (reproducible under resharding)."""
    return base_seed + clip_index


def gather_clips(frames_u8):
    """frames_u8: [F, H, W, 3] uint8 of this rank's clip -> list of world_size tensors (rank order) on every rank."""
    rank, ws = world()
    if ws == 1:
        return [frames_u8]
    out = [torch.empty_like(frames_u8) for _ in range(ws)]
    dist.all_gather(out, frames_u8.contiguous())
    return out


# ------------------------------------------------------------------------------------------------ CFG-pair split
_pair_groups = None


def cfg_split_enabled():
    rank, ws = world()
    return os.environ.get('T2V_CFG_SPLIT') == '1' and ws >= 2 and ws % 2 == 0


def cfg_pair():
    """(pair index, role, process group): role 0 evaluates the conditional branch, role 1 the unconditional one.
    Every rank creates every pair group once (new_group is collective over the whole world)."""
    global _pair_groups
    rank, ws = world()
    if _pair_groups is None:
        _pair_groups = [dist.new_group([2 * i, 2 * i + 1]) for i in range(ws // 2)]
    return rank // 2, rank % 2, _pair_groups[rank // 2]


def units():
    """(index, count) of the unit that renders whole clips: a rank in sample-DP mode, a rank pair in CFG-split mode."""
    rank, ws = world()
    return (rank // 2, ws // 2) if cfg_split_enabled() else (rank, ws)


def exchange_eps(e_mine, group):
    """All-gather of the two branches inside the pair -> (eps_cond, eps_uncond) on both ranks."""
    e_mine = e_mine.contiguous()
    out = [torch.empty_like(e_mine), torch.empty_like(e_mine)]
    dist.all_gather(out, e_mine, group=group)
    return out[0], out[1]


_role_groups = None


def cfg_role_group():
    """CFG split x frame shard (SURVEY.md 8e "2 x 4" layout): the ranks that evaluate the SAME guidance branch form one
    frame-shard group (even ranks = conditional, odd ranks = unconditional); rank 2i and 2i+1 hold the same frames and
    exchange their eps once per step (exchange_eps).  Every rank creates both groups (new_group is collective)."""
    global _role_groups
    rank, ws = world()
    if _role_groups is None:
        _role_groups = [dist.new_group(list(range(r, ws, 2))) for r in (0, 1)]
    return _role_groups[rank % 2]


def pair_shared(noise):
    """Per-step sampler noise in CFG-split mode: both ranks of a pair must apply the IDENTICAL update, but each rank's global
    CUDA generator is its own -- with eta > 0 the latents would silently drift apart after the first step.  Role 0's draw is
    broadcast inside the pair (every rank still advances its own generator, so stream positions stay aligned)."""
    if not cfg_split_enabled():
        return noise
    pair, role, grp = cfg_pair()
    dist.broadcast(noise, src=2 * pair, group=grp)
    return noise


def pair_callback(callback, *args):
    """Runs the per-step host callback; in CFG-split mode the decision to interrupt is made collective inside the pair (a
    callback raising on one rank only would leave its partner blocked in the next eps all-gather)."""
    if not cfg_split_enabled():
        return callback(*args)
    _, _, grp = cfg_pair()
    err = None
    try:
        callback(*args)
    except BaseException as e:            # InterruptedException derives from BaseException in the webui
        err = e
    flag = torch.tensor([1 if err is not None else 0], dtype=torch.int32,
                        device='cuda' if dist.get_backend(grp) == 'nccl' else 'cpu')
    dist.all_reduce(flag, op=dist.ReduceOp.MAX, group=grp)
    if err is not None:
        raise err
    if int(flag.item()) != 0:
        from .samplers import InterruptedException
        raise InterruptedException()


# ------------------------------------------------------------------------------------------------ frame-sharded clip
_frame_shard = None          # the active FrameShardedClip while its sampling loop runs (samplers draw noise through it)


def frame_bounds(F, world_size):
    """Balanced contiguous frame ranges, larger ones first -- the same partition csrc/shard.cuh::shard_partition computes."""
    out, off = [], 0
    for r in range(world_size):
        out.append(off)
        off += F // world_size + (1 if r < F % world_size else 0)
    return out + [off]


def step_noise(like):
    """Per-step sampler noise (eta > 0).  A batch of n clips draws one clip-sized tensor per clip, in clip order, from the
    global CUDA generator: a batched run consumes it step-major (step s of clips 0..n-1, then step s + 1), n sequential runs
    clip-major, so the two give different per-step noise from the same generator state.
    Frame-sharded: every rank draws the FULL clip's noise from its (identically seeded) CUDA generator and keeps its frames,
    so the result does not depend on the number of ranks."""
    fs = _frame_shard
    if fs is None:
        if like.shape[0] > 1:
            return pair_shared(torch.cat([torch.randn_like(like[i:i + 1]) for i in range(like.shape[0])], dim=0))
        return pair_shared(torch.randn_like(like))
    full = torch.randn((like.shape[0], like.shape[1], fs.F) + tuple(like.shape[3:]), device=like.device, dtype=like.dtype)
    return full[:, :, fs.f0:fs.f1].contiguous()


class FrameShardedClip(object):
    """Drives ONE clip over the ranks of `group`: slices x_T, runs the unchanged scheduler classes on this rank's frames
    (the UNet mirror is in shard mode), gathers the final latent once, decodes this rank's frames, gathers the frames."""

    def __init__(self, sd_model, autoencoder, group=None):
        self.sd_model, self.autoencoder, self.group = sd_model, autoencoder, group
        self.rank, self.ws = dist.get_rank(group), dist.get_world_size(group)
        if getattr(sd_model, '_shard', None) is None:
            sd_model.shard_setup(group)
        self.F = self.f0 = self.f1 = None

    def begin(self, F, seed=None):
        global _frame_shard
        self.F = int(F)
        b = frame_bounds(self.F, self.ws)
        self.f0, self.f1 = b[self.rank], b[self.rank + 1]
        self.sd_model.set_clip_frames(self.F)
        if seed is not None:
            torch.cuda.manual_seed(int(seed))          # identical per-step noise streams on every rank (eta > 0)
        _frame_shard = self

    def end(self):
        global _frame_shard
        _frame_shard = None

    def local(self, x_full):
        return x_full[:, :, self.f0:self.f1].contiguous()

    def _gather_frames(self, t, dim):
        """all-gather of per-rank frame slices with ragged counts (padded to the largest slice)."""
        b = frame_bounds(self.F, self.ws)
        nmax = max(b[r + 1] - b[r] for r in range(self.ws))
        pad_shape = list(t.shape)
        pad_shape[dim] = nmax
        buf = torch.zeros(pad_shape, dtype=t.dtype, device=t.device)
        buf.narrow(dim, 0, t.shape[dim]).copy_(t)
        out = [torch.empty_like(buf) for _ in range(self.ws)]
        dist.all_gather(out, buf, group=self.group)
        return torch.cat([out[r].narrow(dim, 0, b[r + 1] - b[r]) for r in range(self.ws)], dim=dim)

    def gather_latent(self, x_local):
        """THE all-gather before the VAE: [1, 4, F_local, h, w] -> [1, 4, F, h, w] on every rank."""
        return self._gather_frames(x_local.contiguous(), 2)

    def decode(self, x0_full, z_scale):
        """Frame-sharded VAE: this rank decodes its own frames (the decoder is per-frame), then one all-gather of uint8 frames."""
        mine = self.autoencoder.decode_video(self.local(x0_full), z_scale, as_uint8=True)      # [F_local, H, W, 3]
        return self._gather_frames(mine, 0)
