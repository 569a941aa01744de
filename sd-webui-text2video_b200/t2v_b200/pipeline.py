"""`TextToVideoSynthesis` -- the pipeline object behind the reference's `process_modelscope` entry point
(scripts/modelscope/t2v_pipeline.py:45-385), with the denoising loop and the VAE decode on the GPU-native library.

Same public surface: `TextToVideoSynthesis(model_dir)`, attributes `.sd_model .autoencoder .clip_encoder .diffusion
.model_dir .keep_in_vram`, and `infer(prompt, n_prompt, steps, frames, seed, scale, width, height, eta, cpu_vae,
device, latents, skip_steps, strength, mask, is_vid2vid, sampler, batch_size=1) -> (list of HxWx3 uint8 BGR frames, last
latent, infotext)`; with batch_size = n > 1 each of the three is a list of n, clip i seeded seed + i.

Differences that are the point of this repo:
  * UNet + samplers + VAE run through libt2v_b200.so (no autocast, no PyTorch kernels on the hot path);
  * the VAE decodes all frames in one batched call and converts to uint8 on the device; ONE D2H copy of the finished
    clip replaces the reference's per-frame `.cpu()` sync (t2v_pipeline.py:347-355);
  * text conditioning is out of the hot path (SURVEY.md section 2, row 4): `prompt` / `n_prompt` may be strings when a
    `clip_encoder` with `.encode(list[str]) -> [1, L, context_dim]` is plugged in, or already-encoded tensors.
"""
import json
import os
import random

import numpy as np
import torch

from . import distributed as _dist
from .modules import UNetSD, AutoencoderKL
from .samplers import Txt2VideoSampler, available_samplers

SCALE_FACTOR = 0.18215          # t2v_pipeline.py:321
BUDGET_MARGIN = 512 << 20       # what a plan build allocates outside its arena (the VAE's rule, DESIGN.md section 2)


def batch_groups(n, fits):
    """Splits n clips into consecutive groups of the largest size k <= n with fits(k) (the B = 2k plan fits the memory
    budget), the last group the remainder.  [] if not even one clip fits."""
    k = n
    while k > 0 and not fits(k):
        k -= 1
    if k == 0:
        return []
    return [k] * (n // k) + ([n % k] if n % k else [])

VAE_DDCONFIG = {'double_z': True, 'z_channels': 4, 'resolution': 256, 'in_channels': 3, 'out_ch': 3, 'ch': 128,
                'ch_mult': [1, 2, 4, 4], 'num_res_blocks': 2, 'attn_resolutions': [], 'dropout': 0.0}   # :117-128

DEFAULT_UNET_CFG = {'unet_in_dim': 4, 'unet_dim': 320, 'unet_y_dim': 768, 'unet_context_dim': 1024, 'unet_out_dim': 4,
                    'unet_dim_mult': [1, 2, 4, 4], 'unet_num_heads': 8, 'unet_head_dim': 64, 'unet_res_blocks': 2,
                    'unet_attn_scales': [1, 0.5, 0.25], 'unet_dropout': 0.1, 'temporal_attention': 'True',
                    'num_timesteps': 1000, 'mean_type': 'eps'}       # public damo-vilab configuration.json values


def linear_sd_betas(num_timesteps=1000, init_beta=0.00085, last_beta=0.0120):
    """'linear_sd' schedule (t2v_model.py:1240-1249 called from t2v_pipeline.py:107-111)."""
    return torch.linspace(init_beta ** 0.5, last_beta ** 0.5, num_timesteps, dtype=torch.float64) ** 2


class TextToVideoSynthesis(object):
    def __init__(self, model_dir=None, *, model_cfg=None, unet_state=None, vae_state=None, clip_encoder=None,
                 device=None):
        """`model_dir` as in the reference (configuration.json + checkpoints).  For synthetic runs pass `model_cfg`
        (dict with the configuration.json `model_cfg` keys) and state dicts directly."""
        self.model_dir = model_dir
        self.device = torch.device(device) if device is not None else torch.device('cuda', torch.cuda.current_device())
        self.keep_in_vram = 'None'
        cfg = dict(DEFAULT_UNET_CFG)
        args = {}
        if model_dir is not None:
            with open(os.path.join(model_dir, 'configuration.json'), 'r') as f:
                conf = json.load(f)
            cfg.update(conf['model']['model_cfg'])
            args = conf['model'].get('model_args', {})
        if model_cfg:
            cfg.update(model_cfg)
        self.config = cfg
        with torch.device(self.device):          # parameters are created on the GPU directly (1.4 B of them)
          self.sd_model = UNetSD(in_dim=cfg['unet_in_dim'], dim=cfg['unet_dim'], y_dim=cfg['unet_y_dim'],
                               context_dim=cfg['unet_context_dim'], out_dim=cfg['unet_out_dim'],
                               dim_mult=cfg['unet_dim_mult'], num_heads=cfg['unet_num_heads'],
                               head_dim=cfg['unet_head_dim'], num_res_blocks=cfg['unet_res_blocks'],
                               attn_scales=cfg['unet_attn_scales'], dropout=cfg['unet_dropout'],
                               parameterization=cfg['mean_type'],
                               temporal_attention=str(cfg['temporal_attention']) == 'True')
        if unet_state is None and model_dir is not None:
            unet_state = torch.load(os.path.join(model_dir, args['ckpt_unet']), map_location='cpu')
        if unet_state is not None:
            self.sd_model.load_state_dict(unet_state, strict=True)
        self.sd_model.eval().half()
        betas = linear_sd_betas(cfg['num_timesteps'])
        self.sd_model.register_schedule(given_betas=betas.numpy())
        self.sd_model.to(self.device)
        self.diffusion = Txt2VideoSampler(self.sd_model, self.device, betas=betas)
        ckpt_vae = os.path.join(model_dir, args['ckpt_autoencoder']) if (model_dir and vae_state is None) else None
        with torch.device(self.device):
            self.autoencoder = AutoencoderKL(VAE_DDCONFIG, 4, ckpt_vae)
        if vae_state is not None:
            own = self.autoencoder.state_dict()
            own.update(vae_state)                    # decoder-only synthetic states are allowed
            self.autoencoder.load_state_dict(own, strict=True)
        self.autoencoder.eval().half().to(self.device)
        if clip_encoder is None and model_dir is not None and args.get('ckpt_clip') and \
                os.path.exists(os.path.join(model_dir, args['ckpt_clip'])):
            # t2v_pipeline.py:64-69: FrozenOpenCLIPEmbedder(version=<model_dir>/<ckpt_clip>, layer='penultimate'); the text
            # transformer runs on the library (t2v_b200/clip.py).  Needs a BPE tokenizer for string prompts (open_clip's).
            from .clip import FrozenOpenCLIPEmbedder
            clip_encoder = FrozenOpenCLIPEmbedder(version=os.path.join(model_dir, args['ckpt_clip']), layer='penultimate')
            clip_encoder.model.half().to(self.device)
        self.clip_encoder = clip_encoder
        self.noise_gen = torch.Generator(device='cpu')
        self.last_tensor = None
        self.frame_shard = None
        # batch_size > 1: bytes of denoiser plan (activation arena) a batch may add; 0 = automatic: free device memory - 512 MB
        self.batch_memory_budget = 0
        self.last_batch_groups = None           # clips per B = 2k forward of the last batched infer()

    def enable_frame_shard(self, group=None):
        """ONE clip over the ranks of `group` (BASELINE config 4): every rank calls infer() with the same arguments and gets
        the same finished clip; the denoiser exchanges activations over NVLink inside its kernels (distributed.py)."""
        from .distributed import FrameShardedClip
        self.frame_shard = FrameShardedClip(self.sd_model, self.autoencoder, group)
        return self.frame_shard

    # ------------------------------------------------------------------------------------------ conditioning
    def preprocess(self, prompt, n_prompt, steps=None):
        def enc(p):
            if torch.is_tensor(p):
                return p.to(self.device, non_blocking=True)
            if self.clip_encoder is None:
                raise RuntimeError('string prompts need a clip_encoder (the OpenCLIP text tower is outside the '
                                   'hot path built here); pass encoded [1, L, context_dim] tensors instead')
            return self.clip_encoder.encode([p]).to(self.device)
        return enc(prompt), enc(n_prompt)

    # ------------------------------------------------------------------------------------------ entry
    def plan_groups(self, n, frames, height, width, L):
        """How n clips of one batched infer() are grouped: the largest k whose B = 2k denoiser plan (context batch 2, host
        dry pass) fits the budget runs first, as many times as it fits, then the remainder.  A cached plan needs no new
        memory.  Raises if a single clip's B = 2 plan does not fit."""
        budget = self.batch_memory_budget or max(torch.cuda.mem_get_info(self.device)[0] - BUDGET_MARGIN, 0)
        h, w = height // 8, width // 8
        need = {}

        def fits(k):
            arena, _, cached = self.sd_model.plan_info(2 * k, frames, h, w, L, ctx_batch=2)
            need[k] = 0 if cached else arena
            return need[k] <= budget
        groups = batch_groups(n, fits)
        if not groups:
            raise RuntimeError(f'batch of {n} clips of {frames} x {height} x {width}: one clip\'s B = 2 denoiser plan needs '
                               f'{need[1] / 1e9:.2f} GB, more than the memory budget of {budget / 1e9:.2f} GB')
        return groups

    @torch.no_grad()
    def infer(self, prompt, n_prompt, steps, frames, seed, scale, width=256, height=256, eta=0.0,
              cpu_vae='GPU (half precision)', device=None, latents=None, skip_steps=0, strength=0, mask=None,
              is_vid2vid=False, sampler=available_samplers[0].name, batch_size=1):
        if 'CPU' in str(cpu_vae):
            raise RuntimeError('the CPU VAE mode of the reference does not exist here: t2v_b200 has no CPU path')
        if batch_size > 1:
            if self.frame_shard is not None:
                raise NotImplementedError('batch_size > 1 with a frame-sharded clip: run the clips one after another')
            if _dist.cfg_split_enabled():
                raise NotImplementedError('batch_size > 1 in CFG-split mode (T2V_CFG_SPLIT=1): run the clips one after another')
        seed = seed if seed != -1 else random.randint(0, 2 ** 32 - 1)
        if batch_size > 1:
            return self._infer_batch(prompt, n_prompt, steps, frames, seed, scale, width, height, eta, cpu_vae, latents,
                                     skip_steps, strength, mask, is_vid2vid, sampler, batch_size)
        vars_ = {'steps': steps, 'frames': frames, 'seed': seed, 'scale': scale, 'width': width, 'height': height,
                 'eta': eta, 'sampler': sampler}
        steps = steps - skip_steps
        c, uc = self.preprocess(prompt, n_prompt, steps)
        strength = None if (strength == 0.0 and not is_vid2vid) else strength
        if latents is not None:
            latents = latents.to(self.device)       # the reference's get_noise discards its `.to(device)` (samplers_common.py:106)
            if 'half precision' in str(cpu_vae):    # t2v_pipeline.py:257: vid2vid latents (and the mask) are rounded to fp16, which
                latents = latents.half()            # also rounds the scheduler's entry latent (`.to(dtype=latent.dtype)`)
        latents, noise, shape = self.diffusion.get_noise(1, 4, frames, height, width, seed=seed, latents=latents)
        self.diffusion.get_sampler(sampler, return_sampler=False)
        fs = self.frame_shard
        if fs is not None:
            # frame-sharded clip: the (identical, CPU-seeded) x_T is cut to this rank's frames; the scheduler never sees more
            fs.begin(shape[2], seed)
            noise = fs.local(noise)
            latents = fs.local(latents) if latents is not None else None
            shape = tuple(noise.shape)
        try:
            x0 = self.diffusion.sample_loop(steps=steps, strength=strength, eta=eta, conditioning=c,
                                            unconditional_conditioning=uc, batch_size=1, guidance_scale=scale,
                                            latents=latents, shape=shape, noise=noise, is_vid2vid=is_vid2vid,
                                            sampler_name=sampler, mask=mask)
        finally:
            if fs is not None:
                fs.end()
        if fs is not None:
            x0 = fs.gather_latent(x0)               # the single NCCL all-gather before the VAE
            self.last_tensor = x0
            frames_u8 = fs.decode(x0, 1.0 / SCALE_FACTOR)
        else:
            self.last_tensor = x0
            frames_u8 = self.autoencoder.decode_video(x0, 1.0 / SCALE_FACTOR, as_uint8=True)     # [F, H, W, 3] RGB, device
        host = torch.empty(frames_u8.shape, dtype=torch.uint8, pin_memory=True)
        host.copy_(frames_u8, non_blocking=True)                                              # the one D2H of the clip
        torch.cuda.current_stream().synchronize()
        rgb = host.numpy()
        video = [np.ascontiguousarray(f[:, :, ::-1]) for f in rgb]       # cv2.COLOR_RGB2BGR (t2v_pipeline.py:431-434)
        return video, self.last_tensor, create_infotext(prompt, n_prompt, vars_)

    def _infer_batch(self, prompt, n_prompt, steps, frames, seed, scale, width, height, eta, cpu_vae, latents, skip_steps,
                     strength, mask, is_vid2vid, sampler, n):
        """infer() of n clips seeded seed, seed + 1, ...: each step guides a group of k clips with ONE B = 2k forward, and
        the VAE decodes all n * frames frames in one call.  Start latents (vid2vid / img2vid): one per clip ([n, ...]), or
        one of batch 1 shared by the clips."""
        seeds = [seed + i for i in range(n)]
        steps_total = steps
        steps = steps - skip_steps
        c, uc = self.preprocess(prompt, n_prompt, steps)
        strength = None if (strength == 0.0 and not is_vid2vid) else strength
        if latents is not None:
            latents = latents.to(self.device)
            if 'half precision' in str(cpu_vae):
                latents = latents.half()
        F = latents.shape[2] if latents is not None else frames     # a vid2vid clip has its input video's frames
        groups = self.plan_groups(n, F, height, width, c.shape[1])
        self.last_batch_groups = groups
        outs, first = [], 0
        if latents is not None and latents.shape[0] not in (1, n):
            raise ValueError(f'{n} clips take start latents of batch 1 or {n}, got {tuple(latents.shape)}')
        for k in groups:
            lat = latents[first:first + k] if latents is not None and latents.shape[0] == n else latents
            mask_k = mask[first:first + k] if mask is not None and mask.shape[0] == n else mask
            lat_k, noise, shape = self.diffusion.get_noise(k, 4, frames, height, width, latents=lat,
                                                           seeds=seeds[first:first + k])
            # a fresh sampler per group, as per infer(): encode_latent rebinds DDIM's .sample for vid2vid
            self.diffusion.get_sampler(sampler, return_sampler=False)
            outs.append(self.diffusion.sample_loop(steps=steps, strength=strength, eta=eta, conditioning=c,
                                                   unconditional_conditioning=uc, batch_size=k, guidance_scale=scale,
                                                   latents=lat_k, shape=shape, noise=noise, is_vid2vid=is_vid2vid,
                                                   sampler_name=sampler, mask=mask_k))
            first += k
        x0 = torch.cat(outs, dim=0)
        self.last_tensor = x0
        frames_u8 = self.autoencoder.decode_video(x0, 1.0 / SCALE_FACTOR, as_uint8=True)        # [n * F, H, W, 3] RGB
        host = torch.empty(frames_u8.shape, dtype=torch.uint8, pin_memory=True)
        host.copy_(frames_u8, non_blocking=True)
        torch.cuda.current_stream().synchronize()
        rgb = host.numpy()
        videos = [[np.ascontiguousarray(f[:, :, ::-1]) for f in rgb[i * F:(i + 1) * F]] for i in range(n)]
        infos = [create_infotext(prompt, n_prompt, {'steps': steps_total, 'frames': frames, 'seed': s, 'scale': scale,
                                                    'width': width, 'height': height, 'eta': eta, 'sampler': sampler})
                 for s in seeds]
        return videos, [x0[i:i + 1] for i in range(n)], infos

    def prepare_frames(self, frames_u8, width, height, cpu_vae='GPU (half precision)'):
        """The reference's frame preparation for compute_latents (process_modelscope.py:115-137, :172-190): every uint8 RGB
        frame ([f, H0, W0, 3] array or CUDA tensor, or a sequence of [H0, W0, 3] arrays / RGB PIL images) resized to
        width x height with PIL's LANCZOS, then x / 255 * 2 - 1, bit for bit, on the device (t2v_frames_resize) ->
        [1, 3, f, height, width] (a view of a dense [f, 3, height, width]): fp16 in the half-precision VAE mode, the value
        compute_latents' `.half()` gives, fp32 otherwise."""
        from . import ops
        dtype = torch.float16 if 'half precision' in str(cpu_vae) else torch.float32
        with torch.cuda.device(self.device):
            out = ops.frames_resize(frames_u8, width, height, dtype)
        return out.permute(1, 0, 2, 3).unsqueeze(0)

    @torch.no_grad()
    def compute_latents(self, vd_out, cpu_vae='GPU (half precision)', device=None):
        """vid2vid / img2vid latent preparation (t2v_pipeline.py:148-194): vd_out [b, 3, f, H, W] in [-1, 1] ->
        latents [b, 4, f, H/8, W/8] fp32 on the CPU = posterior.mean * 0.18215.  All frames are encoded in one batch
        instead of the reference's chunk-of-one loop; `cpu_vae` variants other than the GPU ones raise (no CPU path)."""
        if 'CPU' in cpu_vae:
            raise RuntimeError('t2v_b200 has no CPU VAE path; use "GPU (half precision)"')
        dev = device if device is not None else self.device
        b, c, f, H, W = vd_out.shape
        frames = vd_out.to(dev).permute(0, 2, 1, 3, 4).reshape(b * f, c, H, W)
        frames = frames.half() if 'half precision' in cpu_vae else frames.float()
        mean = self.autoencoder.encode(frames).mean * SCALE_FACTOR
        lat = mean.reshape(b, f, *mean.shape[1:]).permute(0, 2, 1, 3, 4)
        return lat.to(torch.float32).cpu()


def create_infotext(prompt, n_prompt, params):
    p = prompt if isinstance(prompt, str) else '<encoded prompt>'
    n = n_prompt if isinstance(n_prompt, str) else ''
    tail = ', '.join(f'{k}: {v}' for k, v in params.items() if v is not None)
    neg = ('\nNegative prompt: ' + n) if len(n) > 0 else ''
    return f'{p}{neg}\n{tail}'.strip()
