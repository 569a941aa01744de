"""`process_modelscope(args_dict, extra_args)` -- the entry point `t2v_helpers.render.run` dispatches to
(reference: scripts/modelscope/process_modelscope.py:34-266), backed by the GPU-native pipeline.

Kept: the name, the signature, the return type (`list[str]` of data-URL videos, process_modelscope.py:34,:256-262), the
module-global `pipe` cache (reset by render.py:41 through `pipe = None`), the batch loop with `seed + batch`
(process_modelscope.py:160,:221), the argument names of `T2VArgs` (t2v_helpers/args.py:219-236), vid2vid (latent preparation
on the library) and img2vid inpainting: the per-frame weight schedule (`T2VAnimKeys`), the fp64 blend
`image_latents * (1 - mask) + noise * mask` (process_modelscope.py:170-219) as one device kernel, `strength = 1`.
Input frames: `vid2vid_frames_uint8` (the decoded video, RGB) and `inpainting_image` (a PIL image, a uint8 array, a path or
an object with `.name`, as the reference receives it) are resized with PIL's LANCZOS and normalised on the device
(`TextToVideoSynthesis.prepare_frames`, bit for bit), once per call for every clip; `vid2vid_frames_tensor` /
`inpainting_image_tensor` ([-1, 1], already at the output size) take precedence when given.  Out of scope by SURVEY.md
section 2 rows 5/12: decoding video files (ffmpeg / cv2) and the LoRA UI.  Packaging: `video_encoder(frames, args) -> str`
is pluggable (the webui's ffmpeg_stitch_video wrapper); the default (video_encode.py) pipes through an `ffmpeg` binary when one exists and otherwise
returns an uncompressed AVI data URL.  `return_frames=True` in `args_dict` returns the raw BGR frame lists instead.
`batch_size` (default 1) groups the `batch_count` clips into batches of that many, each sampled as one batched run
(`infer(batch_size=...)`, clip i of a batch still seeded seed + i).  The encoded vid2vid video is shared by the clips of a
batch (each clip noises it with its own x_T); img2vid blends one start latent per clip, in clip order, as the sequential
loop does.
"""
import ctypes as C
import os
from types import SimpleNamespace

import numpy as np
import torch

from . import _lib
from .key_frames import T2VAnimKeys
from .pipeline import TextToVideoSynthesis
from .video_encode import default_video_encoder

pipe = None
video_encoder = default_video_encoder        # callable(list_of_bgr_frames, args) -> str (data URL)

_DEFAULTS = dict(prompt='', n_prompt='', steps=30, frames=24, seed=-1, cfg_scale=17, width=256, height=256, eta=0.0,
                 batch_count=1, batch_size=1, sampler='DDIM_Gaussian', cpu_vae='GPU (half precision)', keep_pipe_in_vram='None',
                 do_vid2vid=False, vid2vid_startFrame=0, model='<modelscope>', inpainting_frames=0,
                 inpainting_weights='0:(t/max_i_f), "max_i_f":(1)')          # T2VArgs defaults (t2v_helpers/args.py:219-236)


def inpainting_latents(pipe_, image, frames, height, width, inpainting_frames, inpainting_weights, seed, cpu_vae, noise=None):
    """img2vid start latents + mask (process_modelscope.py:170-219).  `image`: [3, H, W] (or [1, 3, 1, H, W]) in [-1, 1].
    The reference tiles the image to `frames` copies and encodes every copy; the VAE is per-frame, so one encode gives the same
    latent.  `latent_noise` comes from numpy's global generator exactly like the reference (np.random.normal, float64)."""
    keys = T2VAnimKeys(SimpleNamespace(max_frames=frames, inpainting_weights=inpainting_weights), seed, inpainting_frames)
    img = torch.as_tensor(image)
    if img.dim() == 3:
        img = img.view(1, 3, 1, *img.shape[1:])
    image_latents = pipe_.compute_latents(img.float(), cpu_vae, torch.device('cuda'))          # [1, 4, 1, h, w] fp32 (CPU)
    lh, lw = height // 8, width // 8
    if tuple(image_latents.shape[-2:]) != (lh, lw):
        raise ValueError(f'inpainting image must be {height}x{width} (latent {lh}x{lw}), got latent {tuple(image_latents.shape[-2:])}')
    latent_noise = np.random.normal(size=(1, 4, frames, lh, lw)) if noise is None else np.asarray(noise, dtype=np.float64)
    weights = np.asarray([keys.inpainting_weights_series[i] for i in range(frames)], dtype=np.float64)
    dev = torch.device('cuda')
    img_d = image_latents.to(dev, torch.float32).contiguous()
    noise_d = torch.from_numpy(latent_noise).to(dev)
    w_d = torch.from_numpy(weights).to(dev)
    out = torch.empty((1, 4, frames, lh, lw), dtype=torch.float64, device=dev)
    mask = torch.empty_like(out)
    _lib.check(_lib.lib().t2v_latent_blend(_lib.ptr(img_d), int(img_d.shape[2]), _lib.ptr(noise_d), _lib.ptr(w_d), _lib.ptr(out),
                                           _lib.ptr(mask), 4, frames, lh * lw, _lib.stream_ptr()), 'latent_blend')
    return out, mask


def process_modelscope(args_dict, extra_args=None):
    """Runs `batch_count` clips.  `args_dict` uses the reference's key names; additionally `model_dir`,
    `prompt_embeds` / `n_prompt_embeds` ([1, L, 1024] tensors) may be given for head-less use."""
    global pipe
    a = SimpleNamespace(**{**_DEFAULTS, **args_dict})
    vid_latents = None
    if getattr(a, 'do_vid2vid', False):
        # The reference decodes the input video with cv2 (vid2frames, process_modelscope.py:101): webui plumbing.  Head-less use
        # passes the decoded frames (uint8 RGB, resized here as the reference resizes them) or a tensor [1, 3, f, H, W] in
        # [-1, 1]; the latent preparation itself (compute_latents, t2v_pipeline.py:148-194) runs on the library.
        if getattr(a, 'vid2vid_frames_tensor', None) is None and getattr(a, 'vid2vid_frames_uint8', None) is None:
            raise NotImplementedError('vid2vid: pass `vid2vid_frames_uint8` (the decoded video, uint8 RGB [f, H, W, 3]) or '
                                      '`vid2vid_frames_tensor` ([1, 3, f, H, W] in [-1, 1]); decoding video files is webui '
                                      'plumbing outside this package')
    model_dir = getattr(a, 'model_dir', None)
    if pipe is None or (model_dir is not None and pipe.model_dir != model_dir):
        pipe = TextToVideoSynthesis(model_dir, **(extra_args or {}))
    pipe.keep_in_vram = a.keep_pipe_in_vram
    prompt = getattr(a, 'prompt_embeds', None)
    n_prompt = getattr(a, 'n_prompt_embeds', None)
    prompt = a.prompt if prompt is None else prompt
    n_prompt = a.n_prompt if n_prompt is None else n_prompt
    outputs = []
    strength = getattr(a, 'strength', 0.0)
    skip_steps = 0
    if getattr(a, 'do_vid2vid', False):
        vid = getattr(a, 'vid2vid_frames_tensor', None)
        if vid is None:                                                                                                    # :101-137
            video = a.vid2vid_frames_uint8
            used = vid2vid_frame_range(len(video), a.vid2vid_startFrame, a.frames)
            vid = pipe.prepare_frames(video[used.start:used.stop], a.width, a.height, a.cpu_vae)
        vid_latents = pipe.compute_latents(vid, a.cpu_vae, torch.device('cuda')).to(torch.device('cuda'))                 # :141
        skip_steps = int(np.floor(a.steps * max(0, min(1 - strength, 1))))                                                  # :143
    else:
        strength = 1                                                                                                       # :146
    keep_frames = getattr(a, 'return_frames', False) or video_encoder is None
    image = getattr(a, 'inpainting_image_tensor', None)
    if a.inpainting_frames > 0 and image is None and getattr(a, 'inpainting_image', None) is not None:                # :172-190
        image = pipe.prepare_frames([load_rgb_image(a.inpainting_image)], a.width, a.height, a.cpu_vae)
    for batch, n in batch_sizes(a.batch_count, a.batch_size):
        seed = a.seed + batch if a.seed != -1 else -1
        latents, mask = vid_latents, None
        if a.inpainting_frames > 0 and image is not None:                                                                  # :170-219
            # the blended latent IS the clip's x_T: one per clip, drawn in clip order as the sequential loop draws them
            blends = [inpainting_latents(pipe, image, a.frames, a.height, a.width, a.inpainting_frames, a.inpainting_weights,
                                         a.seed, a.cpu_vae, getattr(a, 'inpainting_noise', None)) for _ in range(n)]
            latents, mask = torch.cat([b[0] for b in blends]), torch.cat([b[1] for b in blends])
            strength = 1
        args = (prompt, n_prompt, a.steps, a.frames, seed, a.cfg_scale, a.width, a.height, a.eta, a.cpu_vae, torch.device('cuda'),
                latents, skip_steps, strength, mask, bool(getattr(a, 'do_vid2vid', False)), a.sampler)
        clips = [pipe.infer(*args)[0]] if n == 1 else pipe.infer(*args, batch_size=n)[0]
        outputs.extend(frames if keep_frames else video_encoder(frames, a) for frames in clips)
    return outputs


def batch_sizes(batch_count, batch_size):
    """[(index of the batch's first clip, clips in it)]: `batch_count` clips in batches of `batch_size`, the last the rest."""
    if batch_size < 1:
        raise ValueError(f'batch_size must be >= 1, got {batch_size}')
    return [(i, min(batch_size, batch_count - i)) for i in range(0, batch_count, batch_size)]


def vid2vid_frame_range(n_decoded, start, frames):
    """The frames of a decoded video that the reference loads: vid2frames(extract_from_frame=start,
    extract_to_frame=start + frames) keeps frame `count` while count <= extract_to_frame (t2v_helpers/video_audio_utils.py:
    59-73), so frames + 1 of them from `start`, fewer where the video ends."""
    if not 0 <= start < n_decoded:
        raise ValueError(f'vid2vid start frame {start} is outside the {n_decoded} decoded frames')
    return range(start, min(start + frames + 1, n_decoded))


def load_rgb_image(image):
    """The img2vid image as the reference opens it (process_modelscope.py:175): a path, or an object with `.name` (gradio's
    upload), is opened with PIL and converted to RGB, and so is a PIL image; a uint8 array [H, W, 3] is taken as RGB."""
    if isinstance(image, np.ndarray):
        return image
    from PIL import Image
    if isinstance(image, Image.Image):
        return np.asarray(image.convert('RGB'))
    path = image if isinstance(image, (str, os.PathLike)) else image.name
    with Image.open(path) as im:
        return np.asarray(im.convert('RGB'))
