"""GPU: t2v_frames_resize (PIL's LANCZOS resize + the reference's x / 255 * 2 - 1) equals the CPU restatement
(tests/resize_oracle.py, itself pinned bit for bit to Pillow by test_frame_resize_cpu.py) with torch.equal, fp32 and fp16, on
the CPU test's grid; a batch of different frames in one call, host-staged in chunks and from device memory; nothing written
outside the output view and nothing left unwritten inside it.  End to end: process_modelscope's uint8 vid2vid frames and img2vid
image (a PIL image and a path, as the reference opens it) give the same frames as the `*_tensor` inputs built from the
restatement's resized frames, with batch_size = 2."""
import numpy as np
import pytest
import torch

import resize_oracle as R
from oracle import unet_oracle as UO, vae_oracle as VO
from test_frame_resize_cpu import SHAPES, content

pytestmark = pytest.mark.gpu


def expected(frames, w, h, dtype):
    ref = torch.from_numpy(R.normalise(R.resize(frames, w, h)))
    return ref.half() if dtype == torch.float16 else ref


@pytest.mark.parametrize('dtype', [torch.float32, torch.float16])
@pytest.mark.parametrize('h0,w0,h,w', SHAPES)
def test_kernel_matches_restatement(h0, w0, h, w, dtype):
    from t2v_b200 import ops
    frames = np.stack([content('random', h0, w0, seed=7), content('checkerboard', h0, w0)])
    want = expected(frames, w, h, dtype)
    got = ops.frames_resize(frames, w, h, dtype)                                  # host frames, staged
    assert got.shape == (2, 3, h, w) and got.dtype == dtype
    assert torch.equal(got.cpu(), want)
    dev = ops.frames_resize(torch.from_numpy(frames).cuda(), w, h, dtype)        # device frames
    assert torch.equal(dev.cpu(), want)


def test_250_frame_clip_in_one_call():
    """The UI's longest clip at the ZeroScope XL upscale (576x320 -> 1024x576): 250 different frames, uploaded in three chunks
    of the default staging size, as an array and as a list of frames."""
    from t2v_b200 import ops
    rng = np.random.default_rng(11)
    frames = rng.integers(0, 256, (250, 320, 576, 3), dtype=np.uint8)
    frames[::5, ::2, ::2] = 255                    # every fifth frame half saturated: extremes in the same call
    frames[1::5, 1::2, ::2] = 0
    assert ops.STAGING_BYTES // (320 * 576 * 3) < 125
    got = ops.frames_resize(frames, 1024, 576, torch.float16)
    listed = ops.frames_resize(list(frames), 1024, 576, torch.float16)
    assert torch.equal(got, listed)
    for i in range(0, 250, 50):
        assert torch.equal(got[i:i + 50].cpu(), expected(frames[i:i + 50], 1024, 576, torch.float16)), i


@pytest.mark.parametrize('h0,w0,h,w', [(45, 80, 72, 128), (72, 128, 72, 40), (30, 64, 61, 64)])
def test_output_view_written_exactly(h0, w0, h, w):
    """out is a view in the middle of a NaN-filled buffer: its frames are all written, the frames around it untouched."""
    from t2v_b200 import ops
    frames = np.stack([content('random', h0, w0, seed=s) for s in range(5)])
    buf = torch.full((7, 3, h, w), float('nan'), device='cuda')
    ops.frames_resize(frames, w, h, torch.float32, out=buf[1:6], staging_bytes=2 * h0 * w0 * 3)     # chunks of 2, 2, 1
    assert torch.isnan(buf[0]).all() and torch.isnan(buf[6]).all()
    assert torch.equal(buf[1:6].cpu(), expected(frames, w, h, torch.float32))


def test_wrapper_rejects_bad_inputs():
    from t2v_b200 import ops
    with pytest.raises(ValueError, match='uint8 RGB'):
        ops.frames_resize([np.zeros((4, 4, 3), np.uint8), np.zeros((4, 5, 3), np.uint8)], 8, 8)
    with pytest.raises(ValueError, match='uint8 RGB'):
        ops.frames_resize(np.zeros((2, 4, 4, 3), np.float32), 8, 8)
    with pytest.raises(ValueError, match='out must be'):
        ops.frames_resize(np.zeros((2, 4, 4, 3), np.uint8), 8, 8, out=torch.empty((2, 3, 8, 9), device='cuda'))
    with pytest.raises(RuntimeError, match='every size in'):
        ops.frames_resize(np.zeros((1, 4, 4, 3), np.uint8), 0, 8)


# ------------------------------------------------------------------------------------------------ end to end
SIZE = 64


@pytest.fixture(scope='module')
def pipe():
    from t2v_b200.pipeline import TextToVideoSynthesis
    W = UO.make_weights(UO.param_specs(UO.UNetConfig(dim=64)), seed=1)
    Wv = UO.make_weights(VO.decoder_param_specs(VO.VAEConfig()), seed=3)
    p = TextToVideoSynthesis(None, model_cfg={'unet_dim': 64}, unet_state=W, vae_state=Wv)
    p.autoencoder.load_state_dict(UO.make_weights(VO.encoder_param_specs(VO.VAEConfig()), seed=5), strict=False)
    p.autoencoder.cuda()
    return p


def conds():
    g = torch.Generator().manual_seed(2)
    return torch.randn(1, 77, 1024, generator=g).half(), torch.randn(1, 77, 1024, generator=g).half()


def same_clips(a, b):
    return len(a) == len(b) and all(len(x) == len(y) and all(np.array_equal(f, g) for f, g in zip(x, y)) for x, y in zip(a, b))


@pytest.mark.parametrize('batch_size', [1, 2])
def test_vid2vid_uint8_frames_match_the_tensor_input(pipe, batch_size):
    """A 7-frame 80x45 video from frame 2 with frames = 3: the reference loads frames 2..5 (vid2frames' inclusive range),
    resizes them to 64x64 and normalises; the clip has those 4 frames."""
    from t2v_b200 import process_modelscope as pm
    c, uc = conds()
    video = np.random.default_rng(3).integers(0, 256, (7, 45, 80, 3), dtype=np.uint8)
    base = dict(prompt_embeds=c, n_prompt_embeds=uc, steps=8, frames=3, seed=11, cfg_scale=5.0, width=SIZE, height=SIZE,
                sampler='DDIM', return_frames=True, batch_count=2, batch_size=batch_size, do_vid2vid=True, strength=0.5,
                vid2vid_startFrame=2)
    tensor = torch.from_numpy(R.normalise(R.resize(video[2:6], SIZE, SIZE))).permute(1, 0, 2, 3).unsqueeze(0)
    pm.pipe = pipe
    try:
        got = pm.process_modelscope(dict(base, vid2vid_frames_uint8=video))
        want = pm.process_modelscope(dict(base, vid2vid_frames_tensor=tensor))
        listed = pm.process_modelscope(dict(base, vid2vid_frames_uint8=list(video)))
    finally:
        pm.pipe = None
    assert len(got) == 2 and len(got[0]) == 4 and got[0][0].shape == (SIZE, SIZE, 3)
    assert same_clips(got, want) and same_clips(listed, want)


@pytest.mark.parametrize('batch_size', [1, 2])
def test_img2vid_image_matches_the_tensor_input(pipe, batch_size, tmp_path):
    Image = pytest.importorskip('PIL.Image')
    from t2v_b200 import process_modelscope as pm
    c, uc = conds()
    rgb = np.random.default_rng(4).integers(0, 256, (90, 120, 3), dtype=np.uint8)
    path = tmp_path / 'start.png'
    Image.fromarray(rgb).save(path)
    tensor = torch.from_numpy(R.normalise(R.resize(rgb, SIZE, SIZE)))                # [3, H, W] in [-1, 1]
    noise = np.random.RandomState(5).normal(size=(1, 4, 3, 8, 8))
    base = dict(prompt_embeds=c, n_prompt_embeds=uc, steps=4, frames=3, seed=21, cfg_scale=5.0, width=SIZE, height=SIZE,
                sampler='DDIM_Gaussian', return_frames=True, batch_count=2, batch_size=batch_size, inpainting_frames=2,
                inpainting_noise=noise)
    pm.pipe = pipe
    try:
        want = pm.process_modelscope(dict(base, inpainting_image_tensor=tensor))
        as_image = pm.process_modelscope(dict(base, inpainting_image=Image.fromarray(rgb)))
        as_path = pm.process_modelscope(dict(base, inpainting_image=str(path)))
    finally:
        pm.pipe = None
    assert len(want) == 2 and len(want[0]) == 3
    assert same_clips(as_image, want) and same_clips(as_path, want)
