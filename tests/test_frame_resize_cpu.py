"""CPU: the restatement of Pillow's LANCZOS resize (tests/resize_oracle.py) against Pillow itself, the library's coefficient
tables (t2v_resize_coeffs, host only) against the restatement's, t2v_frames_resize's argument checks, and the host logic of
process_modelscope's uint8 inputs: vid2frames' frame range, the image loading, one resize per call."""
import ctypes as C
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import resize_oracle as R
from t2v_b200 import _lib, ops

# (H0, W0, H, W): the ZeroScope XL upscale and 1080p sources, downsampling, 64^2 -> 1024^2, non-integer ratios, one-pixel
# rows and columns, unchanged sizes, and horizontal-only / vertical-only resizes
SHAPES = [(1080, 1920, 576, 1024), (320, 576, 576, 1024), (720, 1280, 256, 256), (64, 64, 1024, 1024), (7, 13, 5, 29),
          (13, 7, 29, 5), (108, 192, 57, 102), (37, 53, 64, 40), (1, 9, 4, 1), (9, 1, 1, 4), (1, 1, 3, 2), (1, 40, 1, 17),
          (24, 1, 7, 1), (50, 50, 50, 50), (40, 40, 40, 17), (33, 64, 64, 64)]


def content(kind, h, w, seed=0):
    if kind == 'random':
        return np.random.default_rng(seed).integers(0, 256, (h, w, 3), dtype=np.uint8)
    board = (np.indices((h, w)).sum(0) % 2 * 255).astype(np.uint8)      # 0/255: the negative lobes clip
    return np.stack([board, 255 - board, board], axis=-1)


@pytest.mark.parametrize('kind', ['random', 'checkerboard'])
@pytest.mark.parametrize('h0,w0,h,w', SHAPES)
def test_restatement_matches_pillow(h0, w0, h, w, kind):
    Image = pytest.importorskip('PIL.Image')
    a = content(kind, h0, w0)
    ref = np.asarray(Image.fromarray(a).resize((w, h), Image.LANCZOS))
    assert np.array_equal(R.resize(a, w, h), ref)


def test_restatement_resizes_a_batch_frame_by_frame():
    a = np.stack([content('random', 19, 23, seed=s) for s in range(3)])
    got = R.resize(a, 31, 11)
    assert got.shape == (3, 11, 31, 3)
    for i in range(3):
        assert np.array_equal(got[i], R.resize(a[i], 31, 11))
    n = R.normalise(got)
    assert n.shape == (3, 3, 11, 31) and n.dtype == np.float32
    assert np.array_equal(n, (np.float32(2) * (got.astype(np.float32) / np.float32(255)) - np.float32(1)).transpose(0, 3, 1, 2))


@pytest.mark.parametrize('n_in,n_out', [(1920, 1024), (576, 1024), (1280, 256), (64, 1024), (7, 29), (13, 5), (1, 4), (9, 1),
                                        (3, 2), (1000, 1), (57, 58)])
def test_library_tables_match_the_restatement(n_in, n_out):
    bounds, coeffs = ops.resize_coeffs(n_in, n_out)
    rb, rk = R.coeffs(n_in, n_out)
    assert np.array_equal(bounds, rb) and np.array_equal(coeffs, rk)
    used = np.arange(coeffs.shape[1])[None, :] < bounds[:, 1:]
    assert np.all(coeffs[~used] == 0)
    assert np.all(np.abs(coeffs.sum(1) - (1 << 22)) <= coeffs.shape[1])        # normalised weights, rounded per tap


def test_unchanged_size_is_the_identity_table():
    bounds, coeffs = ops.resize_coeffs(48, 48)
    assert coeffs.shape == (48, 1) and np.all(coeffs == 1 << 22)
    assert np.array_equal(bounds, np.stack([np.arange(48), np.ones(48)], axis=1))


def test_coeffs_reject_bad_sizes():
    l = _lib.load_library()
    k = C.c_int(0)
    for a, b in [(0, 4), (4, 0), (-1, 4), (32769, 4), (4, 32769)]:
        assert l.t2v_resize_coeffs(a, b, C.byref(k), None, None) == -1
        assert b'resize_coeffs' in l.t2v_last_error()
    assert l.t2v_resize_coeffs(4, 4, None, None, None) == -1
    assert l.t2v_resize_coeffs(32768, 1, C.byref(k), None, None) == 0 and k.value == 2 * 3 * 32768 + 1


def test_frames_resize_rejects_bad_arguments_before_touching_the_device():
    """Every refusal returns -1 with the reason before any CUDA call, so fake device addresses are safe here."""
    l = _lib.load_library()
    src, out, tmp = C.c_void_p(0x10000), C.c_void_p(0x20000), C.c_void_p(0x40000)

    def call(src=src, n=2, h0=32, w0=48, out=out, h=16, w=24, fp16=0, tmp=tmp, tmp_bytes=2 * 32 * 24 * 3):
        rc = l.t2v_frames_resize(src, n, h0, w0, out, h, w, fp16, tmp, tmp_bytes, None)
        return rc, l.t2v_last_error().decode()
    for kw in [dict(n=0), dict(h0=0), dict(w0=0), dict(h=0), dict(w=0), dict(w=32769), dict(h0=40000)]:
        rc, err = call(**kw)
        assert rc == -1 and 'every size in [1, 32768]' in err, (kw, err)
    rc, err = call(src=None)
    assert rc == -1 and 'src and out are required' in err
    rc, err = call(out=None)
    assert rc == -1 and 'src and out are required' in err
    rc, err = call(out=C.c_void_p(0x20002))                       # fp32 out needs 4-byte alignment
    assert rc == -1 and 'aligned to its element size (4 bytes)' in err
    rc, err = call(out=C.c_void_p(0x20001), fp16=1)               # fp16 out needs 2-byte alignment
    assert rc == -1 and 'aligned to its element size (2 bytes)' in err
    rc, err = call(tmp_bytes=2 * 32 * 24 * 3 - 1)
    assert rc == -1 and 'needs a uint8 buffer of 4608 bytes, got 4607' in err
    rc, err = call(tmp=None)
    assert rc == -1 and 'got 0' in err


def vid2frames_kept(n_video, start, frames):
    """Restates the frame loop of vid2frames (t2v_helpers/video_audio_utils.py:59-73) with n = 1: reading starts at
    extract_from_frame, frame `count` is written while count <= extract_to_frame, until the video ends."""
    kept, count, to = [], start, start + frames
    while count < n_video:
        if count <= to:
            kept.append(count)
        count += 1
    return kept


@pytest.mark.parametrize('n_video,start,frames', [(100, 0, 24), (100, 5, 24), (24, 0, 24), (25, 0, 24), (30, 20, 24),
                                                  (3, 2, 1), (1, 0, 1)])
def test_vid2vid_frame_range_is_vid2frames_inclusive_range(n_video, start, frames):
    from t2v_b200.process_modelscope import vid2vid_frame_range
    assert list(vid2vid_frame_range(n_video, start, frames)) == vid2frames_kept(n_video, start, frames)


def test_vid2vid_frame_range_rejects_a_start_past_the_video():
    from t2v_b200.process_modelscope import vid2vid_frame_range
    with pytest.raises(ValueError, match='outside the 10 decoded frames'):
        vid2vid_frame_range(10, 10, 4)
    with pytest.raises(ValueError):
        vid2vid_frame_range(10, -1, 4)


def test_load_rgb_image_takes_what_the_reference_takes(tmp_path):
    Image = pytest.importorskip('PIL.Image')
    from t2v_b200.process_modelscope import load_rgb_image
    rgba = np.random.default_rng(1).integers(0, 256, (6, 5, 4), dtype=np.uint8)
    im = Image.fromarray(rgba, 'RGBA')
    want = np.asarray(im.convert('RGB'))
    path = tmp_path / 'image.png'
    im.save(path)
    assert np.array_equal(load_rgb_image(im), want)
    assert np.array_equal(load_rgb_image(str(path)), want)
    assert np.array_equal(load_rgb_image(path), want)
    assert np.array_equal(load_rgb_image(SimpleNamespace(name=str(path))), want)      # gradio's upload object
    assert load_rgb_image(want) is want


class FakePipe:
    """Records what process_modelscope hands to prepare_frames / compute_latents / infer."""
    model_dir = None

    def __init__(self):
        self.prepared, self.encoded, self.latents = [], [], []

    def prepare_frames(self, frames, width, height, cpu_vae='GPU (half precision)'):
        self.prepared.append((np.asarray(frames), width, height, cpu_vae))
        return torch.full((1, 3, len(frames), height, width), float(len(self.prepared)))

    def compute_latents(self, vd_out, cpu_vae='GPU (half precision)', device=None):
        self.encoded.append(vd_out)
        return torch.zeros((1, 4, vd_out.shape[2], vd_out.shape[3] // 8, vd_out.shape[4] // 8))

    def infer(self, *args, batch_size=1):
        self.latents.append(args[11])
        clips = [['frame'] for _ in range(batch_size)]
        return (clips[0], None, '') if batch_size == 1 else (clips, None, [''] * batch_size)


def run_with(pipe, monkeypatch, **kw):
    from t2v_b200 import process_modelscope as pm
    monkeypatch.setattr(pm, 'pipe', pipe)
    monkeypatch.setattr(torch.Tensor, 'to', lambda self, *a, **k: self)        # no device here
    args = dict(prompt_embeds=1, n_prompt_embeds=2, seed=3, width=16, height=8, frames=4, return_frames=True, **kw)
    return pm.process_modelscope(args)


def test_vid2vid_uint8_frames_are_prepared_once_from_the_inclusive_range(monkeypatch):
    video = np.arange(10, dtype=np.uint8)[:, None, None, None] * np.ones((10, 5, 7, 3), dtype=np.uint8)
    pipe = FakePipe()
    out = run_with(pipe, monkeypatch, do_vid2vid=True, vid2vid_frames_uint8=video, vid2vid_startFrame=2, strength=0.5,
                   batch_count=3, batch_size=2)
    assert len(out) == 3 and len(pipe.prepared) == 1 and len(pipe.encoded) == 1
    frames, w, h, vae = pipe.prepared[0]
    assert [int(f[0, 0, 0]) for f in frames] == [2, 3, 4, 5, 6] and (w, h) == (16, 8) and vae == 'GPU (half precision)'
    assert pipe.encoded[0].shape == (1, 3, 5, 8, 16)
    assert all(lat.shape[2] == 5 for lat in pipe.latents)          # the clip has its input's frames, as the reference's
    # a list of frames is sliced the same way; the tensor key takes precedence
    pipe = FakePipe()
    run_with(pipe, monkeypatch, do_vid2vid=True, vid2vid_frames_uint8=list(video), strength=0.5)
    assert [int(f[0, 0, 0]) for f in pipe.prepared[0][0]] == [0, 1, 2, 3, 4]
    pipe = FakePipe()
    given = torch.zeros((1, 3, 4, 8, 16))
    run_with(pipe, monkeypatch, do_vid2vid=True, vid2vid_frames_uint8=video, vid2vid_frames_tensor=given, strength=0.5)
    assert pipe.prepared == [] and pipe.encoded[0] is given
    with pytest.raises(NotImplementedError):
        run_with(FakePipe(), monkeypatch, do_vid2vid=True)


def test_inpainting_image_is_prepared_once_per_call(monkeypatch):
    from t2v_b200 import process_modelscope as pm
    blended = []
    monkeypatch.setattr(pm, 'inpainting_latents', lambda p, image, *a: (blended.append(image), (torch.zeros(1), torch.zeros(1)))[1])
    img = np.random.default_rng(2).integers(0, 256, (12, 9, 3), dtype=np.uint8)
    pipe = FakePipe()
    run_with(pipe, monkeypatch, inpainting_frames=2, inpainting_image=img, batch_count=3, batch_size=2)
    assert len(pipe.prepared) == 1 and np.array_equal(pipe.prepared[0][0], img[None])
    assert len(blended) == 3 and all(b is blended[0] for b in blended) and blended[0].shape == (1, 3, 1, 8, 16)
    blended.clear()
    given = torch.zeros((3, 8, 16))
    pipe = FakePipe()
    run_with(pipe, monkeypatch, inpainting_frames=2, inpainting_image=img, inpainting_image_tensor=given)
    assert pipe.prepared == [] and blended == [given]
    blended.clear()
    pipe = FakePipe()
    run_with(pipe, monkeypatch, inpainting_frames=0, inpainting_image=img)          # no inpainting frames: the image is unused
    assert pipe.prepared == [] and blended == []
