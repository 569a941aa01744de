"""Thin Python wrappers over the kernel-level C entry points (t2v_op_*).  Used by the parity tests and by
small host-side utilities (q_sample_blend also by the VideoCrafter sampler's masked mode); the model-level path
(t2v_unet_forward / t2v_vae_decode) does not go through here.

All tensors are CUDA fp16, channels-last token matrices [rows, C] unless stated otherwise.
"""
import ctypes as C

import numpy as np
import torch

from . import _lib

GEMM_GEGLU = 1
GEMM_FORCE_BS, GEMM_NO_BS = 2048, 4096      # bring-up switches of t2v_op_gemm: B-stationary variant on / off
GEMM_OUT_F32 = 2
GEMM_SLAB_OUT = 8192      # test switch of t2v_op_gemm: per-warp slab stores even where the TMA-store epilogue applies


def _ia(vals):
    return (C.c_int * len(vals))(*[int(v) for v in vals])


def gemm(a, w_packed, N, *, K=None, lda=None, dims=None, taps=None, n_alloc=None, b_batch_dim=-1, flags=0, out=None,
         ldo=None, bias=None, bias_rows=0, bias_stride=0, residual=None, ldr=None, alpha=1.0, force_bn=0, force_cg=0):
    """out[row, n] = alpha * sum_tap sum_k a[row + tap, k] w[tap, n, k] (+bias) (+residual)."""
    l = _lib.lib()
    rows = a.shape[0]
    K = K if K is not None else a.shape[1]
    lda = lda if lda is not None else a.stride(0)
    dims = list(dims) if dims is not None else [rows]
    nd = len(dims)
    taps = taps if taps is not None else [[0] * nd]
    flat = [o for t in taps for o in t]
    n_alloc = n_alloc if n_alloc is not None else w_packed.shape[-2]
    ncols = N // 2 if (flags & GEMM_GEGLU) else N
    if out is None:
        out = torch.empty((rows, ncols), device=a.device, dtype=torch.float32 if (flags & GEMM_OUT_F32) else torch.float16)
    ldo = ldo if ldo is not None else out.stride(0)
    ldr = ldr if ldr is not None else (residual.stride(0) if residual is not None else 0)
    rc = l.t2v_op_gemm(_lib.ptr(a), lda, K, nd, _ia(dims), len(taps), _ia(flat), _lib.ptr(w_packed), n_alloc, N,
                       b_batch_dim, flags, _lib.ptr(out), ldo, _lib.ptr(bias), bias_rows, bias_stride,
                       _lib.ptr(residual), ldr, alpha, force_bn, force_cg, _lib.stream_ptr())
    _lib.check(rc, 'op_gemm')
    return out


def gemm_splitk(a, w_packed, N, splits, *, scratch=None, K=None, lda=None, dims=None, taps=None, n_alloc=None, b_batch_dim=-1,
                flags=0, out=None, ldo=None, bias=None, bias_rows=0, bias_stride=0, residual=None, ldr=None, alpha=1.0,
                force_bn=0, force_cg=0):
    """gemm's problem through split-K (fp32 partials per split, then a fix-up pass adding bias and residual).
    scratch: fp32 CUDA tensor, by default [splits, rows, N].  Returns (out, number of splits run)."""
    l = _lib.lib()
    rows = a.shape[0]
    K = K if K is not None else a.shape[1]
    lda = lda if lda is not None else a.stride(0)
    dims = list(dims) if dims is not None else [rows]
    taps = taps if taps is not None else [[0] * len(dims)]
    flat = [o for t in taps for o in t]
    n_alloc = n_alloc if n_alloc is not None else w_packed.shape[-2]
    if out is None:
        out = torch.empty((rows, N), device=a.device, dtype=torch.float16)
    if scratch is None:
        scratch = torch.empty((max(splits, 1), rows, N), device=a.device, dtype=torch.float32)
    ldo = ldo if ldo is not None else out.stride(0)
    ldr = ldr if ldr is not None else (residual.stride(0) if residual is not None else 0)
    used = C.c_int(0)
    rc = l.t2v_op_gemm_splitk(_lib.ptr(a), lda, K, len(dims), _ia(dims), len(taps), _ia(flat), _lib.ptr(w_packed), n_alloc, N,
                              b_batch_dim, flags, _lib.ptr(out), ldo, _lib.ptr(bias), bias_rows, bias_stride,
                              _lib.ptr(residual), ldr, alpha, splits, _lib.ptr(scratch), scratch.numel(), C.byref(used),
                              force_bn, force_cg, _lib.stream_ptr())
    _lib.check(rc, 'op_gemm_splitk')
    return out, used.value


def ln_linear(x, w, bias, gamma, beta, *, flags=0, residual=None, out=None, force_bn=0, force_cg=0):
    """Linear(LayerNorm(x)) (eps 1e-5) with the LayerNorm folded into the GEMM epilogue.  w [N, K] (GEGLU-packed with
    flags=GEMM_GEGLU).  Returns (out, w_folded [N, K] fp16, colsum [N] fp32, bias32 [N] fp32, rowstat [rows, 2] fp32)."""
    l = _lib.lib()
    rows, K = x.shape
    w = w.reshape(-1, K)
    N = w.shape[0]
    ncols = N // 2 if (flags & GEMM_GEGLU) else N
    if out is None:
        out = torch.empty((rows, ncols), device=x.device, dtype=torch.float16)
    wf = torch.empty((N, K), device=x.device, dtype=torch.float16)
    colsum = torch.empty((N,), device=x.device, dtype=torch.float32)
    bias32 = torch.empty((N,), device=x.device, dtype=torch.float32)
    rowstat = torch.empty((rows, 2), device=x.device, dtype=torch.float32)
    rc = l.t2v_op_ln_linear(_lib.ptr(x), x.stride(0), rows, K, _lib.ptr(w), _lib.ptr(bias), _lib.ptr(gamma), _lib.ptr(beta), N,
                            flags, _lib.ptr(wf), _lib.ptr(colsum), _lib.ptr(bias32), _lib.ptr(rowstat), _lib.ptr(residual),
                            residual.stride(0) if residual is not None else 0, _lib.ptr(out), out.stride(0), force_bn, force_cg,
                            _lib.stream_ptr())
    _lib.check(rc, 'op_ln_linear')
    return out, wf, colsum, bias32, rowstat


def upsample2x(x):
    """Nearest 2x upsampling of frames x [nframes, h, w, C] -> [nframes, 2h, 2w, C]."""
    l = _lib.lib()
    nf, h, w, Cc = x.shape
    y = torch.empty((nf, 2 * h, 2 * w, Cc), device=x.device, dtype=torch.float16)
    _lib.check(l.t2v_op_upsample2x(_lib.ptr(x), _lib.ptr(y), nf, h, w, Cc, _lib.stream_ptr()), 'op_upsample2x')
    return y


def im2col_s2(x, pad_lo=1, out=None):
    """Stride-2 3x3 gather: x [nframes, h, w, C] -> [nframes, ho, wo, 9 * C], column tap * C + c with tap = ky * 3 + kx.
    pad_lo = 1: padding 1, ho = ceil(h/2); pad_lo = 0: the ldm Downsample's pad (0,1,0,1), ho = floor(h/2)."""
    l = _lib.lib()
    nf, h, w, Cc = x.shape
    ho, wo = ((h + 1) // 2, (w + 1) // 2) if pad_lo else (h // 2, w // 2)
    col = torch.empty((nf, ho, wo, 9 * Cc), device=x.device, dtype=torch.float16) if out is None else out
    _lib.check(l.t2v_op_im2col_s2(_lib.ptr(x), _lib.ptr(col), nf, h, w, Cc, pad_lo, _lib.stream_ptr()), 'op_im2col_s2')
    return col


def ingest_latent(x, tok, cpad, frame0=0, nframes=None, scale=1.0):
    """Frames [frame0, frame0 + nframes) in (b f) order of the latent x [B, C, F, h, w] (fp32 or fp16, contiguous) into the
    rows of tok [nframes*h*w, ld] fp16 (a row-strided view is fine): fp16(x * scale), columns C..cpad-1 zeroed."""
    l = _lib.lib()
    B, Cc, Fr, h, w = x.shape
    nframes = B * Fr - frame0 if nframes is None else nframes
    rc = l.t2v_op_ingest_latent(_lib.ptr(x), int(x.dtype == torch.float32), _lib.ptr(tok), tok.stride(0), cpad, Cc, Fr, h, w,
                                frame0, nframes, scale, _lib.stream_ptr())
    _lib.check(rc, 'op_ingest_latent')
    return tok


def egress_latent(tok, out):
    """Token rows tok [B*F*h*w, ld] fp16 -> out [B, C, F, h, w] (fp32 or fp16, contiguous)."""
    l = _lib.lib()
    B, Cc, Fr, h, w = out.shape
    rc = l.t2v_op_egress_latent(_lib.ptr(tok), tok.stride(0), _lib.ptr(out), int(out.dtype == torch.float32), B, Cc, Fr, h, w,
                                _lib.stream_ptr())
    _lib.check(rc, 'op_egress_latent')
    return out


def avgpool2x2(x, out=None):
    """nn.AvgPool2d(2, 2) of frames x [nframes, h, w, C] -> [nframes, h // 2, w // 2, C] (fp32 sum, one fp16 rounding)."""
    l = _lib.lib()
    nf, h, w, Cc = x.shape
    y = torch.empty((nf, h // 2, w // 2, Cc), device=x.device, dtype=torch.float16) if out is None else out
    _lib.check(l.t2v_op_avgpool2x2(_lib.ptr(x), _lib.ptr(y), nf, h, w, Cc, _lib.stream_ptr()), 'op_avgpool2x2')
    return y


def pixel_unshuffle(x, out=None):
    """nn.PixelUnshuffle(8) of x [N, Cc, H, W] (fp32 or fp16, contiguous) as tokens [N * H/8 * W/8, 64 * Cc] fp16."""
    l = _lib.lib()
    N, Cc, H, W = x.shape
    tok = torch.empty((N * (H // 8) * (W // 8), 64 * Cc), device=x.device, dtype=torch.float16) if out is None else out
    rc = l.t2v_op_pixel_unshuffle(_lib.ptr(x), int(x.dtype == torch.float32), _lib.ptr(tok), N, Cc, H, W, _lib.stream_ptr())
    _lib.check(rc, 'op_pixel_unshuffle')
    return tok


def relu_(x):
    """nn.ReLU in place on a dense fp16 matrix x [rows, C]."""
    l = _lib.lib()
    _lib.check(l.t2v_op_relu(_lib.ptr(x), x.shape[0], x.shape[1], _lib.stream_ptr()), 'op_relu')
    return x


def feature_add_(x, f, rows_per_sample, f_samples):
    """x[r] += f[(r // rows_per_sample % f_samples) * rows_per_sample + r % rows_per_sample] in place (fp32 add, one rounding);
    x [rows, C] may be a row-strided view, f is dense [f_samples * rows_per_sample, C]."""
    l = _lib.lib()
    rows, Cc = x.shape
    rc = l.t2v_op_feature_add(_lib.ptr(x), x.stride(0), _lib.ptr(f), Cc, rows, rows_per_sample, f_samples, _lib.stream_ptr())
    _lib.check(rc, 'op_feature_add')
    return x


def concat_cols(a, b, out):
    """out[:, :Ca + Cb] = a | b for row-strided fp16 matrices a [rows, Ca], b [rows, Cb], out [rows, >= Ca + Cb]."""
    l = _lib.lib()
    rc = l.t2v_op_concat_cols(_lib.ptr(a), a.stride(0), a.shape[1], _lib.ptr(b), b.stride(0), b.shape[1], _lib.ptr(out),
                              out.stride(0), a.shape[0], _lib.stream_ptr())
    _lib.check(rc, 'op_concat_cols')
    return out


def softmax_rows(x, scale, out=None):
    """Row softmax of fp16(x * scale) for a dense fp16 matrix x [rows, cols]."""
    l = _lib.lib()
    y = torch.empty_like(x) if out is None else out
    _lib.check(l.t2v_op_softmax_rows(_lib.ptr(x), _lib.ptr(y), x.shape[0], x.shape[1], scale, _lib.stream_ptr()), 'op_softmax_rows')
    return y


def transpose_batched(x, out=None):
    """x [nb, R, C] fp16 (contiguous) -> [nb, C, R]."""
    l = _lib.lib()
    nb, R, Cc = x.shape
    y = torch.empty((nb, Cc, R), device=x.device, dtype=torch.float16) if out is None else out
    _lib.check(l.t2v_op_transpose_batched(_lib.ptr(x), _lib.ptr(y), nb, R, Cc, _lib.stream_ptr()), 'op_transpose_batched')
    return y


def frames_to_u8(tok, out=None):
    """Decoded frames tok [pixels, ld] fp16 (RGB in columns 0..2, a row-strided view is fine) -> uint8 [pixels, 3]."""
    l = _lib.lib()
    px = tok.shape[0]
    out = torch.empty((px, 3), device=tok.device, dtype=torch.uint8) if out is None else out
    _lib.check(l.t2v_op_frames_to_u8(_lib.ptr(tok), tok.stride(0), _lib.ptr(out), px, _lib.stream_ptr()), 'op_frames_to_u8')
    return out


def frames_to_f32(tok, n, H, W, out=None):
    """Decoded frames tok [n*H*W, ld] fp16 (RGB in columns 0..2) -> fp32 [n, 3, H, W]."""
    l = _lib.lib()
    out = torch.empty((n, 3, H, W), device=tok.device, dtype=torch.float32) if out is None else out
    _lib.check(l.t2v_op_frames_to_f32(_lib.ptr(tok), tok.stride(0), _lib.ptr(out), n, H, W, _lib.stream_ptr()), 'op_frames_to_f32')
    return out


def convert_to_f16(src, out=None):
    """Contiguous fp32 or fp16 CUDA tensor -> fp16 of the same shape (round to nearest even)."""
    l = _lib.lib()
    out = torch.empty(src.shape, device=src.device, dtype=torch.float16) if out is None else out
    rc = l.t2v_op_convert_to_f16(_lib.ptr(src), int(src.dtype == torch.float32), _lib.ptr(out), src.numel(), _lib.stream_ptr())
    _lib.check(rc, 'op_convert_to_f16')
    return out


def time_sinusoid(t, dim):
    """Timestep embedding [cos(t f_k) | sin(t f_k)], f_k = 10000^(-k / (dim // 2)), fp16 [B, dim] (odd dim: last column 0).
    t: fp32 CUDA [B]."""
    l = _lib.lib()
    out = torch.empty((t.numel(), dim), device=t.device, dtype=torch.float16)
    _lib.check(l.t2v_op_time_sinusoid(_lib.ptr(t), _lib.ptr(out), t.numel(), dim, _lib.stream_ptr()), 'op_time_sinusoid')
    return out


def small_linear(x, w, bias=None, addend=None, silu_in=False):
    """y = fp16(fp16(act(x) @ w^T + bias) + addend) for a few rows x [B, K], w [N, K]; act = SiLU rounded to fp16 when
    silu_in.  Accumulation in fp32."""
    l = _lib.lib()
    B, K = x.shape
    N = w.shape[0]
    y = torch.empty((B, N), device=x.device, dtype=torch.float16)
    rc = l.t2v_op_small_linear(_lib.ptr(x), x.stride(0), _lib.ptr(w), _lib.ptr(bias), _lib.ptr(addend), _lib.ptr(y), y.stride(0),
                               B, N, K, int(silu_in), _lib.stream_ptr())
    _lib.check(rc, 'op_small_linear')
    return y


def pack_conv_weight(w, n_alloc=None, k_alloc=None):
    """w [Cout, Cin, *k] (fp16/fp32, CUDA) -> [taps, n_alloc, k_alloc] fp16."""
    l = _lib.lib()
    w = w.contiguous()
    cout, cin = w.shape[0], w.shape[1]
    taps = 1
    for s in w.shape[2:]:
        taps *= s
    n_alloc = n_alloc or cout
    k_alloc = k_alloc or cin
    dst = torch.empty((taps, n_alloc, k_alloc), device=w.device, dtype=torch.float16)
    rc = l.t2v_op_pack_conv_weight(_lib.ptr(w), int(w.dtype == torch.float32), _lib.ptr(dst), cout, cin, taps, n_alloc,
                                   k_alloc, _lib.stream_ptr())
    _lib.check(rc, 'pack_conv_weight')
    return dst


def pack_geglu_weight(w, b, bn):
    l = _lib.lib()
    w = w.contiguous()
    H = w.shape[0] // 2
    K = w.shape[1]
    wd = torch.empty((1, 2 * H, K), device=w.device, dtype=torch.float16)
    bd = torch.empty((2 * H,), device=w.device, dtype=torch.float16)
    rc = l.t2v_op_pack_geglu_weight(_lib.ptr(w), _lib.ptr(b.contiguous()), int(w.dtype == torch.float32), _lib.ptr(wd),
                                    _lib.ptr(bd), H, K, bn, _lib.stream_ptr())
    _lib.check(rc, 'pack_geglu_weight')
    return wd, bd


def _lora_target(w, out, cols):
    if w.dtype != torch.float16 or not w.is_contiguous():
        raise ValueError('the LoRA target must be a contiguous fp16 tensor (it is updated in place)')
    out = w.shape[0] if out is None else out
    return out, (w.numel() // max(out, 1) if cols is None else cols)


def lora_merge_(w, A, B, alpha, temporal_mean=False, out=None, cols=None):
    """In place: w [out, cols] = fp16(w + fp16(fp16(B @ A) * alpha)), the Stable-LoRA merge of t2v_unet_lora_merge.
    A [rank, cols] (x3 columns with temporal_mean), B [out, rank] fp16.  out / cols default to w's first dimension and
    the rest; given, only the first out * cols elements of w are written."""
    out, cols = _lora_target(w, out, cols)
    A, B = A.to(torch.float16).contiguous(), B.to(torch.float16).contiguous()
    rc = _lib.lib().t2v_op_lora_merge(_lib.ptr(w), _lib.ptr(A), _lib.ptr(B), out, cols, A.shape[0], float(alpha),
                                      int(temporal_mean), _lib.stream_ptr())
    _lib.check(rc, 'op_lora_merge')
    return w


def lora_apply_(w, up, down, alpha, out=None, cols=None):
    """In place: w [out, cols] = fp16(w + alpha * up @ down) in fp32, the VideoCrafter merge of t2v_*_lora_apply.
    up [out, rank], down [rank, cols]: fp32 when either is, else fp16."""
    out, cols = _lora_target(w, out, cols)
    dt = torch.float16 if up.dtype == down.dtype == torch.float16 else torch.float32
    up, down = up.to(dt).contiguous(), down.to(dt).contiguous()
    rc = _lib.lib().t2v_op_lora_apply(_lib.ptr(w), _lib.ptr(up), _lib.ptr(down), int(dt == torch.float32), out, cols,
                                      up.shape[1], float(alpha), _lib.stream_ptr())
    _lib.check(rc, 'op_lora_apply')
    return w


def conv_taps_2d():
    """tap = ky*3+kx over row dims (w, h, frames)."""
    return [[kx - 1, ky - 1, 0] for ky in range(3) for kx in range(3)]


def conv_taps_temporal():
    """tap = kt over row dims (pixels, frames, samples)."""
    return [[0, kt - 1, 0] for kt in range(3)]


def groupnorm(x, gamma, beta, rows_per_inst, eps, silu, phase=0, stats=None, out=None):
    """GroupNorm (32 groups, + SiLU) over instances of rows_per_inst consecutive rows of x [rows, C] (a row-strided view
    is fine).  phase 0: the model's single-GPU path, returns y.  phase 1: statistics only (the frame-sharded plans'
    chunking), returns (mean, rstd) per (instance, group), fp32 [rows // rows_per_inst, 32, 2].  phase 2: apply only with
    the given `stats` in that layout, returns y.  `out`: where y goes (by default a new dense [rows, C])."""
    l = _lib.lib()
    n_inst = x.shape[0] // rows_per_inst if rows_per_inst > 0 else 0
    if phase == 1:
        stats = torch.empty((n_inst, 32, 2), device=x.device, dtype=torch.float32) if stats is None else stats
    elif phase == 2 and (stats is None or stats.dtype != torch.float32 or not stats.is_contiguous()
                         or stats.numel() != n_inst * 64):
        raise ValueError('groupnorm: phase 2 needs contiguous fp32 stats [rows // rows_per_inst, 32, 2]')
    y = out if out is not None else torch.empty(x.shape, device=x.device, dtype=x.dtype)
    rc = l.t2v_op_groupnorm(_lib.ptr(x), x.stride(0), _lib.ptr(y), y.stride(0), x.shape[0], x.shape[1], rows_per_inst,
                            _lib.ptr(gamma), _lib.ptr(beta), eps, int(silu), phase, _lib.ptr(stats), _lib.stream_ptr())
    _lib.check(rc, 'op_groupnorm')
    return stats if phase == 1 else y


def layernorm(x, gamma, beta, eps=1e-5, out=None):
    """LayerNorm over the C columns of every row of x [rows, C] (a row-strided view is fine) -> `out` or a new dense matrix."""
    l = _lib.lib()
    y = out if out is not None else torch.empty(x.shape, device=x.device, dtype=x.dtype)
    rc = l.t2v_op_layernorm(_lib.ptr(x), x.stride(0), _lib.ptr(y), y.stride(0), x.shape[0], x.shape[1], _lib.ptr(gamma),
                            _lib.ptr(beta), eps, _lib.stream_ptr())
    _lib.check(rc, 'op_layernorm')
    return y


def attention(q, k, v, o, q_bs, q_ss, k_bs, k_ss, v_bs, v_ss, o_bs, o_ss, batch, heads, sq, skv, kv_batch_div=1,
              scale=0.125):
    l = _lib.lib()
    rc = l.t2v_op_attention(_lib.ptr(q), _lib.ptr(k), _lib.ptr(v), _lib.ptr(o), q_bs, q_ss, k_bs, k_ss, v_bs, v_ss, o_bs,
                            o_ss, batch, heads, sq, skv, kv_batch_div, scale, _lib.stream_ptr())
    _lib.check(rc, 'op_attention')
    return o


def attention_hd(q, k, v, o, q_bs, q_ss, k_bs, k_ss, v_bs, v_ss, o_bs, o_ss, batch, heads, head_dim, sq, skv, kv_batch_div=1,
                 scale=None, *, b_inner=1, q_bsi=0, k_bsi=0, v_bsi=0, o_bsi=0):
    """softmax(QK^T * scale)V for any supported head_dim (head h at column h*head_dim of the token matrices).
    Two-level batch: batch index b -> (b // b_inner) * X_bs + (b % b_inner) * X_bsi (K / V after the kv_batch_div division)."""
    l = _lib.lib()
    scale = head_dim ** -0.5 if scale is None else scale
    rc = l.t2v_op_attention_hd(_lib.ptr(q), _lib.ptr(k), _lib.ptr(v), _lib.ptr(o), q_bs, q_ss, k_bs, k_ss, v_bs, v_ss, o_bs,
                               o_ss, batch, heads, head_dim, sq, skv, kv_batch_div, scale, b_inner, q_bsi, k_bsi, v_bsi, o_bsi,
                               _lib.stream_ptr())
    _lib.check(rc, 'op_attention_hd')
    return o


def clip_attention(qkv, L, heads, o=None):
    """Causal self-attention of the CLIP text towers: qkv [B*L, 3W] (q | k | v, head width 64) -> o [B*L, W]."""
    l = _lib.lib()
    rows, W3 = qkv.shape
    W = W3 // 3
    if o is None:
        o = torch.empty((rows, W), device=qkv.device, dtype=torch.float16)
    if not (qkv.is_contiguous() and o.is_contiguous()) or W3 != 3 * W or rows % L != 0 or tuple(o.shape) != (rows, W):
        raise ValueError('clip_attention: qkv must be a dense [B*L, 3W] matrix and o a dense [B*L, W] one')
    rc = l.t2v_op_clip_attention(_lib.ptr(qkv), _lib.ptr(o), rows // L, L, W, heads, _lib.stream_ptr())
    _lib.check(rc, 'op_clip_attention')
    return o


def abs_quantile(x, q, out=None, workspace=None):
    """torch.quantile(x.abs(), q, dim=1) of an fp32 CUDA tensor x [B, n] (t2v_abs_quantile), bit for bit, by an exact radix
    select: no sort and no host synchronisation.  NaN for a row holding a NaN; RuntimeError for a row above 2^24 elements.
    `workspace`: a CUDA uint8 tensor of at least t2v_abs_quantile_workspace(B) bytes (allocated when None)."""
    l = _lib.lib()
    if x.dim() != 2 or x.dtype != torch.float32 or not x.is_cuda:
        raise TypeError('abs_quantile: x must be a 2-D fp32 CUDA tensor [B, n]')
    x = x.contiguous()
    B = x.shape[0]
    out = torch.empty(B, device=x.device, dtype=torch.float32) if out is None else out
    if workspace is None:
        workspace = torch.empty(l.t2v_abs_quantile_workspace(B), device=x.device, dtype=torch.uint8)
    rc = l.t2v_abs_quantile(_lib.ptr(x), B, x.shape[1], float(q), _lib.ptr(out), _lib.ptr(workspace), workspace.numel(),
                            _lib.stream_ptr())
    _lib.check(rc, 'abs_quantile')
    return out


def q_sample_blend(x0, noise, a, s, mask=None, img=None, out=None):
    """t2v_q_sample_blend on fp32 CUDA tensors: a[b] * x0 + s[b] * noise (q_sample), or, with `mask` and `img`,
    that * mask + (1 - mask) * img (the masked-DDIM blend), rounded as torch's fp32 ops.  The output has img's shape
    ([B, C, T, h, w]; x0's without img); x0, noise and mask broadcast to it as torch broadcasts.  a, s: [B] fp32.
    `out` may be `img` (in place)."""
    l = _lib.lib()
    shape = tuple((img if img is not None else x0).shape)
    if len(shape) != 5:
        raise ValueError(f'q_sample_blend: the latent must be 5-D [B, C, T, h, w], got {list(shape)}')
    if img is not None:
        img = img.contiguous()
    out = torch.empty(shape, device=x0.device, dtype=torch.float32) if out is None else out
    if not out.is_contiguous() or tuple(out.shape) != shape:
        raise ValueError('q_sample_blend: out must be contiguous with the output shape')
    if a.numel() != shape[0] or s.numel() != shape[0]:
        raise ValueError(f'q_sample_blend: a and s need one coefficient per sample ({shape[0]})')
    ts = [t for t in (x0, noise, a, s, mask, img, out) if t is not None]
    if any(t.dtype != torch.float32 or not t.is_cuda for t in ts):
        raise TypeError('q_sample_blend: every tensor must be fp32 on the GPU')

    def view(t):                                        # (tensor, strides): expand gives stride 0 on broadcast dimensions
        e = t.expand(shape)
        return e, (C.c_longlong * 5)(*e.stride())
    x0e, xs = view(x0)
    ne, ns = view(noise)
    me, ms = view(mask) if mask is not None else (None, None)
    a, s = a.contiguous(), s.contiguous()
    rc = l.t2v_q_sample_blend(_lib.ptr(x0e), xs, _lib.ptr(ne), ns, _lib.ptr(a), _lib.ptr(s), _lib.ptr(me), ms, _lib.ptr(img),
                              _lib.ptr(out), _ia(shape), _lib.stream_ptr())
    _lib.check(rc, 'q_sample_blend')
    return out


def attention_relpos(q, k, v, o, table_k, table_v, n_seq, seq_inner, bs_outer, bs_inner, ss, o_bs_outer, o_bs_inner, o_ss,
                     heads, head_dim, T, max_rel, scale=None):
    """Temporal self-attention with relative-position key / value tables (VideoCrafter TemporalCrossAttention)."""
    l = _lib.lib()
    scale = head_dim ** -0.5 if scale is None else scale
    rc = l.t2v_op_attention_relpos(_lib.ptr(q), _lib.ptr(k), _lib.ptr(v), _lib.ptr(o), _lib.ptr(table_k), _lib.ptr(table_v),
                                   n_seq, seq_inner, bs_outer, bs_inner, ss, o_bs_outer, o_bs_inner, o_ss, heads, head_dim, T,
                                   max_rel, scale, _lib.stream_ptr())
    _lib.check(rc, 'op_attention_relpos')
    return o


def resize_coeffs(in_size, out_size):
    """t2v_resize_coeffs (host only, no GPU needed): Pillow's LANCZOS tables for in_size -> out_size pixels as numpy int32
    bounds [out_size, 2] (first input pixel, taps used) and coeffs [out_size, ksize] (22 fractional bits)."""
    l = _lib.load_library()
    k = C.c_int(0)
    _lib.check(l.t2v_resize_coeffs(in_size, out_size, C.byref(k), None, None), 'resize_coeffs')
    bounds = np.zeros((out_size, 2), dtype=np.int32)
    coeffs = np.zeros((out_size, k.value), dtype=np.int32)
    _lib.check(l.t2v_resize_coeffs(in_size, out_size, C.byref(k), bounds.ctypes.data_as(C.c_void_p),
                                   coeffs.ctypes.data_as(C.c_void_p)), 'resize_coeffs')
    return bounds, coeffs


STAGING_BYTES = 64 << 20      # host frames go to the device in chunks of about this many bytes


def frames_resize(frames, width, height, dtype=torch.float32, out=None, staging_bytes=STAGING_BYTES):
    """PIL's Image.resize((width, height), Image.LANCZOS) of uint8 RGB frames, then the reference's x / 255 * 2 - 1, bit for
    bit (t2v_frames_resize) -> [n, 3, height, width] fp32 or fp16 on the current device, or into `out` (a contiguous CUDA
    tensor of that shape and dtype).  `frames`: a uint8 CUDA tensor [n, H0, W0, 3], or host frames -- an array
    [n, H0, W0, 3] or a sequence of [H0, W0, 3] arrays or RGB PIL images -- copied to the device in chunks of about
    `staging_bytes` through two pinned buffers, so a long high-resolution clip never has its whole uint8 copy on the device
    and the host copy of one chunk overlaps the device's work on the previous one."""
    l = _lib.lib()
    if dtype not in (torch.float32, torch.float16):
        raise TypeError(f'frames_resize: dtype must be torch.float32 or torch.float16, got {dtype}')
    n = len(frames)
    if n == 0:
        raise ValueError('frames_resize: no frames')
    on_device = torch.is_tensor(frames) and frames.is_cuda
    if on_device:
        if frames.dtype != torch.uint8 or frames.dim() != 4 or frames.shape[3] != 3:
            raise ValueError(f'frames_resize: device frames must be uint8 [n, H, W, 3], got {frames.dtype} {list(frames.shape)}')
        H0, W0 = frames.shape[1], frames.shape[2]
    else:
        H0, W0 = _host_frame(frames[0], None).shape[:2]
    dev = frames.device if on_device else torch.device('cuda', torch.cuda.current_device())
    if out is None:
        out = torch.empty((n, 3, height, width), device=dev, dtype=dtype)
    if tuple(out.shape) != (n, 3, height, width) or out.dtype != dtype or not out.is_contiguous() or out.device != dev:
        raise ValueError(f'frames_resize: out must be a contiguous {dtype} tensor [{n}, 3, {height}, {width}] on {dev}')
    chunk = n if on_device else max(1, min(n, staging_bytes // (H0 * W0 * 3)))
    tmp = torch.empty((chunk * H0 * width * 3,), device=dev, dtype=torch.uint8) if width != W0 else None

    def launch(src, i0, k):
        rc = l.t2v_frames_resize(_lib.ptr(src), k, H0, W0, _lib.ptr(out[i0]), height, width, int(dtype == torch.float16),
                                 _lib.ptr(tmp), tmp.numel() if tmp is not None else 0, _lib.stream_ptr())
        _lib.check(rc, 'frames_resize')

    if on_device:
        launch(frames.contiguous(), 0, n)
        return out
    stream = torch.cuda.current_stream(dev)
    nbuf = 1 if chunk == n else 2
    pinned = [torch.empty((chunk, H0, W0, 3), dtype=torch.uint8, pin_memory=True) for _ in range(nbuf)]
    staged = [torch.empty((chunk, H0, W0, 3), dtype=torch.uint8, device=dev) for _ in range(nbuf)]
    copied = [None] * nbuf          # event after the upload that last read each pinned buffer
    for c, i0 in enumerate(range(0, n, chunk)):
        b, k = c % nbuf, min(chunk, n - i0)
        if copied[b] is not None:
            copied[b].synchronize()
        host = pinned[b].numpy()
        for j in range(k):
            host[j] = _host_frame(frames[i0 + j], (H0, W0))
        staged[b][:k].copy_(pinned[b][:k], non_blocking=True)
        copied[b] = torch.cuda.Event()
        copied[b].record(stream)
        launch(staged[b], i0, k)
    return out


def _host_frame(frame, size):
    a = np.asarray(frame)
    if a.dtype != np.uint8 or a.ndim != 3 or a.shape[2] != 3 or (size is not None and a.shape[:2] != size):
        want = f'[{size[0]}, {size[1]}, 3]' if size is not None else '[H, W, 3]'
        raise ValueError(f'frames_resize: every frame must be uint8 RGB {want}, got {a.dtype} {list(a.shape)}')
    return a
