"""`Adapter` -- VideoCrafter's T2I-Adapter (videocrafter/lvdm/models/modules/adapter.py:75-105), the depth-conditioning
network of T2VAdapterDepth, with its arithmetic in libt2v_b200.so (csrc/adapter.cu).

Kept from the reference: the constructor keywords and defaults, the parameter tree (`conv_in`, `body[k].{in_conv, block1,
block2, skep, down_opt.op}`, k = level * nums_rb + block, generated from the library's own parameter table), so an adapter
checkpoint loads with `load_state_dict(strict=True)`, and `forward(x) -> list` of one feature map per level.  The features
are channels-last views of the library's output, [N, C_l, h_l, w_l] with strides of an [N, h_l, w_l, C_l] tensor, which is
the layout `UNetModel.forward(features_adapter=...)` stages without a copy.
"""
import ctypes as C

import torch

from . import _lib
from .modules import _NativeModule, _build_tree


class Adapter(_NativeModule):
    def __init__(self, channels=(320, 640, 1280, 1280), nums_rb=3, cin=64, ksize=3, sk=False, use_conv=True):
        super().__init__()
        channels = [int(c) for c in channels]
        if not 1 <= len(channels) <= 4:
            raise ValueError(f'Adapter: 1 to 4 levels are built (got {len(channels)})')
        self.channels, self.nums_rb, self.cin, self.ksize = channels, int(nums_rb), int(cin), int(ksize)
        self.sk, self.use_conv = bool(sk), bool(use_conv)
        cfg = _lib.AdapterConfigC()
        cfg.cin, cfg.n_levels, cfg.nums_rb, cfg.ksize = self.cin, len(channels), self.nums_rb, self.ksize
        for i, c in enumerate(channels):
            cfg.channels[i] = c
        cfg.sk, cfg.use_conv = int(self.sk), int(self.use_conv)
        try:
            table = self._open('adapter', cfg)
        except RuntimeError:
            raise ValueError(f'Adapter({channels}, nums_rb={nums_rb}, cin={cin}, ksize={ksize}, sk={sk}, use_conv={use_conv}): '
                             f'{_lib.load_library().t2v_last_error().decode()}') from None
        _build_tree(self, table)

    def feature_sizes(self, H, W):
        """[(h_l, w_l)] of a H x W input: PixelUnshuffle(8), then halved per level (stride-2 conv: rounding up, average
        pooling: rounding down)."""
        if H % 8 or W % 8:
            raise ValueError(f'Adapter: input {H}x{W} is not a multiple of 8 (PixelUnshuffle(8))')
        h, w = H // 8, W // 8
        out = []
        for i in range(len(self.channels)):
            if i:
                h, w = ((h + 1) // 2, (w + 1) // 2) if self.use_conv else (h // 2, w // 2)
            if h < 1 or w < 1:
                raise ValueError(f'Adapter: level {i} of a {H}x{W} input would be empty ({h}x{w})')
            out.append((h, w))
        return out

    @torch.no_grad()
    def forward(self, x):
        """x [N, cin/64, H, W] -> [features [N, channels[l], h_l, w_l] fp16 (channels-last views)]."""
        if x.dim() != 4 or x.shape[1] * 64 != self.cin:
            raise ValueError(f'Adapter expects [N, {self.cin // 64}, H, W] condition frames, got {tuple(x.shape)}')
        N, _, H, W = x.shape
        sizes = self.feature_sizes(H, W)
        self.sync_weights()
        if not x.is_cuda:
            raise RuntimeError('Adapter input must be on the GPU (there is no CPU path in t2v_b200)')
        if x.dtype not in (torch.float16, torch.float32):
            x = x.float()
        x = x.contiguous()
        outs = [torch.empty((N, h, w, c), device=x.device, dtype=torch.float16) for (h, w), c in zip(sizes, self.channels)]
        ptrs = (C.c_void_p * len(outs))(*[o.data_ptr() for o in outs])
        _lib.check(_lib.lib().t2v_adapter_encode(self._handle, _lib.ptr(x), int(x.dtype == torch.float32), ptrs, N, H, W,
                                                 _lib.stream_ptr()), 'adapter_encode')
        return [o.permute(0, 3, 1, 2) for o in outs]
