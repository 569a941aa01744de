"""Stable-LoRA merging for the GPU-native denoiser -- the arithmetic of `StableLoraProcessor.process_lora`
(scripts/stable_lora/stable_utils/lora_processor.py:202-246 and :50-96) done on the library's packed weights.

The reference walks `model.named_modules()`, and for every `<name>.lora_A` / `<name>.lora_B` pair in a LoRA file replaces
`m.weight` by `W + alpha * (B @ A)` (Linear; Conv2d with the product viewed as the weight; Conv3d (3,1,1) with the product
viewed [o, i, 3, 3, 1] and averaged over the second kernel axis), undoing the previous selection with `-=` first.  Through
the drop-in mirror that surgery still works (re-assigned Parameters are re-shipped by sync_weights), but it re-packs the whole
model and rebuilds every plan.  `process_lora` below keeps the walk, the key matching and the flags, and sends each pair to
`UNetSD.lora_merge` instead: one small kernel per weight + an in-place re-pack of the variants that depend on it.  Undo is
`lora_clear()` (restores the base copies exactly), so switching LoRAs never accumulates fp16 rounding residue.
"""
import torch

from .modules import UNetSD


class StableLoraProcessor(object):
    def __init__(self):
        self.previous = None          # (lora_files_list, alpha, flags) of the current merge

    @staticmethod
    def is_lora_match(key, name):
        return key == f'{name}.lora_A'            # lora_processor.py:33-41 (key_name_match on 'lora_A')

    @torch.no_grad()
    def process_lora(self, model, lora_files_list, use_bias=False, use_time=True, use_conv=True, use_emb=False, use_linear=True,
                     lora_alpha=1.0, undo_merge=False):
        """`lora_files_list`: list of {key: tensor} dicts (loaded safetensors).  undo_merge=True drops every merge (the
        reference re-applies the previous files with `-=`; here the base copies are restored)."""
        if not isinstance(model, UNetSD):
            raise TypeError('process_lora works on the t2v_b200 UNetSD mirror')
        if use_bias or use_emb:
            raise NotImplementedError('bias / embedding LoRA entries are not part of the denoiser hot path')
        if undo_merge:
            model.lora_clear()
            self.previous = None
            return 0
        merged = 0
        for n, m in model.named_modules():
            for lora_model in lora_files_list:
                ka, kb = f'{n}.lora_A', f'{n}.lora_B'
                if ka not in lora_model or kb not in lora_model:
                    continue
                A, B = lora_model[ka], lora_model[kb]
                if isinstance(m, torch.nn.Linear) and use_linear:
                    if 'proj' in n:                                    # :222-223 squeezes a trailing 1 of Conv1d-style tensors
                        A, B = (t.squeeze(-1) if t.dim() > 2 else t for t in (A, B))
                    model.lora_merge(n + '.weight', A, B, lora_alpha)
                    merged += 1
                elif isinstance(m, (torch.nn.Conv2d, torch.nn.Conv1d)) and use_conv:
                    model.lora_merge(n + '.weight', A, B, lora_alpha)
                    merged += 1
                elif isinstance(m, torch.nn.Conv3d) and use_conv and use_time:
                    model.lora_merge(n + '.weight', A, B, lora_alpha, temporal_mean=True)
                    merged += 1
        self.previous = (lora_files_list, lora_alpha)
        return merged
