"""ctypes binding of libt2v_b200.so (the C ABI declared in include/t2v_b200.h).

There is deliberately NO fallback: if the shared library is missing or the device is not sm_90 the import of
the product path fails loudly (RuntimeError) -- a silent PyTorch path would void every parity/perf claim.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get('T2V_LIB_PATH') or os.path.join(_HERE, 'libt2v_b200.so')      # override: A/B builds of the kernels

c_void_p, c_int, c_ll, c_float, c_char_p, c_double = C.c_void_p, C.c_int, C.c_longlong, C.c_float, C.c_char_p, C.c_double
P = c_void_p

# name -> (restype, [argtypes]); mirrors include/t2v_b200.h one to one
SIGNATURES = {
    't2v_init': (c_int, [c_int]),
    't2v_last_error': (c_char_p, []),
    't2v_num_sms': (c_int, []),
    't2v_version': (c_char_p, []),
    't2v_unet_create': (c_int, [P, C.POINTER(P)]),
    't2v_unet_destroy': (None, [P]),
    't2v_unet_set_param': (c_int, [P, c_char_p, P, c_int, c_int, C.POINTER(C.c_int64), P]),
    't2v_unet_missing_params': (c_int, [P, c_char_p, C.c_size_t]),
    't2v_unet_param_info': (c_int, [P, c_int, c_char_p, C.c_size_t, C.POINTER(C.c_int64), C.POINTER(c_int)]),
    't2v_unet_forward': (c_int, [P, P, c_int, P, P, P, c_int, c_int, c_int, c_int, c_int, c_int, P]),
    't2v_unet_forward_ctx': (c_int, [P, P, c_int, P, P, c_int, P, c_int, c_int, c_int, c_int, c_int, c_int, P]),
    't2v_unet_forward_adapter': (c_int, [P, P, c_int, P, P, P, c_int, c_int, P, c_int, c_int, c_int, c_int, c_int, c_int, P]),
    't2v_unet_flops': (c_double, [P, c_int, c_int, c_int, c_int, c_int]),
    't2v_unet_plan_bytes': (c_int, [P, c_int, c_int, c_int, c_int, c_int, C.POINTER(C.c_size_t)]),
    't2v_unet_plan_info': (c_int, [P, c_int, c_int, c_int, c_int, c_int, c_int, C.POINTER(C.c_size_t), C.POINTER(c_double),
                                   C.POINTER(c_int)]),
    't2v_unet_num_launches': (c_int, [P]),
    't2v_unet_profile': (c_int, [P, c_int, c_int, c_int, c_int, c_int, P, C.POINTER(c_double)]),
    't2v_unet_read_tap': (c_ll, [P, c_char_p, P, c_ll, P]),
    't2v_unet_enable_taps': (c_int, [P, c_int]),
    't2v_unet_tap_info': (c_int, [P, c_char_p, C.POINTER(c_ll), C.POINTER(c_int), C.POINTER(c_int), C.POINTER(c_int)]),
    't2v_unet_lora_merge': (c_int, [P, c_char_p, P, P, c_int, c_float, c_int, P]),
    't2v_unet_lora_clear': (c_int, [P, P]),
    't2v_unet_lora_merged': (c_int, [P]),
    't2v_unet_lora_apply': (c_int, [P, c_char_p, P, P, c_int, c_int, c_float, P]),
    't2v_unet_lora_restore': (c_int, [P, c_char_p, P]),
    't2v_vae_lora_apply': (c_int, [P, c_char_p, P, P, c_int, c_int, c_float, P]),
    't2v_vae_lora_restore': (c_int, [P, c_char_p, P]),
    't2v_vae_lora_clear': (c_int, [P, P]),
    't2v_vae_lora_merged': (c_int, [P]),
    't2v_clip_lora_apply': (c_int, [P, c_char_p, P, P, c_int, c_int, c_float, P]),
    't2v_clip_lora_restore': (c_int, [P, c_char_p, P]),
    't2v_clip_lora_clear': (c_int, [P, P]),
    't2v_clip_lora_merged': (c_int, [P]),
    't2v_adapter_lora_apply': (c_int, [P, c_char_p, P, P, c_int, c_int, c_float, P]),
    't2v_adapter_lora_restore': (c_int, [P, c_char_p, P]),
    't2v_adapter_lora_clear': (c_int, [P, P]),
    't2v_adapter_lora_merged': (c_int, [P]),
    't2v_unet_shard_setup': (c_int, [P, c_int, c_int]),
    't2v_unet_shard_prepare': (c_int, [P, c_int, c_int, c_int, c_int, c_int, P, P]),
    't2v_unet_shard_connect': (c_int, [P, c_int, c_int, c_int, c_int, c_int, P, P]),
    't2v_unet_shard_connected': (c_int, [P, c_int, c_int, c_int, c_int, c_int]),
    't2v_unet_shard_barrier': (c_int, [P, P]),
    't2v_unet_shard_info': (c_int, [P, c_int, C.POINTER(c_int), C.POINTER(c_int), C.POINTER(c_int)]),
    't2v_vae_create': (c_int, [P, C.POINTER(P)]),
    't2v_vae_destroy': (None, [P]),
    't2v_vae_set_param': (c_int, [P, c_char_p, P, c_int, c_int, C.POINTER(C.c_int64), P]),
    't2v_vae_missing_params': (c_int, [P, c_char_p, C.c_size_t]),
    't2v_vae_param_info': (c_int, [P, c_int, c_char_p, C.c_size_t, C.POINTER(C.c_int64), C.POINTER(c_int)]),
    't2v_vae_decode': (c_int, [P, P, c_int, c_float, P, c_int, c_int, c_int, c_int, c_int, P]),
    't2v_vae_encode': (c_int, [P, P, c_int, P, c_int, c_int, c_int, P]),
    't2v_vae_flops': (c_double, [P, c_int, c_int, c_int]),
    't2v_vae_plan_bytes': (c_int, [P, c_int, c_int, c_int, c_int, C.POINTER(C.c_size_t), C.POINTER(C.c_size_t)]),
    't2v_vae_plan_chunks': (c_int, [P, c_int, c_int, c_int, c_int, C.c_size_t, C.POINTER(c_int), C.POINTER(c_int)]),
    't2v_vae_set_memory_budget': (c_int, [P, C.c_size_t]),
    't2v_vae_get_memory_budget': (C.c_size_t, [P]),
    't2v_vae_last_chunking': (c_int, [P, c_int, C.POINTER(c_int), C.POINTER(c_int)]),
    't2v_vae_cached_plans': (c_int, [P, c_int, C.POINTER(C.c_size_t)]),
    't2v_vae_enable_taps': (c_int, [P, c_int, P]),
    't2v_vae_tap_info': (c_int, [P, c_char_p, C.POINTER(c_ll), C.POINTER(c_int), C.POINTER(c_int), C.POINTER(c_int)]),
    't2v_vae_read_tap': (c_ll, [P, c_char_p, P, c_ll, P]),
    't2v_clip_create': (c_int, [P, C.POINTER(P)]),
    't2v_clip_destroy': (None, [P]),
    't2v_clip_set_param': (c_int, [P, c_char_p, P, c_int, c_int, C.POINTER(C.c_int64), P]),
    't2v_clip_param_info': (c_int, [P, c_int, c_char_p, C.c_size_t, C.POINTER(C.c_int64), C.POINTER(c_int)]),
    't2v_clip_encode': (c_int, [P, P, P, c_int, c_int, P]),
    't2v_adapter_create': (c_int, [P, C.POINTER(P)]),
    't2v_adapter_destroy': (None, [P]),
    't2v_adapter_set_param': (c_int, [P, c_char_p, P, c_int, c_int, C.POINTER(C.c_int64), P]),
    't2v_adapter_missing_params': (c_int, [P, c_char_p, C.c_size_t]),
    't2v_adapter_param_info': (c_int, [P, c_int, c_char_p, C.c_size_t, C.POINTER(C.c_int64), C.POINTER(c_int)]),
    't2v_adapter_encode': (c_int, [P, P, c_int, P, c_int, c_int, c_int, P]),
    't2v_ddim_step': (c_int, [P, P, P, c_int, P, c_ll, c_ll, c_int, c_int, c_float, c_int, c_float, c_float, c_float, c_float,
                              c_float, P, c_int, P]),
    't2v_ddim_step_ex': (c_int, [P, P, P, c_int, P, c_ll, c_ll, c_int, c_int, c_float, c_int, c_float, c_float, c_float, c_float,
                                 c_float, P, c_int, c_int, P, P]),
    't2v_cfg_x0': (c_int, [P, P, P, c_int, P, c_ll, c_float, c_float, c_float, c_int, P]),
    't2v_lincomb': (c_int, [P, C.POINTER(P), C.POINTER(c_float), c_int, c_ll, P]),
    't2v_ddim_step_threshold': (c_int, [P, P, P, c_int, P, c_ll, c_ll, c_int, c_int, c_float, c_float, c_float, c_float, c_float,
                                        c_float, P, c_int, c_int, c_float, P, P, c_ll, P]),
    't2v_abs_quantile': (c_int, [P, c_int, c_ll, c_float, P, P, c_ll, P]),
    't2v_abs_quantile_workspace': (c_ll, [c_int]),
    't2v_latent_blend': (c_int, [P, c_int, P, P, P, P, c_int, c_int, c_ll, P]),
    't2v_q_sample_blend': (c_int, [P, C.POINTER(c_ll), P, C.POINTER(c_ll), P, P, P, C.POINTER(c_ll), P, P, C.POINTER(c_int), P]),
    't2v_frames_resize': (c_int, [P, c_int, c_int, c_int, P, c_int, c_int, c_int, P, c_ll, P]),
    't2v_resize_coeffs': (c_int, [c_int, c_int, C.POINTER(c_int), P, P]),
    't2v_op_gemm': (c_int, [P, c_ll, c_int, c_int, C.POINTER(c_int), c_int, C.POINTER(c_int), P, c_int, c_int, c_int,
                            c_int, P, c_ll, P, c_int, c_ll, P, c_ll, c_float, c_int, c_int, P]),
    't2v_op_gemm_splitk': (c_int, [P, c_ll, c_int, c_int, C.POINTER(c_int), c_int, C.POINTER(c_int), P, c_int, c_int, c_int,
                                   c_int, P, c_ll, P, c_int, c_ll, P, c_ll, c_float, c_int, P, c_ll, C.POINTER(c_int), c_int,
                                   c_int, P]),
    't2v_op_ln_linear': (c_int, [P, c_ll, c_ll, c_int, P, P, P, P, c_int, c_int, P, P, P, P, P, c_ll, P, c_ll, c_int, c_int, P]),
    't2v_op_pack_conv_weight': (c_int, [P, c_int, P, c_int, c_int, c_int, c_int, c_int, P]),
    't2v_op_pack_geglu_weight': (c_int, [P, P, c_int, P, P, c_int, c_int, c_int, P]),
    't2v_op_lora_merge': (c_int, [P, P, P, c_int, c_int, c_int, c_float, c_int, P]),
    't2v_op_lora_apply': (c_int, [P, P, P, c_int, c_int, c_int, c_int, c_float, P]),
    't2v_op_groupnorm': (c_int, [P, c_ll, P, c_ll, c_ll, c_int, c_int, P, P, c_float, c_int, c_int, P, P]),
    't2v_op_layernorm': (c_int, [P, c_ll, P, c_ll, c_ll, c_int, P, P, c_float, P]),
    't2v_op_attention': (c_int, [P, P, P, P, c_ll, c_ll, c_ll, c_ll, c_ll, c_ll, c_ll, c_ll, c_int, c_int, c_int, c_int,
                                 c_int, c_float, P]),
    't2v_op_attention_hd': (c_int, [P, P, P, P, c_ll, c_ll, c_ll, c_ll, c_ll, c_ll, c_ll, c_ll, c_int, c_int, c_int, c_int,
                                    c_int, c_int, c_float, c_int, c_ll, c_ll, c_ll, c_ll, P]),
    't2v_op_attention_relpos': (c_int, [P, P, P, P, P, P, c_ll, c_ll, c_ll, c_ll, c_ll, c_ll, c_ll, c_ll, c_int, c_int,
                                        c_int, c_int, c_float, P]),
    't2v_op_clip_attention': (c_int, [P, P, c_int, c_int, c_int, c_int, P]),
    't2v_op_upsample2x': (c_int, [P, P, c_int, c_int, c_int, c_int, P]),
    't2v_op_im2col_s2': (c_int, [P, P, c_int, c_int, c_int, c_int, c_int, P]),
    't2v_op_time_sinusoid': (c_int, [P, P, c_int, c_int, P]),
    't2v_op_small_linear': (c_int, [P, c_ll, P, P, P, P, c_ll, c_int, c_int, c_int, c_int, P]),
    't2v_op_ingest_latent': (c_int, [P, c_int, P, c_ll, c_int, c_int, c_int, c_int, c_int, c_ll, c_ll, c_float, P]),
    't2v_op_egress_latent': (c_int, [P, c_ll, P, c_int, c_int, c_int, c_int, c_int, c_int, P]),
    't2v_op_avgpool2x2': (c_int, [P, P, c_int, c_int, c_int, c_int, P]),
    't2v_op_pixel_unshuffle': (c_int, [P, c_int, P, c_int, c_int, c_int, c_int, P]),
    't2v_op_relu': (c_int, [P, c_ll, c_int, P]),
    't2v_op_feature_add': (c_int, [P, c_ll, P, c_int, c_ll, c_ll, c_int, P]),
    't2v_op_concat_cols': (c_int, [P, c_ll, c_int, P, c_ll, c_int, P, c_ll, c_ll, P]),
    't2v_op_softmax_rows': (c_int, [P, P, c_ll, c_int, c_float, P]),
    't2v_op_transpose_batched': (c_int, [P, P, c_int, c_int, c_int, P]),
    't2v_op_frames_to_u8': (c_int, [P, c_ll, P, c_ll, P]),
    't2v_op_frames_to_f32': (c_int, [P, c_ll, P, c_int, c_int, c_int, P]),
    't2v_op_convert_to_f16': (c_int, [P, c_int, P, c_ll, P]),
}


class UNetConfigC(C.Structure):
    _fields_ = [('in_dim', c_int), ('dim', c_int), ('context_dim', c_int), ('out_dim', c_int),
                ('dim_mult', c_int * 8), ('n_mult', c_int), ('num_heads', c_int), ('head_dim', c_int),
                ('num_res_blocks', c_int), ('attn_scales', c_float * 8), ('n_attn_scales', c_int), ('arch', c_int),
                ('temporal_length', c_int)]


class ShardExportC(C.Structure):
    """t2v_shard_export (include/t2v_b200.h): what the ranks of a frame-sharded clip swap once per shape."""
    _fields_ = [('comm_handle', C.c_ubyte * 64), ('slab_handle', C.c_ubyte * 64), ('rank', c_int), ('nranks', c_int),
                ('n_exchanges', c_int), ('n_groupnorms', c_int), ('dst_offset', c_ll * 192)]


class ClipConfigC(C.Structure):
    _fields_ = [('width', c_int), ('heads', c_int), ('layers_run', c_int), ('context', c_int), ('vocab', c_int), ('arch', c_int)]


class AdapterConfigC(C.Structure):
    _fields_ = [('cin', c_int), ('channels', c_int * 4), ('n_levels', c_int), ('nums_rb', c_int), ('ksize', c_int), ('sk', c_int),
                ('use_conv', c_int)]


class VAEConfigC(C.Structure):
    _fields_ = [('ch', c_int), ('ch_mult', c_int * 8), ('n_mult', c_int), ('num_res_blocks', c_int),
                ('z_channels', c_int), ('out_ch', c_int), ('embed_dim', c_int)]


_lib = None
_inited_device = None


def load_library():
    """dlopen only (no GPU needed): used by the CPU tests to check the exported symbol table."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(f'{LIB_PATH} is missing: build it with `python __graft_entry__.py` '
                               f'(or sd-webui-text2video_b200/csrc/build.sh); there is no CPU fallback')
        lib = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            if os.environ.get('T2V_BRINGUP') == '1' and not hasattr(lib, name):
                continue                 # kernel bring-up scripts only; tests never set this
            fn = getattr(lib, name)      # AttributeError if the .so does not export a declared symbol
            fn.restype = res
            fn.argtypes = args
        _lib = lib
    return _lib


def lib():
    """The library, initialised on the current CUDA device.  Raises if there is no sm_90 GPU."""
    global _inited_device
    import torch
    l = load_library()
    if not torch.cuda.is_available():
        raise RuntimeError('t2v_b200 needs a CUDA device (sm_90a); no CPU fallback exists')
    dev = torch.cuda.current_device()
    if _inited_device != dev:
        torch.cuda.init()
        rc = l.t2v_init(dev)
        if rc != 0:
            raise RuntimeError(f't2v_init failed ({rc}): {l.t2v_last_error().decode()}')
        _inited_device = dev
    return l


def check(rc, what=''):
    if rc != 0:
        raise RuntimeError(f't2v_b200 {what} failed ({rc}): {load_library().t2v_last_error().decode()}')


def stream_ptr():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)
