"""ctypes binding of libfyc_sm90a.so (the C ABI declared in include/fyc.h).

The product path has NO CPU fallback: if the shared library is missing or a call fails, an exception is
raised.  Every call enqueues work on the *current torch CUDA stream* and never synchronises.
"""
import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libfyc_sm90a.so")

F32, BF16, F16 = 0, 1, 2
IMPL_AUTO, IMPL_SIMT, IMPL_TC = 0, 1, 2
EPI_BIAS, EPI_RESIDUAL, EPI_ROWBIAS, EPI_GEGLU, EPI_OUT_F32, EPI_LNFOLD = 1, 2, 4, 8, 16, 32
PRED = {"epsilon": 0, "sample": 1, "v_prediction": 2}

_vp, _i64, _i32, _f32, _sz = C.c_void_p, C.c_int64, C.c_int32, C.c_float, C.c_size_t


class GemmArgs(C.Structure):
    _fields_ = [("A", _vp), ("W", _vp), ("out", _vp), ("bias", _vp), ("residual", _vp), ("rowbias", _vp),
                ("M", _i64), ("N", _i64), ("K", _i64), ("lda", _i64), ("ldw", _i64), ("ldo", _i64), ("ldr", _i64),
                ("batch", _i64), ("strideA", _i64), ("strideW", _i64), ("strideO", _i64), ("rows_per_group", _i64),
                ("alpha", _f32), ("dtype", _i32), ("epilogue", _i32), ("impl", _i32), ("A2", _vp), ("lda2", _i64), ("K1", _i64), ("ln_rowstats", _vp)]


class ConvArgs(C.Structure):
    _fields_ = [("x", _vp), ("w", _vp), ("out", _vp), ("bias", _vp), ("residual", _vp), ("rowbias", _vp),
                ("NB", _i64), ("H", _i64), ("W", _i64), ("Cin", _i64), ("Cout", _i64), ("stride", _i32),
                ("upsample", _i32), ("images_per_group", _i64), ("dtype", _i32), ("epilogue", _i32), ("impl", _i32),
                ("workspace", _vp), ("workspace_bytes", _sz), ("pad_mode", _i32), ("w_phases", _vp), ("ld_rowbias", _i64)]


class AttnArgs(C.Structure):
    _fields_ = [("q", _vp), ("k", _vp), ("v", _vp), ("out", _vp), ("batch", _i64), ("heads", _i64), ("Lq", _i64),
                ("Lk", _i64), ("D", _i64), ("ldq", _i64), ("ldk", _i64), ("ldv", _i64), ("ldo", _i64), ("bsq", _i64),
                ("bsk", _i64), ("bsv", _i64), ("bso", _i64), ("kv_batch_div", _i64), ("scale", _f32),
                ("out_alpha", _f32), ("accumulate", _i32), ("dtype", _i32), ("impl", _i32),
                ("k2", _vp), ("v2", _vp), ("Lk2", _i64), ("ldk2", _i64), ("ldv2", _i64), ("bsk2", _i64), ("bsv2", _i64), ("alpha2", _f32)]


class DdimCoefs(C.Structure):
    _fields_ = [("guidance", _f32), ("sqrt_alpha_t", _f32), ("sqrt_beta_t", _f32), ("sqrt_alpha_prev", _f32),
                ("dir_coef", _f32), ("noise_coef", _f32), ("prediction_type", _i32), ("clip_sample", _i32), ("cfg_pair", _i32)]


# every exported symbol of include/fyc.h: name -> (restype, argtypes)
SIGNATURES = {
    "fyc_version": (_i32, []),
    "fyc_last_error": (C.c_char_p, []),
    "fyc_tcgen05_available": (_i32, []),
    "fyc_gemm": (_i32, [C.POINTER(GemmArgs), _vp]),
    "fyc_conv3x3_workspace_bytes": (_sz, [C.POINTER(ConvArgs)]),
    "fyc_conv3x3": (_i32, [C.POINTER(ConvArgs), _vp]),
    "fyc_conv3x3_up2_eligible": (_i32, [C.POINTER(ConvArgs)]),
    "fyc_conv3x3_tc_route": (_i32, [C.POINTER(ConvArgs)]),
    "fyc_groupnorm_workspace_bytes": (_sz, [_i64, _i64, _i64]),
    "fyc_groupnorm": (_i32, [_vp, _vp, _vp, _vp, _i64, _i64, _i64, _i64, _f32, _i32, _i32, _vp, _sz, _vp]),
    "fyc_groupnorm_concat": (_i32, [_vp, _i64, _vp, _i64, _vp, _vp, _vp, _i64, _i64, _i64, _f32, _i32, _i32, _vp, _sz, _vp]),
    "fyc_layernorm": (_i32, [_vp, _vp, _vp, _vp, _i64, _i64, _f32, _vp, _i64, _i64, _i32, _vp]),
    "fyc_layernorm_stats": (_i32, [_vp, _vp, _vp, _i64, _i64, _f32, _i32, _vp]),
    "fyc_attention": (_i32, [C.POINTER(AttnArgs), _vp]),
    "fyc_temporal_attention": (_i32, [_vp, _vp, _i64, _i64, _i64, _i64, _i64, _f32, _i32, _vp]),
    "fyc_self_attention_tc": (_i32, [_vp, _i64, _i64, _i64, _vp, _vp, _i64, _i64, _i64, _i64, _i64, _f32, _vp]),
    "fyc_self_attention_tc_f16": (_i32, [_vp, _i64, _i64, _i64, _vp, _vp, _i64, _i64, _i64, _i64, _i64, _f32, _vp]),
    "fyc_self_attention_tc_d80": (_i32, [_vp, _i64, _i64, _i64, _vp, _vp, _i64, _i64, _i64, _i64, _f32, _vp]),
    "fyc_self_attention_tc_d80_f16": (_i32, [_vp, _i64, _i64, _i64, _vp, _vp, _i64, _i64, _i64, _i64, _f32, _vp]),
    "fyc_cross_attention_tc": (_i32, [_vp, _i64, _i64, _vp, _i64, _vp, _vp, _i64, _vp, _vp, _i64, _i64, _i64, _i64, _i64, _i64, _i64, _i64, _f32, _f32,
                                      _f32, _vp]),
    "fyc_cross_attention_tc_f16": (_i32, [_vp, _i64, _i64, _vp, _i64, _vp, _vp, _i64, _vp, _vp, _i64, _i64, _i64, _i64, _i64, _i64, _i64, _i64, _f32,
                                          _f32, _f32, _vp]),
    "fyc_transpose_tokens": (_i32, [_vp, _vp, _i64, _i64, _i64, _i64, _i64, _vp]),
    "fyc_softmax_rows": (_i32, [_vp, _vp, _i64, _i64, _i32, _vp]),
    "fyc_timestep_embed": (_i32, [_vp, _vp, _vp, _i64, _i64, _i32, _vp]),
    "fyc_silu": (_i32, [_vp, _vp, _i64, _i32, _vp]),
    "fyc_gelu": (_i32, [_vp, _vp, _i64, _i32, _vp]),
    "fyc_geglu": (_i32, [_vp, _vp, _i64, _i64, _i32, _vp]),
    "fyc_upsample_nearest2x": (_i32, [_vp, _vp, _i64, _i64, _i64, _i64, _i32, _vp]),
    "fyc_concat_channels": (_i32, [_vp, _vp, _vp, _i64, _i64, _i64, _i32, _vp]),
    "fyc_ncfhw_to_nfhwc": (_i32, [_vp, _vp, _i64, _i64, _i64, _i64, _f32, _i32, _vp]),
    "fyc_nfhwc_to_ncfhw": (_i32, [_vp, _vp, _i64, _i64, _i64, _i64, _i64, _i32, _vp]),
    "fyc_build_unet_input": (_i32, [_vp, _vp, _vp, _vp, _i64, _i64, _i64, _i32, _i32, _i32, _vp]),
    "fyc_build_unet_input_first": (_i32, [_vp, _vp, _vp, _i64, _i64, _i64, _i32, _i32, _i32, _i32, _vp]),
    "fyc_first_frame_temb_rows": (_i32, [_vp, _vp, _i64, _i64, _i64, _vp]),
    "fyc_cfg_ddim_step": (_i32, [_vp, _vp, _vp, _vp, _i64, C.POINTER(DdimCoefs), _vp]),
    "fyc_cfg_video_ddim_step": (_i32, [_vp, _vp, _f32, _vp, _vp, _vp, _i64, C.POINTER(DdimCoefs), _vp]),
    "fyc_frames_finalize": (_i32, [_vp, _vp, _i64, _i64, _i64, _i64, _i32, _vp]),
    "fyc_video_grid_u8": (_i32, [_vp, _vp, _i64, _i64, _i64, _i64, _i64, _i64, _i32, _vp]),
}

_lib = None
launch_count = 0          # kernels-launching C-ABI calls made by this process (bench.py reports it)


class FycError(RuntimeError):
    pass


def lib():
    """Load (once) and return the shared library.  Fails loudly if it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise FycError(f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                           "(there is no CPU/PyTorch fallback for the engine)")
        l = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(l, name)
            fn.restype, fn.argtypes = res, args
        _lib = l
    return _lib


def check(status):
    global launch_count
    launch_count += 1
    if status != 0:
        raise FycError(f"libfyc status {status}: {lib().fyc_last_error().decode()}")


def stream_ptr():
    return torch.cuda.current_stream().cuda_stream


def dtype_code(t):
    if t == torch.float32:
        return F32
    if t == torch.bfloat16:
        return BF16
    if t == torch.float16:
        return F16
    raise FycError(f"unsupported activation dtype {t}")


def ptr(t):
    return None if t is None else t.data_ptr()
