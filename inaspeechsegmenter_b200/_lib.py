"""ctypes binding of libiss_b200.so (the C ABI declared in include/iss_b200.h).

This is the thin FFI layer the north-star asks for: Python host code calling
hand-written sm_90a CUDA through a C ABI; torch tensors only supply device
memory (``data_ptr()``) and streams.  There is no fallback: if the library is
missing or a call fails, an exception is raised.
"""
import ctypes
import os

import numpy as np

from . import _build

_c = ctypes
_LIB = None


class IssError(RuntimeError):
    pass


class LayerDesc(_c.Structure):
    _fields_ = [('kind', _c.c_int32), ('kh', _c.c_int32), ('kw', _c.c_int32),
                ('sh', _c.c_int32), ('sw', _c.c_int32),
                ('pad_top', _c.c_int32), ('pad_left', _c.c_int32),
                ('pad_bottom', _c.c_int32), ('pad_right', _c.c_int32),
                ('cin', _c.c_int32), ('cout', _c.c_int32), ('flags', _c.c_int32),
                ('w_off', _c.c_int64), ('bias_off', _c.c_int64),
                ('pre_scale_off', _c.c_int64), ('pre_shift_off', _c.c_int64),
                ('post_scale_off', _c.c_int64), ('post_shift_off', _c.c_int64)]


LAYER_CONV2D, LAYER_DENSE, LAYER_MAXPOOL = 1, 2, 3
F_BIAS, F_AFFINE_PRE, F_RELU, F_AFFINE_POST, F_SOFTMAX, F_SIGMOID = 1, 2, 4, 8, 16, 32
PCM_F32, PCM_S16 = 0, 1
PCM_U8, PCM_S24, PCM_S32, PCM_F64 = 2, 3, 4, 5      # WAV encodings the resampler alone reads
RESAMPLE_END = 1                      # ISS_RESAMPLE_END
VBX_END = 1                           # ISS_VBX_END
FFT_FP32, FFT_FP64 = 0, 1
GEMM_FP32, GEMM_TC_TS, GEMM_TC_F16 = 0, 2, 3     # fp32 CUDA cores | 3xTF32 wgmma | fp16-split wgmma (default)
ABI_VERSION = 9                      # == ISS_ABI_VERSION in include/iss_b200.h

# name -> (restype, argtypes); must list every symbol include/iss_b200.h declares
_vp, _i, _i64, _d = _c.c_void_p, _c.c_int, _c.c_int64, _c.c_double
SIGNATURES = {
    'iss_version': (_i, []),
    'iss_last_error': (_c.c_char_p, []),
    'iss_ctx_create': (_i, [_i, _c.POINTER(_vp)]),
    'iss_ctx_destroy': (_i, [_vp]),
    'iss_launch_count': (_i64, []),
    'iss_set_gemm_mode': (_i, [_i]),
    'iss_get_gemm_mode': (_i, []),
    'iss_sidekit_num_frames': (_i64, [_i64]),
    'iss_sidekit_upload_tables': (_i, [_vp, _vp, _vp]),
    'iss_sidekit_features': (_i, [_vp, _vp, _i, _i64, _i, _vp, _vp, _vp, _vp]),
    'iss_sidekit_features_multi': (_i, [_vp, _i, _vp, _vp, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp]),
    'iss_loge_stats': (_i, [_vp, _vp, _i64, _vp, _vp]),
    'iss_loge_stats_multi': (_i, [_vp, _vp, _vp, _vp, _i, _vp, _vp]),
    'iss_set_energy_viterbi_serial': (_i, [_i]),
    'iss_energy_viterbi': (_i, [_vp, _vp, _i64, _vp, _d, _vp, _vp, _d, _i, _vp, _vp, _vp]),
    'iss_energy_viterbi_multi': (_i, [_vp, _vp, _vp, _i, _vp, _d, _vp, _vp, _d, _i, _vp, _vp, _vp, _vp]),
    'iss_viterbi_segments': (_i, [_vp, _vp, _i, _vp, _i, _vp, _d, _vp, _vp, _vp]),
    'iss_viterbi_work_bytes': (_i64, [_i64, _i]),
    'iss_viterbi_online': (_i, [_vp, _i, _i, _vp, _vp, _i64, _vp, _d, _vp, _vp, _d, _vp, _vp, _i64, _i64, _vp, _i64, _vp,
                                _vp, _vp]),
    'iss_viterbi_online_work_bytes': (_i64, [_i]),
    'iss_energy_transfer': (_i, [_vp, _vp, _i64, _vp, _d, _vp, _vp, _vp, _vp, _vp]),
    'iss_energy_forward': (_i, [_vp, _vp, _i64, _vp, _d, _vp, _vp, _d, _vp, _vp, _vp, _vp, _vp]),
    'iss_energy_emit': (_i, [_vp, _i64, _i, _i, _vp, _vp, _vp]),
    'iss_cnn_create': (_i, [_vp, _c.POINTER(LayerDesc), _i, _vp, _i64, _i, _i, _c.POINTER(_vp)]),
    'iss_cnn_destroy': (_i, [_vp]),
    'iss_cnn_num_classes': (_i, [_vp]),
    'iss_cnn_flops_per_patch': (_d, [_vp]),
    'iss_cnn_workspace_bytes': (_i64, [_vp, _i64, _i]),
    'iss_cnn_forward': (_i, [_vp, _vp, _vp, _i64, _i, _i, _i, _vp, _vp, _i, _vp, _vp, _i64, _vp]),
    'iss_cnn_forward_multi': (_i, [_vp, _vp, _vp, _i64, _i, _vp, _vp, _i, _vp, _vp, _vp, _i, _vp, _vp, _i64, _vp]),
    'iss_vbx_num_frames': (_i64, [_i64]),
    'iss_vbx_upload_tables': (_i, [_vp, _vp, _vp]),
    'iss_vbx_work_bytes': (_i64, [_i64]),
    'iss_vbx_features': (_i, [_vp, _vp, _i, _i64, _vp, _vp, _vp, _vp]),
    'iss_vbx_features_multi': (_i, [_vp, _i, _vp, _vp, _i, _vp, _vp, _vp, _vp, _vp]),
    'iss_vbx_fbank_window_multi': (_i, [_vp, _i, _vp, _vp, _vp, _i, _vp, _vp]),
    'iss_vbx_cmvn_window_multi': (_i, [_vp, _i, _vp, _vp, _vp, _vp]),
    'iss_dither_mt19937_multi': (_i, [_vp, _i, _vp, _vp, _i64, _vp, _vp]),
    'iss_resample_num_frames': (_i64, [_i64, _i]),
    'iss_resample_upload_taps': (_i, [_vp, _i, _vp, _i64]),
    'iss_resample_release_taps': (_i, [_vp, _i]),
    'iss_resample_to16k_multi': (_i, [_vp, _i, _vp, _vp, _i, _i, _i, _vp, _vp, _vp]),
    'iss_resample_window_multi': (_i, [_vp, _i, _vp, _vp, _i, _i, _i, _vp, _vp]),
    'iss_resnet_blob_len': (_i64, [_i, _i, _i, _vp]),
    'iss_resnet_create': (_i, [_vp, _vp, _i64, _i, _i, _i, _vp, _c.POINTER(_vp)]),
    'iss_resnet_destroy': (_i, [_vp]),
    'iss_resnet_flops_per_window': (_d, [_vp, _i]),
    'iss_resnet_workspace_bytes': (_i64, [_vp, _i, _i]),
    'iss_resnet_embed': (_i, [_vp, _vp, _vp, _i64, _vp, _i, _i, _vp, _vp, _i64, _vp]),
    'iss_mlp_create': (_i, [_vp, _c.POINTER(LayerDesc), _i, _vp, _i64, _i, _c.POINTER(_vp)]),
    'iss_mlp_destroy': (_i, [_vp]),
    'iss_mlp_out_dim': (_i, [_vp]),
    'iss_mlp_workspace_bytes': (_i64, [_vp, _i64]),
    'iss_mlp_forward': (_i, [_vp, _vp, _vp, _i64, _vp, _vp, _i64, _vp]),
    'iss_cnn_profile': (_i, [_vp, _i]),
    'iss_cnn_profile_read': (_i, [_vp, _c.POINTER(_d), _c.POINTER(_i64), _c.POINTER(_d)]),
    'iss_cnn_layer_flops': (_d, [_vp, _i]),
    'iss_cnn_num_layers': (_i, [_vp]),
    'iss_gather_halo_rows_bound': (_i, [_i, _i, _i, _i, _i, _i]),
    'iss_gather_halo_smem': (_i, [_i] * 10),
    'iss_gather_pipe_smem': (_i, [_i] * 10),
}


def lib_path():
    return _build.LIB


def load(build_if_missing=True):
    """Loads (building first if the .so is absent and nvcc is available)."""
    global _LIB
    if _LIB is not None:
        return _LIB
    path = lib_path()
    if not os.path.exists(path):
        if not build_if_missing:
            raise IssError('libiss_b200.so is not built (run `python -m inaspeechsegmenter_b200._build`); '
                           'there is no CPU fallback')
        _build.build()
    elif build_if_missing and _build.needs_build() and os.access(_build.NVCC, os.X_OK):
        _build.build()                   # sources newer than the library: never load a stale ABI silently
    lib = _c.CDLL(path)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)          # AttributeError if the symbol is missing
        fn.restype, fn.argtypes = res, args
    if lib.iss_version() != ABI_VERSION:
        raise IssError('libiss_b200.so has ABI version %d, this package binds version %d: rebuild it '
                       '(python -m inaspeechsegmenter_b200._build --force)' % (lib.iss_version(), ABI_VERSION))
    _LIB = lib
    return lib


def check(rc, what=''):
    if rc != 0:
        msg = load().iss_last_error()
        raise IssError('%s failed (%d): %s' % (what, rc, msg.decode() if msg else ''))


def ptr(x):
    """Device/host pointer of a torch tensor or numpy array as c_void_p."""
    if x is None:
        return _c.c_void_p(0)
    if isinstance(x, np.ndarray):
        return _c.c_void_p(x.ctypes.data)
    return _c.c_void_p(x.data_ptr())
