"""ctypes binding of libstb200.so (include/stb200.h) and, for tests/ only, of libstb200_test.so
(include/stb200_test.h: kernel-level hooks that are not part of the product library).  No fallback: a missing
library is a hard error."""
from __future__ import annotations

import ctypes as C
from pathlib import Path

import os

PKG_DIR = Path(__file__).resolve().parent
LIB_PATH = Path(os.environ.get('STB_LIB', PKG_DIR / 'libstb200.so'))   # STB_LIB: A/B a differently built library
TEST_LIB_PATH = PKG_DIR / 'libstb200_test.so'

STB_ERR_INVALID = -1
MAX_LOSS_TERMS = 14   # STB_MAX_LOSS_TERMS
POOLING = {'max': 0, 'average': 1, 'l2': 2}

_lib = None
_tlib = None


class NativeError(RuntimeError):
    pass


def _set(lib, sigs):
    for name, args in sigs.items():
        fn = getattr(lib, name)
        fn.argtypes = args
        fn.restype = C.c_int


def _declare(lib):
    vp, i, f, sz, i64 = C.c_void_p, C.c_int, C.c_float, C.c_size_t, C.c_int64
    pp = C.POINTER(C.c_void_p)
    lib.stb_last_error.restype = C.c_char_p
    lib.stb_last_error.argtypes = []
    _set(lib, {
        'stb_ctx_create': [i, i, pp, pp, vp, pp],
        'stb_workspace_bytes': [vp, i, i, C.POINTER(sz)],
        'stb_bind_workspace': [vp, vp, sz, vp],
        'stb_style_stats': [vp, vp, i, i, pp, pp, vp],
        'stb_content_features': [vp, vp, i, i, vp, vp],
        'stb_set_targets': [vp, i, i, vp, f, pp, pp, C.POINTER(f), f, f, vp],
        'stb_set_layers': [vp, i, C.POINTER(i), i, C.POINTER(i)],
        'stb_content_features_ex': [vp, vp, i, i, pp, vp],
        'stb_set_targets_ex': [vp, i, i, pp, C.POINTER(f), pp, pp, C.POINTER(f), f, f, vp],
        'stb_loss_terms': [vp, vp, i, C.POINTER(i), vp],
        'stb_iterate': [vp, vp, vp, vp, vp, i64, f, f, f, f, f, vp, vp],
        'stb_iterate_ex': [vp, vp, vp, vp, vp, i64, f, f, f, f, f, i, vp, vp, vp],
        'stb_lbfgs_state_bytes': [i, i, C.POINTER(sz)],
        'stb_lbfgs_reset': [vp, i, i, vp],
        'stb_iterate_lbfgs': [vp, vp, vp, vp, sz, i64, f, vp, vp],
        'stb_set_band': [vp, i, i, i, i],
        'stb_stats_block': [vp, i, i, pp, C.POINTER(sz)],
        'stb_iterate_fwd': [vp, vp, vp],
        'stb_iterate_bwd': [vp, vp, vp, vp, vp],
        'stb_adam_update': [vp, vp, vp, vp, vp, i, i, i, i, i64, f, f, f, f, f, vp],
        'stb_set_loss_ring': [vp, vp, i],
        'stb_resize': [vp, i, i, i, vp, i, i, i, i, vp],
        'stb_snapshot': [vp, i, i, C.c_double, i, vp, vp],
        'stb_resample_tmp_bytes': [i, i, i, i, i, i, C.POINTER(sz)],
        'stb_resample_rgb8': [vp, i, i, i, i, i, i, vp, vp, i, vp, vp, i, vp, sz, vp, vp],
        'stb_comm_create': [vp, i, i, i, i, vp, pp],
        'stb_comm_connect_ipc': [vp, vp],
        'stb_comm_connect_local': [vp, pp],
        'stb_comm_disconnect': [vp],
        'stb_comm_alloc_workspace': [vp, sz, vp, pp, vp],
        'stb_comm_connect_ws_ipc': [vp, vp],
        'stb_comm_connect_ws_local': [vp, pp],
        'stb_comm_release_workspace': [vp, i],
        'stb_comm_set_geometry': [vp, i, i, i, i, i, i, i, i],
        'stb_comm_reset': [vp, vp],
        'stb_iterate_banded': [vp, vp, vp, vp, vp, i64, f, f, f, f, f, vp, vp],
        'stb_iterate_lbfgs_banded': [vp, vp, vp, vp, sz, i64, f, vp, vp],
        'stb_graph_status': [vp, C.c_char_p, sz],
        'stb_launch_count': [vp, C.POINTER(i64), C.POINTER(i64), C.POINTER(i)],
        'stb_profile_enable': [vp, i],
        'stb_profile_read': [vp, C.POINTER(f), C.POINTER(i), i],
        'stb_debug_activation': [vp, i, i, i, vp, sz, vp],
        'stb_debug_w2_trace': [vp, vp, sz, C.POINTER(i)],
    })
    lib.stb_ctx_destroy.argtypes = [vp]
    lib.stb_ctx_destroy.restype = None


def _declare_test(lib):
    vp, i, f, sz = C.c_void_p, C.c_int, C.c_float, C.c_size_t
    pp = C.POINTER(C.c_void_p)
    lib.stb_test_last_error.restype = C.c_char_p
    lib.stb_test_last_error.argtypes = []
    _set(lib, {
        'stb_pack_weights': [vp, vp, i, i, i, vp],
        'stb_test_pixel_gemm': [i, i, i, i, i, i, vp, vp, vp, i, i, vp, vp, vp, vp, vp, f, i, i, vp],
        'stb_test_conv0_fwd': [vp, vp, vp, vp, i, i, f, vp, vp, C.POINTER(i), vp],
        'stb_test_tv': [vp, i, i, i, i, i, f, vp, vp, C.POINTER(i), vp],
        'stb_test_conv0_bwd': [vp, vp, vp, vp, i, i, vp],
        'stb_test_conv0_bwd_adam': [vp, vp, vp, vp, i, i, vp, vp, vp, vp, C.c_int64, f, f, f, f, f, i, vp],
        'stb_test_sse': [vp, vp, C.c_long, vp, C.POINTER(i), vp],
        'stb_test_conv_pool': [i, i, i, i, vp, vp, vp, vp, vp, i, vp],
        'stb_test_pool_bwd': [i, vp, vp, vp, i, i, i, vp],
        'stb_test_gram': [vp, C.c_long, i, vp, sz, vp, vp, vp],
        'stb_test_w2': [vp, vp, vp, vp, i, f, f, vp, sz, vp, vp, vp, vp, vp],
        'stb_test_w2_layers': [pp, pp, pp, pp, C.POINTER(f), C.POINTER(f), i, i, vp, sz, vp, pp, pp, pp, pp, pp, vp],
        'stb_test_lbfgs_step': [vp, sz, i, i, vp, vp, vp, f, C.POINTER(i), C.POINTER(f), vp],
        'stb_test_lbfgs_step_banded': [vp, vp, sz, vp, vp, vp, f, i, C.POINTER(i), C.POINTER(f), vp],
        'stb_test_lbfgs_gradient': [vp, sz, i, i, vp, vp],
        'stb_test_comm_info': [vp, C.POINTER(i), C.POINTER(i), C.POINTER(i)],
    })
    lib.stb_test_preload.argtypes = []
    lib.stb_test_preload.restype = C.c_int
    lib.stb_test_gram_partials_floats.argtypes = [C.c_long, i]
    lib.stb_test_gram_partials_floats.restype = sz
    lib.stb_test_w2_workspace_bytes.argtypes = []
    lib.stb_test_w2_workspace_bytes.restype = sz


# every symbol include/stb200.h declares (tests/test_cpu_host.py checks the library against this list and the header)
EXPORTS = [
    'stb_last_error', 'stb_ctx_create', 'stb_ctx_destroy', 'stb_workspace_bytes', 'stb_bind_workspace',
    'stb_style_stats', 'stb_content_features', 'stb_set_targets', 'stb_iterate', 'stb_iterate_ex',
    'stb_set_layers', 'stb_content_features_ex', 'stb_set_targets_ex', 'stb_loss_terms',
    'stb_lbfgs_state_bytes', 'stb_lbfgs_reset', 'stb_iterate_lbfgs',
    'stb_set_band', 'stb_stats_block', 'stb_iterate_fwd', 'stb_iterate_bwd', 'stb_adam_update',
    'stb_set_loss_ring', 'stb_resize', 'stb_snapshot', 'stb_resample_tmp_bytes', 'stb_resample_rgb8',
    'stb_comm_create', 'stb_comm_connect_ipc', 'stb_comm_connect_local', 'stb_comm_disconnect', 'stb_comm_alloc_workspace',
    'stb_comm_connect_ws_ipc', 'stb_comm_connect_ws_local', 'stb_comm_release_workspace',
    'stb_comm_set_geometry', 'stb_comm_reset',
    'stb_iterate_banded', 'stb_iterate_lbfgs_banded', 'stb_graph_status', 'stb_launch_count', 'stb_profile_enable', 'stb_profile_read', 'stb_debug_activation', 'stb_debug_w2_trace',
]
# include/stb200_test.h (libstb200_test.so)
TEST_EXPORTS = [
    'stb_test_last_error', 'stb_pack_weights', 'stb_test_pixel_gemm', 'stb_test_conv0_fwd', 'stb_test_tv',
    'stb_test_conv0_bwd', 'stb_test_conv0_bwd_adam', 'stb_test_sse', 'stb_test_conv_pool', 'stb_test_pool_bwd', 'stb_test_gram',
    'stb_test_gram_partials_floats', 'stb_test_w2', 'stb_test_w2_layers', 'stb_test_w2_workspace_bytes',
    'stb_test_lbfgs_step', 'stb_test_lbfgs_step_banded',
    'stb_test_lbfgs_gradient', 'stb_test_preload', 'stb_test_comm_info',
]


def load():
    """Load libstb200.so (built in-tree by build.py / __graft_entry__.build())."""
    global _lib
    if _lib is None:
        if not LIB_PATH.exists():
            raise NativeError(f'{LIB_PATH} is missing: build it with `python __graft_entry__.py` '
                              '(there is no CPU or PyTorch fallback for the hot path)')
        lib = C.CDLL(str(LIB_PATH))
        _declare(lib)
        _lib = lib
    return _lib


def load_test():
    """Load libstb200_test.so: the product objects plus the kernel-level hooks of csrc/api_test.cu (tests/ only)."""
    global _tlib
    if _tlib is None:
        if not TEST_LIB_PATH.exists():
            raise NativeError(f'{TEST_LIB_PATH} is missing: build it with `python __graft_entry__.py`')
        lib = C.CDLL(str(TEST_LIB_PATH))
        _declare_test(lib)
        _tlib = lib
    return _tlib


def check(rc: int, test_lib: bool = False):
    if rc != 0:
        msg = (load_test().stb_test_last_error() if test_lib else load().stb_last_error()).decode(errors='replace')
        if rc == STB_ERR_INVALID:
            raise ValueError(msg)
        raise NativeError(f'libstb200 error {rc}: {msg}')


def ptr(t):
    return C.c_void_p(0 if t is None else t.data_ptr())


def ptr_array(tensors):
    arr = (C.c_void_p * len(tensors))(*[t.data_ptr() for t in tensors])
    return C.cast(arr, C.POINTER(C.c_void_p)), arr


def cur_stream():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)
