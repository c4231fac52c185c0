"""ctypes binding of include/fastdepth_b200.h -- the only way Python reaches the kernels.

Fails loudly: if libfastdepth_b200.so is missing or a symbol is absent, importing the
binding raises; there is no PyTorch/CPU fallback behind it.
"""
import ctypes
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get('FD_B200_LIB') or os.path.join(HERE, 'libfastdepth_b200.so')   # env: developer A/B of kernel variants

FD_F32, FD_F16, FD_BF16 = 0, 1, 2
FD_STAGE_STEM, FD_STAGE_DWPW, FD_STAGE_HEAD, FD_STAGE_CONV, FD_STAGE_DECONV, FD_STAGE_UPCONV = 0, 1, 2, 3, 4, 5
FD_ACT_RELU, FD_ACT_RELU6 = 0, 1


class StageDesc(ctypes.Structure):
    """fd_stage_desc"""
    _fields_ = [(n, ctypes.c_int32) for n in
                ('kind', 'c_in', 'c_out', 'ksize', 'stride', 'act', 'upsample', 'skip_src', 'skip_mode')]


_c_int_p = ctypes.POINTER(ctypes.c_int)
_c_float_p = ctypes.POINTER(ctypes.c_float)
_c_double_p = ctypes.POINTER(ctypes.c_double)
_vp = ctypes.c_void_p

# name -> (restype, argtypes): must list EVERY function include/fastdepth_b200.h declares
# (tests/test_abi.py parses the header and compares).
SIGNATURES = {
    'fd_abi_version': (ctypes.c_int, []),
    'fd_last_error': (ctypes.c_char_p, []),
    'fd_plan_create': (ctypes.c_int, [ctypes.POINTER(StageDesc), ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                      ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.POINTER(_vp)]),
    'fd_plan_set_stage_weights': (ctypes.c_int, [_vp, ctypes.c_int, _vp, _vp, _vp, _vp, _vp, _vp]),
    'fd_plan_set_option': (ctypes.c_int, [_vp, ctypes.c_char_p, ctypes.c_int]),
    'fd_plan_get_option': (ctypes.c_int, [_vp, ctypes.c_char_p, _c_int_p]),
    'fd_forward': (ctypes.c_int, [_vp, _vp, _vp, _vp]),
    'fd_forward_batch': (ctypes.c_int, [_vp, ctypes.c_int, _vp, _vp, _vp]),
    'fd_forward_shape': (ctypes.c_int, [_vp, ctypes.c_int, ctypes.c_int, ctypes.c_int, _vp, _vp, _vp]),
    'fd_forward_host': (ctypes.c_int, [_vp, _vp, _vp, _vp]),
    'fd_pipeline_submit': (ctypes.c_int, [_vp, _vp, _vp, ctypes.POINTER(ctypes.c_uint64)]),
    'fd_pipeline_wait': (ctypes.c_int, [_vp, ctypes.c_uint64]),
    'fd_stage_buffer': (ctypes.c_int, [_vp, ctypes.c_int, ctypes.c_int, ctypes.POINTER(_vp),
                                       _c_int_p, _c_int_p, _c_int_p, _c_int_p, _c_int_p]),
    'fd_plan_launches_per_forward': (ctypes.c_int, [_vp, _c_int_p]),
    'fd_plan_workspace_bytes': (ctypes.c_int, [_vp, ctypes.POINTER(ctypes.c_size_t)]),
    'fd_plan_step_count': (ctypes.c_int, [_vp, _c_int_p]),
    'fd_plan_step_info': (ctypes.c_int, [_vp, ctypes.c_int, _c_int_p, _c_double_p, _c_double_p,
                                         ctypes.c_char_p, ctypes.c_int]),
    'fd_plan_step_macs': (ctypes.c_int, [_vp, ctypes.c_int, _c_double_p, _c_double_p]),
    'fd_plan_time_steps': (ctypes.c_int, [_vp, _vp, _vp, _vp, ctypes.c_int, ctypes.c_int, ctypes.c_int, _c_float_p]),
    'fd_plan_trace_stage': (ctypes.c_int, [_vp, ctypes.c_int, _vp, _vp, ctypes.POINTER(ctypes.c_uint64), ctypes.c_int,
                                           _c_int_p, _c_int_p]),
    'fd_debug_block_plan': (ctypes.c_int, [ctypes.c_int] * 8 + [_c_int_p, ctypes.c_int]),
    'fd_debug_conv_plan': (ctypes.c_int, [ctypes.c_int] * 7 + [_c_int_p, ctypes.c_int]),
    'fd_debug_front_plan': (ctypes.c_int, [_vp, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                           _c_int_p, ctypes.c_int]),
    'fd_debug_convt_plan': (ctypes.c_int, [ctypes.c_int] * 8 + [_c_int_p, ctypes.c_int]),
    'fd_debug_pw_tf32x3_plan': (ctypes.c_int, [ctypes.c_int] * 7 + [_c_int_p, ctypes.c_int]),
    'fd_debug_pw_plan': (ctypes.c_int, [ctypes.c_int] * 7 + [_c_int_p, ctypes.c_int]),
    'fd_debug_conv_tf32x3_plan': (ctypes.c_int, [ctypes.c_int] * 9 + [_c_int_p, ctypes.c_int]),
    'fd_metrics_accumulate': (ctypes.c_int, [_vp, _vp, ctypes.c_int, ctypes.c_int, ctypes.c_int, _vp,
                                             ctypes.c_int, _vp]),
    'fd_nyu_val_gather': (ctypes.c_int, [_vp, _vp, _vp, _vp] + [ctypes.c_int] * 6 + [_vp, _vp, ctypes.c_int, _vp]),
    'fd_plan_destroy': (None, [_vp]),
}

_lib = None


def load():
    """Load the shared library (once) and bind every symbol; raises if anything is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            "fastdepth_b200: %s not found. Build it with `python -m fastdepth_b200.build` "
            "(or __graft_entry__.build()); there is no fallback path." % LIB_PATH)
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)          # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    if lib.fd_abi_version() != 2:
        raise RuntimeError('fastdepth_b200: ABI version mismatch')
    _lib = lib
    return lib


def check(rc):
    if rc != 0:
        msg = load().fd_last_error()
        raise RuntimeError('fastdepth_b200 error %d: %s' % (rc, msg.decode() if msg else ''))
