"""ctypes binding of libwatsor_b200.so (include/watsor_b200.h).  Fails loudly when the
library has not been built -- there is no CPU fallback."""
import ctypes
import os
from ctypes import (POINTER, Structure, c_char_p, c_double, c_float, c_int, c_int32, c_int64, c_size_t,
                    c_uint8, c_uint32, c_uint64, c_void_p)

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'csrc', 'libwatsor_b200.so')

WB_F_FRAMES_ON_DEVICE, WB_F_FUSE_FILTERS, WB_F_OUT_ON_DEVICE = 1, 2, 4
WB_F_YUV420P, WB_F_NV12 = 8, 16
WB_F_YUYV422, WB_F_UYVY422 = 32, 64
WB_F_BGR24, WB_F_RGBA, WB_F_BGRA = 128, 256, 512
WB_V_LABEL, WB_V_CONFIDENCE, WB_V_AREA, WB_V_MASK, WB_V_PASS = 1, 2, 4, 8, 16
WB_CAM_NO_LABEL_CHECK = 1
WB_MAX_WINDOWS = 16


class ClassFilter(Structure):
    _fields_ = [('label', c_int32), ('has_zone_list', c_int32), ('zone_bits', c_uint32),
                ('_pad', c_int32), ('confidence', c_double), ('area', c_double)]


class FramePlanes(Structure):
    """wb_frame_planes: a frame's planes and the bytes between the rows of each (unused planes NULL)"""
    _fields_ = [('plane', c_void_p * 3), ('pitch', c_int64 * 3)]


class WatsorB200Error(RuntimeError):
    pass


_lib = None


def _point_at_bundled_nccl():
    """`wb_comm_*` binds NCCL with dlopen.  If no copy is loaded yet, make it pick the one PyTorch ships
    (site-packages/nvidia/nccl/lib/libnccl.so.2) rather than a different system version with the same SONAME,
    after which `import torch` would fail to resolve its symbols.  No import of torch or nvidia.* happens here."""
    if os.environ.get('WB_NCCL_LIB'):
        return
    import sys
    for base in sys.path:
        cand = os.path.join(base, 'nvidia', 'nccl', 'lib', 'libnccl.so.2')
        if base and os.path.isfile(cand):
            os.environ['WB_NCCL_LIB'] = cand
            return


def load():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.isfile(LIB_PATH):
        raise WatsorB200Error(
            'libwatsor_b200.so is not built (%s). Build it with '
            '`python -c "import __graft_entry__ as g; g.build()"` or `make -C watsor_b200/csrc`. '
            'There is no CPU fallback.' % LIB_PATH)
    _point_at_bundled_nccl()
    lib = ctypes.CDLL(LIB_PATH)
    P = POINTER
    sig = {
        'wb_abi_version': (c_int, []),
        'wb_last_error': (c_char_p, []),
        'wb_device_count': (c_int, [P(c_int)]),
        'wb_create': (c_int, [c_int, c_void_p, c_size_t, c_int, c_int, P(c_void_p)]),
        'wb_destroy': (c_int, [c_void_p]),
        'wb_device_name': (c_int, [c_void_p, c_char_p, c_size_t]),
        'wb_set_stream': (c_int, [c_void_p, c_uint64]),
        'wb_model_info': (c_int, [c_void_p, P(c_int32), P(c_int32), P(c_int32), P(c_int32), P(c_int32)]),
        'wb_set_camera': (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_int,
                                  P(ClassFilter), c_uint32]),
        'wb_set_camera_windows': (c_int, [c_void_p, c_int, c_int, P(c_int32), c_double]),
        'wb_register_host': (c_int, [c_void_p, c_void_p, c_size_t]),
        'wb_unregister_host': (c_int, [c_void_p, c_void_p]),
        'wb_detect': (c_int, [c_void_p, c_int, P(c_void_p), P(c_int32), c_uint32, P(c_void_p),
                              P(c_void_p), P(c_float)]),
        'wb_submit': (c_int, [c_void_p, c_int, c_int, P(c_void_p), P(c_int32), c_uint32]),
        'wb_collect': (c_int, [c_void_p, c_int, P(c_void_p), P(c_void_p), P(c_float)]),
        'wb_detect_planes': (c_int, [c_void_p, c_int, P(FramePlanes), P(c_int32), c_uint32, P(c_void_p),
                                     P(c_void_p), P(c_float)]),
        'wb_submit_planes': (c_int, [c_void_p, c_int, c_int, P(FramePlanes), P(c_int32), c_uint32]),
        'wb_stream_fence': (c_int, [c_void_p, c_uint64, c_int]),
        'wb_comm_unique_id': (c_int, [c_void_p]),
        'wb_comm_init': (c_int, [c_void_p, c_int, c_int, c_void_p]),
        'wb_scatter_frames': (c_int, [c_void_p, c_int, P(c_void_p), c_void_p, c_size_t, c_uint64]),
        'wb_comm_destroy': (c_int, [c_void_p]),
        'wb_preprocess': (c_int, [c_void_p, c_int, P(c_void_p), P(c_int32), P(c_int32), c_void_p]),
        'wb_backbone': (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_size_t]),
        'wb_backbone_frames': (c_int, [c_void_p, c_int, P(c_void_p), P(c_int32), c_uint32, c_void_p, c_void_p, c_int,
                                       c_void_p, c_size_t, P(c_int32)]),
        'wb_postprocess': (c_int, [c_void_p, c_int, c_void_p, c_void_p, P(c_int32), c_uint32,
                                   P(c_void_p), P(c_void_p), c_void_p, c_void_p, c_void_p, c_void_p]),
        'wb_filter_rows': (c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p]),
        'wb_anchors': (c_int, [c_void_p, c_void_p]),
        'wb_last_launch_count': (c_int, [c_void_p, P(c_int)]),
        'wb_profile_layers': (c_int, [c_void_p, c_int, P(c_void_p), P(c_int32), P(c_float),
                                      P(c_int32), c_int, P(c_int)]),
        'wb_tracker_create': (c_int, [c_int, c_int, P(c_void_p)]),
        'wb_tracker_destroy': (c_int, [c_void_p]),
        'wb_tracker_update': (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_int, P(c_int), P(c_int)]),
        'wb_sieve_rows': (c_int, [c_void_p, c_void_p, c_int, c_void_p, P(c_int)]),
        'wb_debug_pyset_order': (c_int, [P(c_int32), c_int, P(c_int32), P(c_int)]),
        'wb_debug_unused_order': (c_int, [c_int, c_void_p, P(c_int32), P(c_int)]),
        'wb_debug_argsort': (c_int, [c_void_p, c_int, P(c_int32)]),
        'wb_fx_create': (c_int, [c_int, c_void_p, c_int, c_void_p, c_void_p, c_double, P(c_void_p)]),
        'wb_fx_set_camera': (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]),
        'wb_fx_render': (c_int, [c_void_p, c_int, P(c_void_p), P(c_void_p), P(c_int32), P(c_void_p), c_uint32,
                                 P(c_float)]),
        'wb_fx_destroy': (c_int, [c_void_p]),
        'wb_fx_last_error': (c_char_p, []),
    }
    for name, (res, args) in sig.items():
        fn = getattr(lib, name)       # AttributeError if the header and the library disagree
        fn.restype = res
        fn.argtypes = args
    if lib.wb_abi_version() != 1:
        raise WatsorB200Error('libwatsor_b200.so ABI version mismatch')
    _lib = lib
    return lib


EXPORTS = ['wb_abi_version', 'wb_last_error', 'wb_device_count', 'wb_create', 'wb_destroy',
           'wb_device_name', 'wb_set_stream', 'wb_model_info', 'wb_set_camera', 'wb_set_camera_windows',
           'wb_register_host',
           'wb_unregister_host', 'wb_detect', 'wb_submit', 'wb_collect', 'wb_detect_planes', 'wb_submit_planes',
           'wb_stream_fence', 'wb_comm_unique_id', 'wb_comm_init',
           'wb_scatter_frames', 'wb_comm_destroy', 'wb_preprocess', 'wb_backbone', 'wb_backbone_frames',
           'wb_postprocess', 'wb_filter_rows', 'wb_anchors', 'wb_last_launch_count', 'wb_profile_layers',
           'wb_tracker_create', 'wb_tracker_destroy', 'wb_tracker_update', 'wb_sieve_rows', 'wb_debug_pyset_order',
           'wb_debug_unused_order', 'wb_debug_argsort', 'wb_fx_create', 'wb_fx_set_camera', 'wb_fx_render',
           'wb_fx_destroy', 'wb_fx_last_error']


def check(rc):
    if rc != 0:
        raise WatsorB200Error(load().wb_last_error().decode(errors='replace'))


def device_count():
    n = c_int(0)
    check(load().wb_device_count(ctypes.byref(n)))
    return n.value
