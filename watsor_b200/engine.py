"""Thin object wrapper over the C-ABI context (`wb_ctx`, include/watsor_b200.h).

Host code stays Python, as in the reference; every numeric step happens inside
libwatsor_b200.so.  numpy arrays are only argument carriers (frames in, rows out).
"""
import ctypes
from ctypes import POINTER, byref, c_char_p, c_float, c_int, c_int32, c_uint32, c_void_p, cast

import numpy as np

from . import _lib
from ._lib import ClassFilter, check
from .windows import check_windows
from .stream.share import MAX_DETECTIONS, Detection

# wb_create's precision by name (include/watsor_b200.h): fp32 CUDA-core convs; bf16 wgmma; fp32 storage with the dense
# convs as 3xTF32 wgmma (fp32-faithful); 1xTF32 wgmma (diagnostic); fp16 wgmma, activations saturated at +-65504
PRECISIONS = {'fp32': 0, 'bf16': 1, 'tf32x3': 2, 'tf32x1': 3, 'fp16': 4}
PRECISION_FP32, PRECISION_BF16_TC = PRECISIONS['fp32'], PRECISIONS['bf16']
PRECISION_TF32X3, PRECISION_FP16_TC = PRECISIONS['tf32x3'], PRECISIONS['fp16']

# frame layouts the hot path reads, by ffmpeg's -pix_fmt names -> wb_detect / wb_submit flag: RGB24 and YUV ...
PIXEL_FORMATS = {'rgb24': 0, 'yuv420p': _lib.WB_F_YUV420P, 'nv12': _lib.WB_F_NV12,
                 'yuyv422': _lib.WB_F_YUYV422, 'uyvy422': _lib.WB_F_UYVY422}
# ... and the other packed RGB byte orders: BGR24 (OpenCV's frames) and the 4-byte RGBA / BGRA (also rgb0 / bgr0, the
# fourth byte is not read), read as the RGB24 frame cv2.cvtColor makes of them.  Every function here that takes a
# pixel_format accepts these as well, except frame_shape, which keeps its contract (layout_shape covers every layout);
# PIXEL_FORMATS keeps listing the layouts it always listed.
RGB_ORDERS = {'bgr24': _lib.WB_F_BGR24, 'rgba': _lib.WB_F_RGBA, 'bgra': _lib.WB_F_BGRA}
# every layout, by name -> flag
FRAME_FORMATS = dict(PIXEL_FORMATS, **RGB_ORDERS)
_BYTES_PER_PIXEL = {'rgb24': 3, 'bgr24': 3, 'rgba': 4, 'bgra': 4}


def _check_format(pixel_format, formats=FRAME_FORMATS):
    if pixel_format not in formats:
        raise ValueError('pixel_format must be one of %s, not %r%s' % (
            ', '.join(formats), pixel_format,
            ' (engine.layout_shape gives the shape of a %s frame)' % pixel_format if pixel_format in FRAME_FORMATS else ''))


def layout_shape(pixel_format, width, height):
    """numpy shape of one packed uint8 frame of a `width` x `height` camera in any layout of FRAME_FORMATS: (H, W, 3)
    for rgb24 and bgr24, (H, W, 4) for rgba and bgra, (H*3//2, W) for the 4:2:0 formats (luma plane, then the chroma;
    include/watsor_b200.h), which need an even width and height, and (H, W, 2) for the packed 4:2:2 formats (the shape
    cv2.cvtColor takes), which need an even width.  The same shapes hold for the frames the effects pass reads and
    writes (output.effects, `output_format`)."""
    _check_format(pixel_format)
    if pixel_format in _BYTES_PER_PIXEL:
        return (height, width, _BYTES_PER_PIXEL[pixel_format])
    if pixel_format in ('yuyv422', 'uyvy422'):
        if width % 2:
            raise ValueError('%s frames need an even width; the camera is %dx%d' % (pixel_format, width, height))
        return (height, width, 2)
    if width % 2 or height % 2:
        raise ValueError('%s frames need an even width and height; the camera is %dx%d' % (pixel_format, width, height))
    return (height * 3 // 2, width)


def layout_planes(pixel_format, width, height):
    """(rows, row bytes) of each plane of a `width` x `height` frame in `pixel_format`, in the order wb_frame_planes
    takes them (include/watsor_b200.h): one plane for the RGB byte orders and the packed 4:2:2 formats, the pixel rows;
    two for nv12, Y and the interleaved (U, V) pairs; three for yuv420p, Y, U and V.  The sizes layout_shape refuses
    are refused here too."""
    layout_shape(pixel_format, width, height)
    if pixel_format in _BYTES_PER_PIXEL:
        return ((height, width * _BYTES_PER_PIXEL[pixel_format]),)
    if pixel_format in ('yuyv422', 'uyvy422'):
        return ((height, width * 2),)
    if pixel_format == 'nv12':
        return ((height, width), (height // 2, width))
    return ((height, width), (height // 2, width // 2), (height // 2, width // 2))


def plane_address(plane, rows, row_bytes, on_device, where):
    """(address, pitch) of one plane of a frame given as planes.  `plane` is a uint8 numpy array or torch tensor whose
    first dimension counts the plane's `rows` and whose other dimensions hold one row's `row_bytes` densely (a view
    such as big[y0:y1, x0:x1] qualifies): the pitch is the first dimension's stride.  Device planes
    (`on_device`) are CUDA tensors or (address, pitch) pairs from any other library, which the C library checks.
    rows None: a camera this engine does not know, whose size the library checks.  Raises ValueError naming `where`."""
    if isinstance(plane, tuple):
        if not on_device:
            raise ValueError('%s: an (address, pitch) pair is a device plane; pass frames_on_device=True' % where)
        if len(plane) != 2:
            raise ValueError('%s: a device plane is an (address, pitch) pair, not %d values' % (where, len(plane)))
        return int(plane[0]), int(plane[1])
    if isinstance(plane, np.ndarray):
        if on_device:
            raise ValueError('%s: a numpy array is host memory, but frames_on_device is set' % where)
        dtype_ok, shape, strides, addr = plane.dtype == np.uint8, plane.shape, plane.strides, plane.ctypes.data
    elif type(plane).__module__.split('.')[0] == 'torch':
        import torch
        if plane.is_cuda != bool(on_device):
            raise ValueError('%s: a %s tensor, but frames_on_device is %s' % (
                where, 'CUDA' if plane.is_cuda else 'CPU', bool(on_device)))
        dtype_ok, shape, strides = plane.dtype == torch.uint8, tuple(plane.shape), plane.stride()
        addr = plane.data_ptr()
    else:
        raise ValueError('%s: a plane is a uint8 numpy array or torch tensor%s, not %s' % (
            where, ' or an (address, pitch) pair' if on_device else '', type(plane).__name__))
    if not dtype_ok or len(shape) < 1:
        raise ValueError('%s: a plane is a uint8 array of at least one dimension, not %s of shape %s' % (
            where, getattr(plane, 'dtype', '?'), shape))
    dense, step = True, 1
    for n, st in reversed(list(zip(shape[1:], strides[1:]))):
        dense &= n == 1 or st == step
        step *= n
    if not dense:
        raise ValueError('%s: the bytes of a row must be dense (strides %s for shape %s)' % (where, strides, shape))
    if rows is not None and (shape[0] != rows or step != row_bytes):
        raise ValueError('%s: %d rows of %d bytes expected, not %d rows of %d bytes (shape %s)' % (
            where, rows, row_bytes, shape[0], step, shape))
    pitch = strides[0] if shape[0] > 1 or strides[0] >= step else step    # numpy may give one row any stride
    if pitch < step:
        raise ValueError('%s: the row pitch %d is below the row bytes %d (rows overlap or run bottom-up)' % (
            where, pitch, step))
    return addr, pitch


def frame_shape(pixel_format, width, height):
    """layout_shape for the RGB24 and YUV layouts of PIXEL_FORMATS, the names this function has always taken; it
    refuses the other RGB byte orders (bgr24, rgba, bgra) as it always has, and layout_shape gives their shapes."""
    _check_format(pixel_format, PIXEL_FORMATS)
    return layout_shape(pixel_format, width, height)


def check_frames(frames, sizes, pixel_format):
    """Raises ValueError unless every numpy frame is a C-contiguous uint8 array of `layout_shape` for its camera's
    (width, height) in `sizes`.  A size of None (a camera unknown here, which the library reports) and raw addresses
    are passed through unchecked."""
    _check_format(pixel_format)
    for i, (frame, size) in enumerate(zip(frames, sizes)):
        if size is None:
            continue
        shape = layout_shape(pixel_format, *size)
        if isinstance(frame, np.ndarray) and (frame.dtype != np.uint8 or frame.shape != shape or
                                              not frame.flags['C_CONTIGUOUS']):
            raise ValueError('frame %d: a %s frame of a %dx%d camera is a C-contiguous uint8 array of shape %s, not %s %s%s'
                             % (i, pixel_format, size[0], size[1], shape, frame.dtype, frame.shape,
                                '' if frame.flags['C_CONTIGUOUS'] else ' (not C-contiguous)'))


def _ptr_array(ptrs):
    arr = (c_void_p * len(ptrs))()
    for i, p in enumerate(ptrs):
        arr[i] = p
    return arr


def _addr(obj):
    """Address of a numpy array / ctypes object / raw integer (device pointer)."""
    if obj is None:
        return None
    if isinstance(obj, int):
        return obj
    if isinstance(obj, np.ndarray):
        assert obj.flags['C_CONTIGUOUS'], 'arrays handed to libwatsor_b200 must be C-contiguous'
        return obj.ctypes.data
    return ctypes.addressof(obj)


class Engine:
    """One `wb_ctx`: a model resident on one H100 plus per-camera filter tables."""

    def __init__(self, model_blob, device=0, max_batch=8, precision=PRECISION_FP32):
        self.lib = _lib.load()
        self._blob = bytes(model_blob)       # keep alive during wb_create
        self._ctx = c_void_p()
        check(self.lib.wb_create(device, self._blob, len(self._blob), max_batch, precision,
                                 byref(self._ctx)))
        self.device = device
        self.max_batch = max_batch
        self.precision = precision
        ih, iw, nc, na, nl = (c_int32() for _ in range(5))
        check(self.lib.wb_model_info(self._ctx, byref(ih), byref(iw), byref(nc), byref(na), byref(nl)))
        self.input_h, self.input_w = ih.value, iw.value
        self.num_classes, self.num_anchors, self.num_layers = nc.value, na.value, nl.value
        self.cameras = {}
        self.windows = {}                       # cam_id -> [(x, y, w, h)] (set_camera_windows)

    # ------------------------------------------------------------------ life cycle
    def close(self):
        if self._ctx:
            self.lib.wb_destroy(self._ctx)
            self._ctx = c_void_p()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def device_name(self):
        buf = ctypes.create_string_buffer(255)
        check(self.lib.wb_device_name(self._ctx, buf, 255))
        return buf.value.decode()

    def set_stream(self, cuda_stream):
        check(self.lib.wb_set_stream(self._ctx, int(cuda_stream)))

    # ------------------------------------------------------------------- cameras
    def set_camera(self, cam_id, width, height, zone_rasters=None, class_filters=(), flags=0):
        """class_filters: iterable of (label, confidence, area, zones or None).  label -1 = default."""
        arr = (ClassFilter * max(1, len(class_filters)))()
        for i, (label, conf, area, zones) in enumerate(class_filters):
            bits = 0
            for z in (zones or ()):
                bits |= 1 << (z - 1)
            arr[i] = ClassFilter(label, 1 if zones else 0, bits, 0, conf, area)
        n_zones = 0
        raster_ptr = None
        dummy = np.zeros(1, np.uint8)          # stays alive until wb_set_camera has returned
        if zone_rasters is not None:
            zone_rasters = np.ascontiguousarray(zone_rasters, dtype=np.uint8)
            assert zone_rasters.ndim == 3 and zone_rasters.shape[1:] == (height, width)
            n_zones = zone_rasters.shape[0]
            # a mask without any zone is still "has_mask" (MaskFilter would reject everything)
            raster_ptr = zone_rasters.ctypes.data if n_zones else dummy.ctypes.data
        check(self.lib.wb_set_camera(self._ctx, cam_id, width, height, n_zones, raster_ptr,
                                     len(class_filters), arr, flags))
        self.cameras[cam_id] = (width, height)
        self.windows.pop(cam_id, None)          # the library clears them too: the frame size may have changed

    def set_camera_windows(self, cam_id, windows, merge_threshold=0.5):
        """Detection windows of a configured camera: (x, y, w, h) rectangles in its pixels (see windows.grid_windows),
        each of which becomes one model image per frame; max_batch counts model images.  The windows' rows are merged
        into the frame's 100 rows: a row is dropped when a kept row of the same label from another window covers more
        than `merge_threshold` of the smaller box.  An empty list removes the windows."""
        if cam_id not in self.cameras:
            raise ValueError('camera %r has not been configured with set_camera' % (cam_id,))
        windows = check_windows(windows, *self.cameras[cam_id])
        if not 0.0 <= merge_threshold <= 1.0:
            raise ValueError('merge_threshold must be in [0, 1], not %r' % (merge_threshold,))
        xywh = (c_int32 * max(1, 4 * len(windows)))(*[v for win in windows for v in win])
        check(self.lib.wb_set_camera_windows(self._ctx, cam_id, len(windows), xywh, float(merge_threshold)))
        if windows:
            self.windows[cam_id] = windows
        else:
            self.windows.pop(cam_id, None)

    def register_host(self, address, nbytes):
        check(self.lib.wb_register_host(self._ctx, address, nbytes))

    def unregister_host(self, address):
        check(self.lib.wb_unregister_host(self._ctx, address))

    # ------------------------------------------------------------------ hot path
    def _frame_planes(self, frames, cam_ids, pixel_format, on_device):
        """wb_frame_planes of a batch with at least one frame given as a tuple of planes (see plane_address); the
        batch's packed frames become the planes at their packed offsets"""
        arr = (_lib.FramePlanes * len(frames))()
        for i, (frame, cam) in enumerate(zip(frames, cam_ids)):
            size = self.cameras.get(cam)
            layout = layout_planes(pixel_format, *size) if size is not None else None
            if isinstance(frame, tuple):
                if layout is not None and len(frame) != len(layout):
                    raise ValueError('frame %d: a %s frame has %d plane%s, not %d' % (
                        i, pixel_format, len(layout), 's' if len(layout) > 1 else '', len(frame)))
                for k, plane in enumerate(frame[:3]):
                    rows, row_bytes = layout[k] if layout is not None else (None, None)
                    where = 'frame %d (%s) plane %d' % (i, pixel_format, k)
                    arr[i].plane[k], arr[i].pitch[k] = plane_address(plane, rows, row_bytes, on_device, where)
                continue
            if isinstance(frame, np.ndarray) and on_device:
                raise ValueError('frame %d: a numpy array is host memory, but frames_on_device is set' % i)
            addr = _addr(frame)
            offset = 0
            for k, (rows, row_bytes) in enumerate(layout or ((0, 0),)):
                arr[i].plane[k], arr[i].pitch[k] = addr + offset, row_bytes
                offset += rows * row_bytes
        return arr

    def _io(self, frames, cam_ids, out, verdicts, pixel_format='rgb24', flags=0):
        """ctypes arguments of a batch; fp is a wb_frame_planes array when a frame is a tuple of planes, else the
        frames' addresses"""
        n = len(frames)
        assert n == len(cam_ids)
        if any(isinstance(f, tuple) for f in frames):
            fp = self._frame_planes(frames, cam_ids, pixel_format, flags & _lib.WB_F_FRAMES_ON_DEVICE)
        else:
            fp = _ptr_array([_addr(f) for f in frames])
        cams = (c_int32 * n)(*cam_ids)
        op = _ptr_array([_addr(o) for o in out]) if out is not None else None
        vp = _ptr_array([_addr(v) for v in verdicts]) if verdicts is not None else None
        return n, fp, cams, op, vp

    def _format_flags(self, frames, cam_ids, pixel_format):
        check_frames(frames, [self.cameras.get(c) for c in cam_ids], pixel_format)
        for c in set(cam_ids):
            if c in self.windows:
                check_windows(self.windows[c], *self.cameras[c], pixel_format)
        return FRAME_FORMATS[pixel_format]

    def detect(self, frames, cam_ids, out, verdicts=None, flags=0, pixel_format='rgb24'):
        """frames: host uint8 arrays (or device pointers with WB_F_FRAMES_ON_DEVICE) in `pixel_format`
        (a name of FRAME_FORMATS: 'rgb24', 'bgr24', 'rgba', 'bgra', 'yuv420p', 'nv12', 'yuyv422' or 'uyvy422', see
        layout_shape); out: per frame a `Detection*100` ctypes array / address.  A frame may also be a tuple of its
        planes (layout_planes), each an array or tensor with row padding of its own or an (address, pitch) pair on
        the device (plane_address): decoder surfaces and ffmpeg frames, read without packing them first.
        Returns device ms."""
        flags |= self._format_flags(frames, cam_ids, pixel_format)
        n, fp, cams, op, vp = self._io(frames, cam_ids, out, verdicts, pixel_format, flags)
        ms = c_float(0)
        fn = self.lib.wb_detect_planes if fp._type_ is _lib.FramePlanes else self.lib.wb_detect
        check(fn(self._ctx, n, fp, cams, flags, op, vp, byref(ms)))
        return ms.value

    def submit(self, slot, frames, cam_ids, flags=0, pixel_format='rgb24'):
        """`detect`'s frames, enqueued on `slot`; `collect` returns the results.  The frames, and every plane of a
        frame given as planes, must stay valid until then."""
        flags |= self._format_flags(frames, cam_ids, pixel_format)
        n, fp, cams, _, _ = self._io(frames, cam_ids, None, None, pixel_format, flags)
        fn = self.lib.wb_submit_planes if fp._type_ is _lib.FramePlanes else self.lib.wb_submit
        check(fn(self._ctx, slot, n, fp, cams, flags))

    def collect(self, slot, out=None, verdicts=None):
        op = _ptr_array([_addr(o) for o in out]) if out is not None else None
        vp = _ptr_array([_addr(v) for v in verdicts]) if verdicts is not None else None
        ms = c_float(0)
        check(self.lib.wb_collect(self._ctx, slot, op, vp, byref(ms)))
        return ms.value

    def stream_fence(self, cuda_stream, direction):
        """direction 0: slot streams wait for `cuda_stream`; 1: `cuda_stream` waits for the slots."""
        check(self.lib.wb_stream_fence(self._ctx, int(cuda_stream), direction))

    # --------------------------------------------------------------- frame scatter (NCCL behind the C-ABI)
    def comm_unique_id(self):
        """128-byte rendezvous id; the root rank makes it and ships it to the others over any host channel."""
        buf = (ctypes.c_uint8 * 128)()
        check(self.lib.wb_comm_unique_id(buf))
        return bytes(buf)

    def comm_init(self, rank, world, unique_id):
        """Collective over the `world` engines (one per process / GPU)."""
        assert len(unique_id) == 128
        buf = (ctypes.c_uint8 * 128).from_buffer_copy(unique_id)
        check(self.lib.wb_comm_init(self._ctx, rank, world, buf))

    def scatter_frames(self, root, send_ptrs, recv_ptr, nbytes, cuda_stream=0):
        """send_ptrs: on the root, one device pointer per rank (that rank's `nbytes` slab), else None; recv_ptr:
        this rank's device buffer.  cuda_stream 0: later submits on this engine are ordered after the scatter."""
        sp = _ptr_array(send_ptrs) if send_ptrs is not None else None
        check(self.lib.wb_scatter_frames(self._ctx, root, sp, c_void_p(int(recv_ptr)), nbytes, int(cuda_stream)))

    def comm_destroy(self):
        check(self.lib.wb_comm_destroy(self._ctx))

    # --------------------------------------------------------------- stage level
    def preprocess(self, frames):
        n = len(frames)
        fp = _ptr_array([_addr(np.ascontiguousarray(f)) for f in frames])
        w = (c_int32 * n)(*[f.shape[1] for f in frames])
        h = (c_int32 * n)(*[f.shape[0] for f in frames])
        out = np.empty((n, self.input_h, self.input_w, 3), np.float32)
        check(self.lib.wb_preprocess(self._ctx, n, fp, w, h, out.ctypes.data))
        return out

    def backbone(self, pre, stop_layer=-1, layer_shape=None):
        pre = np.ascontiguousarray(pre, dtype=np.float32)
        n = pre.shape[0]
        enc = np.empty((n, self.num_anchors, 4), np.float32)
        logits = np.empty((n, self.num_anchors, self.num_classes + 1), np.float32)
        layer_out = None
        if stop_layer >= 0 and layer_shape is not None:
            layer_out = np.empty((n,) + tuple(layer_shape), np.float32)
        check(self.lib.wb_backbone(self._ctx, n, pre.ctypes.data, enc.ctypes.data, logits.ctypes.data,
                                   stop_layer, layer_out.ctypes.data if layer_out is not None else None,
                                   layer_out.size if layer_out is not None else 0))
        return enc, logits, layer_out

    def backbone_frames(self, frames, cam_ids, stop_layer=-1, layer_shape=None, pixel_format='rgb24',
                        frames_on_device=False, flags=0):
        """`backbone` fed as the product path is: frames as `detect` takes them (host arrays, or device pointers with
        frames_on_device), each camera's detection windows expanded into model images.  stop_layer -1 runs `submit`'s
        kernels (CUDA graph, post stage, window merge) on slot 0.  Returns (enc, logits, layer_out, n_images); the head
        buffers are returned as the run left them, without being cleared first."""
        flags |= self._format_flags(frames, cam_ids, pixel_format)
        if frames_on_device:
            flags |= _lib.WB_F_FRAMES_ON_DEVICE
        windowed = any(c in self.windows for c in cam_ids)
        n_img = sum(max(len(self.windows.get(c, ())), 1) for c in cam_ids) if windowed else len(cam_ids)
        n, fp, cams, _, _ = self._io(frames, cam_ids, None, None)
        enc = np.empty((n_img, self.num_anchors, 4), np.float32)
        logits = np.empty((n_img, self.num_anchors, self.num_classes + 1), np.float32)
        layer_out = None
        if stop_layer >= 0 and layer_shape is not None:
            layer_out = np.empty((n_img,) + tuple(layer_shape), np.float32)
        got = c_int32(0)
        check(self.lib.wb_backbone_frames(self._ctx, n, fp, cams, flags, enc.ctypes.data, logits.ctypes.data,
                                          stop_layer, layer_out.ctypes.data if layer_out is not None else None,
                                          layer_out.size if layer_out is not None else 0, byref(got)))
        assert got.value == n_img, (got.value, n_img)
        return enc, logits, layer_out, got.value

    def postprocess(self, enc, logits, cam_ids, flags=0):
        enc = np.ascontiguousarray(enc, dtype=np.float32)
        logits = np.ascontiguousarray(logits, dtype=np.float32)
        n = enc.shape[0]
        rows = [(Detection * MAX_DETECTIONS)() for _ in range(n)]
        verd = np.zeros((n, MAX_DETECTIONS), np.uint32)
        boxes = np.empty((n, MAX_DETECTIONS, 4), np.float32)
        scores = np.empty((n, MAX_DETECTIONS), np.float32)
        classes = np.empty((n, MAX_DETECTIONS), np.float32)
        num = np.empty(n, np.int32)
        check(self.lib.wb_postprocess(
            self._ctx, n, enc.ctypes.data, logits.ctypes.data, (c_int32 * n)(*cam_ids), flags,
            _ptr_array([ctypes.addressof(r) for r in rows]),
            _ptr_array([verd[i].ctypes.data for i in range(n)]), boxes.ctypes.data, scores.ctypes.data,
            classes.ctypes.data, num.ctypes.data))
        return rows, verd, boxes, scores, classes, num

    def filter_rows(self, cam_id, rows, n_rows=None):
        """rows: ctypes Detection array (updated in place).  Returns uint32 verdicts."""
        n = n_rows if n_rows is not None else len(rows)
        verd = np.zeros(n, np.uint32)
        check(self.lib.wb_filter_rows(self._ctx, cam_id, n, ctypes.addressof(rows), verd.ctypes.data))
        return verd

    def anchors(self):
        out = np.empty((self.num_anchors, 4), np.float32)
        check(self.lib.wb_anchors(self._ctx, out.ctypes.data))
        return out

    def last_launch_count(self):
        n = c_int(0)
        check(self.lib.wb_last_launch_count(self._ctx, byref(n)))
        return n.value

    def profile_layers(self, device_frames, cam_ids):
        n = len(device_frames)
        cap = self.num_layers + 8
        ms = (c_float * cap)()
        kinds = (c_int32 * cap)()
        cnt = c_int(0)
        check(self.lib.wb_profile_layers(self._ctx, n, _ptr_array(list(device_frames)),
                                         (c_int32 * n)(*cam_ids), ms, kinds, cap, byref(cnt)))
        return [(kinds[i], ms[i]) for i in range(cnt.value)]
