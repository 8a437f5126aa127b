"""B200ObjectDetector -- the detector plugin for NVIDIA H100 (sm_90a).

Implements the duck-typed Detector protocol every reference back-end provides
(watsor/detection/tensorflow_cpu.py:8-92, tensorrt_gpu.py:15-91):

    __init__(model_path[, device]);  context manager;  `device_name`;
    detect(image_shape, image_np, detections) -> inference time in ms

and adds the batched form the GPU needs to be busy: one call per tick for all cameras
(`detect_batch`, `submit`/`collect`), with the confidence / area / mask-zone predicates of
watsor/filter fused behind the NMS.  Model selection follows tensorflow_cpu.py:50-53:
`frozen_inference_graph.pb`, else `cpu.pb`, in `model_path` (a pre-compiled `b200.wb200`
wins when present).
"""
import ctypes
import os

import numpy as np

from .. import _lib
from ..engine import PRECISION_BF16_TC, PRECISION_FP16_TC, PRECISION_FP32, PRECISION_TF32X3, PRECISIONS, Engine
from ..model import Model, compile_frozen_graph
from ..stream.share import MAX_DETECTIONS, Detection

MODEL_FILES = ('frozen_inference_graph.pb', 'cpu.pb')
COMPILED_MODEL = 'b200.wb200'


def find_model(model_path):
    """-> ('blob'|'graph', path).  Raises FileNotFoundError like the reference back-ends do
    (the worker turns it into a logged error, detector.py:97-98)."""
    if os.path.isfile(model_path):
        return ('blob' if model_path.endswith('.wb200') else 'graph'), model_path
    compiled = os.path.join(model_path, COMPILED_MODEL)
    if os.path.isfile(compiled):
        return 'blob', compiled
    for name in MODEL_FILES:
        p = os.path.join(model_path, name)
        if os.path.isfile(p):
            return 'graph', p
    raise FileNotFoundError('No {} / {} / {} in {}'.format(COMPILED_MODEL, MODEL_FILES[0], MODEL_FILES[1],
                                                          model_path))


def load_model_blob(model_path):
    kind, path = find_model(model_path)
    if kind == 'blob':
        with open(path, 'rb') as f:
            return f.read()
    return compile_frozen_graph(path).to_blob()


def default_precision():
    """`WATSOR_B200_PRECISION=fp32|tf32x3|bf16|fp16` (or the diagnostic `tf32x1`; the reference's analogous switch is
    TRT_FLOAT_PRECISION, main_for_gpu.py:24).  Default: fp32-faithful tensor-core mode.  `16` selects bf16, as it
    always has; IEEE half is `fp16` (or `half`)."""
    v = os.environ.get('WATSOR_B200_PRECISION', 'tf32x3').lower()
    aliases = {'32': PRECISION_FP32, '16': PRECISION_BF16_TC, 'half': PRECISION_FP16_TC}
    return {**PRECISIONS, **aliases}.get(v, PRECISION_TF32X3)


class B200ObjectDetector(object):

    def __init__(self, model_path, device=0, max_batch=None, precision=None, model_blob=None):
        if max_batch is None:
            max_batch = int(os.environ.get('WATSOR_B200_MAX_BATCH', '64'))
        blob = model_blob if model_blob is not None else load_model_blob(model_path)
        self.engine = Engine(blob, device=device, max_batch=max_batch,
                             precision=default_precision() if precision is None else precision)
        self.max_batch = max_batch
        self._shape_cams = {}          # (H, W) -> anonymous camera id for the single-frame protocol
        self._next_anon = 255

    # ------------------------------------------------------------- Detector protocol
    @property
    def device_name(self):
        return self.engine.device_name

    def __enter__(self):
        return self

    def __exit__(self, exc_type, exc_value, traceback):
        self.engine.close()

    def detect(self, image_shape, image_np, detections):
        """Single-frame protocol call (tensorflow_cpu.py:74-92): fills `detections`
        (label, confidence, bounding_box of all 100 rows) and returns milliseconds."""
        cam = self._camera_for_shape(image_shape)
        return self.engine.detect([image_np], [cam], [detections])

    # ------------------------------------------------------------------ batched API
    def configure_camera(self, cam_id, width, height, camera_config=None):
        """Per-camera filter state (main.py:294-299 builds the same from the camera dict):
        `camera_config` = {'width','height','detect':[{label:{confidence,area,zones}}],['mask']}.
        Optional keys: 'windows', a list of [x, y, w, h] detection windows in the camera's pixels (e.g.
        watsor_b200.windows.grid_windows), and 'window_merge_threshold' (default 0.5), see Engine.set_camera_windows."""
        rasters, filters = camera_tables(camera_config, width, height)
        self.engine.set_camera(cam_id, width, height, rasters, filters)
        windows = (camera_config or {}).get('windows')
        if windows:
            self.engine.set_camera_windows(cam_id, [tuple(w) for w in windows],
                                           camera_config.get('window_merge_threshold', 0.5))

    def register_frame_buffer(self, frame_buffer):
        """Pin the shared-memory images of a FrameBuffer (share.py:76-81) for async H2D."""
        for frame in frame_buffer.frames:
            addr = ctypes.addressof(frame.image.get_obj())
            self.engine.register_host(addr, ctypes.sizeof(frame.image.get_obj()))

    def detect_batch(self, frames, cam_ids, detections, verdicts=None, fuse_filters=True,
                     frames_on_device=False, pixel_format='rgb24'):
        """pixel_format: 'rgb24' (H, W, 3); OpenCV's 'bgr24' (H, W, 3) as cv2.VideoCapture and cv2.imread return it;
        the 4-byte 'rgba' / 'bgra' (H, W, 4) of GPU pipelines (alpha ignored); the 4:2:0 layouts decoders emit,
        'yuv420p' / 'nv12' (H*3//2, W); or the packed 4:2:2 layouts of webcams and capture cards, 'yuyv422' /
        'uyvy422' (H, W, 2).  All are converted on the GPU exactly as cv2.cvtColor converts them to RGB24.  One format
        per batch.  A frame may also be a tuple of its planes (engine.layout_planes) with row pitches of their own:
        arrays or tensors whose first dimension counts rows (an AVFrame's data[i] viewed with linesize[i], a crop of a
        larger frame) or, with frames_on_device, (device address, pitch) pairs such as a decoder surface's.  Device
        planes are read in place; host planes are packed as they are uploaded."""
        flags = (_lib.WB_F_FUSE_FILTERS if fuse_filters else 0) | \
                (_lib.WB_F_FRAMES_ON_DEVICE if frames_on_device else 0)
        return self.engine.detect(frames, cam_ids, detections, verdicts, flags, pixel_format)

    def submit(self, slot, frames, cam_ids, fuse_filters=True, frames_on_device=False, pixel_format='rgb24'):
        """detect_batch's frames (planes too), enqueued on `slot`; they must stay valid until `collect`"""
        flags = (_lib.WB_F_FUSE_FILTERS if fuse_filters else 0) | \
                (_lib.WB_F_FRAMES_ON_DEVICE if frames_on_device else 0)
        self.engine.submit(slot, frames, cam_ids, flags, pixel_format)

    def collect(self, slot, detections=None, verdicts=None):
        return self.engine.collect(slot, detections, verdicts)

    # ----------------------------------------------------------------------- helpers
    def _camera_for_shape(self, image_shape):
        key = (int(image_shape[0]), int(image_shape[1]))
        cam = self._shape_cams.get(key)
        if cam is None:
            cam = self._next_anon
            self._next_anon -= 1
            self.engine.set_camera(cam, key[1], key[0], None, ())
            self._shape_cams[key] = cam
        return cam


def camera_tables(camera_config, width, height):
    """camera dict -> (zone rasters or None, [(label, confidence, area, zones)])."""
    if not camera_config:
        return None, ()
    from ..config.coco import COCO_CLASSES
    from ..filter.mask import mask_tables
    cfg = dict(camera_config)
    cfg.setdefault('width', width)
    cfg.setdefault('height', height)
    rasters, zones_by_label = (None, {})
    if 'mask' in cfg:
        rasters, zones_by_label = mask_tables(cfg)
    max_area = abs(((width - 1) - 0 + 1) * ((height - 1) - 0 + 1))
    rows = []
    for entry in cfg.get('detect', []):
        coco_class = next(iter(entry))
        idx = COCO_CLASSES.index(coco_class)
        p = entry[coco_class]
        rows.append((idx, p.get('confidence', 50) / 100, p.get('area', 10) / 100 * max_area,
                     zones_by_label.get(idx)))
    return rasters, rows
