"""The reference's visual effects (watsor/output/copy.py, blend.py, draw.py) on the GPU.

Same class names, constructors and `apply(image_in, image_out, shape, header_in, header_out)` contract as the
reference, so `Watsor._create_effects` (watsor/main.py:302-312) can return them unchanged; every class is one call
into `wb_fx_render` (include/watsor_b200.h).  `FusedEffects` does what the whole chain of main.py does for a camera
-- copy or blend, then draw, then the zone outlines -- in ONE pass over the frame; `EffectsEngine.render` is the batched
form for several cameras.  Both can write the output as yuv420p or NV12 for an encoder, converted on the GPU as
cv2.cvtColor(COLOR_RGB2YUV_I420) would convert the RGB24 result; the single chained effects stay RGB24, since DrawEffect
draws onto image_out in place.  There is no CPU fallback: without the library and an H100 the constructors raise.

The output bytes are the reference's: BlendEffect's float32 arithmetic is restated (blend.py:15-32), cv2.rectangle at
thickness 1 is the box outline, cv2.addWeighted is one float fused multiply-add rounded half to even, the label text
and the zone outlines come from tables made with the installed OpenCV (font.py, `contour_bits`).
"""
import ctypes
from ctypes import Structure, byref, c_float, c_int32, c_uint8, c_void_p, memmove, sizeof

import numpy as np

from .. import _lib
from ..config.coco import COCO_CLASSES, get_coco_class
from ..engine import check_frames, layout_shape
from ..stream.share import MAX_DETECTIONS, Detection
from .font import FontAtlas

WB_FX_BLEND, WB_FX_DRAW, WB_FX_CONTOURS, WB_FX_ON_DEVICE = 1, 2, 4, 8
WB_FX_YUV420P, WB_FX_NV12 = 16, 32
WB_FX_OUT_YUV420P, WB_FX_OUT_NV12 = 64, 128
WB_FX_YUYV422, WB_FX_UYVY422 = 256, 512
WB_FX_BGR24, WB_FX_RGBA, WB_FX_BGRA = 1024, 2048, 4096
WB_FX_OUT_BGR24 = 8192
_FX_FORMATS = {'rgb24': 0, 'yuv420p': WB_FX_YUV420P, 'nv12': WB_FX_NV12, 'yuyv422': WB_FX_YUYV422,
               'uyvy422': WB_FX_UYVY422, 'bgr24': WB_FX_BGR24, 'rgba': WB_FX_RGBA, 'bgra': WB_FX_BGRA}
_FX_OUT_FORMATS = {'rgb24': 0, 'yuv420p': WB_FX_OUT_YUV420P, 'nv12': WB_FX_OUT_NV12, 'bgr24': WB_FX_OUT_BGR24}


class _Font(Structure):
    _fields_ = [('n_glyphs', c_int32), ('rows', c_int32), ('cols', c_int32), ('y0', c_int32),
                ('text_height', c_int32), ('baseline', c_int32), ('margin', c_int32),
                ('advance', c_void_p), ('lut', c_void_p)]


class _Label(Structure):
    _fields_ = [('box_color', c_uint8 * 3), ('n_prefix', c_uint8), ('prefix', c_uint8 * 60)]


def _check_output_format(output_format):
    # 4:2:2 is an input format only: OpenCV's RGB -> 4:2:2 arithmetic is not the I420 one the kernel restates; RGBA /
    # BGRA are input formats only: an encoder or cv2.imencode takes RGB24, BGR24 or 4:2:0
    if output_format not in _FX_OUT_FORMATS:
        raise ValueError('output_format must be one of %s, not %r' % (', '.join(_FX_OUT_FORMATS), output_format))


def _check(rc):
    if rc != 0:
        raise _lib.WatsorB200Error(_lib.load().wb_fx_last_error().decode(errors='replace'))


def contour_bits(alpha_channel):
    """uint32 [H][W]: bit z-1 set where `cv2.drawContours(image, contours, z-1, color, thickness=1)` of draw.py:103
    paints (the drawing does not depend on the image, so one raster per zone, made once, is exact)."""
    import cv2

    from ..filter.mask import find_contours
    contours = find_contours(alpha_channel)
    assert len(contours) <= 32, 'a mask may hold at most 32 zones'
    bits = np.zeros(alpha_channel.shape, np.uint32)
    for z in range(len(contours)):
        raster = np.zeros(alpha_channel.shape, np.uint8)
        cv2.drawContours(raster, contours, z, 1, thickness=1)
        bits |= raster.astype(np.uint32) << np.uint32(z)
    return bits


class EffectsEngine:
    """One `wb_fx` context: font tables, label styles and per-camera rasters resident on one H100."""

    def __init__(self, device=0, labels=None):
        self.lib = _lib.load()
        labels = list(COCO_CLASSES) if labels is None else list(labels)
        styles = [get_coco_class(i) for i in range(len(labels))]
        for s in styles:
            # the kernel implements the attributes every COCO class has (coco.py:114-119)
            assert s.font_color == (255, 255, 255) and s.box_thickness == 1 and s.font_thickness == 1 \
                and s.font_scale == 0.5, 'only the reference\'s drawing attributes are implemented'
        self.atlas = FontAtlas(''.join(labels) + ': 0123456789%')
        a = self.atlas
        self._advance = np.array([a.advance[c] for c in a.chars], np.int32)
        font = _Font(len(a.chars), a.rows, a.cols, a.y0, a.text_height, a.baseline,
                     int(round(np.ceil(0.1 * a.text_height))),            # draw.py:62
                     self._advance.ctypes.data, a.lut.ctypes.data)
        table = (_Label * len(labels))()
        for i, name in enumerate(labels):
            prefix = [a.index[c] for c in name + ': ']
            assert len(prefix) <= 60, name
            table[i].box_color[:] = styles[i].box_color
            table[i].n_prefix = len(prefix)
            table[i].prefix[:len(prefix)] = prefix
        digits = (c_uint8 * 11)(*[a.index[c] for c in '0123456789%'])
        self._fx = c_void_p()
        _check(self.lib.wb_fx_create(device, byref(font), len(labels), table, digits, styles[0].alpha,
                                     byref(self._fx)))
        self.atlas.lut = None            # 98 MB of host memory: resident on the device now
        self.device = device
        self._next_cam = 0
        self._sizes = {}                 # cam_id -> (width, height)
        self.last_gpu_ms = 0.0

    def close(self):
        if self._fx:
            self.lib.wb_fx_destroy(self._fx)
            self._fx = c_void_p()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def add_camera(self, width, height, alpha_channel=None, contours=None):
        """-> cam_id.  alpha_channel: uint8 [H][W] (BlendEffect); contours: `contour_bits(alpha_channel)`."""
        cam = self._next_cam
        self._next_cam += 1
        alpha = None if alpha_channel is None else np.ascontiguousarray(alpha_channel, np.uint8)
        cont = None if contours is None else np.ascontiguousarray(contours, np.uint32)
        for arr in (alpha, cont):
            assert arr is None or arr.shape == (height, width)
        _check(self.lib.wb_fx_set_camera(self._fx, cam, width, height,
                                         None if alpha is None else alpha.ctypes.data,
                                         None if cont is None else cont.ctypes.data))
        self._sizes[cam] = (width, height)
        return cam

    def render(self, images_in, images_out, cam_ids, rows, flags, pixel_format='rgb24', output_format='rgb24'):
        """images: uint8 arrays (or device pointers with WB_FX_ON_DEVICE); rows: per frame the `Detection * 100`
        array of a frame header (or its address).  pixel_format: layout of images_in, 'rgb24', OpenCV's 'bgr24',
        'rgba' / 'bgra' (alpha ignored), a 4:2:0 layout 'yuv420p' / 'nv12' or a packed 4:2:2 layout 'yuyv422' /
        'uyvy422' (converted as cv2.cvtColor does; see engine.layout_shape).  output_format: layout of images_out,
        'rgb24', 'bgr24' for cv2.imencode (the rendered frame with R and B swapped, cv2.cvtColor(COLOR_RGB2BGR)) or
        'yuv420p' / 'nv12' for an encoder that takes 4:2:0 (the rendered frame converted as
        cv2.cvtColor(COLOR_RGB2YUV_I420) does).  images_out may be images_in only when both are 'rgb24' or 'bgr24'."""
        _check_output_format(output_format)
        sizes = [self._sizes.get(c) for c in cam_ids]
        check_frames(images_in, sizes, pixel_format)
        if output_format != 'rgb24':
            check_frames(images_out, sizes, output_format)
        flags |= _FX_FORMATS[pixel_format] | _FX_OUT_FORMATS[output_format]
        n = len(images_in)

        def addr(x):
            if isinstance(x, int):
                return x
            if isinstance(x, np.ndarray):
                assert x.flags['C_CONTIGUOUS'] and x.dtype == np.uint8
                return x.ctypes.data
            return ctypes.addressof(x)

        pin = (c_void_p * n)(*[addr(x) for x in images_in])
        pout = (c_void_p * n)(*[addr(x) for x in images_out])
        prow = (c_void_p * n)(*[addr(r) for r in rows])
        cams = (c_int32 * n)(*cam_ids)
        ms = c_float()
        _check(self.lib.wb_fx_render(self._fx, n, pin, pout, cams, prow, flags, byref(ms)))
        self.last_gpu_ms = ms.value
        return ms.value


_ENGINE = None


def default_engine():
    """One engine per process (the reference runs one effects process per camera, output/video.py:10-35); the device
    follows the detector's selection rules (CUDA_DEVICE etc., detection/devices.py)."""
    global _ENGINE
    if _ENGINE is None:
        from ..detection.devices import b200_gpus
        devices = [d for d, _ in b200_gpus()]
        if not devices:
            raise _lib.WatsorB200Error('no H100 visible: the GPU visual effects have no CPU fallback')
        _ENGINE = EffectsEngine(devices[0])
    return _ENGINE


def _camera_tables(camera_config, want_alpha, want_contours):
    from ..filter.mask import get_alpha_channel
    alpha, _ = get_alpha_channel(camera_config['mask'], camera_config['width'], camera_config['height'])
    return (alpha if want_alpha else None), (contour_bits(alpha) if want_contours else None)


class _Effect:
    flags = 0

    def __init__(self, engine=None):
        self._engine = engine
        self._cams = {}          # (h, w) -> cam_id for effects that are not tied to a camera_config

    def _engine_or_default(self):
        if self._engine is None:
            self._engine = default_engine()
        return self._engine

    def _cam_for(self, shape):
        key = (int(shape[0]), int(shape[1]))
        if key not in self._cams:
            self._cams[key] = self._engine_or_default().add_camera(key[1], key[0])
        return self._cams[key]

    @staticmethod
    def _rows(header):
        return header.detections


class CopyHeaderEffect:
    """copy.py:6-10 -- the header stays on the host."""

    @staticmethod
    def apply(image_in, image_out, shape, header_in, header_out):
        memmove(ctypes.addressof(header_out.get_obj()), ctypes.addressof(header_in.get_obj()),
                sizeof(header_in.get_obj()))


class CopyImageEffect:
    """copy.py:13-18 (a host copy; inside `FusedEffects` it is the kernel's load/store)."""

    @staticmethod
    def apply(image_in, image_out, shape, header_in, header_out):
        np.copyto(image_out, image_in)


class BlendEffect(_Effect):
    """blend.py:6-32: the frame alpha-blended against white with the mask's alpha channel."""
    flags = WB_FX_BLEND

    def __init__(self, camera_config, engine=None):
        super().__init__(engine)
        alpha, _ = _camera_tables(camera_config, True, False)
        self._cam = self._engine_or_default().add_camera(camera_config['width'], camera_config['height'], alpha)

    def apply(self, image_in, image_out, shape, header_in, header_out):
        self._engine.render([image_in], [image_out], [self._cam], [self._rows(header_out)], self.flags)


class DrawEffect(_Effect):
    """draw.py:7-88: boxes and labels of the detections with label > 0, drawn onto image_out."""
    flags = WB_FX_DRAW

    def apply(self, image_in, image_out, shape, header_in, header_out):
        cam = self._cam_for(shape)
        self._engine.render([image_out], [image_out], [cam], [self._rows(header_out)], self.flags)


class DrawEffectWithContours(DrawEffect):
    """draw.py:91-103: + the outline of every zone a drawn detection lies in."""
    flags = WB_FX_DRAW | WB_FX_CONTOURS

    def __init__(self, camera_config, engine=None):
        super().__init__(engine)
        _, cont = _camera_tables(camera_config, False, True)
        self._cam = self._engine_or_default().add_camera(camera_config['width'], camera_config['height'], None, cont)

    def apply(self, image_in, image_out, shape, header_in, header_out):
        self._engine.render([image_out], [image_out], [self._cam], [self._rows(header_out)], self.flags)


class FusedEffects(_Effect):
    """The image part of the effect chain main.py:302-312 builds for a camera, as one pass:
    with a mask   BlendEffect + DrawEffectWithContours;   without   CopyImageEffect + DrawEffect.
    output_format 'yuv420p' / 'nv12' writes image_out as the 4:2:0 frame an encoder takes (engine.layout_shape), so the
    output FrameBuffer holds w*h*3//2 bytes and no RGB -> 4:2:0 conversion is left to the encoder; 'bgr24' writes the
    BGR24 frame that cv2.imencode takes without a cv2.cvtColor of its own."""

    def __init__(self, camera_config, engine=None, output_format='rgb24'):
        super().__init__(engine)
        _check_output_format(output_format)
        layout_shape(output_format, camera_config['width'], camera_config['height'])   # even sizes
        self.output_format = output_format
        if 'mask' in camera_config:
            alpha, cont = _camera_tables(camera_config, True, True)
            self.flags = WB_FX_BLEND | WB_FX_DRAW | WB_FX_CONTOURS
        else:
            alpha = cont = None
            self.flags = WB_FX_DRAW
        self._cam = self._engine_or_default().add_camera(camera_config['width'], camera_config['height'], alpha, cont)

    def apply(self, image_in, image_out, shape, header_in, header_out):
        self._engine.render([image_in], [image_out], [self._cam], [self._rows(header_out)], self.flags,
                            output_format=self.output_format)


def new_rows():
    """A zeroed `Detection * 100` (tests, bench)."""
    return (Detection * MAX_DETECTIONS)()


__all__ = ['EffectsEngine', 'CopyHeaderEffect', 'CopyImageEffect', 'BlendEffect', 'DrawEffect',
           'DrawEffectWithContours', 'FusedEffects', 'contour_bits', 'new_rows', 'WB_FX_BLEND', 'WB_FX_DRAW',
           'WB_FX_CONTOURS', 'WB_FX_ON_DEVICE', 'WB_FX_YUV420P', 'WB_FX_NV12', 'WB_FX_OUT_YUV420P', 'WB_FX_OUT_NV12',
           'WB_FX_YUYV422', 'WB_FX_UYVY422', 'WB_FX_BGR24', 'WB_FX_RGBA', 'WB_FX_BGRA', 'WB_FX_OUT_BGR24']
