"""numpy restatement of the packed RGB byte orders of watsor_b200/csrc/yuv420.cuh (rgb_layout: bytes per pixel and the
byte offsets of R, G and B) and the byte permutations the kernels apply to them, plus the frames the tests feed them.
The CPU suite pins the table against the header and the permutations against cv2.cvtColor; the GPU tests then show
that the kernels equal cvtColor too."""
import cv2
import numpy as np

FORMATS = ('bgr24', 'rgba', 'bgra')
# fmt -> (bytes per pixel, offset of R, offset of G, offset of B), as rgb_layout in yuv420.cuh
LAYOUT = {'rgb24': (3, 0, 1, 2), 'bgr24': (3, 2, 1, 0), 'rgba': (4, 0, 1, 2), 'bgra': (4, 2, 1, 0)}
CV2_CODE = {'bgr24': cv2.COLOR_BGR2RGB, 'rgba': cv2.COLOR_RGBA2RGB, 'bgra': cv2.COLOR_BGRA2RGB}


def to_rgb(frame, fmt):
    """uint8 [h][w][bpp] frame -> uint8 [h][w][3] RGB24, as the kernels read it: R, G, B from their byte offsets"""
    bpp, r, g, b = LAYOUT[fmt]
    assert frame.shape[2] == bpp, (frame.shape, fmt)
    return np.ascontiguousarray(frame[:, :, [r, g, b]])


def from_rgb(rgb, fmt, rng=None):
    """the frame of `fmt` whose to_rgb is `rgb`; the fourth byte of RGBA / BGRA is random (the kernels must ignore it)"""
    bpp, r, g, b = LAYOUT[fmt]
    h, w = rgb.shape[:2]
    out = np.empty((h, w, bpp), np.uint8)
    if bpp == 4:
        out[:, :, 3] = (rng or np.random.default_rng(0)).integers(0, 256, (h, w), dtype=np.uint8)
    out[:, :, r], out[:, :, g], out[:, :, b] = rgb[:, :, 0], rgb[:, :, 1], rgb[:, :, 2]
    return out


def to_bgr(rgb):
    """the BGR24 output the effects pass writes: its RGB24 result with bytes 0 and 2 swapped"""
    return np.ascontiguousarray(rgb[:, :, ::-1])


def cv2_rgb(frame, fmt):
    return frame if fmt == 'rgb24' else cv2.cvtColor(frame, CV2_CODE[fmt])


def cv2_bgr(rgb):
    return cv2.cvtColor(rgb, cv2.COLOR_RGB2BGR)


def random_frame(rng, w, h, fmt):
    return rng.integers(0, 256, (h, w, LAYOUT[fmt][0]), dtype=np.uint8)
