"""numpy restatement of the packed 4:2:2 -> RGB24 conversion of watsor_b200/csrc/yuv420.cuh (where the Y, U and V of
pixel (x, y) live in a YUYV / UYVY frame, then the same integer arithmetic as tests/yuv_emulation.py), plus the frames
the tests feed it.  The CPU suite pins it against cv2.cvtColor on every (Y, U, V) triple; the GPU tests then show that
the kernels equal cvtColor too."""
import cv2
import numpy as np

FORMATS = ('yuyv422', 'uyvy422')
CV2_CODE = {'yuyv422': cv2.COLOR_YUV2RGB_YUYV, 'uyvy422': cv2.COLOR_YUV2RGB_UYVY}


def sample_offsets(fmt, w, h):
    """byte offsets of the Y, U and V samples of every pixel of a packed w x h frame, as yuv420.cuh computes them:
    luma_origin + y * 2w + x * luma_step, chroma_origin + y * row + (x >> 1) * step, U + v_off"""
    assert fmt in FORMATS and w % 2 == 0, (fmt, w)
    ys, xs = np.mgrid[0:h, 0:w].astype(np.int64)
    luma0, chroma0 = (0, 1) if fmt == 'yuyv422' else (1, 0)
    Y = luma0 + ys * 2 * w + xs * 2
    U = chroma0 + ys * 2 * w + (xs >> 1) * 4
    return Y, U, U + 2


def yuv_to_rgb(Y, U, V):
    """yuv_to_rgb of yuv420.cuh on int arrays -> uint8 [..., 3]"""
    Y, U, V = (np.asarray(a, np.int64) for a in (Y, U, V))
    y = np.maximum(Y - 16, 0) * 1220542 + (1 << 19)
    u, v = U - 128, V - 128
    rgb = [y + 1673527 * v, y - 852492 * v - 409993 * u, y + 2116026 * u]
    return np.stack([np.clip(ch >> 20, 0, 255) for ch in rgb], axis=-1).astype(np.uint8)


def to_rgb(frame, fmt, rows=256):
    """uint8 [h][w][2] 4:2:2 frame -> uint8 [h][w][3] RGB24, as the kernels compute it (in bands of `rows` rows)"""
    h, w = frame.shape[:2]
    out = np.empty((h, w, 3), np.uint8)
    for r0 in range(0, h, rows):
        band = np.ascontiguousarray(frame[r0:r0 + rows])
        flat = band.reshape(-1)
        Y, U, V = sample_offsets(fmt, w, band.shape[0])
        out[r0:r0 + rows] = yuv_to_rgb(flat[Y], flat[U], flat[V])
    return out


def cv2_rgb(frame, fmt):
    return cv2.cvtColor(frame, CV2_CODE[fmt])


def pack(Y, U, V, fmt):
    """Y [h][w], U and V [h][w/2] -> the packed [h][w][2] frame (YUYV: Y0 U Y1 V; UYVY: U Y0 V Y1)"""
    h, w = Y.shape
    out = np.empty((h, w, 2), np.uint8)
    yi, ci = (0, 1) if fmt == 'yuyv422' else (1, 0)
    out[:, :, yi] = Y
    out[:, 0::2, ci] = U
    out[:, 1::2, ci] = V
    return out


def from_rgb(rgb, fmt):
    """an RGB image as a 4:2:2 frame: BT.601 Y of every pixel, U and V of each pair's left pixel (any bytes would do;
    this gives the detector pictures it finds objects in)"""
    yuv = cv2.cvtColor(rgb, cv2.COLOR_RGB2YUV)
    return pack(yuv[:, :, 0], yuv[:, 0::2, 1], yuv[:, 0::2, 2], fmt)


def from_i420(frame, fmt):
    """the 4:2:2 frame with the pixels of a yuv420p frame (each chroma row repeated for its two luma rows), so that
    cvtColor of the two gives the same RGB"""
    h, w = frame.shape[0] * 2 // 3, frame.shape[1]
    flat = frame.reshape(-1)
    U = flat[w * h:w * h * 5 // 4].reshape(h // 2, w // 2)
    V = flat[w * h * 5 // 4:].reshape(h // 2, w // 2)
    return pack(frame[:h], np.repeat(U, 2, axis=0), np.repeat(V, 2, axis=0), fmt)


def random_frame(rng, w, h, fmt='yuyv422'):
    """random 4:2:2 bytes with Y below 16 and above 235 and chroma 0 and 255 present"""
    frame = rng.integers(0, 256, (h, w, 2), dtype=np.uint8)
    Y, U, V = sample_offsets(fmt, w, h)
    flat = frame.reshape(-1)
    n = min(6, w * h)
    flat[Y.reshape(-1)[:n]] = np.array([0, 15, 16, 235, 236, 255], np.uint8)[:n]
    flat[U.reshape(-1)[0]], flat[V.reshape(-1)[0]] = 0, 255
    flat[U.reshape(-1)[-1]] = 255
    return frame


def all_triples(fmt, side, seed=0):
    """8192 x 4096 frame holding every (Y, U, V) triple exactly once: macropixel k (row-major) carries U = k >> 8 & 255,
    V = k & 255 and Y = k >> 16 on its left (side 0) or right (side 1) pixel; the other pixel has a random Y"""
    w, h = 8192, 4096
    k = np.arange(w * h // 2, dtype=np.int64)
    partner = np.random.default_rng(seed).integers(0, 256, k.size, dtype=np.uint8)
    Y = np.empty((k.size, 2), np.uint8)
    Y[:, side] = (k >> 16).astype(np.uint8)
    Y[:, 1 - side] = partner
    return pack(Y.reshape(h, w), ((k >> 8) & 255).astype(np.uint8).reshape(h, w // 2),
                (k & 255).astype(np.uint8).reshape(h, w // 2), fmt)
