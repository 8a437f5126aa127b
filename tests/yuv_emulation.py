"""numpy restatement of the 4:2:0 -> RGB24 conversion of watsor_b200/csrc/yuv420.cuh (the same integer arithmetic
and the same chroma addressing, both layouts), plus the frames the tests feed it.  The CPU suite pins it against
cv2.cvtColor on every (Y, U, V) triple; the GPU tests then show that the kernels equal cvtColor too."""
import cv2
import numpy as np

CV2_CODE = {'yuv420p': cv2.COLOR_YUV2RGB_I420, 'nv12': cv2.COLOR_YUV2RGB_NV12}


def chroma_layout(fmt, w, h):
    """(step, row, v_off) of yuv420.cuh's ChromaLayout."""
    if fmt == 'nv12':
        return 2, w, 1
    assert fmt == 'yuv420p', fmt
    return 1, w // 2, (w // 2) * (h // 2)


def to_rgb(frame, w, h, fmt):
    """uint8 [h*3/2][w] 4:2:0 frame -> uint8 [h][w][3] RGB24, as the kernels compute it."""
    flat = frame.reshape(-1)
    step, row, v_off = chroma_layout(fmt, w, h)
    ys, xs = np.mgrid[0:h, 0:w]
    c = w * h + (ys >> 1) * row + (xs >> 1) * step
    Y = flat[:w * h].reshape(h, w).astype(np.int64)
    U = flat[c].astype(np.int64) - 128
    V = flat[c + v_off].astype(np.int64) - 128
    y = np.maximum(Y - 16, 0) * 1220542 + (1 << 19)
    rgb = [y + 1673527 * V, y - 852492 * V - 409993 * U, y + 2116026 * U]
    return np.stack([np.clip(ch >> 20, 0, 255) for ch in rgb], axis=-1).astype(np.uint8)


def cv2_rgb(frame, fmt):
    return cv2.cvtColor(frame, CV2_CODE[fmt])


def i420_to_nv12(frame, w, h):
    """the same pixels with the chroma interleaved"""
    q = (w // 2) * (h // 2)
    out = frame.copy()
    uv = out[h:].reshape(-1)
    uv[0::2] = frame[h:].reshape(-1)[:q]
    uv[1::2] = frame[h:].reshape(-1)[q:]
    return out


def from_rgb(rgb, fmt):
    """an RGB image as a 4:2:0 frame (OpenCV's forward conversion; any bytes would do)"""
    h, w = rgb.shape[:2]
    i420 = cv2.cvtColor(rgb, cv2.COLOR_RGB2YUV_I420)
    return i420 if fmt == 'yuv420p' else i420_to_nv12(i420, w, h)


def random_frame(rng, w, h):
    """random 4:2:0 bytes with Y below 16 and above 235 and chroma 0 and 255 present"""
    frame = rng.integers(0, 256, (h * 3 // 2, w), dtype=np.uint8)
    flat = frame.reshape(-1)
    n = min(6, w * h)
    flat[:n] = np.array([0, 15, 16, 235, 236, 255], np.uint8)[:n]
    flat[w * h:w * h + 2] = (0, 255)
    flat[-1] = 0
    return frame


def all_triples(fmt):
    """4096 x 4096 frame holding every (Y, U, V) triple exactly once: each 2x2 block carries one (U, V) pair and 4 of
    its 256 Y values, 64 consecutive blocks (in chroma raster order) one pair."""
    w = h = 4096
    k = np.arange((w // 2) * (h // 2), dtype=np.int64)        # block index = chroma raster index
    pair, j = k // 64, k % 64
    Y = np.empty((h, w), np.uint8)
    blocks = (4 * j[:, None] + np.arange(4)[None, :]).astype(np.uint8).reshape(h // 2, w // 2, 2, 2)
    Y[:] = blocks.transpose(0, 2, 1, 3).reshape(h, w)          # (by, dy, bx, dx)
    U, V = (pair >> 8).astype(np.uint8), (pair & 255).astype(np.uint8)
    frame = np.concatenate([Y.reshape(-1), U, V]).reshape(h * 3 // 2, w)
    return frame if fmt == 'yuv420p' else i420_to_nv12(frame, w, h)
