"""numpy restatement of the RGB24 -> 4:2:0 conversion the effects pass writes (rgb_to_yuv in
watsor_b200/csrc/yuv420.cuh and the 4:2:0 store of k_fx_render): the same integer arithmetic and the same siting, U
and V of each 2x2 block from its top-left pixel, for both layouts.  The CPU suite pins it against
cv2.cvtColor(COLOR_RGB2YUV_I420) on every (R, G, B) triple; the GPU tests then show that the kernel equals it."""
import numpy as np

from tests.yuv_emulation import i420_to_nv12

N_TRIPLES = 1 << 24


def rgb_to_yuv(r, g, b):
    """int32 arrays -> (Y, U, V) uint8 arrays"""
    r, g, b = (np.asarray(c, np.int32) for c in (r, g, b))
    y = 269484 * r + 528482 * g + 102760 * b + (1 << 19) + (16 << 20)
    u = -155188 * r - 305135 * g + 460324 * b + (1 << 19) + (128 << 20)
    v = 460324 * r - 385875 * g - 74448 * b + (1 << 19) + (128 << 20)
    return tuple(np.clip(c >> 20, 0, 255).astype(np.uint8) for c in (y, u, v))


def to_yuv420(rgb, fmt):
    """uint8 [h][w][3] RGB24 (w, h even) -> uint8 [h*3/2][w] 4:2:0 frame, as the kernel writes it."""
    h, w = rgb.shape[:2]
    assert w % 2 == 0 and h % 2 == 0, (w, h)
    Y, _, _ = rgb_to_yuv(rgb[..., 0], rgb[..., 1], rgb[..., 2])
    tl = rgb[0::2, 0::2]
    _, U, V = rgb_to_yuv(tl[..., 0], tl[..., 1], tl[..., 2])
    i420 = np.concatenate([Y.reshape(-1), U.reshape(-1), V.reshape(-1)]).reshape(h * 3 // 2, w)
    return i420 if fmt == 'yuv420p' else i420_to_nv12(i420, w, h)


def triple(k):
    """(R, G, B) of triple index k (R in the high byte)"""
    k = np.asarray(k, np.int64)
    return (k >> 16) & 255, (k >> 8) & 255, k & 255


def top_left_frames(rng, n_frames=16, side=2048):
    """n_frames RGB24 frames of side x side whose 2x2 blocks, in frame then chroma raster order, hold every (R, G, B)
    triple once as the top-left pixel; the other three pixels of each block are random."""
    blocks = (side // 2) ** 2
    assert n_frames * blocks == N_TRIPLES
    frames = []
    for f in range(n_frames):
        rgb = rng.integers(0, 256, (side, side, 3), dtype=np.uint8)
        r, g, b = triple(np.arange(f * blocks, (f + 1) * blocks))
        rgb[0::2, 0::2] = np.stack([r, g, b], axis=-1).astype(np.uint8).reshape(side // 2, side // 2, 3)
        frames.append(rgb)
    return frames
