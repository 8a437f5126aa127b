"""Detection windows: parts of a camera's frame that each become one model image.

The model sees a 300x300 image, so on a 1920x1080 frame a person 60 px tall shrinks to 15 px and is lost.  Detecting
on overlapping windows as well as on the whole frame keeps small objects large enough; the library merges the windows'
rows back into the frame's 100 rows on the GPU (include/watsor_b200.h, wb_set_camera_windows).
"""
import math

from ._lib import WB_MAX_WINDOWS

FOUR_TWO_ZERO = ('yuv420p', 'nv12')
FOUR_TWO_TWO = ('yuyv422', 'uyvy422')


def grid_windows(width, height, cols, rows, overlap=0.25, full_frame=True, align=2):
    """[(x, y, w, h), ...]: the whole frame first (unless `full_frame` is False), then a `cols` x `rows` grid of windows
    that cover the frame, neighbours overlapping by at least `overlap` of a window's size (less at most `align` px).
    Origins and sizes are multiples of `align` wherever the frame's size allows (an odd frame size leaves the last
    window of a row or column odd), so align=2 suits the 4:2:0 and 4:2:2 formats."""
    if cols < 1 or rows < 1 or not 0 <= overlap < 1 or align < 1:
        raise ValueError('need cols, rows >= 1, 0 <= overlap < 1 and align >= 1')

    def axis(size, n):
        span = size / (n - (n - 1) * overlap)                  # n windows of `span` with the overlap cover `size`
        span = min(size, int(math.ceil(span / align)) * align)
        out = []
        for i in range(n):
            x = 0 if n == 1 else (i * (size - span) // (n - 1)) // align * align
            out.append((x, size - x if i == n - 1 else span))
        return out

    wins = [(0, 0, width, height)] if full_frame else []
    for y, h in axis(height, rows):
        for x, w in axis(width, cols):
            wins.append((x, y, w, h))
    return wins


def check_windows(windows, width, height, pixel_format='rgb24'):
    """Raises ValueError unless `windows` is a list of at most WB_MAX_WINDOWS (x, y, w, h) integer rectangles with
    w, h >= 1 inside a `width` x `height` frame, with even origins and sizes for the 4:2:0 formats and an even x and w
    for the 4:2:2 formats (their chroma is shared by pixel pairs of a row only).  The packed RGB orders (rgb24, bgr24,
    rgba, bgra) take any window."""
    windows = list(windows)
    if len(windows) > WB_MAX_WINDOWS:
        raise ValueError('a camera may have at most %d detection windows, not %d' % (WB_MAX_WINDOWS, len(windows)))
    for i, win in enumerate(windows):
        if len(win) != 4 or not all(isinstance(v, int) or hasattr(v, '__index__') for v in win):
            raise ValueError('window %d: %r is not four integers (x, y, w, h)' % (i, win))
        x, y, w, h = (int(v) for v in win)
        if w < 1 or h < 1:
            raise ValueError('window %d %r is empty' % (i, tuple(win)))
        if x < 0 or y < 0 or x + w > width or y + h > height:
            raise ValueError('window %d %r is not inside the %dx%d frame' % (i, tuple(win), width, height))
        if pixel_format in FOUR_TWO_ZERO and (x % 2 or y % 2 or w % 2 or h % 2):
            raise ValueError('window %d %r: %s frames need an even window origin, width and height'
                             % (i, tuple(win), pixel_format))
        if pixel_format in FOUR_TWO_TWO and (x % 2 or w % 2):
            raise ValueError('window %d %r: %s frames need an even window x and width' % (i, tuple(win), pixel_format))
    return [tuple(int(v) for v in win) for win in windows]
