"""Zone masks and detection rows at the limits of the mask / area / confidence predicates, shared by
tests/test_zone_masks_host.py and tests/test_gpu_zone_masks.py.

Every mask builder returns an RGBA uint8 image whose alpha channel is 255 inside the zones and 216 elsewhere, as a
watsor mask is drawn (filter/mask.py: a zone is alpha == 255).  Where the number of zones matters the builder checks
it with `find_contours`, and every zone it makes has >= 3 contour points and a positive area (the centroid key of
mask.py divides by m00)."""
import os

import cv2
import numpy as np

from oracle.filters import AreaOracle, ConfidenceOracle, Det, MaskOracle, find_contours

BACKGROUND = 216
I32_MIN, I32_MAX = -2 ** 31, 2 ** 31 - 1
# labels on both sides of every boundary apply_filters has: `label > 0`, the 91 COCO entries, WB_MAX_LABELS = 128
LABELS = (0, -1, -7, I32_MIN, 1, 2, 45, 89, 90, 91, 100, 126, 127, 128, 129, 1000, I32_MAX)


def rgba(alpha):
    out = np.zeros(alpha.shape + (4,), np.uint8)
    out[..., :3] = 128
    out[..., 3] = alpha
    return out


def zones_of(mask):
    """the zone contours of an RGBA mask, in the reference's order"""
    return find_contours(np.ascontiguousarray(mask[..., 3]))


def checked(alpha, n_zones=None):
    mask = rgba(alpha)
    contours = zones_of(mask)
    if n_zones is not None:
        assert len(contours) == n_zones, (len(contours), n_zones)
    for c in contours:
        assert len(c) >= 3 and cv2.moments(c)['m00'] > 0, c[:, 0].tolist()
    return mask


def _blob(alpha, kind, cx, cy, rx, ry):
    if kind == 0:
        cv2.rectangle(alpha, (cx - rx, cy - ry), (cx + rx, cy + ry), 255, -1)
    elif kind == 1:
        cv2.ellipse(alpha, (cx, cy), (rx, ry), 0, 0, 360, 255, -1)
    else:                                        # 45 degree diamond
        r = min(rx, ry)
        cv2.fillConvexPoly(alpha, np.array([(cx, cy - r), (cx + r, cy), (cx, cy + r), (cx - r, cy)], np.int32), 255)


def grid_mask(width, height, n_zones=32, cols=8):
    """`n_zones` blobs on a `cols`-wide grid, cycling rectangle, ellipse, diamond; each blob's centroid lies in its own
    cell, so the reference numbers them by distance from the origin."""
    rows = (n_zones + cols - 1) // cols
    cw, ch = width // cols, height // rows
    alpha = np.full((height, width), BACKGROUND, np.uint8)
    for z in range(n_zones):
        r, c = divmod(z, cols)
        cx, cy = c * cw + cw // 2, r * ch + ch // 2
        _blob(alpha, z % 3, cx, cy, max(2, cw * 3 // 10 + z % 4), max(2, ch * 3 // 10 - z % 3))
    return checked(alpha, n_zones)


def border_mask(width=320, height=240):
    """zones on every frame corner and every edge: 4 corner blocks (one of them a single-pixel-wide L), an edge-hugging
    band on each side and a zone that spans the whole width"""
    a = np.full((height, width), BACKGROUND, np.uint8)
    a[0:12, 0:16] = 255                                   # top left corner
    a[0:9, width - 7:width] = 255                         # top right corner
    a[height - 5:height, 0:20] = 255                      # bottom left corner
    a[height - 30:height, width - 1] = 255                # bottom right corner: 1-px L along two edges
    a[height - 1, width - 30:width] = 255
    a[height - 3:height, width - 3:width] = 255
    a[0:2, 60:140] = 255                                  # top edge, 2 px high
    a[height - 1, 60:140] = 255                           # bottom edge, 1 px high + a 2x2 block
    a[height - 2:height, 99:101] = 255
    a[80:160, 0] = 255                                    # left edge, 1 px wide + a 2x2 block
    a[119:121, 0:2] = 255
    a[70:170, width - 2:width] = 255                      # right edge, 2 px wide
    a[118:122, 4:width - 4] = 255                         # across the frame
    return checked(a, 9)


def thin_mask(width=200, height=150):
    """single-pixel-wide zones: L shapes (each with a 2x2 block so that its area is positive), staircases of steps 2 and
    3, 45 degree bands 2 px wide in both directions, and two blocks joined only through a diagonal pixel"""
    a = np.full((height, width), BACKGROUND, np.uint8)
    a[5:30, 5] = 255                                      # L: down, then right; the block at the elbow
    a[29, 5:40] = 255
    a[28:30, 4:6] = 255
    a[5, 50:80] = 255                                     # L: right, then down; the block at the far end
    a[5:25, 79] = 255
    a[24:26, 78:80] = 255
    for y in range(12):                                   # staircase, step 2
        a[40 + y, 10 + 2 * y:13 + 2 * y] = 255
    for y in range(8):                                    # staircase, step 3
        a[40 + y, 60 + 3 * y:64 + 3 * y] = 255
    for y in range(30):                                   # 45 degree band, 2 px wide, down to the right
        a[60 + y, 100 + y:102 + y] = 255
    for y in range(30):                                   # 45 degree band, 2 px wide, down to the left
        a[60 + y, 190 - y:192 - y] = 255
    a[100:106, 20:26] = 255                               # two blocks meeting at one corner
    a[106:112, 26:32] = 255
    a[120:140, 150] = 255                                 # a vertical 1-px bar with a block at its top
    a[120:122, 149:151] = 255
    return checked(a, 8)


def diagonal_join_mask(width=64, height=48):
    """two blocks that share only a corner: findContours follows 8-connected pixels, so they are ONE zone"""
    a = np.full((height, width), BACKGROUND, np.uint8)
    a[10:20, 10:20] = 255
    a[20:30, 20:30] = 255
    return checked(a, 1)


def tie_mask(width=240, height=240):
    """pairs of zones mirrored about the diagonal x == y: equal centroid keys cx^2 + cy^2, so the stable sort keeps
    findContours' order between them"""
    a = np.full((height, width), BACKGROUND, np.uint8)
    for (x, y, w, h) in ((100, 20, 20, 10), (40, 60, 12, 12), (150, 90, 30, 6)):
        a[y:y + h, x:x + w] = 255
        a[x:x + w, y:y + h] = 255                         # the mirror image
    cv2.circle(a, (180, 180), 12, 255, -1)               # on the diagonal: its own mirror
    return checked(a, 7)


def over_limit_mask(width=640, height=480):
    return grid_mask(width, height, 33, cols=11)


def tiny_zone_mask(width=40, height=30, n_pixels=1):
    """a zone of 1 or 2 pixels: its contour has fewer than 3 points and zero area"""
    a = np.full((height, width), BACKGROUND, np.uint8)
    a[10:20, 10:20] = 255
    a[25, 30:30 + n_pixels] = 255
    return rgba(a)


FAMILIES = {
    'grid32-640x480': lambda: grid_mask(640, 480),
    'grid32-1920x1080': lambda: grid_mask(1920, 1080),
    'grid32-3840x2160': lambda: grid_mask(3840, 2160),
    'border': border_mask,
    'thin': thin_mask,
    'diagonal-join': diagonal_join_mask,
    'ties': tie_mask,
}


def write_mask(directory, name, mask):
    path = os.path.join(str(directory), name + '.png')
    assert cv2.imwrite(path, mask)
    return path


# ------------------------------------------------------------------------------------------------- rows
def zone_edge_boxes(contours, max_vertices=None):
    """boxes at every place where covering a zone pixel or not changes: one pixel, one row and one column on every
    contour vertex (or `max_vertices` of them, evenly spaced), bounding-box corner and the pixels diagonally next to
    them, plus each zone's bounding box and the box one pixel larger"""
    boxes = set()
    for c in contours:
        bx, by, bw, bh = cv2.boundingRect(c)
        corners = [(bx, by), (bx + bw - 1, by), (bx, by + bh - 1), (bx + bw - 1, by + bh - 1)]
        vertices = c[:, 0]
        if max_vertices is not None and len(vertices) > max_vertices:
            vertices = vertices[np.linspace(0, len(vertices) - 1, max_vertices).astype(int)]
        points = {tuple(int(v) for v in p) for p in vertices} | set(corners)
        for (x, y) in points:
            for dx in (-1, 0, 1):
                for dy in (-1, 0, 1):
                    if dx and not dy or dy and not dx:
                        continue
                    px, py = x + dx, y + dy
                    boxes.add((px, py, px, py))
                    boxes.add((px - 5, py, px, py))      # one row ending on the pixel
                    boxes.add((px, py, px + 5, py))
                    boxes.add((px, py - 5, px, py))      # one column
                    boxes.add((px, py, px, py + 5))
        boxes.add((bx, by, bx + bw - 1, by + bh - 1))
        boxes.add((bx - 1, by - 1, bx + bw, by + bh))
    return sorted(boxes)


def frame_edge_boxes(width, height):
    """the whole frame, boxes partly outside it on each side, wholly outside it, with unordered corners, and the
    extreme int32 coordinates (spans of 2^32 and 3e9)"""
    w, h = width, height
    out = [(0, 0, w - 1, h - 1), (-5, -5, w + 5, h + 5), (w - 1, h - 1, 0, 0), (I32_MIN, I32_MIN, I32_MAX, I32_MAX),
           (-10, 10, 5, h // 2), (w - 5, 10, w + 10, h // 2), (10, -10, w // 2, 5), (10, h - 5, w // 2, h + 10),
           (-20, -20, -1, -1), (w, 0, w + 10, 10), (0, h, 10, h + 10), (-30, h // 2, -1, h // 2 + 3),
           (w, h, w + 50, h + 50), (w // 2, h // 2, 0, 0), (w - 1, 0, 0, h - 1), (0, h - 1, w - 1, 0),
           (I32_MIN, 0, I32_MAX, 0), (0, I32_MIN, 0, I32_MAX), (I32_MIN, 10, I32_MAX, 12), (I32_MAX, 10, I32_MIN, 12),
           (-1500000000, 0, 1500000000, h - 1), (0, -1500000000, w - 1, 1500000000),
           (I32_MIN, I32_MIN, I32_MIN, I32_MIN), (I32_MAX, I32_MAX, I32_MAX, I32_MAX), (I32_MIN, 0, -1, h - 1),
           (w, I32_MIN, I32_MAX, I32_MAX), (I32_MAX, I32_MAX, I32_MIN, I32_MIN)]
    return out


def random_boxes(rng, width, height, n):
    out = []
    for i in range(n):
        x0, x1 = (int(v) for v in rng.integers(-8, width + 8, 2))
        y0, y1 = (int(v) for v in rng.integers(-8, height + 8, 2))
        if i % 3 == 0:
            x1, y1 = x0 + int(rng.integers(-3, 4)), y0 + int(rng.integers(-3, 4))
        out.append((x0, y0, x1, y1))
    return out


def edge_rows(mask, rng, n_random=200, max_vertices=6, thresholds=(0.5,), labels=LABELS, limit=None):
    """-> [(label, confidence, box)]: the zone and frame edge boxes and random ones, each with a label and a
    confidence cycled so that every label meets boxes of every kind; confidences are random float32 values, each
    threshold exactly, the float32 just below it, 0, 1 and NaN.  `limit`: at most that many zone edge boxes, drawn
    at random (the frame edge boxes are always there)."""
    h, w = mask.shape[:2]
    zone_boxes = zone_edge_boxes(zones_of(mask), max_vertices)
    if limit is not None and len(zone_boxes) > limit:
        zone_boxes = [zone_boxes[i] for i in sorted(rng.choice(len(zone_boxes), limit, replace=False))]
    boxes = zone_boxes + frame_edge_boxes(w, h) + random_boxes(rng, w, h, n_random)
    confs = [float('nan'), 0.0, 1.0]
    for t in thresholds:
        confs += [t, float(np.nextafter(np.float32(t), np.float32(0)))]
    out = []
    for i, box in enumerate(boxes):
        label = labels[(i * 7) % len(labels)]
        conf = confs[i % len(confs)] if i % 3 == 0 else float(np.float32(rng.random()))
        out.append((label, conf, box))
    return out


def to_detections(rows):
    from watsor_b200.stream.share import Detection
    arr = (Detection * len(rows))()
    for d, (label, conf, (x0, y0, x1, y1)) in zip(arr, rows):
        d.label, d.confidence = label, conf
        d.bounding_box.x_min, d.bounding_box.y_min, d.bounding_box.x_max, d.bounding_box.y_max = x0, y0, x1, y1
    return arr


def to_dets(rows):
    return [Det(label, conf, box) for label, conf, box in rows]


# ------------------------------------------------------------------------------------------------- oracles
def table_oracles(mask_path, width, height, table):
    """oracle/filters.py predicates for a camera table as `Engine.set_camera` takes it, [(label, confidence, area,
    zones or None)]: the oracles are built from an empty camera config and their per-label dicts filled from the table.
    The default row (label -1) stands for every label without a row of its own, as apply_filters reads it; labels
    are expanded over LABELS, the only ones the tests use."""
    cfg = {'width': width, 'height': height, 'mask': mask_path, 'detect': []}
    conf, area, mask = ConfidenceOracle(cfg), AreaOracle(cfg), MaskOracle(cfg)
    rows = {label: (c, a, z) for label, c, a, z in table}
    default = rows.get(-1)
    for label in LABELS:
        entry = rows.get(label) if 0 <= label < 128 else None
        entry = entry if entry is not None else default
        if entry is None:
            continue
        c, a, zones = entry
        conf.idx[label] = c
        area.idx[label] = a
        if zones:
            mask.by_zone[label] = [p if i + 1 in zones else None for i, p in enumerate(mask.polygons)]
        else:
            mask.by_zone[label] = mask.polygons
    return [conf, area, mask]


def chain_verdicts(dets, filters, check_label=True):
    """apply_predicates (track.py:26) as verdict bits WB_V_*; with check_label False (WB_CAM_NO_LABEL_CHECK) the
    `label > 0` gate is skipped and its bit is never set"""
    out = []
    for d in dets:
        v = 0
        if check_label:
            if not d.label > 0:
                out.append(0)
                continue
            v = 1
        ok = True
        for bit, f in enumerate(filters):
            if not f(d):
                ok = False
                break
            v |= 2 << bit
        out.append(v | (16 if ok else 0))
    return out
