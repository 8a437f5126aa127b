"""CPU restatement of watsor/filter/{confidence,area,mask,track,sieve}.py.

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).  Pinned by the reference's
known-answer tests watsor/test/test_filter.py:14-96 (re-run in
tests/test_oracle_filters.py).

shapely (mask.py:2) is not installed, so `bounding_box.intersects(polygon)`
(mask.py:54) is restated as an exact integer-geometry predicate on closed point
sets: the closed rectangle spanned by the detection's corners meets the closed
polygon region iff a polygon vertex lies in the rectangle, or a polygon edge meets
the rectangle, or a rectangle corner lies inside the polygon.  cv2 *is* installed
and is used exactly where the reference uses it (imread, threshold, findContours,
moments -- mask.py:62-88).
"""
from collections import defaultdict, deque

import cv2
import numpy as np

from .coco_labels import COCO_CLASSES


class Det:
    """Plain stand-in for watsor.stream.share.Detection (share.py:19-24)."""
    __slots__ = ('label', 'zones', 'confidence', 'x_min', 'y_min', 'x_max', 'y_max')

    def __init__(self, label=0, confidence=0.0, box=(0, 0, 0, 0), zones=None):
        self.label = label
        self.confidence = confidence
        self.x_min, self.y_min, self.x_max, self.y_max = box
        self.zones = list(zones) if zones is not None else [0] * 10

    def key(self):
        return (self.label, tuple(self.zones), self.confidence,
                self.x_min, self.y_min, self.x_max, self.y_max)

    def clone(self):
        return Det(self.label, self.confidence,
                   (self.x_min, self.y_min, self.x_max, self.y_max), self.zones)


class ConfidenceOracle:
    """confidence.py:10-19"""

    def __init__(self, camera_config):
        self.idx = {}
        for entry in camera_config['detect']:
            coco_class = next(iter(entry))
            self.idx[COCO_CLASSES.index(coco_class)] = entry[coco_class]['confidence'] / 100

    def __call__(self, d):
        c = self.idx.get(d.label, None)
        return c is not None and d.confidence >= c


class AreaOracle:
    """area.py:10-26"""

    def __init__(self, camera_config):
        self.idx = {}
        for entry in camera_config['detect']:
            coco_class = next(iter(entry))
            w, h = camera_config['width'], camera_config['height']
            max_area = abs((w - 1 - 0 + 1) * (h - 1 - 0 + 1))
            self.idx[COCO_CLASSES.index(coco_class)] = entry[coco_class]['area'] / 100 * max_area

    def __call__(self, d):
        a = self.idx.get(d.label, None)
        return a is not None and abs((d.x_max - d.x_min + 1) * (d.y_max - d.y_min + 1)) >= a


# ------------------------------------------------------------------ mask geometry
def get_alpha_channel(filename, width=None, height=None):
    """mask.py:62-75 (same cv2 call, same assertion messages)."""
    mask_image = cv2.imread(filename, cv2.IMREAD_UNCHANGED)
    assert mask_image is not None, "Error reading mask file {}".format(filename)
    assert len(mask_image.shape) == 3 and mask_image.shape[2] == 4, \
        "Mask image {} is not of 32 bit color".format(filename)
    if width is not None and height is not None:
        assert mask_image.shape[0] == height and mask_image.shape[1] == width, \
            "The size of mask image {} doesn't match {}x{}".format(filename, width, height)
    return mask_image[:, :, 3], mask_image


def find_contours(alpha_channel):
    """mask.py:78-88: zone = alpha==255; external contours sorted by the squared
    distance of the int-truncated moment centroid from the origin."""
    _, thresh = cv2.threshold(255 - alpha_channel, 0, 255, cv2.THRESH_BINARY_INV)
    contours, _ = cv2.findContours(thresh, cv2.RETR_EXTERNAL, cv2.CHAIN_APPROX_SIMPLE)[-2:]

    def key(contour):
        m = cv2.moments(contour)
        cx, cy = int(m['m10'] / m['m00']), int(m['m01'] / m['m00'])
        return cx * cx + cy * cy

    return sorted(contours, key=key)


def _orient(ax, ay, bx, by, cx, cy):
    return (bx - ax) * (cy - ay) - (by - ay) * (cx - ax)


def _seg_hits_seg(p, q, a, b):
    """Closed segments p-q (arrays of many) vs a-b (one); exact in int64."""
    px, py, qx, qy = p[:, 0], p[:, 1], q[:, 0], q[:, 1]
    ax, ay, bx, by = a[0], a[1], b[0], b[1]
    d1 = _orient(px, py, qx, qy, ax, ay)
    d2 = _orient(px, py, qx, qy, bx, by)
    d3 = _orient(ax, ay, bx, by, px, py)
    d4 = _orient(ax, ay, bx, by, qx, qy)
    proper = (np.sign(d1) * np.sign(d2) < 0) & (np.sign(d3) * np.sign(d4) < 0)

    def on(ux, uy, vx, vy, wx, wy, d):       # w on segment u-v given collinear
        return (d == 0) & (np.minimum(ux, vx) <= wx) & (wx <= np.maximum(ux, vx)) & \
               (np.minimum(uy, vy) <= wy) & (wy <= np.maximum(uy, vy))
    touch = on(px, py, qx, qy, ax, ay, d1) | on(px, py, qx, qy, bx, by, d2) | \
        on(ax, ay, bx, by, px, py, d3) | on(ax, ay, bx, by, qx, qy, d4)
    return proper | touch


def _point_in_polygon(x, y, P, Q):
    """Closed even-odd test for an integer point; boundary counts as inside."""
    px, py, qx, qy = P[:, 0], P[:, 1], Q[:, 0], Q[:, 1]
    d = _orient(px, py, qx, qy, x, y)
    on_edge = (d == 0) & (np.minimum(px, qx) <= x) & (x <= np.maximum(px, qx)) & \
              (np.minimum(py, qy) <= y) & (y <= np.maximum(py, qy))
    if on_edge.any():
        return True
    # ray to +x: edge straddles the horizontal line y (half-open rule)
    straddle = (py <= y) != (qy <= y)
    # x-coordinate of the crossing > x  <=>  sign test without division
    # crossing_x - x = ((qx-px)*(y-py) + (px - x)*(qy-py)) / (qy-py)
    num = (qx - px) * (y - py) + (px - x) * (qy - py)
    den = (qy - py)
    right = np.where(den > 0, num > 0, num < 0)
    return bool(np.count_nonzero(straddle & right) % 2)


def rect_intersects_polygon(x0, y0, x1, y1, poly):
    """closed rect (corners as given in mask.py:45-48) vs closed polygon region."""
    P = np.asarray(poly, dtype=np.int64).reshape(-1, 2)
    if max(abs(int(v)) for v in (x0, y0, x1, y1)) >= 2 ** 30:
        # int32 corners: the orientation products of a rectangle edge reach 2^64, so compute in Python integers
        P = P.astype(object)
        x0, y0, x1, y1 = (int(v) for v in (x0, y0, x1, y1))
    Q = np.roll(P, -1, axis=0)
    xa, xb = min(x0, x1), max(x0, x1)
    ya, yb = min(y0, y1), max(y0, y1)
    if xb < P[:, 0].min() or xa > P[:, 0].max() or yb < P[:, 1].min() or ya > P[:, 1].max():
        return False                          # disjoint from the polygon's bounding box
    inside = (P[:, 0] >= xa) & (P[:, 0] <= xb) & (P[:, 1] >= ya) & (P[:, 1] <= yb)
    if inside.any():
        return True
    corners = [(xa, ya), (xb, ya), (xb, yb), (xa, yb)]
    for k in range(4):
        if _seg_hits_seg(P, Q, corners[k], corners[(k + 1) % 4]).any():
            return True
    return _point_in_polygon(xa, ya, P, Q)


class MaskOracle:
    """mask.py:8-59"""

    def __init__(self, camera_config):
        filename = camera_config['mask']
        alpha, _ = get_alpha_channel(filename, camera_config['width'], camera_config['height'])
        contours = find_contours(alpha)
        self.polygons = [c[:, 0] for c in contours]
        for p in self.polygons:
            # shapely's Polygon() (mask.py:26) raises below 3 coordinates
            assert len(p) >= 3, "A LinearRing must have at least 3 coordinate tuples"
        self.by_zone = {}
        for entry in camera_config['detect']:
            coco_class = next(iter(entry))
            index = COCO_CLASSES.index(coco_class)
            zones = entry[coco_class]['zones']
            if len(zones) == 0:
                continue
            for z in zones:
                assert 0 < z <= len(self.polygons), \
                    "There is no zone {} in mask {}".format(z, filename)
            self.by_zone[index] = [p if idx + 1 in zones else None
                                   for idx, p in enumerate(self.polygons)]

    def __call__(self, d):
        polygons = self.by_zone.get(d.label, self.polygons)
        result = False
        z = 0
        p = 0
        while p < len(polygons) and z < len(d.zones):
            if polygons[p] is not None and rect_intersects_polygon(
                    d.x_min, d.y_min, d.x_max, d.y_max, polygons[p]):
                d.zones[z] = p + 1
                z += 1
                result = True
            p += 1
        return result


def apply_predicates(dets, filters):
    """track.py:25-27 first line: `d.label > 0 and all(f(d) for f in filters)`,
    lazily (a later filter only runs -- and MaskFilter only writes zones -- when the
    earlier ones passed).  Returns (kept list, verdict bit list)."""
    kept, verdicts = [], []
    for d in dets:
        v = 0
        ok = d.label > 0
        if ok:
            v |= 1
            for bit, f in enumerate(filters):
                if not f(d):
                    ok = False
                    break
                v |= 2 << bit
        verdicts.append(v)
        if ok:
            kept.append(d)
    return kept, verdicts


class TrackOracle:
    """track.py:8-149 (centroid tracker + predicate application)."""

    def __init__(self, filters=None, sensitivity=5, history=10):
        from scipy.spatial import distance
        self._cdist = distance.cdist
        self.sensitivity = sensitivity
        self.history = history
        self.filters = [] if filters is None else filters
        self.by_label = defaultdict(list)

    def __call__(self, detections):
        kept, _ = apply_predicates(detections, self.filters)
        return self._group_and_update(kept)

    @staticmethod
    def _centroid(d):
        return int((d.x_min + d.x_max) / 2.0), int((d.y_min + d.y_max) / 2.0)

    def _group_and_update(self, detections):
        groups = defaultdict(list)
        for d in detections:
            groups[d.label].append(d)
        suspicious = len(groups) > 0
        for label in list(self.by_label.keys()):
            if label not in groups:
                del self.by_label[label]
        for label, dets in groups.items():
            n_in = len(dets)
            inp = np.zeros((n_in, 2), dtype="int")
            for i, d in enumerate(dets):
                inp[i] = self._centroid(d)
            n_ex = len(self.by_label[label])
            ex = np.zeros((n_ex, 2), dtype="int")
            for i, h in enumerate(self.by_label[label]):
                ex[i] = self._centroid(h[0])
            dist = self._cdist(np.array(ex), inp)
            if len(dist.shape) == 2 and dist.shape[0] > 0 and dist.shape[1] > 0:
                rows = np.argsort(np.amin(dist, axis=1))
                cols = np.argmin(dist, axis=1)[rows]
            else:
                rows, cols = [], []
            used_r, used_c = set(), set()
            for r, c in zip(rows, cols):
                if r in used_r or c in used_c:
                    continue
                self.by_label[label][r].append(dets[c])
                used_r.add(r)
                used_c.add(c)
            for r in sorted(set(range(n_ex)) - used_r, reverse=True):
                del self.by_label[label][r]
            for c in set(range(n_in)) - used_c:
                self.by_label[label].append(deque([dets[c]], maxlen=self.history))
        result = []
        for label, hs in self.by_label.items():
            for h in hs:
                if len(h) < self.sensitivity:
                    continue
                result.append(self._combine(h))
        return result, suspicious

    @staticmethod
    def _combine(h):
        n = h[0].clone()
        n.zones = [0] * 10
        for d in list(h)[1:]:
            n.confidence = max(n.confidence, d.confidence)
            n.x_min = min(n.x_min, d.x_min)
            n.y_min = min(n.y_min, d.y_min)
            n.x_max = max(n.x_max, d.x_max)
            n.y_max = max(n.y_max, d.y_max)
        zones = set()
        for d in h:
            for z in d.zones:
                if z > 0:
                    zones.add(z)
        for i, z in enumerate(zones):
            if i < 10:
                n.zones[i] = z
        return n
