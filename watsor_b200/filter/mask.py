"""MaskFilter -- contract of watsor/filter/mask.py:8-88.

Set-up (host, once per camera, same OpenCV calls as the reference): read the RGBA mask,
zone = pixels with alpha == 255, external contours sorted by the squared distance of the
int-truncated moment centroid from the origin (mask.py:62-88).  Instead of shapely
polygons each zone becomes a filled-contour raster; libwatsor_b200 turns the rasters into
summed-area tables in HBM, and "bounding box intersects zone polygon" (mask.py:54) becomes
"the box covers at least one raster pixel" -- 4 loads per (detection, zone).  Both are the
same predicate because contour vertices are pixel centres joined by 8-connected unit steps
(DESIGN.md section 5; tests/test_oracle_filters.py::test_raster_sat_equals_exact_polygon_intersection checks the raster /
summed-area form against exact integer geometry on porch.png and random masks with holes and islands, including
zero-width / zero-height boxes; tests/test_zone_masks_host.py checks it on 32-zone grids of rectangles, ellipses and
45-degree diamonds at 640x480, 1920x1080 and 3840x2160, zones on every frame edge and corner, single-pixel-wide L shapes
and bars, staircases, 2-pixel 45-degree bands, two blocks joined only through a diagonal pixel (findContours makes them
one zone whose ring touches itself) and zones with equal centroid keys, each with edge boxes on every corner and
outside the frame).  The claim held on every family, so no kind of zone is refused beyond what the reference refuses.
Not covered: GEOS' own treatment of invalid self-touching rings (1-pixel-wide parts, diagonal joins), which the exact
integer geometry of oracle/filters.py stands in for.  Zones of fewer than 3 contour points have zero area and fail,
as in the reference, in the centroid key (ZeroDivisionError) before the 3-point assertion is reached.  One visible difference from the reference: the fused detector path
(`WB_F_FUSE_FILTERS`) clears `zones[]` of every row before judging it, whereas `TensorFlowObjectDetector.detect`
never touches zones (ref:tensorflow_cpu.py:79-90; the reference's sieve works on a zeroed clone, sieve.py:24-27, so
the published rows agree).
"""
import cv2
import numpy as np

from .. import _lib
from ..config.coco import COCO_CLASSES
from ._gpu import NEG_INF, GpuPredicate

MAX_CAMERA_ZONES = 32


def get_alpha_channel(filename, width=None, height=None):
    mask_image = cv2.imread(filename, cv2.IMREAD_UNCHANGED)
    assert mask_image is not None, "Error reading mask file {}".format(filename)
    assert len(mask_image.shape) == 3 and mask_image.shape[2] == 4, \
        "Mask image {} is not of 32 bit color".format(filename)
    if width is not None and height is not None:
        assert mask_image.shape[0] == height and mask_image.shape[1] == width, \
            "The size of mask image {} doesn't match {}x{}".format(filename, width, height)
    return mask_image[:, :, 3], mask_image


def contours_key(contour):
    moments = cv2.moments(contour)
    cx, cy = int(moments['m10'] / moments['m00']), int(moments['m01'] / moments['m00'])
    return cx * cx + cy * cy


def find_contours(alpha_channel):
    _, thresh = cv2.threshold(255 - alpha_channel, 0, 255, cv2.THRESH_BINARY_INV)
    contours, _ = cv2.findContours(thresh, cv2.RETR_EXTERNAL, cv2.CHAIN_APPROX_SIMPLE)[-2:]
    return sorted(contours, key=contours_key)


def zone_rasters(contours, width, height):
    """uint8 [n_zones][H][W]: 1 where the pixel lies inside or on the zone's outer contour."""
    out = np.zeros((len(contours), height, width), np.uint8)
    for i, c in enumerate(contours):
        cv2.drawContours(out[i], [c], -1, 1, thickness=cv2.FILLED)
    return out


def mask_tables(camera_config):
    """-> (zone rasters, {label: [zone numbers]}) for a camera config with a 'mask' key."""
    filename = camera_config['mask']
    alpha, _ = get_alpha_channel(filename, camera_config['width'], camera_config['height'])
    contours = find_contours(alpha)
    for c in contours:
        assert len(c) >= 3, "A zone of mask {} has fewer than 3 contour points".format(filename)
    assert len(contours) <= MAX_CAMERA_ZONES, "Mask {} has more than {} zones".format(filename, MAX_CAMERA_ZONES)
    zones_by_label = {}
    for entry in camera_config['detect']:
        coco_class = next(iter(entry))
        zones = entry[coco_class]['zones']
        if len(zones) == 0:
            continue
        for z in zones:
            assert 0 < z <= len(contours), "There is no zone {} in mask {}".format(z, filename)
        zones_by_label[COCO_CLASSES.index(coco_class)] = list(zones)
    return zone_rasters(contours, camera_config['width'], camera_config['height']), zones_by_label


class MaskFilter(GpuPredicate):
    verdict_bit = _lib.WB_V_MASK

    def __init__(self, camera_config):
        rasters, self.zones_by_label = mask_tables(camera_config)
        self.n_zones = rasters.shape[0]
        rows = [(-1, NEG_INF, 0.0, None)]                       # unlisted label: every zone (mask.py:50)
        rows += [(label, NEG_INF, 0.0, zones) for label, zones in self.zones_by_label.items()]
        super().__init__(camera_config['width'], camera_config['height'], rows, rasters)
