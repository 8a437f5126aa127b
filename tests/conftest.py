import json
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN_DIR = os.path.join(ROOT, 'tests', 'golden')
from oracle.reference_build import MODEL_BLOB, REF_SITE, reference_dir, reference_pb  # noqa: E402

REF_DIR = reference_dir()
REF_PB = reference_pb()


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs an H100 (run with `pytest -m gpu`)')


def has_gpu():
    from watsor_b200 import _lib
    try:
        return _lib.device_count() > 0
    except Exception:
        return False


@pytest.fixture(scope='session')
def golden():
    with open(os.path.join(GOLDEN_DIR, 'ssd_shapes_golden.json')) as f:
        return json.load(f)


@pytest.fixture(scope='session')
def shapes_model():
    """The upstream 3-class SSD-MobileNet-v1 test model (real weights) as a compiled blob, built by
    __graft_entry__.build() from an upstream checkout (oracle/reference_build.py)."""
    from watsor_b200.model import Model
    if not os.path.isfile(MODEL_BLOB):
        pytest.skip('oracle/_ref model blob missing (run __graft_entry__.build() with an upstream checkout)')
    return Model.load(MODEL_BLOB)


@pytest.fixture(scope='session')
def shapes_oracle(shapes_model):
    from oracle.ssd_model import SsdModelOracle
    return SsdModelOracle(shapes_model)


@pytest.fixture(scope='session')
def shapes_oracle64(shapes_model):
    from oracle.ssd_model import SsdModelOracle
    return SsdModelOracle(shapes_model, dtype=np.float64)


@pytest.fixture(scope='session')
def coco_model():
    """SSD-MobileNet-v1 with 90-class heads and seeded synthetic weights (no COCO weights exist
    offline); threshold 1e-8 as in the TF model-zoo graphs."""
    from watsor_b200.model import synthetic_ssd_mobilenet_v1
    return synthetic_ssd_mobilenet_v1(num_classes=90, seed=0, score_thr=1e-8)


def load_golden_frame(name):
    from PIL import Image
    return np.array(Image.open(os.path.join(GOLDEN_DIR, 'frames', name + '.png')).convert('RGB'))


PORCH_CONFIG = {
    'width': 640, 'height': 480, 'mask': os.path.join(GOLDEN_DIR, 'porch.png'),
    'detect': [{'person': {'confidence': 50, 'area': 1, 'zones': []}},
               {'bicycle': {'confidence': 50, 'area': 1, 'zones': [2]}},
               {'car': {'confidence': 50, 'area': 10, 'zones': []}}]}
