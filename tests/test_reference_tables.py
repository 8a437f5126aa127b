"""Small tables and containers the filters and the frame ABI depend on, against the reference modules imported
from the read-only tree: the COCO label table (watsor/config/coco.py:14-131) and the Frame / FrameBuffer views
(watsor/stream/share.py:37-113).  CPU only; without an upstream checkout the upstream results come from
tests/golden/reference/ (tests/reference_golden.py)."""
import ctypes
import sys

import numpy as np
import pytest

from tests.conftest import REF_DIR as REF  # noqa: E402
from tests.reference_golden import upstream  # noqa: E402


def ref_module(name):
    sys.path.insert(0, REF)
    try:
        import importlib
        return importlib.import_module(name)
    finally:
        sys.path.remove(REF)


def test_coco_table_equals_reference():
    from watsor_b200.config import coco

    def theirs():
        ref_coco = ref_module('watsor.config.coco')
        out = {'classes': list(ref_coco.COCO_CLASSES)}
        for idx in list(range(-3, 95)) + [1000]:
            try:
                out[str(idx)] = ref_coco.get_coco_class(idx).label
            except Exception as e:
                out[str(idx)] = 'raises ' + type(e).__name__
        return out
    ref = upstream('tables', 'coco', theirs)
    assert [list(c) if isinstance(c, tuple) else c for c in coco.COCO_CLASSES] == ref['classes']
    for idx in list(range(-3, 95)) + [1000]:
        want = ref[str(idx)]
        if want.startswith('raises '):                          # whatever the reference does out of range ...
            with pytest.raises(Exception) as e:                  # ... we do the same
                coco.get_coco_class(idx)
            assert type(e.value).__name__ == want[7:], idx
            continue
        # the reference record also carries drawing attributes (colours, font) of the out-of-scope output stage
        assert coco.get_coco_class(idx).label == want, idx


def test_frame_views_equal_reference():
    from watsor_b200.stream import share

    def theirs():
        ref_share = ref_module('watsor.stream.share')
        out = []
        for w, h in ((64, 48), (1, 1), (320, 240)):
            t = ref_share.Frame(w, h, 3, 'B')
            st, it = t.get_numpy_image(np.uint8)
            out.append({'shape': list(st), 'array_shape': list(it.shape), 'dtype': str(it.dtype),
                        'header_bytes': ctypes.sizeof(t.header.get_obj()),
                        'whc': [t.header.width, t.header.height, t.header.channels]})
        return {'frames': out, 'buffer_frames': len(ref_share.FrameBuffer(3, 32, 16).frames)}
    ref = upstream('tables', 'frames', theirs)
    for (w, h), theirs in zip(((64, 48), (1, 1), (320, 240)), ref['frames']):
        ours = share.Frame(w, h)
        so, io = ours.get_numpy_image(np.uint8)
        assert list(so) == theirs['shape'] == [h, w, 3] and list(io.shape) == theirs['array_shape']
        assert str(io.dtype) == theirs['dtype']
        assert ctypes.sizeof(ours.header.get_obj()) == theirs['header_bytes'] == 7224
        assert [ours.header.width, ours.header.height, ours.header.channels] == theirs['whc']
        io[...] = 7
        ours.header.detections[99].label = 5
        ours.clear()
        assert not io.any() and ours.header.detections[99].label == 0
    assert len(share.FrameBuffer(3, 32, 16).frames) == ref['buffer_frames'] == 3
