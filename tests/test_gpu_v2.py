"""SSD-MobileNet-v2 (the model BASELINE.json's 640x480 configs name): architecture descriptor with
seeded synthetic weights -- no v2 weights exist offline -- checked GPU-vs-oracle: inverted residual
blocks (1x1 expand, depthwise, linear projection, residual add), 24-channel tensors (K not a multiple of
16), 576/1280-wide taps; and the BASELINE configs[2] workload itself (tests/workload.py): 90 classes at
score threshold 1e-8, a mask on each of the 8 cameras, schema-default thresholds -- row for row, in the
reported precision (tf32x3) and on the CUDA-core path."""
import numpy as np
import pytest

from tests import workload
from tests.artist import artist_frame
from tests.gpu_util import compare_rows, new_rows, rows_bytes, rows_to_tuples, zones_of
from watsor_b200 import _lib
from watsor_b200.detection.b200 import B200ObjectDetector
from watsor_b200.engine import Engine
from watsor_b200.model import OP_HEAD, synthetic_ssd_mobilenet_v2
from watsor_b200.stream.share import Detection

pytestmark = pytest.mark.gpu
PRECISIONS = dict(argvalues=[0, 2], ids=['fp32-cuda-cores', 'fp32-3xtf32-tcgen05'])


@pytest.fixture(scope='module')
def v2():
    from oracle.ssd_model import SsdModelOracle
    m = synthetic_ssd_mobilenet_v2(num_classes=3, seed=2, score_thr=0.3)   # 9..14 detections per frame
    return m, SsdModelOracle(m), SsdModelOracle(m, dtype=np.float64)


@pytest.fixture(scope='module')
def v2coco():
    """configs[2]'s model + both oracles + the float64 tie analysis of the test frames (computed once)."""
    from oracle.ssd_graph import to_detections
    from oracle.ssd_model import SsdModelOracle
    from oracle.ties import analyse
    m = workload.v2_coco_model()
    o32, o64 = SsdModelOracle(m), SsdModelOracle(m, dtype=np.float64)
    frames = []
    for cam in range(8):                              # one frame per camera of the configs[2] batch
        img = artist_frame(640, 480, cam, cam % 3)
        pre = o32.preprocess(img)
        e32, l32 = o32.raw_heads(pre)
        e64, l64 = o64.raw_heads(pre)
        b, s, cl, n = o32.postprocess(e32, l32)
        frames.append({'cam': cam, 'img': img, 'pre': pre, 'heads32': (e32, l32), 'heads64': (e64, l64),
                       'want': to_detections(b, cl, s, img.shape), 'n': n,
                       'ties': analyse(o64, e64, l64, img.shape)})
    return m, o32, o64, frames


@pytest.mark.parametrize('precision', **PRECISIONS)
def test_v2_layer_by_layer(v2, precision):
    m, oracle, _ = v2
    pre = oracle.preprocess(artist_frame(640, 480, 1, 0))
    enc, lg, memo = oracle.raw_heads(pre, return_memo=True)
    with Engine(m.to_blob(), device=0, max_batch=2, precision=precision) as e:
        for li, layer in enumerate(m.layers):
            if layer.op == OP_HEAD:
                continue
            want = oracle.feature(memo, li)
            _, _, got = e.backbone(pre[None], stop_layer=li, layer_shape=want.shape)
            err, scale = np.abs(got[0] - want).max(), max(1.0, float(np.abs(want).max()))
            # random weights + residual adds amplify rounding differences ~5x more than the trained v1 net
            assert err <= (1e-4 if precision == 0 else 4e-4) * scale, (li, layer.name, err, scale)
        genc, glg, _ = e.backbone(pre[None])
    assert np.abs(genc[0] - enc).max() <= 1e-3 and np.abs(glg[0] - lg).max() <= 3e-3


@pytest.mark.parametrize('precision', **PRECISIONS)
def test_v2_detect_rows(v2, precision):
    """3-class v2 at threshold 0.3 (few candidates, n_valid < 100: padding rows, threshold edge)."""
    from oracle.ssd_graph import to_detections
    from oracle.ties import analyse, compare_with_ties
    m, oracle, oracle64 = v2
    stats = {'strict_frames': 0, 'tie_frames': 0}
    with B200ObjectDetector(None, device=0, max_batch=4, precision=precision, model_blob=m.to_blob()) as det:
        for frame in range(4):
            img = artist_frame(640, 480, 2, frame)
            rows = (Detection * 100)()
            det.detect(img.shape, img, rows)
            got = rows_to_tuples(rows)
            _check_frame(got, img, oracle, oracle64, stats, to_detections, analyse, compare_with_ties)
    print('v2 3-class:', stats)
    assert stats['strict_frames'] + stats['tie_frames'] == 4


def _check_frame(got, img, o32, o64, stats, to_detections, analyse, compare_with_ties, cached=None):
    """Row-exact against the fp32 oracle; when that fails, every difference must be a tie the float64
    evaluation classifies (oracle/ties.py) -- never a set comparison."""
    if cached is None:
        pre = o32.preprocess(img)
        e32, l32 = o32.raw_heads(pre)
        b, s, cl, n = o32.postprocess(e32, l32)
        want = to_detections(b, cl, s, img.shape)
        e64, l64 = o64.raw_heads(pre)
        an = analyse(o64, e64, l64, img.shape)
        b64 = o64.postprocess(e64, l64)[0]
    else:
        want, n, an = cached['want'], cached['n'], cached['ties']
        b64 = o64.postprocess(*cached['heads64'])[0]
    try:
        flips = compare_rows(got, want, b64, img.shape)
        stats['strict_frames'] += 1
        stats['flips'] = stats.get('flips', 0) + flips
        return
    except AssertionError:
        pass
    res = compare_with_ties(got, an)
    # the fp32 CPU oracle must need the same allowance (the classification is not hiding a GPU-only error)
    compare_with_ties(want, an)
    n_out = res['n_out']
    assert all(g == (1, 0.0, 0, 0, 0, 0) for g in got[n_out:]) or n_out == 100
    stats['tie_frames'] += 1
    for k in ('strict', 'in_group', 'unchecked'):
        stats[k] = stats.get(k, 0) + res[k]


@pytest.mark.parametrize('precision', **PRECISIONS)
def test_configs2_heads_vs_float64(v2coco, precision):
    """Raw head tensors of the 90-class v2 net (53 conv layers deep, logits of magnitude ~8) against the float64
    evaluation of the same layer program: within 5e-4 absolute (a confidence error <= 1.3e-4, the north star allows
    1e-3) and within 6x of the fp32 CPU oracle's own distance from float64 (measured: CUDA cores 1x, 3xTF32 3..4.5x --
    the tensor core accumulates with truncation, DESIGN.md 4.1)."""
    m, o32, o64, frames = v2coco
    with Engine(m.to_blob(), device=0, max_batch=2, precision=precision) as e:
        for fr in frames[:3]:
            genc, glg, _ = e.backbone(fr['pre'][None])
            (e32, l32), (e64, l64) = fr['heads32'], fr['heads64']
            for g, a, b in ((genc[0], e32, e64), (glg[0], l32, l64)):
                err_gpu, err_cpu = np.abs(g - b).max(), np.abs(a - b).max()
                assert err_gpu <= 5e-4 and err_gpu <= 6 * err_cpu + 2e-5, (err_gpu, err_cpu)


@pytest.mark.parametrize('precision', **PRECISIONS)
def test_configs2_rows_exact_end_to_end(v2coco, precision):
    """BASELINE configs[2] as bench.py runs it: the 8-camera batch, 90 classes at 1e-8, one mask per camera,
    schema-default thresholds, predicates fused.  Per frame:
      (a) Detection rows equal the fp32 oracle's rows exactly (label, integer box; confidence 1e-3), or every
          difference is a float64-classified rounding tie;
      (b) the GPU post stage on the GPU's own head tensors is bit-identical to the oracle's post stage on those
          tensors (so (a)'s ties come from conv rounding only);
      (c) verdict bits and zones equal the oracle predicates applied to the same rows."""
    from oracle.filters import AreaOracle, ConfidenceOracle, Det, MaskOracle, apply_predicates
    from oracle.ssd_graph import to_detections
    from oracle.ties import analyse, compare_with_ties
    m, o32, o64, frames = v2coco
    stats = {'strict_frames': 0, 'tie_frames': 0}
    with B200ObjectDetector(None, device=0, max_batch=8, precision=precision, model_blob=m.to_blob()) as det:
        cfgs = [workload.camera_config(c) for c in range(8)]
        for c in range(8):
            det.configure_camera(c, 640, 480, cfgs[c])
        rows = new_rows(8)
        verd = np.zeros((8, 100), np.uint32)
        det.detect_batch([f['img'] for f in frames], list(range(8)), rows, [verd[i] for i in range(8)],
                         fuse_filters=True)
        # determinism of the full batch
        rows2 = new_rows(8)
        det.detect_batch([f['img'] for f in frames], list(range(8)), rows2, fuse_filters=True)
        assert all(rows_bytes(a) == rows_bytes(b) for a, b in zip(rows, rows2))
        passed = 0
        for i, fr in enumerate(frames):
            got = rows_to_tuples(rows[i])
            _check_frame(got, fr['img'], o32, o64, stats, to_detections, analyse, compare_with_ties, cached=fr)
            # (c) predicates on the GPU's own rows
            cfg = cfgs[i]
            dets = [Det(g[0], g[1], tuple(g[2:])) for g in got]
            _, want_v = apply_predicates(dets, [ConfidenceOracle(cfg), AreaOracle(cfg), MaskOracle(cfg)])
            assert [int(v) & 15 for v in verd[i]] == want_v, (i, [int(v) for v in verd[i]][:10], want_v[:10])
            assert [int(v) >> 4 for v in verd[i]] == [1 if v == 15 else 0 for v in want_v]
            assert zones_of(rows[i]) == [d.zones for d in dets]
            passed += sum(1 for v in want_v if v == 15)
        # (b) post stage on the GPU's own heads, frame by frame through the stage-level ABI
        for i, fr in enumerate(frames[:4]):
            genc, glg, _ = det.engine.backbone(fr['pre'][None])
            prow, _, _, _, _, num = det.engine.postprocess(genc, glg, [i])
            b, s, cl, n = o32.postprocess(genc[0], glg[0])
            assert num[0] == n
            assert [t[:1] + t[2:] for t in rows_to_tuples(prow[0])] == \
                [t[:1] + t[2:] for t in to_detections(b, cl, s, fr['img'].shape)]
            assert max(abs(x[1] - y[1]) for x, y in zip(rows_to_tuples(prow[0]), to_detections(b, cl, s, fr['img'].shape))) <= 2e-7
    print('configs[2] rows:', stats, 'rows passing all predicates:', passed)
    checked = 100 * stats['strict_frames'] + stats.get('strict', 0) + stats.get('in_group', 0)
    assert stats['strict_frames'] + stats['tie_frames'] == 8
    assert checked >= 0.75 * 800, stats          # fragile NMS decisions may leave part of a frame unasserted
    # (area >= 10 % of the frame and a zone hit: with these synthetic heads hardly any row passes all predicates;
    #  what is asserted above is that every verdict bit equals the oracle's)


def test_configs2_single_frame_equals_batch_rows(v2coco):
    """One frame alone vs inside the 8-camera batch (different split-K plans): same detections."""
    m, o32, o64, frames = v2coco
    with B200ObjectDetector(None, device=0, max_batch=8, precision=2, model_blob=m.to_blob()) as det:
        for c in range(8):
            det.configure_camera(c, 640, 480, None)
        batch = new_rows(8)
        det.detect_batch([f['img'] for f in frames], list(range(8)), batch, fuse_filters=False)
        single = new_rows(1)
        det.detect_batch([frames[3]['img']], [3], single, fuse_filters=False)
        a, b = rows_to_tuples(batch[3]), rows_to_tuples(single[0])
        same = sum(1 for x, y in zip(a, b) if x[0] == y[0] and x[2:] == y[2:])
        assert same >= 90 and max(abs(x[1] - y[1]) for x, y in zip(a, b)) < 1e-3
