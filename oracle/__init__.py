"""CPU oracle for the watsor detection hot path -- TEST INFRASTRUCTURE ONLY.

Nothing under ``oracle/`` is product code.  Only ``tests/``,
``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` / ``--impl
reference`` legs may import it, and only as the checker or the reported CPU
baseline.  ``watsor_b200`` never imports it; the product path fails loudly when
the CUDA library is missing.

What it restates (all citations into upstream asmirnou/watsor @127f125):

* watsor/detection/tensorflow_cpu.py:74-121 -- feed a uint8 HWC frame to the
  frozen TF Object-Detection graph, fetch detection_boxes/scores/classes, convert
  the normalised boxes to integer pixel coordinates.
* the arithmetic of the frozen graph itself (watsor/test/model/cpu.pb, produced by
  watsor/test/model/prepare.py:19-198).  TensorFlow -- an un-pinned, un-vendored
  dependency (setup.py:51-53, docker/Dockerfile.base:39) -- is NOT installed here,
  so the graph is restated op-group by op-group from the GraphDef with numpy /
  torch-CPU fp32 (see oracle/ssd_graph.py).  Every constant is read from the
  GraphDef, none is hard-coded.
* watsor/filter/{confidence,area,mask,track}.py and watsor/filter/sieve.py.
  shapely (mask.py:2) is absent, so bbox/polygon intersection is restated as an
  exact integer-geometry test (oracle/filters.py).

PARITY PINNING STATUS
  - filter stage: pinned by the reference's own known-answer tests
    (watsor/test/test_filter.py:14-96), re-run against this oracle in
    tests/test_oracle_filters.py.
  - struct ABI: pinned by ctypes sizes/offsets of watsor/stream/share.py:11-32.
  - conv / batch-norm / activation / bias numerics (backbone + heads, 99 % of the
    arithmetic): pinned by an INDEPENDENT EXECUTOR of the reference's own graph --
    OpenCV 4.13's dnn module run on the backbone + heads sub-graph of
    watsor/test/model/cpu.pb (tools/make_golden_cvdnn.py, vectors in
    tests/golden/cvdnn_heads.npz labelled "OpenCV-dnn, not TensorFlow",
    tests/test_oracle_cvdnn.py: agreement to 4e-5 on tensors of range 21).
  - legacy ResizeBilinear: pinned by OpenCV-dnn executing the reference's own
    ResizeBilinear node (attributes untouched) with its own kernel, 8 frame sizes,
    up- and down-scaling, agreement to 2.4e-7 (tests/test_oracle_cvdnn_resize.py).
  - box decode, per-class greedy NMS, cross-class top-100: pinned by OpenCV-dnn's
    DetectionOutputLayer (the SSD post-processing of the Caffe / OpenCV model zoos:
    CENTER_SIZE coding with variances = the graph's scale factors, strict
    thresholds, greedy order), same detections to 2e-6 on 3-class and 90-class
    heads with real suppression going on (tests/test_oracle_cvdnn_post.py).
  - anchors: not restated at all -- constant-folded from the reference's own graph.
  - still **parity unpinned** (no second executor; TensorFlow cannot run here and
    the reference's only model test asserts a detection count,
    watsor/test/test_detect.py:28-77): TF's order for EXACTLY equal scores (lower
    anchor index first) and the placement of ClipToWindow / zero-area pruning
    between NMS and the final top-100.  Both follow the GraphDef node order quoted
    in oracle/ssd_graph.py.
  - oracle/ties.py: float64 classification of rounding ties in the ranking (used by
    the 90-class end-to-end tests); test infrastructure like the rest.
"""
