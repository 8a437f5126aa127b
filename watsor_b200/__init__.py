"""watsor_b200 -- H100-native (sm_90a) implementation of watsor's per-frame detection
hot path behind the reference's plugin surface:

    watsor_b200.detection   <-> watsor/detection/*   (Detector protocol, create_object_detectors)
    watsor_b200.filter      <-> watsor/filter/*      (Confidence/Area/Mask/Track filters, sieve)
    watsor_b200.stream      <-> watsor/stream/share.py (the shared-memory frame ABI only)
    watsor_b200.config.coco <-> watsor/config/coco.py  (label table used by the filters)

All arithmetic runs in hand-written CUDA kernels inside csrc/libwatsor_b200.so, reached
through the ctypes C-ABI declared in include/watsor_b200.h.  There is no CPU fallback:
importing the compute classes without the built library raises.
"""
__version__ = '0.1.0'
