"""numpy restatement of k_window_merge (watsor_b200/csrc/kernels_post.cu): a frame's window rows -> its 100 rows.

A row is a tuple (label, confidence, x_min, y_min, x_max, y_max) in the window's pixels."""
import numpy as np

from tests.gpu_util import rows_to_tuples


def valid_rows(rows):
    """The valid rows of one window's Detection[100] as the existing path writes them: scores are > the model's score
    threshold >= 0, so the valid rows are the leading rows with a positive confidence (padding has confidence 0)."""
    out = []
    for t in rows_to_tuples(rows):
        if not t[1] > 0:
            break
        out.append(t)
    return out


def ios_exceeds(a, b, thr):
    """intersection over the smaller inclusive pixel box > thr, on integers and float64 as the kernel computes it"""
    iw = min(a[4], b[4]) - max(a[2], b[2]) + 1
    ih = min(a[5], b[5]) - max(a[3], b[3]) + 1
    inter = iw * ih if iw > 0 and ih > 0 else 0
    area = [(r[4] - r[2] + 1) * (r[5] - r[3] + 1) for r in (a, b)]
    return float(inter) > float(np.float64(thr) * np.float64(min(area)))


def merge_windows(window_rows, origins, merge_threshold=0.5, class_offset=1.0, max_total=100):
    """window_rows[k]: the valid rows of window k; origins[k] = (x, y) of window k.  Returns the frame's 100 rows."""
    cand = []
    for k, (rows, (x, y)) in enumerate(zip(window_rows, origins)):
        for r, (lab, conf, x0, y0, x1, y1) in enumerate(rows):
            cand.append(((-np.float32(conf), k, r), k, (lab, conf, x0 + x, y0 + y, x1 + x, y1 + y)))
    cand.sort(key=lambda c: c[0])
    kept = []
    for _, k, row in cand:
        if len(kept) >= max_total:
            break
        if any(kk != k and kr[0] == row[0] and ios_exceeds(row, kr, merge_threshold) for kk, kr in kept):
            continue
        kept.append((k, row))
    out = [row for _, row in kept]
    pad = (int(np.float32(0) + np.float32(class_offset)), 0.0, 0, 0, 0, 0)
    return out + [pad] * (100 - len(out))
