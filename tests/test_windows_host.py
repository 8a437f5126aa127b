"""Detection windows on the CPU: known answers of the merge restatement (tests/window_merge.py), grid_windows,
check_windows, and the worker's per-tick frame limit when cameras have windows."""
import pytest

from tests.window_merge import ios_exceeds, merge_windows
from watsor_b200.detection import detector as det_mod
from watsor_b200.windows import check_windows, grid_windows

PAD = (1, 0.0, 0, 0, 0, 0)


def test_part_box_inside_whole_box_of_another_window_is_dropped():
    whole = [(1, 0.9, 100, 100, 199, 299)]             # full-frame window
    part = [(1, 0.95, 0, 0, 49, 199)]                  # window at (150, 100): the left half of the same person
    got = merge_windows([whole, part], [(0, 0), (150, 100)])
    assert got[0] == (1, 0.95, 150, 100, 199, 299) and got[1] == PAD   # the higher score is kept
    got = merge_windows([[(1, 0.99, 100, 100, 199, 299)], part], [(0, 0), (150, 100)])
    assert got[0] == (1, 0.99, 100, 100, 199, 299) and got[1] == PAD


def test_rows_of_one_window_never_suppress_each_other():
    rows = [(1, 0.9, 10, 10, 50, 50), (1, 0.8, 10, 10, 50, 50)]
    assert merge_windows([rows], [(0, 0)])[:3] == rows + [PAD]


def test_different_labels_are_both_kept():
    got = merge_windows([[(1, 0.9, 10, 10, 50, 50)], [(2, 0.8, 10, 10, 50, 50)]], [(0, 0), (0, 0)])
    assert got[:2] == [(1, 0.9, 10, 10, 50, 50), (2, 0.8, 10, 10, 50, 50)]


def test_threshold_one_keeps_everything():
    a, b = [(3, 0.7, 0, 0, 9, 9)], [(3, 0.6, 0, 0, 9, 9)]
    assert merge_windows([a, b], [(0, 0), (0, 0)], 1.0)[:2] == a + b
    assert merge_windows([a, b], [(0, 0), (0, 0)], 0.999)[:2] == a + [PAD]
    assert not ios_exceeds(a[0], b[0], 1.0) and ios_exceeds(a[0], b[0], 0.0)
    # touching boxes share one pixel column: inter = 10, smaller area 100 -> IoS 0.1
    assert ios_exceeds((1, 0, 0, 0, 9, 9), (1, 0, 9, 0, 20, 9), 0.09)
    assert not ios_exceeds((1, 0, 0, 0, 9, 9), (1, 0, 9, 0, 20, 9), 0.1)
    assert not ios_exceeds((1, 0, 0, 0, 9, 9), (1, 0, 10, 0, 20, 9), 0.0)


def test_ties_are_ordered_by_window_then_row():
    w0 = [(5, 0.5, 0, 0, 1, 1), (6, 0.5, 0, 0, 1, 1)]
    w1 = [(7, 0.5, 0, 0, 1, 1), (8, 0.75, 0, 0, 1, 1)]
    got = merge_windows([w0, w1], [(0, 0), (100, 0)])
    assert [r[0] for r in got[:4]] == [8, 5, 6, 7]


def test_more_than_100_kept_rows_are_cut_and_padding_follows():
    rows = [[(1 + (r % 3), 0.9 - 0.001 * r, 2 * r, 0, 2 * r + 1, 1) for r in range(60)] for _ in range(2)]
    got = merge_windows(rows, [(0, 0), (0, 500)])
    assert len(got) == 100 and PAD not in got
    assert [r[1] for r in got] == sorted([r[1] for r in got], reverse=True)
    got = merge_windows([rows[0][:30]], [(0, 0)], class_offset=0.0)
    assert got[30:] == [(0, 0.0, 0, 0, 0, 0)] * 70
    assert merge_windows([[], []], [(0, 0), (1, 1)]) == [PAD] * 100


def test_grid_windows_cover_overlap_and_align():
    for (w, h, cols, rows) in [(1920, 1080, 2, 2), (1920, 1080, 3, 2), (640, 480, 4, 3), (2560, 1440, 3, 3), (300, 300, 1, 1)]:
        wins = grid_windows(w, h, cols, rows)
        assert wins[0] == (0, 0, w, h) and len(wins) == 1 + cols * rows
        grid = wins[1:]
        for x, y, ww, hh in grid:
            assert x % 2 == 0 and y % 2 == 0 and ww % 2 == 0 and hh % 2 == 0
            assert x >= 0 and y >= 0 and x + ww <= w and y + hh <= h
        xs = sorted({(x, ww) for x, _, ww, _ in grid})
        ys = sorted({(y, hh) for _, y, _, hh in grid})
        assert xs[0][0] == 0 and xs[-1][0] + xs[-1][1] == w and ys[0][0] == 0 and ys[-1][0] + ys[-1][1] == h
        for axis in (xs, ys):
            for (a, la), (b, _) in zip(axis, axis[1:]):
                assert a + la - b >= 0.25 * la - 2              # neighbours overlap by a quarter of a window
        for cx in list(range(0, w, 7)) + [w - 1]:
            for cy in list(range(0, h, 7)) + [h - 1]:
                assert any(x <= cx < x + ww and y <= cy < y + hh for x, y, ww, hh in grid), (cx, cy)
        check_windows(wins, w, h, 'nv12')
    assert grid_windows(641, 481, 2, 2, full_frame=False)[-1] == (272, 204, 369, 277)   # odd frame: last one odd
    assert grid_windows(100, 100, 1, 1, overlap=0.5, full_frame=False) == [(0, 0, 100, 100)]


def test_check_windows_errors():
    check_windows([(0, 0, 640, 480), (1, 3, 5, 7)], 640, 480)
    with pytest.raises(ValueError, match='not inside'):
        check_windows([(600, 0, 41, 10)], 640, 480)
    with pytest.raises(ValueError, match='not inside'):
        check_windows([(-2, 0, 10, 10)], 640, 480)
    with pytest.raises(ValueError, match='empty'):
        check_windows([(0, 0, 0, 10)], 640, 480)
    with pytest.raises(ValueError, match='at most 16'):
        check_windows([(0, 0, 10, 10)] * 17, 640, 480)
    for fmt in ('yuv420p', 'nv12'):
        for win in [(1, 0, 10, 10), (0, 1, 10, 10), (0, 0, 11, 10), (0, 0, 10, 11)]:
            with pytest.raises(ValueError, match='even window origin'):
                check_windows([win], 640, 480, fmt)
        check_windows([(2, 4, 10, 12)], 640, 480, fmt)
    with pytest.raises(ValueError, match='four integers'):
        check_windows([(0, 0, 10)], 640, 480)


def test_worker_drains_max_batch_over_max_windows_frames():
    from tests.fake_backend import FakeB200
    from tests.test_detector_worker import make_fb, run_worker

    sizes = []

    class Recording(FakeB200):
        max_batch = 8

        def submit(self, slot, images, cams, fuse_filters=False):
            sizes.append(len(images))
            super().submit(slot, images, cams, fuse_filters)

    assert det_mod.max_windows(None) == 1 and det_mod.max_windows({'a': {}, 'b': None}) == 1
    configs = {'cam': {'windows': [[0, 0, 16, 8], [0, 0, 8, 8], [8, 0, 8, 8]]}, 'other': {'windows': []}}
    assert det_mod.max_windows(configs) == 3
    fb = make_fb(8)
    run_worker(Recording, range(8), fb, {'camera_configs': configs})
    assert [f.latch.count for f in fb.frames] == [1] * 8
    assert sum(sizes) == 8 and max(sizes) <= 8 // 3
    sizes.clear()
    fb = make_fb(8)
    run_worker(Recording, range(8), fb, {'camera_configs': {'cam': {'detect': []}}})
    assert sum(sizes) == 8 and max(sizes) <= 8
