"""The merge of a page's four turned readings (DESIGN 4.15): CPU checks with the kernels' bodies run on the host
(tests/emu/turn_merge_emu.cpp) against oracle/turn_merge_ref.py, bit for bit, on the reference's four readings of one
page (tests/golden/omni_page_turns.npz, merged_*), on fabricated readings and on hand-made cases."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle import page_turn_ref as PT
from oracle import tile_ref
from oracle import turn_merge_ref as R
from tests.support import assert_same, emu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
PAD, EOS = 1096, 1099


def bind(lib):
    """Bind tests/emu/turn_merge_emu.cpp (host compile of the kernels' bodies)."""
    lib.emu_merge_turns.restype = C.c_long
    lib.emu_merge_turns.argtypes = ([C.c_int] + [C.c_void_p] * 6 + [C.c_int, C.c_int64, C.c_int64, C.c_double] +
                                    [C.c_void_p] * 7)
    lib.emu_map_row.restype = None
    lib.emu_map_row.argtypes = [C.c_void_p] * 3 + [C.c_int, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p]


def emu_merge(count, offset, pts, polys, rec, prob, pad=PAD, eos=EOS, iou=0.5):
    """alm_omni_merge_turns' three launches on the host -> the dict merge_turns / turn_merge_ref.merge return."""
    lib = emu('turn_merge_emu', bind)
    count = np.ascontiguousarray(count, np.int32)
    offset = np.ascontiguousarray(offset, np.int32)
    pts = np.ascontiguousarray(pts, np.float64).reshape(-1, 2)
    polys = np.ascontiguousarray(polys, np.float64).reshape(-1, 32)
    rec = np.ascontiguousarray(rec, np.int64)
    prob = np.ascontiguousarray(prob, np.float32)
    P, L, K = len(count) // 4, rec.shape[1], max(pts.shape[0], 1)
    out = dict(count=np.zeros(P, np.int32), offset=np.zeros(P, np.int32), pts=np.zeros((K, 2)),
               polys=np.zeros((K, 32)), rec=np.zeros((K, L), np.int64), prob=np.zeros((K, L), np.float32),
               source=np.zeros((K, 2), np.int32))
    n = lib.emu_merge_turns(P, count.ctypes.data, offset.ctypes.data, pts.ctypes.data, polys.ctypes.data,
                            rec.ctypes.data, prob.ctypes.data, L, pad, eos, iou,
                            *[out[k].ctypes.data for k in ('count', 'offset', 'pts', 'polys', 'rec', 'prob', 'source')])
    for k in ('pts', 'polys', 'rec', 'prob', 'source'):
        out[k] = out[k][:n]
    return out


def gold():
    return np.load(os.path.join(GOLD, 'omni_page_turns.npz'))


def fixture_rows():
    """The fixture's four merged readings (turns 0..3 of one page) as the input of one page's turn merge."""
    g = gold()
    return ((g['merged_count'], g['merged_offset'], g['merged_pts'], g['merged_polys'], g['merged_rec'],
             g['merged_prob']), int(g['recog_pad_index']), int(g['rec_eos_index']))


def poly_of(x0, y0, x1, y1):
    """16 vertices of an axis-aligned word: top boundary left to right, bottom right to left."""
    xs = np.concatenate([np.linspace(x0, x1, 8), np.linspace(x1, x0, 8)])
    ys = np.concatenate([np.full(8, y0), np.full(8, y1)])
    return np.stack([xs, ys], 1).reshape(-1)


def make(readings, L=4):
    """Rows from readings [4 P] of lists of (x0, y0, x1, y1, q): one recognised token of probability q then eos, so
    the row's score is q / (1 + 1e-5) and equal q give equal scores."""
    count = np.array([len(r) for r in readings], np.int32)
    offset = (np.cumsum(count) - count).astype(np.int32)
    rows = [w for r in readings for w in r]
    N = len(rows)
    polys = np.array([poly_of(*w[:4]) for w in rows], np.float64).reshape(N, 32)
    pts = np.array([((w[0] + w[2]) / 2, (w[1] + w[3]) / 2) for w in rows], np.float64).reshape(N, 2)
    rec = np.full((N, L), EOS, np.int64)
    rec[:, 0] = 1000
    prob = np.zeros((N, L), np.float32)
    prob[:, 0] = [w[4] for w in rows]
    return count, offset, pts, polys, rec, prob


def fabricate(rng, P, max_rows=600):
    """Readings of P pages of random words: each reading sees a random subset of its page's words with jittered
    boxes (cross-turn IoU spread around 0.5) and a few junk rows; probabilities from a small set (exact score ties
    are common); some readings and pages are empty, some readings exceed one 128-row block."""
    readings = []
    for p in range(P):
        n_words = int(rng.choice([0, 3, 20, 150, max_rows, 2 * max_rows]))
        words = [(rng.uniform(0, 900), rng.uniform(0, 900), rng.uniform(8, 90), rng.uniform(5, 40))
                 for _ in range(n_words)]
        for k in range(4):
            rows = []
            if rng.random() < 0.15:
                readings.append(rows)
                continue
            for x, y, w, h in words:
                if rng.random() < 0.5:
                    continue
                j = rng.normal(0, 0.18, 4)
                rows.append((x + j[0] * w, y + j[1] * h, x + w + j[2] * w, y + h + j[3] * h,
                             float(rng.choice([0.25, 0.5, 0.75, 0.875, 1.0]))))
            rows = rows[:max_rows]
            readings.append(rows)
    out = make(readings, L=6)
    count, offset, pts, polys, rec, prob = out
    # multi-token rows too, with skipped 'unknown' ids and a row that stops at once
    N = len(pts)
    if N:
        pick = rng.random(N) < 0.3
        rec[pick, 1:] = rng.choice([1001, PAD - 1, PAD, EOS], (int(pick.sum()), rec.shape[1] - 1))
        prob[pick, 1:] = rng.choice([0.5, 0.25, 1.0], (int(pick.sum()), rec.shape[1] - 1)).astype(np.float32)
    return out


def drop_directions(count, offset, polys, rec, prob, pad=PAD, eos=EOS, iou=0.5):
    """Per dropped row, whether a lower or a higher turn dropped it -> the set of directions seen, and the number of
    dropped rows (by the oracle's own functions)."""
    polys = np.asarray(polys).reshape(-1, 32)
    box = [R.box(v) for v in polys]
    s = [PT.spot_score(rec[n], prob[n], pad, eos) for n in range(len(polys))]
    seen, dropped = set(), 0
    for p in range(len(count) // 4):
        rows = [[int(offset[4 * p + k]) + i for i in range(int(count[4 * p + k]))] for k in range(4)]
        for ka in range(4):
            for ia, a in enumerate(rows[ka]):
                by = {('lower' if kb < ka else 'higher') for kb in range(4) if kb != ka
                      for ib, b in enumerate(rows[kb])
                      if R.above(s[b], kb, ib, s[a], ka, ia) and tile_ref.iou_at_least(box[b], box[a], iou)}
                seen |= by
                dropped += bool(by)
    return seen, dropped


def test_the_fixture_equals_the_oracle():
    """The reference's tiled readings of one page at turns 0..3: emulation == oracle bit for bit; rows are dropped."""
    args, pad, eos = fixture_rows()
    got = emu_merge(*args, pad=pad, eos=eos)
    assert_same(got, R.merge(*args, pad, eos))
    n_in = int(args[0].sum())
    assert 0 < int(got['count'][0]) < n_in
    _, dropped = drop_directions(args[0], args[1], args[3], args[4], args[5], pad, eos)
    assert dropped == n_in - int(got['count'][0])


def test_fabricated_readings_equal_the_oracle():
    """Many pages, 0..600 rows per reading, cross-turn overlaps around theta and exact score ties, at three
    thresholds: emulation == oracle bit for bit."""
    rng = np.random.default_rng(11)
    for P, iou in ((9, 0.5), (7, 0.3), (7, 0.75), (3, 1.0)):
        args = fabricate(rng, P)
        got = emu_merge(*args, iou=iou)
        assert_same(got, R.merge(*args, PAD, EOS, iou))
        assert iou == 1.0 or got['count'].sum() < args[0].sum()


def test_suppression_runs_both_ways():
    """Between the fixture and the fabricated readings, a lower turn drops a higher one and a higher turn drops a
    lower one."""
    args, pad, eos = fixture_rows()
    seen, _ = drop_directions(args[0], args[1], args[3], args[4], args[5], pad, eos)
    c, o, _, polys, rec, prob = fabricate(np.random.default_rng(11), 9)
    seen |= drop_directions(c, o, polys, rec, prob)[0]
    assert seen == {'lower', 'higher'}


def check(readings, want_sources, iou=0.5):
    """Emulation == oracle, and the kept (turn, index) per page are want_sources."""
    args = make(readings)
    got = emu_merge(*args, iou=iou)
    assert_same(got, R.merge(*args, PAD, EOS, iou))
    pages = [got['source'][o:o + c].tolist() for c, o in zip(got['count'], got['offset'])]
    assert pages == want_sources
    return got


W = (10.0, 20.0, 50.0, 30.0)  # a word's box


def test_a_word_read_at_two_turns_keeps_the_higher_score():
    check([[(*W, 0.6)], [], [(*W, 0.9)], []], [[[2, 0]]])
    check([[(*W, 0.9)], [], [(*W, 0.6)], []], [[[0, 0]]])


def test_equal_scores_keep_the_lower_turn():
    check([[], [(*W, 0.7)], [], [(*W, 0.7)]], [[[1, 0]]])
    check([[(*W, 0.7)], [(*W, 0.7)], [(*W, 0.7)], [(*W, 0.7)]], [[[0, 0]]])


def test_overlapping_rows_of_one_turn_both_stay():
    check([[(*W, 0.6), (*W, 0.9)], [], [], []], [[[0, 0], [0, 1]]])
    # and a better row at another turn drops them both
    check([[(*W, 0.6), (*W, 0.7)], [], [], [(*W, 0.8)]], [[[3, 0]]])


def test_a_non_transitive_chain_drops_two_rows():
    """a (turn 0) < b (turn 1) < c (turn 2); IoU(a, b) = IoU(b, c) = 7 / 13 >= 0.5, IoU(a, c) = 1 / 4: b drops a and c
    drops b, so only c stays (greedy NMS would keep a as well)."""
    a, b, c = (0, 0, 10, 10, 0.5), (3, 0, 13, 10, 0.6), (6, 0, 16, 10, 0.7)
    check([[a], [b], [c], []], [[[2, 0]]])


def test_non_finite_rows_are_kept_and_drop_nothing():
    """A row with a NaN vertex never matches; a row with a NaN score never ranks above another and none ranks above
    it: both are kept, and so are the rows they overlap.  An infinite vertex never matches either."""
    args = make([[(*W, 0.5)], [(*W, 0.99)], [], [],
                 [(*W, float('nan'))], [], [], [(*W, 0.1)],
                 [(*W, 0.5)], [], [(*W, 0.9)], []])
    count, offset, pts, polys, rec, prob = args
    polys[1, 7] = np.nan            # page 0, turn 1: a NaN vertex on the best row
    polys[5, 0] = np.inf            # page 2, turn 2: an infinite vertex on the better row
    got = emu_merge(*args)
    assert_same(got, R.merge(*args, PAD, EOS))
    pages = [got['source'][o:o + c].tolist() for c, o in zip(got['count'], got['offset'])]
    assert pages == [[[0, 0], [1, 0]], [[0, 0], [3, 0]], [[0, 0], [2, 0]]]
    assert np.isnan(R.box(polys[1])).all() and np.isnan(R.box(polys[5])).all()
    box, score = np.zeros(4), np.zeros(1)
    lib = emu('turn_merge_emu', bind)
    lib.emu_map_row(polys[1].ctypes.data, rec[1].ctypes.data, prob[1].ctypes.data, rec.shape[1], PAD, EOS,
                    box.ctypes.data, score.ctypes.data)
    assert np.isnan(box).all() and score[0] == PT.spot_score(rec[1], prob[1], PAD, EOS)


def test_empty_readings_and_empty_pages():
    check([[], [], [], []], [[]])
    check([[], [], [], [], [(*W, 0.5)], [], [], [], [], [], [], []], [[], [[0, 0]], []])
    got = check([[]] * 4 + [[], [], [], [(*W, 0.5)]] + [[]] * 8, [[], [[3, 0]], [], []])
    assert got['offset'].tolist() == [0, 0, 1, 1]


def test_one_non_empty_reading_comes_back_unchanged():
    """A page read with words at one turn only keeps that reading's rows, unchanged and in order, over several
    blocks of rows."""
    rng = np.random.default_rng(5)
    for k in range(4):
        rows = [(x, y, x + 30, y + 9, float(rng.choice([0.5, 1.0]))) for x, y in rng.uniform(0, 50, (300, 2))]
        readings = [[] for _ in range(8)]
        readings[k] = rows[:5]
        readings[4 + k] = rows
        args = make(readings)
        got = check(readings, [[[k, i] for i in range(5)], [[k, i] for i in range(300)]])
        for key, a in zip(('pts', 'polys', 'rec', 'prob'), args[2:]):
            assert np.array_equal(got[key], a), key


def test_the_python_wrapper_refuses_bad_arguments():
    """merge_turns raises ValueError on the host, before any library call: iou outside (0, 1] or not finite, a count
    that is not four readings per page, negative counts, offsets that are not the counts' prefix sum, row arrays that
    disagree with the counts."""
    from advancedliteratemachinery_b200.omniparser import merge_turns
    args = make([[(*W, 0.5)], [(*W, 0.6)], [], []])
    count, offset, pts, polys, rec, prob = args
    for iou in (0.0, -0.1, 1.5, float('nan'), float('inf')):
        with pytest.raises(ValueError):
            merge_turns(None, *args, PAD, EOS, iou=iou)
    bad = [
        (count[:3], offset[:3], pts, polys, rec, prob),
        (count, offset[:2], pts, polys, rec, prob),
        (np.array([3, 0, 0, 0]), np.array([0, 3, 3, 3]), pts, polys, rec, prob),
        (np.array([3, -1, 0, 0]), np.array([0, 3, 2, 2]), pts, polys, rec, prob),
        (count, np.array([0, 0, 2, 2]), pts, polys, rec, prob),
        (count, offset, pts[:1], polys, rec, prob),
        (count, offset, pts, polys[:1], rec, prob),
        (count, offset, pts, polys, rec, prob[:, :2]),
        (count, offset, pts, polys, rec[:, :0], prob[:, :0]),
    ]
    for b in bad:
        with pytest.raises(ValueError):
            merge_turns(None, *b, PAD, EOS)
