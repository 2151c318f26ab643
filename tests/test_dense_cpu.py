"""Dense pages read in spatial windows (DESIGN 4.16): CPU checks of the rule's bodies run on the host
(tests/emu/dense_emu.cpp) against oracle/dense_ref.py.  The window table must be the training code's grids, ownership
must partition the page, the point filter must keep exactly the owned points, and the merge of n window readings must
equal the oracle bit for bit (and alm_omni_merge_turns' emulation at n = 4)."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle import dense_ref as D
from tests.support import assert_same, emu
from tests.test_turn_merge_cpu import EOS, PAD, emu_merge, fixture_rows, poly_of

_EMU = None
NB = 1000


def bind(lib):
    """Bind tests/emu/dense_emu.cpp (host compile of the kernels' bodies)."""
    lib.emu_window.argtypes = [C.c_int] * 4 + [C.c_void_p]
    lib.emu_owns.argtypes = [C.c_void_p, C.c_int64, C.c_int64]
    lib.emu_trained_grid.argtypes = [C.c_int, C.c_int]
    lib.emu_own_points.argtypes = [C.c_void_p] + [C.c_int] * 6 + [C.c_void_p]
    lib.emu_merge_readings.restype = C.c_long
    lib.emu_merge_readings.argtypes = ([C.c_int, C.c_int] + [C.c_void_p] * 6 + [C.c_int, C.c_int64, C.c_int64, C.c_double]
                                       + [C.c_void_p] * 7)


def emu_window(nx, ny, w, nb=NB):
    box = np.zeros(4, np.int32)
    emu('dense_emu', bind).emu_window(nb, nx, ny, w, box.ctypes.data)
    return box.tolist()


def emu_merge_readings(nr, count, offset, pts, polys, rec, prob, pad=PAD, eos=EOS, iou=0.5):
    """alm_omni_merge_readings' three launches on the host -> the dict merge_readings / dense_ref.merge return."""
    lib = emu('dense_emu', bind)
    count = np.ascontiguousarray(count, np.int32)
    offset = np.ascontiguousarray(offset, np.int32)
    pts = np.ascontiguousarray(pts, np.float64).reshape(-1, 2)
    polys = np.ascontiguousarray(polys, np.float64).reshape(-1, 32)
    rec = np.ascontiguousarray(rec, np.int64)
    prob = np.ascontiguousarray(prob, np.float32)
    P, L, K = len(count) // nr, rec.shape[1], max(pts.shape[0], 1)
    out = dict(count=np.zeros(P, np.int32), offset=np.zeros(P, np.int32), pts=np.zeros((K, 2)),
               polys=np.zeros((K, 32)), rec=np.zeros((K, L), np.int64), prob=np.zeros((K, L), np.float32),
               source=np.zeros((K, 2), np.int32))
    n = lib.emu_merge_readings(P, nr, count.ctypes.data, offset.ctypes.data, pts.ctypes.data, polys.ctypes.data,
                               rec.ctypes.data, prob.ctypes.data, L, pad, eos, iou,
                               *[out[k].ctypes.data for k in ('count', 'offset', 'pts', 'polys', 'rec', 'prob',
                                                              'source')])
    for k in ('pts', 'polys', 'rec', 'prob', 'source'):
        out[k] = out[k][:n]
    return out


def rows_of(readings, L=4):
    """Rows from readings [nr P] of lists of (x0, y0, x1, y1, q) in bins: one token of probability q then eos."""
    count = np.array([len(r) for r in readings], np.int32)
    offset = (np.cumsum(count) - count).astype(np.int32)
    rows = [w for r in readings for w in r]
    N = len(rows)
    polys = np.array([poly_of(*w[:4]) for w in rows], np.float64).reshape(N, 32)
    pts = np.array([((w[0] + w[2]) // 2, (w[1] + w[3]) // 2) for w in rows], np.float64).reshape(N, 2)
    rec = np.full((N, L), EOS, np.int64)
    rec[:, 0] = 1000
    prob = np.zeros((N, L), np.float32)
    prob[:, 0] = [w[4] for w in rows]
    return count, offset, pts, polys, rec, prob


def fabricate(rng, P, nr, max_rows=600):
    """Window readings of P pages in integer bins: every window reads the words of its page near it, jittered so that
    the IoU of two readings of a word spreads around 0.5, probabilities from a small set (exact score ties); some
    windows and pages are empty, some exceed one 128-row block."""
    readings = []
    for p in range(P):
        n_words = int(rng.choice([0, 5, 40, 300, max_rows]))
        words = [(int(rng.integers(0, 950)), int(rng.integers(0, 970)), int(rng.integers(4, 50)),
                  int(rng.integers(3, 30))) for _ in range(n_words)]
        for k in range(nr):
            rows = []
            if rng.random() < 0.1:
                readings.append(rows)
                continue
            for x, y, w, h in words:
                if rng.random() < 1.0 - 1.5 / nr:
                    continue
                j = rng.integers(-2, 3, 4)
                rows.append((x + j[0], y + j[1], x + w + j[2], y + h + j[3],
                             float(rng.choice([0.25, 0.5, 0.75, 1.0]))))
            readings.append(rows[:max_rows])
    return rows_of(readings, L=5)


# ---------------------------------------------------------------------------------------------------- windows
@pytest.mark.parametrize('nx,ny', D.TRAINED)
def test_window_table_is_the_training_grid(nx, ny):
    want = D.collate_windows(nx, ny, NB)
    got = [emu_window(nx, ny, w) for w in range(nx * ny)]
    assert sorted(got) == sorted(want)
    assert got == D.windows(nx, ny, NB)
    # row-major: top to bottom, then left to right
    assert [(b[1], b[0]) for b in got] == sorted((b[1], b[0]) for b in got)


def test_window_table_at_1000_bins():
    assert [emu_window(1, 1, 0)] == [[0, 0, 999, 999]]
    assert [emu_window(2, 1, w)[0::2] for w in range(2)] == [[0, 500], [500, 999]]
    assert [emu_window(3, 1, w)[0::2] for w in range(3)] == [[0, 333], [333, 666], [666, 999]]


def test_only_the_trained_grids_are_allowed():
    lib = emu('dense_emu', bind)
    for nx in range(-1, 6):
        for ny in range(-1, 6):
            assert lib.emu_trained_grid(nx, ny) == ((nx, ny) in D.TRAINED)


@pytest.mark.parametrize('nx,ny', D.TRAINED)
@pytest.mark.parametrize('nb', [1000, 7, 3])
def test_ownership_partitions_the_page(nx, ny, nb):
    lib = emu('dense_emu', bind)
    boxes = [np.array(emu_window(nx, ny, w, nb), np.int32) for w in range(nx * ny)]
    v = np.arange(nb)
    for x in v[::max(1, nb // 97)].tolist() + [nb - 1]:
        for y in v[::max(1, nb // 89)].tolist() + [nb - 1]:
            owners = [w for w, b in enumerate(boxes) if lib.emu_owns(b.ctypes.data, x, y)]
            assert len(owners) == 1, (x, y, owners)
            assert owners == [w for w, b in enumerate(boxes) if D.owns(b.tolist(), x, y)]
    # tokens outside the bins belong to no window
    for x, y in [(-1, 0), (0, nb), (nb + 5, 3)]:
        assert not any(lib.emu_owns(b.ctypes.data, x, y) for b in boxes)


def test_point_filter_keeps_the_owned_points_in_order():
    lib = emu('dense_emu', bind)
    rng = np.random.default_rng(3)
    for nx, ny in D.TRAINED:
        for w in range(nx * ny):
            n_prompt = 7
            n = int(rng.integers(0, 40))
            tok = np.concatenate([np.arange(n_prompt), rng.integers(0, NB + 3, n)]).astype(np.int32)
            xy = np.zeros(2 * max(1, n), np.int32)
            k = lib.emu_own_points(tok.ctypes.data, n_prompt, n, NB, nx, ny, w, xy.ctypes.data)
            want = D.owned_points(D.windows(nx, ny)[w], tok[n_prompt:n_prompt + n])
            assert [tuple(p) for p in xy[:2 * k].reshape(-1, 2).tolist()] == want


# ---------------------------------------------------------------------------------------------------- merge
@pytest.mark.parametrize('nr', [2, 4, 9])
@pytest.mark.parametrize('seed', [0, 1, 2])
def test_merge_equals_the_oracle_on_fabricated_pages(nr, seed):
    rng = np.random.default_rng(100 * nr + seed)
    rows = fabricate(rng, 3, nr)
    count = rows[0]
    dropped = 0
    for iou in (0.5, 0.3, 1.0):
        got = emu_merge_readings(nr, *rows, iou=iou)
        assert_same(got, D.merge(nr, *rows, PAD, EOS, iou))
        dropped += int(count.sum() - got['count'].sum())
    assert dropped > 0


def test_merge_equals_the_oracle_at_600_rows_per_window():
    rng = np.random.default_rng(7)
    readings = []
    for k in range(9):
        readings.append([(int(x), int(y), int(x) + 20, int(y) + 10, float(q))
                         for x, y, q in zip(rng.integers(0, 200, 600), rng.integers(0, 200, 600),
                                            rng.choice([0.5, 1.0], 600))])
    rows = rows_of(readings)
    assert_same(emu_merge_readings(9, *rows), D.merge(9, *rows, PAD, EOS, 0.5))


def test_merge_at_four_readings_is_the_turn_merge():
    rows, pad, eos = fixture_rows()
    assert_same(emu_merge_readings(4, *rows, pad=pad, eos=eos), emu_merge(*rows, pad=pad, eos=eos))
    rng = np.random.default_rng(11)
    rows = fabricate(rng, 4, 4)
    assert_same(emu_merge_readings(4, *rows), emu_merge(*rows))


def hand(readings, nr=4, iou=0.5):
    rows = rows_of(readings)
    got = emu_merge_readings(nr, *rows, iou=iou)
    assert_same(got, D.merge(nr, *rows, PAD, EOS, iou))
    return got


def test_a_word_straddling_a_seam_is_kept_once():
    # windows 0 and 1 of a 2 x 2 grid both read the word at x = 495..510; window 1 reads it better
    got = hand([[(495, 10, 510, 20, 0.5)], [(496, 10, 510, 20, 0.75)], [], []])
    assert got['source'].tolist() == [[1, 0]]


def test_equal_scores_keep_the_lower_window():
    got = hand([[], [], [(100, 100, 140, 120, 1.0)], [(100, 101, 140, 120, 1.0)]])
    assert got['source'].tolist() == [[2, 0]]


def test_rows_of_one_window_never_drop_each_other():
    got = hand([[(0, 0, 40, 20, 1.0), (0, 0, 40, 20, 0.5)], [], [], []])
    assert got['source'].tolist() == [[0, 0], [0, 1]]


def test_empty_windows_and_pages():
    got = hand([[]] * 9 + [[(5, 5, 9, 9, 0.5)]] + [[]] * 8, nr=9)
    assert got['count'].tolist() == [0, 1] and got['source'].tolist() == [[0, 0]]


def test_nan_rows_never_match_and_are_never_dropped():
    rows = rows_of([[(0, 0, 40, 20, 0.5)], [(0, 0, 40, 20, 1.0)], [], []])
    count, offset, pts, polys, rec, prob = rows
    polys[1, 3] = np.nan
    prob[0, 0] = np.nan
    got = emu_merge_readings(4, *rows)
    assert_same(got, D.merge(4, *rows, PAD, EOS, 0.5))
    assert got['source'].tolist() == [[0, 0], [1, 0]]


# ---------------------------------------------------------------------------------------------------- reference fixture
def dense_gold():
    return np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'omni_dense.npz'))


def test_fixture_levels_follow_the_auto_rule():
    g = dense_gold()
    flags = {1: [bool(g['sat0'][0])], 2: g['sat2'].tolist(), 3: g['sat3'].tolist()}
    side, kept = D.auto_reading(lambda n: [(None, s) for s in flags[n]])
    assert side == 3 and [s for _, s in kept] == flags[3]
    assert flags[1] == [True] and any(flags[2]) and not all(flags[2]) and not all(flags[3])


def test_merge_equals_the_reference_fixture():
    g = dense_gold()
    rows = tuple(g[f'win_{k}'] for k in ('count', 'offset', 'pts', 'polys', 'rec', 'prob'))
    pad, eos, iou = int(g['recog_pad_index'][0]), int(g['rec_eos_index'][0]), float(g['iou'][0])
    got = emu_merge_readings(9, *rows, pad=pad, eos=eos, iou=iou)
    assert_same(got, {k: g[f'merged_{k}'] for k in ('count', 'offset', 'pts', 'polys', 'rec', 'prob', 'source')})
    assert_same(got, D.merge(9, *rows, pad, eos, iou))
    for w in range(9):  # every stored row is owned by its window
        box = D.windows(3, 3)[w]
        lo = int(rows[1][w])
        assert all(D.owns(box, int(x), int(y)) for x, y in rows[2][lo:lo + int(rows[0][w])])
