"""Words that cross tile seams, recovered from a whole-page reading (DESIGN 4.17): CPU checks with the kernels' bodies
run on the host (tests/emu/whole_page_emu.cpp) against oracle/whole_page_ref.py, bit for bit, on the reference's
readings of one page (tests/golden/omni_whole_page.npz), on fabricated pages and on hand-made cases, plus the rule's
stated properties."""
import ctypes as C
import math
import os

import numpy as np
import pytest

from oracle import tile_ref
from oracle import whole_page_ref as R
from tests.support import assert_same, emu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
NB = 1000
A4 = (3508, 2480)


def bind(lib):
    """Bind tests/emu/whole_page_emu.cpp (host compile of the kernels' bodies)."""
    lib.emu_merge_whole_page.restype = C.c_long
    lib.emu_merge_whole_page.argtypes = ([C.c_int] + [C.c_void_p] * 3 + [C.c_int, C.c_int, C.c_double, C.c_int] +
                                         [C.c_void_p] * 12 + [C.c_int, C.c_int] + [C.c_void_p] * 7)
    lib.emu_inside.restype = C.c_int
    lib.emu_inside.argtypes = [C.c_double, C.c_double, C.c_void_p]


def emu_merge(sizes, turns, T, ov, margin, num_bins, tiles, n_inst, pt, poly, rec, prob):
    """alm_omni_merge_whole_page's three launches on the host -> the dict merge_whole_page / whole_page_ref.merge
    return."""
    lib = emu('whole_page_emu', bind)
    P = len(sizes)
    hs = np.ascontiguousarray([s[0] for s in sizes], np.int32)
    ws = np.ascontiguousarray([s[1] for s in sizes], np.int32)
    tr = None if turns is None else np.ascontiguousarray(turns, np.int32)
    t = {k: np.ascontiguousarray(tiles[k], d) for k, d in
         (('count', np.int32), ('offset', np.int32), ('pts', np.float64), ('polys', np.float64), ('rec', np.int64),
          ('prob', np.float32), ('source', np.int32))}
    n_inst = np.ascontiguousarray(n_inst, np.int32)
    pt, poly, rec = (np.ascontiguousarray(a, np.int64) for a in (pt, poly, rec))
    prob = np.ascontiguousarray(prob, np.float32)
    L, cap = rec.shape[2], pt.shape[1]
    K = max(t['pts'].shape[0] + int(n_inst.sum()), 1)
    out = dict(count=np.zeros(P, np.int32), offset=np.zeros(P, np.int32), pts=np.zeros((K, 2)),
               polys=np.zeros((K, 32)), rec=np.zeros((K, L), np.int64), prob=np.zeros((K, L), np.float32),
               source=np.zeros((K, 2), np.int32))
    n = lib.emu_merge_whole_page(P, hs.ctypes.data, ws.ctypes.data, None if tr is None else tr.ctypes.data, T, ov,
                                 margin, num_bins,
                                 *[t[k].ctypes.data for k in ('count', 'offset', 'pts', 'polys', 'rec', 'prob',
                                                              'source')],
                                 n_inst.ctypes.data, pt.ctypes.data, poly.ctypes.data, rec.ctypes.data,
                                 prob.ctypes.data, cap, L,
                                 *[out[k].ctypes.data for k in ('count', 'offset', 'pts', 'polys', 'rec', 'prob',
                                                                'source')])
    for k in ('pts', 'polys', 'rec', 'prob', 'source'):
        out[k] = out[k][:n]
    return out


def both(*args):
    """The emulation equals the oracle bit for bit; returns the result."""
    got = emu_merge(*args)
    want = R.merge(*args)
    assert_same(got, want)
    return got


# ---- fabrication -------------------------------------------------------------------------------------------------


def band_poly(x0, y0, x1, y1, slant=0.0):
    """16 vertices of a word from (x0, y0) to (x1, y1) (top-left, bottom-right of the upright box), the bottom edge
    shifted by slant in x: top boundary left to right, bottom right to left."""
    xs = np.concatenate([np.linspace(x0, x1, 8), np.linspace(x1, x0, 8) + slant])
    ys = np.concatenate([np.full(8, y0), np.full(8, y1)])
    return np.stack([xs, ys], 1).reshape(-1)


def to_bins(poly, tw, th):
    """Page-frame vertices [32] -> coordinate ids in a tw x th frame (clamped to the bins)."""
    v = np.asarray(poly, np.float64).copy()
    v[0::2] = np.floor(v[0::2] / tw * NB)
    v[1::2] = np.floor(v[1::2] / th * NB)
    return np.clip(v, 0, NB - 1).astype(np.int64)


def tile_rows(rows, P, L=3):
    """Tile rows from per page lists of (pts (x, y), polys [32]) -> the tile merge's dict."""
    count = np.array([len(r) for r in rows], np.int32)
    flat = [x for r in rows for x in r]
    N = len(flat)
    rng = np.random.default_rng(N)
    return dict(count=count, offset=(np.cumsum(count) - count).astype(np.int32),
                pts=np.array([x[0] for x in flat], np.float64).reshape(N, 2),
                polys=np.array([x[1] for x in flat], np.float64).reshape(N, 32),
                rec=rng.integers(0, 1100, (N, L)).astype(np.int64), prob=rng.random((N, L)).astype(np.float32),
                source=np.stack([np.arange(N), np.arange(N) % 7], 1).astype(np.int32).reshape(N, 2))


def whole_readings(words, P, cap=None, L=3):
    """Whole-page readings from per page lists of (pt ids [2], poly ids [32]) -> (n_inst, pt, poly, rec, prob)."""
    cap = max([len(w) for w in words] + [1]) if cap is None else cap
    n_inst = np.array([len(w) for w in words], np.int32)
    pt = np.zeros((P, cap, 2), np.int64)
    poly = np.zeros((P, cap, 32), np.int64)
    for p, ws in enumerate(words):
        for i, (a, b) in enumerate(ws):
            pt[p, i], poly[p, i] = a, b
    rng = np.random.default_rng(int(n_inst.sum()))
    return (n_inst, pt, poly, rng.integers(0, 1100, (P, cap, L)).astype(np.int64),
            rng.random((P, cap, L)).astype(np.float32))


def fabricate(rng, P, max_rows):
    """P pages of random sizes and turns under one random layout: whole-page words of every width (many wider than
    the overlap, some slanted), tile rows scattered over the page and on the whole words' polygons and boxes."""
    T = int(rng.integers(64, 700))
    ov = int(rng.integers(0, T // 2 + 1))
    sizes = [(int(rng.integers(20, 4 * T)), int(rng.integers(20, 4 * T))) for _ in range(P)]
    sizes[0] = (min(sizes[0][0], T), min(sizes[0][1], T))  # one single-tile page
    turns = rng.integers(0, 4, P).astype(np.int32)
    words, rows = [], []
    for p, (H, W) in enumerate(sizes):
        th, tw = R.turned(H, W, int(turns[p]))
        n = int(rng.choice([0, 1, 5, max_rows]))
        ws, page_words = [], []
        for _ in range(n):
            w, h = rng.uniform(2, tw) * rng.choice([0.05, 0.3, 1.0]), rng.uniform(2, th) * rng.choice([0.05, 0.3])
            x, y = rng.uniform(0, max(tw - w, 1)), rng.uniform(0, max(th - h, 1))
            v = band_poly(x, y, x + w, y + h, rng.choice([0.0, rng.uniform(-w, w)]))
            ws.append((to_bins([x + w / 2, y + h / 2], tw, th), to_bins(v, tw, th)))
            page_words.append(R.whole_rows([(H, W)], [turns[p]], T, ov, 4.0, [1], ws[-1][0][None, None],
                                           ws[-1][1][None, None], NB)[0][0][2])
        words.append(ws)
        tr = []
        for _ in range(int(rng.choice([0, 3, max_rows]))):
            if page_words and rng.random() < 0.6:
                v = np.asarray(page_words[int(rng.integers(len(page_words)))]).reshape(16, 2)
                a, b = v[int(rng.integers(16))], v[int(rng.integers(16))]
                pt_ = a + (b - a) * rng.random()  # on a chord of a whole polygon: inside or on its border
                if rng.random() < 0.3:
                    pt_ = np.array([rng.uniform(v[:, 0].min(), v[:, 0].max()),
                                    rng.uniform(v[:, 1].min(), v[:, 1].max())])  # in its box
            else:
                pt_ = np.array([rng.uniform(0, W), rng.uniform(0, H)])
            tr.append((pt_, band_poly(pt_[0] - 5, pt_[1] - 3, pt_[0] + 5, pt_[1] + 3)))
        rows.append(tr)
    return sizes, turns, T, ov, tile_rows(rows, P), whole_readings(words, P)


@pytest.mark.parametrize('seed', range(6))
def test_emulation_equals_the_oracle_on_fabricated_pages(seed):
    rng = np.random.default_rng(seed)
    sizes, turns, T, ov, tiles, whole = fabricate(rng, int(rng.integers(1, 5)), 250)
    for tr in (turns, None):
        got = both(sizes, tr, T, ov, 4.0, NB, tiles, *whole)
        assert got['count'].sum() <= tiles['count'].sum() + whole[0].sum()


def test_fabrication_exercises_both_decisions():
    kept_whole = dropped = 0
    for seed in range(6):
        rng = np.random.default_rng(seed)
        sizes, turns, T, ov, tiles, whole = fabricate(rng, int(rng.integers(1, 5)), 250)
        got = emu_merge(sizes, turns, T, ov, 4.0, NB, tiles, *whole)
        kept_whole += int((got['source'][:, 0] < 0).sum())
        dropped += int(tiles['count'].sum()) - int((got['source'][:, 0] >= 0).sum())
    assert kept_whole > 20 and dropped > 20


# ---- the reference fixture ---------------------------------------------------------------------------------------


def gold():
    """The fixture, with its page: omni_tiles.npz's (the same page seed)."""
    g = dict(np.load(os.path.join(GOLD, 'omni_whole_page.npz')))
    t = np.load(os.path.join(GOLD, 'omni_tiles.npz'))
    assert int(g['seed']) == int(t['seed'])
    g['page'] = t['page']
    return g


def test_fixture_merge_equals_the_emulation_and_the_oracle():
    g = gold()
    size = tuple(int(x) for x in g['page'].shape[:2])
    T, ov, nb = int(g['tile']), int(g['overlap']), int(g['num_bins'])
    tm = tile_ref.merge([size], T, ov, g['n_inst'], g['pt'], g['poly'], g['rec'], g['prob'], nb)
    assert_same(tm, {k: g[f'tiles_{k}'] for k in tm})
    args = ([size], None, T, ov, float(g['margin']), nb, tm, g['whole_n_inst'], g['whole_pt'], g['whole_poly'],
            g['whole_rec'], g['whole_prob'])
    got = both(*args)
    assert_same(got, {k: g[f'merged_{k}'] for k in got})
    whole = got['source'][:, 0] < 0
    assert whole.sum() >= 1 and (~whole).sum() < tm['count'].sum()  # a whole row kept, a tile row dropped
    # the whole rows' coordinates are decode_pred_seq's of the reference's whole-page reading
    inst = got['source'][whole, 1]
    assert np.array_equal(got['pts'][whole], g['whole_ref_pts'][0][inst])
    assert np.array_equal(got['polys'][whole], g['whole_ref_polys'][0][inst])


# ---- hand-made cases ---------------------------------------------------------------------------------------------


def a4_tile_decode(words, T=1200, ov=256, max_inst=4, L=3):
    """Tile decodes of an A4 page from page-frame words [(x0, y0, x1, y1)]: every tile reads the part of each word it
    sees (clipped to the tile)."""
    plan = tile_ref.plan([A4], T, ov)
    nt = len(plan)
    n_inst = np.zeros(nt, np.int32)
    pt = np.zeros((nt, max_inst, 2), np.int64)
    poly = np.zeros((nt, max_inst, 32), np.int64)
    for k, (_, y0, x0, h, w) in enumerate(plan):
        for (a, b, c, d) in words:
            if c <= x0 or a >= x0 + w or d <= y0 or b >= y0 + h:
                continue
            a_, b_, c_, d_ = max(a, x0) - x0, max(b, y0) - y0, min(c, x0 + w) - x0, min(d, y0 + h) - y0
            i = n_inst[k]
            poly[k, i] = np.clip(np.round(band_poly(a_, b_, c_, d_) / np.tile([w, h], 16) * NB), 0, NB - 1)
            pt[k, i] = np.round(np.array([(a_ + c_) / 2 / w, (b_ + d_) / 2 / h]) * NB)
            n_inst[k] += 1
    rng = np.random.default_rng(0)
    return (n_inst, pt, poly, rng.integers(0, 1100, (nt, max_inst, L)).astype(np.int64),
            rng.random((nt, max_inst, L)).astype(np.float32))


def whole_word(x0, y0, x1, y1, size=A4, slant=0.0):
    H, W = size
    return to_bins([(x0 + x1) / 2, (y0 + y1) / 2], W, H), to_bins(band_poly(x0, y0, x1, y1, slant), W, H)


def test_a4_seam_word_is_lost_by_the_tiles_and_recovered_whole():
    """Columns [0, 1200), [944, 2144), [1280, 2480): a word over x = 944 .. 1200 is cut in every tile that sees it, so
    the tile merge loses it; tile 0's partial reading (stopping 20 px short of its edge) survives the tile merge."""
    assert tile_ref.axis(A4[1], 1200, 256) == [0, 944, 1280]
    tm = tile_ref.merge([A4], 1200, 256, *a4_tile_decode([(944, 500, 1200, 560)]), NB)
    assert tm['count'][0] == 0  # cut in every tile
    tm = tile_ref.merge([A4], 1200, 256, *a4_tile_decode([(944, 500, 1200, 560), (950, 505, 1180, 555)]), NB)
    assert tm['count'][0] == 1 and tuple(tm['source'][0]) == (0, 1)  # the fragment, read by tile 0 only
    whole = whole_readings([[whole_word(944, 500, 1200, 560)]], 1)
    got = both([A4], None, 1200, 256, 4.0, NB, tm, *whole)
    assert got['count'][0] == 1 and tuple(got['source'][0]) == (-1, 0)
    assert got['polys'][0][0] < 944 and got['polys'][0][14] > 1200 - 4  # the word, whole


def test_a_word_one_tile_sees_whole_stays_with_the_tile():
    tm = tile_ref.merge([A4], 1200, 256, *a4_tile_decode([(300, 500, 700, 560)]), NB)
    assert tm['count'][0] == 1
    whole = whole_readings([[whole_word(300, 500, 700, 560)]], 1)
    got = both([A4], None, 1200, 256, 4.0, NB, tm, *whole)
    assert_same(got, tm)


def test_a_slanted_whole_word_drops_by_its_polygon_not_its_box():
    """A kept whole word slanting from x ~ 900 at its top to ~ 1400 at its bottom: a tile word inside its box but
    outside its polygon stays, one on the polygon is dropped."""
    pts = [(1350.0, 430.0), (1150.0, 600.0)]  # box only, polygon
    tm = tile_rows([[(np.array(p), band_poly(p[0] - 5, p[1] - 3, p[0] + 5, p[1] + 3)) for p in pts]], 1)
    whole = whole_readings([[whole_word(900, 400, 1200, 800, slant=250.0)]], 1)
    got = both([A4], None, 1200, 256, 4.0, NB, tm, *whole)
    assert got['source'][:, 0].tolist() == [0, -1]
    v = R.whole_rows([A4], None, 1200, 256, 4.0, *whole[:3], NB)[0][0][2]
    assert min(v[0::2]) <= pts[0][0] <= max(v[0::2]) and min(v[1::2]) <= pts[0][1] <= max(v[1::2])


def test_a_word_over_a_four_tile_corner():
    size = (2000, 2000)  # 2 x 2 tiles, origins 0 and 800
    assert tile_ref.axis(2000, 1200, 256) == [0, 800]
    tm = tile_rows([[(np.array([1000.0, 1000.0]), band_poly(995, 997, 1005, 1003))]], 1)
    for box, kept in (((780, 780, 1220, 1220), True), ((780, 850, 1220, 1150), True), ((850, 850, 1150, 1150), False)):
        whole = whole_readings([[whole_word(*box, size=size)]], 1)
        got = both([size], None, 1200, 256, 4.0, NB, tm, *whole)
        assert got['source'][:, 0].tolist() == ([-1] if kept else [0])


def test_the_clamped_last_tile():
    size = (500, 1300)  # columns [0, 1200) and [100, 1300): the last one clamped
    assert tile_ref.axis(1300, 1200, 256) == [0, 100]
    tm = tile_rows([[]], 1)
    for box, kept in (((95, 100, 1205, 150), True), ((150, 100, 1150, 150), False), ((50, 100, 1250, 150), True)):
        whole = whole_readings([[whole_word(*box, size=size)]], 1)
        got = both([size], None, 1200, 256, 4.0, NB, tm, *whole)
        assert got['count'][0] == int(kept)


def test_single_tile_pages_keep_no_whole_row():
    """Property (b): the page fits in one tile, so nothing is cut; the tile rows come back unchanged."""
    rng = np.random.default_rng(3)
    sizes = [(300, 220), (1200, 1200), (64, 900)]
    words = [[(rng.integers(0, NB, 2), rng.integers(0, NB, 32)) for _ in range(40)] for _ in sizes]
    tm = tile_rows([[(np.array([rng.uniform(0, W), rng.uniform(0, H)]), rng.uniform(0, 900, 32)) for _ in range(30)]
                    for H, W in sizes], 3)
    whole = whole_readings(words, 3)
    for turns in (None, [0, 1, 3]):
        got = both(sizes, turns, 1200, 256, 4.0, NB, tm, *whole)
        assert_same(got, tm)


def test_nan_coordinates_are_never_inside():
    lib = emu('whole_page_emu', bind)
    sq = np.ascontiguousarray(band_poly(0, 0, 10, 10))
    assert lib.emu_inside(5.0, 5.0, sq.ctypes.data) and R.inside(5.0, 5.0, sq)
    for x, y in ((math.nan, 5.0), (5.0, math.nan), (math.nan, math.nan)):
        assert not lib.emu_inside(x, y, sq.ctypes.data) and not R.inside(x, y, sq)
    nan_sq = sq.copy()
    nan_sq[4] = math.nan
    assert lib.emu_inside(5.0, 5.0, nan_sq.ctypes.data) == R.inside(5.0, 5.0, nan_sq)
    tm = tile_rows([[(np.array([math.nan, 530.0]), band_poly(1000, 500, 1100, 560)),
                     (np.array([1000.0, math.nan]), np.full(32, math.nan)),
                     (np.array([1000.0, 530.0]), band_poly(1000, 500, 1100, 560))]], 1)
    whole = whole_readings([[whole_word(944, 500, 1200, 560)]], 1)
    got = both([A4], None, 1200, 256, 4.0, NB, tm, *whole)
    assert got['source'][:, 0].tolist() == [0, 1, -1]


def test_empty_pages_and_readings():
    sizes = [A4, (2000, 2000), A4]
    tm = tile_rows([[], [(np.array([1000.0, 1000.0]), band_poly(995, 997, 1005, 1003))], []], 3)
    whole = whole_readings([[], [], [whole_word(944, 500, 1200, 560)]], 3)
    got = both(sizes, None, 1200, 256, 4.0, NB, tm, *whole)
    assert got['count'].tolist() == [0, 1, 1] and got['offset'].tolist() == [0, 0, 1]
    got = both(sizes, None, 1200, 256, 4.0, NB, tile_rows([[], [], []], 3), *whole_readings([[], [], []], 3))
    assert got['count'].tolist() == [0, 0, 0] and got['pts'].shape == (0, 2)


# ---- properties ------------------------------------------------------------------------------------------------


@pytest.mark.parametrize('seed', range(4))
def test_narrow_whole_rows_are_never_kept(seed):
    """Property (a): a whole row whose box is narrower than ov - 2m and shorter than ov - 2m is kept by no plan."""
    rng = np.random.default_rng(100 + seed)
    m = 4.0
    for _ in range(300):
        T = int(rng.integers(64, 1500))
        ov = int(rng.integers(2 * m + 2, T // 2 + 1))
        H, W = int(rng.integers(1, 6 * T)), int(rng.integers(1, 6 * T))
        k = int(rng.integers(0, 4))
        th, tw = R.turned(H, W, k)
        lim = ov - 2 * m
        w, h = rng.uniform(0, lim), rng.uniform(0, lim)
        x, y = rng.uniform(-5, tw + 5), rng.uniform(-5, th + 5)
        xs = np.concatenate([np.linspace(x, x + w, 8), np.linspace(x + w, x, 8)])
        ys = np.concatenate([np.full(8, y), np.full(8, y + h)])
        xs, ys = [float(np.float32(v)) for v in xs], [float(np.float32(v)) for v in ys]
        if max(xs) - min(xs) >= lim or max(ys) - min(ys) >= lim:
            continue
        assert not R.cut_by_every_tile(xs, ys, th, tw, T, ov, m)
    # and through the emulation, on binned rows
    sizes, turns, T, ov, tiles, whole = fabricate(rng, 3, 200)
    if ov > 2 * m:
        got = emu_merge(sizes, turns, T, ov, m, NB, tiles, *whole)
        for p, rows in enumerate(R.whole_rows(sizes, turns, T, ov, m, *whole[:3], NB)):
            for i, _, polys, kept in rows:
                xs, ys = polys[0::2], polys[1::2]
                if max(xs) - min(xs) < ov - 2 * m and max(ys) - min(ys) < ov - 2 * m:
                    assert not kept
                    mine = got['source'][got['offset'][p]:got['offset'][p] + got['count'][p]]
                    assert (-1, i) not in [tuple(s) for s in mine]


@pytest.mark.parametrize('seed', range(3))
def test_the_result_does_not_depend_on_row_order(seed):
    """Property (c): shuffling the tile rows and the whole rows of every page permutes the output the same way."""
    rng = np.random.default_rng(200 + seed)
    sizes, turns, T, ov, tiles, whole = fabricate(rng, 3, 200)
    got = emu_merge(sizes, turns, T, ov, 4.0, NB, tiles, *whole)
    P = len(sizes)
    perm_t = np.concatenate([o + rng.permutation(c) for o, c in zip(tiles['offset'], tiles['count'])]).astype(int)
    t2 = {k: (v if k in ('count', 'offset') else v[perm_t]) for k, v in tiles.items()}
    n_inst, pt, poly, rec, prob = whole
    perm_w = [rng.permutation(int(n)) for n in n_inst]
    w2 = [n_inst] + [a.copy() for a in (pt, poly, rec, prob)]
    for p in range(P):
        for a, b in zip(w2[1:], (pt, poly, rec, prob)):
            a[p, :n_inst[p]] = b[p, perm_w[p]]
    got2 = emu_merge(sizes, turns, T, ov, 4.0, NB, t2, *w2)
    assert got2['count'].tolist() == got['count'].tolist()
    for p in range(P):
        def rowset(res, wperm):
            rows = set()
            for r in range(int(res['offset'][p]), int(res['offset'][p]) + int(res['count'][p])):
                s = tuple(res['source'][r])
                key = ('w', int(wperm[s[1]])) if s[0] < 0 else ('t', s)
                rows.add((key, res['pts'][r].tobytes(), res['polys'][r].tobytes(), res['rec'][r].tobytes()))
            return rows
        assert rowset(got, np.arange(int(n_inst[p]))) == rowset(got2, perm_w[p])
