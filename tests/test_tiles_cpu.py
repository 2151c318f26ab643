"""Pages spotted in overlapping tiles: CPU checks of the tile layout (its properties, the library's host entry point)
and of the merge kernels' bodies run on the host (tests/emu/tile_emu.cpp) against oracle/tile_ref.py, bit for bit, on
random fabricated tile outputs, on hand-made seam cases, on the reference's coordinates (tests/golden/post_omni.json)
and on tests/golden/omni_tiles.npz (the reference run on every tile of a page by oracle/gen_golden_tiles.py)."""
import ctypes as C
import json
import os

import numpy as np
import pytest

from tests.support import emu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


def bind(lib):
    """Bind tests/emu/tile_emu.cpp (host compile of the merge kernels' bodies)."""
    lib.emu_tile_axis.restype = C.c_int
    lib.emu_tile_axis.argtypes = [C.c_int] * 3 + [C.c_void_p, C.c_int]
    lib.emu_merge_tiles.restype = C.c_long
    lib.emu_merge_tiles.argtypes = ([C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int] + [C.c_void_p] * 5 +
                                    [C.c_int] * 3 + [C.c_double] * 3 + [C.c_void_p] * 7)


def emu_merge(sizes, T, ov, n_inst, pt, poly, rec, prob, num_bins, margin=4.0, band=None, iou=0.5):
    """alm_omni_merge_tiles' three launches on the host -> the dict merge_tiles / tile_ref.merge return."""
    lib = emu('tile_emu', bind)
    band = ov / 4 if band is None else band
    hs = np.ascontiguousarray([s[0] for s in sizes], np.int32)
    ws = np.ascontiguousarray([s[1] for s in sizes], np.int32)
    n_inst = np.ascontiguousarray(n_inst, np.int32)
    pt, poly, rec = (np.ascontiguousarray(a, np.int64) for a in (pt, poly, rec))
    prob = np.ascontiguousarray(prob, np.float32)
    maxi, L = pt.shape[1], rec.shape[2]
    K = max(int(n_inst.sum()), 1)
    out = dict(count=np.zeros(len(sizes), np.int32), offset=np.zeros(len(sizes), np.int32), pts=np.zeros((K, 2)),
               polys=np.zeros((K, 32)), rec=np.zeros((K, L), np.int64), prob=np.zeros((K, L), np.float32),
               source=np.zeros((K, 2), np.int32))
    n = lib.emu_merge_tiles(hs.ctypes.data, ws.ctypes.data, len(sizes), T, ov, n_inst.ctypes.data, pt.ctypes.data,
                            poly.ctypes.data, rec.ctypes.data, prob.ctypes.data, maxi, L, num_bins, margin, band, iou,
                            *[out[k].ctypes.data for k in ('count', 'offset', 'pts', 'polys', 'rec', 'prob', 'source')])
    for k in ('pts', 'polys', 'rec', 'prob', 'source'):
        out[k] = out[k][:n]
    return out


def assert_same(a, b):
    """Two merge results are equal, floats bit for bit."""
    assert a.keys() == b.keys()
    for k in a:
        x, y = np.asarray(a[k]), np.asarray(b[k])
        assert x.shape == y.shape and x.dtype == y.dtype, k
        if x.dtype.kind == 'f':
            x, y = x.view(np.uint64 if x.itemsize == 8 else np.uint32), y.view(np.uint64 if y.itemsize == 8 else np.uint32)
        assert np.array_equal(x, y), k


def random_layouts(rng, n):
    T = rng.integers(64, 2000, n)
    ov = (rng.uniform(0, 1, n) * (T // 2 + 1)).astype(np.int64)
    ov[:3] = [0, T[1] // 2, T[2] // 2]
    L = np.maximum(1, T[:, None] * rng.choice([0.3, 1, 1.0001, 1.5, 2, 3.7, 9, 40], (n, 2)) * rng.uniform(0.9, 1.1, (n, 2)))
    L[3:6] = T[3:6, None]      # exactly one tile
    L[6:9] = T[6:9, None] + 1  # two tiles, the second clamped
    return np.concatenate([L.astype(np.int64), T[:, None], ov[:, None]], 1)


def test_layout_properties():
    """Per axis: tiles start at 0, end at L and cover it, stride <= T - ov (overlap >= ov), one tile iff L <= T, all of
    size min(T, L); the seams increase and sit inside their overlap, so the cores partition the page; the library's
    entry point and the emulation equal the oracle."""
    from advancedliteratemachinery_b200 import preprocess as P
    from oracle import tile_ref as R
    lib = emu('tile_emu', bind)
    buf = np.zeros(1 << 16, np.int32)
    for H, W, T, ov in random_layouts(np.random.default_rng(0), 5000).tolist():
        for L in (H, W):
            x0 = R.axis(L, T, ov)
            tw = min(T, L)
            assert x0[0] == 0 and x0[-1] + tw == L and (len(x0) == 1) == (L <= T)
            assert all(0 < b - a <= T - ov for a, b in zip(x0, x0[1:]))
            s = R.seams(x0, tw)
            assert all(a < b for a, b in zip(s, s[1:]))
            assert all(x0[i + 1] <= s[i] <= x0[i] + tw for i in range(len(s)))
            n = lib.emu_tile_axis(L, T, ov, buf.ctypes.data, len(buf))
            assert buf[:n].tolist() == x0
        plan = P.omni_tile_plan([(H, W)], T, ov)
        assert plan.tolist() == [list(r) for r in R.plan([(H, W)], T, ov)]


def test_tile_plan_entry_point():
    """Several pages in order, row-major within a page; bad layouts and sides are refused."""
    from advancedliteratemachinery_b200 import _lib, preprocess as P
    plan = P.omni_tile_plan([(3508, 2480), (100, 100)], 1200, 256)
    assert len(plan) == 13 and (plan[:12, 0] == 0).all() and plan[12].tolist() == [1, 0, 0, 100, 100]
    assert plan[:12, 1].tolist() == [0] * 3 + [944] * 3 + [1888] * 3 + [2308] * 3
    assert plan[:3, 2].tolist() == [0, 944, 1280] and (plan[:12, 3:] == 1200).all()
    assert P.omni_tile_plan([], 1200, 256).shape == (0, 5)
    for bad in (dict(tile=63, overlap=0), dict(tile=100, overlap=51), dict(tile=100, overlap=-1)):
        with pytest.raises(_lib.AlmError):
            P.omni_tile_plan([(500, 500)], **bad)
    for size in ((0, 5), (5, 0)):
        with pytest.raises(_lib.AlmError):
            P.omni_tile_plan([size], 100, 10)


def fabricate(rng, sizes, T, ov, max_inst, L, num_bins, n_words):
    """Tile outputs of pages holding random words: every tile that sees a word reads it, its polygon and point binned
    in the tile's frame with a bin or two of noise (so readings of one word differ between tiles), plus junk."""
    from oracle import tile_ref as R
    plan = R.plan(sizes, T, ov)
    nt = len(plan)
    n_inst = np.zeros(nt, np.int32)
    pt = np.zeros((nt, max_inst, 2), np.int64)
    poly = np.zeros((nt, max_inst, 32), np.int64)
    rec = rng.integers(0, 100, (nt, max_inst, L)).astype(np.int64)
    prob = rng.uniform(0, 1, (nt, max_inst, L)).astype(np.float32)
    words = []
    for p, (H, W) in enumerate(sizes):
        for _ in range(n_words):
            w, h = rng.uniform(5, 0.4 * min(T, W)), rng.uniform(3, 0.2 * min(T, H))
            x, y = rng.uniform(0, W - w), rng.uniform(0, H - h)
            words.append((p, x, y, w, h))
    for k, (p, y0, x0, th, tw) in enumerate(plan):
        for wp, x, y, w, h in words:
            if wp != p or n_inst[k] == max_inst or x + w <= x0 or x >= x0 + tw or y + h <= y0 or y >= y0 + th:
                continue
            if rng.random() < 0.1:
                continue  # a tile that misses a word now and then
            xs = np.clip(np.concatenate([np.linspace(x, x + w, 8), np.linspace(x + w, x, 8)]), x0, x0 + tw - 1e-9)
            ys = np.clip(np.concatenate([np.full(8, y), np.full(8, y + h)]), y0, y0 + th - 1e-9)
            bx = np.floor((xs - x0) / tw * num_bins) + rng.integers(-1, 2, 16)
            by = np.floor((ys - y0) / th * num_bins) + rng.integers(-1, 2, 16)
            i = n_inst[k]
            poly[k, i, 0::2] = np.clip(bx, 0, num_bins - 1)
            poly[k, i, 1::2] = np.clip(by, 0, num_bins - 1)
            px, py = np.clip(x + w / 2 + rng.uniform(-2, 2), x0, x0 + tw - 1e-9), np.clip(y + h / 2, y0, y0 + th - 1e-9)
            pt[k, i] = [np.floor((px - x0) / tw * num_bins), np.floor((py - y0) / th * num_bins)]
            n_inst[k] += 1
        junk = min(int(rng.integers(0, 3)), max_inst - n_inst[k])
        for i in range(n_inst[k], n_inst[k] + junk):
            pt[k, i] = rng.integers(0, num_bins, 2)
            poly[k, i] = rng.integers(0, num_bins, 32)
        n_inst[k] += junk
    return n_inst, pt, poly, rec, prob


def merge_both(sizes, T, ov, outs, num_bins, **kw):
    from oracle import tile_ref as R
    got = emu_merge(sizes, T, ov, *outs, num_bins, **kw)
    assert_same(got, R.merge(sizes, T, ov, *outs, num_bins, **kw))
    return got


@pytest.mark.parametrize('seed', range(6))
def test_merge_on_the_host_equals_oracle(seed):
    """Random pages, layouts, parameters and fabricated tile outputs: the emulated kernels equal the oracle bit for bit,
    and the cases reach every branch (cuts, candidates outside the core, suppression across seams)."""
    from oracle import tile_ref as R
    rng = np.random.default_rng(100 + seed)
    T = int(rng.choice([64, 128, 200, 1200]))
    ov = int(rng.integers(0, T // 2 + 1))
    sizes = [(int(rng.integers(1, 4 * T)), int(rng.integers(1, 4 * T))) for _ in range(int(rng.integers(1, 5)))]
    sizes[0] = (3 * T, 2 * T + 7)
    num_bins = int(rng.choice([1000, 97]))
    outs = fabricate(rng, sizes, T, ov, 24, 5, num_bins, 30)
    kw = dict(margin=float(rng.choice([0.0, 4.0, 2.5])), band=None if seed % 2 else float(rng.uniform(0, ov / 2 + 1)),
              iou=float(rng.choice([0.5, 0.3, 1.0])))
    got = merge_both(sizes, T, ov, outs, num_bins, **kw)
    assert int(got['count'].sum()) < int(outs[0].sum())
    tiles = R.tile_grid(sizes, T, ov, ov / 4 if kw['band'] is None else kw['band'])
    flags = [R.instance(tiles[k], outs[1][k, i], outs[2][k, i], num_bins, kw['margin'])
             for k in range(len(tiles)) for i in range(int(outs[0][k]))]
    assert any(f['cand'] for f in flags) and not all(f['cand'] for f in flags)


# hand-made cases: T = 100, num_bins = 100, so a bin is a page pixel in the tile's frame
NB = 100


def page_instance(x0, y0, box, point):
    """ids of a word with page box (x_0, y_0, x_1, y_1) and point (x, y), read by the tile at (x0, y0)."""
    a, b, c, d = box
    xs = np.concatenate([np.linspace(a, c, 8), np.linspace(c, a, 8)]) - x0
    ys = np.concatenate([np.full(8, b), np.full(8, d)]) - y0
    poly = np.zeros(32, np.int64)
    poly[0::2], poly[1::2] = np.round(xs), np.round(ys)
    return np.array([point[0] - x0, point[1] - y0], np.int64), poly


def outputs(plan, readings, L=3):
    """readings: [(tile, page box, point)] -> per-tile outputs in the decode layout."""
    nt = len(plan)
    per = [[r for r in readings if r[0] == k] for k in range(nt)]
    maxi = max(1, max(len(p) for p in per))
    n_inst = np.array([len(p) for p in per], np.int32)
    pt, poly = np.zeros((nt, maxi, 2), np.int64), np.zeros((nt, maxi, 32), np.int64)
    rec = np.zeros((nt, maxi, L), np.int64)
    prob = np.zeros((nt, maxi, L), np.float32)
    for k, p in enumerate(per):
        for i, (_, box, point) in enumerate(p):
            pt[k, i], poly[k, i] = page_instance(plan[k][2], plan[k][1], box, point)
            rec[k, i] = 10 * k + i
            prob[k, i] = 0.5
    return n_inst, pt, poly, rec, prob


def kept(res):
    return [tuple(s) for s in res['source'].tolist()]


def test_seam_cases():
    """A 100 x 160 page, T 100, ov 40: tiles at x 0 and 60, seam 80, band 10, interior edges x = 100 (tile 0) and
    x = 60 (tile 1).  Host bodies and oracle agree on each case."""
    from oracle import tile_ref as R
    sizes, T, ov = [(100, 160)], 100, 40
    plan = R.plan(sizes, T, ov)
    assert [p[2] for p in plan] == [0, 60] and R.seams([0, 60], 100) == [80.0]
    run = lambda readings, **kw: merge_both(sizes, T, ov, outputs(plan, readings), NB, **kw)
    # a word on the seam read by both tiles: kept once, from the tile whose interior edge is farther (tile 1: 12 px)
    assert kept(run([(0, (72, 40, 90, 50), (81, 45)), (1, (72, 40, 90, 50), (81, 45))])) == [(1, 0)]
    # equal distance to both interior edges (10 px): the lower tile wins
    assert kept(run([(0, (70, 40, 90, 50), (80, 45)), (1, (70, 40, 90, 50), (80, 45))])) == [(0, 0)]
    # each reading's point in the other tile's core: kept once through the band, lost without it
    two = [(0, (70, 40, 92, 50), (83, 45)), (1, (71, 40, 92, 50), (77, 45))]
    assert kept(run(two)) == [(1, 0)]
    assert kept(run(two, band=0.0)) == []
    # a word cut by tile 0's interior edge: dropped there, kept from tile 1
    assert kept(run([(0, (90, 40, 99, 50), (95, 45)), (1, (90, 40, 115, 50), (102, 45))])) == [(1, 0)]
    # cut means within the margin: 4 px from the edge is cut, 5 px is not
    assert kept(run([(0, (30, 40, 96, 50), (50, 45))])) == []
    assert kept(run([(0, (30, 40, 95, 50), (50, 45))])) == [(0, 0)]
    # page-border edges never cut; same-tile overlaps are both kept
    border = [(0, (0, 0, 30, 99), (10, 50)), (0, (0, 0, 30, 99), (12, 50)), (1, (130, 40, 159, 50), (150, 45))]
    assert kept(run(border)) == [(0, 0), (0, 1), (1, 0)]
    # an IoU below theta keeps both readings; theta 1 needs identical boxes
    near = [(0, (60, 40, 80, 50), (70, 45)), (1, (70, 40, 90, 50), (85, 45))]
    assert kept(run(near)) == [(0, 0), (1, 0)]
    res = run([(0, (70, 40, 90, 50), (80, 45)), (1, (70, 40, 90, 51), (80, 45))], iou=1.0)
    assert kept(res) == [(0, 0), (1, 0)]
    # page coordinates: tile origin + the tile-frame coordinate
    res = run([(1, (130, 40, 159, 50), (150, 45))])
    assert res['pts'].tolist() == [[150.0, 45.0]] and res['polys'][0, 0] == 130.0 and res['rec'][0].tolist() == [10] * 3


def test_four_tile_corner_and_empty_pages():
    """A word at the corner of four tiles is kept once, from the tile where it is farthest from interior edges; pages
    and tiles without instances give count 0 and do not shift the other pages' offsets."""
    from oracle import tile_ref as R
    sizes, T, ov = [(50, 50), (160, 160), (300, 90)], 100, 40
    plan = R.plan(sizes, T, ov)
    assert len(plan) == 1 + 4 + 5
    box = (74, 72, 88, 86)   # d of the four tiles at (x0, y0) = (0, 0), (60, 0), (0, 60), (60, 60): 12, 14, 12, 12
    readings = [(k, box, (80, 80)) for k in range(1, 5)]
    res = merge_both(sizes, T, ov, outputs(plan, readings), NB)
    assert kept(res) == [(2, 0)] and res['count'].tolist() == [0, 1, 0] and res['offset'].tolist() == [0, 0, 1]
    res = merge_both(sizes, T, ov, outputs(plan, []), NB)
    assert res['count'].tolist() == [0, 0, 0] and res['pts'].shape == (0, 2)


def test_single_tile_page_reproduces_decode_pred_seq():
    """A page no larger than one tile keeps every instance at decode_pred_seq's coordinates: the reference's own values
    in tests/golden/post_omni.json, bit for bit (the float32 arithmetic both share)."""
    from oracle import tile_ref as R
    for c in json.load(open(os.path.join(GOLD, 'post_omni.json'))):
        h, w = c['orig']
        pt = np.asarray(c['pt'], np.int64).reshape(1, -1, 2)
        n = pt.shape[1]
        if n == 0:
            continue
        poly = np.asarray(c['poly'], np.int64).reshape(1, n, 32)
        L = int(c['rec_length'])
        outs = (np.array([n], np.int32), pt, poly, np.zeros((1, n, L), np.int64), np.zeros((1, n, L), np.float32))
        T = max(64, h, w)
        got = merge_both([(h, w)], T, T // 4, outs, 1000)
        assert kept(got) == [(0, i) for i in range(n)]
        assert got['pts'].tolist() == [r['pts'][0] for r in c['results']]
        assert got['polys'].tolist() == [sum(r['polys'], []) for r in c['results']]
        assert [R.coord(i, 1000, w) for i in pt[0, :, 0]] == [r['pts'][0][0] for r in c['results']]


def test_fixture_merge():
    """tests/golden/omni_tiles.npz: the reference's decode_pred_seq of every tile (with the tile's own orig_size) is the
    tile-frame coordinate the merge uses, and the emulated merge of the reference's tile outputs equals the fixture's
    merge (written by the oracle)."""
    from oracle import tile_ref as R
    z = np.load(os.path.join(GOLD, 'omni_tiles.npz'))
    sizes, T, ov = [tuple(z['page'].shape[:2])], int(z['tile']), int(z['overlap'])
    outs = (z['n_inst'], z['pt'], z['poly'], z['rec'], z['prob'])
    got = merge_both(sizes, T, ov, outs, int(z['num_bins']))
    for k in ('count', 'offset', 'pts', 'polys', 'rec', 'prob', 'source'):
        assert np.array_equal(got[k], z[f'merged_{k}']), k
    plan = z['plan']
    for k in range(len(plan)):
        for i in range(int(z['n_inst'][k])):
            loc = z['ref_pts'][k, i]   # the reference's decode_pred_seq 'pts' of this tile, in the tile's frame
            assert [R.coord(z['pt'][k, i, 0], int(z['num_bins']), plan[k, 4]),
                    R.coord(z['pt'][k, i, 1], int(z['num_bins']), plan[k, 3])] == loc.tolist()
            assert [R.coord(v, int(z['num_bins']), plan[k, 4 - j % 2]) for j, v in enumerate(z['poly'][k, i])] == \
                z['ref_polys'][k, i].tolist()
    assert int(z['n_inst'].sum()) > int(got['count'].sum()) > 0
