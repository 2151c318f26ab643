"""KIE entities that cross tile seams, recovered from a whole-page KIE reading (DESIGN 4.22): CPU checks of the merge,
with the kernels' bodies run on the host (tests/emu/kie_whole_page_emu.cpp) against oracle/kie_whole_page_ref.py, bit
for bit: on fabricated decodes of many pages, layouts and turns, on hand-made seam cases, on the rule's properties and
on tests/golden/omni_kie_tiles.npz (the reference's tile decodes and its whole-page probes).  Also: the binding's
refusals."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle import kie_whole_page_ref as KW
from oracle import page_turn_ref as PT
from tests.support import assert_same, emu
from tests.test_kie_tiles_cpu import BASE, NB, NCLS, emu_merge, fabricate

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
ENT = ('cls', 'prob', 'word_offset', 'word_count', 'source')
WORD = ('rect', 'poly', 'word_source')
RAW = (('n_tok', np.int32), ('tokens', np.int64), ('probs', np.float32), ('n_inst', np.int32), ('inst_pos', np.int32),
       ('poly', np.int64))


def bind(lib):
    """Bind tests/emu/kie_whole_page_emu.cpp (host compile of the kernels' bodies)."""
    lib.emu_merge_kie_whole_page.restype = C.c_long
    lib.emu_merge_kie_whole_page.argtypes = ([C.c_void_p] * 3 + [C.c_int] * 3 + [C.c_double] + [C.c_int] * 3 +
                                             [C.c_void_p] * 13 + [C.c_int] + [C.c_void_p] * 3 + [C.c_int] +
                                             [C.c_void_p] * 11)


def emu_whole(sizes, T, ov, tiles, whole, margin=4.0, turns=None, num_bins=NB, class_base=BASE, n_classes=NCLS):
    """alm_omni_merge_kie_whole_page's launches on the host -> the dict merge_kie_whole_page returns (None: a walk
    failed).  tiles: merge_kie_tiles' dict; whole: the pages' whole readings (RAW keys, one row per page)."""
    lib = emu('kie_whole_page_emu', bind)
    hs = np.ascontiguousarray([s[0] for s in sizes], np.int32)
    ws = np.ascontiguousarray([s[1] for s in sizes], np.int32)
    ts = None if turns is None else np.ascontiguousarray(turns, np.int32)
    t = {k: np.ascontiguousarray(tiles[k], d) for k, d in (
        ('count', np.int32), ('offset', np.int32), ('cls', np.int32), ('prob', np.float32), ('word_offset', np.int32),
        ('word_count', np.int32), ('source', np.int32), ('rect', np.float64), ('poly', np.float64),
        ('word_source', np.int32))}
    a = {k: np.ascontiguousarray(whole[k], d) for k, d in RAW}
    E = max(len(t['cls']) + int(a['n_tok'].sum()), 1)
    N = max(len(t['rect']) + int(a['n_inst'].sum()), 1)
    P = len(sizes)
    out = dict(count=np.zeros(P, np.int32), offset=np.zeros(P, np.int32), cls=np.zeros(E, np.int32),
               prob=np.zeros(E, np.float32), word_offset=np.zeros(E, np.int32), word_count=np.zeros(E, np.int32),
               source=np.zeros((E, 2), np.int32), rect=np.zeros((N, 4)), poly=np.zeros((N, 32)),
               word_source=np.zeros((N, 2), np.int32))
    nw = C.c_long()
    n = lib.emu_merge_kie_whole_page(
        hs.ctypes.data, ws.ctypes.data, None if ts is None else ts.ctypes.data, P, T, ov, margin, num_bins, class_base,
        n_classes, t['count'].ctypes.data, t['offset'].ctypes.data, *[t[k].ctypes.data for k in ENT + WORD],
        a['n_tok'].ctypes.data, a['tokens'].ctypes.data, a['probs'].ctypes.data, a['tokens'].shape[1],
        a['n_inst'].ctypes.data, a['inst_pos'].ctypes.data, a['poly'].ctypes.data, a['inst_pos'].shape[1],
        *[out[k].ctypes.data for k in ('count', 'offset') + ENT + WORD], C.byref(nw))
    if n < 0:
        return None
    for k in ENT:
        out[k] = out[k][:n]
    for k in WORD:
        out[k] = out[k][:nw.value]
    return out


def check(sizes, T, ov, tiles, whole, turns=None, margin=4.0, **kw):
    """The host bodies equal the oracle bit for bit; returns the merge."""
    got = emu_whole(sizes, T, ov, tiles, whole, margin, turns, **kw)
    nb, base, ncls = kw.get('num_bins', NB), kw.get('class_base', BASE), kw.get('n_classes', NCLS)
    ref = KW.merge(sizes, turns, T, ov, margin, nb, base, ncls, tiles, whole)
    assert_same(got, ref)
    return got


def reading(frames, num_bins=NB, rng=None):
    """Decodes of images, one per frame (h, w, [entities]); an entity is (class, [boxes (x0, y0, x1, y1) in the
    image's pixels]).  Each word's polygon spans its box (8 points on top, 8 on the bottom), binned in the image."""
    n = len(frames)
    max_inst = 1 + max(sum(len(bx) for _, bx in f[2]) for f in frames)
    max_tok = 1 + max(sum(2 * len(bx) + 1 for _, bx in f[2]) for f in frames)
    raw = dict(n_tok=np.zeros(n, np.int32), tokens=np.zeros((n, max_tok), np.int64),
               probs=np.full((n, max_tok), 0.5, np.float32), n_inst=np.zeros(n, np.int32),
               inst_pos=np.zeros((n, max_inst), np.int32), poly=np.zeros((n, max_inst, 32), np.int64))
    if rng is not None:
        raw['probs'] = rng.uniform(0, 1, (n, max_tok)).astype(np.float32)
    for k, (h, w, ents) in enumerate(frames):
        for cls, boxes in ents:
            for a, b, c, d in boxes:
                i, t = raw['n_inst'][k], raw['n_tok'][k]
                xs = np.concatenate([np.linspace(a, c, 8), np.linspace(c, a, 8)])
                ys = np.concatenate([np.full(8, b), np.full(8, d)])
                raw['poly'][k, i, 0::2] = np.clip(np.round(xs / w * num_bins), 0, num_bins - 1)
                raw['poly'][k, i, 1::2] = np.clip(np.round(ys / h * num_bins), 0, num_bins - 1)
                raw['inst_pos'][k, i] = t
                raw['tokens'][k, t:t + 2] = raw['poly'][k, i, :2]
                raw['n_inst'][k] += 1
                raw['n_tok'][k] += 2
            raw['tokens'][k, raw['n_tok'][k]] = BASE + cls
            raw['n_tok'][k] += 1
    return raw


def clip(boxes, y0, x0, h, w):
    """The parts of page boxes a tile at (y0, x0) of h x w sees, in its pixels."""
    out = []
    for a, b, c, d in boxes:
        a, b, c, d = max(a - x0, 0), max(b - y0, 0), min(c - x0, w - 0.5), min(d - y0, h - 0.5)
        if a < c and b < d:
            out.append((a, b, c, d))
    return out


def read_page(sizes, T, ov, ents, turns=None):
    """Every tile of the pages' plan and every page read whole, of entities given per page as (class, [page boxes of
    the turned page]): a tile reads the part of an entity it sees -> (tile merge, whole readings)."""
    turns = [0] * len(sizes) if turns is None else turns
    plan = PT.plan(sizes, turns, T, ov)
    tiles = reading([(h, w, [(c, clip(bx, y0, x0, h, w)) for c, bx in ents[p] if clip(bx, y0, x0, h, w) or not bx])
                     for p, y0, x0, h, w in np.asarray(plan).tolist()])
    whole = reading([PT.turned_size(H, W, k) + ([(c, bx) for c, bx in ents[p]],)
                     for p, ((H, W), k) in enumerate(zip(sizes, turns))])
    return emu_merge(sizes, T, ov, tiles, turns=turns), whole


def sources(m, p=0):
    rows = range(int(m['offset'][p]), int(m['offset'][p]) + int(m['count'][p]))
    return [tuple(m['source'][r]) for r in rows]


def test_receipt_entity_across_a_horizontal_seam():
    """A three-line entity over the seam of a 160 x 100 page (tiles at y 0 and 60): each tile keeps a two-line
    fragment (no IoU between them), so without the whole reading the middle line is read twice and the entity is never
    read whole.  The whole reading is cut by both tiles and kept; both fragments' anchors lie in its box, one of them
    in the gap between two of its words, and both are dropped."""
    sizes = [(160, 100)]
    lines = [(10, 30, 60, 45), (10, 70, 60, 85), (10, 115, 60, 130)]
    tiles, whole = read_page(sizes, 100, 40, [[(1, lines)]])
    assert sources(tiles) == [(0, 0), (1, 0)] and tiles['word_count'].tolist() == [2, 2]
    ay = (tiles['rect'][2:4, 1].min() + tiles['rect'][2:4, 3].max()) / 2   # tile 1's fragment, in page pixels
    assert 85 < ay < 115   # between the second and the third line
    got = check(sizes, 100, 40, tiles, whole)
    assert sources(got) == [(-1, 0)] and got['word_count'].tolist() == [3]
    assert got['word_source'].tolist() == [[-1, 0], [-1, 1], [-1, 2]]
    # one line taller than the overlap, which no tile reads whole: lost without the option, recovered with it
    tiles, whole = read_page(sizes, 100, 40, [[(2, [(10, 50, 60, 110)])]])
    assert sources(tiles) == []
    assert sources(check(sizes, 100, 40, tiles, whole)) == [(-1, 0)]


def test_entity_one_tile_holds_keeps_the_tile_reading():
    sizes = [(160, 100)]
    tiles, whole = read_page(sizes, 100, 40, [[(0, [(10, 10, 60, 40)]), (3, [(10, 120, 60, 150)])]])
    got = check(sizes, 100, 40, tiles, whole)
    assert sources(got) == sources(tiles) == [(0, 0), (1, 0)]


def test_four_tile_corner_and_clamped_tile():
    # 160 x 160: tiles at (0, 0), (0, 60), (60, 0), (60, 60); a box over both seams is cut by all four
    tiles, whole = read_page([(160, 160)], 100, 40, [[(1, [(30, 30, 130, 130)])]])
    assert sources(check([(160, 160)], 100, 40, tiles, whole)) == [(-1, 0)]
    # 130 x 100: the last tile is clamped to y 30; a box over y 20 .. 120 is cut by both, one over 35 .. 95 is not cut
    # by tile 0 (5 px from its bottom edge)
    tiles, whole = read_page([(130, 100)], 100, 40, [[(1, [(10, 20, 60, 120)]), (2, [(70, 35, 90, 95)])]])
    got = check([(130, 100)], 100, 40, tiles, whole)
    assert [s for s in sources(got) if s[0] < 0] == [(-1, 0)]


def test_single_tile_pages_keep_nothing_whole():
    """Property (b): a page that fits in one tile keeps its tile entities, wordless ones included, and nothing whole."""
    sizes = [(90, 80), (100, 100)]
    ents = [[(1, [(5, 5, 85, 75)]), (2, [])], [(0, [(0, 0, 99, 99)])]]
    tiles, whole = read_page(sizes, 100, 40, ents)
    got = check(sizes, 100, 40, tiles, whole)
    assert_same(got, tiles)


def test_nan_wordless_and_empty_readings():
    sizes = [(160, 100)]
    lines = [(10, 30, 60, 45), (10, 70, 60, 85), (10, 115, 60, 130)]
    tiles, whole = read_page(sizes, 100, 40, [[(1, lines)]])
    # a NaN in a fragment's rect: its anchor is NaN, never inside, so the fragment stays
    bad = {k: v.copy() for k, v in tiles.items()}
    bad['rect'][0, 1] = np.nan
    got = check(sizes, 100, 40, bad, whole)
    assert sources(got) == [(0, 0), (-1, 0)]
    bad['rect'][0, 1] = np.inf
    assert sources(check(sizes, 100, 40, bad, whole)) == [(0, 0), (-1, 0)]
    # a wordless whole entity is never kept; an empty reading keeps nothing
    wl = reading([(160, 100, [(1, []), (2, [])])])
    assert sources(check(sizes, 100, 40, tiles, wl)) == sources(tiles)
    empty = reading([(160, 100, [])])
    assert_same(check(sizes, 100, 40, tiles, empty), tiles)


def fabricate_whole(rng, sizes, T, ov, turns, n_ent=12, max_words=8):
    """Whole readings of the pages: entities of 1..max_words words laid out as lines, many taller or wider than the
    overlap, some wordless, in the turned frame."""
    frames = []
    for (H, W), k in zip(sizes, turns):
        h, w = PT.turned_size(H, W, k)
        ents = []
        for _ in range(n_ent):
            nw = int(rng.choice([0, 1, 2, 3, max_words]))
            big = rng.random() < 0.5
            ew, eh = rng.uniform(4, (1.5 if big else 0.3) * min(T, w)), rng.uniform(3, (1.5 if big else 0.2) * min(T, h))
            x, y = rng.uniform(0, max(w - ew, 1)), rng.uniform(0, max(h - eh, 1))
            boxes = []
            for j in range(nw):   # words on up to three lines
                line, col = j % 3, j // 3
                lh = eh / 3
                boxes.append((min(x + col * ew / 3, w - 2), min(y + line * lh, h - 2),
                              min(x + (col + 0.8) * ew / 3, w - 1), min(y + (line + 0.7) * lh, h - 1)))
            ents.append((int(rng.integers(0, NCLS)), boxes))
        frames.append((h, w, ents))
    return reading(frames, rng=rng)


@pytest.mark.parametrize('seed', range(8))
def test_merge_on_the_host_equals_oracle(seed):
    """Random pages, layouts, turns 0..3, margins and fabricated tile and whole decodes (1..8 words per entity,
    wordless entities, empty readings): the emulated kernels equal the oracle, and both decisions are frequent."""
    rng = np.random.default_rng(700 + seed)
    T = int(rng.choice([64, 128, 200]))
    ov = int(rng.integers(4, T // 2 + 1))
    sizes = [(int(rng.integers(T + 1, 4 * T)), int(rng.integers(T + 1, 4 * T))) for _ in range(int(rng.integers(2, 5)))]
    sizes.append((T // 2, T - 1))   # a page that is one tile
    turns = None if seed % 2 == 0 else rng.integers(0, 4, len(sizes)).tolist()
    tr = [0] * len(sizes) if turns is None else turns
    raw = fabricate(rng, sizes, T, ov, turns, n_ent=30, max_tok=512, max_inst=200)
    tiles = emu_merge(sizes, T, ov, raw, turns=turns)
    whole = fabricate_whole(rng, sizes, T, ov, tr, n_ent=40 if seed < 4 else 120)
    margin = float(rng.choice([0.0, 4.0, 2.5]))
    got = check(sizes, T, ov, tiles, whole, turns, margin)
    kept_whole = int((got['source'][:, 0] < 0).sum())
    kept_tile = int((got['source'][:, 0] >= 0).sum())
    assert kept_whole > 0 and 0 < kept_tile < len(tiles['cls'])


def test_properties():
    """(a) a whole entity smaller than ov - 2m on both axes is never kept; (b) see test_single_tile_pages_keep_nothing
    _whole; (c) reversing the order of the whole entities and of the tile entities keeps the same entities."""
    rng = np.random.default_rng(5)
    T, ov, m = 128, 48, 4.0
    sizes = [(500, 400), (400, 500)]
    ents = []
    for (H, W) in sizes:
        page = []
        for _ in range(200):
            w, h = rng.uniform(1, ov - 2 * m - 2), rng.uniform(1, ov - 2 * m - 2)
            x, y = rng.uniform(0, W - w - 1), rng.uniform(0, H - h - 1)
            page.append((int(rng.integers(0, NCLS)), [(x, y, x + w, y + h)]))
        ents.append(page)
    tiles, whole = read_page(sizes, T, ov, ents)
    got = check(sizes, T, ov, tiles, whole, margin=m)
    assert (got['source'][:, 0] >= 0).all()
    # (c): rows reversed
    raw = fabricate(rng, sizes, T, ov, None, n_ent=30, max_tok=512, max_inst=200)
    tiles = emu_merge(sizes, T, ov, raw)
    whole = fabricate_whole(rng, sizes, T, ov, [0, 0], n_ent=60)
    a = check(sizes, T, ov, tiles, whole)

    def reverse_tiles(t):
        out = {k: [] for k in t}
        out['count'] = t['count'].copy()
        for p in range(len(sizes)):
            for r in reversed(range(int(t['offset'][p]), int(t['offset'][p]) + int(t['count'][p]))):
                ws = slice(int(t['word_offset'][r]), int(t['word_offset'][r]) + int(t['word_count'][r]))
                for k in ('cls', 'prob', 'word_count', 'source'):
                    out[k].append(t[k][r])
                for k in WORD:
                    out[k].extend(t[k][ws])
        wc = np.array(out['word_count'], np.int32)
        res = {k: np.array(v) for k, v in out.items()}
        res.update(offset=t['offset'], word_count=wc, word_offset=(np.cumsum(wc) - wc).astype(np.int32))
        return res

    whole_ents = []
    for p, (H, W) in enumerate(sizes):
        nt, ni = int(whole['n_tok'][p]), int(whole['n_inst'][p])
        ws = KW.K.walk(whole['tokens'][p][:nt], whole['probs'][p][:nt], whole['inst_pos'][p][:ni], NB, BASE, NCLS)
        whole_ents.append([(c, [tuple(whole['poly'][p][i]) for i in w]) for c, _, w in ws][::-1])
    rw = dict(n_tok=np.zeros_like(whole['n_tok']), tokens=np.zeros_like(whole['tokens']), probs=whole['probs'],
              n_inst=np.zeros_like(whole['n_inst']), inst_pos=np.zeros_like(whole['inst_pos']),
              poly=np.zeros_like(whole['poly']))
    for p, es in enumerate(whole_ents):
        for c, polys in es:
            for pl in polys:
                i, t = rw['n_inst'][p], rw['n_tok'][p]
                rw['poly'][p, i] = pl
                rw['inst_pos'][p, i] = t
                rw['tokens'][p, t:t + 2] = pl[:2]
                rw['n_inst'][p] += 1
                rw['n_tok'][p] += 2
            rw['tokens'][p, rw['n_tok'][p]] = BASE + c
            rw['n_tok'][p] += 1
    b = check(sizes, T, ov, reverse_tiles(tiles), rw)

    def kept(m):
        return sorted((tuple(m['rect'][w].tolist()) for w in range(len(m['rect']))))
    assert kept(a) == kept(b) and a['count'].tolist() == b['count'].tolist()
    assert (a['source'][:, 0] < 0).any() and (a['source'][:, 0] >= 0).any()


def test_fixture_whole_readings():
    """tests/golden/omni_kie_tiles.npz: the reference's whole-page probes at turns 0..3 are the whole readings of the
    fixture page read at that turn.  Merged with the emulated tile merge of the reference's tile decodes (turn 0) the
    whole reading keeps entities that every tile cuts and drops the tile entities inside them."""
    g = np.load(os.path.join(GOLD, 'omni_kie_tiles.npz'))
    T, ov, base = int(g['tile']), int(g['overlap']), int(g['class_base'])
    sizes = [tuple(g['page'].shape[:2])]
    raw = {k: g[k] for k in ('n_tok', 'tokens', 'probs', 'n_inst', 'inst_pos', 'poly')}
    tiles = emu_merge(sizes, T, ov, raw, class_base=base)
    whole = {k: g['probe_' + k][0:1] for k in ('n_tok', 'tokens', 'probs', 'n_inst', 'inst_pos', 'poly')}
    got = check(sizes, T, ov, tiles, whole, class_base=base)
    assert (got['source'][:, 0] < 0).any() and int(got['count'][0]) < len(tiles['cls']) + 2
    assert len([s for s in got['source'].tolist() if s[0] >= 0]) < len(tiles['cls'])
    for k in (1, 2, 3):
        whole = {n: g['probe_' + n][k:k + 1] for n in ('n_tok', 'tokens', 'probs', 'n_inst', 'inst_pos', 'poly')}
        check(sizes, T, ov, emu_merge(sizes, T, ov, raw, class_base=base, turns=[0]), whole, class_base=base)


def test_binding_refusals():
    """merge_kie_whole_page refuses a bad margin, bad turns and arrays that do not match the pages before it reaches
    the library."""
    from advancedliteratemachinery_b200.omniparser import merge_kie_whole_page
    sizes = [(160, 100)]
    tiles, whole = read_page(sizes, 100, 40, [[(1, [(10, 30, 60, 130)])]])
    args = [whole[k] for k in ('n_tok', 'tokens', 'probs', 'n_inst', 'inst_pos', 'poly')]
    for bad in (dict(margin=-1.0), dict(margin=float('nan')), dict(turns=[4]), dict(turns=[0, 1])):
        with pytest.raises(ValueError):
            merge_kie_whole_page(None, sizes, 100, 40, tiles, *args, NB, BASE, NCLS, **bad)
    with pytest.raises(ValueError):   # one whole reading for two pages
        merge_kie_whole_page(None, sizes * 2, 100, 40, tiles, *args, NB, BASE, NCLS)
    short = dict(tiles, rect=tiles['rect'][:, :3])
    with pytest.raises(ValueError):
        merge_kie_whole_page(None, sizes, 100, 40, short, *args, NB, BASE, NCLS)
