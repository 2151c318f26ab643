"""KIE on tiled and turned pages (DESIGN 4.18): CPU checks of the entity merge, with the kernels' bodies run on the host
(tests/emu/kie_tile_emu.cpp) against oracle/kie_tile_ref.py, bit for bit: on fabricated tile decodes of many pages,
layouts and turns, on hand-made seam cases, and on tests/golden/omni_kie_tiles.npz (the reference run on every tile of
a page by oracle/gen_golden_kie_tiles.py).  Also: the shared entity walk still gives alm_post_omni_kie_json's output."""
import ctypes as C
import json
import os

import numpy as np
import pytest

from oracle import kie_tile_ref as K
from oracle import tile_ref as R
from oracle import page_turn_ref as PT
from tests.support import emu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
NB, BASE, NCLS = 1000, 1104, 4   # num_bins, class_base (padding_index + 1), SROIE classes


def bind(lib):
    """Bind tests/emu/kie_tile_emu.cpp (host compile of the kernels' bodies)."""
    lib.emu_merge_kie_tiles.restype = C.c_long
    lib.emu_merge_kie_tiles.argtypes = ([C.c_void_p] * 3 + [C.c_int] * 3 + [C.c_void_p] * 3 + [C.c_int] +
                                        [C.c_void_p] * 3 + [C.c_int] * 4 + [C.c_double] * 3 + [C.c_void_p] * 11)


def emu_merge(sizes, T, ov, raw, margin=4.0, band=None, iou=0.5, turns=None, num_bins=NB, class_base=BASE,
              n_classes=NCLS):
    """alm_omni_merge_kie_tiles' launches on the host -> the dict merge_kie_tiles returns (None: a walk failed)."""
    lib = emu('kie_tile_emu', bind)
    band = ov / 4 if band is None else band
    hs = np.ascontiguousarray([s[0] for s in sizes], np.int32)
    ws = np.ascontiguousarray([s[1] for s in sizes], np.int32)
    ts = None if turns is None else np.ascontiguousarray(turns, np.int32)
    a = {k: np.ascontiguousarray(raw[k], d) for k, d in (
        ('n_tok', np.int32), ('tokens', np.int64), ('probs', np.float32), ('n_inst', np.int32),
        ('inst_pos', np.int32), ('poly', np.int64))}
    E, N = max(int(a['n_tok'].sum()), 1), max(int(a['n_inst'].sum()), 1)
    P = len(sizes)
    out = dict(count=np.zeros(P, np.int32), offset=np.zeros(P, np.int32), cls=np.zeros(E, np.int32),
               prob=np.zeros(E, np.float32), word_offset=np.zeros(E, np.int32), word_count=np.zeros(E, np.int32),
               source=np.zeros((E, 2), np.int32), rect=np.zeros((N, 4)), poly=np.zeros((N, 32)),
               word_source=np.zeros((N, 2), np.int32))
    nw = C.c_long()
    n = lib.emu_merge_kie_tiles(hs.ctypes.data, ws.ctypes.data, None if ts is None else ts.ctypes.data, P, T, ov,
                                a['n_tok'].ctypes.data, a['tokens'].ctypes.data, a['probs'].ctypes.data,
                                a['tokens'].shape[1], a['n_inst'].ctypes.data, a['inst_pos'].ctypes.data,
                                a['poly'].ctypes.data, a['inst_pos'].shape[1], num_bins, class_base, n_classes,
                                margin, band, iou, *[out[k].ctypes.data for k in (
                                    'count', 'offset', 'cls', 'prob', 'word_offset', 'word_count', 'source', 'rect',
                                    'poly', 'word_source')], C.byref(nw))
    if n < 0:
        return None
    for k in ('cls', 'prob', 'word_offset', 'word_count', 'source'):
        out[k] = out[k][:n]
    for k in ('rect', 'poly', 'word_source'):
        out[k] = out[k][:nw.value]
    return out


def oracle_of(sizes, T, ov, raw, turns=None, **kw):
    """oracle/kie_tile_ref.merge of the tiles' entity tuples, each word's text its '(tile, instance)'."""
    plan = PT.plan(sizes, [0] * len(sizes) if turns is None else turns, T, ov)
    ents = []
    for k, (_, _, _, h, w) in enumerate(plan):
        nt, ni = int(raw['n_tok'][k]), int(raw['n_inst'][k])
        ents.append(K.tile_entities(raw['tokens'][k][:nt], raw['probs'][k][:nt], raw['inst_pos'][k][:ni],
                                    raw['poly'][k][:ni], h, w, NB, BASE, NCLS, [f'{k}:{i}' for i in range(ni)]))
    return K.merge(sizes, T, ov, ents, turns=turns, **kw)


def check(sizes, T, ov, raw, turns=None, **kw):
    """The host bodies equal the oracle: entities, classes, probabilities, word rects and word sources."""
    got = emu_merge(sizes, T, ov, raw, turns=turns, **kw)
    ref = oracle_of(sizes, T, ov, raw, turns=turns, **kw)
    for p in range(len(sizes)):
        rows = range(int(got['offset'][p]), int(got['offset'][p]) + int(got['count'][p]))
        assert [tuple(got['source'][r]) for r in rows] == ref['source'][p]
        mine = []
        for r in rows:
            ws = range(int(got['word_offset'][r]), int(got['word_offset'][r]) + int(got['word_count'][r]))
            mine.append((' '.join(f'{s[0]}:{s[1]}' for s in got['word_source'][ws].tolist()), int(got['cls'][r]),
                         float(got['prob'][r]), got['rect'][ws].tolist()))
        assert mine == ref['entities'][p]
    return got


def fabricate(rng, sizes, T, ov, turns=None, n_ent=6, max_words=8, max_tok=96, max_inst=40):
    """Tile decodes of pages holding random entities of 0..max_words words: every tile that sees an entity reads it
    (words binned in the tile's frame with a bin of noise, so readings differ between tiles), sometimes with another
    class, plus lone bins and trailing words of no entity."""
    turns = [0] * len(sizes) if turns is None else list(turns)
    read = [PT.turned_size(H, W, k) for (H, W), k in zip(sizes, turns)]
    plan = R.plan(read, T, ov)
    ents = []
    for p, (H, W) in enumerate(read):
        for _ in range(n_ent):
            nw = int(rng.choice([0, 1, 1, 2, 3, max_words]))
            x, y = rng.uniform(0, W * 0.9), rng.uniform(0, H * 0.9)
            words = []
            for j in range(nw):
                w, h = rng.uniform(3, 0.3 * min(T, W)), rng.uniform(2, 0.1 * min(T, H))
                wx, wy = min(x + j * w * 1.1, W - w), min(y, H - h)
                words.append((wx, wy, w, h))
            ents.append((p, int(rng.integers(0, NCLS)), words))
    nt = len(plan)
    raw = dict(n_tok=np.zeros(nt, np.int32), tokens=np.zeros((nt, max_tok), np.int64),
               probs=rng.uniform(0, 1, (nt, max_tok)).astype(np.float32), n_inst=np.zeros(nt, np.int32),
               inst_pos=np.zeros((nt, max_inst), np.int32), poly=np.zeros((nt, max_inst, 32), np.int64))
    for k, (p, y0, x0, th, tw) in enumerate(plan):
        toks, pos, polys = [], [], []

        def word(wx, wy, w, h):
            xs = np.clip(np.concatenate([np.linspace(wx, wx + w, 8), np.linspace(wx + w, wx, 8)]), x0, x0 + tw - 1e-9)
            ys = np.clip(np.concatenate([np.full(8, wy), np.full(8, wy + h)]), y0, y0 + th - 1e-9)
            poly = np.zeros(32, np.int64)
            poly[0::2] = np.clip(np.floor((xs - x0) / tw * NB) + rng.integers(-1, 2, 16), 0, NB - 1)
            poly[1::2] = np.clip(np.floor((ys - y0) / th * NB) + rng.integers(-1, 2, 16), 0, NB - 1)
            pos.append(len(toks))
            toks.extend([int(poly[0]), int(poly[1])])
            polys.append(poly)

        for ep, cls, words in ents:
            seen = [w for w in words if not (w[0] + w[2] <= x0 or w[0] >= x0 + tw or w[1] + w[3] <= y0 or
                                             w[1] >= y0 + th)]
            if ep != p or (words and not seen) or rng.random() < 0.1 or len(pos) + len(seen) + 2 > max_inst:
                continue
            if not words and rng.random() < 0.5:
                continue
            for w in seen:
                word(*w)
            if rng.random() < 0.2:
                toks.append(int(rng.integers(0, NB)))   # a lone bin before the class
            toks.append(BASE + (cls if rng.random() < 0.8 else int(rng.integers(0, NCLS))))
        if rng.random() < 0.5:  # a trailing word of no entity
            word(x0 + 1, y0 + 1, 5, 3)
        assert len(toks) <= max_tok
        raw['n_tok'][k], raw['n_inst'][k] = len(toks), len(pos)
        raw['tokens'][k, :len(toks)] = toks
        raw['inst_pos'][k, :len(pos)] = pos
        if polys:
            raw['poly'][k, :len(polys)] = polys
    return raw


@pytest.mark.parametrize('seed', range(8))
def test_merge_on_the_host_equals_oracle(seed):
    """Random pages, layouts, turns 0..3, parameters and fabricated decodes (empty tiles, wordless entities, 1-8
    words): the emulated kernels equal the oracle, and the cases reach cuts, candidates and suppression."""
    rng = np.random.default_rng(300 + seed)
    T = int(rng.choice([64, 128, 200]))
    ov = int(rng.integers(0, T // 2 + 1))
    sizes = [(int(rng.integers(1, 4 * T)), int(rng.integers(1, 4 * T))) for _ in range(int(rng.integers(1, 5)))]
    sizes[0] = (3 * T, 2 * T + 7)
    sizes.append((T // 2, T - 1))   # a page that is one tile
    turns = None if seed % 2 == 0 else rng.integers(0, 4, len(sizes)).tolist()
    raw = fabricate(rng, sizes, T, ov, turns)
    kw = dict(margin=float(rng.choice([0.0, 4.0, 2.5])), band=None if seed % 3 else float(rng.uniform(0, ov / 2 + 1)),
              iou=float(rng.choice([0.5, 0.3, 1.0])))
    got = check(sizes, T, ov, raw, turns, **kw)
    ents = sum(len(K.walk(raw['tokens'][k][:raw['n_tok'][k]], raw['probs'][k], raw['inst_pos'][k][:raw['n_inst'][k]],
                          NB, BASE, NCLS)) for k in range(len(raw['n_tok'])))
    assert 0 < int(got['count'].sum()) < ents
    assert (raw['n_tok'] == 0).any() or (raw['n_inst'] == 0).any() or seed % 2


# hand-made cases: a 100 x 160 page, T 100, ov 40: tiles at x 0 and 60, seam 80, band 10; num_bins 100 so a bin is a
# pixel of the tile's frame
def hand(readings, n_tiles=2):
    """readings: [(tile, class, [page boxes of its words])] -> tile decodes (boxes in page pixels, tile at x0)."""
    x0s = [0, 60, 0, 60]
    raw = dict(n_tok=np.zeros(n_tiles, np.int32), tokens=np.zeros((n_tiles, 32), np.int64),
               probs=np.full((n_tiles, 32), 0.5, np.float32), n_inst=np.zeros(n_tiles, np.int32),
               inst_pos=np.zeros((n_tiles, 8), np.int32), poly=np.zeros((n_tiles, 8, 32), np.int64))
    for k, cls, boxes in readings:
        for a, b, c, d in boxes:
            i, t = raw['n_inst'][k], raw['n_tok'][k]
            xs = np.concatenate([np.linspace(a, c, 8), np.linspace(c, a, 8)]) - x0s[k]
            ys = np.concatenate([np.full(8, b), np.full(8, d)])
            raw['poly'][k, i, 0::2], raw['poly'][k, i, 1::2] = np.round(xs), np.round(ys)
            raw['inst_pos'][k, i] = t
            raw['tokens'][k, t:t + 2] = raw['poly'][k, i, :2]
            raw['n_inst'][k] += 1
            raw['n_tok'][k] += 2
        raw['tokens'][k, raw['n_tok'][k]] = 104 + cls
        raw['n_tok'][k] += 1
    return raw


def kept(sizes, raw, **kw):
    lib_kw = dict(num_bins=100, class_base=104)
    got = emu_merge(sizes, 100, 40, raw, **kw, **lib_kw)
    return [tuple(s) for s in got['source'].tolist()], got


def test_seam_cases():
    """Each rule of the merge on a hand-made case."""
    S = [(100, 160)]
    # an entity in the overlap read by both tiles: kept once, from the tile where it lies farther from an interior edge
    # (tile 0: 100 - 90 = 10 px, tile 1: 72 - 60 = 12 px)
    assert kept(S, hand([(0, 1, [(72, 40, 80, 50), (82, 40, 90, 50)]), (1, 1, [(72, 40, 90, 50)])]))[0] == [(1, 0)]
    # two readings with different classes are resolved by the rule, not by the class
    src, got = kept(S, hand([(0, 0, [(72, 40, 90, 50)]), (1, 3, [(72, 40, 90, 50)])]))
    assert src == [(1, 0)] and got['cls'].tolist() == [3]
    # ties (10 px each) go to the lower tile
    assert kept(S, hand([(0, 2, [(70, 40, 90, 50)]), (1, 2, [(70, 40, 90, 50)])]))[0] == [(0, 0)]
    # an entity cut by an interior edge (4 px from x = 100 in tile 0) is dropped; 5 px is not cut
    assert kept(S, hand([(0, 1, [(30, 40, 96, 50)])]))[0] == []
    assert kept(S, hand([(0, 1, [(30, 40, 95, 50)])]))[0] == [(0, 0)]
    # the anchor decides the tile: centre x 84 lies in tile 1's widened core only with the band
    assert kept(S, hand([(0, 1, [(78, 40, 90, 50)])]))[0] == [(0, 0)]
    assert kept(S, hand([(0, 1, [(80, 40, 94, 50)])]), band=0.0)[0] == []
    # entities of one tile never suppress each other
    assert kept(S, hand([(0, 1, [(10, 10, 30, 20)]), (0, 2, [(10, 10, 30, 20)])]))[0] == [(0, 0), (0, 1)]
    # a wordless entity is dropped on a page of several tiles and kept on a page that is one tile
    assert kept(S, hand([(0, 1, [])]))[0] == []
    src, got = kept([(100, 90)], hand([(0, 1, [])], n_tiles=1))
    assert src == [(0, 0)] and got['word_count'].tolist() == [0]
    # rects: tile origin + w * min / num_bins
    src, got = kept(S, hand([(1, 0, [(130, 40, 159, 50)])]))
    assert got['rect'].tolist() == [[130.0, 40.0, 159.0, 50.0]] and got['word_source'].tolist() == [[1, 0]]


def test_walk_failures():
    """A mismatched inst_pos and a token that is neither a bin nor a class fail the walk, in the host bodies and the
    oracle."""
    raw = hand([(0, 1, [(10, 10, 30, 20)])])
    bad = {k: v.copy() for k, v in raw.items()}
    bad['inst_pos'][0, 0] = 1
    assert emu_merge([(100, 160)], 100, 40, bad, num_bins=100, class_base=104) is None
    bad = {k: v.copy() for k, v in raw.items()}
    bad['tokens'][0, 2] = 104 + 4
    assert emu_merge([(100, 160)], 100, 40, bad, num_bins=100, class_base=104) is None
    with pytest.raises(ValueError):
        K.walk([5, 6, 200], [1] * 3, [0], 100, 104, 4)
    with pytest.raises(ValueError):
        K.walk([5, 6, 104], [1] * 3, [1], 100, 104, 4)


def post_cases():
    """tests/golden/post_kie.json: the reference's own decode_vie_pt_poly_rec_seq on scripted decodes."""
    for c in json.load(open(os.path.join(GOLD, 'post_kie.json'))):
        probs = np.frombuffer(bytes.fromhex(c['probs_f32_hex']), dtype='<f4').copy()
        yield c, probs


def test_single_tile_page_is_the_reference_walk():
    """A page that is one upright tile keeps every entity, wordless ones included, with decode_vie_pt_poly_rec_seq's
    classes, probabilities and rects bit for bit: the reference's own values in tests/golden/post_kie.json."""
    for c, probs in post_cases():
        h, w = (int(v) for v in c['orig'])
        toks = np.asarray(c['tokens'], np.int64).reshape(1, -1)
        pos = np.asarray(c['pos'], np.int32).reshape(1, -1)
        n = pos.shape[1]
        raw = dict(n_tok=np.array([toks.shape[1]], np.int32), tokens=np.pad(toks, ((0, 0), (0, 1))),
                   probs=np.pad(probs.reshape(1, -1), ((0, 0), (0, 1))), n_inst=np.array([n], np.int32),
                   inst_pos=np.pad(pos, ((0, 0), (0, 1))),
                   poly=np.pad(np.asarray(c['poly'], np.int64).reshape(1, n, 32), ((0, 0), (0, 1), (0, 0))))
        got = emu_merge([(h, w)], max(64, h, w), 0, raw, class_base=c['class_base'], n_classes=len(c['classes']))
        exp = json.loads(c['json'])
        assert int(got['count'][0]) == len(exp)
        for r, e in enumerate(exp):
            ws = range(int(got['word_offset'][r]), int(got['word_offset'][r]) + int(got['word_count'][r]))
            assert got['rect'][ws].tolist() == e[3]
            assert float(got['prob'][r]) == e[2] and c['classes'][int(got['cls'][r])] == e[1]


def test_shared_walk_gives_the_kie_json():
    """alm_post_omni_kie_json, now on the shared walk, still gives the reference's json.dumps of every case of
    tests/golden/post_kie.json, and its entities are the oracle walk's."""
    from types import SimpleNamespace

    from advancedliteratemachinery_b200 import postprocess as P
    for c, probs in post_cases():
        a = SimpleNamespace(chars=c['chars'], num_bins=1000, rec_length=c['rec_length'])
        a.recog_pad_index = a.num_bins + len(a.chars) + 1
        a.rec_eos_index = a.recog_pad_index + 3
        text = P.kie_json(c['tokens'], probs, c['pos'], np.asarray(c['poly'], dtype=np.int64).reshape(-1, 32),
                          np.asarray(c['rec'], dtype=np.int64).reshape(-1, a.rec_length), c['orig'], a, c['classes'],
                          c['class_base'])
        assert text == c['json']
        walked = K.walk(c['tokens'], probs, c['pos'], 1000, c['class_base'], len(c['classes']))
        assert [(c['classes'][e[0]], e[1], len(e[2])) for e in walked] == \
            [(e[1], e[2], len(e[3])) for e in json.loads(text)]


def test_fixture_merge():
    """tests/golden/omni_kie_tiles.npz: the reference's entity tuples of every tile are the walk of the stored raw
    decodes, and the emulated merge of those decodes equals the oracle's merge of the reference's tuples."""
    g = np.load(os.path.join(GOLD, 'omni_kie_tiles.npz'))
    T, ov, base = int(g['tile']), int(g['overlap']), int(g['class_base'])
    page = [tuple(g['page'].shape[:2])]
    raw = {k: g[k] for k in ('n_tok', 'tokens', 'probs', 'n_inst', 'inst_pos', 'poly')}
    ref_ents = [[] for _ in range(len(g['plan']))]
    for (k, i, c), p, r, t in zip(g['ref_ent'].tolist(), g['ref_prob'].tolist(), g['ref_rect'].tolist(),
                                  g['ref_text'].tolist()):
        if i == len(ref_ents[k]):
            ref_ents[k].append((t, c, p, []))
        ref_ents[k][i][3].append(r)
    assert [len(e) for e in ref_ents] == g['ref_n_ent'].tolist()
    for k, (_, _, _, h, w) in enumerate(g['plan'].tolist()):
        nt, ni = int(raw['n_tok'][k]), int(raw['n_inst'][k])
        mine = K.tile_entities(raw['tokens'][k][:nt], raw['probs'][k][:nt], raw['inst_pos'][k][:ni],
                               raw['poly'][k][:ni], h, w, int(g['num_bins']), base, int(g['vie']))
        assert [(e[1], e[3]) for e in mine] == [(e[1], e[3]) for e in ref_ents[k]]
        assert all(abs(a[2] - b[2]) < 1e-6 for a, b in zip(mine, ref_ents[k]))
    ref = K.merge(page, T, ov, ref_ents)
    got = emu_merge(page, T, ov, raw, class_base=base)
    assert [tuple(s) for s in got['source'].tolist()] == ref['source'][0]
    assert 0 < int(got['count'][0]) < sum(len(e) for e in ref_ents)
    for r, e in enumerate(ref['entities'][0]):
        ws = range(int(got['word_offset'][r]), int(got['word_offset'][r]) + int(got['word_count'][r]))
        assert got['rect'][ws].tolist() == e[3] and int(got['cls'][r]) == e[1]
