"""GPU: caller-given regions read at quarter-turns (DESIGN 4.21; read_regions(orientation=...),
alm_pre_omni_tiles_at_turned, alm_omni_select_regions).

* turn 0 for every region is 'upright' bit for bit, for points, boxes, quads, polygons and a region read whole;
* a region read at turn k is the region read upright on np.rot90(page, k) at its turned point or box, mapped back;
* per-region turns mixed in one call agree with the single-turn calls region by region;
* 'auto': the candidate turns, the scores, the kept turn and the kept outputs;
* candidates, beams and character boxes follow the kept reading;
* the new C entries against the emulation and the range entry, their refusals, and the Python refusals.
"""
import numpy as np
import pytest
import torch

from tests.support import golden, kw, omni_model, release_models
from tests.test_region_turns_cpu import EOS, NB, PAD, emu_select, fabricate

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

ERR_INVALID = -1
def spot_model(wseed=0, pt_eos_bias=-30.0, pt_seq_length=8, rec_length=25):
    return omni_model(dict(wseed=wseed, pt_eos_bias=pt_eos_bias, pt_seq_length=pt_seq_length, rec_length=rec_length))


def tiles_fixture():
    """the omni_tiles.npz model and page (300 x 220, read in 128-pixel tiles), and spot_tiled's words on it"""
    gold = golden('omni_tiles.npz')
    return gold, omni_model(gold), kw(gold)


def fixture_regions(m, page, kw):
    """the fixture page's words as points, integer boxes, quads and polygons, plus a box wider than a tile (read
    whole)"""
    words = m.spot_tiled([page], **kw)[0]
    polys = np.array([w['polys'] for w in words], np.float64)
    H, W = page.shape[:2]
    lo = np.floor(polys.min(1)).clip(0, [W, H])
    hi = np.ceil(polys.max(1)).clip(0, [W, H])
    boxes = np.concatenate([np.concatenate([lo, hi], 1), [[10, 100, 200, 130]]])
    return dict(point=np.round(np.array([w['pts'][0] for w in words])), box=boxes,
                quad=np.round(polys[:, [0, 7, 8, 15]]), polygon=polys)


def bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint32) if a.dtype == np.float32 else a


def same_chars(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert x['char'] == y['char']
        for k in ('centre', 'cov', 'box'):
            assert np.array_equal(x[k], y[k]), k


def same_results(got, want, keys=('pts', 'score', 'polys', 'rec', 'page', 'tile')):
    assert len(got) == len(want)
    for g, w in zip(got, want):
        for k in keys:
            assert g[k] == w[k], k
        if 'chars' in w:
            same_chars(g['chars'], w['chars'])


def map_back(k, xy, H, W):
    """numpy map_back of points [n, 2] of np.rot90(page, k) to the upright H x W page"""
    u, v = xy[:, 0], xy[:, 1]
    x, y = {0: (u, v), 1: (W - v, u), 2: (W - u, H - v), 3: (v, H - u)}[k]
    return np.stack([x, y], 1)


def a4_pages(seed=9):
    rng = np.random.default_rng(seed)
    return [rng.integers(0, 256, (3508, 2480, 3), dtype=np.uint8), rng.integers(0, 256, (500, 700, 3), dtype=np.uint8)]


def a4_boxes(seed=10, R=30):
    """integer boxes on the A4 page (wide, tall, and one across two column seams) and three on the small page"""
    rng = np.random.default_rng(seed)
    xy = rng.integers([0, 0], [2480 - 400, 3508 - 400], (R, 2))
    wh = np.where(rng.random((R, 1)) < 0.5, rng.integers([30, 12], [400, 60], (R, 2)),
                  rng.integers([12, 30], [60, 400], (R, 2)))
    boxes = np.concatenate([xy, xy + wh], 1).astype(np.float64)
    boxes[R - 1] = [1100, 1500, 2200, 1540]
    boxes = np.concatenate([boxes, [[10, 10, 100, 40], [600, 450, 700, 500], [0, 0, 700, 500]]])
    pi = np.zeros(R + 3, int)
    pi[-3:] = 1
    return boxes, pi


# ------------------------------------------------------------------------------------------------ turn 0
def test_turn_zero_is_upright_bit_for_bit():
    gold, m, kw = tiles_fixture()
    page = gold['page']
    for kind, regions in fixture_regions(m, page, kw).items():
        R = len(regions)
        pi = np.zeros(R, int)
        want = m.read_regions([page], regions, pi, kind=kind, max_batch=3, rec_locations=True, **kw)
        lw = m.last_rec_locations
        got = m.read_regions([page], regions, pi, kind=kind, max_batch=3, rec_locations=True,
                             orientation=np.zeros(R, np.int64), **kw)
        same_results(got, want)
        assert all(g['turns'] == 0 for g in got) and np.array_equal(bits(m.last_rec_locations), bits(lw)), kind
        if kind == 'box':
            assert got[-1]['tile'] == -1
    m._set_rec_candidates(0)


def test_turn_zero_on_an_a4_page():
    m = spot_model(0, -30.0, 12, 25)
    pages = a4_pages()
    boxes, pi = a4_boxes()
    kw = dict(tile=1200, overlap=256, test_min_size=1200, test_max_size=1920)
    want = m.read_regions(pages, boxes, pi, kind='box', max_batch=4, **kw)
    got = m.read_regions(pages, boxes, pi, kind='box', max_batch=4, orientation=np.zeros(len(boxes), np.int32), **kw)
    same_results(got, want)
    assert got[len(boxes) - 4]['tile'] == -1


# ------------------------------------------------------------------------------------------------ one turn
def check_turned(m, page, regions, kind, k, kw, max_batch):
    """orientation=[k] * R against upright read_regions on np.rot90(page, k) at the turned points / boxes"""
    from advancedliteratemachinery_b200 import postprocess as P
    from advancedliteratemachinery_b200.omniparser import region_boxes, turn_boxes, turn_points
    H, W = page.shape[:2]
    R = len(regions)
    pi = np.zeros(R, int)
    hw = np.tile([H, W], (R, 1))
    got = m.read_regions([page], regions, pi, kind=kind, max_batch=max_batch, orientation=np.full(R, k), **kw)
    lg = m.last_regions
    rot = np.ascontiguousarray(np.rot90(page, k))
    if kind == 'box':
        tregions = turn_boxes(region_boxes(regions, 'box'), hw, np.full(R, k))
    else:
        tregions = turn_points(P.region_points(regions, kind), hw, np.full(R, k))
    want = m.read_regions([rot], tregions, pi, kind='box' if kind == 'box' else 'point', max_batch=max_batch, **kw)
    lw = m.last_regions
    assert [c['kind'] for c in lg['chunks']] == [c['kind'] for c in lw['chunks']]
    for a, b in zip(lg['chunks'], lw['chunks']):
        assert np.array_equal(a['index'], b['index'])
        for key in ('n', 'pt', 'poly', 'rec'):
            assert np.array_equal(a[key], b[key]), key
        assert np.array_equal(bits(a['prob']), bits(b['prob']))
    for g, w in zip(got, want):
        assert g['rec'] == w['rec'] and g['score'] == w['score'] and g['tile'] == w['tile'] and g['turns'] == k
        assert np.array_equal(np.array(g['pts']), map_back(k, np.array(w['pts']), H, W))
        assert np.array_equal(np.array(g['polys']), map_back(k, np.array(w['polys']), H, W))
    return got


@pytest.mark.parametrize('k', [1, 2, 3])
def test_a_turn_is_a_turned_page(k):
    gold, m, kw = tiles_fixture()
    regions = fixture_regions(m, gold['page'], kw)
    for kind in ('point', 'box'):
        check_turned(m, gold['page'], regions[kind], kind, k, kw, max_batch=3)


def test_a_turn_on_an_a4_page():
    m = spot_model(0, -30.0, 12, 25)
    page = a4_pages()[0]
    boxes, pi = a4_boxes(R=24)
    kw = dict(tile=1200, overlap=256, test_min_size=1200, test_max_size=1920)
    got = check_turned(m, page, boxes[pi == 0], 'box', 1, kw, max_batch=5)
    assert got[-1]['tile'] == -1


# ------------------------------------------------------------------------------------------------ mixed turns
def test_mixed_turns_agree_with_single_turn_calls():
    gold, m, kw = tiles_fixture()
    page = gold['page']
    other = np.ascontiguousarray(np.rot90(page, 1)[40:, :250])
    boxes = fixture_regions(m, page, kw)['box']
    boxes = np.concatenate([boxes, boxes[:8]])
    pi = np.zeros(len(boxes), int)
    pi[-8:] = 1
    ok = (boxes[:, 2] <= np.where(pi == 1, other.shape[1], page.shape[1])) & \
        (boxes[:, 3] <= np.where(pi == 1, other.shape[0], page.shape[0]))
    boxes, pi = boxes[ok], pi[ok]
    R = len(boxes)
    turns = np.random.default_rng(5).integers(0, 4, R)
    got = m.read_regions([page, other], boxes, pi, kind='box', max_batch=4, orientation=turns, **kw)
    rows = m.last_regions['rec'][:, 0]
    probs = m.last_regions['prob'][:, 0]
    assert len(m.last_regions['readings']) > 4
    for k in range(4):
        want = m.read_regions([page, other], boxes, pi, kind='box', max_batch=4, orientation=np.full(R, k), **kw)
        sel = np.nonzero(turns == k)[0]
        assert np.array_equal(rows[sel], m.last_regions['rec'][sel, 0])
        np.testing.assert_allclose(probs[sel], m.last_regions['prob'][sel, 0], rtol=5e-5, atol=0)
        for r in sel:
            assert got[r]['rec'] == want[r]['rec'] and got[r]['tile'] == want[r]['tile'] and got[r]['turns'] == k
            assert got[r]['pts'] == want[r]['pts'] and got[r]['polys'] == want[r]['polys']


# ------------------------------------------------------------------------------------------------ 'auto'
def host_score(rec, prob):
    s, n = 0.0, 0
    for t, p in zip(rec.tolist(), prob.tolist()):
        if t in (PAD, EOS):
            break
        if t == PAD - 1:
            continue
        s, n = s + float(p), n + 1
    return s / (n + 1e-5)


def check_auto(m, pages, regions, pi, kind, kw, max_batch, **extra):
    from advancedliteratemachinery_b200.omniparser import region_turn_candidates
    sizes = [p.shape[:2] for p in pages]
    got = m.read_regions(pages, regions, pi, kind=kind, max_batch=max_batch, orientation='auto', **extra, **kw)
    lr = m.last_regions
    cand = region_turn_candidates(sizes, regions, pi, kind)
    assert np.array_equal(lr['candidates'], cand)
    R = len(regions)
    want_scores = np.array([[host_score(lr['rec'][r, c], lr['prob'][r, c]) for c in range(2)] for r in range(R)])
    assert np.array_equal(lr['scores'], want_scores)
    kept = np.where(want_scores[:, 1] > want_scores[:, 0], 1, 0)   # the lower turn on a tie
    assert np.array_equal(lr['turns'], cand[np.arange(R), kept])
    assert [g['turns'] for g in got] == lr['turns'].tolist()
    return got, kept


def test_auto_keeps_the_better_reading():
    gold, m, kw = tiles_fixture()
    page = gold['page']
    regions = fixture_regions(m, page, kw)
    tall = np.array([[20, 20, 40, 120], [150, 30, 170, 200]], np.float64)   # 2 h >= 3 w: turns 1 and 3
    boxes = np.concatenate([regions['box'], tall])
    R = len(boxes)
    got, kept = check_auto(m, [page], boxes, np.zeros(R, int), 'box', kw, 3)
    turns = m.last_regions['turns']
    assert (m.last_regions['candidates'][-2:] == [1, 3]).all() and (m.last_regions['candidates'][0] == [0, 2]).all()
    rows, probs = m.last_regions['rec'], m.last_regions['prob']
    for k in np.unique(turns).tolist():
        want = m.read_regions([page], boxes, np.zeros(R, int), kind='box', max_batch=3, orientation=np.full(R, k), **kw)
        for r in np.nonzero(turns == k)[0]:
            assert np.array_equal(rows[r, kept[r]], m.last_regions['rec'][r, 0])
            np.testing.assert_allclose(probs[r, kept[r]], m.last_regions['prob'][r, 0], rtol=5e-5, atol=0)
            assert got[r]['rec'] == want[r]['rec'] and got[r]['tile'] == want[r]['tile']
            assert got[r]['pts'] == want[r]['pts'] and got[r]['polys'] == want[r]['polys']
    for kind in ('quad', 'polygon', 'point'):
        check_auto(m, [page], regions[kind], np.zeros(len(regions[kind]), int), kind, kw, 16)


def test_auto_on_an_a4_page():
    m = spot_model(0, -30.0, 12, 25)
    pages = a4_pages()
    boxes, pi = a4_boxes()
    kw = dict(tile=1200, overlap=256, test_min_size=1200, test_max_size=1920)
    check_auto(m, pages, boxes, pi, 'box', kw, 4)
    first = m.last_regions['candidates'][:, 0]
    assert (first == 1).any() and (first == 0).any(), 'tall and wide regions'


# ------------------------------------------------------------------------------------------------ lists
def test_candidates_beams_and_chars_follow_the_kept_reading():
    from advancedliteratemachinery_b200.omniparser import char_boxes, char_dicts
    gold, m, kw = tiles_fixture()
    page = gold['page']
    boxes = fixture_regions(m, page, kw)['box']
    R = len(boxes)
    pi = np.zeros(R, int)
    base = m.read_regions([page], boxes, pi, kind='box', max_batch=3, orientation='auto', **kw)
    kept = m.last_regions['turns']
    k_idx = np.where(kept == m.last_regions['candidates'][:, 0], 0, 1)
    got = m.read_regions([page], boxes, pi, kind='box', max_batch=3, orientation='auto', rec_candidates=3, **kw)
    ids, probs = m.last_rec_candidates
    assert ids.shape == (R, m.vocab.rec_length, 3) and [g['rec'] for g in got] == [b['rec'] for b in base]
    assert np.array_equal(ids[:, :, 0], m.last_regions['rec'][np.arange(R), k_idx])
    assert np.array_equal(bits(probs[:, :, 0]), bits(m.last_regions['prob'][np.arange(R), k_idx]))
    m.read_regions([page], boxes, pi, kind='box', max_batch=3, orientation='auto', rec_beams=2, **kw)
    lr = m.last_regions
    kb = np.where(lr['turns'] == lr['candidates'][:, 0], 0, 1)
    assert m.last_rec_beams[0].shape == (R, 2, m.vocab.rec_length)
    assert np.array_equal(m.last_rec_beams[0][:, 0], lr['rec'][np.arange(R), kb])
    got = m.read_regions([page], boxes, pi, kind='box', max_batch=3, orientation='auto', rec_locations=True, **kw)
    lr = m.last_regions
    kl = np.where(lr['turns'] == lr['candidates'][:, 0], 0, 1)
    assert [g['rec'] for g in got] == [b['rec'] for b in base]
    g = np.arange(R) * 2 + kl
    f = lr['frames'][lr['frame_index'].reshape(-1)[g]]
    sizes = [(int(a), int(b)) for a, b in f[:, :2]]
    tiles = np.stack([np.arange(R), f[:, 3], f[:, 4], f[:, 5], f[:, 6]], 1)
    rec = lr['rec'][np.arange(R), kl]
    polys = np.array([x['polys'] for x in got]).reshape(R, 32)
    hand = char_dicts(char_boxes(m.ctx, sizes, tiles, polys, rec, m.last_rec_locations, np.arange(R), PAD, EOS,
                                 turns=f[:, 2]), rec, m.vocab)
    assert any(len(c) for c in hand)
    for x, c in zip(got, hand):
        same_chars(x['chars'], c)
    m._set_rec_candidates(0)


# ------------------------------------------------------------------------------------------------ C entries
def test_tiles_at_turned_equal_the_turned_range_entry():
    from advancedliteratemachinery_b200 import _lib, preprocess as P
    ctx = _lib.Context(0)
    try:
        rng = np.random.default_rng(2)
        base = [rng.integers(0, 256, s + (3,), dtype=np.uint8) for s in ((1900, 1300), (700, 1500))]
        pages = [base[0], base[1], base[0]]          # page 0 listed again at another turn
        turns = np.array([1, 2, 3], np.int32)
        plan = P.omni_tile_plan(P.turned_sizes([p.shape[:2] for p in pages], turns), 1200, 256)
        for idx in ([2, 3, 4], [len(plan) - 1, 0, 5, 5], list(range(len(plan)))):
            got = P.omni_tiles_at(ctx, pages, idx, 1200, 256, 1200, 1920, turns=turns)
            for j, i in enumerate(idx):
                want = P.omni_tiles(ctx, pages, 1200, 256, 1200, 1920, i, 1, turns=turns)
                h, w = want.tensors.shape[2:]
                assert torch.equal(got.tensors[j, :, :h, :w].view(torch.int32), want.tensors[0].view(torch.int32))
                assert torch.equal(got.mask[j, :h, :w], want.mask[0]) and bool(got.mask[j, h:].all())
        zero = P.omni_tiles_at(ctx, base, [0, 3], 1200, 256, 1200, 1920, turns=[0, 0])
        want = P.omni_tiles_at(ctx, base, [0, 3], 1200, 256, 1200, 1920)
        assert torch.equal(zero.tensors.view(torch.int32), want.tensors.view(torch.int32))
        with pytest.raises(ValueError):
            P.omni_tiles_at(ctx, base, [0], 1200, 256, 1200, 1920, turns=[0, 4])
        keep, ptrs, hs, ws, n = P._image_args(base)
        idx = np.zeros(1, np.int32)
        t = torch.empty(1, 3, 1200, 1200, device='cuda')
        mk = torch.empty(1, 1200, 1200, dtype=torch.uint8, device='cuda')
        for bad in (None, np.array([0, 4], np.int32), np.array([-1, 0], np.int32)):
            assert ctx.lib.alm_pre_omni_tiles_at_turned(
                ctx.h, ptrs, hs.ctypes.data, ws.ctypes.data, n, None if bad is None else bad.ctypes.data, 1200, 256,
                idx.ctypes.data, 1, 1200, 1920, t.data_ptr(), mk.data_ptr()) == ERR_INVALID
    finally:
        ctx.close()


def test_select_regions_equals_the_emulation():
    from advancedliteratemachinery_b200 import _lib
    from advancedliteratemachinery_b200.omniparser import select_regions
    ctx = _lib.Context(0)
    try:
        cases = [fabricate(0, Cn=1), fabricate(1, Cn=2), fabricate(3, Cn=4), fabricate(5, R=40, L=1021),
                 fabricate(6, R=20000, Cn=2, F=64)]
        frames, fidx, pt, poly, rec, prob = fabricate(7, R=50)
        rec[:15, :, 0] = NB + 1
        prob[:10, 0, 0] = np.nan     # NaN scores: never kept over a number
        prob[10:15, :, 0] = np.nan
        cases.append((frames, fidx, pt, poly, rec, prob))
        for data in cases:
            got = select_regions(ctx, *data, NB, PAD, EOS)
            want = emu_select(*data)
            for k, w in zip(('kept', 'scores', 'pts', 'polys'), want):
                assert np.array_equal(got[k], w, equal_nan=True), k
        assert (got['kept'][:10] == 1).all() and (got['kept'][10:15] == 0).all()
        frames, fidx, pt, poly, rec, prob = fabricate(8, R=30)
        rec[:, 1], prob[:, 1] = rec[:, 0], prob[:, 0]   # a region read twice at identical rows
        got = select_regions(ctx, frames, fidx, pt, poly, rec, prob, NB, PAD, EOS)
        turns = frames[fidx, 2]
        assert np.array_equal(got['scores'][:, 0], got['scores'][:, 1])
        assert np.array_equal(got['kept'], np.where(turns[:, 1] < turns[:, 0], 1, 0))
        empty = select_regions(ctx, frames, fidx[:0], pt[:0], poly[:0], rec[:0], prob[:0], NB, PAD, EOS)
        assert empty['kept'].shape == (0,)
    finally:
        ctx.close()


def test_select_regions_refusals_leave_the_context_usable():
    from advancedliteratemachinery_b200.omniparser import select_regions
    gold, m, kw = tiles_fixture()
    frames, fidx, pt, poly, rec, prob = fabricate(9, R=12)
    ok = select_regions(m.ctx, frames, fidx, pt, poly, rec, prob, NB, PAD, EOS)
    lib, h = m.lib, m.ctx.h
    R, Cn = fidx.shape

    def call(fr=frames, fi=fidx, c=Cn, nf=None, null=None, L=rec.shape[2], nb=NB):
        fr = np.ascontiguousarray(fr, np.int32)
        fi = np.ascontiguousarray(fi, np.int32)
        bufs = [fi, fr, np.ascontiguousarray(pt), np.ascontiguousarray(poly), np.ascontiguousarray(rec),
                np.ascontiguousarray(prob)]
        outs = [np.zeros(R, np.int32), np.zeros((R, 4)), np.zeros((R, 2)), np.zeros((R, 32))]
        ptrs = [None if null == i else a.ctypes.data for i, a in enumerate(bufs + outs)]
        return lib.alm_omni_select_regions(h, R, c, ptrs[0], len(fr) if nf is None else nf, ptrs[1], *ptrs[2:6], L,
                                           nb, PAD, EOS, *ptrs[6:])
    bad_turn, bad_size, outside = frames.copy(), frames.copy(), frames.copy()
    bad_turn[3, 2] = 4
    bad_size[2, 5] = 0
    outside[1, 4] = max(outside[1, 0], outside[1, 1]) + 1
    neg = fidx.copy()
    neg[2, 1] = -1
    big = fidx.copy()
    big[0, 0] = len(frames)
    refusals = [dict(null=i) for i in range(10)] + [dict(c=0), dict(c=5), dict(fi=neg), dict(fi=big),
                                                   dict(fr=bad_turn), dict(fr=bad_size), dict(fr=outside), dict(nf=0),
                                                   dict(L=0), dict(nb=0)]
    n0 = m.ctx.launch_count()
    for bad in refusals:
        assert call(**bad) == ERR_INVALID, bad
    assert m.ctx.launch_count() == n0, 'refused before any device work'
    again = select_regions(m.ctx, frames, fidx, pt, poly, rec, prob, NB, PAD, EOS)
    for k in ok:
        assert np.array_equal(ok[k], again[k]), k
    page = gold['page']
    m.read_regions([page], [[50, 50]], [0], kind='point', orientation='auto', **kw)   # a decode still works


# ------------------------------------------------------------------------------------------------ Python refusals
def test_python_refusals_come_before_any_device_work():
    from advancedliteratemachinery_b200 import OmniParserB200, OmniVocab
    from advancedliteratemachinery_b200 import synthetic as W
    from oracle.gen_golden import KIE_CASES
    gold, m, kw = tiles_fixture()
    page = gold['page']
    pts = np.array([[50, 50], [100, 200]])
    m.read_regions([page], pts, [0, 0], kind='point', orientation=[1, 3], **kw)
    n0 = m.ctx.launch_count()
    for bad in ('mixed', 'sideways', 'Upright', [1], [1, 2, 3], np.array([1.0, 2.0]), [0, 4], [-1, 0], [[1, 2]]):
        with pytest.raises(ValueError):
            m.read_regions([page], pts, [0, 0], kind='point', orientation=bad, **kw)
    with pytest.raises(ValueError):
        m.read_regions([page], pts, [0, 0], kind='point', orientation='auto', rec_locations=True, rec_beams=2, **kw)
    assert m.ctx.launch_count() == n0
    c = KIE_CASES['kie']
    kie = OmniParserB200(W.omniparser_state_dict(seed=c['wseed'], vie_categories=c['vie'], pt_eos_bias=c['pt_eos_bias']),
                         OmniVocab(vie_categories=c['vie'], pt_seq_length=c['pt_seq_length']), workspace_mb=1024)
    try:
        n1 = kie.ctx.launch_count()
        for o in ('auto', [1, 2]):
            with pytest.raises(ValueError):
                kie.read_regions([page], pts, [0, 0], kind='point', orientation=o, **kw)
        assert kie.ctx.launch_count() == n1
    finally:
        kie.ctx.close()
