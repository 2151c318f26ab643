"""GPU: reading at caller points (alm_omni_decode_at / OmniParserB200.read_at) and regions of raw pages (read_regions).

* reference parity: the fixture of oracle/gen_golden_points.py (the reference's own polygon and recognition loops on
  chosen points) and the small decode fixtures read at their own points;
* decode followed by read_at at its points, on the same encoded batch, is decode bit for bit -- ids, probabilities,
  candidates, n-best lists and character locations -- under the decode schedules and for a mixed-size batch: the rows,
  Ncap and therefore every launch are the ones decode ran;
* batch invariance, the refusals, and read_regions on the tiled-page fixture and an A4-size page.
"""
import os

import numpy as np
import pytest
import torch

from tests.support import golden, kw, omni_model, options, release_models
from tests.test_read_at_cpu import brute_route

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

ERR_INVALID, ERR_STATE = -1, -4
def spot_model(wseed=0, pt_eos_bias=-30.0, pt_seq_length=8, rec_length=25):
    return omni_model(dict(wseed=wseed, pt_eos_bias=pt_eos_bias, pt_seq_length=pt_seq_length, rec_length=rec_length))


def case(name, golden_dir):
    from oracle.gen_golden import OMNI_CASES, omni_inputs
    c = OMNI_CASES[name]
    img, mask = omni_inputs(c)
    return c, np.load(os.path.join(golden_dir, f'omni_{name}.npz')), img, mask


def bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint32) if a.dtype == np.float32 else a


def assert_same(a, b, what):
    if isinstance(a, (tuple, list)):
        assert len(a) == len(b), what
        for i, (x, y) in enumerate(zip(a, b)):
            assert_same(x, y, f'{what}[{i}]')
    elif a is None or b is None:
        assert a is None and b is None, what
    else:
        assert a.shape == b.shape and np.array_equal(bits(a), bits(b)), what


# ----------------------------------------------------------------------------------------------- reference parity
@pytest.mark.parametrize('name', ['full', 'odd'])
def test_reference_polygon_and_recognition_loops_at_points(name, golden_dir):
    from oracle.gen_golden import OMNI_CASES, omni_inputs
    gold = np.load(os.path.join(golden_dir, 'omni_points.npz'))
    c = OMNI_CASES[name]
    m = spot_model(c['wseed'], c['pt_eos_bias'], c['pt_seq_length'], c['rec_length'])
    img, mask = omni_inputs(c)
    m.encode(img, mask)
    pts = gold[f'{name}_pts']
    (pt, poly, rec), (probs,) = m.read_at([pts])[0]
    assert np.array_equal(pt.numpy().reshape(-1, 2), pts)
    assert np.array_equal(poly.numpy().reshape(-1, 32), gold[f'{name}_poly']), 'polygon ids'
    assert np.array_equal(rec.numpy()[0], gold[f'{name}_rec']), 'recognition ids'
    np.testing.assert_allclose(probs.numpy(), gold[f'{name}_probs'], rtol=2e-3, atol=1e-7)
    if name == 'full':   # the duplicated point is read twice, identically
        assert np.array_equal(poly.numpy().reshape(-1, 32)[0], poly.numpy().reshape(-1, 32)[3])


@pytest.mark.parametrize('name', ['full', 'masked', 'odd', 'oddlen', 'eos'])
def test_decode_fixtures_read_at_their_own_points(name, golden_dir):
    c, gold, img, mask = case(name, golden_dir)
    m = spot_model(c['wseed'], c['pt_eos_bias'], c['pt_seq_length'], c['rec_length'])
    m.encode(img, mask)
    (pt, poly, rec), _ = m.read_at([gold['pt'].reshape(-1, 2)])[0]
    assert np.array_equal(poly.numpy(), gold['poly']) and np.array_equal(rec.numpy(), gold['rec']), name


# ----------------------------------------------------------------------------------------------- round trip
EXTRAS = [dict(), dict(rec_candidates=5), dict(rec_beams=1), dict(rec_beams=4, length_penalty=0.5),
          dict(rec_locations=True)]
SETTINGS = [dict(joint_decode=1), dict(joint_decode=0), dict(decode_streams=1), dict(use_graphs=0)]


def round_trip(m, encode):
    """decode, then read_at at decode's points on the same encoded batch, with every extra: bit for bit"""
    for extra in EXTRAS:
        encode()
        dec = m._decode_arrays(**extra)
        lists = (m.last_rec_candidates, m.last_rec_beams, m.last_rec_locations)
        n, pt = dec[0], dec[1]
        assert n.sum() > 0
        got = m._read_at_arrays([pt[b, :n[b]] for b in range(len(n))], **extra)
        assert np.array_equal(got[0], n)
        for k, what in zip(range(1, 5), ('pt', 'poly', 'rec', 'prob')):
            assert_same(got[k], dec[k], f'{what} {extra}')
        assert_same((m.last_rec_candidates, m.last_rec_beams, m.last_rec_locations), lists, f'lists {extra}')
    m._set_rec_candidates(0)


@pytest.mark.parametrize('setting', SETTINGS, ids=lambda s: '-'.join(f'{k}{v}' for k, v in s.items()))
def test_decode_then_read_at_its_points_is_decode(setting, golden_dir):
    _, _, img0, mask0 = case('full', golden_dir)
    _, _, img1, mask1 = case('masked', golden_dir)
    img, mask = torch.cat([img0, img1, img0]), torch.cat([mask0, mask1, mask0])
    m = spot_model(0, -30.0, 8, 25)
    with options(m.ctx, **setting):
        round_trip(m, lambda: m.encode(img, mask))


def test_decode_then_read_at_on_pages_of_different_sizes():
    g = torch.Generator().manual_seed(31)
    t = torch.zeros(3, 3, 96, 128)
    sizes = [(96, 128), (64, 80), (72, 112)]
    for b, (h, w) in enumerate(sizes):
        t[b, :, :h, :w] = torch.randn(3, h, w, generator=g)
    m = spot_model(0, -30.0, 8, 25)
    round_trip(m, lambda: m.encode_pages(t, sizes))


# ----------------------------------------------------------------------------------------------- batch invariance
def test_a_page_read_alone_or_in_a_batch(golden_dir):
    _, gold, img, mask = case('full', golden_dir)
    m = spot_model(0, -30.0, 8, 25)
    maxi = 4
    rng = np.random.default_rng(3)
    pts = gold['pt'].reshape(-1, 2)                       # 4 points: Ncap 4 alone
    one = np.load(os.path.join(golden_dir, 'omni_points.npz'))['full_pts'][2:3]   # clear of near-ties on this page
    m.encode(img, mask)
    alone = m._read_at_arrays([pts])
    alone1 = m._read_at_arrays([one])
    m.encode(img.repeat(4, 1, 1, 1), mask.repeat(4, 1, 1))
    batch = m._read_at_arrays([pts, np.zeros((0, 2), int), one, rng.integers(0, 1000, (maxi, 2))])
    assert batch[0].tolist() == [4, 0, 1, maxi]
    for k in range(1, 4):   # ids of every page equal alone; the page with no points has no rows
        assert np.array_equal(batch[k][0], alone[k][0]) and np.array_equal(batch[k][2, :1], alone1[k][0, :1])
        assert not batch[k][1].any()
    assert np.array_equal(bits(batch[4][0]), bits(alone[4][0])), 'same Ncap: probabilities bit for bit'
    np.testing.assert_allclose(batch[4][2, :1], alone1[4][0, :1], rtol=5e-5, atol=0)


def test_more_points_than_max_instances_read_in_several_calls(golden_dir):
    _, _, img, mask = case('full', golden_dir)
    m = spot_model(0, -30.0, 8, 25)
    m.encode(img, mask)
    rng = np.random.default_rng(4)
    pts = rng.integers(0, 1000, (11, 2))
    n, pt, poly, rec, prob = m._read_at_arrays([pts], rec_candidates=2)
    assert n.tolist() == [11] and pt.shape[1] == 12 and m.last_rec_candidates[0].shape[1] == 12
    for i0 in range(0, 11, 4):
        part = m._read_at_arrays([pts[i0:i0 + 4]], rec_candidates=2)
        k = len(pts[i0:i0 + 4])
        assert np.array_equal(poly[0, i0:i0 + k], part[2][0, :k]) and np.array_equal(rec[0, i0:i0 + k], part[3][0, :k])
        assert np.array_equal(bits(prob[0, i0:i0 + k]), bits(part[4][0, :k]))


# ----------------------------------------------------------------------------------------------- refusals
def _decode_at(m, xy, count, cap, **cfg_over):
    import ctypes as C
    B = len(count)
    cfg = m._cfg(max(1, m.vocab.pt_seq_length // 2))
    for k, v in cfg_over.items():
        setattr(cfg, k, v)
    xy = np.ascontiguousarray(np.asarray(xy, np.int32).reshape(B, cap, 2))
    count = np.ascontiguousarray(count, np.int32)
    out = [np.zeros((B, cap, 32), np.int64), np.zeros((B, cap, m.vocab.rec_length), np.int64),
           np.zeros((B, cap, m.vocab.rec_length), np.float32)]
    return m.lib.alm_omni_decode_at(m.ctx.h, xy.ctypes.data, count.ctypes.data, cap, C.byref(cfg),
                                    *(a.ctypes.data for a in out))


def test_refusals_leave_the_context_usable(golden_dir):
    from advancedliteratemachinery_b200 import OmniParserB200, OmniVocab
    from tests.conftest import omni_sd
    _, gold, img, mask = case('full', golden_dir)
    pts = gold['pt'].reshape(-1, 2)
    fresh = OmniParserB200(omni_sd(0, -30.0), OmniVocab(pt_seq_length=8))
    try:
        assert _decode_at(fresh, np.zeros(8), [1], 4) == ERR_STATE, 'before encode'
        with pytest.raises(Exception):
            fresh.read_at([pts])
    finally:
        fresh.ctx.close()
    m = spot_model(0, -30.0, 8, 25)
    m.encode(img, mask)
    want = m._read_at_arrays([pts])
    good = np.zeros((1, 4, 2), np.int32)
    good[0, :4] = pts
    for what, args, kw in [('bin = num_bins', (np.full(8, 1000), [1], 4), {}),
                           ('negative bin', (np.full(8, -1), [1], 4), {}),
                           ('count > cap', (np.zeros(6), [4], 3), {}),
                           ('count < 0', (good, [-1], 4), {}),
                           ('count > max_instances', (np.zeros(16), [5], 8), {}),
                           ('cap 0', (np.zeros(0), [0], 0), {}),
                           ('poly_length', (good, [4], 4), dict(poly_length=31)),
                           ('vie_categories', (good, [4], 4), dict(vie_categories=4))]:
        rc = _decode_at(m, *args, **kw)
        assert rc == ERR_INVALID, (what, rc)
        assert_same(m._read_at_arrays([pts]), want, f'after refusing {what}')
    with options(m.ctx, kv_decoders=1):
        m.encode(img, mask)
        assert _decode_at(m, good, [4], 4) == ERR_STATE, 'kv_decoders < 3'
    m.encode(img, mask)
    assert_same(m._read_at_arrays([pts]), want, 'after refusing kv_decoders < 3')
    # candidates together with beams: refused by the setters, in Python and in the library
    with pytest.raises(ValueError):
        m.read_at([pts], rec_candidates=2, rec_beams=2)
    m.ctx.check(m.lib.alm_omni_set_rec_candidates(m.ctx.h, 2))
    assert m.lib.alm_omni_set_rec_beams(m.ctx.h, 2, 1.0) == ERR_INVALID
    m.ctx.check(m.lib.alm_omni_set_rec_candidates(m.ctx.h, 0))
    m._rec_k = 0
    for bad in ([pts + 1000], [pts.astype(float)], [pts[:, :1]], [pts, pts]):
        with pytest.raises(ValueError):
            m.read_at(bad)
    assert_same(m._read_at_arrays([pts]), want, 'after the ValueErrors')
    # a device slot given a host pointer
    from advancedliteratemachinery_b200 import preprocess as Pre
    page = np.zeros((64, 64, 3), np.uint8)
    keep, ptrs, hs, ws, n = Pre._image_args([page])
    idx = np.zeros(1, np.int32)
    host = np.zeros((1, 3, 64, 64), np.float32)
    hmask = np.zeros((1, 64, 64), np.uint8)
    assert m.lib.alm_pre_omni_tiles_at(m.ctx.h, ptrs, hs.ctypes.data, ws.ctypes.data, 1, 64, 0, idx.ctypes.data, 1, 64,
                                       64, host.ctypes.data, hmask.ctypes.data) == ERR_INVALID
    with pytest.raises(ValueError):
        Pre.omni_tiles_at(m.ctx, [page], [1], 64, 0, 64, 64)
    assert_same(m._read_at_arrays([pts]), want, 'after the tile refusals')


def test_kie_checkpoint_is_refused():
    from advancedliteratemachinery_b200 import OmniParserB200, OmniVocab
    from advancedliteratemachinery_b200 import synthetic as W
    from oracle.gen_golden import KIE_CASES, omni_inputs
    c = KIE_CASES['kie']
    m = OmniParserB200(W.omniparser_state_dict(seed=c['wseed'], vie_categories=c['vie'], pt_eos_bias=c['pt_eos_bias']),
                       OmniVocab(vie_categories=c['vie'], pt_seq_length=c['pt_seq_length']), workspace_mb=1024)
    try:
        img, mask = omni_inputs(c)
        m.encode(img, mask)
        assert _decode_at(m, np.zeros(8), [1], 4, vie_categories=c['vie']) == ERR_INVALID
        with pytest.raises(ValueError):
            m.read_at([np.zeros((1, 2), int)])
        with pytest.raises(ValueError):
            m.read_regions([np.zeros((64, 64, 3), np.uint8)], [[3, 3]], [0], kind='point')
        m.decode_kie([c['canvas']])   # still usable
    finally:
        m.ctx.close()


# ----------------------------------------------------------------------------------------------- read_regions
def tiles_fixture():
    gold = golden('omni_tiles.npz')
    return gold, omni_model(gold), kw(gold)


def check_regions(m, pages, regions, pi, kind, kw, max_batch=16):
    """read_regions against the rule: brute-force routing, each tile / whole page encoded alone and read_at at its
    points padded to the chunk's Ncap (ids equal; probabilities bit for bit when the chunk is that one image, else
    within 5e-5 relative), points and polygons by the merge arithmetic"""
    from advancedliteratemachinery_b200 import postprocess as P
    from advancedliteratemachinery_b200 import preprocess as Pre
    from advancedliteratemachinery_b200.omniparser import region_boxes, tile_to_page
    res = m.read_regions(pages, regions, pi, kind=kind, max_batch=max_batch, **kw)
    lr = m.last_regions
    sizes = [p.shape[:2] for p in pages]
    route = brute_route(sizes, lr['plan'], region_boxes(regions, kind), pi)
    assert np.array_equal(lr['route'], route)
    tiles = sorted(set(route[route >= 0].tolist()))
    encoded = [i for c in lr['chunks'] if c['kind'] == 'tile' for i in c['index'].tolist()]
    assert encoded == tiles, 'only the tiles holding a region are encoded'
    assert all(len(c['index']) <= max_batch for c in lr['chunks'])
    nb = m.vocab.num_bins
    for c in lr['chunks']:
        Ncap = int(c['n'].max())
        for j, i in enumerate(c['index'].tolist()):
            if c['kind'] == 'tile':
                y0, x0, h, w = (int(v) for v in lr['plan'][i, 1:])
                rows = np.nonzero(route == i)[0]
                nt = Pre.omni_tiles_at(m.ctx, pages, [i], **kw)
            else:
                (h, w), y0, x0 = sizes[i], 0, 0
                rows = np.nonzero((route < 0) & (np.asarray(pi) == i))[0]
                nt = Pre.omni_tiles(m.ctx, [pages[i]], max(64, max(h, w)), 0, kw['test_min_size'], kw['test_max_size'])
            m.encode(nt.tensors)
            local = P.point_bins(lr['points'][rows] - [x0, y0], (h, w), nb)
            k = len(rows)
            n, pt, poly, rec, prob = m._read_at_arrays([np.concatenate([local, local[-1:].repeat(Ncap - k, 0)])])
            assert np.array_equal(c['pt'][j, :k], pt[0, :k]) and np.array_equal(c['poly'][j, :k], poly[0, :k])
            assert np.array_equal(c['rec'][j, :k], rec[0, :k])
            if len(c['index']) == 1:   # the same batch shape: bit for bit
                assert np.array_equal(bits(c['prob'][j, :k]), bits(prob[0, :k]))
            else:                      # another batch shape moves the last bits (as for decode_dense)
                np.testing.assert_allclose(c['prob'][j, :k], prob[0, :k], rtol=5e-5, atol=0)
            for r, q in zip(rows, range(k)):
                d = res[r]
                assert d['page'] == int(pi[r])
                assert d['pts'] == [tile_to_page((y0, x0), (h, w), pt[0, q], nb)[0].tolist()]
                assert d['polys'] == tile_to_page((y0, x0), (h, w), poly[0, q].reshape(-1, 2), nb).tolist()
    return res


def test_read_regions_on_the_tiled_page():
    from advancedliteratemachinery_b200.omniparser import tile_to_page
    gold, m, kw = tiles_fixture()
    page = gold['page']
    words = m.spot_tiled([page], **kw)[0]
    mg, plan = m.last_tiles['merged'], m.last_tiles['plan']
    pts = np.array([w_['pts'][0] for w_ in words])
    res = check_regions(m, [page], pts, np.zeros(len(pts), int), 'point', kw)
    # a point of spot_tiled routed to the word's own tile reads the word: its ids, and the polygon the merge computed
    same = [r for r, w_ in enumerate(words) if w_['tile'] >= 0 and m.last_regions['route'][r] == w_['tile']]
    assert same, 'no word was routed to its source tile'
    for r in same:
        t = int(m.last_regions['route'][r])
        c = next(c for c in m.last_regions['chunks'] if c['kind'] == 'tile' and t in c['index'].tolist())
        j = c['index'].tolist().index(t)
        q = np.nonzero(m.last_regions['route'] == t)[0].tolist().index(r)
        assert np.array_equal(c['rec'][j, q], mg['rec'][r]), r
        if np.array_equal(c['poly'][j, q], m.last_tiles['poly'][mg['source'][r, 0], mg['source'][r, 1]]):
            assert res[r]['polys'] == mg['polys'][r].reshape(16, 2).tolist()
        assert res[r]['rec'] == words[r]['rec'] and res[r]['pts'] == words[r]['pts']
    # the same words as boxes and as their polygons; a region wider than the overlap across a seam is read whole
    polys = mg['polys'].reshape(-1, 16, 2)
    seam = np.array([[[40, 60], [200, 60], [200, 80], [40, 80]]], np.float64)
    quads = np.concatenate([polys[:, [0, 7, 8, 15]], seam])
    res = check_regions(m, [page], quads, np.zeros(len(quads), int), 'quad', kw, max_batch=2)
    assert res[-1]['tile'] == -1 and m.last_regions['chunks'][-1]['kind'] == 'whole'
    check_regions(m, [page], polys, np.zeros(len(polys), int), 'polygon', kw)


def test_read_regions_on_an_a4_page_with_candidates_and_beams():
    m = spot_model(0, -30.0, 12, 25)
    rng = np.random.default_rng(9)
    a4 = rng.integers(0, 256, (3508, 2480, 3), dtype=np.uint8)
    small = rng.integers(0, 256, (500, 700, 3), dtype=np.uint8)
    empty = np.zeros((1300, 900, 3), np.uint8)   # two tiles and no region, before a page with regions
    pages = [a4, empty, small]
    kw = dict(tile=1200, overlap=256, test_min_size=1200, test_max_size=1920)
    R = 40
    xy = rng.uniform([0, 0], [2480 - 400, 3508 - 60], (R, 2))   # every centre on the page
    wh = rng.uniform([30, 12], [400, 60], (R, 2))
    boxes = np.concatenate([xy, xy + wh], 1)
    boxes[R - 1] = [1100, 1500, 2200, 1540]   # across two column seams, in no tile: read whole
    pi = np.zeros(R + 3, int)
    pi[-3:] = 2
    boxes = np.concatenate([boxes, [[10, 10, 100, 40], [600, 450, 700, 500], [0, 0, 700, 500]]])
    res = check_regions(m, pages, boxes, pi, 'box', kw, max_batch=3)
    assert res[R - 1]['tile'] == -1 and all(r['tile'] == 0 for r in res[R:])
    for extra in (dict(rec_candidates=3), dict(rec_beams=2)):
        got = m.read_regions(pages, boxes, pi, kind='box', max_batch=3, **extra, **kw)
        if 'rec_candidates' in extra:   # candidate 0 is the greedy reading
            assert [g['rec'] for g in got] == [r['rec'] for r in res]
        lst = m.last_rec_candidates if 'rec_candidates' in extra else m.last_rec_beams
        assert lst[0].shape[0] == len(boxes)
        ids = lst[0][:, :, 0] if 'rec_candidates' in extra else lst[0][:, 0]
        recs = np.concatenate([c['rec'][j, :int(c['n'][j])] for c in m.last_regions['chunks'] for j in
                               range(len(c['index']))])
        order = np.concatenate([np.nonzero(m.last_regions['route'] == i)[0] if c['kind'] == 'tile' else
                                np.nonzero((m.last_regions['route'] < 0) & (pi == i))[0]
                                for c in m.last_regions['chunks'] for i in c['index'].tolist()])
        assert np.array_equal(ids[order], recs), extra
    m._set_rec_candidates(0)


def test_tiles_at_an_index_list_equal_the_range_entry():
    from advancedliteratemachinery_b200 import _lib, preprocess as P
    ctx = _lib.Context(0)
    try:
        rng = np.random.default_rng(2)
        pages = [rng.integers(0, 256, s + (3,), dtype=np.uint8) for s in ((3508, 2480), (900, 1500))]
        plan = P.omni_tile_plan([p.shape[:2] for p in pages], 1200, 256)
        for idx in ([2, 3, 4], [len(plan) - 1, 0, 5, 5], list(range(len(plan)))):
            got = P.omni_tiles_at(ctx, pages, idx, 1200, 256, 1200, 1920)
            for j, i in enumerate(idx):
                want = P.omni_tiles(ctx, pages, 1200, 256, 1200, 1920, i, 1)
                h, w = want.tensors.shape[2:]
                assert torch.equal(got.tensors[j, :, :h, :w].view(torch.int32), want.tensors[0].view(torch.int32))
                assert torch.equal(got.mask[j, :h, :w], want.mask[0]) and bool(got.mask[j, h:].all())
            if idx == [2, 3, 4]:
                want = P.omni_tiles(ctx, pages, 1200, 256, 1200, 1920, 2, 3)
                assert torch.equal(got.tensors.view(torch.int32), want.tensors.view(torch.int32))
    finally:
        ctx.close()
