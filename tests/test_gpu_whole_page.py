"""GPU: words that cross tile seams, recovered from a whole-page reading (DESIGN 4.17; alm_omni_merge_whole_page,
OmniParserB200.spot_tiled(whole_page=True)).  On the fixture page spot_tiled equals tests/golden/omni_whole_page.npz
(the unmodified reference on every tile and on the whole page, merged by oracle/tile_ref.py and
oracle/whole_page_ref.py); the device merge equals the host build of the same bodies (tests/emu/whole_page_emu.cpp) bit
for bit, on the device's own readings and on 16 pages x 12 tiles of fabricated rows; every orientation mode, chunk size
and page kind agrees with the rule."""
import numpy as np
import pytest
import torch

from oracle import turn_merge_ref as TM
from oracle import whole_page_ref as WP
from tests import support
from tests.support import assert_same, golden, omni_model, release_models, same
from tests.test_whole_page_cpu import band_poly, emu_merge

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

ERR_INVALID = -1  # include/alm_ocr.h ALM_ERR_INVALID


def fixture():
    """The fixture, with its page: omni_tiles.npz's (the same page seed)."""
    g = dict(golden('omni_whole_page.npz'))
    t = golden('omni_tiles.npz')
    assert int(g['seed']) == int(t['seed'])
    g['page'] = t['page']
    return g


def kw(gold, **extra):
    return support.kw(gold, margin=float(gold['margin']), **extra)


def pages(gold):
    """The fixture page (larger than T), a page of 2 x 3 tiles and one smaller than a tile."""
    rng = np.random.default_rng(21)
    return [gold['page'], rng.integers(0, 256, (230, 301, 3), dtype=np.uint8),
            rng.integers(0, 256, (97, 120, 3), dtype=np.uint8)]


def emu_of(m, sizes, turns, gold, tiles, whole):
    return emu_merge(sizes, turns, int(gold['tile']), int(gold['overlap']), float(gold['margin']), m.vocab.num_bins,
                     tiles, *whole)


def oracle_of(m, sizes, turns, gold, tiles, whole):
    return WP.merge(sizes, turns, int(gold['tile']), int(gold['overlap']), float(gold['margin']), m.vocab.num_bins,
                    tiles, *whole)


def test_spot_tiled_equals_the_fixture():
    """ids exact, coordinates exact, probabilities close; the merge equals the emulation fed the device's own
    readings in every field."""
    gold = fixture()
    m = omni_model(gold)
    page = gold['page']
    size = page.shape[:2]
    got = m.spot_tiled([page], whole_page=True, **kw(gold))[0]
    t = m.last_tiles
    for k in ('n_inst', 'pt', 'poly', 'rec'):
        assert np.array_equal(t[k], gold[k]), k
    np.testing.assert_allclose(t['prob'], gold['prob'], rtol=1e-5, atol=1e-6)
    n, pt, poly, rec, prob = t['whole']
    wn = int(gold['whole_n_inst'][0])
    assert n.tolist() == [wn]
    for a, k in ((pt, 'whole_pt'), (poly, 'whole_poly'), (rec, 'whole_rec')):
        assert np.array_equal(a[0, :wn], gold[k][0, :wn]), k
    np.testing.assert_allclose(prob[0, :wn], gold['whole_prob'][0, :wn], rtol=1e-5, atol=1e-6)
    wm = t['whole_merge']
    for k in ('count', 'offset', 'pts', 'polys', 'rec', 'source'):
        assert np.array_equal(wm[k], gold[f'merged_{k}']), k
    assert_same(wm, emu_of(m, [size], None, gold, t['merged'], t['whole']))
    assert len(got) == int(wm['count'][0]) and [d['tile'] for d in got].count(-1) >= 1
    for d, (tl, i), pts in zip(got, wm['source'], wm['pts']):
        assert d['instance'] == i and d['pts'] == [pts.tolist()] and (d['tile'] == -1) == (tl < 0)


def large_input(rng, P=16, n=4096, w=509, L=25, num_bins=1000):
    """P A4 pages (3 x 4 tiles of 1200 / 256), n tile rows and w whole rows per page: whole words of every width,
    tile points scattered and on the whole words."""
    sizes = [(3508, 2480)] * P
    turns = rng.integers(0, 4, P).astype(np.int32)
    pt = rng.integers(0, num_bins, (P, w, 2))
    x0 = rng.integers(0, num_bins - 20, (P, w))
    y0 = rng.integers(0, num_bins - 10, (P, w))
    wd = np.minimum(num_bins - 1 - x0, rng.choice([5, 50, 200], (P, w)))
    ht = np.minimum(num_bins - 1 - y0, rng.choice([4, 20], (P, w)))
    xs = np.concatenate([np.linspace(0, 1, 8), np.linspace(1, 0, 8)])
    poly = np.zeros((P, w, 32), np.int64)
    poly[..., 0::2] = np.round(x0[..., None] + wd[..., None] * xs)
    poly[..., 1::2] = np.round(y0[..., None] + ht[..., None] * np.repeat([0.0, 1.0], 8))
    pts = rng.uniform(0, 2480, (P * n, 2))
    pts[:, 1] = rng.uniform(0, 3508, P * n)
    polys = band_poly(-5, -3, 5, 3)[None] + np.tile(pts, 16)  # a 10 x 6 word around every point
    whole = (np.full(P, w, np.int32), pt, poly, rng.integers(0, 1100, (P, w, L)),
             rng.random((P, w, L)).astype(np.float32))
    count = np.full(P, n, np.int32)
    tiles = dict(count=count, offset=(np.cumsum(count) - count).astype(np.int32), pts=pts, polys=polys,
                 rec=rng.integers(0, 1100, (P * n, L)), prob=rng.random((P * n, L)).astype(np.float32),
                 source=rng.integers(0, 12, (P * n, 2)).astype(np.int32))
    return sizes, turns, tiles, whole


def test_device_merge_equals_the_emulation_at_16_pages_x_12_tiles():
    from advancedliteratemachinery_b200.omniparser import merge_whole_page
    gold = fixture()
    m = omni_model(gold)
    sizes, turns, tiles, whole = large_input(np.random.default_rng(7))
    m.ctx.launch_count(reset=True)
    got = merge_whole_page(m.ctx, sizes, 1200, 256, tiles, *whole, 1000, 4.0, turns=turns)
    assert m.ctx.launch_count() == 3
    want = emu_merge(sizes, turns, 1200, 256, 4.0, 1000, tiles, *whole)
    assert_same(got, want)
    kept_whole = int((got['source'][:, 0] < 0).sum())
    assert 0 < kept_whole < int(whole[0].sum()) and int(got['count'].sum()) - kept_whole < int(tiles['count'].sum())


def test_single_tile_pages_are_not_read_again():
    gold = fixture()
    m = omni_model(gold)
    pg = [pages(gold)[2], gold['page'][:100, :110]]
    m.ctx.launch_count(reset=True)
    want = m.spot_tiled(pg, **kw(gold))
    launches = m.ctx.launch_count(reset=True)
    got = m.spot_tiled(pg, whole_page=True, **kw(gold))
    assert m.ctx.launch_count() == launches
    same(got, want)
    assert 'whole' not in m.last_tiles


def test_auto_reuses_its_probe():
    """'auto': the whole-page reading is the probe at the chosen turn; only the merge's three launches are added."""
    gold = fixture()
    m = omni_model(gold)
    pg = pages(gold)
    m.ctx.launch_count(reset=True)
    m.spot_tiled(pg, orientation='auto', **kw(gold))
    launches = m.ctx.launch_count(reset=True)
    tiles_only = m.last_tiles
    got = m.spot_tiled(pg, orientation='auto', whole_page=True, **kw(gold))
    assert m.ctx.launch_count() == launches + 3
    t = m.last_tiles
    r = 4 * np.arange(len(pg)) + t['turns']
    for a, b in zip(t['whole'], t['probe']):
        assert np.array_equal(a, b[r])
    assert_same(t['merged'], tiles_only['merged'])
    sizes = [p.shape[:2] for p in pg]
    assert_same(t['whole_merge'], oracle_of(m, sizes, t['turns'], gold, t['merged'], t['whole']))
    assert len(got) == len(pg)


@pytest.mark.parametrize('k', [1, 2, 3])
def test_explicit_turns_read_the_fixture(k):
    """The page np.rot90(page, -k) read at turn k is the fixture page: the whole-page reading is the reference's, and
    the merge is the oracle's on the device's readings, in the turned page's pixels."""
    gold = fixture()
    m = omni_model(gold)
    page = np.ascontiguousarray(np.rot90(gold['page'], -k))
    m.spot_tiled([page], orientation=[k], whole_page=True, **kw(gold))
    t = m.last_tiles
    wn = int(gold['whole_n_inst'][0])
    assert t['whole'][0].tolist() == [wn]
    for a, g in zip(t['whole'][1:4], ('whole_pt', 'whole_poly', 'whole_rec')):
        assert np.array_equal(a[0, :wn], gold[g][0, :wn]), g
    for f in ('count', 'source'):
        assert np.array_equal(t['whole_merge'][f], gold[f'merged_{f}']), f
    assert_same(t['whole_merge'], oracle_of(m, [page.shape[:2]], [k], gold, t['merged'], t['whole']))


def test_mixed_on_the_fixture():
    """Each of the four readings is merged with its own whole-page partner (reading 0 is the fixture's), then
    merge_turns runs on the result."""
    gold = fixture()
    m = omni_model(gold)
    v = m.vocab
    page = gold['page']
    got = m.spot_tiled([page], orientation='mixed', whole_page=True, **kw(gold))[0]
    t = m.last_tiles
    wn = int(gold['whole_n_inst'][0])
    assert t['whole'][0][0] == wn and np.array_equal(t['whole'][2][0, :wn], gold['whole_poly'][0, :wn])
    sizes4 = [page.shape[:2]] * 4
    wm = t['whole_merge']
    assert_same(wm, oracle_of(m, sizes4, [0, 1, 2, 3], gold, t['readings'], t['whole']))
    for f in ('count', 'source'):
        assert np.array_equal(wm[f][:1] if f == 'count' else wm[f][:int(wm['count'][0])], gold[f'merged_{f}']), f
    assert_same(t['turn_merge'], TM.merge(wm['count'], wm['offset'], wm['pts'], wm['polys'], wm['rec'], wm['prob'],
                                          v.recog_pad_index, v.rec_eos_index))
    assert len(got) == int(t['turn_merge']['count'][0])


def test_a_saturated_whole_page_does_not_raise():
    gold = fixture()
    m = omni_model(gold)
    keep = m.vocab.pt_seq_length
    m.vocab.pt_seq_length = 2
    try:
        res = m.spot_tiled(pages(gold), whole_page=True, **kw(gold))
        assert m.last_dense.saturated.any() and len(res) == 3
    finally:
        m.vocab.pt_seq_length = keep


def test_chunk_sizes_agree_and_later_calls_are_unchanged():
    gold = fixture()
    m = omni_model(gold)
    pg = pages(gold)
    before = [m.spot_tiled(pg, **kw(gold)), m.spot_tiled(pg, orientation=[1, 0, 3], **kw(gold))]
    m.encode_pages(*_encoded(m, pg[1]))
    dec = m.decode()
    base = m.spot_tiled(pg, max_batch=5, whole_page=True, **kw(gold))
    assert any(d['tile'] == -1 for d in base[0])
    same(m.spot_tiled(pg, max_batch=1, whole_page=True, **kw(gold)), base)
    big = m.spot_tiled(pg, max_batch=16, whole_page=True, **kw(gold))
    drop = lambda res: [[{k: x for k, x in d.items() if k != 'score'} for d in r] for r in res]
    same(drop(big), drop(base))
    np.testing.assert_allclose([d['score'] for r in big for d in r], [d['score'] for r in base for d in r],
                               rtol=1e-5, atol=0)
    same(m.spot_tiled(pg, **kw(gold)), before[0])
    same(m.spot_tiled(pg, orientation=[1, 0, 3], **kw(gold)), before[1])
    m.encode_pages(*_encoded(m, pg[1]))
    after = m.decode()
    assert len(after) == len(dec)
    for a, b in zip(after, dec):
        assert (a is None) == (b is None)
        if a is not None:
            for x, y in zip(a[0], b[0]):
                assert torch.equal(x, y)


def _encoded(m, page):
    from advancedliteratemachinery_b200 import preprocess as P
    nt = P.omni_pages(m.ctx, [page], 128, 256)
    return nt.tensors, P.omni_plan([page.shape[:2]], 128, 256)[0]


def test_group_lines_takes_the_result_as_it_is():
    gold = fixture()
    m = omni_model(gold)
    res = m.spot_tiled(pages(gold), whole_page=True, **kw(gold))
    for r, ls in zip(res, m.group_lines(res)):
        assert sorted(w for line in ls for w in line['words']) == list(range(len(r)))


def test_error_paths_leave_the_context_usable():
    from advancedliteratemachinery_b200.omniparser import merge_whole_page
    gold = fixture()
    m = omni_model(gold)
    lib, h = m.ctx.lib, m.ctx.h
    sizes, turns, tiles, whole = large_input(np.random.default_rng(3), P=2, n=200, w=30)
    hs = np.array([s[0] for s in sizes], np.int32)
    ws = np.array([s[1] for s in sizes], np.int32)
    t = {k: np.ascontiguousarray(tiles[k]) for k in ('count', 'offset', 'pts', 'polys', 'rec', 'prob', 'source')}
    t['rec'] = t['rec'].astype(np.int64)
    n_inst, pt, poly, rec, prob = (np.ascontiguousarray(a) for a in whole)
    pt, poly, rec = (a.astype(np.int64) for a in (pt, poly, rec))
    N, L, cap_in = t['pts'].shape[0], t['rec'].shape[1], pt.shape[1]
    K = N + int(n_inst.sum())
    out = [np.zeros(2, np.int32), np.zeros(2, np.int32), np.zeros((K, 2)), np.zeros((K, 32)),
           np.zeros((K, L), np.int64), np.zeros((K, L), np.float32), np.zeros((K, 2), np.int32)]

    def call(T=1200, ov=256, margin=4.0, tr=turns, cnt=None, off=None, n=None, cap=K, null=None):
        ins = [(cnt if cnt is not None else t['count']).ctypes.data,
               (off if off is not None else t['offset']).ctypes.data] + \
              [t[k].ctypes.data for k in ('pts', 'polys', 'rec', 'prob', 'source')] + \
              [(n if n is not None else n_inst).ctypes.data] + [a.ctypes.data for a in (pt, poly, rec, prob)]
        outs = [o.ctypes.data for o in out]
        if null is not None:
            if null < len(ins):
                ins[null] = None
            else:
                outs[null - len(ins)] = None
        return lib.alm_omni_merge_whole_page(h, hs.ctypes.data, ws.ctypes.data, 2,
                                             None if tr is None else tr.ctypes.data, T, ov, margin, 1000, *ins,
                                             cap_in, L, *outs, cap)

    assert call() == 0 and call(tr=None) == 0
    for bad in (dict(T=32), dict(ov=700), dict(ov=-1), dict(margin=-1.0), dict(margin=float('nan')),
                dict(margin=float('inf')), dict(tr=np.array([0, 4], np.int32)), dict(tr=np.array([-1, 0], np.int32)),
                dict(cnt=np.array([200, -1], np.int32)), dict(off=np.array([0, 199], np.int32)),
                dict(off=np.array([1, 200], np.int32)), dict(n=np.array([30, 31], np.int32)),
                dict(n=np.array([-1, 30], np.int32)), dict(cap=K - 1)):
        assert call(**bad) == ERR_INVALID, bad
    for slot in range(19):
        assert call(null=slot) == ERR_INVALID, slot
    assert_same(merge_whole_page(m.ctx, sizes, 1200, 256, tiles, *whole, 1000, 4.0, turns=turns),
                emu_merge(sizes, turns, 1200, 256, 4.0, 1000, tiles, *whole))
