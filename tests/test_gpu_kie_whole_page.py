"""GPU: KIE entities that cross tile seams, recovered from a whole-page KIE reading, and character boxes for every entity
word (OmniParserB200.kie_tiled(whole_page=True, rec_locations=True), alm_omni_merge_kie_whole_page; DESIGN 4.22).
kie_tiled(whole_page=True) on the fixture page must equal the oracle's merge of the unmodified reference's tile decodes
and whole-page probes (tests/golden/omni_kie_tiles.npz); the device merge must equal the host build of the same bodies
(tests/emu/kie_whole_page_emu.cpp) bit for bit in three launches; single-tile pages and 'auto' must add nothing but the
merge; character boxes must be the host rule's on the device's own locations; and the calls without the new options,
and refused calls, must leave everything as it was."""

import ctypes as C

import numpy as np
import pytest
import torch

from oracle import kie_whole_page_ref as KW
from oracle import page_turn_ref as PT
from oracle import rec_box_ref as RB
from tests.support import assert_same, golden, kw, omni_model, release_models  # noqa: F401
from tests.test_kie_tiles_cpu import emu_merge, fabricate
from tests.test_kie_whole_page_cpu import emu_whole, fabricate_whole

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

RAW = ('n_tok', 'tokens', 'probs', 'n_inst', 'inst_pos', 'poly')
MERGE_LAUNCHES = 3


def whole_of(arrays):
    """kie_tiled's whole-page decode arrays (``_decode_kie_arrays``' order) -> the RAW dict of the merge."""
    n_inst, pos, poly, _, _, n_tok, toks, tprob = arrays[:8]
    return dict(n_tok=n_tok, tokens=toks, probs=tprob, n_inst=n_inst, inst_pos=pos, poly=poly)


def probe(g, k):
    return {n: g['probe_' + n][k:k + 1] for n in RAW}


def oracle_entities(m, sizes, g, tiles, whole, wrec, turns=None):
    """The oracle's merge -> the reference's entity tuples, each word's text from its rec row (tile: the tile decode's
    rec; whole: wrec [P, max_inst, L])."""
    v = m.vocab
    ref = KW.merge(sizes, turns, int(g['tile']), int(g['overlap']), 4.0, v.num_bins, int(g['class_base']),
                   v.vie_categories, tiles, whole)
    out = []
    for p in range(len(sizes)):
        ents = []
        for r in range(int(ref['offset'][p]), int(ref['offset'][p]) + int(ref['count'][p])):
            ws = range(int(ref['word_offset'][r]), int(ref['word_offset'][r]) + int(ref['word_count'][r]))
            text = ' '.join(m._kie_word(m.last_tiles['rec'][t, i] if t >= 0 else wrec[p, i])
                            for t, i in ref['word_source'][ws].tolist())
            ents.append((text, v.classes[int(ref['cls'][r])], float(ref['prob'][r]), ref['rect'][ws].tolist()))
        out.append(ents)
    return out, ref


def same_entities(a, b, rtol=0.0):
    assert [(e[0], e[1], e[3]) for e in a] == [(e[0], e[1], e[3]) for e in b]
    np.testing.assert_allclose([e[2] for e in a], [e[2] for e in b], rtol=rtol)


def test_fixture_page_equals_reference_merge():
    """Texts, classes and rects exact, probabilities within 2e-3: the oracle's merge of the reference's tile decodes
    and its whole-page probe at turn 0.  The whole reading is the reference's probe token for token, the device merge
    equals the host build bit for bit, a whole entity is kept and a tile entity dropped."""
    g = golden('omni_kie_tiles.npz')
    m = omni_model(g, kie=True)
    page = g['page']
    sizes = [page.shape[:2]]
    got = m.kie_tiled([page], whole_page=True, **kw(g))
    t = m.last_tiles
    w = whole_of(t['whole'])
    n = int(g['probe_n_tok'][0])
    assert int(w['n_tok'][0]) == n and np.array_equal(w['tokens'][0, :n], g['probe_tokens'][0, :n])
    ni = int(g['probe_n_inst'][0])
    assert np.array_equal(w['poly'][0, :ni], g['probe_poly'][0, :ni])
    ref_tiles = emu_merge(sizes, int(g['tile']), int(g['overlap']), {k: g[k] for k in RAW},
                          class_base=int(g['class_base']))
    exp, ref = oracle_entities(m, sizes, g, ref_tiles, probe(g, 0), g['probe_rec'][0:1])
    same_entities(got[0], exp[0], rtol=2e-3)
    assert (ref['source'][:, 0] < 0).any() and (ref['source'][:, 0] >= 0).sum() < len(ref_tiles['cls'])
    emu = emu_whole(sizes, int(g['tile']), int(g['overlap']), t['merged'], w, class_base=int(g['class_base']))
    assert_same(t['whole_merge'], emu)


def test_turns_equal_the_oracle():
    """Explicit turns 1..3: the whole reading is the reference's probe at that turn, and the result is the oracle's
    merge of the device's own tile merge and that probe."""
    g = golden('omni_kie_tiles.npz')
    m = omni_model(g, kie=True)
    page = g['page']
    sizes = [page.shape[:2]]
    for k in (1, 2, 3):
        got = m.kie_tiled([page], orientation=[k], whole_page=True, **kw(g))
        t = m.last_tiles
        w = whole_of(t['whole'])
        n = int(g['probe_n_tok'][k])
        assert np.array_equal(w['tokens'][0, :n], g['probe_tokens'][k, :n])
        exp, _ = oracle_entities(m, sizes, g, t['merged'], probe(g, k), g['probe_rec'][k:k + 1], turns=[k])
        same_entities(got[0], exp[0], rtol=2e-3)


def test_single_tile_pages_add_nothing():
    """Pages that fit in one tile: whole_page=True returns what whole_page=False returns, with the same launches."""
    g = golden('omni_kie_tiles.npz')
    m = omni_model(g, kie=True)
    pages = [np.ascontiguousarray(g['page'][:100, :90]), np.ascontiguousarray(g['page'][:120, :128])]
    n0 = m.ctx.launch_count()
    off = m.kie_tiled(pages, **kw(g))
    n1 = m.ctx.launch_count()
    on = m.kie_tiled(pages, whole_page=True, **kw(g))
    assert on == off and m.ctx.launch_count() - n1 == n1 - n0
    assert 'whole' not in m.last_tiles


def test_auto_adds_only_the_merge():
    """'auto' reuses its probe at the chosen turn as the whole reading: the merge's launches are the only extra ones,
    and the result is the oracle's merge of the reference's probe."""
    g = golden('omni_kie_tiles.npz')
    m = omni_model(g, kie=True)
    page = g['page']
    n0 = m.ctx.launch_count()
    off = m.kie_tiled([page], orientation='auto', **kw(g))
    n1 = m.ctx.launch_count()
    on = m.kie_tiled([page], orientation='auto', whole_page=True, **kw(g))
    assert m.ctx.launch_count() - n1 == n1 - n0 + MERGE_LAUNCHES
    t = m.last_tiles
    k = int(g['probe_turn'][0])
    assert t['turns'].tolist() == [k] and off != on
    exp, _ = oracle_entities(m, [page.shape[:2]], g, t['merged'], probe(g, k), g['probe_rec'][k:k + 1], turns=[k])
    same_entities(on[0], exp[0], rtol=2e-3)


def test_max_batch_gives_the_same_entities():
    g = golden('omni_kie_tiles.npz')
    m = omni_model(g, kie=True)
    pages = [g['page'], np.ascontiguousarray(g['page'][:100, :90]), np.ascontiguousarray(np.rot90(g['page'], 1))]
    ref = m.kie_tiled(pages, max_batch=1, whole_page=True, rec_locations=True, **kw(g))
    for b in (5, 16):
        got = m.kie_tiled(pages, max_batch=b, whole_page=True, rec_locations=True, **kw(g))
        assert [[e[:4] for e in p] for p in got] == [[e[:4] for e in p] for p in ref]
        for p, q in zip(got, ref):
            for e, f in zip(p, q):
                for a, b_ in zip(e[4], f[4]):
                    assert len(a) == len(b_) and all(x['char'] == y['char'] and np.array_equal(x['box'], y['box'])
                                                     for x, y in zip(a, b_))


def test_merge_at_scale_equals_host_build():
    """16 A4 pages at 300 dpi x 12 tiles of fabricated tile entities and whole readings (1..8 words, wordless ones,
    some pages turned): the device merge equals the host build bit for bit, in three launches."""
    from advancedliteratemachinery_b200.omniparser import merge_kie_tiles, merge_kie_whole_page
    g = golden('omni_kie_tiles.npz')
    m = omni_model(g, kie=True)
    rng = np.random.default_rng(12)
    sizes = [(3508, 2480)] * 16
    turns = [0] * 8 + [1, 2, 3, 0, 1, 2, 3, 0]
    raw = fabricate(rng, sizes, 1200, 256, turns, n_ent=60, max_tok=1024, max_inst=400)
    plan = PT.plan(sizes, turns, 1200, 256)
    assert len(plan) == 16 * 12
    tiles = merge_kie_tiles(m.ctx, sizes, 1200, 256, plan, *[raw[k] for k in RAW], 1000, 1104, 4, turns=turns)
    whole = fabricate_whole(rng, sizes, 1200, 256, turns, n_ent=200)
    n0 = m.ctx.launch_count()
    dev = merge_kie_whole_page(m.ctx, sizes, 1200, 256, tiles, *[whole[k] for k in RAW], 1000, 1104, 4, turns=turns)
    assert m.ctx.launch_count() == n0 + MERGE_LAUNCHES
    assert_same(dev, emu_whole(sizes, 1200, 256, tiles, whole, turns=turns))
    assert (dev['source'][:, 0] < 0).any() and (dev['source'][:, 0] >= 0).sum() < len(tiles['cls'])


def chars_equal(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert x['char'] == y['char']
        for k in ('centre', 'cov', 'box'):
            assert np.array_equal(x[k], y[k], equal_nan=True), k


def test_one_tile_page_chars_are_rec_char_boxes():
    """On a page that fits in one tile every word's chars are postprocess.rec_char_boxes on decode_kie(
    rec_locations=True)'s own outputs, and the entities are decode_kie's.  Characters exact; centres, covariances and
    boxes within 1e-4 px: the entity words' polygons are decode_pred_seq's float32 coordinates, where rec_char_boxes
    scales the bins in double."""
    from advancedliteratemachinery_b200 import postprocess
    from advancedliteratemachinery_b200 import preprocess as P
    g = golden('omni_kie_tiles.npz')
    m = omni_model(g, kie=True)
    page = np.ascontiguousarray(g['page'][:100, :90])
    got = m.kie_tiled([page], rec_locations=True, **kw(g))[0]
    inst = m.last_tiles['merged']['word_source'][:, 1].tolist()   # each entity word's instance
    assert got and [e[:4] for e in got] == m.kie_tiled([page], **kw(g))[0]
    v = m.vocab
    nt = P.omni_pages(m.ctx, [page], int(g['test_min_size']), int(g['test_max_size']))
    seqs = [v.pt_prompt(), torch.tensor([[v.poly_sos_index]]), torch.tensor([[v.rec_sos_index]]),
            torch.tensor([[100, 90]])]
    exp = m.forward_pages(nt, seqs, rec_locations=True)[0]
    raw, loc = m.last_kie_raw, m.last_rec_locations
    assert [e[:4] for e in got] == exp
    n = int(raw['n_inst'][0])
    want = postprocess.rec_char_boxes(raw['poly'][0, :n], raw['rec'][0, :n], loc[0, :n], (100, 90), m.vocab)
    words = [w for e in got for w in e[4]]
    assert len(words) == len(inst) > 0 and max(inst) < n
    for a, i in zip(words, inst):
        assert [c['char'] for c in a] == [c['char'] for c in want[i]] and a
        for x, y in zip(a, want[i]):
            for k in ('centre', 'cov', 'box'):
                np.testing.assert_allclose(x[k], y[k], rtol=0, atol=1e-4, err_msg=k)


@pytest.mark.parametrize('orientation', ['upright', [1], [3], 'auto'])
def test_tiled_chars_are_the_host_rule_on_the_device_locations(orientation):
    """Tiled and turned pages, with and without whole_page: every word's chars are the host rule (oracle/rec_box_ref)
    fed the device's own locations, tile words in their tile's frame and whole-page words in the page read whole; the
    entities are those without locations."""
    g = golden('omni_kie_tiles.npz')
    m = omni_model(g, kie=True)
    v = m.vocab
    page = g['page']
    H, W = page.shape[:2]
    for whole_page in (False, True):
        base = m.kie_tiled([page], orientation=orientation, whole_page=whole_page, **kw(g))[0]
        got = m.kie_tiled([page], orientation=orientation, whole_page=whole_page, rec_locations=True, **kw(g))[0]
        assert [e[:4] for e in got] == base
        t = m.last_tiles
        mg = t['whole_merge'] if whole_page else t['merged']
        turn = 0 if orientation == 'upright' else int(t['turns'][0])
        th, tw = PT.turned_size(H, W, turn)
        plan = t['plan']
        frames = [(H, W, turn, y0, x0, h, w) for _, y0, x0, h, w in plan.tolist()] + [(H, W, turn, 0, 0, th, tw)]
        src = mg['word_source'].astype(np.int64)
        tile = src[:, 0] >= 0
        rec = np.where(tile[:, None], t['rec'][src[:, 0].clip(0), src[:, 1]],
                       t['whole'][3][0, src[:, 1]] if whole_page else 0)
        loc = np.where(tile[:, None, None], t['loc'][src[:, 0].clip(0), src[:, 1]],
                       t['whole'][8][0, src[:, 1]] if whole_page else 0)
        fi = np.where(tile, src[:, 0], len(plan))
        from advancedliteratemachinery_b200.omniparser import char_dicts
        want = char_dicts(RB.char_boxes(mg['poly'], rec, loc, fi, frames, v.recog_pad_index, v.rec_eos_index), rec, v)
        words = [w for e in got for w in e[4]]
        assert len(words) == len(want) and (not whole_page or (~tile).any())
        for a, b in zip(words, want):
            chars_equal(a, b)


def test_other_calls_unchanged_and_errors_leave_the_context_usable():
    """kie_tiled, spot_tiled and decode_kie without the new options give what they gave before a call that used them;
    refused calls (candidates, beams, 'mixed', a spotting checkpoint, bad C-entry arguments) change nothing."""
    from advancedliteratemachinery_b200 import AlmError, OmniParserB200, OmniVocab
    from advancedliteratemachinery_b200 import preprocess as P
    from advancedliteratemachinery_b200.omniparser import merge_kie_whole_page
    from tests.conftest import omni_sd
    g = golden('omni_kie_tiles.npz')
    m = omni_model(g, kie=True)
    page = g['page']
    small = np.ascontiguousarray(page[:100, :90])
    v = m.vocab
    seqs = [v.pt_prompt(), torch.tensor([[v.poly_sos_index]]), torch.tensor([[v.rec_sos_index]]),
            torch.tensor([[100, 90]])]

    def fwd():
        return m.forward_pages(P.omni_pages(m.ctx, [small], int(g['test_min_size']), int(g['test_max_size'])), seqs)

    before, tiled = fwd(), m.kie_tiled([page], **kw(g))
    m.kie_tiled([page], whole_page=True, rec_locations=True, orientation='auto', **kw(g))
    t = m.last_tiles
    tiles, whole = t['merged'], whole_of(t['whole'])
    T, ov = int(g['tile']), int(g['overlap'])
    sz = [page.shape[:2]]
    args = [whole[k] for k in RAW]
    for bad in (dict(rec_candidates=2), dict(rec_beams=2), dict(orientation='mixed')):
        with pytest.raises(ValueError):
            m.kie_tiled([page], whole_page=True, **bad, **kw(g))
    with pytest.raises(AlmError):
        merge_kie_whole_page(m.ctx, sz, 63, 0, tiles, *args, 1000, int(g['class_base']), 4)
    bad = {k: a.copy() for k, a in whole.items()}
    bad['inst_pos'][0, 0] += 1
    with pytest.raises(AlmError):
        merge_kie_whole_page(m.ctx, sz, T, ov, tiles, *[bad[k] for k in RAW], 1000, int(g['class_base']), 4)
    bad = {k: a.copy() for k, a in whole.items()}
    bad['tokens'][0, 2] = int(g['class_base']) + 4
    with pytest.raises(AlmError):
        merge_kie_whole_page(m.ctx, sz, T, ov, tiles, *[bad[k] for k in RAW], 1000, int(g['class_base']), 4)
    tb = dict(tiles, word_offset=tiles['word_offset'] + 1)
    with pytest.raises(AlmError):
        merge_kie_whole_page(m.ctx, sz, T, ov, tb, *args, 1000, int(g['class_base']), 4)
    # a capacity below the entities: the entry itself, with cap_ent 0
    hs, ws = np.array([sz[0][0]], np.int32), np.array([sz[0][1]], np.int32)
    tt = {k: np.ascontiguousarray(a) for k, a in tiles.items()}
    w = {k: np.ascontiguousarray(a) for k, a in whole.items()}
    outs = [np.zeros(256, np.int32) for _ in range(7)]
    rc = m.lib.alm_omni_merge_kie_whole_page(
        m.ctx.h, hs.ctypes.data, ws.ctypes.data, 1, None, T, ov, 4.0, 1000, int(g['class_base']), 4,
        *[tt[k].ctypes.data for k in ('count', 'offset', 'cls', 'prob', 'word_offset', 'word_count', 'source', 'rect',
                                      'poly', 'word_source')],
        w['n_tok'].ctypes.data, w['tokens'].ctypes.data, w['probs'].ctypes.data, w['tokens'].shape[1],
        w['n_inst'].ctypes.data, w['inst_pos'].ctypes.data, w['poly'].ctypes.data, w['inst_pos'].shape[1],
        *[o.ctypes.data for o in outs], C.c_long(0), np.zeros((256, 4)).ctypes.data, np.zeros((256, 32)).ctypes.data,
        np.zeros((256, 2), np.int32).ctypes.data, C.c_long(256))
    assert rc != 0
    assert fwd() == before
    assert m.kie_tiled([page], **kw(g)) == tiled
    # a spotting checkpoint is refused; its spot_tiled is unchanged by a KIE model's calls
    tg = golden('omni_tiles.npz')
    s = OmniParserB200(omni_sd(int(tg['wseed']), float(tg['pt_eos_bias'])),
                       OmniVocab(pt_seq_length=int(tg['pt_seq_length']), rec_length=int(tg['rec_length'])),
                       workspace_mb=4096)
    try:
        tkw = kw(tg)
        spot = s.spot_tiled([tg['page']], **tkw)
        spot_whole = s.spot_tiled([tg['page']], whole_page=True, **tkw)
        with pytest.raises(ValueError):
            s.kie_tiled([tg['page']], whole_page=True, **tkw)
        assert s.spot_tiled([tg['page']], **tkw) == spot
        assert s.spot_tiled([tg['page']], whole_page=True, **tkw) == spot_whole
    finally:
        s.ctx.close()
