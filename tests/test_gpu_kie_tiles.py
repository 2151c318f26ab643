"""GPU: KIE on pages larger than the model's input and on turned pages (OmniParserB200.kie_tiled,
alm_omni_merge_kie_tiles; DESIGN 4.18).  kie_tiled on the fixture page must equal the oracle's merge of the unmodified
reference's per-tile outputs (tests/golden/omni_kie_tiles.npz); a one-tile page must give decode_kie's list; explicit
turns must give the reading of np.rot90(page, k) mapped back; 'auto' must pick the reference probes' turn; the device
merge must equal the host build of the same bodies (tests/emu/kie_tile_emu.cpp) bit for bit; and refused calls leave
the context and every other decode unchanged."""

import numpy as np
import pytest
import torch

from oracle import kie_tile_ref as K
from oracle import page_turn_ref as PT
from tests.support import assert_same, golden, kw, omni_model, release_models
from tests.test_kie_tiles_cpu import emu_merge, fabricate

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)


def ref_tiles(g):
    """The reference's entity tuples of every tile, class names resolved."""
    from advancedliteratemachinery_b200.omniparser import CLASSES_SROIE
    ents = [[] for _ in range(len(g['plan']))]
    for (k, i, c), p, r, t in zip(g['ref_ent'].tolist(), g['ref_prob'].tolist(), g['ref_rect'].tolist(),
                                  g['ref_text'].tolist()):
        if i == len(ents[k]):
            ents[k].append((t, CLASSES_SROIE[c], p, []))
        ents[k][i][3].append(r)
    return ents


def same_entities(a, b, rtol=0.0):
    assert [(e[0], e[1], e[3]) for e in a] == [(e[0], e[1], e[3]) for e in b]
    if rtol:
        np.testing.assert_allclose([e[2] for e in a], [e[2] for e in b], rtol=rtol)
    else:
        assert [e[2] for e in a] == [e[2] for e in b]


def test_fixture_page_equals_reference_merge():
    """Texts, classes and rects bit for bit, probabilities within the decoder's tolerance; every tile's token ids are
    the reference's; the device merge of the device's own tile decodes equals the host build bit for bit."""
    g = golden('omni_kie_tiles.npz')
    m = omni_model(g, kie=True)
    page = g['page']
    got = m.kie_tiled([page], **kw(g))
    ref = K.merge([page.shape[:2]], int(g['tile']), int(g['overlap']), ref_tiles(g))
    same_entities(got[0], ref['entities'][0], rtol=2e-3)
    t = m.last_tiles
    assert np.array_equal(t['plan'], g['plan'])
    for k in range(len(g['plan'])):
        n = int(g['n_tok'][k])
        assert int(t['n_tok'][k]) == n and np.array_equal(t['tokens'][k, :n], g['tokens'][k, :n])
        ni = int(g['n_inst'][k])
        assert np.array_equal(t['poly'][k, :ni], g['poly'][k, :ni]) and np.array_equal(t['rec'][k, :ni], g['rec'][k, :ni])
    raw = {k: t[k] for k in ('n_tok', 'tokens', 'probs', 'n_inst', 'inst_pos', 'poly')}
    emu = emu_merge([page.shape[:2]], int(g['tile']), int(g['overlap']), raw, class_base=int(g['class_base']))
    assert_same(t['merged'], emu)
    assert [tuple(s) for s in t['merged']['source'].tolist()] == ref['source'][0]


def test_one_tile_page_is_decode_kie():
    """A page that fits in one tile gives exactly decode_kie's list from forward_pages on the whole page."""
    from advancedliteratemachinery_b200 import preprocess as P
    g = golden('omni_kie_tiles.npz')
    m = omni_model(g, kie=True)
    page = np.ascontiguousarray(g['page'][:100, :90])
    got = m.kie_tiled([page], **kw(g))
    v = m.vocab
    nt = P.omni_pages(m.ctx, [page], int(g['test_min_size']), int(g['test_max_size']))
    seqs = [v.pt_prompt(), torch.tensor([[v.poly_sos_index]]), torch.tensor([[v.rec_sos_index]]),
            torch.tensor([[100, 90]])]
    exp = m.forward_pages(nt, seqs)[0] or []
    assert exp and got[0] == exp


def test_turns_map_back():
    """Explicit turns k = 1..3 give kie_tiled(np.rot90(page, k)) with every rect and vertex mapped back; 'upright' and
    all-zero turns give the same result."""
    g = golden('omni_kie_tiles.npz')
    m = omni_model(g, kie=True)
    page = g['page']
    H, W = page.shape[:2]
    up = m.kie_tiled([page], **kw(g))
    up_poly = m.last_tiles['merged']['poly'].copy()
    assert m.kie_tiled([page], orientation=[0], **kw(g)) == up
    assert np.array_equal(m.last_tiles['merged']['poly'], up_poly)
    for k in (1, 2, 3):
        rot = np.ascontiguousarray(np.rot90(page, k))
        ref = m.kie_tiled([rot], **kw(g))[0]
        ref_poly = m.last_tiles['merged']['poly'].copy()
        got = m.kie_tiled([page], orientation=[k], **kw(g))[0]
        mapped = []
        for text, cls, prob, rects in ref:
            rs = []
            for r in rects:
                x0, y0 = PT.map_back(r[0], r[1], k, H, W)
                x1, y1 = PT.map_back(r[2], r[3], k, H, W)
                rs.append([min(x0, x1), min(y0, y1), max(x0, x1), max(y0, y1)])
            mapped.append((text, cls, prob, rs))
        same_entities(got, mapped)
        t = m.last_tiles
        assert t['turns'].tolist() == [k]
        pv = np.array([PT.map_back(u, v, k, H, W) for u, v in ref_poly.reshape(-1, 2)]).reshape(-1, 32)
        assert np.array_equal(t['merged']['poly'], pv)


def test_auto_picks_the_reference_turn():
    """'auto' chooses the turn of the reference's probes with their scores, and reads the page at that turn."""
    g = golden('omni_kie_tiles.npz')
    m = omni_model(g, kie=True)
    page = g['page']
    got = m.kie_tiled([page], orientation='auto', **kw(g))
    t = m.last_tiles
    assert t['turns'].tolist() == g['probe_turn'].tolist()
    np.testing.assert_allclose(t['page_scores'], g['probe_scores'], rtol=1e-3)
    assert np.array_equal(t['probe'][5], g['probe_n_tok'])
    assert got == m.kie_tiled([page], orientation=g['probe_turn'].tolist(), **kw(g))


def test_max_batch_gives_the_same_entities():
    g = golden('omni_kie_tiles.npz')
    m = omni_model(g, kie=True)
    pages = [g['page'], np.ascontiguousarray(g['page'][:100, :90]), np.ascontiguousarray(g['page'][:, :150])]
    ref = m.kie_tiled(pages, max_batch=1, **kw(g))
    n = len(m.last_tiles['plan'])
    for b in (3, n):
        assert m.kie_tiled(pages, max_batch=b, **kw(g)) == ref


def test_merge_at_scale_equals_host_build():
    """16 A4 pages at 300 dpi x 12 tiles of fabricated entities (1..8 words, wordless ones, some turned): the device
    merge equals the host build of the same bodies bit for bit."""
    from advancedliteratemachinery_b200.omniparser import merge_kie_tiles
    g = golden('omni_kie_tiles.npz')
    m = omni_model(g, kie=True)
    rng = np.random.default_rng(11)
    sizes = [(3508, 2480)] * 16
    turns = [0] * 8 + [1, 2, 3, 0, 1, 2, 3, 0]
    raw = fabricate(rng, sizes, 1200, 256, turns, n_ent=60, max_tok=1024, max_inst=400)
    plan = PT.plan(sizes, turns, 1200, 256)
    assert len(plan) == 16 * 12
    for tr in (None, turns):
        if tr is None:
            raw0 = fabricate(rng, sizes, 1200, 256, None, n_ent=60, max_tok=1024, max_inst=400)
            plan0 = PT.plan(sizes, [0] * 16, 1200, 256)
        else:
            raw0, plan0 = raw, plan
        dev = merge_kie_tiles(m.ctx, sizes, 1200, 256, plan0, raw0['n_tok'], raw0['tokens'], raw0['probs'],
                              raw0['n_inst'], raw0['inst_pos'], raw0['poly'], 1000, 1104, 4, turns=tr)
        emu = emu_merge(sizes, 1200, 256, raw0, turns=tr)
        assert_same(dev, emu)
        assert 0 < int(dev['count'].sum()) and (dev['word_count'] > 1).any()


def test_errors_leave_everything_usable():
    """A spotting checkpoint, a bad layout, a bad turn, a mismatched inst_pos and a too-small capacity are refused;
    afterwards decode_kie / forward_pages, kie_tiled and spot_tiled give what they gave before."""
    import ctypes as C

    from advancedliteratemachinery_b200 import AlmError, OmniParserB200, OmniVocab
    from advancedliteratemachinery_b200 import preprocess as P
    from advancedliteratemachinery_b200.omniparser import merge_kie_tiles
    from tests.conftest import omni_sd
    g = golden('omni_kie_tiles.npz')
    m = omni_model(g, kie=True)
    page = g['page']
    v = m.vocab
    small = np.ascontiguousarray(page[:100, :90])
    seqs = [v.pt_prompt(), torch.tensor([[v.poly_sos_index]]), torch.tensor([[v.rec_sos_index]]),
            torch.tensor([[100, 90]])]

    def fwd():
        return m.forward_pages(P.omni_pages(m.ctx, [small], int(g['test_min_size']), int(g['test_max_size'])), seqs)

    before, tiled = fwd(), m.kie_tiled([page], **kw(g))
    raw = {k: m.last_tiles[k].copy() for k in ('n_tok', 'tokens', 'probs', 'n_inst', 'inst_pos', 'poly')}
    plan = m.last_tiles['plan']
    args = lambda r: (r['n_tok'], r['tokens'], r['probs'], r['n_inst'], r['inst_pos'], r['poly'], 1000,  # noqa: E731
                      int(g['class_base']), 4)
    sz = [page.shape[:2]]
    T, ov = int(g['tile']), int(g['overlap'])
    with pytest.raises((AlmError, ValueError)):
        m.kie_tiled([page], tile=63, overlap=0)
    with pytest.raises(ValueError):
        m.kie_tiled([page], orientation=[4], **kw(g))
    with pytest.raises(ValueError):
        m.kie_tiled([page], orientation='mixed', **kw(g))
    with pytest.raises(ValueError):
        m.kie_tiled([page], rec_candidates=2, **kw(g))
    with pytest.raises(AlmError):
        merge_kie_tiles(m.ctx, sz, 63, 0, plan, *args(raw))
    with pytest.raises(ValueError):
        merge_kie_tiles(m.ctx, sz, T, ov, plan, *args(raw), turns=[4])
    bad = {k: a.copy() for k, a in raw.items()}
    k = int(np.argmax(bad['n_inst'] > 0))
    bad['inst_pos'][k, 0] += 1
    with pytest.raises(AlmError):
        merge_kie_tiles(m.ctx, sz, T, ov, plan, *args(bad))
    bad = {k: a.copy() for k, a in raw.items()}
    bad['tokens'][k, 2] = int(g['class_base']) + 4
    with pytest.raises(AlmError):
        merge_kie_tiles(m.ctx, sz, T, ov, plan, *args(bad))
    # a capacity below the entities: the entry itself, with cap_ent 0
    hs, ws = np.array([sz[0][0]], np.int32), np.array([sz[0][1]], np.int32)
    tp, to = np.ascontiguousarray(plan[:, 0]), np.ascontiguousarray(plan[:, 1:3])
    r = {k: np.ascontiguousarray(a) for k, a in raw.items()}
    outs = [np.zeros(64, np.int32) for _ in range(7)]
    rc = m.lib.alm_omni_merge_kie_tiles(
        m.ctx.h, hs.ctypes.data, ws.ctypes.data, 1, None, T, ov, len(plan), tp.ctypes.data, to.ctypes.data,
        r['n_tok'].ctypes.data, r['tokens'].ctypes.data, r['probs'].ctypes.data, r['tokens'].shape[1],
        r['n_inst'].ctypes.data, r['inst_pos'].ctypes.data, r['poly'].ctypes.data, r['inst_pos'].shape[1], 1000,
        int(g['class_base']), 4, 4.0, 8.0, 0.5, *[o.ctypes.data for o in outs], C.c_long(0),
        np.zeros((64, 4)).ctypes.data, np.zeros((64, 32)).ctypes.data, np.zeros((64, 2), np.int32).ctypes.data,
        C.c_long(64))
    assert rc != 0
    assert fwd() == before
    assert m.kie_tiled([page], **kw(g)) == tiled
    # a spotting checkpoint is refused; its context keeps working
    tg = golden('omni_tiles.npz')
    s = OmniParserB200(omni_sd(int(tg['wseed']), float(tg['pt_eos_bias'])),
                       OmniVocab(pt_seq_length=int(tg['pt_seq_length']), rec_length=int(tg['rec_length'])),
                       workspace_mb=4096)
    try:
        tkw = kw(tg)
        spot = s.spot_tiled([tg['page']], **tkw)
        with pytest.raises(ValueError):
            s.kie_tiled([tg['page']], **tkw)
        with pytest.raises(AlmError):
            merge_kie_tiles(s.ctx, sz, T, ov, plan, *args(bad))
        assert s.spot_tiled([tg['page']], **tkw) == spot
    finally:
        s.ctx.close()
