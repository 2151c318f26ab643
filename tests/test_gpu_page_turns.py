"""GPU: pages read turned by quarter-turns (preprocess.omni_tiles(turns=), merge_tiles(turns=), orient_select,
OmniParserB200.spot_tiled(orientation=); DESIGN 4.14).  Turned tile inputs must equal those of the host-turned pages
bit for bit; a page read at turn k must equal spot_tiled of np.rot90(page, k) with its rows mapped back by
oracle/page_turn_ref.py; 'upright' and all-zero turns must be today's result; 'auto' must choose what the oracle
chooses from the device's own probe readings and then equal the explicit reading at that turn; and
tests/golden/omni_page_turns.npz (the unmodified reference on np.rot90 of a page) must be reproduced."""
import numpy as np
import pytest
import torch

from oracle import page_turn_ref as R
from tests.support import assert_same, golden, kw, omni_model, release_models, same

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

ERR_INVALID = -1  # include/alm_ocr.h ALM_ERR_INVALID


def pages(gold):
    """The fixture page (two tiles upright, two turned), a page of 2 x 3 tiles and one smaller than a tile."""
    rng = np.random.default_rng(21)
    return [gold['page'], rng.integers(0, 256, (230, 301, 3), dtype=np.uint8),
            rng.integers(0, 256, (97, 120, 3), dtype=np.uint8)]


def mapped(res, k, H, W):
    """spot_tiled dicts of np.rot90(page, k) with their points and vertices mapped back to the H x W page by the
    oracle, vertex order kept, and 'turns' added."""
    out = []
    for d in res:
        e = dict(d)
        e['pts'] = [list(R.map_back(*d['pts'][0], k, H, W))]
        e['polys'] = [list(R.map_back(u, v, k, H, W)) for u, v in d['polys']]
        e['turns'] = k
        out.append(e)
    return out


def test_turned_tile_inputs_equal_omni_tiles_of_turned_pages():
    """All four turns, pages smaller and larger than T and of odd sizes, host and device pages, whole plan and
    sub-ranges: tensors and mask bit for bit."""
    from advancedliteratemachinery_b200 import _lib, preprocess as P
    ctx = _lib.Context(0)
    try:
        rng = np.random.default_rng(2)
        pg = [rng.integers(0, 256, s + (3,), dtype=np.uint8) for s in ((301, 219), (91, 400), (128, 128), (77, 61))]
        for T, ov, mn, mx in ((128, 32, 128, 256), (100, 50, 80, 333)):
            for turns in ([0, 1, 2, 3], [1, 3, 2, 1], [2, 2, 0, 3], [3, 0, 1, 1]):
                rot = [np.ascontiguousarray(np.rot90(p, k)) for p, k in zip(pg, turns)]
                n = len(P.omni_tile_plan([r.shape[:2] for r in rot], T, ov))
                for first, count in ((0, None), (1, 3), (n - 2, 2)):
                    src = pg if first else [torch.from_numpy(p).cuda() for p in pg]
                    got = P.omni_tiles(ctx, src, T, ov, mn, mx, first, count, turns=turns)
                    want = P.omni_tiles(ctx, rot, T, ov, mn, mx, first, count)
                    assert torch.equal(got.tensors.view(torch.int32), want.tensors.view(torch.int32))
                    assert torch.equal(got.mask, want.mask)
    finally:
        ctx.close()


def test_explicit_turns_equal_the_rotated_pages_mapped_back():
    """Every page at every turn: spot_tiled(orientation=turns) equals spot_tiled of np.rot90(page, k) with the rows
    mapped back by the oracle, in every field (vertex j maps to vertex j: the order is kept)."""
    gold = golden('omni_page_turns.npz')
    m = omni_model(gold)
    pg = pages(gold)
    for turns in ([1, 2, 3], [3, 0, 2], [2, 3, 1]):
        got = m.spot_tiled(pg, max_batch=1, orientation=np.array(turns), **kw(gold))
        assert m.last_tiles['turns'].tolist() == turns and 'page_scores' not in m.last_tiles
        want = [mapped(m.spot_tiled([np.rot90(p, k)], max_batch=1, **kw(gold))[0], k, *p.shape[:2])
                for p, k in zip(pg, turns)]
        same(got, want)
        assert sum(len(r) for r in got) > 0
    # chunks of several turned tiles agree with one tile per chunk
    same(m.spot_tiled(pg, max_batch=5, orientation=[1, 2, 3], **kw(gold)),
         m.spot_tiled(pg, max_batch=1, orientation=[1, 2, 3], **kw(gold)))


def test_the_fixture_at_every_turn():
    """The fixture page read at turns 0..3 as four pages: tile decodes equal the reference's (ids exact,
    probabilities close), the merge equals the oracle's (coordinates exact), and the device merge equals the host build
    fed the device's own tile outputs."""
    from tests.test_page_turns_cpu import emu_merge_turned
    gold = golden('omni_page_turns.npz')
    m = omni_model(gold)
    page = gold['page']
    m.spot_tiled([page] * 4, orientation=[0, 1, 2, 3], **kw(gold))
    t = m.last_tiles
    assert np.array_equal(t['plan'], gold['plan'])
    for k in ('n_inst', 'pt', 'poly', 'rec'):
        assert np.array_equal(t[k], gold[k]), k
    np.testing.assert_allclose(t['prob'], gold['prob'], rtol=2e-3, atol=1e-7)
    for k in ('count', 'offset', 'pts', 'polys', 'rec', 'source'):
        assert np.array_equal(t['merged'][k], gold[f'merged_{k}']), k
    assert_same(t['merged'], emu_merge_turned([page.shape[:2]] * 4, [0, 1, 2, 3], int(gold['tile']),
                                              int(gold['overlap']), t['n_inst'], t['pt'], t['poly'], t['rec'],
                                              t['prob'], m.vocab.num_bins))


def test_upright_and_zero_turns_are_todays_result():
    """'upright' is the default path (no new keys, same last_tiles); all-zero turns give the same rows bit for bit."""
    gold = golden('omni_page_turns.npz')
    m = omni_model(gold)
    pg = pages(gold)
    base = m.spot_tiled(pg, **kw(gold))
    t0 = m.last_tiles
    up = m.spot_tiled(pg, orientation='upright', **kw(gold))
    assert set(m.last_tiles) == set(t0) and np.array_equal(m.last_tiles['plan'], t0['plan'])
    same(up, base)
    assert all(set(d) == {'pts', 'score', 'polys', 'rec', 'tile', 'instance'} for r in up for d in r)
    zero = m.spot_tiled(pg, orientation=[0, 0, 0], **kw(gold))
    same(zero, [[dict(d, turns=0) for d in r] for r in base])


def test_auto_chooses_what_the_oracle_chooses_and_reads_at_that_turn():
    """'auto': the probe readings are the reference's on the fixture page; turns and page_scores equal the oracle's
    choice from the device's own probe readings; the result equals explicit-turn spot_tiled at the chosen turns (a
    page of several tiles read again in tiles, the others kept from their probe); only P turns and P x 4 scores come
    back from the one-launch selection."""
    from advancedliteratemachinery_b200.omniparser import orient_select
    gold = golden('omni_page_turns.npz')
    m = omni_model(gold)
    v = m.vocab
    pg = pages(gold)
    P = len(pg)
    got = m.spot_tiled(pg, max_batch=1, orientation='auto', **kw(gold))
    t = m.last_tiles
    n_inst, _, _, rec, prob = t['probe']
    assert n_inst.shape == (4 * P,)
    want_t, want_s = R.choose(n_inst.reshape(P, 4), rec.reshape((P, 4) + rec.shape[1:]),
                              prob.reshape((P, 4) + prob.shape[1:]), v.recog_pad_index, v.rec_eos_index)
    assert t['turns'].tolist() == want_t.tolist()
    assert t['page_scores'].view(np.uint64).tolist() == want_s.view(np.uint64).tolist()
    for k in ('n_inst', 'pt', 'poly', 'rec'):
        assert np.array_equal(t['probe'][('n_inst', 'pt', 'poly', 'rec').index(k)][:4], gold[f'probe_{k}']), k
    assert int(t['turns'][0]) == int(gold['probe_turn'])
    np.testing.assert_allclose(t['page_scores'][0], gold['probe_page_scores'], rtol=1e-5)
    same(got, m.spot_tiled(pg, max_batch=1, orientation=t['turns'], **kw(gold)))
    assert all(d['turns'] == int(t['turns'][p]) for p, r in enumerate(got) for d in r)
    # the selection alone: one launch, P turns and P x 4 scores
    m.ctx.launch_count(reset=True)
    turns, scores = orient_select(m.ctx, n_inst.reshape(P, 4), rec.reshape((P, 4) + rec.shape[1:]),
                                  prob.reshape((P, 4) + prob.shape[1:]), v.recog_pad_index, v.rec_eos_index)
    assert m.ctx.launch_count() == 1 and turns.shape == (P,) and scores.shape == (P, 4)
    assert np.array_equal(turns, t['turns']) and np.array_equal(scores, t['page_scores'])


def test_auto_on_many_pages_and_chunks():
    """'auto' over several chunks equals 'auto' one page at a time, and the selection at scale equals the oracle."""
    from advancedliteratemachinery_b200.omniparser import orient_select
    gold = golden('omni_page_turns.npz')
    m = omni_model(gold)
    pg = pages(gold)
    same(m.spot_tiled(pg, max_batch=3, orientation='auto', **kw(gold)),
         [m.spot_tiled([p], max_batch=3, orientation='auto', **kw(gold))[0] for p in pg])
    rng = np.random.default_rng(4)
    P, maxi, L = 300, 512, 25
    n_inst = rng.integers(0, maxi + 1, (P, 4)).astype(np.int32)
    n_inst[0], n_inst[1], n_inst[2] = 0, maxi, [0, 3, 0, 0]
    rec = rng.choice([1096, 1099, 1095, 1000, 1010], (P, 4, maxi, L), p=[.05, .05, .1, .4, .4])
    prob = rng.uniform(0, 1, (P, 4, maxi, L)).astype(np.float32)
    turns, scores = orient_select(m.ctx, n_inst, rec, prob, 1096, 1099)
    want_t, want_s = R.choose(n_inst, rec, prob, 1096, 1099)
    assert np.array_equal(turns, want_t) and np.array_equal(scores.view(np.uint64), want_s.view(np.uint64))


def test_error_paths_leave_the_context_usable():
    """Unknown orientation strings, turns of the wrong length or outside 0..3 and a KIE checkpoint raise ValueError;
    the C entries refuse bad turns and bad counts before any device work; the context reads correctly afterwards."""
    import ctypes as C
    from advancedliteratemachinery_b200 import OmniParserB200, _lib, preprocess as Pre
    from advancedliteratemachinery_b200.omniparser import merge_tiles
    gold = golden('omni_page_turns.npz')
    m = omni_model(gold)
    pg = pages(gold)
    for bad in ('sideways', 'Auto', [0, 1], [0, 1, 4], [0, -1, 0], np.zeros(3)):
        with pytest.raises(ValueError):
            m.spot_tiled(pg, orientation=bad, **kw(gold))
    with pytest.raises(ValueError):
        Pre.omni_tiles(m.ctx, pg, 128, 32, turns=[0, 1])
    lib, h = m.ctx.lib, m.ctx.h
    page = np.ascontiguousarray(gold['page'])
    ptrs = (C.c_void_p * 1)(page.ctypes.data)
    hs, ws = np.array([page.shape[0]], np.int32), np.array([page.shape[1]], np.int32)
    out = torch.empty(8, 3, 256, 256, device='cuda')
    mask = torch.empty(8, 256, 256, dtype=torch.uint8, device='cuda')
    for t in (4, -1):
        turns = np.array([t], np.int32)
        assert lib.alm_pre_omni_tiles_turned(h, ptrs, hs.ctypes.data, ws.ctypes.data, 1, turns.ctypes.data, 128, 32,
                                             0, 1, 128, 256, out.data_ptr(), mask.data_ptr()) == ERR_INVALID
    assert lib.alm_pre_omni_tiles_turned(h, ptrs, hs.ctypes.data, ws.ctypes.data, 1, None, 128, 32, 0, 1, 128, 256,
                                         out.data_ptr(), mask.data_ptr()) == ERR_INVALID
    n_inst = np.array([0, 1, 7, 0], np.int32)   # 7 > max_inst
    rec, prob = np.zeros((4, 6, 25), np.int64), np.zeros((4, 6, 25), np.float32)
    tt, sc = np.zeros(1, np.int32), np.zeros(4)
    assert lib.alm_omni_orient_select(h, 1, n_inst.ctypes.data, rec.ctypes.data, prob.ctypes.data, 6, 25, 1096, 1099,
                                      tt.ctypes.data, sc.ctypes.data) == ERR_INVALID
    assert lib.alm_omni_orient_select(h, 0, n_inst.ctypes.data, rec.ctypes.data, prob.ctypes.data, 6, 25, 1096, 1099,
                                      tt.ctypes.data, sc.ctypes.data) == ERR_INVALID
    plan = gold['plan'][:2]
    outs = [gold[k][:2] for k in ('n_inst', 'pt', 'poly', 'rec', 'prob')]
    with pytest.raises(_lib.AlmError):   # the plan of the upright page is not the plan of the page turned once
        merge_tiles(m.ctx, [page.shape[:2]], 128, 32, plan, *outs, 1000, turns=[1])
    got = merge_tiles(m.ctx, [page.shape[:2]], 128, 32, plan, *outs, 1000, turns=[0])
    assert np.array_equal(got['source'], gold['merged_source'][:int(gold['merged_count'][0])])
    kie = OmniParserB200(None, type(m.vocab)(vie_categories=4))
    with pytest.raises(ValueError):
        kie.spot_tiled(pg, orientation='auto')
    kie.ctx.close()
