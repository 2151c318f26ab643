"""GPU: recognition candidates and n-best beams for the words of pages read in tiles (OmniParserB200.spot_tiled(
rec_candidates=, rec_beams=, length_penalty=); DESIGN 4.11, 4.14, 4.15).

* candidates change no word: every dict equals spot_tiled() bit for bit, candidate 0 is the word's rec ids and
  probabilities, and each word's row is its tile instance's row of the tile decodes, which equal
  decode(rec_candidates=k) of forward_pages on the host-sliced tiles;
* a page of one tile gets decode's candidates and beams of the batch-1 reading;
* W = 1 is spot_tiled() up to each word's first terminal token; W = 4 keeps the points, polygons, 'tile' and
  'instance' for 'upright' and explicit turns, and every n-best list is its tile instance's;
* explicit turns, 'auto' and 'mixed' follow each word back to its (reading, tile, instance); 'auto''s one-tile pages
  keep their probe's lists; candidates with rec_locations keep the 'chars' of rec_locations alone;
* refusals come before any device work, and a later plain call is spot_tiled() with the lists reset;
* max_batch 1 / 5 / 16 give the same lists.
"""
import numpy as np
import pytest
import torch

from tests.support import golden, kw, omni_model, release_models, same

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)


def setup():
    gold = golden('omni_tiles.npz')
    return gold, omni_model(gold)


def pages():
    """The fixture pages of omni_tiles.npz (2 x 3 tiles) and omni_page_turns.npz (two tiles upright, two turned), a page
    of one tile and one of 2 x 3 tiles of noise."""
    rng = np.random.default_rng(5)
    return [golden('omni_tiles.npz')['page'], golden('omni_page_turns.npz')['page'],
            rng.integers(0, 256, (97, 120, 3), dtype=np.uint8), rng.integers(0, 256, (230, 301, 3), dtype=np.uint8)]


def one_tile_page():
    return np.random.default_rng(5).integers(0, 256, (100, 90, 3), dtype=np.uint8)


def sliced(pages, plan):
    return [np.ascontiguousarray(pages[p][y:y + h, x:x + w]) for p, y, x, h, w in plan.tolist()]


def same_arrays(a, b, tag=''):
    """Two tuples of arrays are equal, floats bit for bit."""
    assert len(a) == len(b), tag
    for i, (x, y) in enumerate(zip(a, b)):
        assert x.shape == y.shape and x.dtype == y.dtype, (tag, i, x.shape, y.shape)
        if x.dtype == np.float32:
            x, y = np.ascontiguousarray(x).view(np.uint32), np.ascontiguousarray(y).view(np.uint32)
        assert np.array_equal(x, y), (tag, i)


def followed_back(m, res):
    """Each returned word's (tile row of last_tiles' plan, instance), in result order, from its 'tile' / 'instance'
    (and for 'mixed', whose plan is that of the 4 P readings, its 'turns')."""
    t = m.last_tiles
    mixed = 'turn_merge' in t
    first = np.searchsorted(t['plan'][:, 0], np.arange(int(t['plan'][:, 0].max()) + 1))
    rows = [(first[4 * p + d['turns'] if mixed else p] + d['tile'], d['instance'])
            for p, r in enumerate(res) for d in r]
    return np.array(rows, np.int64).reshape(-1, 2)


def rows_of(lists, src):
    return tuple(a[src[:, 0], src[:, 1]] for a in lists)


def without(res, keys):
    return [[{k: v for k, v in d.items() if k not in keys} for d in r] for r in res]


def terminal_end(v, row):
    """index after the first rec_eos / recog_pad of a rec row (its length when there is none)"""
    for i, c in enumerate(row.tolist()):
        if c in (v.rec_eos_index, v.recog_pad_index):
            return i + 1
    return len(row)


# ------------------------------------------------------------------------------------------------ candidates
@pytest.mark.parametrize('k', [1, 3, 8])
def test_candidates_are_free_and_are_the_tiles_decode(k):
    from advancedliteratemachinery_b200 import preprocess as P
    from advancedliteratemachinery_b200.omniparser import slot_candidates
    gold, m = setup()
    page = gold['page']
    base = m.spot_tiled([page], **kw(gold))
    got = m.spot_tiled([page], rec_candidates=k, **kw(gold))
    same(got, base)
    t = m.last_tiles
    ids, probs = m.last_rec_candidates
    N, L = len(got[0]), m.vocab.rec_length
    assert N > 0 and ids.shape == (N, L, k) and probs.shape == (N, L, k) and ids.dtype == np.int64
    assert m.last_rec_beams is None and 'beams' not in t
    same_arrays((ids[:, :, 0], probs[:, :, 0]), (t['merged']['rec'], t['merged']['prob']), 'candidate 0')
    src = followed_back(m, got)
    assert np.array_equal(src, t['merged']['source'])
    same_arrays((ids, probs), rows_of(t['candidates'], src), 'rows')
    assert t['candidates'][0].shape == t['rec'].shape + (k,)
    # every tile's candidates: decode(rec_candidates=k) of forward_pages on the host-sliced tiles
    nt = P.omni_pages(m.ctx, sliced([page], t['plan']), int(gold['test_min_size']), int(gold['test_max_size']))
    outs = m.forward_pages(nt, rec_candidates=k)
    want = slot_candidates(t['n_inst'], *m.last_rec_candidates)
    for j, (o, w) in enumerate(zip(outs, want)):
        n = int(t['n_inst'][j])
        assert (o is None) == (w is None) == (n == 0)
        if w is not None:
            same_arrays(w, (t['candidates'][0][j, :n], t['candidates'][1][j, :n]), f'tile {j}')


def test_one_tile_page_gets_decodes_candidates_and_beams():
    from advancedliteratemachinery_b200 import preprocess as P
    from advancedliteratemachinery_b200.omniparser import slot_beams, slot_candidates
    gold, m = setup()
    page = one_tile_page()
    nt = P.omni_pages(m.ctx, [page], int(gold['test_min_size']), int(gold['test_max_size']))
    for extra in (dict(rec_candidates=3), dict(rec_beams=4), dict(rec_beams=3, length_penalty=0.5)):
        cand = 'rec_candidates' in extra
        res = m.spot_tiled([page], **kw(gold, **extra))[0]
        assert res and [(d['tile'], d['instance']) for d in res] == [(0, i) for i in range(len(res))]
        got = m.last_rec_candidates if cand else m.last_rec_beams
        out = m.forward_pages(nt, **extra)[0]
        n = out[0][0].numel() // 2
        assert n == len(res)
        want = slot_candidates(np.array([n]), *m.last_rec_candidates) if cand else \
            slot_beams(np.array([n]), *m.last_rec_beams)
        same_arrays(got, want[0], str(extra))


# ------------------------------------------------------------------------------------------------ beams
def test_width_one_is_spot_tiled_up_to_the_first_terminal_token():
    gold, m = setup()
    v = m.vocab
    pg = pages()
    for orientation in ('upright', [1, 0, 3, 2], 'mixed'):
        base = m.spot_tiled(pg, orientation=orientation, **kw(gold))
        mg = m.last_tiles['turn_merge' if orientation == 'mixed' else 'merged']
        got = m.spot_tiled(pg, orientation=orientation, rec_beams=1, **kw(gold))
        same(got, base)   # 'rec' and 'score' read up to the first terminal token
        ids, probs, scores = m.last_rec_beams
        assert ids.shape == (len(mg['rec']), 1, v.rec_length) and scores.shape == (len(mg['rec']), 1)
        for i in range(len(mg['rec'])):
            e = terminal_end(v, mg['rec'][i])
            assert np.array_equal(ids[i, 0, :e], mg['rec'][i, :e]), (orientation, i)
            assert np.array_equal(probs[i, 0, :e].view(np.uint32), mg['prob'][i, :e].view(np.uint32)), (orientation, i)
            assert (ids[i, 0, e:] == v.recog_pad_index).all() and (probs[i, 0, e:] == 0).all(), (orientation, i)


def test_beams_keep_the_greedy_geometry_and_are_the_tiles_decode():
    """W = 4: points, polygons, 'tile', 'instance' (and 'turns') as spot_tiled(), 'rec' / 'score' hypothesis 0's; every
    word's n-best list is its tile instance's, and those of the fixture page's tiles are decode(rec_beams=4) of
    forward_pages on the host-sliced tiles."""
    from advancedliteratemachinery_b200 import postprocess, preprocess as P
    from advancedliteratemachinery_b200.omniparser import slot_beams
    gold, m = setup()
    v = m.vocab
    pg = pages()
    for orientation in ('upright', [1, 0, 3, 2], [2, 2, 2, 2], [3, 1, 1, 3]):
        base = m.spot_tiled(pg, orientation=orientation, **kw(gold))
        got = m.spot_tiled(pg, orientation=orientation, rec_beams=4, length_penalty=0.7, **kw(gold))
        assert without(got, ('rec', 'score')) == without(base, ('rec', 'score')), orientation
        t = m.last_tiles
        ids, probs, scores = m.last_rec_beams
        N = sum(len(r) for r in got)
        assert N > 0 and ids.shape == (N, 4, v.rec_length) and probs.shape == ids.shape and scores.shape == (N, 4)
        assert m.last_rec_candidates is None and 'candidates' not in t
        texts, sc = postprocess.rec_texts(ids[:, 0], probs[:, 0], v)
        assert [d['rec'] for r in got for d in r] == texts and [d['score'] for r in got for d in r] == sc.tolist()
        same_arrays((ids[:, 0], probs[:, 0]), (t['merged']['rec'], t['merged']['prob']), 'hypothesis 0')
        src = followed_back(m, got)
        same_arrays((ids, probs, scores), rows_of(t['beams'], src), str(orientation))
    m.spot_tiled(pg[:1], rec_beams=4, length_penalty=0.7, **kw(gold))
    t = m.last_tiles
    nt = P.omni_pages(m.ctx, sliced(pg[:1], t['plan']), int(gold['test_min_size']), int(gold['test_max_size']))
    m.forward_pages(nt, rec_beams=4, length_penalty=0.7)
    want = slot_beams(t['n_inst'], *m.last_rec_beams)
    for j, w in enumerate(want):
        n = int(t['n_inst'][j])
        assert (w is None) == (n == 0)
        if w is not None:
            same_arrays(w, tuple(a[j, :n] for a in t['beams']), f'tile {j}')


def test_turned_lists_equal_the_turned_page_read_upright():
    """Turn k reads the tiles of np.rot90(page, k) bit for bit, so its tiles' lists are those of that page read
    upright."""
    gold, m = setup()
    page = pages()[1]
    for extra in (dict(rec_candidates=5), dict(rec_beams=4)):
        name = 'candidates' if 'rec_candidates' in extra else 'beams'
        for k in range(4):
            m.spot_tiled([page], orientation=[k], **kw(gold, **extra))
            got = m.last_tiles[name]
            m.spot_tiled([np.ascontiguousarray(np.rot90(page, k))], **kw(gold, **extra))
            same_arrays(got, m.last_tiles[name], f'{name} turn {k}')


# ------------------------------------------------------------------------------------------------ orientation
@pytest.mark.parametrize('orientation', ['upright', 'turns', 'auto', 'mixed'])
def test_rows_follow_each_word_back_to_its_tile_instance(orientation):
    gold, m = setup()
    pg = pages()
    o = [1, 0, 3, 2] if orientation == 'turns' else orientation
    base = m.spot_tiled(pg, orientation=o, max_batch=5, **kw(gold))
    got = m.spot_tiled(pg, orientation=o, max_batch=5, rec_candidates=4, **kw(gold))
    same(got, base)
    t = m.last_tiles
    src = followed_back(m, got)
    assert len(src) > 0
    same_arrays(m.last_rec_candidates, rows_of(t['candidates'], src), 'candidates')
    mg = t['turn_merge' if orientation == 'mixed' else 'merged']
    same_arrays((m.last_rec_candidates[0][:, :, 0], m.last_rec_candidates[1][:, :, 0]), (mg['rec'], mg['prob']))
    got = m.spot_tiled(pg, orientation=o, max_batch=5, rec_beams=4, **kw(gold))
    t = m.last_tiles
    src = followed_back(m, got)
    same_arrays(m.last_rec_beams, rows_of(t['beams'], src), 'beams')
    mg = t['turn_merge' if orientation == 'mixed' else 'merged']
    same_arrays((m.last_rec_beams[0][:, 0], m.last_rec_beams[1][:, 0]), (mg['rec'], mg['prob']))
    if orientation == 'auto':   # the one-tile page's tile row is its probe reading at the chosen turn, lists included
        p = 2
        j = int(np.nonzero(t['plan'][:, 0] == p)[0][0])
        r = 4 * p + int(t['turns'][p])
        same_arrays(tuple(a[j] for a in t['beams']), tuple(a[r] for a in t['probe'][5:]), 'probe')
        assert len(t['probe']) == 8


def test_candidates_with_locations_keep_the_chars():
    from tests.test_gpu_page_char_boxes import same_chars
    gold, m = setup()
    pg = pages()
    for orientation in ('upright', 'auto', 'mixed'):
        alone = m.spot_tiled(pg, orientation=orientation, rec_locations=True, **kw(gold))
        loc = m.last_tiles['loc']
        cand = m.spot_tiled(pg, orientation=orientation, rec_candidates=3, **kw(gold))
        lists = m.last_rec_candidates
        both = m.spot_tiled(pg, orientation=orientation, rec_candidates=3, rec_locations=True, **kw(gold))
        assert without(both, ('chars',)) == without(alone, ('chars',)) == cand
        for ra, rb in zip(both, alone):
            for a, b in zip(ra, rb):
                same_chars(a['chars'], b['chars'])
        same_arrays(m.last_rec_candidates, lists, orientation)
        same_arrays((m.last_tiles['loc'],), (loc,), orientation)


# ------------------------------------------------------------------------------------------------ refusals and reset
def test_refusals_come_before_any_device_work_and_a_plain_call_resets(monkeypatch):
    gold, m = setup()
    pg = pages()
    base = m.spot_tiled(pg, **kw(gold))
    for extra in (dict(rec_candidates=3), dict(rec_beams=2)):   # a plain call after one with lists
        m.spot_tiled(pg, **kw(gold, **extra))
        assert m.last_rec_candidates is not None or m.last_rec_beams is not None
        same(m.spot_tiled(pg, **kw(gold)), base)
        assert m.last_rec_candidates is None and m.last_rec_beams is None
        assert 'candidates' not in m.last_tiles and 'beams' not in m.last_tiles
    encoded = []
    monkeypatch.setattr(m, 'encode', lambda *a, **k: encoded.append('encode'))
    monkeypatch.setattr(m, 'encode_pages', lambda *a, **k: encoded.append('encode_pages'))
    n0 = m.ctx.launch_count()
    bad = [dict(rec_candidates=2, whole_page=True), dict(rec_beams=2, whole_page=True),
           dict(rec_beams=1, whole_page=True, orientation='mixed'), dict(rec_candidates=9), dict(rec_candidates=-1),
           dict(rec_beams=9), dict(rec_beams=-1), dict(rec_beams=2, length_penalty=2.5),
           dict(rec_beams=2, length_penalty=-0.1), dict(rec_candidates=2, rec_beams=2),
           dict(rec_beams=2, rec_locations=True), dict(rec_beams=2, rec_locations=True, orientation='auto')]
    for extra in bad:
        with pytest.raises(ValueError):
            m.spot_tiled(pg, **kw(gold, **extra))
    assert encoded == [] and m.ctx.launch_count() == n0
    monkeypatch.undo()
    same(m.spot_tiled(pg, **kw(gold)), base)
    assert m.last_rec_candidates is None and m.last_rec_beams is None


# ------------------------------------------------------------------------------------------------ chunks
def test_chunk_sizes_give_the_same_lists():
    """max_batch 1 / 5 / 16 over two pages of different sizes (chunks through encode and encode_pages): the same words
    and candidates bit for bit.  Beams with W > 1 run the tensor-core decoder path, whose probabilities move in the
    last bits with the batch shape (DESIGN 4.4, as test_gpu_beams checks for decode): the same words and hypothesis
    ids, probabilities and scores within 5e-5 relative."""
    gold, m = setup()
    pg = [gold['page'], one_tile_page()]
    runs, lists = [], []
    for mb in (1, 5, 16):
        runs.append(m.spot_tiled(pg, max_batch=mb, **kw(gold, rec_candidates=3)))
        lists.append(m.last_rec_candidates)
    assert runs[0] == runs[1] == runs[2] and len(runs[0][1]) > 0
    for other in lists[1:]:
        same_arrays(other, lists[0], 'candidates')
    runs, lists = [], []
    for mb in (1, 5, 16):
        runs.append(m.spot_tiled(pg, max_batch=mb, **kw(gold, rec_beams=4)))
        lists.append(m.last_rec_beams)
    for res, (ids, probs, scores) in zip(runs[1:], lists[1:]):
        assert without(res, ('score',)) == without(runs[0], ('score',))
        np.testing.assert_allclose([d['score'] for r in res for d in r], [d['score'] for r in runs[0] for d in r],
                                   rtol=5e-5, atol=0)
        assert np.array_equal(ids, lists[0][0])
        np.testing.assert_allclose(probs, lists[0][1], rtol=5e-5, atol=0)
        np.testing.assert_allclose(scores, lists[0][2], rtol=5e-5, atol=1e-6)
