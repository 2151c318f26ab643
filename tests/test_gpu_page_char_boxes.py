"""GPU: character boxes in page pixels of words read in tiles (DESIGN 4.20; alm_omni_char_boxes,
omniparser.char_boxes, spot_tiled / read_regions with rec_locations=True).  The device entry must equal the host build
of the same bodies (tests/emu/rec_box_emu.cpp) in every field, bit for bit, on the fabricated sets of
tests/test_page_char_boxes_cpu.py and at 16 pages x 4 096 words in one launch; a page read turned must give the boxes
of np.rot90(page, k) read upright, mapped by the rule, bit for bit; locations must change nothing else; every word's
boxes must come from the reading the merges kept; and rec_locations=False must be today's path."""
import numpy as np
import pytest
import torch

from oracle import rec_box_ref as R
from oracle.whole_page_ref import map_back
from tests.support import ctx, golden, kw, omni_model, release_models
from tests.test_page_char_boxes_cpu import (EOS, KEYS, PAD, assert_same, emu_boxes, fabricate, frames_to_tiles,
                                           hand_made_words)

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

ERR_INVALID = -1  # include/alm_ocr.h ALM_ERR_INVALID


def device(ctx, polys, rec, loc, fi, frames):
    from advancedliteratemachinery_b200.omniparser import char_boxes
    sizes, tiles, turns = frames_to_tiles(frames)
    return char_boxes(ctx, sizes, tiles, polys, rec, loc, fi, PAD, EOS, turns=turns)


def pages():
    """The fixture pages of omni_tiles.npz (2 x 3 tiles) and omni_page_turns.npz (two tiles upright, two turned), a page
    of one tile and one of 2 x 3 tiles of noise."""
    rng = np.random.default_rng(5)
    return [golden('omni_tiles.npz')['page'], golden('omni_page_turns.npz')['page'],
            rng.integers(0, 256, (97, 120, 3), dtype=np.uint8), rng.integers(0, 256, (230, 301, 3), dtype=np.uint8)]


def without_chars(res):
    return [[{k: v for k, v in d.items() if k != 'chars'} for d in r] for r in res]


def same_chars(a, b):
    """Two lists of 'chars' equal, floats bit for bit."""
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert x['char'] == y['char']
        for k in ('centre', 'cov', 'box'):
            assert np.array_equal(x[k], y[k], equal_nan=True), k


def oracle_chars(m, sizes, plan, turns, polys, rec, loc, tile_index):
    from advancedliteratemachinery_b200.omniparser import char_dicts
    v = m.vocab
    H = np.array([sizes[p][0] for p in plan[:, 0]])
    W = np.array([sizes[p][1] for p in plan[:, 0]])
    t = np.zeros(len(plan), np.int64) if turns is None else np.asarray(turns)[plan[:, 0]]
    frames = np.stack([H, W, t, plan[:, 1], plan[:, 2], plan[:, 3], plan[:, 4]], 1)
    return char_dicts(R.char_boxes(polys, rec, loc, tile_index, frames, v.recog_pad_index, v.rec_eos_index), rec, v)


# ---- the entry against the host build


@pytest.mark.parametrize('seed', range(3))
def test_device_equals_the_emulation_on_fabricated_words(ctx, seed):
    args = fabricate(seed)
    n0 = ctx.launch_count()
    assert_same(device(ctx, *args), emu_boxes(*args))
    assert ctx.launch_count() == n0 + 1


@pytest.mark.parametrize('L', [1, 1021])
def test_device_equals_the_emulation_at_the_rec_length_bounds(ctx, L):
    args = fabricate(10 + L, N=24 if L > 1 else 200, L=L)
    assert_same(device(ctx, *args), emu_boxes(*args))


def test_device_equals_the_emulation_on_hand_made_words(ctx):
    args = hand_made_words()
    assert_same(device(ctx, *args), emu_boxes(*args))


def test_device_equals_the_emulation_at_16_pages_x_4096_words_in_one_launch(ctx):
    polys, rec, loc, fi, frames = fabricate(99, N=16 * 4096, F=16 * 12, nan=0.001)
    n0 = ctx.launch_count()
    got = device(ctx, polys, rec, loc, fi, frames)
    assert ctx.launch_count() == n0 + 1
    assert_same(got, emu_boxes(polys, rec, loc, fi, frames))
    assert int(got['n_chars'].sum()) > 16 * 4096 * 5


def test_no_words_no_launch(ctx):
    args = fabricate(1, N=0)
    n0 = ctx.launch_count()
    got = device(ctx, *args)
    assert ctx.launch_count() == n0 and got['n_chars'].shape == (0,)


def test_refusals_return_invalid_and_leave_the_context_usable(ctx):
    c = ctx
    polys, rec, loc, fi, frames = fabricate(4, N=8)
    frames = np.ascontiguousarray(frames, np.int32)
    N, L = rec.shape
    outs = [np.zeros(N, np.int32), np.zeros((N, L), np.int32), np.zeros((N, L, 2)), np.zeros((N, L, 3)),
            np.zeros((N, L, 8))]
    polys, rec, loc, fi = (np.ascontiguousarray(a, d) for a, d in
                           ((polys, np.float64), (rec, np.int64), (loc, np.float32), (fi, np.int32)))

    def call(n=N, l=L, p=polys, r=rec, lo=loc, f=fi, nf=len(frames), fr=frames, out=None):
        ptr = lambda a: None if a is None else a.ctypes.data
        o = [ptr(a) for a in (outs if out is None else out)]
        return c.lib.alm_omni_char_boxes(c.h, n, l, ptr(p), ptr(r), ptr(lo), ptr(f), nf, ptr(fr), PAD, EOS, *o)

    def bad_frame(col, value):
        fr = frames.copy()
        fr[0, col] = value
        return fr

    n0 = c.launch_count()
    tall = frames.copy()
    th = tall[0, 1] if tall[0, 2] % 2 else tall[0, 0]
    tall[0, 3], tall[0, 5] = 1, th
    for rc in [call(n=-1), call(l=0), call(l=1022), call(p=None), call(r=None), call(lo=None), call(f=None),
               call(fr=None), call(out=[None] + outs[1:]), call(out=outs[:4] + [None]), call(nf=0),
               call(f=np.full(N, len(frames), np.int32)), call(f=np.full(N, -1, np.int32)), call(fr=bad_frame(2, 4)),
               call(fr=bad_frame(2, -1)), call(fr=bad_frame(0, 0)), call(fr=bad_frame(1, -3)), call(fr=bad_frame(5, 0)),
               call(fr=bad_frame(6, -1)), call(fr=bad_frame(3, -1)), call(fr=bad_frame(4, -1)), call(fr=tall)]:
        assert rc == ERR_INVALID
    assert c.launch_count() == n0
    assert call(n=0, p=None, r=None, lo=None, f=None, fr=None, nf=0) == 0   # nothing to do, nothing read
    assert call() == 0
    want = emu_boxes(polys, rec, loc, fi, frames)
    assert_same(dict(zip(KEYS, outs)), want)


# ---- spot_tiled and read_regions


def test_turned_pages_give_the_boxes_of_the_turned_page_read_upright():
    """Turn k of the two fixture pages: the words' 'chars' equal the rule applied to np.rot90(page, k) read upright
    (its polygons mapped to the page, its ids and locations), bit for bit: the turned tiles are pixel permutations."""
    gold = golden('omni_page_turns.npz')
    m = omni_model(gold)
    for page in pages()[:2]:
        H, W = page.shape[:2]
        for k in range(4):
            got = m.spot_tiled([page], orientation=[k], rec_locations=True, **kw(gold))[0]
            up = m.spot_tiled([np.ascontiguousarray(np.rot90(page, k))], rec_locations=True, **kw(gold))[0]
            t = m.last_tiles
            assert len(got) == len(up) and len(got) > 0
            src = t['merged']['source']
            polys = np.array([map_back(k, x, y, H, W) for x, y in t['merged']['polys'].reshape(-1, 2)]).reshape(-1, 32)
            assert np.array_equal(polys, np.array([d['polys'] for d in got]).reshape(-1, 32))
            want = oracle_chars(m, [(H, W)], t['plan'], [k], polys, t['merged']['rec'], t['loc'][src[:, 0], src[:, 1]],
                                src[:, 0])
            assert sum(len(c) for c in want) > 0
            for d, w_ in zip(got, want):
                same_chars(d['chars'], w_)


def test_locations_change_nothing_else():
    gold = golden('omni_page_turns.npz')
    m = omni_model(gold)
    pg = pages()
    for orientation in ['upright', [1, 0, 3, 2], 'auto', 'mixed']:
        off = m.spot_tiled(pg, orientation=orientation, **kw(gold))
        on = m.spot_tiled(pg, orientation=orientation, rec_locations=True, **kw(gold))
        assert without_chars(on) == off
        assert all('chars' in d for r in on for d in r)
        assert all(len(d['chars']) == len(d['rec']) for r in on for d in r)


@pytest.mark.parametrize('orientation', ['auto', 'mixed', 'upright'])
def test_chars_come_from_the_kept_reading(orientation):
    """Each word's 'chars' are the rule applied to the locations of the tile instance its 'tile' / 'instance' (and,
    for 'mixed', 'turns') name; 'auto' reads the one-tile page from its probe.  max_batch 1 / 5 / 16 agree."""
    gold = golden('omni_page_turns.npz')
    m = omni_model(gold)
    pg = pages()
    sizes = [p.shape[:2] for p in pg]
    res = m.spot_tiled(pg, orientation=orientation, max_batch=5, rec_locations=True, **kw(gold))
    t = m.last_tiles
    plan = t['plan']
    mixed = orientation == 'mixed'
    reading = lambda p, d: 4 * p + d['turns'] if mixed else p
    first = np.searchsorted(plan[:, 0], np.arange(4 * len(pg) if mixed else len(pg)))
    words = [(p, d) for p, r in enumerate(res) for d in r]
    assert words
    tile = np.array([first[reading(p, d)] + d['tile'] for p, d in words])
    inst = np.array([d['instance'] for _, d in words])
    rec = (t['turn_merge'] if mixed else t['merged'])['rec']
    polys = np.array([d['polys'] for _, d in words]).reshape(-1, 32)
    want = oracle_chars(m, [s for s in sizes for _ in range(4)] if mixed else sizes, plan,
                        t.get('turns'), polys, rec, t['loc'][tile, inst], tile)
    for (_, d), w_ in zip(words, want):
        same_chars(d['chars'], w_)
    if orientation == 'auto':   # the one-tile page's tile row is its probe reading at the chosen turn
        p = 2
        j = int(np.nonzero(plan[:, 0] == p)[0][0])
        assert np.array_equal(t['loc'][j], t['probe'][5][4 * p + int(t['turns'][p])])
    for mb in (1, 16):
        other = m.spot_tiled(pg, orientation=orientation, max_batch=mb, rec_locations=True, **kw(gold))
        assert without_chars(other) == without_chars(res) or mb == 16
        for ra, rb in zip(other, res):
            assert len(ra) == len(rb)
            for a, b in zip(ra, rb):
                assert [c['char'] for c in a['chars']] == [c['char'] for c in b['chars']]
                for ca, cb in zip(a['chars'], b['chars']):
                    assert np.abs(ca['centre'] - cb['centre']).max() <= 0.02
                    assert np.abs(ca['cov'] - cb['cov']).max() <= 1e-3 * np.trace(cb['cov']) + 0.02
                    assert np.abs(ca['box'] - cb['box']).max() <= 0.1


def test_read_regions_at_decode_points_gives_spot_tiled_chars():
    """On a page of one tile, read_regions at the words' own points reproduces the decode (read_at), so its 'chars'
    equal spot_tiled's bit for bit; on the larger pages each region's chars follow the rule in its own frame."""
    gold = golden('omni_page_turns.npz')
    m = omni_model(gold)
    pg = pages()
    res = m.spot_tiled([pg[2]], rec_locations=True, **kw(gold))[0]
    assert res
    pts = np.array([d['pts'][0] for d in res])
    reg = m.read_regions([pg[2]], pts, np.zeros(len(pts), np.int64), kind='point', rec_locations=True, **kw(gold))
    for a, b in zip(reg, res):
        assert a['rec'] == b['rec'] and a['polys'] == b['polys']
        same_chars(a['chars'], b['chars'])
    # every page, in tiles and on pages read whole: the rule on each region's own reading in its own frame
    sizes = [p.shape[:2] for p in pg]
    words = m.spot_tiled(pg, **kw(gold))
    whole = lambda H, W: np.concatenate([np.stack([np.linspace(1, W - 1, 8), np.full(8, 1.0)], 1),
                                         np.stack([np.linspace(W - 1, 1, 8), np.full(8, H - 1.0)], 1)])
    polys = np.array([d['polys'] for r in words for d in r] + [whole(*sizes[0]), whole(*sizes[3])], np.float32)
    page_index = np.concatenate([np.repeat(np.arange(len(pg)), [len(r) for r in words]), [0, 3]])
    reg = m.read_regions(pg, polys, page_index, kind='polygon', rec_locations=True, **kw(gold))
    lr = m.last_regions
    assert (lr['route'] < 0).any() and (lr['route'] >= 0).any()
    frames = np.concatenate([lr['plan'], [(p, 0, 0) + tuple(sizes[p]) for p in range(len(pg))]])
    fi = np.where(lr['route'] >= 0, lr['route'], len(lr['plan']) + page_index)
    rec = np.zeros((len(reg), m.vocab.rec_length), np.int64)   # each region's ids, from its chunk's image
    for c in lr['chunks']:
        for j, i in enumerate(c['index']):
            rows = np.nonzero(lr['route'] == i)[0] if c['kind'] == 'tile' else \
                np.nonzero((lr['route'] < 0) & (page_index == i))[0]
            rec[rows] = c['rec'][j, :len(rows)]
    want = oracle_chars(m, sizes, frames, None, np.array([d['polys'] for d in reg]).reshape(-1, 32), rec,
                        m.last_rec_locations, fi)
    for d, w_ in zip(reg, want):
        same_chars(d['chars'], w_)


def test_off_by_default_and_refusals():
    """rec_locations=False is the default: the same words and launches; with locations on, launches are added, and a
    later call without them is back to the default's words and launches."""
    gold = golden('omni_page_turns.npz')
    m = omni_model(gold)
    pg = pages()

    def run(**extra):
        n0 = m.ctx.launch_count()
        res = m.spot_tiled(pg, **kw(gold, **extra))
        return res, m.ctx.launch_count() - n0

    base, n = run()
    assert run(rec_locations=False) == (base, n)
    assert not any('chars' in d for r in base for d in r) and 'loc' not in m.last_tiles
    assert run(rec_locations=True)[1] > n
    assert run() == (base, n)
    with pytest.raises(ValueError):
        m.spot_tiled(pg, whole_page=True, rec_locations=True, **kw(gold))
    with pytest.raises(ValueError):
        m.read_regions(pg[:1], np.array([[10.0, 10.0]]), [0], kind='point', rec_beams=2, rec_locations=True,
                       **kw(gold))
    assert run() == (base, n)
