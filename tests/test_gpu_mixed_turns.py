"""GPU: pages read at all four quarter-turns and merged (omniparser.merge_turns, OmniParserB200.spot_tiled(
orientation='mixed'); DESIGN 4.15).  The device merge must equal the host build of its kernels' bodies bit for bit
in three launches; each of the four readings must be the explicit-turn reading; the merged result must equal
oracle/turn_merge_ref.py on tests/golden/omni_page_turns.npz (the reference's four readings of one page) and on the
device's own readings; and no other orientation may change."""
import numpy as np
import pytest
import torch

from oracle import turn_merge_ref as R
from tests.support import assert_same, golden, kw, omni_model, release_models, same
from tests.test_turn_merge_cpu import EOS, PAD, emu_merge, fixture_rows

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

ERR_INVALID = -1  # include/alm_ocr.h ALM_ERR_INVALID


def pages(gold):
    """The fixture page (larger than T), a page of 2 x 3 tiles and one smaller than a tile."""
    rng = np.random.default_rng(21)
    return [gold['page'], rng.integers(0, 256, (230, 301, 3), dtype=np.uint8),
            rng.integers(0, 256, (97, 120, 3), dtype=np.uint8)]


def large_rows(rng, P=16, n=4096, L=25):
    """P pages x 4 readings x n rows of words on a 2 000 x 2 000 page: every reading sees jittered copies of the
    page's words, scores from a few probabilities (ties), so that cross-turn overlaps around 0.5 are common."""
    R4 = 4 * P
    count = np.full(R4, n, np.int32)
    offset = (np.cumsum(count) - count).astype(np.int32)
    words = rng.uniform(0, 2000, (P, n, 2))
    size = rng.uniform([10, 5], [120, 40], (P, n, 2))
    base = np.repeat(np.concatenate([words, words + size], 2), 4, 0)  # [R4, n, 4]
    box = base + rng.normal(0, 0.15, base.shape) * np.tile(np.repeat(size, 4, 0), 2)
    t = np.linspace(0, 1, 8)
    xs = np.concatenate([box[..., :1] + t * (box[..., 2:3] - box[..., :1]),
                         box[..., 2:3] + t * (box[..., :1] - box[..., 2:3])], -1)
    ys = np.concatenate([np.repeat(box[..., 1:2], 8, -1), np.repeat(box[..., 3:4], 8, -1)], -1)
    polys = np.stack([xs, ys], -1).reshape(-1, 32)
    pts = np.stack([(box[..., 0] + box[..., 2]) / 2, (box[..., 1] + box[..., 3]) / 2], -1).reshape(-1, 2)
    N = R4 * n
    rec = rng.choice([1000, 1001, PAD - 1, PAD, EOS], (N, L), p=[.4, .3, .1, .1, .1]).astype(np.int64)
    prob = rng.choice([0.25, 0.5, 0.75, 1.0], (N, L)).astype(np.float32)
    return count, offset, pts, polys, rec, prob


def test_device_merge_equals_the_emulation():
    """The fixture's four readings and 16 pages x 4 readings x 4 096 fabricated rows: every output field of the
    device merge equals the host build fed the same inputs, bit for bit, in three launches."""
    from advancedliteratemachinery_b200.omniparser import merge_turns
    m = omni_model(golden('omni_page_turns.npz'))
    args, pad, eos = fixture_rows()
    m.ctx.launch_count(reset=True)
    got = merge_turns(m.ctx, *args, pad, eos)
    assert m.ctx.launch_count() == 3
    assert_same(got, emu_merge(*args, pad=pad, eos=eos))
    big = large_rows(np.random.default_rng(7))
    for iou in (0.5, 0.3):
        m.ctx.launch_count(reset=True)
        got = merge_turns(m.ctx, *big, PAD, EOS, iou)
        assert m.ctx.launch_count() == 3
        want = emu_merge(*big, iou=iou)
        assert_same(got, want)
        assert 0 < int(got['count'].sum()) < len(big[2])


def test_mixed_on_the_fixture():
    """The fixture page at tile 128: the four readings are the explicit-turn readings (and the reference's); the
    result is turn_merge_ref of the fixture's merged_* rows, with 'turns' / 'tile' / 'instance' from the oracle's
    sources, and turn_merge_ref of the device's own readings bit for bit."""
    from advancedliteratemachinery_b200 import postprocess
    gold = golden('omni_page_turns.npz')
    m = omni_model(gold)
    v = m.vocab
    page = gold['page']
    got = m.spot_tiled([page], orientation='mixed', **kw(gold))[0]
    t = m.last_tiles
    assert t['turns'].tolist() == [0, 1, 2, 3] and np.array_equal(t['plan'], gold['plan'])
    rd = t['readings']
    m.spot_tiled([page] * 4, orientation=[0, 1, 2, 3], **kw(gold))
    assert_same(rd, m.last_tiles['merged'])
    first = np.searchsorted(gold['plan'][:, 0], np.arange(4))
    for k in range(4):  # each reading is spot_tiled at that turn
        m.spot_tiled([page], orientation=[k], **kw(gold))
        e = m.last_tiles['merged']
        rows = slice(int(rd['offset'][k]), int(rd['offset'][k] + rd['count'][k]))
        assert_same({f: rd[f][rows] for f in ('pts', 'polys', 'rec', 'prob')},
                    {f: e[f] for f in ('pts', 'polys', 'rec', 'prob')})
        assert np.array_equal(rd['source'][rows] - [first[k], 0], e['source'])
    for k in ('count', 'offset', 'pts', 'polys', 'rec', 'source'):
        assert np.array_equal(rd[k], gold[f'merged_{k}']), k
    pad, eos = v.recog_pad_index, v.rec_eos_index
    assert_same(t['turn_merge'], R.merge(rd['count'], rd['offset'], rd['pts'], rd['polys'], rd['rec'], rd['prob'],
                                         pad, eos))
    want = R.merge(gold['merged_count'], gold['merged_offset'], gold['merged_pts'], gold['merged_polys'],
                   gold['merged_rec'], gold['merged_prob'], pad, eos)
    for k in ('count', 'offset', 'pts', 'polys', 'rec', 'source'):
        assert np.array_equal(t['turn_merge'][k], want[k]), k
    texts, _ = postprocess.rec_texts(want['rec'], want['prob'], v)
    assert len(got) == len(want['source']) > 0
    for d, (k, i), pts, poly, txt in zip(got, want['source'], want['pts'], want['polys'], texts):
        tile, inst = gold['merged_source'][gold['merged_offset'][k] + i]
        assert (d['turns'], d['tile'], d['instance']) == (k, tile - first[k], inst)
        assert d['pts'] == [pts.tolist()] and d['polys'] == poly.reshape(-1, 2).tolist() and d['rec'] == txt


def test_single_tile_pages_read_the_auto_probes():
    """Pages no larger than T: the four tiled readings are 'auto''s probe readings, array for array."""
    gold = golden('omni_page_turns.npz')
    m = omni_model(gold)
    pg = [gold['page'], pages(gold)[2]]
    args = dict(kw(gold), tile=256, overlap=32)
    m.spot_tiled(pg, orientation='auto', **args)
    probe = m.last_tiles['probe']
    m.spot_tiled(pg, orientation='mixed', **args)
    t = m.last_tiles
    assert len(t['plan']) == 4 * len(pg)
    for k, a in zip(('n_inst', 'pt', 'poly', 'rec', 'prob'), probe):
        assert np.array_equal(t[k], a), k


def test_mixed_agrees_across_chunks_page_kinds_and_sizes():
    """max_batch 1 / 5 / 16, host and CUDA pages, every page alone and with the others (pages smaller and larger
    than T): the same result.  In chunks of 16 tiles the decoder's probabilities differ from those of smaller chunks
    in the last bits (its ids and coordinates do not; so do the upright and explicit-turn paths), so there the words,
    their turns, tiles, coordinates and texts are compared exactly and the scores to 1e-5."""
    gold = golden('omni_page_turns.npz')
    m = omni_model(gold)
    pg = pages(gold)
    base = m.spot_tiled(pg, max_batch=5, orientation='mixed', **kw(gold))
    assert all(len(r) > 0 for r in base)
    assert len({d['turns'] for r in base for d in r}) > 1
    same(m.spot_tiled(pg, max_batch=1, orientation='mixed', **kw(gold)), base)
    same(m.spot_tiled([torch.from_numpy(p).cuda() for p in pg], max_batch=5, orientation='mixed', **kw(gold)), base)
    same([m.spot_tiled([p], max_batch=5, orientation='mixed', **kw(gold))[0] for p in pg], base)
    big = m.spot_tiled(pg, max_batch=16, orientation='mixed', **kw(gold))
    drop = lambda res: [[{k: v for k, v in d.items() if k != 'score'} for d in r] for r in res]
    same(drop(big), drop(base))
    np.testing.assert_allclose([d['score'] for r in big for d in r], [d['score'] for r in base for d in r],
                               rtol=1e-5, atol=0)


def test_group_lines_takes_the_result_as_it_is():
    gold = golden('omni_page_turns.npz')
    m = omni_model(gold)
    res = m.spot_tiled(pages(gold), orientation='mixed', **kw(gold))
    lines = m.group_lines(res)
    assert len(lines) == len(res)
    for r, ls in zip(res, lines):
        words = sorted(w for line in ls for w in line['words'])
        assert words == list(range(len(r)))


def test_other_orientations_are_unchanged_by_a_mixed_call():
    gold = golden('omni_page_turns.npz')
    m = omni_model(gold)
    pg = pages(gold)
    modes = ('upright', [1, 3, 2], 'auto')
    before = [m.spot_tiled(pg, orientation=o, **kw(gold)) for o in modes]
    m.spot_tiled(pg, orientation='mixed', **kw(gold))
    for o, b in zip(modes, before):
        same(m.spot_tiled(pg, orientation=o, **kw(gold)), b)


def test_error_paths_leave_the_context_usable():
    """The C entry refuses bad pages / lengths, null buffers, negative counts, offsets that are not the counts'
    prefix sum, a bad iou and a small cap before any device work; the Python entries refuse bad orientations and a
    KIE checkpoint; the context merges correctly afterwards."""
    from advancedliteratemachinery_b200 import OmniParserB200
    from advancedliteratemachinery_b200.omniparser import merge_turns
    gold = golden('omni_page_turns.npz')
    m = omni_model(gold)
    lib, h = m.ctx.lib, m.ctx.h
    args, pad, eos = fixture_rows()
    count, offset = (np.ascontiguousarray(a, np.int32) for a in args[:2])
    pts, polys = (np.ascontiguousarray(a, np.float64) for a in args[2:4])
    rec, prob = np.ascontiguousarray(args[4], np.int64), np.ascontiguousarray(args[5], np.float32)
    N, L = rec.shape
    out = [np.zeros(1, np.int32), np.zeros(1, np.int32), np.zeros((N, 2)), np.zeros((N, 32)),
           np.zeros((N, L), np.int64), np.zeros((N, L), np.float32), np.zeros((N, 2), np.int32)]

    def call(n_pages=1, cnt=count, off=offset, L_=L, iou=0.5, cap=N, null=None):
        ins = [cnt.ctypes.data, off.ctypes.data, pts.ctypes.data, polys.ctypes.data, rec.ctypes.data, prob.ctypes.data]
        outs = [o.ctypes.data for o in out]
        if null is not None:
            if null < len(ins):
                ins[null] = None
            else:
                outs[null - len(ins)] = None
        return lib.alm_omni_merge_turns(h, n_pages, ins[0], ins[1], *ins[2:], L_, pad, eos, iou, *outs[:2],
                                        *outs[2:], cap)

    assert call() == 0
    for bad in (dict(n_pages=0), dict(L_=0), dict(iou=0.0), dict(iou=1.5), dict(iou=float('nan')), dict(cap=N - 1),
                dict(cnt=np.array([6, -1, 7, 5], np.int32)), dict(off=np.array([0, 6, 12, 20], np.int32)),
                dict(off=np.array([1, 7, 14, 21], np.int32))):
        assert call(**bad) == ERR_INVALID, bad
    for slot in range(13):
        assert call(null=slot) == ERR_INVALID, slot
    pg = pages(gold)
    for bad in ('Mixed', 'mixed ', ['mixed']):
        with pytest.raises(ValueError):
            m.spot_tiled(pg, orientation=bad, **kw(gold))
    assert_same(merge_turns(m.ctx, *args, pad, eos), emu_merge(*args, pad=pad, eos=eos))
    kie = OmniParserB200(None, type(m.vocab)(vie_categories=4))
    with pytest.raises(ValueError):
        kie.spot_tiled(pg, orientation='mixed')
    kie.ctx.close()
