"""GPU: pages spotted in overlapping tiles (preprocess.omni_tiles, alm_omni_merge_tiles, OmniParserB200.spot_tiled).
Tile inputs must equal omni_pages of the host-sliced tiles bit for bit; every tile must get forward_pages' result;
spot_tiled on the fixture page must equal tests/golden/omni_tiles.npz (the unmodified reference run on every tile and
merged by oracle/tile_ref.py); and the device merge must equal the host build of the same bodies (tests/emu/tile_emu.cpp)
bit for bit, on the device's own tile outputs and on 16 pages x 12 tiles x 512 fabricated instances."""
import numpy as np
import pytest
import torch

from tests.support import assert_same, golden, kw, omni_model, release_models
from tests.test_tiles_cpu import emu_merge, fabricate

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)


def sliced(pages, plan):
    return [np.ascontiguousarray(pages[p][y:y + h, x:x + w]) for p, y, x, h, w in plan.tolist()]


def second_page():
    """A page no larger than one tile of the fixture's layout, of another size (its tiles need encode_pages)."""
    return np.random.default_rng(5).integers(0, 256, (100, 90, 3), dtype=np.uint8)


def test_tile_inputs_equal_omni_pages_of_sliced_tiles():
    """Several pages (one smaller than a tile on one axis, host and device pages), whole plan and sub-ranges."""
    from advancedliteratemachinery_b200 import _lib, preprocess as P
    ctx = _lib.Context(0)
    try:
        rng = np.random.default_rng(1)
        pages = [rng.integers(0, 256, s + (3,), dtype=np.uint8) for s in ((300, 220), (90, 400), (128, 128), (77, 60))]
        for T, ov, mn, mx in ((128, 32, 128, 256), (100, 50, 80, 333), (200, 0, 256, 256)):
            plan = P.omni_tile_plan([p.shape[:2] for p in pages], T, ov)
            for first, count in ((0, None), (1, 3), (len(plan) - 2, 2)):
                src = pages if first else [torch.from_numpy(p).cuda() for p in pages]
                got = P.omni_tiles(ctx, src, T, ov, mn, mx, first, count)
                sel = plan[first:first + (len(plan) - first if count is None else count)]
                want = P.omni_pages(ctx, sliced(pages, sel), mn, mx)
                assert torch.equal(got.tensors.view(torch.int32), want.tensors.view(torch.int32))
                assert torch.equal(got.mask, want.mask)
    finally:
        ctx.close()


def test_spot_tiled_equals_the_fixture():
    """ids exact, coordinates exact (page and tile frame), probabilities close; every tile's decode equals
    forward_pages on the sliced tiles bit for bit; the merge equals the emulation fed the device's own tile outputs."""
    from advancedliteratemachinery_b200 import preprocess as P
    gold = golden('omni_tiles.npz')
    m = omni_model(gold)
    page = gold['page']
    res = m.spot_tiled([page], **kw(gold))
    t = m.last_tiles
    assert np.array_equal(t['plan'], gold['plan'])
    for k in ('n_inst', 'pt', 'poly', 'rec'):
        assert np.array_equal(t[k], gold[k]), k
    np.testing.assert_allclose(t['prob'], gold['prob'], rtol=2e-3, atol=1e-7)
    mg = t['merged']
    for k in ('count', 'offset', 'pts', 'polys', 'rec', 'source'):
        assert np.array_equal(mg[k], gold[f'merged_{k}']), k
    # the device merge == the host build of the same bodies on the device's own tile outputs, probabilities included
    assert_same(mg, emu_merge([page.shape[:2]], int(gold['tile']), int(gold['overlap']), t['n_inst'], t['pt'], t['poly'],
                              t['rec'], t['prob'], m.vocab.num_bins))
    # every tile: forward_pages of the host-sliced tiles, bit for bit
    nt = P.omni_pages(m.ctx, sliced([page], t['plan']), int(gold['test_min_size']), int(gold['test_max_size']))
    outs = m.forward_pages(nt)
    for k, o in enumerate(outs):
        n = int(t['n_inst'][k])
        assert (o is None) == (n == 0)
        if o is None:
            continue
        (pt, poly, rec), (prob,) = o
        assert np.array_equal(pt.numpy().reshape(n, 2), t['pt'][k, :n])
        assert np.array_equal(poly.numpy().reshape(n, 32), t['poly'][k, :n])
        assert np.array_equal(rec.numpy()[0], t['rec'][k, :n])
        assert np.array_equal(prob.numpy().view(np.uint32), t['prob'][k, :n].view(np.uint32))
    assert len(res) == 1 and len(res[0]) == int(gold['merged_count'][0])
    for r, d in enumerate(res[0]):
        assert d['pts'] == [gold['merged_pts'][r].tolist()] and d['polys'] == gold['merged_polys'][r].reshape(16, 2).tolist()
        assert (d['tile'], d['instance']) == tuple(gold['merged_source'][r])


def test_single_tile_page_equals_decode_pred_seq():
    """A page no larger than one tile: exactly decode_pred_seq of forward_pages on that page."""
    from advancedliteratemachinery_b200 import postprocess as Post, preprocess as P
    gold = golden('omni_tiles.npz')
    m = omni_model(gold)
    page = second_page()
    res = m.spot_tiled([page], **kw(gold))[0]
    out = m.forward_pages(P.omni_pages(m.ctx, [page], int(gold['test_min_size']), int(gold['test_max_size'])))[0]
    assert out is not None
    want = Post.decode_pred_seq(out[0], out[1], {'file_name': 'p', 'orig_size': page.shape[:2]}, m.vocab)
    assert [{k: v for k, v in d.items() if k not in ('tile', 'instance')} for d in res] == \
        [{k: v for k, v in d.items() if k != 'image_id'} for d in want]
    assert [(d['tile'], d['instance']) for d in res] == [(0, i) for i in range(len(want))]


def test_chunk_sizes_agree_and_other_outputs_are_unchanged():
    """max_batch 1 / 5 / 16 over two pages of different sizes (chunks through encode and encode_pages) give one
    result; decode / forward_pages on other inputs are the same before and after a tiled call; the merge is three
    launches."""
    from advancedliteratemachinery_b200 import NestedTensor, OmniParserB200, preprocess as P
    from advancedliteratemachinery_b200.omniparser import merge_tiles
    gold = golden('omni_tiles.npz')
    m = omni_model(gold)
    pages = [gold['page'], second_page()]
    probe = P.omni_pages(m.ctx, [second_page(), gold['page'][:120, :150]], 128, 256)
    before = m.forward_pages(probe)
    m.encode(probe.tensors[:1, :, :142, :128])
    dec_before = m.decode()
    runs = [m.spot_tiled(pages, max_batch=b, **kw(gold)) for b in (1, 5, 16)]
    assert runs[0] == runs[1] == runs[2] and len(runs[0]) == 2 and len(runs[0][1]) > 0
    t = m.last_tiles
    m.ctx.launch_count(reset=True)
    merge_tiles(m.ctx, [p.shape[:2] for p in pages], int(gold['tile']), int(gold['overlap']), t['plan'], t['n_inst'],
                t['pt'], t['poly'], t['rec'], t['prob'], m.vocab.num_bins)
    assert m.ctx.launch_count() == 3
    after = m.forward_pages(NestedTensor(probe.tensors, probe.mask))
    m.encode(probe.tensors[:1, :, :142, :128])
    assert repr(m.decode()) == repr(dec_before) and repr(after) == repr(before)
    kie = OmniParserB200(None, type(m.vocab)(vie_categories=4))
    with pytest.raises(ValueError):
        kie.spot_tiled(pages)
    kie.ctx.close()


def test_merge_at_scale_equals_the_emulation():
    """16 pages x 12 tiles x 512 fabricated instances (2480 x 3508 pages, T 1200, ov 256): device == host build."""
    from advancedliteratemachinery_b200 import _lib
    from advancedliteratemachinery_b200.omniparser import merge_tiles
    from advancedliteratemachinery_b200 import preprocess as P
    rng = np.random.default_rng(11)
    sizes = [(3508, 2480)] * 16
    plan = P.omni_tile_plan(sizes, 1200, 256)
    assert len(plan) == 192
    outs = fabricate(rng, sizes, 1200, 256, 512, 25, 1000, 3000)
    assert (outs[0] == 512).mean() > 0.5
    ctx = _lib.Context(0)
    try:
        got = merge_tiles(ctx, sizes, 1200, 256, plan, *outs, 1000)
        assert_same(got, emu_merge(sizes, 1200, 256, *outs, 1000))
        assert 0 < int(got['count'].sum()) < int(outs[0].sum())
        got = merge_tiles(ctx, sizes, 1200, 256, plan, *outs, 1000, margin=0.0, band=0.0, iou=0.3)
        assert_same(got, emu_merge(sizes, 1200, 256, *outs, 1000, margin=0.0, band=0.0, iou=0.3))
    finally:
        ctx.close()


def test_error_paths_leave_the_context_usable():
    """Bad tile / overlap / margin / band / iou, a page index out of range, tiles that are not the plan's, n_inst out
    of range and a short capacity are refused before any device work; the context merges correctly afterwards."""
    from advancedliteratemachinery_b200 import _lib, preprocess as P
    from advancedliteratemachinery_b200.omniparser import merge_tiles
    gold = golden('omni_tiles.npz')
    m = omni_model(gold)
    sizes = [gold['page'].shape[:2]]
    T, ov = int(gold['tile']), int(gold['overlap'])
    plan = gold['plan']
    outs = [gold[k] for k in ('n_inst', 'pt', 'poly', 'rec', 'prob')]
    for bad in (dict(margin=float('nan')), dict(margin=-1), dict(band=float('inf')), dict(iou=0.0), dict(iou=1.5)):
        with pytest.raises(ValueError):
            merge_tiles(m.ctx, sizes, T, ov, plan, *outs, 1000, **bad)
    with pytest.raises(_lib.AlmError):
        merge_tiles(m.ctx, sizes, 63, 0, plan, *outs, 1000)
    with pytest.raises(_lib.AlmError):
        merge_tiles(m.ctx, sizes, T, T // 2 + 1, plan, *outs, 1000)
    for col, val in ((0, 1), (0, -1), (1, 5)):   # page index out of range, origin not the plan's
        p2 = plan.copy()
        p2[2, col] = val
        with pytest.raises(_lib.AlmError):
            merge_tiles(m.ctx, sizes, T, ov, p2, *outs, 1000)
    n2 = outs[0].copy()
    n2[0] = outs[1].shape[1] + 1
    with pytest.raises((_lib.AlmError, ValueError)):
        merge_tiles(m.ctx, sizes, T, ov, plan, n2, *outs[1:], 1000)
    with pytest.raises(_lib.AlmError):
        P.omni_tiles(m.ctx, [gold['page']], 63, 0)
    with pytest.raises(ValueError):
        P.omni_tiles(m.ctx, [gold['page']], T, ov, first=len(plan))
    got = merge_tiles(m.ctx, sizes, T, ov, plan, *outs, 1000)
    assert np.array_equal(got['source'], gold['merged_source'])
