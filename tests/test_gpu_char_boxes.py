"""GPU: where each recognised character is -- char_box_kernel reduces MGP-STR's A^3 maps to page-space boxes
(alm_mgpstr_forward_boxes, recognize* with char_boxes=True).  Bar: the device boxes equal the oracle bit for bit when
the oracle is fed the device's own maps (read back through forward(is_eval=True)); ids and probabilities are the same
bits with boxes on and off; boxes add exactly one launch per head."""
import numpy as np
import pytest
import torch

from tests.support import emu, mgp_model, options, release_models
from tests.test_char_boxes_cpu import bind, emu_char_boxes
from tests.test_curve_crops_cpu import curve_fixture, curve_regions
from tests.test_quad_crops_cpu import quad_fixture

pytestmark = pytest.mark.gpu
ALM_ERR_INVALID, ALM_ERR_STATE = -1, -4


@pytest.fixture(scope='module')
def model():
    return mgp_model()


def device_maps(m, crops):
    """The A^3 maps [3][B, 27, 257] and top-1 ids [3, B, 27] the device computes for crops."""
    out = m.forward(crops, is_eval=True, want_logits=False)
    return [a.numpy() for a in out[0]], m.last_ids.numpy().copy()


def chunked_maps(m, crop, pages, regions, pidx, max_batch):
    maps, ids = [], []
    for s in range(0, len(pidx), max_batch):
        a, i = device_maps(m, crop(m.ctx, pages, regions[s:s + max_batch], pidx[s:s + max_batch]))
        maps.append(a)
        ids.append(i)
    return [np.concatenate([a[h] for a in maps]) for h in range(3)], np.concatenate(ids, axis=1)


def assert_oracle(maps, ids, got, kind, sizes=None, geom=None, rows=None):
    from oracle import char_box_ref as V
    n, boxes, centres = (np.asarray(v) for v in got)
    rows = np.arange(ids.shape[1]) if rows is None else rows
    for h in range(3):
        want = V.char_boxes(maps[h][rows], ids[h][rows], h, kind, None if sizes is None else sizes[rows],
                            None if geom is None else geom[rows])
        assert np.array_equal(n[h][rows], want[0]), h
        assert np.array_equal(boxes[h][rows].view(np.uint32), want[1].view(np.uint32)), h
        assert np.array_equal(centres[h][rows].view(np.uint32), want[2].view(np.uint32)), h


@pytest.mark.parametrize('nsplit', [3, 1])
def test_boxes_equal_oracle_on_device_maps(model, nsplit):
    """recognize, recognize_regions (quad fixture, chunks of 7) and recognize_polygons (curve fixture, chunks of 16):
    every box and centre equals the oracle's on the device's own maps and ids, and ids / probs equal the path
    without boxes bit for bit."""
    from advancedliteratemachinery_b200 import _lib, preprocess as P
    m = model
    with options(m.ctx, nsplit=nsplit):
        zc, cpages, ccrops, _ = curve_fixture()
        crops = P.mgp_crops(m.ctx, ccrops)
        ref_ids, ref_prob = m.recognize(crops)
        ids, prob, *got = m.recognize(crops, char_boxes=True)
        assert torch.equal(ids, ref_ids) and torch.equal(prob.view(torch.int32), ref_prob.view(torch.int32))
        maps, dids = device_maps(m, crops)
        assert np.array_equal(dids, ids.numpy())
        assert_oracle(maps, dids, got, _lib.BOX_CROP)
        assert (got[0][1:] > 0).any()

        zq, qpages, _, _ = quad_fixture()
        ref = m.recognize_regions(qpages, zq['quads'], zq['page_index'], max_batch=7)
        ids, prob, *got = m.recognize_regions(qpages, zq['quads'], zq['page_index'], max_batch=7, char_boxes=True)
        assert torch.equal(ids, ref[0]) and torch.equal(prob.view(torch.int32), ref[1].view(torch.int32))
        dev = [torch.from_numpy(p).cuda() for p in qpages]
        maps, dids = chunked_maps(m, P.quad_crops, dev, zq['quads'], zq['page_index'], 7)
        assert np.array_equal(dids, ids.numpy())
        plan = P.quad_plan([p.shape[:2] for p in qpages], zq['quads'], zq['page_index'])
        assert_oracle(maps, dids, got, _lib.BOX_QUAD, plan['sizes'], plan['minv'])

        ref = m.recognize_polygons(cpages, zc['polys'], zc['page_index'], max_batch=16)
        ids, prob, *got = m.recognize_polygons(cpages, zc['polys'], zc['page_index'], max_batch=16, char_boxes=True)
        assert torch.equal(ids, ref[0]) and torch.equal(prob.view(torch.int32), ref[1].view(torch.int32))
        dev = [torch.from_numpy(p).cuda() for p in cpages]
        maps, dids = chunked_maps(m, P.curve_crops, dev, zc['polys'], zc['page_index'], 16)
        assert np.array_equal(dids, ids.numpy())
        plan = P.curve_plan([p.shape[:2] for p in cpages], zc['polys'], zc['page_index'])
        assert_oracle(maps, dids, got, _lib.BOX_CURVE, plan['sizes'], plan['ctrl'])


def test_thousand_regions_equal_oracle(model):
    """1 024 curved regions on 16 pages (two chunks of 512) through recognize_polygons, and their corner quads through
    recognize_regions: every box equals the host run of the kernel body on the device's maps, and the oracle on 64
    regions spread over both chunks."""
    from advancedliteratemachinery_b200 import _lib, postprocess as Post, preprocess as P
    m = model
    pages, polys, pidx = curve_regions(seed=5)
    dev = [torch.from_numpy(p).cuda() for p in pages]
    sizes = [p.shape[:2] for p in pages]
    lib = emu('char_box_emu', bind)
    rows = np.arange(0, 1024, 16)
    quads = Post.quads_from_polygons(polys)
    for kind, crop, regions, recog, planner in (
            (_lib.BOX_CURVE, P.curve_crops, polys, m.recognize_polygons, lambda: P.curve_plan(sizes, polys, pidx)),
            (_lib.BOX_QUAD, P.quad_crops, quads, m.recognize_regions, lambda: P.quad_plan(sizes, quads, pidx))):
        ids, prob, *got = recog(dev, regions, pidx, char_boxes=True)
        assert ids.shape == (3, 1024, 27) and got[1].shape == (3, 1024, 26, 4, 2)
        maps, dids = chunked_maps(m, crop, dev, regions, pidx, 512)
        assert np.array_equal(dids, ids.numpy())
        plan = planner()
        geom = plan['ctrl'] if kind == _lib.BOX_CURVE else plan['minv']
        for h in range(3):
            want = emu_char_boxes(lib, maps[h], dids[h], h, kind, plan['sizes'], geom)
            assert np.array_equal(got[0][h].numpy(), want[0])
            assert np.array_equal(got[1][h].numpy().view(np.uint32), want[1].view(np.uint32))
            assert np.array_equal(got[2][h].numpy().view(np.uint32), want[2].view(np.uint32))
        assert_oracle(maps, dids, got, kind, plan['sizes'], geom, rows)


def test_launches_empty_input_and_candidates(model):
    """Boxes on adds exactly n_a3 launches per chunk; R = 0 gives empty outputs; with k candidates the ids / probs
    are recognize_polygons(k=4)'s and the boxes follow the top-1 ids."""
    m = model
    zc, cpages, _, _ = curve_fixture()
    dev = [torch.from_numpy(p).cuda() for p in cpages]
    R = len(zc['page_index'])
    counts = []
    for boxes in (False, True):
        m.ctx.launch_count(reset=True)
        m.recognize_polygons(dev, zc['polys'], zc['page_index'], max_batch=32, char_boxes=boxes)
        counts.append(m.ctx.launch_count())
    chunks = -(-R // 32)
    assert counts[1] - counts[0] == 3 * chunks, counts
    out = m.recognize_polygons(dev, np.zeros((0, 16, 2)), [], char_boxes=True)
    assert [tuple(t.shape) for t in out] == [(3, 0, 27), (3, 0, 27), (3, 0), (3, 0, 26, 4, 2), (3, 0, 26, 2)]
    ref = m.recognize_polygons(dev, zc['polys'], zc['page_index'], k=4, max_batch=16)
    top1 = m.recognize_polygons(dev, zc['polys'], zc['page_index'], max_batch=16, char_boxes=True)
    ids, prob, *got = m.recognize_polygons(dev, zc['polys'], zc['page_index'], k=4, max_batch=16, char_boxes=True)
    assert torch.equal(ids, ref[0]) and torch.equal(prob.view(torch.int32), ref[1].view(torch.int32))
    for a, b in zip(got, top1[2:]):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))


def test_fused_boxes_follow_the_winning_head(model):
    from advancedliteratemachinery_b200 import postprocess as Post, preprocess as P
    from oracle.char_box_ref import CHAR_TABLE
    m = model
    _, _, ccrops, _ = curve_fixture()
    ids, prob, n, boxes, centres = m.recognize(P.mgp_crops(m.ctx, ccrops), char_boxes=True)
    fuse = Post.mgp_fuse(ids, prob, CHAR_TABLE, [f'b{i}' for i in range(50257)], [f'w{i}' for i in range(30522)])
    out = Post.fused_boxes(fuse, n, boxes, centres)
    assert len(out) == ids.shape[1]
    for b, d in enumerate(out):
        src = int(fuse['source'][b])
        k = int(n[src, b]) if src >= 0 else 0
        assert d['text'] == fuse['fused'][b] and d['boxes'].shape == (k, 4, 2)
        if k:
            assert np.array_equal(d['boxes'], boxes[src, b, :k].numpy()) and np.array_equal(d['centres'],
                                                                                          centres[src, b, :k].numpy())


def test_charstr_gives_char_boxes_only():
    from advancedliteratemachinery_b200 import MGPSTRB200, _lib, preprocess as P
    from advancedliteratemachinery_b200 import synthetic as W
    dim, depth, heads = W.MGP_VARIANTS['base']
    m = MGPSTRB200(W.mgpstr_state_dict(seed=3, dim=dim, depth=depth, heads=heads, char_only=True))
    try:
        _, _, ccrops, _ = curve_fixture()
        crops = P.mgp_crops(m.ctx, ccrops[:12])
        ids, prob, n, boxes, centres = m.recognize(crops, char_boxes=True)
        ref_ids, _ = m.recognize(crops)
        assert torch.equal(ids[0], ref_ids[0])
        assert not n[1:].any() and not boxes[1:].any() and not centres[1:].any()
        maps, dids = device_maps(m, crops)
        from oracle import char_box_ref as V
        want = V.char_boxes(maps[0], dids[0], 0, _lib.BOX_CROP)
        assert np.array_equal(n[0].numpy(), want[0]) and np.array_equal(boxes[0].numpy().view(np.uint32),
                                                                         want[1].view(np.uint32))
        # three head planes against a one-head checkpoint
        raw = _raw_call(m, crops, n_heads=3)
        assert raw == ALM_ERR_INVALID
    finally:
        m.ctx.close()


def _raw_call(m, crops, B=None, k=0, kind=0, n_geom=None, sizes=None, geom=None, n_heads=None):
    B = crops.shape[0] if B is None else B
    bufs = [np.zeros(3 * B * 27 * max(k, 1), np.int32), np.zeros(3 * B * 27 * max(k, 1), np.float32),
            np.zeros(3 * B, np.int32), np.zeros(3 * B * 26 * 8, np.float32), np.zeros(3 * B * 26 * 2, np.float32)]
    ptr = lambda a: a.ctypes.data if a is not None else None
    return m.lib.alm_mgpstr_forward_boxes(m.ctx.h, crops.data_ptr(), B, k, kind, B if n_geom is None else n_geom,
                                          ptr(sizes), ptr(geom), m.info()['n_a3'] if n_heads is None else n_heads,
                                          *[b.ctypes.data for b in bufs])


def test_error_paths_leave_the_context_usable(model):
    from advancedliteratemachinery_b200 import _lib, preprocess as P
    m = model
    _, _, ccrops, _ = curve_fixture()
    crops = P.mgp_crops(m.ctx, ccrops[:4])
    sizes = np.full((4, 2), 20, np.int32)
    quad = np.tile(np.eye(3).reshape(1, 9), (4, 1))
    curve = np.zeros((4, 16))
    nan = quad.copy(); nan[2, 4] = np.nan
    inf = curve.copy(); inf[1, 9] = np.inf
    zero = sizes.copy(); zero[3, 0] = 0
    cases = [dict(kind=3), dict(kind=-1), dict(kind=1, n_geom=3, sizes=sizes, geom=quad), dict(kind=1, geom=quad),
             dict(kind=2, sizes=sizes), dict(kind=1, sizes=sizes, geom=nan), dict(kind=2, sizes=sizes, geom=inf),
             dict(kind=1, sizes=zero, geom=quad), dict(n_heads=1), dict(k=9), dict(k=-1), dict(B=0)]
    for kw in cases:
        assert _raw_call(m, crops, **kw) == ALM_ERR_INVALID, kw
    empty = _lib.Context(0)
    buf = np.zeros(3 * 4 * 26 * 8, np.float32)
    try:
        rc = empty.lib.alm_mgpstr_forward_boxes(empty.h, crops.data_ptr(), 4, 0, 0, 4, None, None, 3,
                                                *[buf.ctypes.data] * 5)
        assert rc == ALM_ERR_STATE
    finally:
        empty.close()
    assert _raw_call(m, crops, kind=1, sizes=sizes, geom=quad) == 0
    ref_ids, ref_prob = m.recognize(crops)
    ids, prob, *got = m.recognize(crops, char_boxes=True)
    assert torch.equal(ids, ref_ids) and torch.equal(prob.view(torch.int32), ref_prob.view(torch.int32))
    maps, dids = device_maps(m, crops)
    assert_oracle(maps, dids, got, _lib.BOX_CROP)
