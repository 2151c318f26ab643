"""GPU: text read at quarter-turns (alm_pre_turned_crops, alm_mgpstr_forward_oriented, the orientation= argument of
recognize_regions / recognize_polygons / recognize_lines).  Bar: turned crops equal the host emulation bit for bit in
three launches; 'auto' equals, on every output, the explicit reading whose host alm_post_mgp_fuse confidence is larger
(the lower turn on a tie); a single upright reading equals today's entry points; errors leave the context usable."""
import numpy as np
import pytest
import torch

from tests import support
from tests.support import mgp_model, release_models
from tests.test_curve_crops_cpu import curve_fixture, random_polygons
from tests.test_orientation_cpu import CHAR_TABLE, bind, emu_turned_crops
from tests.test_quad_crops_cpu import quad_fixture, random_quads

pytestmark = pytest.mark.gpu
ALM_ERR_INVALID = -1
BPE = [f'b{i}' for i in range(2)] + ['#'] + [f'b{i}' for i in range(3, 50257)]
WP = [f'w{i}' for i in range(102)] + ['[SEP]'] + [f'w{i}' for i in range(103, 30522)]


@pytest.fixture(scope='module')
def model():
    return mgp_model()


@pytest.fixture(scope='module')
def emu():
    return support.emu('orient_emu', bind)


def bits(a, b):
    a, b = np.asarray(a), np.asarray(b)
    assert a.shape == b.shape and a.dtype == b.dtype
    assert np.array_equal(a.view(np.uint32) if a.dtype == np.float32 else a, b.view(np.uint32) if b.dtype == np.float32
                          else b)


def regions(kind, n, seed):
    rng = np.random.default_rng(seed)
    big = rng.integers(0, 256, (256, 320, 3), dtype=np.uint8)
    if kind == 'quad':
        z, pages, _, _ = quad_fixture()
        r = np.concatenate([z['quads'], random_quads(rng, n, 256, 320)])
    else:
        z, pages, _, _ = curve_fixture()
        r = np.concatenate([z['polys'].reshape(-1, 32), random_polygons(rng, n, 256, 320).reshape(-1, 32)])
    pi = np.concatenate([z['page_index'], np.full(n, len(pages), np.int32)]).astype(np.int32)
    return list(pages) + [big], r.astype(np.float32), pi


@pytest.mark.parametrize('kind', ['quad', 'curve'])
def test_turned_crops_equal_emulation(model, emu, kind):
    """Fixture + 1 000 random regions at every turn: the device tensor equals the host emulation bit for bit."""
    from advancedliteratemachinery_b200 import preprocess as P
    pages, r, pi = regions(kind, 1000, 11)
    for q in range(4):
        t = np.full(len(r), q, np.int32)
        got = P.turned_crops(model.ctx, pages, r, pi, t, kind).cpu().numpy()
        _, want, _ = emu_turned_crops(emu, pages, r, pi, t, kind)
        bits(got, want)
    # mixed turns in one call are each region's own turn
    t = np.random.default_rng(1).integers(0, 4, len(r)).astype(np.int32)
    got = P.turned_crops(model.ctx, pages, r, pi, t, kind).cpu().numpy()
    bits(got, emu_turned_crops(emu, pages, r, pi, t, kind)[1])


@pytest.mark.parametrize('kind', ['quad', 'curve'])
def test_turned_line_windows_equal_emulation(model, emu, kind):
    """alm_pre_turned_crops(lines=1): the windows of every turned crop equal the host emulation bit for bit, for every
    turn and for mixed turns."""
    from advancedliteratemachinery_b200 import preprocess as P
    from tests.test_orientation_cpu import emu_turned_line_crops
    pages, r, pi = regions(kind, 300, 19)
    rng = np.random.default_rng(4)
    for t in [np.full(len(r), q, np.int32) for q in range(4)] + [rng.integers(0, 4, len(r)).astype(np.int32)]:
        got = P.turned_crops(model.ctx, pages, r, pi, t, kind, lines=True).cpu().numpy()
        bits(got, emu_turned_line_crops(emu, pages, r, pi, t, kind)[1])


@pytest.mark.parametrize('kind', ['quad', 'curve'])
def test_turned_char_boxes_equal_emulation_on_device_maps(model, emu, kind):
    """Char boxes of readings at mixed turns through the oriented entry equal the host body (itself checked against
    the oracle through np.rot90's index map) fed the device's own A^3 maps of the same turned crops."""
    from advancedliteratemachinery_b200 import preprocess as P
    from tests.test_orientation_cpu import emu_turned_char_boxes
    pages, r, pi = regions(kind, 60, 20)
    R = len(r)
    t = np.random.default_rng(5).integers(0, 4, R).astype(np.int32)
    fn = model.recognize_regions if kind == 'quad' else model.recognize_polygons
    ids, probs, n, boxes, centres, kept, _ = fn(pages, r, pi, char_boxes=True, orientation=t)
    assert np.array_equal(kept.numpy(), t)
    crops = P.turned_crops(model.ctx, pages, r, pi, t, kind)
    out = model.forward(crops, is_eval=True, want_logits=False)
    maps, dids = [a.numpy() for a in out[0]], model.last_ids.numpy()
    bits(ids.numpy(), dids)
    plan = (P.quad_plan if kind == 'quad' else P.curve_plan)([p.shape[:2] for p in pages], r, pi)
    geom = plan['minv'].reshape(R, 9) if kind == 'quad' else plan['ctrl'].reshape(R, 16)
    for h in range(3):
        wn, wb, wc = emu_turned_char_boxes(emu, maps[h], dids[h], h, 1 if kind == 'quad' else 2, plan['sizes'], geom, t)
        bits(n[h].numpy(), wn)
        bits(boxes[h].numpy(), wb)
        bits(centres[h].numpy(), wc)
    assert (n.numpy() > 0).any()


def test_three_launches_whatever_the_count(model):
    from advancedliteratemachinery_b200 import preprocess as P
    pages, r, pi = regions('quad', 1100, 12)
    rng = np.random.default_rng(2)
    for R in (1, 64, 1024):
        for lines in (False, True):
            model.ctx.launch_count(reset=True)
            P.turned_crops(model.ctx, pages, r[:R], pi[:R], rng.integers(0, 4, R), 'quad', lines)
            assert model.ctx.launch_count() == 3, (R, lines)


def fuse_conf(ids, probs):
    from advancedliteratemachinery_b200 import postprocess as Post
    return Post.mgp_fuse(ids, probs, CHAR_TABLE, BPE, WP)['conf'].max(0)


def explicit(call, q, R):
    return call(np.full(R, q, np.int32))


@pytest.mark.parametrize('kind,k,boxes,max_batch', [('quad', None, False, 512), ('quad', 3, True, 6),
                                                    ('curve', None, True, 512), ('curve', 2, False, 9)])
def test_auto_keeps_the_more_confident_reading(model, kind, k, boxes, max_batch):
    """'auto' == per region the explicit reading with the larger host fused confidence, on every output; tall regions
    are read at {1, 3}, the others at {0, 2}."""
    from advancedliteratemachinery_b200 import preprocess as P
    pages, r, pi = regions(kind, 60, 13)
    R = len(r)
    fn = model.recognize_regions if kind == 'quad' else model.recognize_polygons
    call = lambda o: fn(pages, r, pi, k=k, max_batch=max_batch, char_boxes=boxes, orientation=o)
    auto = call('auto')
    sizes = (P.quad_plan if kind == 'quad' else P.curve_plan)([p.shape[:2] for p in pages], r, pi)['sizes']
    tall = 2 * sizes[:, 1].astype(np.int64) >= 3 * sizes[:, 0]
    assert (~tall).any() and (tall.any() or kind == 'curve')
    outs = {q: explicit(call, q, R) for q in range(4)}
    kept = np.zeros(R, np.int32)
    for i in range(R):
        qa, qb = (1, 3) if tall[i] else (0, 2)
        ca, cb = (fuse_conf(outs[q][0][:, i:i + 1, ..., 0] if k else outs[q][0][:, i:i + 1],
                            outs[q][1][:, i:i + 1, ..., 0] if k else outs[q][1][:, i:i + 1])[0] for q in (qa, qb))
        kept[i] = qa if ca >= cb else qb
        for a, b in zip(auto[:-2], outs[kept[i]][:-2]):
            bits(a[:, i].numpy(), b[:, i].numpy())
        bits(auto[-1][i:i + 1].numpy(), np.array([max(ca, cb)], np.float32))
    bits(auto[-2].numpy(), kept)
    for q in range(4):  # explicit readings report their own turn
        assert (outs[q][-2].numpy() == q).all()


def test_lines_auto_and_vertical_lines(model):
    """recognize_lines with 'auto' equals the explicit reading the host fusion prefers; a vertical line read at
    turn 1 or 3 is windowed along its length."""
    pages, r, pi = regions('quad', 0, 14)
    h, w = 200, 480
    page = np.random.default_rng(3).integers(0, 256, (h, w, 3), dtype=np.uint8)
    vert = np.array([[[10, 5], [40, 5], [40, 190], [10, 190]], [[100, 20], [470, 20], [470, 50], [100, 50]]],
                    np.float32)
    lp, lr = list(pages) + [page], np.concatenate([r, vert])
    lpi = np.concatenate([pi, [len(pages)] * 2]).astype(np.int32)
    R = len(lr)
    call = lambda o: model.recognize_lines(lp, lr, lpi, 'quad', max_batch=40, orientation=o)
    auto = call('auto')
    outs = {q: call(np.full(R, q, np.int32)) for q in range(4)}
    assert outs[1][5][R - 2] > 1 and outs[0][5][R - 2] == 1  # the vertical line: windows only when turned
    for i in range(R):
        q = int(auto[-2][i])
        for a, b in zip(auto[:-2], outs[q][:-2]):
            if a.dim() == 1:
                assert int(a[i]) == int(b[i])
            else:
                bits(a[:, i].numpy(), b[:, i].numpy())
        cands = [c for c in ((0, 2) if q in (0, 2) else (1, 3))]
        confs = [fuse_conf(outs[c][0][:, i:i + 1], outs[c][1][:, i:i + 1])[0] for c in cands]
        assert q == cands[int(np.argmax(confs))]
        bits(auto[-1][i:i + 1].numpy(), np.array([max(confs)], np.float32))


def test_upright_reading_equals_existing_entries(model):
    """orientation=[0]*R through the new entry == the default path bit for bit (regions, polygons, lines)."""
    pages, r, pi = regions('quad', 40, 15)
    R = len(r)
    zero = np.zeros(R, np.int32)
    for kw in (dict(), dict(k=4), dict(char_boxes=True)):
        a = model.recognize_regions(pages, r, pi, **kw)
        b = model.recognize_regions(pages, r, pi, orientation=zero, **kw)
        for x, y in zip(a, b[:-2]):
            bits(x.numpy(), y.numpy())
    cpages, c, cpi = regions('curve', 20, 16)
    a = model.recognize_polygons(cpages, c, cpi, char_boxes=True)
    b = model.recognize_polygons(cpages, c, cpi, char_boxes=True, orientation=np.zeros(len(c), np.int32))
    for x, y in zip(a, b[:-2]):
        bits(x.numpy(), y.numpy())
    a = model.recognize_lines(pages, r, pi)
    b = model.recognize_lines(pages, r, pi, orientation=zero)
    for x, y in zip(a, b[:-2]):
        bits(x.numpy(), y.numpy())


def test_one_selection_launch_and_r_rows(model):
    """The oriented forward costs the plain forward's launches plus one; the host outputs hold R rows."""
    pages, r, pi = regions('quad', 30, 17)
    R = len(r)
    model.ctx.launch_count(reset=True)
    model.recognize_regions(pages, r, pi, char_boxes=True)
    plain = model.ctx.launch_count()
    model.ctx.launch_count(reset=True)
    out = model.recognize_regions(pages, r, pi, char_boxes=True, orientation=np.zeros(R, np.int32))
    assert model.ctx.launch_count() == plain + 1
    assert out[0].shape == (3, R, 27) and out[3].shape == (3, R, 26, 4, 2) and out[-1].shape == (R,)


def test_error_paths_leave_the_context_usable(model):
    import ctypes as C
    from advancedliteratemachinery_b200 import preprocess as P
    pages, r, pi = regions('quad', 10, 18)
    R = len(r)
    before = model.recognize_regions(pages, r, pi)
    lines_before = model.recognize_lines(pages, r, pi)
    crops = P.turned_crops(model.ctx, pages, r, pi, np.zeros(R, np.int32))
    lib, h = model.lib, model.ctx.h
    i32 = lambda v: np.ascontiguousarray(np.asarray(v, dtype=np.int32))
    out = [torch.zeros(3, R, 27, dtype=torch.int32), torch.zeros(3, R, 27)]
    kept, conf = torch.zeros(R, dtype=torch.int32), torch.zeros(R)

    def fwd(turns, readings, N=R, Rr=R):
        t, rd = i32(turns), i32(readings)
        return lib.alm_mgpstr_forward_oriented(h, crops.data_ptr(), R, N, t.ctypes.data, Rr, rd.ctypes.data, 0, 0, 0,
                                               None, None, None, 3, out[0].data_ptr(), out[1].data_ptr(), None, None,
                                               None, kept.data_ptr(), conf.data_ptr())
    assert fwd([0] * (R - 1) + [4], [1] * R) == ALM_ERR_INVALID
    assert fwd([0] * (R - 1) + [-1], [1] * R) == ALM_ERR_INVALID
    assert fwd([0] * R, [1] * (R - 2) + [3], Rr=R - 1) == ALM_ERR_INVALID
    assert fwd([0] * R, [1] * (R - 1) + [0]) == ALM_ERR_INVALID
    assert fwd([0] * R, [1] * (R - 1), Rr=R - 1) == ALM_ERR_INVALID  # readings sum to R - 1, not N
    keep, ptrs, hs, ws, n = P._image_args(pages)
    bad = i32([5] + [0] * (R - 1))
    dst = torch.empty(R, 3, 32, 128, device='cuda')
    q = np.ascontiguousarray(r)
    assert lib.alm_pre_turned_crops(h, ptrs, hs.ctypes.data, ws.ctypes.data, n, 1, q.ctypes.data, i32(pi).ctypes.data,
                                    R, bad.ctypes.data, 0, dst.data_ptr()) == ALM_ERR_INVALID
    assert lib.alm_pre_turned_crops(h, ptrs, hs.ctypes.data, ws.ctypes.data, n, 1, q.ctypes.data, i32(pi).ctypes.data,
                                    R, i32([0] * R).ctypes.data, 2, dst.data_ptr()) == ALM_ERR_INVALID
    with pytest.raises(ValueError):
        model.recognize_regions(pages, r, pi, orientation='auto', max_batch=1)
    for x, y in zip(before, model.recognize_regions(pages, r, pi)):
        bits(x.numpy(), y.numpy())
    for x, y in zip(lines_before, model.recognize_lines(pages, r, pi)):
        bits(x.numpy(), y.numpy())
