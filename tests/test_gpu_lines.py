"""GPU: text lines longer than MGP-STR's input, read in overlapping windows (alm_pre_line_crops, alm_mgpstr_forward_lines,
MGPSTRB200.recognize_lines).  Bar: window crops equal tests/golden/pre_lines.npz bit for bit; the stitched ids, probs,
counts, boxes and centres equal oracle/line_ref.py bit for bit when it is fed the device's own per-window maps (read
back through forward(is_eval=True) on the same window crops); a one-window line is what recognize_regions /
recognize_polygons give for its crop."""
import numpy as np
import pytest
import torch

from tests.support import emu, mgp_model, options, release_models
from tests.test_curve_crops_cpu import curve_fixture, curve_regions
from tests.test_lines_cpu import bind, emu_line_stitch, line_fixture
from tests.test_quad_crops_cpu import quad_fixture, text_regions

pytestmark = pytest.mark.gpu
ALM_ERR_INVALID, ALM_ERR_STATE = -1, -4
CODE = {'quad': 1, 'curve': 2}


@pytest.fixture(scope='module')
def model():
    return mgp_model()


def chunks(n, max_batch):
    """recognize_lines' chunks: whole regions, at most max_batch windows each -> [(s, e)]."""
    out, s = [], 0
    while s < len(n):
        e, w = s, 0
        while e < len(n) and w + int(n[e]) <= max_batch:
            w += int(n[e])
            e += 1
        out.append((s, e))
        s = e
    return out


def device_windows(m, pages, regions, pidx, kind, max_batch=512):
    """Per chunk of recognize_lines: the window crops' A^3 maps [3][B, 27, 257], top-1 ids and probs [3, B, 27], read
    back through forward(is_eval=True), concatenated over the chunks."""
    from advancedliteratemachinery_b200 import preprocess as P
    plan = P.line_plan([tuple(p.shape[:2]) for p in pages], regions, pidx, kind)
    maps, ids, probs = [], [], []
    for s, e in chunks(plan['n'], max_batch):
        crops = P.line_crops(m.ctx, pages, regions[s:e], pidx[s:e], kind)
        out = m.forward(crops, is_eval=True, want_logits=False)
        maps.append([a.numpy() for a in out[0]])
        ids.append(m.last_ids.numpy().copy())
        probs.append(m.last_prob.numpy().copy())
    n_h = len(maps[0])
    return ([np.concatenate([a[h] for a in maps]) for h in range(n_h)], np.concatenate(ids, 1),
            np.concatenate(probs, 1), plan)


def assert_equal_bits(got, want):
    g, w = np.asarray(got), np.asarray(want)
    assert g.shape == w.shape
    if g.dtype == np.float32:
        g, w = g.view(np.uint32), w.view(np.uint32)
    assert np.array_equal(g, w)


def assert_lines_oracle(out, maps, ids, probs, plan, kind, heads=(0, 1, 2), rows=None):
    from oracle import line_ref as L
    rows = np.arange(len(plan['n'])) if rows is None else rows
    start = np.concatenate([[0], np.cumsum(plan['n'])])
    for h in heads:
        for r in rows:
            b0, b1 = start[r], start[r + 1]
            want = L.stitch(maps[h][b0:b1], ids[h][b0:b1], probs[h][b0:b1], h, CODE[kind], int(plan['sizes'][r][0]),
                            int(plan['sizes'][r][1]), plan['geom'][r])
            assert_equal_bits(out[0][h, r].numpy(), want[0])
            assert_equal_bits(out[1][h, r].numpy(), want[1])
            assert int(out[2][h, r]) == want[2]
            assert_equal_bits(out[3][h, r].numpy(), want[3])
            assert_equal_bits(out[4][h, r].numpy(), want[4])


@pytest.mark.parametrize('kind', ['quad', 'curve'])
def test_line_crops_equal_fixture(model, kind):
    """alm_pre_line_crops reproduces every fixture window bit for bit, from host and from device pages."""
    from advancedliteratemachinery_b200 import preprocess as P
    z, pages = line_fixture()
    regions, pidx = (z['quads'], z['quad_page_index']) if kind == 'quad' else (z['polys'], z['curve_page_index'])
    want = torch.from_numpy(z[f'{kind}_out_u8']).to(torch.float32).div(255)
    m = model
    for pg in (pages, [torch.from_numpy(p).cuda() for p in pages]):
        m.ctx.launch_count(reset=True)
        got = P.line_crops(m.ctx, pg, regions, pidx, kind)
        assert m.ctx.launch_count() == 3
        assert torch.equal(got.cpu(), want)


@pytest.mark.parametrize('nsplit', [3, 1])
def test_stitch_equals_oracle_on_device_maps(model, nsplit):
    """recognize_lines on the fixture's quads (chunks of at most 16 windows) and curves: every stitched id, probability,
    count, box and centre equals the oracle's on the device's own maps, ids and probabilities."""
    m = model
    with options(m.ctx, nsplit=nsplit):
        z, pages = line_fixture()
        dev = [torch.from_numpy(p).cuda() for p in pages]
        for kind, regions, pidx, mb in (('quad', z['quads'], z['quad_page_index'], 16),
                                        ('curve', z['polys'], z['curve_page_index'], 512)):
            out = m.recognize_lines(pages, regions, pidx, kind=kind, max_batch=mb)
            maps, ids, probs, plan = device_windows(m, dev, regions, pidx, kind, mb)
            assert np.array_equal(out[5].numpy(), plan['n'])
            assert_lines_oracle(out, maps, ids, probs, plan, kind)
            assert (out[2] > 26).any() or kind == 'curve'


def fuse(ids, probs):
    from advancedliteratemachinery_b200 import postprocess as Post
    from oracle.char_box_ref import CHAR_TABLE
    bpe, wp = [f'b{i}' for i in range(50257)], [f'w{i}' for i in range(30522)]
    bpe[2], wp[102] = '#', '[SEP]'  # the end tokens of GPT-2 and BERT, whose strings mgp_fuse looks for
    return Post.mgp_fuse(ids, probs, CHAR_TABLE, bpe, wp)


@pytest.mark.parametrize('kind', ['quad', 'curve'])
def test_single_window_lines_equal_region_recognition(model, kind):
    """Regions of one window: ids / probs through each head's end token, the BPE / WordPiece boxes, and -- wherever no
    '[GO]' precedes the char head's '[s]' -- the char boxes and mgp_fuse's fused text, source and confidence equal
    recognize_regions / recognize_polygons with char_boxes=True."""
    from advancedliteratemachinery_b200 import preprocess as P
    m = model
    z, pages, _, _ = quad_fixture() if kind == 'quad' else curve_fixture()
    regions = z['quads'] if kind == 'quad' else z['polys']
    plan = P.line_plan([p.shape[:2] for p in pages], regions, z['page_index'], kind)
    rows = np.flatnonzero(plan['n'] == 1)
    assert len(rows) > 10
    regions, pidx = regions[rows], z['page_index'][rows]
    recog = m.recognize_regions if kind == 'quad' else m.recognize_polygons
    ids, probs, n, boxes, centres = recog(pages, regions, pidx, char_boxes=True)
    lids, lprobs, ln, lboxes, lcentres, wins = m.recognize_lines(pages, regions, pidx, kind=kind)
    assert (wins == 1).all()
    ids, probs, lids, lprobs = ids.numpy(), probs.numpy(), lids.numpy(), lprobs.numpy()
    for h, end in ((0, 1), (1, 2), (2, 102)):
        for b in range(len(rows)):
            row = ids[h, b]
            e = int(np.argmax(row[1:] == end)) + 1 if (row[1:] == end).any() else 27
            top = min(e + 1, 27)
            assert np.array_equal(lids[h, b, :top], row[:top]) and np.array_equal(
                lprobs[h, b, :top].view(np.uint32), probs[h, b, :top].view(np.uint32))
            if h > 0 or (e < 27 and not (row[1:e] == 0).any()):  # the char head: '[s]' with no '[GO]' before it
                k = int(n[h, b])
                assert int(ln[h, b]) == k
                assert_equal_bits(lboxes[h, b, :k].numpy(), boxes[h, b, :k].numpy())
                assert_equal_bits(lcentres[h, b, :k].numpy(), centres[h, b, :k].numpy())
    # mgp_fuse: the char head's string-index slice differs only when '[GO]' comes before '[s]'
    fr, fl = fuse(ids, probs), fuse(lids, lprobs)
    ok = []
    for b in range(len(rows)):
        row = ids[0, b, 1:]
        e = int(np.argmax(row == 1)) if (row == 1).any() else 26
        if not (row[:e] == 0).any():
            ok.append(b)
    assert ok
    for b in ok:
        assert fr['fused'][b] == fl['fused'][b] and fr['source'][b] == fl['source'][b]
        assert np.array_equal(fr['conf'][:, b].view(np.uint32), fl['conf'][:, b].view(np.uint32))


def test_chunking_empty_and_a_thousand_lines(model):
    """max_batch 8, 9 and 512 give the same bits; R = 0 gives empty outputs; 1 024 lines on 16 pages (several chunks)
    equal the host run of the kernel bodies on the device's maps, and the oracle on 32 of them; max_batch < 8 is
    refused."""
    from advancedliteratemachinery_b200 import preprocess as P
    m = model
    z, pages = line_fixture()
    ref = m.recognize_lines(pages, z['quads'], z['quad_page_index'], max_batch=512)
    for mb in (8, 9):
        got = m.recognize_lines(pages, z['quads'], z['quad_page_index'], max_batch=mb)
        for a, b in zip(got, ref):
            assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    with pytest.raises(ValueError):
        m.recognize_lines(pages, z['quads'], z['quad_page_index'], max_batch=7)
    out = m.recognize_lines(pages, np.zeros((0, 4, 2)), [])
    assert [tuple(t.shape) for t in out] == [(3, 0, 210), (3, 0, 210), (3, 0), (3, 0, 208, 4, 2), (3, 0, 208, 2), (0,)]
    out = m.recognize_lines(pages, np.zeros((0, 16, 2)), [], kind='curve')
    assert out[0].shape == (3, 0, 210)

    lib = emu('line_emu', bind)
    for kind, (pg, regions, pidx) in (('quad', text_regions(seed=11)), ('curve', curve_regions(seed=12))):
        dev = [torch.from_numpy(p).cuda() for p in pg]
        out = m.recognize_lines(dev, regions, pidx, kind=kind)
        maps, ids, probs, plan = device_windows(m, dev, regions, pidx, kind)
        assert out[0].shape == (3, 1024, 210) and int(plan['n'].sum()) > 1024
        for h in range(3):
            want = emu_line_stitch(lib, maps[h], ids[h], probs[h], h, CODE[kind], plan['sizes'], plan['geom'])
            for g, w in zip((out[0][h], out[1][h], out[2][h], out[3][h], out[4][h]), want):
                assert_equal_bits(g.numpy(), w)
        assert_lines_oracle(out, maps, ids, probs, plan, kind, rows=np.arange(0, 1024, 32))
    assert P.line_plan([(10, 10)], np.zeros((0, 4, 2)), [])['n'].shape == (0,)


def test_launches_per_chunk(model):
    """Per chunk: 3 crop launches, the forward's launches, and 2 per head (box reduction, stitch)."""
    from advancedliteratemachinery_b200 import preprocess as P
    m = model
    z, pages = line_fixture()
    dev = [torch.from_numpy(p).cuda() for p in pages]
    regions, pidx = z['quads'], z['quad_page_index']
    plan = P.line_plan([p.shape[:2] for p in pages], regions, pidx, 'quad')
    parts = chunks(plan['n'], 32)
    assert len(parts) > 2
    m.ctx.launch_count(reset=True)
    m.recognize_lines(dev, regions, pidx, max_batch=32)
    lines = m.ctx.launch_count()
    m.ctx.launch_count(reset=True)
    for s, e in parts:
        m.recognize(P.line_crops(m.ctx, dev, regions[s:e], pidx[s:e]))
    plain = m.ctx.launch_count()
    assert lines - plain == 6 * len(parts), (lines, plain, len(parts))


def test_charstr_writes_plane_zero_only():
    from advancedliteratemachinery_b200 import MGPSTRB200
    from advancedliteratemachinery_b200 import synthetic as W
    dim, depth, heads = W.MGP_VARIANTS['base']
    m = MGPSTRB200(W.mgpstr_state_dict(seed=3, dim=dim, depth=depth, heads=heads, char_only=True))
    try:
        z, pages = line_fixture()
        dev = [torch.from_numpy(p).cuda() for p in pages]
        regions, pidx = z['polys'], z['curve_page_index']
        out = m.recognize_lines(dev, regions, pidx, kind='curve')
        for t in out[:5]:
            assert not t[1:].any()
        assert out[2][0].any()
        maps, ids, probs, plan = device_windows(m, dev, regions, pidx, 'curve')
        assert_lines_oracle(out, maps, ids, probs, plan, 'curve', heads=(0,))
    finally:
        m.ctx.close()


def _raw_lines(m, crops, R, windows, kind, sizes, geom, B=None, n_heads=None):
    B = crops.shape[0] if B is None else B
    bufs = [np.zeros(3 * R * 210, np.int32), np.zeros(3 * R * 210, np.float32), np.zeros(3 * R, np.int32),
            np.zeros(3 * R * 208 * 8, np.float32), np.zeros(3 * R * 208 * 2, np.float32)]
    w = np.ascontiguousarray(windows, np.int32) if windows is not None else None
    s = np.ascontiguousarray(sizes, np.int32) if sizes is not None else None
    g = np.ascontiguousarray(geom, np.float64) if geom is not None else None
    ptr = lambda a: a.ctypes.data if a is not None else None
    return m.lib.alm_mgpstr_forward_lines(m.ctx.h, crops.data_ptr(), B, R, ptr(w), kind, ptr(s), ptr(g),
                                          m.info()['n_a3'] if n_heads is None else n_heads,
                                          *[b.ctypes.data for b in bufs])


def test_error_paths_leave_the_context_usable(model):
    """Bad arguments return ALM_ERR_INVALID (no checkpoint: ALM_ERR_STATE) and the next calls give the same bits;
    recognize_regions on the same context is bit-identical before and after recognize_lines."""
    from advancedliteratemachinery_b200 import _lib, preprocess as P
    m = model
    zq, qpages, _, _ = quad_fixture()
    before = m.recognize_regions(qpages, zq['quads'], zq['page_index'], char_boxes=True)
    z, pages = line_fixture()
    regions, pidx = z['quads'][:4], z['quad_page_index'][:4]
    plan = P.line_plan([p.shape[:2] for p in pages], regions, pidx, 'quad')
    crops = P.line_crops(m.ctx, pages, regions, pidx)
    R, wins, sizes, geom = 4, plan['n'].astype(np.int32), plan['sizes'], plan['geom']
    nan = geom.copy(); nan[1, 3] = np.nan
    zero = sizes.copy(); zero[2, 1] = 0
    more = wins.copy(); more[3] += 1
    cases = [dict(kind=0), dict(kind=3), dict(windows=None), dict(sizes=None), dict(geom=None), dict(geom=nan),
             dict(sizes=zero), dict(windows=more), dict(B=int(wins.sum()) - 1), dict(n_heads=1), dict(R=0)]
    for kw in cases:
        args = dict(windows=wins, kind=1, sizes=sizes, geom=geom)
        args.update(kw)
        Rk = args.pop('R', R)
        assert _raw_lines(m, crops, Rk, **args) == ALM_ERR_INVALID, kw
    keep, ptrs, hs, ws, n = P._image_args(pages)
    rc = m.lib.alm_pre_line_crops(m.ctx.h, ptrs, hs.ctypes.data, ws.ctypes.data, n, 0, regions.ctypes.data,
                                  pidx.ctypes.data, 4, crops.data_ptr())
    assert rc == ALM_ERR_INVALID
    empty = _lib.Context(0)
    buf = np.zeros(3 * 4 * 208 * 8, np.float32)
    try:
        rc = empty.lib.alm_mgpstr_forward_lines(empty.h, crops.data_ptr(), crops.shape[0], 4, wins.ctypes.data, 1,
                                                sizes.ctypes.data, geom.ctypes.data, 3, *[buf.ctypes.data] * 5)
        assert rc == ALM_ERR_STATE
    finally:
        empty.close()
    assert _raw_lines(m, crops, R, wins, 1, sizes, geom) == 0
    out = m.recognize_lines(pages, regions, pidx)
    maps, ids, probs, _ = device_windows(m, [torch.from_numpy(p).cuda() for p in pages], regions, pidx, 'quad')
    assert_lines_oracle(out, maps, ids, probs, plan, 'quad')
    after = m.recognize_regions(qpages, zq['quads'], zq['page_index'], char_boxes=True)
    for a, b in zip(before, after):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))
