"""Reading text that does not run upright in its crop (DESIGN 4.13): CPU checks of the turned-pixel index map, of the
turned crops the kernels cut (their per-pixel bodies run on the host by tests/emu/orient_emu.cpp) against np.rot90 of
the upright crops and against the oracle crops + np.rot90 + Pillow's resize, and of the confidence rule and choice of
the selection kernel against alm_post_mgp_fuse.  Bar: bit-exact everywhere."""
import ctypes as C
import os

import numpy as np
import pytest

from tests import support
from tests.test_curve_crops_cpu import curve_fixture, random_polygons
from tests.test_quad_crops_cpu import quad_fixture, random_quads

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
CHAR_TABLE = ['[GO]', '[s]'] + list('0123456789abcdefghijklmnopqrstuvwxyz')


@pytest.fixture(scope='module')
def emu():
    return support.emu('orient_emu', bind)


def bind(lib):
    """Bind tests/emu/orient_emu.cpp (host compile of the kernels' bodies)."""
    for f in ('emu_unturn', 'emu_turn_px', 'emu_turned_crops', 'emu_head_conf', 'emu_select'):
        getattr(lib, f).restype = None
    lib.emu_unturn.argtypes = lib.emu_turn_px.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p]
    lib.emu_turned_crops.argtypes = [C.c_int, C.c_int] + [C.c_void_p] * 12 + [C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    lib.emu_head_conf.argtypes = [C.c_int] * 4 + [C.c_void_p] * 3
    lib.emu_select.argtypes = [C.c_int] * 4 + [C.c_void_p] * 2 + [C.c_int] + [C.c_void_p] * 4


def i32(v):
    return np.ascontiguousarray(np.asarray(v, dtype=np.int32))


def emu_turned_crops(lib, pages, regions, page_index, turns, kind):
    """alm_pre_turned_crops' three launches on the host with the library's plan and weights -> (turned natural-size
    crops [R] of u8 [th, tw, 3], out f32 [R, 3, 32, 128])."""
    from advancedliteratemachinery_b200 import preprocess as P
    pages = [np.ascontiguousarray(p) for p in pages]
    sizes = [p.shape[:2] for p in pages]
    if kind == 'quad':
        p = P.quad_plan(sizes, regions, page_index)
        geom = np.ascontiguousarray(p['minv'].reshape(-1, 9))
    else:
        p = P.curve_plan(sizes, regions, page_index)
        geom = np.ascontiguousarray(p['ctrl'].reshape(-1, 16))
    cs = p['sizes']
    turns = i32(turns)
    ts = np.where((turns & 1)[:, None] == 1, cs[:, ::-1], cs)
    coefs, where = [], {}

    def weights(n_in, n_out):
        if (n_in, n_out) not in where:
            b, k = P.resample_coeffs(n_in, n_out, 'bicubic')
            where[(n_in, n_out)] = (sum(a.size for a in coefs), k.shape[1])
            coefs.extend([b.ravel(), k.ravel()])
        return where[(n_in, n_out)]

    hw = [weights(int(w), 128) for w, _ in ts]
    vw = [weights(int(h), 32) for _, h in ts]
    coef = i32(np.concatenate(coefs))
    hb, hk, vb, vk = i32([a for a, _ in hw]), i32([k for _, k in hw]), i32([a for a, _ in vw]), i32([k for _, k in vw])
    ptrs = (C.c_void_p * len(pages))(*[q.ctypes.data for q in pages])
    ph, pw, pi = i32([q.shape[0] for q in pages]), i32([q.shape[1] for q in pages]), i32(page_index)
    R, cs32 = len(cs), i32(cs)
    warped = np.zeros((int((cs[:, 0].astype(np.int64) * cs[:, 1]).sum()), 3), np.uint8)
    out = np.zeros((R, 3, 32, 128), np.float32)
    lib.emu_turned_crops(1 if kind == 'quad' else 2, R, ptrs, ph.ctypes.data, pw.ctypes.data, pi.ctypes.data,
                         geom.ctypes.data, cs32.ctypes.data, turns.ctypes.data, coef.ctypes.data, hb.ctypes.data,
                         hk.ctypes.data, vb.ctypes.data, vk.ctypes.data, 32, 128, warped.ctypes.data, out.ctypes.data)
    crops, off = [], 0
    for w, h in ts:
        crops.append(warped[off:off + w * h].reshape(h, w, 3))
        off += w * h
    return crops, out, cs


def _regions(kind, n_random, seed):
    """The fixture regions of pre_quads / pre_curves and pre_lines, plus n_random random ones on a 256 x 320 page."""
    rng = np.random.default_rng(seed)
    zl = np.load(os.path.join(GOLD, 'pre_lines.npz'))
    lpages = [zl[f'page{i}'] for i in range(int(zl['n_pages']))]
    if kind == 'quad':
        z, pages, _, _ = quad_fixture()
        regs = [z['quads'], zl['quads'], random_quads(rng, n_random, 256, 320)]
        pis = [z['page_index'], zl['quad_page_index']]
    else:
        z, pages, _, _ = curve_fixture()
        regs = [z['polys'], zl['polys'].reshape(-1, 32), random_polygons(rng, n_random, 256, 320).reshape(-1, 32)]
        regs[0] = regs[0].reshape(-1, 32)
        pis = [z['page_index'], zl['curve_page_index']]
    pis = [pis[0], pis[1] + len(pages), np.full(n_random, len(pages) + len(lpages), np.int32)]
    big = np.random.default_rng(seed + 1).integers(0, 256, (256, 320, 3), dtype=np.uint8)
    return list(pages) + lpages + [big], np.concatenate(regs).astype(np.float32), np.concatenate(pis).astype(np.int32)


def test_index_map_is_the_rot90_bijection(emu):
    """unturn maps every pixel of np.rot90(crop, q) to the upright pixel it holds, one to one; turn_px inverts it."""
    for cw, ch in ((1, 1), (1, 7), (9, 1), (5, 3), (32, 8), (17, 40)):
        up = np.arange(cw * ch, dtype=np.int64).reshape(ch, cw)
        for q in range(4):
            t = np.rot90(up, q)
            th, tw = t.shape
            yy, xx = np.mgrid[0:th, 0:tw]
            xy = i32(np.stack([xx.ravel(), yy.ravel()], 1))
            u = np.zeros_like(xy)
            emu.emu_unturn(q, xy.shape[0], xy.ctypes.data, tw, th, u.ctypes.data)
            assert np.array_equal(u[:, 1] * cw + u[:, 0], t.ravel()), (cw, ch, q)
            assert len(np.unique(u[:, 1] * cw + u[:, 0])) == cw * ch
            back = np.zeros_like(u)
            emu.emu_turn_px(q, u.shape[0], u.ctypes.data, cw, ch, back.ctypes.data)
            assert np.array_equal(back, xy), (cw, ch, q)


@pytest.mark.parametrize('kind', ['quad', 'curve'])
def test_turned_crops_are_rot90_of_the_upright_crops(emu, kind):
    """Fixture regions of pre_quads / pre_curves / pre_lines and 1 000 random ones, page-size fallbacks included:
    the turned natural-size crop is np.rot90 of the upright one, bit for bit, for every turn."""
    pages, regs, pi = _regions(kind, 1000, 5)
    up, _, cs = emu_turned_crops(emu, pages, regs, pi, np.zeros(len(regs)), kind)
    if kind == 'quad':
        n_fallback = sum(1 for r in range(len(regs)) if tuple(cs[r]) == tuple(pages[pi[r]].shape[1::-1]))
        assert n_fallback > 0
    for q in range(1, 4):
        got, _, _ = emu_turned_crops(emu, pages, regs, pi, np.full(len(regs), q), kind)
        for r in range(len(regs)):
            assert np.array_equal(got[r], np.rot90(up[r], q)), (kind, q, r)


@pytest.mark.parametrize('kind', ['quad', 'curve'])
def test_turned_tensor_equals_oracle_rot90_pillow(emu, kind):
    """The final tensor == ToTensor(Image.fromarray(np.rot90(oracle crop, q)).resize((128, 32), BICUBIC)), bit for bit,
    on the fixture regions, for every turn."""
    pytest.importorskip('cv2')
    pytest.importorskip('PIL')
    from oracle import preprocess_ref as O
    if kind == 'quad':
        from oracle import quad_crop_ref as Q
        z, pages, _, _ = quad_fixture()
        regs, pi = z['quads'], z['page_index']
        crops, _ = Q.quad_crops(pages, regs, pi)
    else:
        from oracle import curve_crop_ref as Cr
        from advancedliteratemachinery_b200 import preprocess as P
        z, pages, _, _ = curve_fixture()
        regs, pi = z['polys'], z['page_index']
        plan = P.curve_plan([p.shape[:2] for p in pages], regs, pi)
        crops, _ = Cr.curve_crops(pages, regs, pi, plans=[(c, int(s[0]), int(s[1])) for c, s in
                                                          zip(plan['ctrl'], plan['sizes'])])
    for q in range(4):
        _, got, _ = emu_turned_crops(emu, pages, regs, pi, np.full(len(regs), q), kind)
        ref = O.mgp_crops([np.ascontiguousarray(np.rot90(c, q)) for c in crops], 32, 128).numpy()
        assert np.array_equal(got.view(np.uint32), ref.view(np.uint32)), (kind, q)


def _random_heads(rng, B, T):
    """ids / probs [3, B, T] with end tokens at random places (sometimes none), '[GO]' among the characters."""
    ids = np.zeros((3, B, T), np.int32)
    ids[0] = rng.integers(2, 38, (B, T))
    ids[0][rng.random((B, T)) < 0.05] = 0
    ids[1] = rng.integers(3, 50, (B, T))
    ids[2] = rng.integers(103, 200, (B, T))
    for h, end in enumerate((1, 2, 102)):
        pos = rng.integers(1, T + 6, B)  # past T: no end token
        for b in range(B):
            if pos[b] < T:
                ids[h, b, pos[b]] = end
                if rng.random() < 0.3 and pos[b] + 2 < T:
                    ids[h, b, pos[b] + 2] = end
    probs = rng.uniform(0.3, 1.0, (3, B, T)).astype(np.float32)
    return ids, probs


BPE = ['x', 'y', '#'] + [f'b{i}' for i in range(3, 50)]
WP = [f'w{i}' for i in range(102)] + ['[SEP]'] + [f'w{i}' for i in range(103, 200)]


@pytest.mark.parametrize('T', [27, 210])
def test_conf_rule_equals_mgp_fuse(emu, T):
    """fuse_core's per-head confidence == alm_post_mgp_fuse's conf, bit for bit (38-entry char table)."""
    from advancedliteratemachinery_b200 import postprocess as Post
    rng = np.random.default_rng(T)
    B = 400
    ids, probs = _random_heads(rng, B, T)
    ref = Post.mgp_fuse(ids, probs, CHAR_TABLE, BPE, WP)['conf']
    assert (ref == 0).any() and (ref > 0).any()
    for h in range(3):
        got = np.zeros(B, np.float32)
        a, p = np.ascontiguousarray(ids[h]), np.ascontiguousarray(probs[h])
        emu.emu_head_conf(B, T, 1, h, a.ctypes.data, p.ctypes.data, got.ctypes.data)
        assert np.array_equal(got.view(np.uint32), ref[h].view(np.uint32)), h


def test_selection_keeps_the_larger_fused_confidence(emu):
    """emu_select == the argmax of the host fused confidence per region; equal confidence goes to the lower turn."""
    from advancedliteratemachinery_b200 import postprocess as Post
    rng = np.random.default_rng(3)
    R, T = 300, 27
    readings = rng.integers(1, 3, R)
    readings[:40] = 2
    N = int(readings.sum())
    rstart = i32(np.concatenate([[0], np.cumsum(readings)]))
    ids, probs = _random_heads(rng, N, T)
    turns = np.zeros(N, np.int32)
    for r in range(R):
        a = rstart[r]
        turns[a:rstart[r + 1]] = rng.permutation([0, 2] if rng.random() < 0.5 else [1, 3])[:readings[r]]
    for r in range(20):  # identical readings: a tie, which the lower turn wins
        ids[:, rstart[r] + 1], probs[:, rstart[r] + 1] = ids[:, rstart[r]], probs[:, rstart[r]]
    conf = Post.mgp_fuse(ids, probs, CHAR_TABLE, BPE, WP)['conf'].max(0)
    kept, got = np.zeros(R, np.int32), np.zeros(R, np.float32)
    emu.emu_select(3, N, T, 1, np.ascontiguousarray(ids).ctypes.data, np.ascontiguousarray(probs).ctypes.data, R,
                   rstart.ctypes.data, turns.ctypes.data, kept.ctypes.data, got.ctypes.data)
    for r in range(R):
        cand = list(range(rstart[r], rstart[r + 1]))
        best = max(cand, key=lambda i: (conf[i], -turns[i]))
        assert kept[r] == best, r
        assert got[r].view(np.uint32) == np.float32(max(conf[best], 0)).view(np.uint32)
    assert all(turns[kept[r]] == turns[rstart[r]:rstart[r] + 2].min() for r in range(20))


def test_invalid_orientation_is_rejected_before_device_work():
    """Turns outside 0..3, a wrong count, an unknown string or a max_batch that would split a region's readings raise
    ValueError before anything touches the device."""
    from advancedliteratemachinery_b200.mgp_str import MGPSTRB200
    m = object.__new__(MGPSTRB200)  # no context: any device work would fail with something else
    page = np.zeros((64, 64, 3), np.uint8)
    q = np.array([[[2, 2], [40, 2], [40, 12], [2, 12]]] * 2, np.float32)
    for orientation, mb in (([0, 4], 512), ([0, -1], 512), ([0], 512), ('sideways', 512), ([0.5, 1], 512),
                            ('auto', 1)):
        with pytest.raises(ValueError):
            m.recognize_regions([page], q, [0, 0], orientation=orientation, max_batch=mb)
    with pytest.raises(ValueError):
        m.recognize_lines([page], q, [0, 0], orientation='auto', max_batch=15)


def rot90_map(q, cw, ch):
    """(A, b): upright pixel = A (x, y) + b for pixel (x, y) of np.rot90(crop, q), crop cw x ch, read off np.rot90 of the
    upright pixels' own coordinates."""
    def grids(w, h):
        ux, uy = np.meshgrid(np.arange(w), np.arange(h))
        return np.rot90(ux, q), np.rot90(uy, q)
    ex, ey = grids(5, 3)  # the linear part does not depend on the size
    A = np.array([[ex[0, 1] - ex[0, 0], ex[1, 0] - ex[0, 0]], [ey[0, 1] - ey[0, 0], ey[1, 0] - ey[0, 0]]], np.float64)
    gx, gy = grids(cw, ch)
    return A, (float(gx[0, 0]), float(gy[0, 0]))


def unturned(q, cw, ch):
    """A point (X, Y) of np.rot90(crop, q) -> the same point of the upright crop, in double."""
    A, b = rot90_map(q, cw, ch)
    return lambda X, Y: ((A[0, 0] * X + A[0, 1] * Y) + b[0], (A[1, 0] * X + A[1, 1] * Y) + b[1])


def turned_char_box_ref(a, kind, cw, ch, g, q):
    """oracle/char_box_ref's box of a map read on np.rot90(crop, q), taken back to the upright crop through np.rot90's
    index map and to the page through the region's plan."""
    from oracle import char_box_ref as V
    tw, th = (ch, cw) if q & 1 else (cw, ch)
    back = unturned(q, cw, ch)
    page = lambda X, Y: V.to_page(*back(X, Y), kind, cw, ch, g)
    L, R, xc, yc = V.reduce_map(a)
    XL, XR = (L * tw) / 128.0 - 0.5, (R * tw) / 128.0 - 0.5
    Yt, Yb = 0.0, float(th - 1)
    box = np.array([page(XL, Yt), page(XR, Yt), page(XR, Yb), page(XL, Yb)], np.float32)
    return box, np.array(page((xc * tw) / 128.0 - 0.5, (yc * th) / 32.0 - 0.5), np.float32)


def emu_turned_char_boxes(lib, maps, ids, head, kind, sizes, geom, turns):
    B = maps.shape[0]
    n, boxes, centres = np.zeros(B, np.int32), np.zeros((B, 26, 4, 2), np.float32), np.zeros((B, 26, 2), np.float32)
    lib.emu_turned_char_boxes.restype = None
    lib.emu_turned_char_boxes.argtypes = [C.c_int] * 3 + [C.c_void_p] * 8
    args = [np.ascontiguousarray(maps, np.float32), i32(ids), i32(sizes),
            np.ascontiguousarray(np.asarray(geom, np.float64).reshape(B, -1)), i32(turns), n, boxes, centres]
    lib.emu_turned_char_boxes(B, head, kind, *[x.ctypes.data for x in args])
    return n, boxes, centres


@pytest.mark.parametrize('kind', [1, 2])
def test_turned_char_boxes_equal_oracle_through_rot90(emu, kind):
    """char_box_kernel's body on crops read at q = 0..3 equals oracle/char_box_ref's box computed in np.rot90(crop, q)
    and taken back through np.rot90's index map, bit for bit, on quad and curve plans and every head."""
    from oracle import char_box_ref as V
    from tests.test_char_boxes_cpu import plans, random_ids, random_maps
    rng = np.random.default_rng(40 + kind)
    B = 48
    maps, ids = random_maps(rng, B), random_ids(rng, B)
    q, cv = plans(rng, B)
    sizes, geom = (q['sizes'], q['minv'].reshape(B, 9)) if kind == 1 else (cv['sizes'], cv['ctrl'].reshape(B, 16))
    for turn in range(4):
        turns = np.full(B, turn, np.int32)
        turns[::3] = (turn + 1) % 4  # mixed turns in one grid
        for head in (0, 1, 2):
            hid = ids if head == 0 else np.where(ids == 1, V.END_ID[head], ids)
            n, boxes, centres = emu_turned_char_boxes(emu, maps, hid, head, kind, sizes, geom, turns)
            assert np.array_equal(n, V.char_boxes(maps, hid, head)[0])
            for b in range(B):
                for s in range(n[b]):
                    box, centre = turned_char_box_ref(maps[b, s + 1], kind, int(sizes[b][0]), int(sizes[b][1]),
                                                      geom[b], int(turns[b]))
                    assert np.array_equal(boxes[b, s].view(np.uint32), box.view(np.uint32)), (turn, head, b, s)
                    assert np.array_equal(centres[b, s].view(np.uint32), centre.view(np.uint32)), (turn, head, b, s)
                assert not boxes[b, n[b]:].any()


def test_upside_down_reading_puts_top_left_at_the_word_bottom_right(emu):
    """An axis-aligned word read at q = 2: a character at the left of the turned crop lies at the word's right on the
    page, and its 'top-left' corner sits on the word's bottom edge."""
    from advancedliteratemachinery_b200 import preprocess as P
    quad = np.array([[[100, 50], [300, 50], [300, 90], [100, 90]]], np.float32)
    plan = P.quad_plan([(200, 400)], quad, [0])
    a = np.zeros((1, 27, 257), np.float32)
    a[0, 1, 1 + np.arange(8) * 32] = 1.0  # token 1: all its mass in the first patch column
    ids = np.full((1, 27), 5, np.int32)
    ids[0, 2] = 1
    n, boxes, centres = emu_turned_char_boxes(emu, a, ids, 0, 1, plan['sizes'], plan['minv'].reshape(1, 9), [2])
    assert n[0] == 1
    tl, tr, br, bl = boxes[0, 0]
    assert tl[0] > 290 and tl[1] > 85 and br[1] < 55  # top-left at the bottom-right, bottom-right on the top edge
    assert tr[0] < tl[0] and 290 < centres[0, 0, 0] < 300


def emu_turned_line_crops(lib, pages, regions, page_index, turns, kind):
    """alm_pre_turned_crops(lines=1) on the host -> (window crops u8 [th, wn, 3], out f32 [N, 3, 32, 128])."""
    from advancedliteratemachinery_b200 import preprocess as P
    pages = [np.ascontiguousarray(p) for p in pages]
    plan = P.line_plan([p.shape[:2] for p in pages], regions, page_index, kind)
    cs, turns = plan['sizes'], i32(turns)
    ts = np.where((turns & 1)[:, None] == 1, cs[:, ::-1], cs)
    n, _, wn = P.line_windows(ts)
    coefs, where, hw, vw = [], {}, [], []

    def weights(n_in, n_out):
        if (n_in, n_out) not in where:
            b, k = P.resample_coeffs(n_in, n_out, 'bicubic')
            where[(n_in, n_out)] = (sum(x.size for x in coefs), k.shape[1])
            coefs.extend([b.ravel(), k.ravel()])
        return where[(n_in, n_out)]

    shapes = []
    for r in range(len(cs)):
        for _ in range(n[r]):
            hw.append(weights(int(wn[r]), 128))
            vw.append(weights(int(ts[r][1]), 32))
            shapes.append((int(ts[r][1]), int(wn[r])))
    hb, hk, vb, vk = i32([a for a, _ in hw]), i32([k for _, k in hw]), i32([a for a, _ in vw]), i32([k for _, k in vw])
    ptrs = (C.c_void_p * len(pages))(*[q.ctypes.data for q in pages])
    ph, pw = i32([q.shape[0] for q in pages]), i32([q.shape[1] for q in pages])
    warped = np.zeros((sum(h * w for h, w in shapes), 3), np.uint8)
    out = np.zeros((len(shapes), 3, 32, 128), np.float32)
    lib.emu_turned_line_crops.restype = None
    lib.emu_turned_line_crops.argtypes = [C.c_int, C.c_int] + [C.c_void_p] * 12 + [C.c_int, C.c_int, C.c_void_p,
                                                                                  C.c_void_p]
    args = [ph, pw, i32(page_index), np.ascontiguousarray(plan['geom']), i32(cs), turns, i32(np.concatenate(coefs)),
            hb, hk, vb, vk]
    lib.emu_turned_line_crops(1 if kind == 'quad' else 2, len(cs), ptrs, *[x.ctypes.data for x in args], 32, 128,
                              warped.ctypes.data, out.ctypes.data)
    wins, off = [], 0
    for h, w in shapes:
        wins.append(warped[off:off + h * w].reshape(h, w, 3))
        off += h * w
    return wins, out


@pytest.mark.parametrize('kind', ['quad', 'curve'])
def test_turned_line_windows_are_windows_of_the_rot90_crop(emu, kind):
    """alm_pre_turned_crops(lines=1) on the host: the windows are oracle/line_ref's windows of np.rot90 of the upright
    crop, bit for bit, for every turn; a tall line read at an odd turn gets several windows."""
    from oracle import line_ref as L
    pages, regs, pi = _regions(kind, 200, 7)
    up, _, _ = emu_turned_crops(emu, pages, regs, pi, np.zeros(len(regs)), kind)
    for q in range(4):
        wins, _ = emu_turned_line_crops(emu, pages, regs, pi, np.full(len(regs), q), kind)
        want = [w for c in up for w in L.window_crops(np.rot90(c, q))]
        assert len(wins) == len(want)
        assert all(np.array_equal(a, b) for a, b in zip(wins, want)), (kind, q)
    tall = [r for r, c in enumerate(up) if c.shape[0] > 4 * c.shape[1]]
    assert (tall or kind == 'curve') and all(len(L.window_crops(np.rot90(up[r], 1))) > 1 for r in tall)


def turned_stitch_ref(maps, ids, probs, head, kind, sizes, geom, turns):
    """oracle/line_ref.stitch_lines for regions read at turns: windows laid out on np.rot90(crop, q), every point taken
    back to the upright crop through np.rot90's index map before the plan maps it."""
    from oracle import line_ref as L
    out = [], [], [], [], []
    orig, b = L.V.to_page, 0
    try:
        for (cw, ch), g, q in zip(np.asarray(sizes), np.asarray(geom).reshape(len(sizes), -1), turns):
            cw, ch, q = int(cw), int(ch), int(q)
            tw, th = (ch, cw) if q & 1 else (cw, ch)
            back = unturned(q, cw, ch)
            L.V.to_page = lambda X, Y, k_, _w, _h, g_, back=back, cw=cw, ch=ch: orig(*back(X, Y), k_, cw, ch, g_)
            nw = L.windows(tw, th)[0]
            for lst, v in zip(out, L.stitch(maps[b:b + nw], ids[b:b + nw], probs[b:b + nw], head, kind, tw, th, g)):
                lst.append(v)
            b += nw
    finally:
        L.V.to_page = orig
    assert b == len(ids)
    return [np.stack(x) for x in out]


@pytest.mark.parametrize('kind', ['quad', 'curve'])
def test_turned_line_stitch_equals_oracle_through_rot90(emu, kind):
    """line_box_kernel + line_stitch_kernel's bodies on lines read at q = 0..3 (seams and X in the turned crop) equal
    oracle/line_ref's stitch on np.rot90's windows, taken back through np.rot90's index map, bit for bit."""
    from advancedliteratemachinery_b200 import preprocess as P
    from tests.test_lines_cpu import line_ids, line_plans, random_probs
    from tests.test_char_boxes_cpu import random_maps
    rng = np.random.default_rng(50 + (kind == 'curve'))
    plan = line_plans(rng, 30)[kind == 'curve']
    code = 1 if kind == 'quad' else 2
    sizes, geom = plan['sizes'], np.ascontiguousarray(plan['geom'])
    R = len(sizes)
    lib = emu
    lib.emu_turned_line_stitch.restype = None
    lib.emu_turned_line_stitch.argtypes = [C.c_int] * 4 + [C.c_void_p] * 11
    for turn in range(4):
        turns = i32((np.arange(R) + turn) % 4)
        ts = np.where((turns & 1)[:, None] == 1, sizes[:, ::-1], sizes)
        B = int(P.line_windows(ts)[0].sum())
        maps, probs = random_maps(rng, B), random_probs(rng, B)
        for head in (0, 1, 2):
            ids = line_ids(rng, B, head)
            got = [np.zeros((R, 210), np.int32), np.zeros((R, 210), np.float32), np.zeros(R, np.int32),
                   np.zeros((R, 208, 4, 2), np.float32), np.zeros((R, 208, 2), np.float32)]
            args = [np.ascontiguousarray(maps, np.float32), i32(ids), np.ascontiguousarray(probs, np.float32),
                    i32(sizes), geom, turns] + got
            lib.emu_turned_line_stitch(B, R, head, code, *[x.ctypes.data for x in args])
            want = turned_stitch_ref(maps, ids, probs, head, code, sizes, geom, turns)
            for g, w in zip(got, want):
                assert np.array_equal(g.view(np.uint32) if g.dtype == np.float32 else g,
                                      w.view(np.uint32) if w.dtype == np.float32 else w), (turn, head)
