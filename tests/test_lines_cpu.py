"""Text lines read in overlapping windows: CPU checks of the window layout (its properties, the library's host entry
point), of the kernels' bodies run on the host against tests/golden/pre_lines.npz (window crops cut from the
unmodified reference crops by oracle/gen_golden_lines.py) and of the stitch against oracle/line_ref.py, bit for bit."""
import ctypes as C
import functools
import os

import numpy as np
import pytest
import torch

from tests.support import emu
from tests.test_char_boxes_cpu import random_maps
from tests.test_curve_crops_cpu import random_polygons

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


def line_fixture():
    z = np.load(os.path.join(GOLD, 'pre_lines.npz'))
    pages = [z[f'page{i}'] for i in range(int(z['n_pages']))]
    return z, pages


def bind(lib):
    """Bind tests/emu/line_emu.cpp (host compile of the line kernels' bodies)."""
    lib.emu_line_windows.restype = None
    lib.emu_line_windows.argtypes = [C.c_int] + [C.c_void_p] * 4
    lib.emu_line_crops.restype = None
    lib.emu_line_crops.argtypes = [C.c_int, C.c_int] + [C.c_void_p] * 11 + [C.c_int, C.c_int, C.c_void_p]
    lib.emu_line_stitch.restype = None
    lib.emu_line_stitch.argtypes = [C.c_int] * 4 + [C.c_void_p] * 10


# the emulation under the name tools/bench_lines.py loads it by
build_emu = functools.partial(emu, 'line_emu', bind)


def i32(v):
    return np.ascontiguousarray(np.asarray(v, dtype=np.int32))


def emu_line_crops(lib, pages, regions, page_index, kind):
    """alm_pre_line_crops' three launches on the host with the library's own plan -> f32 [sum n, 3, 32, 128]."""
    from advancedliteratemachinery_b200 import preprocess as P
    pages = [np.ascontiguousarray(p) for p in pages]
    plan = P.line_plan([p.shape[:2] for p in pages], regions, page_index, kind)
    coefs, where = [], {}

    def weights(n_in, n_out):
        if (n_in, n_out) not in where:
            b, k = P.resample_coeffs(n_in, n_out, 'bicubic')
            where[(n_in, n_out)] = (sum(a.size for a in coefs), k.shape[1])
            coefs.extend([b.ravel(), k.ravel()])
        return where[(n_in, n_out)]

    hw, vw = [], []
    for (cw, ch), n, wn in zip(plan['sizes'], plan['n'], plan['wn']):
        hw += [weights(int(wn), 128)] * int(n)
        vw += [weights(int(ch), 32)] * int(n)
    coef = i32(np.concatenate(coefs))
    hb, hk, vb, vk = i32([a for a, _ in hw]), i32([k for _, k in hw]), i32([a for a, _ in vw]), i32([k for _, k in vw])
    ptrs = (C.c_void_p * len(pages))(*[p.ctypes.data for p in pages])
    ph, pw, pi = i32([p.shape[0] for p in pages]), i32([p.shape[1] for p in pages]), i32(page_index)
    out = np.zeros((int(plan['n'].sum()), 3, 32, 128), np.float32)
    code = 1 if kind == 'quad' else 2
    lib.emu_line_crops(code, len(pi), ptrs, ph.ctypes.data, pw.ctypes.data, pi.ctypes.data, plan['geom'].ctypes.data,
                       i32(plan['sizes']).ctypes.data, coef.ctypes.data, hb.ctypes.data, hk.ctypes.data, vb.ctypes.data,
                       vk.ctypes.data, 32, 128, out.ctypes.data)
    return out, plan


def emu_line_stitch(lib, maps, ids, probs, head, kind, sizes, geom):
    """line_box_kernel + line_stitch_kernel of one head on the host -> (ids, probs, n, boxes, centres)."""
    maps = np.ascontiguousarray(maps, np.float32)
    probs = np.ascontiguousarray(probs, np.float32)
    sizes, ids = i32(sizes), i32(ids)
    geom = np.ascontiguousarray(np.asarray(geom, np.float64).reshape(len(sizes), -1))
    R = len(sizes)
    out = (np.zeros((R, 210), np.int32), np.zeros((R, 210), np.float32), np.zeros(R, np.int32),
           np.zeros((R, 208, 4, 2), np.float32), np.zeros((R, 208, 2), np.float32))
    lib.emu_line_stitch(maps.shape[0], R, head, kind, maps.ctypes.data, ids.ctypes.data, probs.ctypes.data,
                        sizes.ctypes.data, geom.ctypes.data, *[o.ctypes.data for o in out])
    return out


def random_sizes(rng, n):
    ch = rng.integers(1, 80, n)
    aspect = rng.choice([0.3, 1, 3.9, 4, 4.1, 7, 12, 25, 25.3, 40, 200], n) * rng.uniform(0.9, 1.1, n)
    cw = np.maximum(1, (ch * aspect).astype(np.int64))
    s = np.stack([cw, ch], 1)
    s[:4] = [[1, 1], [4, 1], [5, 1], [100000, 3]]
    return s.astype(np.int32)


def test_layout_properties():
    """Windows cover [0, cw), neighbours overlap by >= ch, one window iff cw <= 4 ch, at most 8 windows and widened
    exactly as stated, x_i = min(i (wn - ov), cw - wn), seams increase."""
    from oracle import line_ref as L
    rng = np.random.default_rng(0)
    for cw, ch in random_sizes(rng, 5000).tolist():
        n, wn, x0 = L.windows(cw, ch)
        assert (n == 1) == (cw <= 4 * ch)
        assert 1 <= n <= 8 and len(x0) == n and x0[0] == 0 and x0[-1] + wn == cw and 1 <= wn <= cw
        if n == 1:
            assert wn == cw
            continue
        natural = 1 + -(-(cw - 4 * ch) // (3 * ch))
        assert wn == (4 * ch if natural <= 8 else -(-(cw + 7 * ch) // 8))
        assert n == min(natural, 8) and wn >= 4 * ch
        assert x0 == [min(i * (wn - ch), cw - wn) for i in range(n)]
        for a, b in zip(x0, x0[1:]):
            # covered, overlap of at least one line height; widened windows of lines 1 or 2 px high can coincide
            assert a + wn - b >= ch and (a < b or (n == 8 and ch <= 2))
        c = L.seams(x0, wn)
        assert all(a < b for a, b in zip(c, c[1:]))
        assert all(x0[i + 1] <= c[i] < x0[i] + wn for i in range(n - 1))  # each seam inside its overlap


def test_host_entry_point_equals_rule():
    """alm_pre_line_windows (through preprocess.line_windows) and the emulation's layout equal the Python rule; a side
    < 1 is refused."""
    from advancedliteratemachinery_b200 import _lib, preprocess as P
    from oracle import line_ref as L
    sizes = random_sizes(np.random.default_rng(1), 3000)
    n, x0, wn = P.line_windows(sizes)
    lib = emu('line_emu', bind)
    en, ex0, ewn = np.zeros_like(n), np.zeros_like(x0), np.zeros_like(wn)
    lib.emu_line_windows(len(sizes), i32(sizes).ctypes.data, en.ctypes.data, ex0.ctypes.data, ewn.ctypes.data)
    assert np.array_equal(n, en) and np.array_equal(x0, ex0) and np.array_equal(wn, ewn)
    for r, (cw, ch) in enumerate(sizes.tolist()):
        n_, wn_, xs = L.windows(cw, ch)
        assert n[r] == n_ and wn[r] == wn_ and x0[r, :n_].tolist() == xs and not x0[r, n_:].any()
    assert P.line_windows(np.zeros((0, 2)))[0].shape == (0,)
    for bad in ([[0, 5]], [[5, 0]], [[3, -1]]):
        with pytest.raises(_lib.AlmError):
            P.line_windows(bad)


def test_oracle_window_crops_equal_fixture():
    """The oracle's windows (full crop, column slice, Pillow resize) of its own restated crops equal the fixture."""
    pytest.importorskip('cv2')
    from oracle import curve_crop_ref as V
    from oracle import line_ref as L
    from oracle import quad_crop_ref as Q
    z, pages = line_fixture()
    qcrops = [Q.crop_image(pages[p], Q.order_point(q)) for q, p in zip(z['quads'], z['quad_page_index'])]
    ccrops = [V.curve_crop(pages[p], *V.curve_plan(poly)) for poly, p in zip(z['polys'], z['curve_page_index'])]
    for name, crops in (('quad', qcrops), ('curve', ccrops)):
        assert np.array_equal([[c.shape[1], c.shape[0]] for c in crops], z[f'{name}_sizes'])
        want = torch.from_numpy(z[f'{name}_out_u8']).to(torch.float32).div(255)
        assert torch.equal(L.line_crops(crops)[1], want)


@pytest.mark.parametrize('kind', ['quad', 'curve'])
def test_kernel_bodies_on_the_host_equal_fixture(kind):
    """The three window-crop launches (line_warp_kernel with the full crop's warp, then the Pillow passes) run on the
    host with the library's plan reproduce every fixture window bit for bit, and the plan's sizes and window counts
    are the fixture's."""
    z, pages = line_fixture()
    regions, pidx = (z['quads'], z['quad_page_index']) if kind == 'quad' else (z['polys'], z['curve_page_index'])
    got, plan = emu_line_crops(emu('line_emu', bind), pages, regions, pidx, kind)
    assert np.array_equal(plan['sizes'], z[f'{kind}_sizes']) and np.array_equal(plan['n'], z[f'{kind}_n'])
    want = torch.from_numpy(z[f'{kind}_out_u8']).to(torch.float32).div(255).numpy()
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


def random_probs(rng, B):
    return rng.uniform(0.01, 1.0, (B, 27)).astype(np.float32)


def line_ids(rng, B, head):
    """Top-1 ids of B windows: an end id at a random position or none, '[GO]' (0) now and then."""
    end = {0: 1, 1: 2, 2: 102}[head]
    ids = rng.integers(3, 100, (B, 27))
    for b in range(B):
        k = rng.integers(0, 32)
        if k < 27:
            ids[b, k] = end
        if rng.random() < 0.3:
            ids[b, rng.integers(1, 27)] = 0
    return ids.astype(np.int32)


def line_plans(rng, R):
    """(quad plan, curve plan) of R random lines from the library's planners: long rotated lines, short words, a
    page-size-fallback quad and curved bands."""
    from advancedliteratemachinery_b200 import preprocess as P
    c = rng.uniform(100, 900, (R, 2))
    w, h, t = rng.uniform(10, 900, R), rng.uniform(1, 40, R), rng.uniform(-0.5, 0.5, R)
    box = np.stack([np.stack([-w, -h], 1), np.stack([w, -h], 1), np.stack([w, h], 1), np.stack([-w, h], 1)], 1) / 2
    rot = np.stack([np.stack([np.cos(t), -np.sin(t)], 1), np.stack([np.sin(t), np.cos(t)], 1)], 1)
    quads = (np.einsum('nij,nkj->nki', rot, box) + c[:, None]).astype(np.float32)
    quads[0] = c[0] + rng.uniform(-0.4, 0.4, (4, 2))  # page-size fallback: 1200 x 1000
    q = P.line_plan([(1000, 1200)], quads, np.zeros(R, np.int32), 'quad')
    polys = random_polygons(rng, R, 1000, 1000)
    cv = P.line_plan([(1000, 1000)], polys, np.zeros(R, np.int32), 'curve')
    assert (q['n'] == 1).any() and (q['n'] == 8).any() and (cv['n'] > 1).any()
    return q, cv


@pytest.mark.parametrize('kind', ['quad', 'curve'])
def test_stitch_on_the_host_equals_oracle(kind):
    """line_box_kernel + line_stitch_kernel's bodies on the host equal oracle/line_ref.stitch_lines bit for bit on
    random maps, ids and probabilities, for every head."""
    from oracle import line_ref as L
    rng = np.random.default_rng(20 + (kind == 'curve'))
    plan = line_plans(rng, 40)[kind == 'curve']
    B = int(plan['n'].sum())
    maps, probs = random_maps(rng, B), random_probs(rng, B)
    lib = emu('line_emu', bind)
    code = 1 if kind == 'quad' else 2
    for head in (0, 1, 2):
        ids = line_ids(rng, B, head)
        got = emu_line_stitch(lib, maps, ids, probs, head, code, plan['sizes'], plan['geom'])
        want = L.stitch_lines(maps, ids, probs, head, code, plan['sizes'], plan['geom'])
        for g, w in zip(got, want):
            assert np.array_equal(g.view(np.uint32) if g.dtype == np.float32 else g,
                                  w.view(np.uint32) if w.dtype == np.float32 else w)
        assert (got[2] > 26).any() and (got[2] < 26).any()


def mix(u0, w0, u1, w1):
    """A map with mass w0 / w1 in the patch columns centred at u0 / u1 (u = 4x + 2), one row: centroid w0 u0 + w1 u1."""
    a = np.zeros(257, np.float32)
    a[1 + 32 * 2 + (u0 - 2) // 4] += w0
    a[1 + 32 * 2 + (u1 - 2) // 4] += w1
    return a


def test_seams_overlap_and_missing_ends():
    """Hand-made two-window lines: a character seen by both windows of the overlap appears once, a token whose centre
    lies exactly on a seam goes to the right window, a window without an end token contributes all 26 tokens, and a
    last window without an end token ends the line with probability 0.  Host bodies and oracle agree on each."""
    from oracle import line_ref as L
    lib = emu('line_emu', bind)
    geom = np.eye(3).reshape(1, 9)

    def both(maps, ids, probs, cw):
        got = emu_line_stitch(lib, maps, ids, probs, 1, 1, [[cw, 32]], geom)
        want = L.stitch_lines(maps, ids, probs, 1, 1, [[cw, 32]], geom)
        for g, w in zip(got, want):
            assert np.array_equal(g, w)
        return got

    # cw 192: windows [0, 128) and [64, 192), seam 95.5; X = x_i + u - 0.5
    assert L.windows(192, 32) == (2, 128, [0, 64]) and L.seams([0, 64], 128) == [95.5]
    maps = np.zeros((2, 27, 257), np.float32)
    ids = np.full((2, 27), 7, np.int32)
    probs = np.full((2, 27), 0.5, np.float32)
    for s, u in enumerate([10, 94, 98]):    # X = 9.5, 93.5 (kept), 97.5 (right of the seam: dropped)
        maps[0, s + 1] = mix(u, 1.0, u, 0.0)
        ids[0, s + 1] = 10 + s
    for s, u in enumerate([30, 34, 58]):    # X = 93.5 (window 0 has it: dropped), 97.5, 121.5
        maps[1, s + 1] = mix(u, 1.0, u, 0.0)
        ids[1, s + 1] = 20 + s
    ids[:, 4] = 2
    probs[1, 4] = 0.25
    got = both(maps, ids, probs, 192)
    assert got[2][0] == 4 and got[0][0, :7].tolist() == [7, 10, 11, 21, 22, 2, 2]
    assert got[1][0, 5] == np.float32(0.25) and (got[1][0, 6:] == 1.0).all()
    assert np.array_equal(got[4][0, :4, 0], np.float32([9.5, 93.5, 97.5, 121.5]))

    # cw 193: windows [0, 128) and [65, 193), seam 96.0; a centre exactly on it goes right
    assert L.windows(193, 32) == (2, 128, [0, 65]) and L.seams([0, 65], 128) == [96.0]
    on = np.zeros((2, 27, 257), np.float32)
    on[0, 1] = mix(94, 0.375, 98, 0.625)    # centroid 96.5: X = 96.0 in window 0 -> not kept there
    on[1, 1] = mix(30, 0.625, 34, 0.375)    # centroid 31.5: X = 65 + 31.5 - 0.5 = 96.0 in window 1 -> kept
    assert L.window_box(on[0, 1], 0, 128, 1, 193, 32, geom)[2] == 96.0
    assert L.window_box(on[1, 1], 65, 128, 1, 193, 32, geom)[2] == 96.0
    ids3 = np.full((2, 27), 7, np.int32)
    ids3[0, 1], ids3[1, 1] = 40, 41
    ids3[:, 2] = 2
    got = both(on, ids3, probs, 193)
    assert got[2][0] == 1 and got[0][0, 1] == 41

    # no end token in either window: 26 tokens each before the seam test, and the line ends with probability 0
    mr = random_maps(np.random.default_rng(5), 2)
    noend = np.full((2, 27), 9, np.int32)
    got = both(mr, noend, probs, 192)
    n = got[2][0]
    assert n >= 26 and got[0][0, n + 1] == 2 and got[1][0, n + 1] == 0.0 and got[1][0, n + 2] == 1.0
    # only the first window lacks one: the last window's end probability closes the line
    ends = noend.copy()
    ends[1, 5] = 2
    probs2 = probs.copy()
    probs2[1, 5] = 0.125
    got = both(mr, ends, probs2, 192)
    assert got[1][0, got[2][0] + 1] == np.float32(0.125)


def test_single_window_lines_equal_char_boxes():
    """A line of one window stitches to the crop's own ids through the end token and to char_box_ref's boxes."""
    from oracle import char_box_ref as V
    from oracle import line_ref as L
    rng = np.random.default_rng(7)
    q, _ = line_plans(rng, 60)
    rows = np.flatnonzero(q['n'] == 1)
    sizes, geom = q['sizes'][rows], q['geom'][rows]
    B = len(rows)
    maps, probs = random_maps(rng, B), random_probs(rng, B)
    lib = emu('line_emu', bind)
    for head in (1, 2):
        ids = line_ids(rng, B, head)
        got = emu_line_stitch(lib, maps, ids, probs, head, 1, sizes, geom)
        n, boxes, centres = V.char_boxes(maps, ids, head, 1, sizes, geom)
        assert np.array_equal(got[2], n)
        assert np.array_equal(got[3][:, :26].view(np.uint32), boxes.view(np.uint32))
        assert np.array_equal(got[4][:, :26].view(np.uint32), centres.view(np.uint32))
        for b in range(B):
            e = n[b] + 2 if n[b] < 26 else 27
            assert np.array_equal(got[0][b, :e], ids[b, :e]) and np.array_equal(got[1][b, :e], probs[b, :e])
        assert L.LINE_LEN == 210


def test_mgp_fuse_reads_stitched_lines():
    """postprocess.mgp_fuse takes stitched [3, R, 210] sequences: the text of each head is its kept tokens."""
    from advancedliteratemachinery_b200 import postprocess as Post
    from oracle.char_box_ref import CHAR_TABLE
    ids = np.zeros((3, 1, 210), np.int32)
    ids[0, 0, 1:41] = np.arange(40) % 36 + 2
    ids[0, 0, 41:] = 1
    ids[1, 0, 1:] = 2
    ids[2, 0, 1:] = 102
    probs = np.ones((3, 1, 210), np.float32)
    fuse = Post.mgp_fuse(ids, probs, CHAR_TABLE, ['x'] * 50257, ['y'] * 30522)
    assert fuse['texts'][0][0] == ''.join(CHAR_TABLE[i] for i in ids[0, 0, 1:41]) and fuse['fused'][0] == fuse['texts'][0][0]
