"""Boxes of the recognised characters from MGP-STR's A^3 maps: CPU checks of the oracle's map selection against the
reference's own slicing (OCR/MGP-STR/demo.py:119-124) on the fixture maps, of the kernel's per-slot body run on the
host against the oracle (bit for bit), and of the geometry the boxes land in."""
import ctypes as C
import os

import numpy as np
import pytest

from tests.support import emu
from tests.test_curve_crops_cpu import random_polygons

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


def bind(lib):
    """Bind tests/emu/char_box_emu.cpp (host compile of char_box_kernel's body)."""
    lib.emu_char_boxes.restype = None
    lib.emu_char_boxes.argtypes = [C.c_int, C.c_int, C.c_int] + [C.c_void_p] * 7


def emu_char_boxes(lib, maps, ids, head, kind=0, sizes=None, geom=None):
    """char_box_kernel's grid on the host -> (n [B], boxes [B, 26, 4, 2], centres [B, 26, 2])."""
    maps = np.ascontiguousarray(maps, np.float32)
    ids = np.ascontiguousarray(ids, np.int32)
    B = maps.shape[0]
    sz = np.ascontiguousarray(sizes if sizes is not None else np.zeros((B, 2)), np.int32)
    g = np.ascontiguousarray(np.asarray(geom, np.float64).reshape(B, -1) if geom is not None else np.zeros((B, 16)))
    n = np.zeros(B, np.int32)
    boxes = np.zeros((B, 26, 4, 2), np.float32)
    centres = np.zeros((B, 26, 2), np.float32)
    lib.emu_char_boxes(B, head, kind, maps.ctypes.data, ids.ctypes.data, sz.ctypes.data, g.ctypes.data, n.ctypes.data,
                       boxes.ctypes.data, centres.ctypes.data)
    return n, boxes, centres


def fixture_maps():
    """(maps [B, 27, 257], char ids [B, 27]) of the MGP-STR and CHAR-STR reference fixtures, and the BPE / WordPiece
    ids of the MGP-STR one."""
    out = []
    for name in ('mgp_b3', 'mgp_charstr', 'mgp_b1'):
        z = np.load(os.path.join(GOLD, f'{name}.npz'))
        extra = {h: z[k] for h, k in ((1, 'bpe_ids'), (2, 'wp_ids')) if k in z.files}
        out.append((z['char_attn'], z['char'].argmax(-1), extra))
    return out


def id_variants(rng, ids):
    """The fixture's ids plus the cases the rule has to get right: '[GO]' (4 characters) before '[s]', no '[s]',
    '[s]' first, and enough '[GO]'s to pass the 26-slot cap."""
    v = [ids.copy()]
    a = ids.copy(); a[1:4] = [5, 0, 7]; a[4] = 1; v.append(a)            # [GO] inside the word
    b = ids.copy(); b[b == 1] = 9; v.append(b)                          # no [s]: n = 0
    c = ids.copy(); c[1] = 1; v.append(c)                               # [s] first: n = 0
    d = ids.copy(); d[1:9] = 0; d[9] = 1; v.append(d)                   # 8 x '[GO]' = 32 characters: cap at 26
    e = rng.integers(0, 38, 27); v.append(e)
    return v


def test_map_selection_equals_reference_slice():
    """The oracle's count selects exactly the maps of attens[h][b][:, 1:].view(-1, 8, 32)[1:EOS+1] (char head, EOS the
    string index of '[s]') and of the first end id (BPE / WordPiece), on the fixture maps."""
    from oracle import char_box_ref as V
    rng = np.random.default_rng(1)
    seen = set()
    for maps, char_ids, extra in fixture_maps():
        for b in range(maps.shape[0]):
            for ids in id_variants(rng, char_ids[b]):
                n = V.box_count(ids, 0)
                want = V.reference_maps(maps[b], ids, 0)
                assert want.shape[0] == n
                assert np.array_equal(maps[b, 1:n + 1, 1:].reshape(n, 8, 32), want)
                seen.add(n if n in (0, 26) else 'mid')
            for head, hid in extra.items():
                for ids in (hid[b], np.where(hid[b] == V.END_ID[head], 3, hid[b])):
                    n = V.box_count(ids, head)
                    assert V.reference_maps(maps[b], ids, head).shape[0] == n
                    assert np.array_equal(maps[b, 1:n + 1, 1:].reshape(n, 8, 32), V.reference_maps(maps[b], ids, head))
    assert seen == {0, 26, 'mid'}


def test_char_count_equals_mgp_fuse_string_index():
    """The ids-only count is the string index of '[s]' that postprocess.mgp_fuse finds in its char_decode: the fused
    char text has exactly n characters whenever '[s]' occurs below the cap."""
    from advancedliteratemachinery_b200 import postprocess as Post
    from oracle import char_box_ref as V
    rng = np.random.default_rng(2)
    ids = np.stack([v for _, cids, _ in fixture_maps() for b in range(cids.shape[0]) for v in id_variants(rng, cids[b])])
    ids = np.concatenate([ids, rng.integers(0, 38, (200, 27))]).astype(np.int32)
    ids3 = np.stack([ids, np.full_like(ids, 2), np.full_like(ids, 102)])
    fused = Post.mgp_fuse(ids3, np.ones(ids3.shape, np.float32), V.CHAR_TABLE, ['x'] * 3, ['y'] * 103)
    checked = 0
    for b, row in enumerate(ids):
        n = V.box_count(row, 0)
        if 1 in row[1:] and n < 26:
            assert len(fused['texts'][0][b]) == n, (b, row)
            checked += 1
    assert checked > 50


def random_maps(rng, B):
    """A^3-like maps [B, 27, 257]: softmaxes at several temperatures, one-hot patches, all mass on cls (mass 0 over
    the patches) and a few exact zeros."""
    logits = rng.standard_normal((B, 27, 257)) * rng.choice([0.5, 3.0, 12.0], (B, 1, 1))
    m = np.exp(logits - logits.max(-1, keepdims=True))
    m = (m / m.sum(-1, keepdims=True)).astype(np.float32)
    m[0, 1] = 0; m[0, 1, 0] = 1                       # cls only
    m[0, 2] = 0; m[0, 2, 1 + 32 * 3 + 17] = 1         # one patch
    m[-1, 1:, 1 + 32 * 5:1 + 32 * 6] = 0              # a zero row
    return m


def random_ids(rng, B):
    ids = rng.integers(2, 38, (B, 27))
    for b in range(B):
        k = rng.integers(0, 30)
        if k < 27:
            ids[b, k] = 1
        if rng.random() < 0.3:
            ids[b, rng.integers(1, 27)] = 0
    return ids.astype(np.int32)


def plans(rng, B):
    """(quad plan, curve plan) of B random regions, from the library's own planners: includes quads that fall back
    to the page size and 1-pixel crop sides."""
    from advancedliteratemachinery_b200 import preprocess as P
    c = rng.uniform(50, 950, (B, 1, 2))
    quads = c + rng.uniform(-80, 80, (B, 4, 2))
    quads[:4] = c[:4] + rng.uniform(-0.4, 0.4, (4, 4, 2))         # truncated size 0: warped at the page's size
    q = P.quad_plan([(1000, 1200)], quads.astype(np.float32), np.zeros(B, np.int32))
    polys = random_polygons(rng, B, 1000, 1000)
    polys[:3] = np.float32(300.0) + rng.uniform(0, 0.3, (3, 16, 2)).astype(np.float32)  # 1 x 1 crops
    cv = P.curve_plan([(1000, 1000)], polys, np.zeros(B, np.int32))
    assert (q['sizes'] == [1200, 1000]).all(1).any() and (cv['sizes'] == 1).any()
    return q, cv


@pytest.mark.parametrize('kind', [0, 1, 2])
def test_kernel_body_on_the_host_equals_oracle(kind):
    """char_box_kernel's per-slot body (csrc/box_core.h) compiled for the host equals the oracle bit for bit on random
    maps and ids, for plain, quad and curve crops and all three heads."""
    from oracle import char_box_ref as V
    rng = np.random.default_rng(10 + kind)
    B = 48
    maps, ids = random_maps(rng, B), random_ids(rng, B)
    q, cv = plans(rng, B)
    sizes, geom = {0: (None, None), 1: (q['sizes'], q['minv']), 2: (cv['sizes'], cv['ctrl'])}[kind]
    lib = emu('char_box_emu', bind)
    for head in (0, 1, 2):
        hid = ids if head == 0 else np.where(ids == 1, V.END_ID[head], ids)
        got = emu_char_boxes(lib, maps, hid, head, kind, sizes, geom)
        want = V.char_boxes(maps, hid, head, kind, sizes, geom)
        assert np.array_equal(got[0], want[0])
        assert np.array_equal(got[1].view(np.uint32), want[1].view(np.uint32))
        assert np.array_equal(got[2].view(np.uint32), want[2].view(np.uint32))
        assert (got[0] > 0).sum() > B // 3


def test_one_hot_column_maps_to_its_span():
    """All of a map's patch mass in column x: the band is that column's 10 % .. 90 % span, 4x + [0.4, 3.6] in the
    input's edge coordinates, the centre the column's middle; and the host kernel body agrees."""
    from oracle import char_box_ref as V
    rng = np.random.default_rng(3)
    maps = np.zeros((1, 27, 257), np.float32)
    for x in range(26):
        col = rng.random(8).astype(np.float32)
        maps[0, x + 1, 1 + 32 * np.arange(8) + x] = col / col.sum()
    ids = np.full((1, 27), 5, np.int32); ids[0, 0] = 0
    n, boxes, centres = emu_char_boxes(emu('char_box_emu', bind), maps, ids, 1)  # BPE head without an end id: 26 boxes
    assert n[0] == 26
    for x in range(26):
        L, R, xc, _ = V.reduce_map(maps[0, x + 1])
        assert abs(L - (4 * x + 0.4)) < 1e-12 and abs(R - (4 * x + 3.6)) < 1e-12 and abs(xc - (4 * x + 2)) < 1e-12
        want = np.float32([[4 * x - 0.1, 0], [4 * x + 3.1, 0], [4 * x + 3.1, 31], [4 * x - 0.1, 31]])
        assert np.abs(boxes[0, x] - want).max() < 1e-5, x
        assert abs(centres[0, x, 0] - (4 * x + 1.5)) < 1e-5


def test_axis_aligned_region_gives_affine_boxes():
    """An axis-aligned rectangle: every box is an axis-aligned rectangle whose sides are the input coordinates scaled
    by the crop's map, and whose top and bottom are the region's."""
    from advancedliteratemachinery_b200 import preprocess as P
    from oracle import char_box_ref as V
    rng = np.random.default_rng(4)
    x0, y0, x1, y1 = 120.0, 40.0, 420.0, 90.0
    quad = np.float32([[[x0, y0], [x1, y0], [x1, y1], [x0, y1]]])
    plan = P.quad_plan([(500, 600)], quad, [0])
    cw, ch = (int(v) for v in plan['sizes'][0])
    maps, ids = random_maps(rng, 1), random_ids(rng, 1)
    ids[0, 20] = 1; ids[0, :20] = 7
    n, boxes, centres = emu_char_boxes(emu('char_box_emu', bind), maps, ids, 0, 1, plan['sizes'], plan['minv'])
    assert n[0] == 19
    sx, sy = (x1 - x0) / (cw - 1), (y1 - y0) / (ch - 1)
    for j in range(n[0]):
        L, R, xc, yc = V.reduce_map(maps[0, j + 1])
        X = np.array([L, R]) * cw / 128 - 0.5
        want = np.array([[x0 + X[0] * sx, y0], [x0 + X[1] * sx, y0], [x0 + X[1] * sx, y1], [x0 + X[0] * sx, y1]])
        assert np.abs(boxes[0, j] - want).max() < 1e-3, j
        assert boxes[0, j, 0, 1] == boxes[0, j, 1, 1] and boxes[0, j, 0, 0] == boxes[0, j, 3, 0]
        c = [x0 + (xc * cw / 128 - 0.5) * sx, y0 + (yc * ch / 32 - 0.5) * sy]
        assert np.abs(centres[0, j] - c).max() < 1e-3
    assert not boxes[0, n[0]:].any() and not centres[0, n[0]:].any()


def test_curved_boxes_follow_the_arc():
    """A 100 degree annular sector (radii 300 and 252): the top corners of every box lie on the top Bezier, the
    bottom corners on the bottom one (within 1e-6 x the region's extent), and all of them within 1 px of their
    circle; boxes advance along the arc with their maps' mass."""
    from advancedliteratemachinery_b200 import preprocess as P
    from oracle import char_box_ref as V
    from oracle.curve_crop_ref import _bezier
    cx, cy, r_top, r_bottom = 400.0, 420.0, 300.0, 252.0
    phi = np.radians(90 + 50 - 100 * np.arange(8) / 7)
    ring = lambda r: np.stack([cx + r * np.cos(phi), cy - r * np.sin(phi)], 1)
    poly = np.concatenate([ring(r_top), ring(r_bottom)[::-1]]).astype(np.float32)
    plan = P.curve_plan([(800, 800)], poly[None], [0])
    cw, ch = (int(v) for v in plan['sizes'][0])
    ctrl = plan['ctrl'][0]
    rng = np.random.default_rng(6)
    maps = random_maps(rng, 1)
    ids = np.full((1, 27), 9, np.int32); ids[0, 0] = 0
    n, boxes, centres = emu_char_boxes(emu('char_box_emu', bind), maps, ids, 2, 2, plan['sizes'], plan['ctrl'])
    assert n[0] == 26
    extent = float(np.ptp(poly, axis=0).max())
    for j in range(26):
        L, R, _, _ = V.reduce_map(maps[0, j + 1])
        t = (np.array([L, R]) * cw / 128 - 0.5) / (cw - 1)
        top, bottom = _bezier(ctrl[0], t), _bezier(ctrl[1], 1 - t)
        assert np.abs(boxes[0, j, [0, 1]] - top).max() <= 1e-6 * extent, j
        assert np.abs(boxes[0, j, [3, 2]] - bottom).max() <= 1e-6 * extent, j
        rad = np.hypot(boxes[0, j, :, 0] - cx, boxes[0, j, :, 1] - cy)
        assert np.abs(rad - [r_top, r_top, r_bottom, r_bottom]).max() < 1.0, j
    # a one-hot column at the left and at the right end of the input sits at the arc's two ends
    maps[0, 1:] = 0
    maps[0, 1, 1] = 1
    maps[0, 2, 1 + 31] = 1
    _, boxes, _ = emu_char_boxes(emu('char_box_emu', bind), maps, ids, 2, 2, plan['sizes'], plan['ctrl'])
    assert np.abs(boxes[0, 0, 0] - poly[0]).max() < 3 and np.abs(boxes[0, 1, 1] - poly[7]).max() < 3


def test_fused_boxes_pairs_the_source_head():
    from advancedliteratemachinery_b200 import postprocess as Post
    n = np.array([[2, 0, 1], [5, 26, 0], [1, 3, 4]], np.int32)
    boxes = np.arange(3 * 3 * 26 * 8, dtype=np.float32).reshape(3, 3, 26, 4, 2)
    centres = np.arange(3 * 3 * 26 * 2, dtype=np.float32).reshape(3, 3, 26, 2)
    fuse = {'fused': ['ab', 'xyz', ''], 'source': np.array([0, 1, -1], np.int32)}
    out = Post.fused_boxes(fuse, n, boxes, centres)
    assert [d['text'] for d in out] == ['ab', 'xyz', ''] and [d['source'] for d in out] == [0, 1, -1]
    assert np.array_equal(out[0]['boxes'], boxes[0, 0, :2]) and np.array_equal(out[1]['centres'], centres[1, 1, :26])
    assert out[2]['boxes'].shape == (0, 4, 2) and out[2]['centres'].shape == (0, 2)
