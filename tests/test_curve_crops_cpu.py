"""Curved text rectified along the Bezier curves of OmniParser's 16-point polygons, then MGP-STR's resize + ToTensor:
CPU checks of the oracle, of the library's host plan and of the kernels' per-pixel bodies run on the host, against
tests/golden/pre_curves.npz (control points from the unmodified reference's bezier_fit_quad, written by
oracle/gen_golden_curves.py).  Bar: bit-exact crops and tensors everywhere; control points within 1e-9 x the
polygon's extent of bezier_fit_quad (the library solves the same least-squares problem in its own code)."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from tests.support import emu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
REF_MISC = '/root/reference/OCR/OmniParser/utils/misc.py'


def curve_fixture():
    z = np.load(os.path.join(GOLD, 'pre_curves.npz'))
    pages = [z[f'page{i}'] for i in range(int(z['n_pages']))]
    crops = [z[f'crop{i}'] for i in range(int(z['n']))]
    out = torch.from_numpy(z['out_u8']).to(torch.float32).div(255)  # ToTensor of the reference's resized crops
    return z, pages, crops, out


def _bernstein(Cp, t):
    t = t[:, None]
    u = 1 - t
    return u ** 3 * Cp[0] + 3 * t * u ** 2 * Cp[1] + 3 * t ** 2 * u * Cp[2] + t ** 3 * Cp[3]


def random_polygons(rng, n, h, w, max_len=400.0):
    """Curved bands (random cubic top boundary, bottom offset along its normal, any rotation), free 16-point
    scribbles, slivers, regions off the page and boundaries with only 2 or 3 distinct points -> f32 [n, 16, 2]."""
    out = np.empty((n, 16, 2))
    ts = np.linspace(0, 1, 8)
    for i in range(n):
        c = rng.uniform([-0.1 * w, -0.1 * h], [1.1 * w, 1.1 * h])
        kind = rng.integers(0, 5)
        if kind == 2:  # free
            out[i] = c + rng.uniform(-60, 60, (16, 2))
            continue
        L = rng.uniform(0.2, max_len) if kind != 3 else rng.uniform(0.05, 0.8)
        Cp = np.array([[0, 0], [L / 3, rng.normal(0, L / 4)], [2 * L / 3, rng.normal(0, L / 4)], [L, rng.normal(0, L / 8)]])
        top = _bernstein(Cp, ts)
        d = np.gradient(top, axis=0)
        nrm = np.stack([-d[:, 1], d[:, 0]], 1) / np.maximum(np.linalg.norm(d, axis=1, keepdims=True), 1e-9)
        bottom = top + nrm * rng.uniform(0.5, 60) * (1 + 0.1 * rng.standard_normal((8, 1)))
        if kind == 4:  # rank-deficient boundary: 2 or 3 distinct positions
            k = int(rng.integers(2, 4))
            idx = np.sort(np.concatenate([np.arange(k), rng.integers(0, k, 8 - k)]))
            pick = np.round(np.linspace(0, 7, k)).astype(int)
            if rng.random() < 0.5:
                top = top[pick][idx]
            else:
                bottom = bottom[pick][idx]
        a = rng.uniform(-np.pi, np.pi)
        rot = np.array([[np.cos(a), -np.sin(a)], [np.sin(a), np.cos(a)]])
        out[i] = np.concatenate([top, bottom[::-1]]) @ rot.T + c
    return out.astype(np.float32)


def curve_regions(seed, n_pages=16, per_page=64, size=1024):
    """A detection-sized workload: n_pages random pages with per_page curved text lines each -> (pages, polys,
    page_index)."""
    rng = np.random.default_rng(seed)
    pages = [rng.integers(0, 256, (size, size, 3), dtype=np.uint8) for _ in range(n_pages)]
    polys = random_polygons(rng, n_pages * per_page, size, size)
    return pages, polys, np.repeat(np.arange(n_pages, dtype=np.int32), per_page)


def bind(lib):
    """Bind tests/emu/curve_emu.cpp (host compile of the kernels' per-pixel bodies)."""
    lib.emu_curve_crops.restype = None
    lib.emu_curve_crops.argtypes = [C.c_int] + [C.c_void_p] * 11 + [C.c_int, C.c_int, C.c_void_p, C.c_void_p]


def emu_curve_crops(lib, pages, polys, page_index, imgH=32, imgW=128):
    """The three launches of alm_pre_curve_crops on the host, with the library's own plan and resize weights ->
    (packed crops u8 [sum w*h, 3], plan dict, out f32 [R, 3, imgH, imgW])."""
    from advancedliteratemachinery_b200 import preprocess as P
    pages = [np.ascontiguousarray(p) for p in pages]
    plan = P.curve_plan([p.shape[:2] for p in pages], polys, page_index)
    sizes, ctrl = plan['sizes'], np.ascontiguousarray(plan['ctrl'])
    R = len(sizes)
    coefs, where = [], {}

    def weights(n_in, n_out):
        if (n_in, n_out) not in where:
            b, k = P.resample_coeffs(n_in, n_out, 'bicubic')
            where[(n_in, n_out)] = (sum(a.size for a in coefs), k.shape[1])
            coefs.extend([b.ravel(), k.ravel()])
        return where[(n_in, n_out)]

    hw = [weights(int(w), imgW) for w, _ in sizes]
    vw = [weights(int(h), imgH) for _, h in sizes]
    coef = np.ascontiguousarray(np.concatenate(coefs).astype(np.int32)) if coefs else np.zeros(1, np.int32)
    i32 = lambda v: np.ascontiguousarray(np.asarray(v, dtype=np.int32))
    hb, hk, vb, vk = i32([a for a, _ in hw]), i32([k for _, k in hw]), i32([a for a, _ in vw]), i32([k for _, k in vw])
    ptrs = (C.c_void_p * len(pages))(*[p.ctypes.data for p in pages])
    ph, pw, pi = i32([p.shape[0] for p in pages]), i32([p.shape[1] for p in pages]), i32(page_index)
    warped = np.zeros((int((sizes[:, 0].astype(np.int64) * sizes[:, 1]).sum()), 3), np.uint8)
    out = np.zeros((R, 3, imgH, imgW), np.float32)
    lib.emu_curve_crops(R, ptrs, ph.ctypes.data, pw.ctypes.data, pi.ctypes.data, ctrl.ctypes.data, i32(sizes).ctypes.data,
                        coef.ctypes.data, hb.ctypes.data, hk.ctypes.data, vb.ctypes.data, vk.ctypes.data, imgH, imgW,
                        warped.ctypes.data, out.ctypes.data)
    return warped, plan, out


def unpack(warped, sizes):
    crops, off = [], 0
    for w, h in sizes:
        crops.append(warped[off:off + w * h].reshape(h, w, 3))
        off += w * h
    assert off == warped.shape[0]
    return crops


def test_oracle_equals_fixture():
    pytest.importorskip('cv2')
    from oracle import curve_crop_ref as V
    z, pages, crops, out = curve_fixture()
    plans = [V.curve_plan(p) for p in z['polys']]
    for r, (ctrl, cw, ch) in enumerate(plans):
        assert np.array_equal(ctrl, z['ctrl'][r]) and (cw, ch) == tuple(z['sizes'][r]), r
    got_crops, got = V.curve_crops(pages, z['polys'], z['page_index'])
    assert all(np.array_equal(a, b) for a, b in zip(got_crops, crops))
    assert torch.equal(got, out)
    assert np.array_equal(crops[0], pages[0][30:60, 20:119])  # axis-aligned box: a plain slice of the page


def test_generator_check_against_unmodified_reference():
    """What oracle/gen_golden_curves.py asserts before it writes the fixture: the restated fit equals the reference's
    own bezier_fit_quad (utils/misc.py imported unmodified), on the fixture and on random boundaries."""
    if not os.path.isfile(REF_MISC):
        pytest.skip('reference sources not present')
    from oracle import curve_crop_ref as V
    from oracle import gen_golden_curves as G
    ref = G.reference_module()
    z, _, _, _ = curve_fixture()
    for r, poly in enumerate(z['polys']):
        assert np.array_equal(G.reference_ctrl(ref, poly), z['ctrl'][r]), r
    rng = np.random.default_rng(5)
    for poly in random_polygons(rng, 300, 1024, 1024):
        p = poly.astype(np.float64)
        for side in (p[:8], p[8:]):
            assert np.array_equal(V.side_ctrl(side), ref.bezier_fit_quad(side[:, 0], side[:, 1]))


def _fixture_and_random(n, seed):
    z, pages, _, _ = curve_fixture()
    rng = np.random.default_rng(seed)
    sizes = [p.shape[:2] for p in pages] + [(1024, 1024)]
    polys = np.concatenate([z['polys'], random_polygons(rng, n, 1024, 1024)])
    pidx = np.concatenate([z['page_index'], np.full(n, len(pages), np.int32)])
    return sizes, polys, pidx


def test_plan_sizes_equal_oracle():
    from advancedliteratemachinery_b200 import preprocess as P
    from oracle import curve_crop_ref as V
    sizes, polys, pidx = _fixture_and_random(10000, 11)
    plan = P.curve_plan(sizes, polys, pidx)
    want = np.asarray([V.crop_size(p) for p in polys], np.int32)
    assert np.array_equal(plan['sizes'], want)
    assert (want == 1).all(axis=1).any()  # the sub-pixel case


def test_plan_control_points_match_bezier_fit_quad():
    """Within 1e-9 x max(1, polygon extent) of the (reference-equal) restated fit on the fixture and 10 000 random
    polygons, rank-deficient boundaries included.  The library takes the pseudo-inverse by a Jacobi eigen-decomposition,
    numpy by LAPACK's SVD, so the last bits differ; the worst distance is printed."""
    from advancedliteratemachinery_b200 import preprocess as P
    from oracle import curve_crop_ref as V
    sizes, polys, pidx = _fixture_and_random(10000, 12)
    ctrl = P.curve_plan(sizes, polys, pidx)['ctrl']
    worst, n_rank = 0.0, 0
    for r, poly in enumerate(polys):
        p = poly.astype(np.float64)
        want = np.stack([V.side_ctrl(p[:8]), V.side_ctrl(p[8:])])
        scale = max(1.0, float(np.ptp(p, axis=0).max()))
        err = float(np.abs(ctrl[r] - want).max()) / scale
        assert err <= 1e-9, (r, err)
        worst = max(worst, err)
        n_rank += any(len(np.unique(s, axis=0)) in (2, 3) for s in (p[:8], p[8:]))
    assert n_rank > 100
    print(f'\ncontrol points: worst distance to bezier_fit_quad {worst:.2e} x extent over {len(polys)} polygons '
          f'({n_rank} with a rank-deficient boundary)')


def test_zero_length_boundary():
    """A boundary whose points all coincide (bezier_fit_quad raises LinAlgError there) gets four control points equal
    to its first point; the other boundary is fitted as usual."""
    from advancedliteratemachinery_b200 import preprocess as P
    from oracle import curve_crop_ref as V
    top = np.tile([[40.5, 30.25]], (8, 1))
    bottom = np.stack([np.linspace(90, 10, 8), np.full(8, 60.0)], 1)
    poly = np.concatenate([top, bottom]).astype(np.float32)
    plan = P.curve_plan([(100, 120)], poly[None], [0])
    assert np.array_equal(plan['ctrl'][0, 0], np.tile([[40.5, 30.25]], (4, 1)))
    assert np.abs(plan['ctrl'][0, 1] - V.side_ctrl(poly[8:].astype(np.float64))).max() < 1e-9 * 80
    assert tuple(plan['sizes'][0]) == V.crop_size(poly)
    both = np.tile([[7.0, 9.0]], (16, 1)).astype(np.float32)
    plan = P.curve_plan([(100, 120)], both[None], [0])
    assert np.array_equal(plan['ctrl'][0], np.tile([[7.0, 9.0]], (2, 4, 1))) and tuple(plan['sizes'][0]) == (1, 1)


def test_plan_rejects_bad_regions():
    from advancedliteratemachinery_b200 import _lib, preprocess as P
    z, _, _, _ = curve_fixture()
    p = z['polys'][1:2].copy()
    nan, inf = p.copy(), p.copy()
    nan[0, 3, 1] = np.nan
    inf[0, 12, 0] = -np.inf
    far = p + np.float32(1.1e6)                                   # control points beyond 2^20
    xs = np.linspace(0, 40000, 8)
    long = np.concatenate([np.stack([xs, np.zeros(8)], 1), np.stack([xs[::-1], np.full(8, 20.0)], 1)])[None]
    tall = np.concatenate([np.stack([np.linspace(0, 20, 8), np.zeros(8)], 1),   # crop sides above 32766
                           np.stack([np.linspace(20, 0, 8), np.full(8, 40000.0)], 1)])[None]
    for polys, pidx in ((p, [1]), (p, [-1]), (nan, [0]), (inf, [0]), (far, [0]), (long, [0]), (tall, [0])):
        with pytest.raises(_lib.AlmError) as e:
            P.curve_plan([(100, 120)], polys, pidx)
        assert e.value.code == -1
    ok = long.copy()
    ok[..., 0] *= 32765.0 / 40000  # just inside cv2.remap's limit
    assert P.curve_plan([(100, 120)], ok, [0])['sizes'][0, 0] == 32766
    assert P.curve_plan([(100, 120)], np.zeros((0, 16, 2)), [])['sizes'].shape == (0, 2)


def test_kernel_bodies_on_the_host_equal_fixture():
    """The per-pixel functions the CUDA kernels execute (csrc/quad_core.h, preproc_core.h), compiled for the host and
    run over every launch's grid with the library's plan and weights, reproduce every reference crop and the final
    tensor bit for bit."""
    z, pages, crops, out = curve_fixture()
    warped, plan, got = emu_curve_crops(emu('curve_emu', bind), pages, z['polys'], z['page_index'])
    assert np.array_equal(plan['sizes'], z['sizes'])
    for r, (a, b) in enumerate(zip(unpack(warped, plan['sizes']), crops)):
        assert np.array_equal(a, b), r
    assert np.array_equal(got.view(np.uint32), out.numpy().view(np.uint32))


def test_kernel_bodies_equal_oracle_on_random_polygons():
    """1 000 random polygons on a 1024 x 1024 page: the host run of the kernel bodies equals the oracle (numpy map +
    cv2.remap + Pillow) fed with the library's plan, bit for bit."""
    pytest.importorskip('cv2')
    from oracle import curve_crop_ref as V
    rng = np.random.default_rng(21)
    pages = [rng.integers(0, 256, (1024, 1024, 3), dtype=np.uint8)]
    polys = random_polygons(rng, 1000, 1024, 1024)
    pidx = np.zeros(1000, np.int32)
    warped, plan, got = emu_curve_crops(emu('curve_emu', bind), pages, polys, pidx)
    plans = [(plan['ctrl'][r], int(w), int(h)) for r, (w, h) in enumerate(plan['sizes'])]
    crops, ref = V.curve_crops(pages, polys, pidx, plans=plans)
    for r, (a, b) in enumerate(zip(unpack(warped, plan['sizes']), crops)):
        assert np.array_equal(a, b), r
    assert np.array_equal(got.view(np.uint32), ref.numpy().view(np.uint32))


def test_rectification_follows_an_arc():
    """A 100 degree annular sector (radii 300 and 252): every map point lies within 1 px of the radius its row should
    have, where the chord through the end points would be up to ~38 px off."""
    from advancedliteratemachinery_b200 import preprocess as P
    from oracle import curve_crop_ref as V
    cx, cy, r_top, r_bottom = 400.0, 420.0, 300.0, 252.0
    phi = np.radians(90 + 50 - 100 * np.arange(8) / 7)
    ring = lambda r: np.stack([cx + r * np.cos(phi), cy - r * np.sin(phi)], 1)
    poly = np.concatenate([ring(r_top), ring(r_bottom)[::-1]]).astype(np.float32)
    plan = P.curve_plan([(800, 800)], poly[None], [0])
    cw, ch = (int(v) for v in plan['sizes'][0])
    mx, my = V.curve_map(plan['ctrl'][0], cw, ch)
    s = np.arange(ch)[:, None] / (ch - 1)
    radius = np.hypot(mx.astype(np.float64) - cx, my.astype(np.float64) - cy)
    err = np.abs(radius - (r_top + (r_bottom - r_top) * s))
    assert err.max() < 1.0, err.max()
    assert abs(cw - 0.5 * (r_top + r_bottom) * np.radians(100)) < 2  # the crop is as wide as the arc is long


def test_polygons_array():
    from advancedliteratemachinery_b200 import postprocess as Post
    polys = np.arange(2 * 32, dtype=np.float64).reshape(2, 32)
    p = Post.polygons_array(polys)
    assert p.dtype == np.float32 and p.shape == (2, 16, 2)
    assert np.array_equal(p, polys.reshape(2, 16, 2).astype(np.float32))
    assert np.array_equal(Post.polygons_array([{'polys': p[i].tolist()} for i in range(2)]), p)
