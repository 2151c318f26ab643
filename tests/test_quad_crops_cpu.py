"""Perspective crops of detected text regions (DocXChain's TextRecognition.order_point + crop_image, then MGP-STR's
resize + ToTensor): CPU checks of the oracle, of the library's host plan and of the kernels' per-pixel bodies run on
the host, against tests/golden/pre_quads.npz (generated from the unmodified reference module by
oracle/gen_golden_quads.py).  Bar: bit-exact everywhere; the inverse maps equal cv2.invert's (the closed form warpPerspective
itself uses) bit for bit."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from tests.support import emu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
REF_MODULES = '/root/reference/Applications/DocXChain/modules'


def quad_fixture():
    z = np.load(os.path.join(GOLD, 'pre_quads.npz'))
    pages = [z[f'page{i}'] for i in range(int(z['n_pages']))]
    crops = [z[f'crop{i}'] for i in range(int(z['n']))]
    out = torch.from_numpy(z['out_u8']).to(torch.float32).div(255)  # ToTensor of the reference's resized crops
    return z, pages, crops, out


def random_quads(rng, n, h, w):
    """Rotated boxes, free quads, slivers and regions partly or wholly off the page."""
    kind = rng.integers(0, 4, n)
    c = rng.uniform([-0.1 * w, -0.1 * h], [1.1 * w, 1.1 * h], (n, 2))
    bw, bh = rng.uniform(2, 0.5 * w, n), rng.uniform(1, 0.2 * h, n)
    t = rng.uniform(-np.pi, np.pi, n)
    box = np.stack([np.stack([-bw, -bh], 1), np.stack([bw, -bh], 1), np.stack([bw, bh], 1), np.stack([-bw, bh], 1)], 1) / 2
    rot = np.stack([np.stack([np.cos(t), -np.sin(t)], 1), np.stack([np.sin(t), np.cos(t)], 1)], 1)
    q = np.einsum('nij,nkj->nki', rot, box) + c[:, None]
    q[kind == 1] += rng.uniform(-0.1, 0.1, (int((kind == 1).sum()), 4, 2)) * bw[kind == 1, None, None]  # perspective
    q[kind == 2] = c[kind == 2, None] + rng.uniform(-60, 60, (int((kind == 2).sum()), 4, 2))          # free
    q[kind == 3] = c[kind == 3, None] + rng.uniform(-0.6, 0.6, (int((kind == 3).sum()), 4, 2))        # sub-pixel
    perm = np.argsort(rng.random((n, 4)), 1)                                                           # any order
    return np.take_along_axis(q, perm[:, :, None], 1).astype(np.float32)


def text_regions(seed, n_pages=16, per_page=64, size=1024):
    """A detection-sized workload: n_pages random pages with per_page text-like quads each (rotated words and lines,
    some with perspective, some reaching past the page edge, two sub-pixel ones) -> (pages, quads, page_index)."""
    rng = np.random.default_rng(seed)
    pages = [rng.integers(0, 256, (size, size, 3), dtype=np.uint8) for _ in range(n_pages)]
    n = n_pages * per_page
    c = rng.uniform(-0.05 * size, 1.05 * size, (n, 2))
    bw, bh = rng.uniform(16, 0.4 * size, n), rng.uniform(8, 64, n)
    t = rng.normal(0, 0.3, n)
    box = np.stack([np.stack([-bw, -bh], 1), np.stack([bw, -bh], 1), np.stack([bw, bh], 1), np.stack([-bw, bh], 1)], 1) / 2
    rot = np.stack([np.stack([np.cos(t), -np.sin(t)], 1), np.stack([np.sin(t), np.cos(t)], 1)], 1)
    q = np.einsum('nij,nkj->nki', rot, box) + c[:, None] + rng.uniform(-4, 4, (n, 4, 2))
    q[[5, n // 2]] = c[[5, n // 2], None] + rng.uniform(-0.4, 0.4, (2, 4, 2))
    perm = np.argsort(rng.random((n, 4)), 1)
    q = np.take_along_axis(q, perm[:, :, None], 1).astype(np.float32)
    return pages, q, np.repeat(np.arange(n_pages, dtype=np.int32), per_page)


def bind(lib):
    """Bind tests/emu/quad_emu.cpp (host compile of the kernels' per-pixel bodies)."""
    lib.emu_quad_crops.restype = None
    lib.emu_quad_crops.argtypes = [C.c_int] + [C.c_void_p] * 11 + [C.c_int, C.c_int, C.c_void_p, C.c_void_p]


def emu_quad_crops(lib, pages, quads, page_index, imgH=32, imgW=128):
    """quadcrop.cu's three launches on the host, with the library's own plan and resize weights ->
    (packed crops u8 [sum w*h, 3], sizes [R, 2] (w, h), out f32 [R, 3, imgH, imgW])."""
    from advancedliteratemachinery_b200 import preprocess as P
    pages = [np.ascontiguousarray(p) for p in pages]
    plan = P.quad_plan([p.shape[:2] for p in pages], quads, page_index)
    sizes, minv = plan['sizes'], np.ascontiguousarray(plan['minv'])
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
    coef = np.ascontiguousarray(np.concatenate(coefs).astype(np.int32))
    i32 = lambda v: np.ascontiguousarray(np.asarray(v, dtype=np.int32))
    hb, hk, vb, vk = i32([a for a, _ in hw]), i32([k for _, k in hw]), i32([a for a, _ in vw]), i32([k for _, k in vw])
    ptrs = (C.c_void_p * len(pages))(*[p.ctypes.data for p in pages])
    ph, pw, pi = i32([p.shape[0] for p in pages]), i32([p.shape[1] for p in pages]), i32(page_index)
    warped = np.zeros((int((sizes[:, 0].astype(np.int64) * sizes[:, 1]).sum()), 3), np.uint8)
    out = np.zeros((R, 3, imgH, imgW), np.float32)
    lib.emu_quad_crops(R, ptrs, ph.ctypes.data, pw.ctypes.data, pi.ctypes.data, minv.ctypes.data, i32(sizes).ctypes.data,
                       coef.ctypes.data, hb.ctypes.data, hk.ctypes.data, vb.ctypes.data, vk.ctypes.data, imgH, imgW,
                       warped.ctypes.data, out.ctypes.data)
    return warped, sizes, out


def test_oracle_equals_fixture():
    pytest.importorskip('cv2')
    from oracle import quad_crop_ref as Q
    z, pages, crops, out = quad_fixture()
    got_crops, got = Q.quad_crops(pages, z['quads'], z['page_index'])
    assert all(np.array_equal(a, b) for a, b in zip(got_crops, crops))
    assert torch.equal(got, out)


def test_generator_check_against_unmodified_reference():
    """What oracle/gen_golden_quads.py asserts before it writes the fixture: the restatement equals the reference's own
    TextRecognition.order_point / crop_image, imported unmodified."""
    cv2 = pytest.importorskip('cv2')
    if not os.path.isdir(REF_MODULES):
        pytest.skip('reference sources not present')
    from oracle import gen_golden_quads as G
    from oracle import quad_crop_ref as Q
    ref = G.reference_module()
    z, pages, crops, _ = quad_fixture()
    for q, p, crop in zip(z['quads'], z['page_index'], crops):
        pts = ref.order_point(q)
        assert np.array_equal(pts, Q.order_point(q))
        assert np.array_equal(ref.crop_image(pages[p], pts), crop)


def test_plan_equals_reference_arithmetic():
    """alm_pre_quad_plan == order_point / crop_image's corners and crop sizes exactly, on the fixture quads and 10 000
    random ones; its inverse maps == cv2.invert(cv2.getPerspectiveTransform(...)) bit for bit.  Their distance to
    numpy's LAPACK inverse of the same matrix is printed for scale: cv2's closed-form 3x3 inverse (adjugate / det)
    is not LU, and on these matrices (entries from ~1e-6 to ~1e3) the two differ by far more than a few ulp, so it
    is cv2.invert that the crops must follow."""
    from advancedliteratemachinery_b200 import preprocess as P
    from oracle import quad_crop_ref as Q
    z, pages, _, _ = quad_fixture()
    rng = np.random.default_rng(17)
    sizes = [p.shape[:2] for p in pages] + [(1024, 1024)]
    quads = np.concatenate([z['quads'], random_quads(rng, 10000, 1024, 1024)])
    pidx = np.concatenate([z['page_index'], np.full(10000, len(pages), np.int32)])
    plan = P.quad_plan(sizes, quads, pidx)
    cv2 = None
    try:
        import cv2
    except ImportError:
        pass
    dev, n_fallback = [], 0
    for r, (q, p) in enumerate(zip(quads, pidx)):
        pts = Q.order_point(q)
        corners, dst, w, h = Q.crop_plan(pts)
        assert np.array_equal(plan['ordered'][r], pts), r
        assert np.array_equal(plan['corners'][r], corners), r
        cw, ch = int(w), int(h)
        if cw <= 0 or ch <= 0:
            ch, cw = sizes[p]
            n_fallback += 1
        assert tuple(plan['sizes'][r]) == (cw, ch), r
        if cv2 is not None:
            M = cv2.getPerspectiveTransform(corners, dst)
            ok, Mi = cv2.invert(M)
            assert np.array_equal(plan['minv'][r].view(np.uint64), Mi.view(np.uint64)), r
            ref = np.linalg.inv(M)
            scale = np.spacing(np.abs(ref).max(axis=1, keepdims=True))
            dev.append(float((np.abs(plan['minv'][r] - ref) / scale).max()))
    assert n_fallback > 0  # the sub-pixel cases took the page-size fallback
    if cv2 is not None:
        q50, q99, worst = np.percentile(dev, [50, 99, 100])
        print(f'\ninverse maps: bit-identical to cv2.invert for {len(quads)} regions; distance to np.linalg.inv in ulp '
              f'of the row\'s largest entry: median {q50:.0f}, 99th percentile {q99:.0f}, max {worst:.3g}')


def test_plan_rejects_bad_regions():
    from advancedliteratemachinery_b200 import _lib, preprocess as P
    q = np.array([[[10, 10], [50, 12], [49, 30], [9, 28]]], np.float32)
    for quads, pidx in ((q, [1]), (q, [-1]), (np.where(np.arange(8).reshape(1, 4, 2) == 3, np.nan, q), [0]),
                        (np.where(np.arange(8).reshape(1, 4, 2) == 0, np.inf, q), [0])):
        with pytest.raises(_lib.AlmError) as e:
            P.quad_plan([(100, 120)], quads, pidx)
        assert e.value.code == -1
    assert P.quad_plan([(100, 120)], np.zeros((0, 4, 2)), [])['sizes'].shape == (0, 2)


def test_kernel_bodies_on_the_host_equal_fixture():
    """The per-pixel functions the CUDA kernels execute (csrc/quad_core.h, preproc_core.h), compiled for the host and
    run over every launch's grid with the library's plan and weights, reproduce every reference crop and the final
    tensor bit for bit."""
    z, pages, crops, out = quad_fixture()
    warped, sizes, got = emu_quad_crops(emu('quad_emu', bind), pages, z['quads'], z['page_index'])
    assert np.array_equal(sizes, z['sizes'])
    off = 0
    for r, crop in enumerate(crops):
        n = crop.shape[0] * crop.shape[1]
        assert np.array_equal(warped[off:off + n].reshape(crop.shape), crop), r
        off += n
    assert off == warped.shape[0]
    assert np.array_equal(got.view(np.uint32), out.numpy().view(np.uint32))


def test_quads_from_polygons():
    from advancedliteratemachinery_b200 import postprocess as Post
    polys = np.arange(2 * 32, dtype=np.float64).reshape(2, 32)
    q = Post.quads_from_polygons(polys)
    assert q.dtype == np.float32 and q.shape == (2, 4, 2)
    p = polys.reshape(2, 16, 2)
    assert np.array_equal(q, p[:, [0, 7, 8, 15]].astype(np.float32))
    dicts = [{'polys': p[i].tolist()} for i in range(2)]
    assert np.array_equal(Post.quads_from_polygons(dicts), q)
