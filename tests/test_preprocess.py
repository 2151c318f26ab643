"""Test-time image pipeline: CPU checks of the oracle and of the host-side size planning against fixtures generated
from the reference's own transforms + Pillow (oracle/gen_golden_pre.py), and the GPU parity tests of the CUDA path.
Bar: bit-exact (integer resampling; ToTensor / Normalize are single IEEE float32 operations per element)."""
import os

import numpy as np
import pytest
import torch

from tests.support import emu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


def _omni():
    z = np.load(os.path.join(GOLD, 'pre_omni.npz'))
    pages = [z[f'page{i}'] for i in range(int(z['n_pages']))]
    return z, pages


def _mgp():
    z = np.load(os.path.join(GOLD, 'pre_mgp.npz'))
    return z, [z[f'crop{i}'] for i in range(int(z['n']))]


def test_oracle_equals_reference_fixtures():
    from oracle import preprocess_ref as O
    z, pages = _omni()
    t, m = O.omni_pages(pages, int(z['min_size']), int(z['max_size']))
    assert torch.equal(t, torch.from_numpy(z['tensors'])) and torch.equal(m, torch.from_numpy(z['mask']))
    zc, crops = _mgp()
    assert torch.equal(O.mgp_crops(crops, 32, 128), torch.from_numpy(zc['out']))


def test_oracle_resample_equals_pillow():
    Image = pytest.importorskip('PIL.Image')
    from oracle import preprocess_ref as O
    rng = np.random.default_rng(3)
    for _ in range(25):
        h, w, oh, ow = (int(v) for v in rng.integers(1, 60, 4))
        img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        for name, flt in (('bilinear', Image.BILINEAR), ('bicubic', Image.BICUBIC)):
            assert np.array_equal(np.asarray(Image.fromarray(img).resize((ow, oh), flt)), O.resize(img, oh, ow, name))


def test_kernel_weights_equal_the_pinned_oracle():
    """The host-side weight computation the CUDA passes consume (alm_pre_coeffs) == the oracle's, which is pinned to
    Pillow: up- and down-scaling, both filters, degenerate 1-pixel lengths."""
    from advancedliteratemachinery_b200 import preprocess as P
    from oracle import preprocess_ref as O
    rng = np.random.default_rng(11)
    cases = [(1, 1), (1, 9), (9, 1), (1024, 1024), (1500, 1024), (333, 1824), (4000, 32), (31, 128)]
    cases += [tuple(int(v) for v in rng.integers(1, 700, 2)) for _ in range(60)]
    for in_size, out_size in cases:
        for name in ('bilinear', 'bicubic'):
            bounds, coefs = P.resample_coeffs(in_size, out_size, name)
            ob, ok = O.precompute(in_size, out_size, name)
            assert np.array_equal(bounds, ob) and np.array_equal(coefs, ok), (in_size, out_size, name)


def bind(lib):
    """Bind tests/emu/preproc_emu.cpp (host compile of the kernels' per-pixel bodies)."""
    import ctypes as C
    for f in (lib.emu_resize_norm, lib.emu_pad_mask):
        f.restype = None
    lib.emu_resize_norm.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p,
                                    C.c_void_p, C.c_int, C.c_void_p, C.c_long, C.c_int, C.c_void_p, C.c_void_p, C.c_int]
    lib.emu_pad_mask.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p]


def _emu_batch(lib, images, sizes, canvas, filter_name, normalize):
    """The launch sequence of pre_resize_batch (preproc.cu) on the host emulation."""
    from advancedliteratemachinery_b200 import preprocess as P
    Hc, Wc = canvas
    n = len(images)
    out = np.zeros((n, 3, Hc, Wc), dtype=np.float32)              # cudaMemsetAsync(out, 0)
    mean = np.asarray([0.485, 0.456, 0.406], dtype=np.float32)
    sd = np.asarray([0.229, 0.224, 0.225], dtype=np.float32)
    for b, (im, (oh, ow)) in enumerate(zip(images, sizes)):
        im = np.ascontiguousarray(im)
        hb, hk = P.resample_coeffs(im.shape[1], ow, filter_name)
        vb, vk = P.resample_coeffs(im.shape[0], oh, filter_name)
        lib.emu_resize_norm(im.ctypes.data, im.shape[0], im.shape[1], oh, ow, hb.ctypes.data, hk.ctypes.data, hk.shape[1],
                            vb.ctypes.data, vk.ctypes.data, vk.shape[1], out[b].ctypes.data, Hc * Wc, Wc, mean.ctypes.data,
                            sd.ctypes.data, 1 if normalize else 0)
    mask = np.zeros((n, Hc, Wc), dtype=np.uint8)
    sz = np.asarray(sizes, dtype=np.int32)
    lib.emu_pad_mask(mask.ctypes.data, n, Hc, Wc, sz.ctypes.data)
    return out, mask


def test_kernel_bodies_on_the_host_equal_reference_fixtures():
    """The per-pixel functions the CUDA kernels execute (csrc/preproc_core.h), compiled for the host and driven in the
    kernels' launch order with the library's own size plan and weights, reproduce the reference outputs bit for bit."""
    from advancedliteratemachinery_b200 import preprocess as P
    lib = emu('preproc_emu', bind)
    z, pages = _omni()
    sizes, canvas = P.omni_plan([p.shape[:2] for p in pages], int(z['min_size']), int(z['max_size']))
    out, mask = _emu_batch(lib, pages, sizes, canvas, 'bilinear', True)
    assert np.array_equal(out.view(np.uint32), z['tensors'].view(np.uint32))     # bit pattern, not just value
    assert np.array_equal(mask.astype(bool), z['mask'])
    zc, crops = _mgp()
    out, _ = _emu_batch(lib, crops, [(32, 128)] * len(crops), (32, 128), 'bicubic', False)
    assert np.array_equal(out.view(np.uint32), zc['out'].view(np.uint32))


def test_size_plan_equals_reference_rule():
    """alm_pre_omni_plan (host-only C entry point) == RandomResize.get_size_with_aspect_ratio on 400 recorded cases."""
    from advancedliteratemachinery_b200 import preprocess as P
    z, _ = _omni()
    for (h, w, mn, mx), ref in zip(z['sizes_in'].tolist(), z['sizes_out'].tolist()):
        sizes, canvas = P.omni_plan([(h, w)], mn, mx)
        assert sizes[0] == tuple(ref) and canvas == tuple(ref), (h, w, mn, mx)
    sizes, canvas = P.omni_plan([(480, 640), (1000, 500), (64, 64)], 64, 96)
    assert canvas == (max(s[0] for s in sizes), max(s[1] for s in sizes))


@pytest.mark.gpu
@pytest.mark.parametrize('on_device', [False, True])
def test_gpu_omni_pages_equal_reference(on_device):
    from advancedliteratemachinery_b200 import _lib, preprocess as P
    z, pages = _omni()
    ctx = _lib.Context(0)
    ims = [torch.from_numpy(p).cuda() if on_device else p for p in pages]
    nt = P.omni_pages(ctx, ims, int(z['min_size']), int(z['max_size']))
    assert torch.equal(nt.tensors.cpu(), torch.from_numpy(z['tensors']))
    assert torch.equal(nt.mask.cpu(), torch.from_numpy(z['mask']))
    ctx.close()


@pytest.mark.gpu
def test_gpu_mgp_crops_equal_reference():
    from advancedliteratemachinery_b200 import _lib, preprocess as P
    z, crops = _mgp()
    ctx = _lib.Context(0)
    out = P.mgp_crops(ctx, crops, 32, 128)
    assert torch.equal(out.cpu(), torch.from_numpy(z['out']))
    ctx.close()


@pytest.mark.gpu
def test_gpu_page_scale_resize_matches_oracle():
    """A real page size (1500 x 1100 -> shorter side 1024): bit-exact against the oracle."""
    from advancedliteratemachinery_b200 import _lib, preprocess as P
    from oracle import preprocess_ref as O
    rng = np.random.default_rng(5)
    page = rng.integers(0, 256, (1500, 1100, 3), dtype=np.uint8)
    ctx = _lib.Context(0)
    nt = P.omni_pages(ctx, [page], 1024, 1824)
    t, m = O.omni_pages([page], 1024, 1824)
    assert torch.equal(nt.tensors.cpu(), t) and torch.equal(nt.mask.cpu(), m)
    ctx.close()
