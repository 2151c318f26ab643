"""Test-time image pipeline on the GPU through the C ABI.

    omni_plan(sizes, test_min_size, test_max_size)   RandomResize.get_size_with_aspect_ratio per page + batch canvas
                                                     (OCR/OmniParser/dataset/transforms.py:275-296; host only)
    omni_pages(ctx, images, ...) -> NestedTensor     RandomResize -> ToTensor -> Normalize -> nested_tensor_from_tensor_list
                                                     (dataset/__init__.py:109-113, transforms.py:249-298,312-322,
                                                      utils/nested_tensor.py:37-54), on the device
    mgp_crops(ctx, images, imgH, imgW) -> tensor     PIL bicubic resize + ToTensor (OCR/MGP-STR/demo.py:126-132)
    quad_plan(sizes, quads, page_index) -> dict      order_point + crop_image's corners, crop sizes, inverse maps
                                                     (Applications/DocXChain/modules/text_recognition.py:84-145; host)
    quad_crops(ctx, pages, quads, page_index, ...)   perspective crop of every region + mgp_crops, on the device
    curve_plan(sizes, polys, page_index) -> dict     Bezier control points (OCR/OmniParser/utils/misc.py:81-110) and
                                                     crop sizes of 16-point polygons (host)
    curve_crops(ctx, pages, polys, page_index, ...)  curved text rectified along its boundary curves + mgp_crops, on
                                                     the device
    line_windows(sizes) / line_plan(...)             the overlapping 4:1 windows a long text line is read in (host)
    line_crops(ctx, pages, regions, page_index, kind) every window of every quad / curved line + mgp_crops, on the
                                                     device
    omni_tile_plan(sizes, tile, overlap)             the overlapping tiles a page larger than OmniParser's input is
                                                     spotted in (host)
    omni_tiles(ctx, pages, tile, overlap, ...)       those tiles cut from the pages (optionally turned by quarter-turns)
                                                     + omni_pages' transform, on the device
    omni_tiles_at(ctx, pages, index, tile, overlap, ...)  the tiles of a list of plan indices, cut the same way
                                                     (optionally of turned pages)

`images`: decoded 8-bit RGB pages, each a uint8 array / tensor [h, w, 3] (host numpy / torch, or CUDA torch).
"""
from __future__ import annotations

import ctypes as C
from typing import List, Sequence, Tuple

import numpy as np
import torch

from . import _lib
from .nested_tensor import NestedTensor


def omni_plan(sizes: Sequence[Tuple[int, int]], test_min_size: int, test_max_size: int):
    """sizes: (h, w) per page -> (resized [(h, w), ...], (Hmax, Wmax))."""
    lib = _lib.load()
    n = len(sizes)
    hs = np.asarray([s[0] for s in sizes], dtype=np.int32)
    ws = np.asarray([s[1] for s in sizes], dtype=np.int32)
    out = np.zeros((max(n, 1), 2), dtype=np.int32)
    hm, wm = C.c_int(0), C.c_int(0)
    rc = lib.alm_pre_omni_plan(hs.ctypes.data, ws.ctypes.data, n, test_min_size, test_max_size, out.ctypes.data,
                               C.byref(hm), C.byref(wm))
    if rc != 0:
        raise _lib.AlmError(rc, 'alm_pre_omni_plan: invalid sizes')
    return [tuple(int(v) for v in out[i]) for i in range(n)], (hm.value, wm.value)


def resample_coeffs(in_size: int, out_size: int, filter: str = 'bilinear'):
    """(bounds [out,2], coefs [out,ksize]) int32: the fixed-point weights one resampling pass of the kernels uses."""
    lib = _lib.load()
    f = {'bilinear': 0, 'bicubic': 1}[filter]
    k = C.c_int(0)
    lib.alm_pre_coeffs(in_size, out_size, f, C.byref(k), None, None, 0)
    bounds = np.zeros((out_size, 2), dtype=np.int32)
    coefs = np.zeros((out_size, k.value), dtype=np.int32)
    rc = lib.alm_pre_coeffs(in_size, out_size, f, C.byref(k), bounds.ctypes.data, coefs.ctypes.data, coefs.size)
    if rc != 0:
        raise _lib.AlmError(rc, 'alm_pre_coeffs')
    return bounds, coefs


def _image_args(images):
    keep, ptrs, hs, ws = [], [], [], []
    for im in images:
        t = im if isinstance(im, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(im))
        assert t.dtype == torch.uint8 and t.dim() == 3 and t.shape[2] == 3, 'pages must be uint8 [h, w, 3]'
        t = t.contiguous()
        keep.append(t)
        ptrs.append(t.data_ptr())
        hs.append(t.shape[0])
        ws.append(t.shape[1])
    n = len(keep)
    return keep, (C.c_void_p * n)(*ptrs), np.asarray(hs, dtype=np.int32), np.asarray(ws, dtype=np.int32), n


def omni_pages(ctx: _lib.Context, images: List, test_min_size: int, test_max_size: int) -> NestedTensor:
    """The reference's validation transform + batching, on the GPU: returns the NestedTensor `model(samples, seqs)` takes
    (tensors f32 [n,3,Hmax,Wmax] normalised and zero padded, mask bool [n,Hmax,Wmax], both on the context's device)."""
    keep, ptrs, hs, ws, n = _image_args(images)
    _, (Hc, Wc) = omni_plan(list(zip(hs.tolist(), ws.tolist())), test_min_size, test_max_size)
    dev = torch.device('cuda', ctx.device)
    tensors = torch.empty(n, 3, Hc, Wc, dtype=torch.float32, device=dev)
    mask = torch.empty(n, Hc, Wc, dtype=torch.uint8, device=dev)
    ctx.wait_torch(*keep)
    ctx.check(ctx.lib.alm_pre_omni_pages(ctx.h, ptrs, hs.ctypes.data, ws.ctypes.data, n, test_min_size, test_max_size,
                                         tensors.data_ptr(), mask.data_ptr()))
    ctx.synchronize()
    return NestedTensor(tensors, mask.bool())


def mgp_crops(ctx: _lib.Context, images: List, imgH: int = 32, imgW: int = 128) -> torch.Tensor:
    """[n,3,imgH,imgW] f32 in [0,1] on the device: `img.resize((imgW, imgH), Image.BICUBIC)` + ToTensor per crop."""
    keep, ptrs, hs, ws, n = _image_args(images)
    out = torch.empty(n, 3, imgH, imgW, dtype=torch.float32, device=torch.device('cuda', ctx.device))
    ctx.wait_torch(*keep)
    ctx.check(ctx.lib.alm_pre_mgp_crops(ctx.h, ptrs, hs.ctypes.data, ws.ctypes.data, n, imgH, imgW, out.data_ptr()))
    ctx.synchronize()
    return out


def _quad_args(quads, page_index):
    q = np.ascontiguousarray(np.asarray(quads, dtype=np.float32).reshape(-1, 4, 2))
    pi = np.ascontiguousarray(np.asarray(page_index, dtype=np.int32).reshape(-1))
    if pi.shape[0] != q.shape[0]:
        raise ValueError(f'{q.shape[0]} quads but {pi.shape[0]} page indices')
    return q, pi


def quad_plan(sizes: Sequence[Tuple[int, int]], quads, page_index):
    """sizes: (h, w) per page; quads: f32 [R, 4, 2] (x, y) page pixel coordinates; page_index: [R] -> dict(ordered f32
    [R,4,2] = TextRecognition.order_point, corners f32 [R,4,2] = crop_image's source corners, sizes int32 [R,2] = crop
    (width, height), minv f64 [R,3,3] = inverse perspective map) exactly as alm_pre_quad_crops uses them (host only)."""
    lib = _lib.load()
    q, pi = _quad_args(quads, page_index)
    R = q.shape[0]
    hs = np.asarray([s[0] for s in sizes], dtype=np.int32)
    ws = np.asarray([s[1] for s in sizes], dtype=np.int32)
    out = dict(ordered=np.zeros((R, 4, 2), np.float32), corners=np.zeros((R, 4, 2), np.float32),
               sizes=np.zeros((R, 2), np.int32), minv=np.zeros((R, 3, 3), np.float64))
    rc = lib.alm_pre_quad_plan(hs.ctypes.data, ws.ctypes.data, len(hs), q.ctypes.data, pi.ctypes.data, R,
                               out['ordered'].ctypes.data, out['corners'].ctypes.data, out['sizes'].ctypes.data,
                               out['minv'].ctypes.data)
    if rc != 0:
        raise _lib.AlmError(rc, 'alm_pre_quad_plan: invalid page index, page size or coordinate')
    return out


def quad_crops(ctx: _lib.Context, pages: List, quads, page_index, imgH: int = 32, imgW: int = 128) -> torch.Tensor:
    """[R,3,imgH,imgW] f32 in [0,1] on the device, the MGP-STR input of every detected region: region r is
    `ToTensor(Image.fromarray(crop_image(pages[page_index[r]], order_point(quads[r]))).resize((imgW, imgH), BICUBIC))`
    (DocXChain's TextRecognition + MGP-STR's transform), bit for bit, in three kernel launches for all regions.
    pages: uint8 [h, w, 3] each (host or CUDA); quads: [R, 4, 2] (x, y) in page pixels, any point order."""
    q, pi = _quad_args(quads, page_index)
    R = q.shape[0]
    out = torch.empty(R, 3, imgH, imgW, dtype=torch.float32, device=torch.device('cuda', ctx.device))
    if R == 0:
        return out
    keep, ptrs, hs, ws, n = _image_args(pages)
    ctx.wait_torch(*keep)
    ctx.check(ctx.lib.alm_pre_quad_crops(ctx.h, ptrs, hs.ctypes.data, ws.ctypes.data, n, q.ctypes.data, pi.ctypes.data, R,
                                         imgH, imgW, out.data_ptr()))
    ctx.synchronize()
    return out


def _poly_args(polys, page_index):
    from .postprocess import polygons_array
    p = polygons_array(polys)
    pi = np.ascontiguousarray(np.asarray(page_index, dtype=np.int32).reshape(-1))
    if pi.shape[0] != p.shape[0]:
        raise ValueError(f'{p.shape[0]} polygons but {pi.shape[0]} page indices')
    return p, pi


def curve_plan(sizes: Sequence[Tuple[int, int]], polys, page_index):
    """sizes: (h, w) per page; polys: OmniParser's 16-point polygons [R, 16, 2] / [R, 32] (x, y) in page pixels, or
    `decode_pred_seq` result dicts; page_index: [R] -> dict(ctrl f64 [R,2,4,2] = control points of the top and the
    bottom boundary, sizes int32 [R,2] = crop (width, height)) exactly as alm_pre_curve_crops uses them (host only)."""
    lib = _lib.load()
    p, pi = _poly_args(polys, page_index)
    R = p.shape[0]
    hs = np.asarray([s[0] for s in sizes], dtype=np.int32)
    ws = np.asarray([s[1] for s in sizes], dtype=np.int32)
    out = dict(ctrl=np.zeros((R, 2, 4, 2), np.float64), sizes=np.zeros((R, 2), np.int32))
    rc = lib.alm_pre_curve_plan(hs.ctypes.data, ws.ctypes.data, len(hs), p.ctypes.data, pi.ctypes.data, R,
                                out['ctrl'].ctypes.data, out['sizes'].ctypes.data)
    if rc != 0:
        raise _lib.AlmError(rc, 'alm_pre_curve_plan: invalid page index, page size, coordinate or crop size')
    return out


def curve_crops(ctx: _lib.Context, pages: List, polys, page_index, imgH: int = 32, imgW: int = 128) -> torch.Tensor:
    """[R,3,imgH,imgW] f32 in [0,1] on the device, the MGP-STR input of every curved text region: region r's polygon
    rectified along the cubic Beziers fitted to its top and bottom boundary (`bezier_fit_quad`), sampled as
    cv2.remap(INTER_LINEAR, BORDER_CONSTANT 0) does it, then `Image.resize((imgW, imgH), BICUBIC)` + ToTensor, bit for
    bit, in three kernel launches for all regions (the rule: include/alm_ocr.h, alm_pre_curve_crops).
    pages: uint8 [h, w, 3] each (host or CUDA); polys: [R, 16, 2] / [R, 32] (x, y) in page pixels, top boundary left
    -> right then bottom boundary right -> left, or `decode_pred_seq` result dicts."""
    p, pi = _poly_args(polys, page_index)
    R = p.shape[0]
    out = torch.empty(R, 3, imgH, imgW, dtype=torch.float32, device=torch.device('cuda', ctx.device))
    if R == 0:
        return out
    keep, ptrs, hs, ws, n = _image_args(pages)
    ctx.wait_torch(*keep)
    ctx.check(ctx.lib.alm_pre_curve_crops(ctx.h, ptrs, hs.ctypes.data, ws.ctypes.data, n, p.ctypes.data, pi.ctypes.data,
                                          R, imgH, imgW, out.data_ptr()))
    ctx.synchronize()
    return out


def line_windows(sizes):
    """sizes: int [R, 2] natural crop (width, height) per region -> (n int32 [R], x0 int32 [R, 8], wn int32 [R]): the
    overlapping 4:1 windows a text line is read in (the rule: include/alm_ocr.h, alm_pre_line_windows; host only)."""
    lib = _lib.load()
    s = np.ascontiguousarray(np.asarray(sizes, dtype=np.int32).reshape(-1, 2))
    R = s.shape[0]
    n, x0, wn = np.zeros(R, np.int32), np.zeros((R, _lib.MAX_LINE_WINDOWS), np.int32), np.zeros(R, np.int32)
    rc = lib.alm_pre_line_windows(s.ctypes.data, R, n.ctypes.data, x0.ctypes.data, wn.ctypes.data)
    if rc != 0:
        raise _lib.AlmError(rc, 'alm_pre_line_windows: a crop side < 1')
    return n, x0, wn


def _line_regions(regions, page_index, kind):
    if kind == 'quad':
        return (_lib.BOX_QUAD,) + _quad_args(regions, page_index)
    if kind == 'curve':
        return (_lib.BOX_CURVE,) + _poly_args(regions, page_index)
    raise ValueError(f"kind must be 'quad' or 'curve', got {kind!r}")


def line_plan(sizes: Sequence[Tuple[int, int]], regions, page_index, kind: str = 'quad'):
    """Text lines read in windows: sizes: (h, w) per page; regions: quads [R, 4, 2] (kind 'quad', as quad_plan) or
    16-point polygons (kind 'curve', as curve_plan) -> dict(sizes int32 [R, 2] natural crop (width, height), geom f64
    [R, 9] inverse perspective maps or [R, 16] control points, n int32 [R] windows per region, x0 int32 [R, 8] window
    origins, wn int32 [R] window width), exactly as alm_pre_line_crops and alm_mgpstr_forward_lines use them (host)."""
    code, _, _ = _line_regions(regions, page_index, kind)
    if code == _lib.BOX_QUAD:
        p = quad_plan(sizes, regions, page_index)
        geom = p['minv'].reshape(-1, 9)
    else:
        p = curve_plan(sizes, regions, page_index)
        geom = p['ctrl'].reshape(-1, 16)
    n, x0, wn = line_windows(p['sizes'])
    return dict(sizes=p['sizes'], geom=np.ascontiguousarray(geom), n=n, x0=x0, wn=wn)


def line_crops(ctx: _lib.Context, pages: List, regions, page_index, kind: str = 'quad') -> torch.Tensor:
    """[sum of windows, 3, 32, 128] f32 in [0, 1] on the device, the MGP-STR inputs of text lines of any length: every
    window of line_plan's layout, region after region, is columns [x0, x0 + wn) of the crop quad_crops / curve_crops cut
    before resizing, then `Image.resize((128, 32), BICUBIC)` + ToTensor, bit for bit, in three kernel launches for all
    regions.  pages: uint8 [h, w, 3] each (host or CUDA); regions and kind as line_plan."""
    code, r, pi = _line_regions(regions, page_index, kind)
    R = r.shape[0]
    if R == 0:
        return torch.empty(0, 3, 32, 128, dtype=torch.float32, device=torch.device('cuda', ctx.device))
    keep, ptrs, hs, ws, n = _image_args(pages)
    plan = line_plan(list(zip(hs.tolist(), ws.tolist())), r, pi, kind)
    out = torch.empty(int(plan['n'].sum()), 3, 32, 128, dtype=torch.float32, device=torch.device('cuda', ctx.device))
    ctx.wait_torch(*keep)
    ctx.check(ctx.lib.alm_pre_line_crops(ctx.h, ptrs, hs.ctypes.data, ws.ctypes.data, n, code, r.ctypes.data,
                                         pi.ctypes.data, R, out.data_ptr()))
    ctx.synchronize()
    return out


def turned_crops(ctx: _lib.Context, pages: List, regions, page_index, turns, kind: str = 'quad',
                 lines: bool = False) -> torch.Tensor:
    """MGP-STR inputs of regions read at turns [R] (0..3): region r is ``np.rot90(crop, turns[r])`` of the crop
    quad_crops / curve_crops cut before resizing, then resized + ToTensor'ed, bit for bit -> [R, 3, 32, 128] on the
    device.  lines: the windows of line_plan laid out on each turned crop instead -> [sum of windows, 3, 32, 128]
    (the rule: include/alm_ocr.h, alm_pre_turned_crops).  regions and kind as line_plan."""
    code, r, pi = _line_regions(regions, page_index, kind)
    t = np.ascontiguousarray(np.asarray(turns, dtype=np.int32).reshape(-1))
    R = r.shape[0]
    if t.shape[0] != R:
        raise ValueError(f'{R} regions but {t.shape[0]} turns')
    keep, ptrs, hs, ws, n = _image_args(pages)
    if lines and R:
        p = line_plan(list(zip(hs.tolist(), ws.tolist())), r, pi, kind)['sizes']
        B = int(line_windows(np.where((t & 1)[:, None] == 1, p[:, ::-1], p))[0].sum())
    else:
        B = R
    out = torch.empty(B, 3, 32, 128, dtype=torch.float32, device=torch.device('cuda', ctx.device))
    if R == 0:
        return out
    ctx.wait_torch(*keep)
    ctx.check(ctx.lib.alm_pre_turned_crops(ctx.h, ptrs, hs.ctypes.data, ws.ctypes.data, n, code, r.ctypes.data,
                                           pi.ctypes.data, R, t.ctypes.data, int(lines), out.data_ptr()))
    ctx.synchronize()
    return out


def omni_tile_plan(sizes: Sequence[Tuple[int, int]], tile: int = 1200, overlap: int = 256) -> np.ndarray:
    """sizes: (h, w) per page -> int32 [n_tiles, 5] = (page, y0, x0, h, w): the overlapping tiles of every page, pages in
    order and each page's tiles row-major (the rule: include/alm_ocr.h, alm_pre_omni_tile_plan; host only)."""
    lib = _lib.load()
    rows = []
    for p, (h, w) in enumerate(sizes):
        ny, nx = C.c_int(0), C.c_int(0)
        rc = lib.alm_pre_omni_tile_plan(int(h), int(w), int(tile), int(overlap), C.byref(ny), C.byref(nx), None, None, 0)
        if rc != 0:
            raise _lib.AlmError(rc, f'alm_pre_omni_tile_plan: page {p} ({h} x {w}), tile {tile}, overlap {overlap} '
                                    '(need sides >= 1, tile >= 64, 0 <= 2 overlap <= tile)')
        cap = max(ny.value, nx.value)
        y0, x0 = np.zeros(cap, np.int32), np.zeros(cap, np.int32)
        rc = lib.alm_pre_omni_tile_plan(int(h), int(w), int(tile), int(overlap), C.byref(ny), C.byref(nx),
                                        y0.ctypes.data, x0.ctypes.data, cap)
        if rc != 0:
            raise _lib.AlmError(rc, 'alm_pre_omni_tile_plan')
        th, tw = min(int(tile), int(h)), min(int(tile), int(w))
        rows += [(p, y, x, th, tw) for y in y0[:ny.value].tolist() for x in x0[:nx.value].tolist()]
    return np.asarray(rows, dtype=np.int32).reshape(-1, 5)


def check_turns(turns, n: int) -> np.ndarray:
    """Quarter-turns of n pages as int32 [n] (ValueError for another length, a non-integer type or a turn outside
    0..3)."""
    t = np.asarray(turns)
    if t.ndim != 1 or t.shape[0] != n or (t.size and t.dtype.kind not in 'iu'):
        raise ValueError(f'turns must be {n} integers, got {t.dtype} {t.shape}')
    if t.size and not ((t >= 0) & (t <= 3)).all():
        raise ValueError(f'turns must be in 0..3, got {t.tolist()}')
    return np.ascontiguousarray(t, dtype=np.int32)


def turned_sizes(sizes: Sequence[Tuple[int, int]], turns) -> List[Tuple[int, int]]:
    """(h, w) of np.rot90(page, k) for every page's (h, w) and turn k."""
    return [(int(w), int(h)) if int(k) & 1 else (int(h), int(w)) for (h, w), k in zip(sizes, turns)]


def omni_tiles(ctx: _lib.Context, pages: List, tile: int = 1200, overlap: int = 256, test_min_size: int = 1200,
               test_max_size: int = 1920, first: int = 0, count: int = None, turns=None) -> NestedTensor:
    """Tiles first .. first + count - 1 of omni_tile_plan (all by default) cut from the pages and put through the
    reference's validation transform, each as an image of its own: equal, bit for bit, to
    ``omni_pages(ctx, [page[y0:y0+h, x0:x0+w] for each tile], test_min_size, test_max_size)``.
    pages: uint8 [h, w, 3] each (host or CUDA).  turns: None, or int [P] in 0..3: page p is read as
    ``np.rot90(page_p, turns[p])`` and the plan is omni_tile_plan of the turned sizes (rule: include/alm_ocr.h,
    alm_pre_omni_tiles_turned)."""
    keep, ptrs, hs, ws, n = _image_args(pages)
    sizes = list(zip(hs.tolist(), ws.tolist()))
    if turns is not None:
        turns = check_turns(turns, n)
        sizes = turned_sizes(sizes, turns)
    plan = omni_tile_plan(sizes, tile, overlap)
    count = len(plan) - first if count is None else count
    if first < 0 or count < 1 or first + count > len(plan):
        raise ValueError(f'tiles {first} .. {first + count - 1} outside the plan of {len(plan)} tiles')
    sel = plan[first:first + count]
    _, (Hc, Wc) = omni_plan([(int(h), int(w)) for h, w in sel[:, 3:5]], test_min_size, test_max_size)
    dev = torch.device('cuda', ctx.device)
    tensors = torch.empty(count, 3, Hc, Wc, dtype=torch.float32, device=dev)
    mask = torch.empty(count, Hc, Wc, dtype=torch.uint8, device=dev)
    ctx.wait_torch(*keep)
    if turns is None:
        ctx.check(ctx.lib.alm_pre_omni_tiles(ctx.h, ptrs, hs.ctypes.data, ws.ctypes.data, n, tile, overlap, first,
                                             count, test_min_size, test_max_size, tensors.data_ptr(), mask.data_ptr()))
    else:
        ctx.check(ctx.lib.alm_pre_omni_tiles_turned(ctx.h, ptrs, hs.ctypes.data, ws.ctypes.data, n, turns.ctypes.data,
                                                    tile, overlap, first, count, test_min_size, test_max_size,
                                                    tensors.data_ptr(), mask.data_ptr()))
    ctx.synchronize()
    return NestedTensor(tensors, mask.bool())


def omni_tiles_at(ctx: _lib.Context, pages: List, index, tile: int = 1200, overlap: int = 256,
                  test_min_size: int = 1200, test_max_size: int = 1920, turns=None) -> NestedTensor:
    """The tiles index[0], index[1], ... of omni_tile_plan(sizes, tile, overlap) (any order, repeats allowed) cut from
    the pages and put through the validation transform, each as an image of its own: what omni_tiles gives for each
    of those tiles, bit for bit (``alm_pre_omni_tiles_at``).  pages: uint8 [h, w, 3] each (host or CUDA).  turns:
    None, or int [P] in 0..3: the plan is that of the turned pages, as in omni_tiles
    (``alm_pre_omni_tiles_at_turned``)."""
    keep, ptrs, hs, ws, n = _image_args(pages)
    sizes = list(zip(hs.tolist(), ws.tolist()))
    if turns is not None:
        turns = check_turns(turns, n)
        sizes = turned_sizes(sizes, turns)
    plan = omni_tile_plan(sizes, tile, overlap)
    idx = np.ascontiguousarray(np.asarray(index).reshape(-1), dtype=np.int32)
    if idx.size == 0 or ((idx < 0) | (idx >= len(plan))).any():
        raise ValueError(f'tile indices must be a non-empty list in 0 .. {len(plan) - 1}')
    sel = plan[idx]
    _, (Hc, Wc) = omni_plan([(int(h), int(w)) for h, w in sel[:, 3:5]], test_min_size, test_max_size)
    dev = torch.device('cuda', ctx.device)
    tensors = torch.empty(len(idx), 3, Hc, Wc, dtype=torch.float32, device=dev)
    mask = torch.empty(len(idx), Hc, Wc, dtype=torch.uint8, device=dev)
    ctx.wait_torch(*keep)
    if turns is None:
        ctx.check(ctx.lib.alm_pre_omni_tiles_at(ctx.h, ptrs, hs.ctypes.data, ws.ctypes.data, n, tile, overlap,
                                                idx.ctypes.data, len(idx), test_min_size, test_max_size,
                                                tensors.data_ptr(), mask.data_ptr()))
    else:
        ctx.check(ctx.lib.alm_pre_omni_tiles_at_turned(ctx.h, ptrs, hs.ctypes.data, ws.ctypes.data, n,
                                                       turns.ctypes.data, tile, overlap, idx.ctypes.data, len(idx),
                                                       test_min_size, test_max_size, tensors.data_ptr(),
                                                       mask.data_ptr()))
    ctx.synchronize()
    return NestedTensor(tensors, mask.bool())
