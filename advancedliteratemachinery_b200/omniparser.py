"""OmniParserB200: the reference's ``OmniParser.forward`` call site served by libalm_ocr.so.

Reference boundary (relative to /root/reference/OCR/OmniParser/):
  ``output = model(samples, seqs)``                      engine/val.py:35
  OmniParser.forward                                     model/omniparser.py:19-32
  token-id layout                                        utils/parser.py:16,88-105
  checkpoint layout ``torch.load(path)['model']``        utils/checkpointer.py:20,44-47
"""
from __future__ import annotations

import ctypes as C
import math
from dataclasses import dataclass
from types import SimpleNamespace
from typing import List, Optional

import numpy as np
import torch

from . import _lib
from .nested_tensor import NestedTensor

DEFAULT_CHARS = ' !"#$%&\'()*+,-./0123456789:;<=>?@ABCDEFGHIJKLMNOPQRSTUVWXYZ[\\]^_`abcdefghijklmnopqrstuvwxyz{|}~'


# entity classes of the two KIE datasets the reference supports (model/transformer.py:49-61); class id =
# padding_index + 1 + position
CLASSES_CORD = ['menu.cnt', 'menu.discountprice', 'menu.etc', 'menu.itemsubtotal', 'menu.nm', 'menu.num', 'menu.price',
                'menu.sub.cnt', 'menu.sub.nm', 'menu.sub.price', 'menu.sub.unitprice', 'menu.unitprice', 'menu.vatyn',
                'sub_total.discount_price', 'sub_total.etc', 'sub_total.othersvc_price', 'sub_total.service_price',
                'sub_total.subtotal_price', 'sub_total.tax_price', 'total.cashprice', 'total.changeprice',
                'total.creditcardprice', 'total.emoneyprice', 'total.menuqty_cnt', 'total.menutype_cnt', 'total.total_etc',
                'total.total_price', 'void_menu.nm', 'void_menu.price']
CLASSES_SROIE = ['company', 'address', 'date', 'total']


@dataclass
class OmniVocab:
    """Same derivation as DefaultParser.parse_args (utils/parser.py:88-105)."""
    chars: str = DEFAULT_CHARS
    num_bins: int = 1000
    rec_length: int = 25
    pt_seq_length: int = 1024
    vie_categories: int = 0
    use_char_window_prompt: bool = True
    classes: Optional[List[str]] = None   # KIE entity names; default: SROIE for 4 categories, CORD for 29

    def __post_init__(self):
        if self.vie_categories and self.classes is None:
            self.classes = {4: CLASSES_SROIE, 29: CLASSES_CORD}.get(self.vie_categories)
        n_char = len(self.chars) + 1
        self.recog_pad_index = self.num_bins + n_char
        self.pt_eos_index = self.recog_pad_index + 1
        self.poly_eos_index = self.pt_eos_index + 1
        self.rec_eos_index = self.poly_eos_index + 1
        self.pt_sos_index = self.rec_eos_index + 1
        self.poly_sos_index = self.pt_sos_index + 1
        self.rec_sos_index = self.poly_sos_index + 1
        self.padding_index = self.rec_sos_index + 1
        self.num_classes = self.padding_index + 1 + self.vie_categories

    def pt_prompt(self) -> torch.Tensor:
        """engine/val.py:25-28"""
        if self.use_char_window_prompt:
            p = [0, 0, self.num_bins - 1, self.num_bins - 1, self.num_bins, self.num_bins + len(self.chars),
                 self.pt_sos_index]
        else:
            p = [0, 0, self.num_bins - 1, self.num_bins - 1, self.pt_sos_index]
        return torch.tensor([p], dtype=torch.long)

    def window_prompt(self, box=None, image_size=None, chars=None) -> torch.Tensor:
        """Spatial / character window prompt [1, 7] (dataset/collate_fn.py:46-115); [1, 5] without the character window
        (``use_char_window_prompt`` False).  No arguments: the global window, equal to ``pt_prompt()``.

        box = (x0, y0, x1, y1) in pixels of image_size = (h, w), binned like the dataset bins point centres:
        clip(floor(v / size * num_bins), 0, num_bins - 1) (dataset/text_spotting.py:78-79).  The model was trained to
        emit the centres with x0 < x <= x1 and y0 < y <= y1 in bins (collate_fn.py:80-82), so a centre in the first bin
        row / column of the box is outside it.
        chars = (first, last), two characters of ``chars``: only words whose first character lies in that class range
        are read (collate_fn.py:105-110)."""
        nb = self.num_bins
        if box is None:
            x0, y0, x1, y1 = 0, 0, nb - 1, nb - 1
        else:
            if image_size is None:
                raise ValueError('box needs image_size = (h, w)')
            h, w = (float(s) for s in image_size)
            x0, y0, x1, y1 = (min(max(int(np.floor(float(v) / size * nb)), 0), nb - 1)
                              for v, size in zip(box, (w, h, w, h)))
        p = [x0, y0, x1, y1]
        if self.use_char_window_prompt:
            lo, hi = (0, len(self.chars)) if chars is None else (self.chars.index(chars[0]), self.chars.index(chars[1]))
            p += [nb + lo, nb + hi]
        elif chars is not None:
            raise ValueError('a character window needs use_char_window_prompt')
        return torch.tensor([p + [self.pt_sos_index]], dtype=torch.long)


def page_sizes_from_mask(mask: torch.Tensor) -> List[tuple]:
    """(h, w) of every page of a NestedTensor mask [B, H, W] (True / nonzero = padding), as
    ``nested_tensor_from_tensor_list`` lays pages out: page b must be the top-left h x w rectangle of its slot and
    everything else padding.  Raises ValueError for any other valid region."""
    m = torch.as_tensor(mask).to(torch.bool).cpu()
    if m.dim() != 3:
        raise ValueError(f'mask must be [B, H, W], got {tuple(m.shape)}')
    sizes = []
    for b in range(m.shape[0]):
        valid = ~m[b]
        h = int(valid.any(dim=1).sum())
        w = int(valid.any(dim=0).sum())
        rect = torch.zeros_like(valid)
        rect[:h, :w] = True
        if h == 0 or w == 0 or not torch.equal(valid, rect):
            raise ValueError(f'page {b}: the valid region of the mask is not a top-left rectangle')
        sizes.append((h, w))
    return sizes


def _spotting_result(n, pt, poly, rec, prob):
    """One image's text-spotting output rows -> the reference's ``([pt, poly, rec], [probs])``, or None
    (transformer.py:240-241,286)."""
    n = int(n)
    if n == 0:
        return None
    return ([torch.from_numpy(pt[:n].reshape(1, -1).copy()), torch.from_numpy(poly[:n].reshape(1, -1).copy()),
             torch.from_numpy(rec[:n][None].copy())], [torch.from_numpy(prob[:n].copy())])


def slot_candidates(n_inst, ids, probs):
    """Recognition candidates [..., max_inst, rec_length, k] -> per slot (image, or [image][prompt]) the candidates of
    its n_inst decoded instances, (ids int64 [n, rec_length, k], probs f32 [n, rec_length, k]) aligned with the slot's
    ``rec[0]``, or None where nothing was decoded (the slot's result is None)."""
    n_inst = np.asarray(n_inst)
    if n_inst.ndim == 0:
        n = int(n_inst)
        return None if n == 0 else (ids[:n].copy(), probs[:n].copy())
    return [slot_candidates(n_inst[i], ids[i], probs[i]) for i in range(n_inst.shape[0])]


def slot_beams(n_inst, ids, probs, scores):
    """n-best lists (``last_rec_beams``: ids / probs [..., max_inst, W, rec_length], scores [..., max_inst, W]) -> per
    slot (image, or [image][prompt]) those of its n_inst decoded instances, (ids int64 [n, W, rec_length], probs f32
    [n, W, rec_length], scores f32 [n, W]) with hypothesis 0 = the slot's ``rec[0]``, or None where nothing was
    decoded (the slot's result is None)."""
    n_inst = np.asarray(n_inst)
    if n_inst.ndim == 0:
        n = int(n_inst)
        return None if n == 0 else (ids[:n].copy(), probs[:n].copy(), scores[:n].copy())
    return [slot_beams(n_inst[i], ids[i], probs[i], scores[i]) for i in range(n_inst.shape[0])]


def slot_locations(n_inst, loc):
    """Character locations (``last_rec_locations``: [..., max_inst, rec_length, 5]) -> per slot (image, or
    [image][prompt]) those of its n_inst decoded instances, f32 [n, rec_length, 5] aligned with the slot's ``rec[0]``,
    or None where nothing was decoded (the slot's result is None)."""
    n_inst = np.asarray(n_inst)
    if n_inst.ndim == 0:
        n = int(n_inst)
        return None if n == 0 else loc[:n].copy()
    return [slot_locations(n_inst[i], loc[i]) for i in range(n_inst.shape[0])]


def check_merge_args(margin, band, iou):
    """The merge parameters alm_omni_merge_tiles accepts (ValueError otherwise): margin, band finite and >= 0, iou in
    (0, 1]."""
    margin, band, iou = float(margin), float(band), float(iou)
    if not (math.isfinite(margin) and margin >= 0 and math.isfinite(band) and band >= 0):
        raise ValueError(f'margin and band must be finite and >= 0, got {margin}, {band}')
    if not (math.isfinite(iou) and 0 < iou <= 1):
        raise ValueError(f'iou must be in (0, 1], got {iou}')
    return margin, band, iou


def check_rec_args(k, beams, length_penalty, locations):
    """The recognition options every decode accepts (ValueError otherwise), as (k, beams, length_penalty, locations):
    rec_candidates k in 0..MAX_CANDIDATES, rec_beams in 0..MAX_BEAMS, length_penalty in [0, 2], beams with neither
    candidates nor locations."""
    k, beams, lp, locations = int(k), int(beams), float(length_penalty), bool(locations)
    if not 0 <= k <= _lib.MAX_CANDIDATES:
        raise ValueError(f'rec_candidates must be 0..{_lib.MAX_CANDIDATES}, got {k}')
    if not 0 <= beams <= _lib.MAX_BEAMS:
        raise ValueError(f'rec_beams must be 0..{_lib.MAX_BEAMS}, got {beams}')
    if not 0.0 <= lp <= 2.0:
        raise ValueError(f'length_penalty must be in [0, 2], got {lp}')
    if k and beams:
        raise ValueError('rec_candidates and rec_beams cannot be combined')
    if locations and beams:
        raise ValueError('rec_locations and rec_beams cannot be combined')
    return k, beams, lp, locations


def check_rec_charset(charset, chars: str, rows: Optional[int] = None):
    """A rec_charset argument (ValueError otherwise) as the sets ``alm_omni_set_rec_charset`` takes (rule: DESIGN 4.23):
    None for no set, else (allowed uint8 [n_sets, len(chars)], row_set int32 [rows] or None).  charset: None; a string
    of characters of `chars`, at least one, for every row (row_set None: set 0); or, where rows is given, a sequence of
    `rows` such strings or None, one per row (None: the row reads unconstrained, with the full set).  Strings naming
    the same characters share one set, in order of first appearance; a sequence of None alone is no set."""
    def one(s, where):
        if not isinstance(s, str) or not s:
            raise ValueError(f'rec_charset{where} must be a non-empty string of the vocabulary\'s characters, got {s!r}')
        bad = sorted(set(s) - set(chars))
        if bad:
            raise ValueError(f'rec_charset{where} has characters outside the vocabulary: {"".join(bad)!r}')
        return frozenset(s)
    if charset is None:
        return None
    if isinstance(charset, str) or rows is None:
        sets, row_set = [one(charset, '')], None
    else:
        items = list(charset)
        if len(items) != rows:
            raise ValueError(f'rec_charset must hold one string or None per row: {len(items)} for {rows} rows')
        if all(s is None for s in items):
            return None
        keys = [frozenset(chars) if s is None else one(s, f'[{i}]') for i, s in enumerate(items)]
        sets = list(dict.fromkeys(keys))
        index = {k: i for i, k in enumerate(sets)}
        row_set = np.array([index[k] for k in keys], dtype=np.int32)
    if len(sets) > _lib.MAX_CHARSETS:
        raise ValueError(f'rec_charset names {len(sets)} distinct sets; at most {_lib.MAX_CHARSETS}')
    allowed = np.array([[c in k for c in chars] for k in sets], dtype=np.uint8).reshape(len(sets), len(chars))
    return allowed, row_set


def _check_max_batch(max_batch) -> int:
    """The most tiles or pages a reader encodes at once, >= 1 (ValueError otherwise)."""
    if int(max_batch) < 1:
        raise ValueError(f'max_batch must be >= 1, got {max_batch}')
    return int(max_batch)


def _parse_orientation(orientation, n: int, modes, per: str):
    """A reader's orientation -> (mode, turns): one of the strings modes with turns None, or None with turns int32 [n],
    one turn per `per` (``preprocess.check_turns``).  ValueError otherwise."""
    from .preprocess import check_turns
    if isinstance(orientation, str):
        if orientation not in modes:
            raise ValueError(f"orientation must be {', '.join(repr(m) for m in modes)} or one turn per {per}, got "
                             f"{orientation!r}")
        return orientation, None
    return None, check_turns(orientation, n)


def _size_arrays(sizes):
    """The heights and widths int32 [P] of pages given as (h, w) sizes."""
    hs = np.ascontiguousarray([int(s[0]) for s in sizes], dtype=np.int32)
    ws = np.ascontiguousarray([int(s[1]) for s in sizes], dtype=np.int32)
    return hs, ws


_ROW_MERGE_OUT = ('count', 'offset', 'pts', 'polys', 'rec', 'prob', 'source')  # in the order of the C arguments


def _row_merge_out(P: int, K: int, L: int) -> dict:
    """The output buffers of a row merge (alm_omni_merge_tiles, _readings, _whole_page): count / offset int32 [P] and
    room for K >= 1 rows of rec_length L."""
    return dict(count=np.zeros(P, np.int32), offset=np.zeros(P, np.int32), pts=np.zeros((K, 2)),
                polys=np.zeros((K, 32)), rec=np.zeros((K, L), np.int64), prob=np.zeros((K, L), np.float32),
                source=np.zeros((K, 2), np.int32))


def _trim(out: dict, keys, n: int) -> dict:
    """out with the arrays under keys cut to their first n rows."""
    for k in keys:
        out[k] = out[k][:n]
    return out


def merge_tiles(ctx: _lib.Context, sizes, tile: int, overlap: int, plan, n_inst, pt, poly, rec, prob, num_bins: int,
                margin: float = 4.0, band: Optional[float] = None, iou: float = 0.5, turns=None) -> dict:
    """The instances decoded from every tile of ``preprocess.omni_tile_plan(sizes, tile, overlap)`` (``plan``, in plan
    order; n_inst / pt / poly / rec / prob in the layout of ``alm_omni_decode``, one row per tile) merged into page
    coordinates on the device (``alm_omni_merge_tiles``; rule: DESIGN 4.11).  band defaults to overlap / 4.
    turns: None, or int [P] in 0..3: page p (sizes are the upright ones) was read as ``np.rot90(page_p, turns[p])`` in
    the tiles of the turned sizes' plan; the merge runs in the turned frame and the kept points and vertices are
    mapped back to the page (``alm_omni_merge_tiles_turned``; rule: DESIGN 4.14).
    Returns dict(count int32 [P], offset int32 [P], pts f64 [K, 2], polys f64 [K, 32], rec int64 [K, L], prob f32
    [K, L], source int32 [K, 2] = (tile, instance)); page p's kept instances are rows offset[p] .. offset[p] + count[p]
    - 1, in (tile, instance) order."""
    from .preprocess import check_turns
    margin, band, iou = check_merge_args(margin, overlap / 4 if band is None else band, iou)
    if turns is not None:
        turns = check_turns(turns, len(sizes))
    hs, ws = _size_arrays(sizes)
    plan = np.asarray(plan, dtype=np.int32).reshape(-1, 5)
    tpage = np.ascontiguousarray(plan[:, 0])
    torigin = np.ascontiguousarray(plan[:, 1:3])
    n_inst = np.ascontiguousarray(n_inst, dtype=np.int32)
    pt, poly, rec = (np.ascontiguousarray(a, dtype=np.int64) for a in (pt, poly, rec))
    prob = np.ascontiguousarray(prob, dtype=np.float32)
    T, maxi, L = pt.shape[0], pt.shape[1], rec.shape[2]
    if not (len(n_inst) == T == len(plan) and poly.shape == (T, maxi, 32) and rec.shape == (T, maxi, L) and
            prob.shape == rec.shape):
        raise ValueError('merge_tiles: per-tile outputs do not match the plan')
    K = max(int(n_inst.sum()), 1)
    P = len(hs)
    out = _row_merge_out(P, K, L)
    args = (int(tile), int(overlap), T, tpage.ctypes.data, torigin.ctypes.data, n_inst.ctypes.data, pt.ctypes.data,
            poly.ctypes.data, rec.ctypes.data, prob.ctypes.data, maxi, L, int(num_bins), margin, band, iou,
            *[out[k].ctypes.data for k in _ROW_MERGE_OUT], K)
    if turns is None:
        ctx.check(ctx.lib.alm_omni_merge_tiles(ctx.h, hs.ctypes.data, ws.ctypes.data, P, *args))
    else:
        ctx.check(ctx.lib.alm_omni_merge_tiles_turned(ctx.h, hs.ctypes.data, ws.ctypes.data, P, turns.ctypes.data,
                                                      *args))
    return _trim(out, _ROW_MERGE_OUT[2:], int(out['count'].sum()))


MAX_REC_LENGTH = 1021  # alm_omni_char_boxes' bound on rec_length, as alm_omni_decode's


def char_boxes(ctx: _lib.Context, sizes, tiles, polys, rec, loc, tile_index, recog_pad_index: int, rec_eos_index: int,
               turns=None) -> dict:
    """One box per recognised character of words read in tiles, in page pixels, on the device
    (``alm_omni_char_boxes``; rule: DESIGN 4.20): ``postprocess.rec_char_boxes`` for the words of ``merge_tiles``,
    ``merge_turns`` and ``read_regions``.  sizes: the upright (h, w) of every page; tiles int [F, 5] = (page, y0, x0, h,
    w) in the layout of ``preprocess.omni_tile_plan`` (a page read whole: (page, 0, 0, h, w) of its turned size); turns:
    None, or int [P] in 0..3, page p read as ``np.rot90(page_p, turns[p])``.  Word n: polys f64 [N, 32] (its vertices
    in page pixels), rec int64 [N, L], loc f32 [N, L, 5] (the locations of the tile instance it came from,
    ``last_rec_locations``' layout) and tile_index int [N] into tiles.
    Returns dict(n_chars int32 [N], step int32 [N, L], centre f64 [N, L, 2], cov f64 [N, L, 3] = (sxx, sxy, syy), box
    f64 [N, L, 8] = four corners (x, y)): character i of word n is slot [n, i], the i-th step decode_seq keeps; slots
    past n_chars are 0.  ValueError for shapes that do not match, a tile index out of range, a turn outside 0..3, a
    non-positive size or a tile outside its turned page."""
    from .preprocess import check_turns
    P = len(sizes)
    turns = np.zeros(P, np.int32) if turns is None else check_turns(turns, P)
    tiles = np.asarray(tiles, dtype=np.int64).reshape(-1, 5)
    rec = np.ascontiguousarray(rec, dtype=np.int64)
    if rec.ndim != 2:
        raise ValueError(f'char_boxes: rec must be [N, L], got {rec.shape}')
    N, L = rec.shape
    polys = np.ascontiguousarray(polys, dtype=np.float64)
    loc = np.ascontiguousarray(loc, dtype=np.float32)
    tile_index = np.asarray(tile_index).reshape(-1)
    if polys.shape not in ((N, 32), (N, 16, 2)):
        raise ValueError(f'char_boxes: polys must be [{N}, 32], got {polys.shape}')
    if loc.shape != (N, L, 5) or len(tile_index) != N or not 1 <= L <= MAX_REC_LENGTH:
        raise ValueError(f'char_boxes: rec {rec.shape} (rec_length in 1..{MAX_REC_LENGTH}), loc {loc.shape} and '
                         f'tile_index {tile_index.shape} do not match')
    if N and (tile_index.dtype.kind not in 'iu' or tile_index.min() < 0 or tile_index.max() >= len(tiles)):
        raise ValueError(f'char_boxes: tile indices must be integers in 0 .. {len(tiles) - 1}')
    if len(tiles) and (tiles[:, 0].min() < 0 or tiles[:, 0].max() >= P):
        raise ValueError(f'char_boxes: tile pages must be in 0 .. {P - 1}')
    hw = np.array([(int(h), int(w)) for h, w in sizes], dtype=np.int64).reshape(-1, 2)
    frames = np.zeros((len(tiles), 7), np.int32)
    if len(tiles):
        p = tiles[:, 0]
        frames[:] = np.stack([hw[p, 0], hw[p, 1], turns[p], tiles[:, 1], tiles[:, 2], tiles[:, 3], tiles[:, 4]], 1)
        odd = turns[p] % 2 == 1
        th, tw = np.where(odd, hw[p, 1], hw[p, 0]), np.where(odd, hw[p, 0], hw[p, 1])
        ok = (hw[p] >= 1).all(1) & (tiles[:, 3] >= 1) & (tiles[:, 4] >= 1) & (tiles[:, 1] >= 0) & (tiles[:, 2] >= 0) & \
            (tiles[:, 1] + tiles[:, 3] <= th) & (tiles[:, 2] + tiles[:, 4] <= tw)
        if not ok.all():
            raise ValueError(f'char_boxes: tile {int(np.argmin(ok))} is empty or outside its turned page')
    out = dict(n_chars=np.zeros(N, np.int32), step=np.zeros((N, L), np.int32), centre=np.zeros((N, L, 2)),
               cov=np.zeros((N, L, 3)), box=np.zeros((N, L, 8)))
    if N == 0:
        return out
    fi = np.ascontiguousarray(tile_index, dtype=np.int32)
    ctx.check(ctx.lib.alm_omni_char_boxes(ctx.h, N, L, polys.ctypes.data, rec.ctypes.data, loc.ctypes.data,
                                          fi.ctypes.data, len(frames), frames.ctypes.data, int(recog_pad_index),
                                          int(rec_eos_index), *[out[k].ctypes.data for k in
                                                                ('n_chars', 'step', 'centre', 'cov', 'box')]))
    return out


def char_dicts(boxes: dict, rec, vocab) -> List[List[dict]]:
    """``char_boxes``' result -> per word the list ``postprocess.rec_char_boxes`` gives: dict(char, centre [2], cov
    [[sxx, sxy], [sxy, syy]], box [4, 2]) per character, in page pixels."""
    rec = np.asarray(rec)
    out = []
    for n, k in enumerate(boxes['n_chars'].tolist()):
        chars = []
        for i in range(k):
            sxx, sxy, syy = boxes['cov'][n, i]
            chars.append({'char': vocab.chars[int(rec[n, boxes['step'][n, i]]) - vocab.num_bins],
                          'centre': boxes['centre'][n, i].copy(), 'cov': np.array([[sxx, sxy], [sxy, syy]]),
                          'box': boxes['box'][n, i].reshape(4, 2).copy()})
        out.append(chars)
    return out


def orient_select(ctx: _lib.Context, n_inst, rec, prob, recog_pad_index: int, rec_eos_index: int):
    """Per page the turn its four probe readings choose, on the device (``alm_omni_orient_select``; rule: DESIGN
    4.14).  n_inst int [P, 4], rec int64 [P, 4, max_inst, L], prob f32 [..]: reading [p, k] = page p read whole at turn
    k, in the layout of ``alm_omni_decode``.  A reading scores the sum, in instance order and in double, of
    decode_pred_seq's 'score' of its instances; the larger score wins, the lower turn on a tie.
    Returns (turns int32 [P], scores f64 [P, 4])."""
    n_inst = np.ascontiguousarray(n_inst, dtype=np.int32).reshape(-1, 4)
    P = n_inst.shape[0]
    rec = np.ascontiguousarray(rec, dtype=np.int64)
    prob = np.ascontiguousarray(prob, dtype=np.float32)
    if P < 1 or rec.ndim != 4 or rec.shape[:2] != (P, 4) or prob.shape != rec.shape:
        raise ValueError(f'orient_select: {P} pages, rec {rec.shape}, prob {prob.shape}')
    turns = np.zeros(P, np.int32)
    scores = np.zeros((P, 4))
    ctx.check(ctx.lib.alm_omni_orient_select(ctx.h, P, n_inst.ctypes.data, rec.ctypes.data, prob.ctypes.data,
                                             rec.shape[2], rec.shape[3], int(recog_pad_index), int(rec_eos_index),
                                             turns.ctypes.data, scores.ctypes.data))
    return turns, scores


def merge_turns(ctx: _lib.Context, count, offset, pts, polys, rec, prob, recog_pad_index: int, rec_eos_index: int,
                iou: float = 0.5) -> dict:
    """The four turned readings of every page merged into one set of words on the device (``alm_omni_merge_turns``;
    rule: DESIGN 4.15).  Input: what ``merge_tiles(..., turns=[0, 1, 2, 3] * P)`` returns for the 4 P readings, reading
    4 p + k = page p read at turn k: count / offset int [4 P] (offset the exclusive prefix sum of count), pts f64
    [N, 2], polys f64 [N, 32], rec int64 [N, L], prob f32 [N, L], in page pixels.  Of two rows of one page at
    different turns whose boxes overlap by IoU >= iou, the one with the lower decode_pred_seq 'score' is dropped (on
    equal scores the one at the higher turn); rows of one reading never drop each other.
    Returns dict(count int32 [P], offset int32 [P], pts, polys, rec, prob, source int32 [K, 2] = (turn, index within
    that reading)); page p's kept rows are offset[p] .. offset[p] + count[p] - 1, in (turn, row) order."""
    return _merge_readings(ctx, 4, count, offset, pts, polys, rec, prob, recog_pad_index, rec_eos_index, iou,
                           'merge_turns')


def merge_readings(ctx: _lib.Context, n_readings: int, count, offset, pts, polys, rec, prob, recog_pad_index: int,
                   rec_eos_index: int, iou: float = 0.5) -> dict:
    """``merge_turns``' rule over n_readings readings per page (``alm_omni_merge_readings``): reading
    n_readings p + k = page p's reading k, source = (k, index within that reading).  The window readings of a dense
    page (``OmniParserB200.decode_dense``, DESIGN 4.16) are merged with it, reading k = window k, boxes in bins."""
    n = int(n_readings)
    if not 1 <= n <= 64:
        raise ValueError(f'n_readings must be in 1..64, got {n_readings}')
    return _merge_readings(ctx, n, count, offset, pts, polys, rec, prob, recog_pad_index, rec_eos_index, iou,
                           'merge_readings')


def merge_whole_page(ctx: _lib.Context, sizes, tile: int, overlap: int, tiles: dict, n_inst, pt, poly, rec, prob,
                     num_bins: int, margin: float = 4.0, turns=None) -> dict:
    """Words that cross tile seams recovered from a whole-page reading of every page, on the device
    (``alm_omni_merge_whole_page``; rule: DESIGN 4.17).  tiles: what ``merge_tiles(ctx, sizes, tile, overlap, ...,
    margin=margin, turns=turns)`` returned for the pages; n_inst / pt / poly / rec / prob: each page's whole-page reading
    (``np.rot90(page_p, turns[p])`` decoded as one image) in the layout of ``alm_omni_decode`` / ``decode_dense``, one
    row per page.  A whole-page instance is kept iff every tile of the page's plan cuts it (a vertex within margin of an
    interior edge); a tile row is dropped iff its point lies inside the polygon of a kept whole-page instance.
    Returns merge_tiles' dict: page p's kept tile rows in their order, then its kept whole-page instances in instance
    order (mapped to the page), source = (tile, instance) for tile rows and (-1, instance) for whole-page rows."""
    from .preprocess import check_turns
    margin = float(margin)
    if not (math.isfinite(margin) and margin >= 0):
        raise ValueError(f'margin must be finite and >= 0, got {margin}')
    if turns is not None:
        turns = check_turns(turns, len(sizes))
    hs, ws = _size_arrays(sizes)
    P = len(hs)
    t = {k: np.ascontiguousarray(tiles[k], dtype=d) for k, d in
         (('count', np.int32), ('offset', np.int32), ('pts', np.float64), ('polys', np.float64), ('rec', np.int64),
          ('prob', np.float32), ('source', np.int32))}
    n_inst = np.ascontiguousarray(n_inst, dtype=np.int32).reshape(-1)
    pt, poly, rec = (np.ascontiguousarray(a, dtype=np.int64) for a in (pt, poly, rec))
    prob = np.ascontiguousarray(prob, dtype=np.float32)
    L = t['rec'].shape[1]
    cap_in = pt.shape[1] if pt.ndim == 3 else 0
    N = t['pts'].shape[0]
    if not (cap_in >= 1 and len(t['count']) == len(t['offset']) == len(n_inst) == P and t['polys'].shape == (N, 32) and
            t['rec'].shape == (N, L) and t['prob'].shape == (N, L) and t['source'].shape == (N, 2) and
            pt.shape == (P, cap_in, 2) and poly.shape == (P, cap_in, 32) and rec.shape == (P, cap_in, L) and
            prob.shape == rec.shape):
        raise ValueError('merge_whole_page: tile rows or whole-page readings do not match the pages')
    K = max(N + int(n_inst.sum()), 1)
    out = _row_merge_out(P, K, L)
    ctx.check(ctx.lib.alm_omni_merge_whole_page(
        ctx.h, hs.ctypes.data, ws.ctypes.data, P, None if turns is None else turns.ctypes.data, int(tile),
        int(overlap), margin, int(num_bins), *[t[k].ctypes.data for k in _ROW_MERGE_OUT],
        n_inst.ctypes.data, pt.ctypes.data, poly.ctypes.data, rec.ctypes.data, prob.ctypes.data, cap_in, L,
        *[out[k].ctypes.data for k in _ROW_MERGE_OUT], K))
    return _trim(out, _ROW_MERGE_OUT[2:], int(out['count'].sum()))


def merge_kie_tiles(ctx: _lib.Context, sizes, tile: int, overlap: int, plan, n_tok, tokens, tok_prob, n_inst, inst_pos,
                    poly, num_bins: int, class_base: int, n_classes: int, margin: float = 4.0,
                    band: Optional[float] = None, iou: float = 0.5, turns=None) -> dict:
    """The KIE entities decoded from every tile of ``preprocess.omni_tile_plan`` of the pages (turned by turns unless
    None; ``plan`` in plan order) merged into page coordinates on the device (``alm_omni_merge_kie_tiles``; rule: DESIGN
    4.18).  n_tok / tokens / tok_prob / n_inst / inst_pos / poly: each tile's KIE decode in the layout of
    ``alm_omni_decode_kie``, one row per tile.  band defaults to overlap / 4.  An entity (the token walk of
    decode_vie_pt_poly_rec_seq) is dropped when its box lies within margin of an interior tile edge, when its anchor lies
    outside the tile's widened core, or when a neighbouring tile's candidate entity overlaps it by box IoU >= iou and
    lies farther from its own interior edges; an entity without words is kept only on a page that is one tile.
    Returns dict(count int32 [P], offset int32 [P], cls int32 [E], prob f32 [E], word_offset int32 [E], word_count
    int32 [E], source int32 [E, 2] = (tile, entity), rect f64 [N, 4], poly f64 [N, 32], word_source int32 [N, 2] =
    (tile, instance)): page p's kept entities are rows offset[p] .. offset[p] + count[p] - 1 in (tile, entity) order,
    entity r's words rows word_offset[r] .. + word_count[r] - 1, in pixels of the upright page."""
    from .preprocess import check_turns
    margin, band, iou = check_merge_args(margin, overlap / 4 if band is None else band, iou)
    if turns is not None:
        turns = check_turns(turns, len(sizes))
    hs, ws = _size_arrays(sizes)
    plan = np.asarray(plan, dtype=np.int32).reshape(-1, 5)
    tpage = np.ascontiguousarray(plan[:, 0])
    torigin = np.ascontiguousarray(plan[:, 1:3])
    n_tok, n_inst, inst_pos = (np.ascontiguousarray(a, dtype=np.int32) for a in (n_tok, n_inst, inst_pos))
    tokens, poly = (np.ascontiguousarray(a, dtype=np.int64) for a in (tokens, poly))
    tok_prob = np.ascontiguousarray(tok_prob, dtype=np.float32)
    T = len(plan)
    if not (n_tok.shape == (T,) and tokens.ndim == 2 and tokens.shape[0] == T and tok_prob.shape == tokens.shape and
            n_inst.shape == (T,) and inst_pos.ndim == 2 and inst_pos.shape[0] == T and
            poly.shape == inst_pos.shape + (32,)):
        raise ValueError('merge_kie_tiles: per-tile outputs do not match the plan')
    # every token could close an entity, and every instance belongs to at most one
    E, N = max(int(n_tok.clip(min=0).sum()), 1), max(int(n_inst.clip(min=0).sum()), 1)
    P = len(hs)
    out = dict(count=np.zeros(P, np.int32), offset=np.zeros(P, np.int32), cls=np.zeros(E, np.int32),
               prob=np.zeros(E, np.float32), word_offset=np.zeros(E, np.int32), word_count=np.zeros(E, np.int32),
               source=np.zeros((E, 2), np.int32), rect=np.zeros((N, 4)), poly=np.zeros((N, 32)),
               word_source=np.zeros((N, 2), np.int32))
    ctx.check(ctx.lib.alm_omni_merge_kie_tiles(
        ctx.h, hs.ctypes.data, ws.ctypes.data, P, None if turns is None else turns.ctypes.data, int(tile),
        int(overlap), T, tpage.ctypes.data, torigin.ctypes.data, n_tok.ctypes.data, tokens.ctypes.data,
        tok_prob.ctypes.data, tokens.shape[1], n_inst.ctypes.data, inst_pos.ctypes.data, poly.ctypes.data,
        inst_pos.shape[1], int(num_bins), int(class_base), int(n_classes), margin, band, iou,
        *[out[k].ctypes.data for k in ('count', 'offset', 'cls', 'prob', 'word_offset', 'word_count', 'source')], E,
        *[out[k].ctypes.data for k in ('rect', 'poly', 'word_source')], N))
    _trim(out, ('cls', 'prob', 'word_offset', 'word_count', 'source'), int(out['count'].sum()))
    return _trim(out, ('rect', 'poly', 'word_source'), int(out['word_count'].sum()))


_KIE_ENT = ('cls', 'prob', 'word_offset', 'word_count', 'source')   # merge_kie_tiles' entity and word arrays, in the
_KIE_WORD = ('rect', 'poly', 'word_source')                         # order of the C arguments


def merge_kie_whole_page(ctx: _lib.Context, sizes, tile: int, overlap: int, tiles: dict, n_tok, tokens, tok_prob,
                         n_inst, inst_pos, poly, num_bins: int, class_base: int, n_classes: int, margin: float = 4.0,
                         turns=None) -> dict:
    """KIE entities that cross tile seams recovered from a whole-page KIE reading of every page, on the device
    (``alm_omni_merge_kie_whole_page``; rule: DESIGN 4.22).  tiles: what ``merge_kie_tiles(ctx, sizes, tile, overlap,
    ..., margin=margin, turns=turns)`` returned for the pages; n_tok / tokens / tok_prob / n_inst / inst_pos / poly: each
    page's whole-page KIE reading (``np.rot90(page_p, turns[p])`` decoded as one image) in the layout of
    ``alm_omni_decode_kie``, one row per page.  A whole-page entity is kept iff it has words and every tile of the
    page's plan cuts its box (an edge within margin of an interior edge); a tile entity is dropped iff its anchor, the
    centre of its box, lies inside the box of a kept whole-page entity.
    Returns merge_kie_tiles' dict: page p's kept tile entities in their order, then its kept whole-page entities in
    entity order (words mapped to the page), source = (tile, entity) / word_source = (tile, instance) for tile entities
    and (-1, entity) / (-1, instance) for whole-page ones."""
    from .preprocess import check_turns
    margin = float(margin)
    if not (math.isfinite(margin) and margin >= 0):
        raise ValueError(f'margin must be finite and >= 0, got {margin}')
    if turns is not None:
        turns = check_turns(turns, len(sizes))
    hs, ws = _size_arrays(sizes)
    P = len(hs)
    t = {k: np.ascontiguousarray(tiles[k], dtype=d) for k, d in (
        ('count', np.int32), ('offset', np.int32), ('cls', np.int32), ('prob', np.float32), ('word_offset', np.int32),
        ('word_count', np.int32), ('source', np.int32), ('rect', np.float64), ('poly', np.float64),
        ('word_source', np.int32))}
    n_tok, n_inst, inst_pos = (np.ascontiguousarray(a, dtype=np.int32) for a in (n_tok, n_inst, inst_pos))
    tokens, poly = (np.ascontiguousarray(a, dtype=np.int64) for a in (tokens, poly))
    tok_prob = np.ascontiguousarray(tok_prob, dtype=np.float32)
    E, N = len(t['cls']), len(t['rect'])
    if not (t['count'].shape == t['offset'].shape == (P,) and all(t[k].shape[:1] == (E,) for k in _KIE_ENT) and
            t['source'].shape == (E, 2) and t['rect'].shape == (N, 4) and t['poly'].shape == (N, 32) and
            t['word_source'].shape == (N, 2) and n_tok.shape == (P,) and tokens.ndim == 2 and
            tokens.shape[0] == P and tok_prob.shape == tokens.shape and n_inst.shape == (P,) and
            inst_pos.ndim == 2 and inst_pos.shape[0] == P and poly.shape == inst_pos.shape + (32,)):
        raise ValueError('merge_kie_whole_page: tile entities or whole-page readings do not match the pages')
    # every token of a whole reading could close an entity, and every instance belongs to at most one
    EK, NK = max(E + int(n_tok.clip(min=0).sum()), 1), max(N + int(n_inst.clip(min=0).sum()), 1)
    out = dict(count=np.zeros(P, np.int32), offset=np.zeros(P, np.int32), cls=np.zeros(EK, np.int32),
               prob=np.zeros(EK, np.float32), word_offset=np.zeros(EK, np.int32), word_count=np.zeros(EK, np.int32),
               source=np.zeros((EK, 2), np.int32), rect=np.zeros((NK, 4)), poly=np.zeros((NK, 32)),
               word_source=np.zeros((NK, 2), np.int32))
    ctx.check(ctx.lib.alm_omni_merge_kie_whole_page(
        ctx.h, hs.ctypes.data, ws.ctypes.data, P, None if turns is None else turns.ctypes.data, int(tile),
        int(overlap), margin, int(num_bins), int(class_base), int(n_classes), t['count'].ctypes.data,
        t['offset'].ctypes.data, *[t[k].ctypes.data for k in _KIE_ENT + _KIE_WORD], n_tok.ctypes.data,
        tokens.ctypes.data, tok_prob.ctypes.data, tokens.shape[1], n_inst.ctypes.data, inst_pos.ctypes.data,
        poly.ctypes.data, inst_pos.shape[1], out['count'].ctypes.data, out['offset'].ctypes.data,
        *[out[k].ctypes.data for k in _KIE_ENT], EK, *[out[k].ctypes.data for k in _KIE_WORD], NK))
    _trim(out, _KIE_ENT, int(out['count'].sum()))
    return _trim(out, _KIE_WORD, int(out['word_count'].sum()))


def _tile_of(source_tile, first_tile):
    """A merged row's 'tile' within its page: -1 for a whole-page row (merge_whole_page's source -1)."""
    return -1 if source_tile < 0 else int(source_tile - first_tile)


def _merge_readings(ctx, nr, count, offset, pts, polys, rec, prob, recog_pad_index, rec_eos_index, iou, name):
    iou = float(iou)
    if not (math.isfinite(iou) and 0 < iou <= 1):
        raise ValueError(f'iou must be in (0, 1], got {iou}')
    count = np.ascontiguousarray(count, dtype=np.int32).reshape(-1)
    offset = np.ascontiguousarray(offset, dtype=np.int32).reshape(-1)
    pts = np.ascontiguousarray(pts, dtype=np.float64).reshape(-1, 2)
    polys = np.ascontiguousarray(polys, dtype=np.float64).reshape(-1, 32)
    rec = np.ascontiguousarray(rec, dtype=np.int64)
    prob = np.ascontiguousarray(prob, dtype=np.float32)
    R, N = len(count), pts.shape[0]
    if R < nr or R % nr or len(offset) != R:
        words = 'four readings' if nr == 4 else f'{nr} readings'
        raise ValueError(f'{name}: count / offset must hold {words} per page, got {R} and {len(offset)}')
    if (count < 0).any() or not np.array_equal(offset, np.cumsum(count) - count):
        raise ValueError(f'{name}: counts must be >= 0 and offsets their exclusive prefix sum')
    if int(count.sum()) != N or polys.shape[0] != N or rec.ndim != 2 or rec.shape[0] != N or rec.shape[1] < 1 or \
            prob.shape != rec.shape:
        raise ValueError(f'{name}: {int(count.sum())} rows counted, pts {pts.shape}, polys {polys.shape}, '
                         f'rec {rec.shape}, prob {prob.shape}')
    P, L, cap = R // nr, rec.shape[1], max(N, 1)
    out = _row_merge_out(P, cap, L)
    args = (count.ctypes.data, offset.ctypes.data, pts.ctypes.data, polys.ctypes.data, rec.ctypes.data,
            prob.ctypes.data, L, int(recog_pad_index), int(rec_eos_index), iou,
            *[out[k].ctypes.data for k in _ROW_MERGE_OUT], cap)
    if nr == 4 and name == 'merge_turns':
        ctx.check(ctx.lib.alm_omni_merge_turns(ctx.h, P, *args))
    else:
        ctx.check(ctx.lib.alm_omni_merge_readings(ctx.h, P, nr, *args))
    return _trim(out, _ROW_MERGE_OUT[2:], int(out['count'].sum()))


GROUP_DEFAULTS = dict(cos_tol=math.cos(math.radians(15.0)), height_ratio=0.5, max_offset=0.5, max_overlap=0.5,
                      max_gap=1.5)


def check_group_args(**params):
    """The grouping parameters alm_omni_group_lines accepts, defaults filled in (ValueError otherwise): cos_tol in
    [-1, 1], height_ratio in [0, 1], max_offset / max_overlap / max_gap finite and >= 0."""
    unknown = set(params) - set(GROUP_DEFAULTS)
    if unknown:
        raise ValueError(f'unknown grouping parameters {sorted(unknown)}')
    p = {k: float(v) for k, v in dict(GROUP_DEFAULTS, **params).items()}
    if not -1 <= p['cos_tol'] <= 1:
        raise ValueError(f'cos_tol must be in [-1, 1], got {p["cos_tol"]}')
    if not 0 <= p['height_ratio'] <= 1:
        raise ValueError(f'height_ratio must be in [0, 1], got {p["height_ratio"]}')
    for k in ('max_offset', 'max_overlap', 'max_gap'):
        if not (math.isfinite(p[k]) and p[k] >= 0):
            raise ValueError(f'{k} must be finite and >= 0, got {p[k]}')
    return p


def group_lines(ctx: _lib.Context, polys, count, offset, **params) -> dict:
    """Spotted words grouped into text lines in reading order on the device (``alm_omni_group_lines``; rule: DESIGN
    4.12).  polys f64 [N, 32] (or [N, 16, 2]), count / offset int32 [P]: page p's words are rows offset[p] ..
    offset[p] + count[p] - 1 -- what ``merge_tiles`` returns as 'polys', 'count', 'offset'.  params: cos_tol,
    height_ratio, max_offset, max_overlap, max_gap (``GROUP_DEFAULTS``).
    Returns dict(n_lines int32 [P], line_offset int32 [P], line_first int32 [K], line_words int32 [K], order int32 [N],
    line_of int32 [N], rank_of int32 [N], line_polys f64 [K, 32]): page p's lines are line_offset[p] .. + n_lines[p] - 1,
    top to bottom; line l's words, left to right, are the rows order[line_first[l] : line_first[l] + line_words[l]]."""
    p = check_group_args(**params)
    count = np.ascontiguousarray(count, dtype=np.int32).reshape(-1)
    offset = np.ascontiguousarray(offset, dtype=np.int32).reshape(-1)
    polys = np.ascontiguousarray(polys, dtype=np.float64).reshape(-1, 32)
    P, N = len(count), polys.shape[0]
    if len(offset) != P:
        raise ValueError('group_lines: count and offset differ in length')
    if P and int(count.clip(min=0).sum()) != N:
        raise ValueError(f'group_lines: {N} polygons, the pages hold {int(count.clip(min=0).sum())}')
    cap = max(N, 1)
    out = dict(n_lines=np.zeros(P, np.int32), line_offset=np.zeros(P, np.int32), line_first=np.zeros(cap, np.int32),
               line_words=np.zeros(cap, np.int32), order=np.zeros(cap, np.int32), line_of=np.zeros(cap, np.int32),
               rank_of=np.zeros(cap, np.int32), line_polys=np.zeros((cap, 32)))
    ctx.check(ctx.lib.alm_omni_group_lines(
        ctx.h, P, count.ctypes.data, offset.ctypes.data, polys.ctypes.data, p['cos_tol'], p['height_ratio'],
        p['max_offset'], p['max_overlap'], p['max_gap'], *[out[k].ctypes.data for k in (
            'n_lines', 'line_offset', 'line_first', 'line_words', 'order', 'line_of', 'rank_of', 'line_polys')], cap))
    K = int(out['n_lines'].sum())
    for k in ('line_first', 'line_words', 'line_polys'):
        out[k] = out[k][:K]
    for k in ('order', 'line_of', 'rank_of'):
        out[k] = out[k][:N]
    return out


def region_boxes(regions, kind: str) -> np.ndarray:
    """Bounding box f64 [R, 4] = (x0, y0, x1, y1) of each region of ``postprocess.region_points``' kinds ('point': the
    point itself, a box of size 0): what ``route_regions`` places in a tile."""
    from .postprocess import REGION_KINDS, polygons_array
    if kind == 'polygon':
        r = polygons_array(regions).astype(np.float64)
    else:
        r = np.asarray(regions, dtype=np.float64)
        r = r.reshape((-1,) + REGION_KINDS[kind]) if kind in REGION_KINDS else r
    if kind == 'point':
        return np.concatenate([r, r], axis=1)
    if kind == 'box':
        return np.stack([np.minimum(r[:, 0], r[:, 2]), np.minimum(r[:, 1], r[:, 3]), np.maximum(r[:, 0], r[:, 2]),
                         np.maximum(r[:, 1], r[:, 3])], axis=1)
    return np.concatenate([r.min(axis=1), r.max(axis=1)], axis=1)


def route_regions(sizes, plan, boxes, page_index) -> np.ndarray:
    """The tile each region is read in (rule: DESIGN 4.19), int64 [R]: an index into ``plan`` (``preprocess.
    omni_tile_plan(sizes, ...)``), or -1 for the whole-page reading.  A page with one tile reads every region in that
    tile, the page read whole.  On a larger page a region goes to the tile that contains its box (boxes f64 [R, 4] =
    (x0, y0, x1, y1) in page pixels, edges included) with the largest distance d from the box to that tile's interior
    edges (in the tile's frame, as ``merge_tiles`` ranks two readings), the lower tile index on a tie; -1 when no tile
    contains it."""
    plan = np.asarray(plan, dtype=np.int64).reshape(-1, 5)
    boxes = np.asarray(boxes, dtype=np.float64).reshape(-1, 4)
    page_index = np.asarray(page_index, dtype=np.int64).reshape(-1)
    route = np.full(len(boxes), -1, np.int64)
    for p in range(len(sizes)):
        rows = np.nonzero(page_index == p)[0]
        tiles = np.nonzero(plan[:, 0] == p)[0]
        if len(rows) == 0:
            continue
        if len(tiles) == 1:
            route[rows] = tiles[0]
            continue
        H, W = (int(v) for v in sizes[p])
        y0, x0, th, tw = (plan[tiles, k][None].astype(np.float64) for k in (1, 2, 3, 4))
        b = boxes[rows]
        bx0, by0 = b[:, 0:1] - x0, b[:, 1:2] - y0   # the box in each tile's frame
        bx1, by1 = b[:, 2:3] - x0, b[:, 3:4] - y0
        inside = (bx0 >= 0) & (by0 >= 0) & (bx1 <= tw) & (by1 <= th)
        d = np.full(inside.shape, np.inf)
        d = np.where(x0 > 0, np.minimum(d, bx0), d)
        d = np.where(x0 + tw < W, np.minimum(d, tw - bx1), d)
        d = np.where(y0 > 0, np.minimum(d, by0), d)
        d = np.where(y0 + th < H, np.minimum(d, th - by1), d)
        d = np.where(inside, d, -np.inf)
        best = np.argmax(d, axis=1)   # the first of equal maxima: the lower tile index
        route[rows] = np.where(inside.any(axis=1), tiles[best], -1)
    return route


def tile_to_page(origin, size, ids, num_bins: int) -> np.ndarray:
    """Bins (x, y) of a reading of the tile at origin = (y0, x0) of size = (h, w) -> page pixels f64, as
    ``alm_omni_merge_tiles`` maps them: origin + f32(f32(id / num_bins) * side), the sum in double."""
    ids = np.asarray(ids).reshape(-1, 2)
    nb = np.float32(num_bins)
    side = np.array([size[1], size[0]], dtype=np.float32)
    v = (ids.astype(np.float32) / nb) * side
    return np.array([origin[1], origin[0]], dtype=np.float64) + v.astype(np.float64)


def turn_points(points, hw, turns) -> np.ndarray:
    """Points (x, y) f64 [N, 2] in pixels of upright pages of size hw [N, 2] = (h, w) -> the same points on
    ``np.rot90(page, turns[n])``, pixel-edge coordinates: k = 1: (y, W - x), k = 2: (W - x, H - y), k = 3: (H - y, x).
    The inverse of ``tile_core::map_back`` (exactly, on integer inputs)."""
    p = np.asarray(points, dtype=np.float64).reshape(-1, 2)
    hw = np.asarray(hw, dtype=np.float64).reshape(-1, 2)
    k = np.asarray(turns).reshape(-1)
    x, y, H, W = p[:, 0], p[:, 1], hw[:, 0], hw[:, 1]
    u = np.select([k == 1, k == 2, k == 3], [y, W - x, H - y], x)
    v = np.select([k == 1, k == 2, k == 3], [W - x, H - y, x], y)
    return np.stack([u, v], axis=1)


def turn_boxes(boxes, hw, turns) -> np.ndarray:
    """Boxes (x0, y0, x1, y1) f64 [N, 4] of upright pages of size hw [N, 2] -> the boxes of their corners turned by
    ``turn_points``: what ``route_regions`` places in the tiles of the turned page."""
    b = np.asarray(boxes, dtype=np.float64).reshape(-1, 4)
    a, c = turn_points(b[:, :2], hw, turns), turn_points(b[:, 2:], hw, turns)
    return np.concatenate([np.minimum(a, c), np.maximum(a, c)], axis=1)


def region_turn_candidates(sizes, regions, page_index, kind: str) -> np.ndarray:
    """The two turns ``read_regions(orientation='auto')`` reads each region at, int32 [R, 2] (rule: DESIGN 4.21): 1 and
    3 for a tall region (2 h >= 3 w, MGP-STR's rule), else 0 and 2.  h and w: the crop size ``preprocess.quad_plan`` /
    ``curve_plan`` give a 'quad' / 'polygon' on its page, a 'box''s own size; a 'point' is never tall."""
    from . import preprocess as Pre
    pi = np.asarray(page_index).reshape(-1)
    if kind == 'point':
        tall = np.zeros(len(pi), bool)
    elif kind == 'box':
        b = region_boxes(regions, kind)
        tall = 2 * (b[:, 3] - b[:, 1]) >= 3 * (b[:, 2] - b[:, 0])
    else:
        plan = Pre.quad_plan if kind == 'quad' else Pre.curve_plan
        cs = plan(sizes, regions, pi)['sizes'].astype(np.int64)  # (width, height)
        tall = 2 * cs[:, 1] >= 3 * cs[:, 0]
    return np.stack([np.where(tall, 1, 0), np.where(tall, 3, 2)], axis=1).astype(np.int32)


def plan_region_turns(sizes, boxes, page_index, turns, tile: int = 1200, overlap: int = 256) -> dict:
    """Where ``read_regions`` reads each region at each of its candidate turns (rule: DESIGN 4.21).  sizes: the upright
    (h, w) of every page; boxes f64 [R, 4] in page pixels (``region_boxes``); turns int [R, C].  A reading is a distinct
    (page, turn) pair that holds a region, and is a page of its own: np.rot90(page, turn), tiled by
    ``preprocess.omni_tile_plan``.  Candidate (r, c) is routed by ``route_regions`` on its reading with the box's
    corners turned (``turn_boxes``).
    Returns dict(readings int32 [n, 2] = (page, turn) in (page, turn) order, reading int64 [R, C] (the candidate's
    reading), plan int32 [tiles, 5] (the readings' plan, 'page' = reading), route int64 [R, C] (an index into plan, or
    -1 for the reading read whole))."""
    from . import preprocess as Pre
    pi = np.asarray(page_index, dtype=np.int64).reshape(-1)
    t = np.asarray(turns, dtype=np.int64).reshape(len(pi), -1)
    R, C = t.shape
    uniq, inv = np.unique(pi[:, None] * 4 + t, return_inverse=True)
    readings = np.stack([uniq // 4, uniq % 4], axis=1).astype(np.int32).reshape(-1, 2)
    reading = inv.reshape(R, C).astype(np.int64)
    read = Pre.turned_sizes([sizes[p] for p in readings[:, 0]], readings[:, 1])
    plan = Pre.omni_tile_plan(read, tile, overlap)
    hw = np.asarray(sizes, dtype=np.float64).reshape(-1, 2)[np.repeat(pi, C)]
    tb = turn_boxes(np.repeat(np.asarray(boxes, dtype=np.float64).reshape(-1, 4), C, axis=0), hw, t.reshape(-1))
    route = route_regions(read, plan, tb, reading.reshape(-1)).reshape(R, C)
    return dict(readings=readings, reading=reading, plan=plan, route=route)


def select_regions(ctx: _lib.Context, frames, frame_index, pt, poly, rec, prob, num_bins: int, recog_pad_index: int,
                   rec_eos_index: int) -> dict:
    """Of every region's C (1..4) candidate readings the one kept, and its point and polygon in upright page pixels, on
    the device (``alm_omni_select_regions``; rule: DESIGN 4.21).  frames int [F, 7] = (H, W, turn, y0, x0, h, w)
    (``alm_omni_char_boxes``' frames), frame_index int [R, C]; candidate (r, c)'s ``read_at`` outputs in bins of its
    frame: pt int64 [R, C, 2], poly [R, C, 32], rec [R, C, L], prob f32 [R, C, L].  A candidate scores
    ``decode_pred_seq``'s 'score'; the larger score is kept, the lower turn on a tie, and a NaN score never ranks above
    another.
    Returns dict(kept int32 [R] (the candidate), scores f64 [R, C], pts f64 [R, 2], polys f64 [R, 32])."""
    fi = np.ascontiguousarray(frame_index, dtype=np.int32)
    frames = np.ascontiguousarray(frames, dtype=np.int32).reshape(-1, 7)
    pt, poly, rec = (np.ascontiguousarray(a, dtype=np.int64) for a in (pt, poly, rec))
    prob = np.ascontiguousarray(prob, dtype=np.float32)
    if fi.ndim != 2 or rec.ndim != 3:
        raise ValueError(f'select_regions: frame_index must be [R, C] and rec [R, C, L], got {fi.shape}, {rec.shape}')
    R, C = fi.shape
    if pt.shape != (R, C, 2) or poly.shape != (R, C, 32) or rec.shape[:2] != (R, C) or prob.shape != rec.shape:
        raise ValueError(f'select_regions: pt {pt.shape}, poly {poly.shape}, rec {rec.shape} and prob {prob.shape} '
                         f'do not match frame_index {fi.shape}')
    out = dict(kept=np.zeros(R, np.int32), scores=np.zeros((R, C)), pts=np.zeros((R, 2)), polys=np.zeros((R, 32)))
    ctx.check(ctx.lib.alm_omni_select_regions(ctx.h, R, C, fi.ctypes.data, len(frames), frames.ctypes.data,
                                              pt.ctypes.data, poly.ctypes.data, rec.ctypes.data, prob.ctypes.data,
                                              rec.shape[2], int(num_bins), int(recog_pad_index), int(rec_eos_index),
                                              *[out[k].ctypes.data for k in ('kept', 'scores', 'pts', 'polys')]))
    return out


class OmniParserB200:
    """Inference-only stand-in for the reference ``OmniParser`` module (``--tfm_pre_norm --use_fpn``)."""

    def __init__(self, state_dict, vocab: Optional[OmniVocab] = None, device: int = 0, stream: Optional[int] = None,
                 ctx: Optional[_lib.Context] = None, workspace_mb: Optional[int] = None,
                 share_from: Optional['OmniParserB200'] = None):
        """state_dict: the reference checkpoint ``torch.load(path)['model']``; or None together with
        ``share_from=other`` (another OmniParserB200 on the same GPU): this instance becomes a second execution
        context over the SAME device weights (alm_share_weights) -- one model, several batches in flight; or None
        when the weights were already put into ``ctx`` (multi-GPU start-up, dist.load_weights_broadcast).

        Device inputs: the context enqueues on its own stream; CUDA tensors handed to encode()/forward() are ordered
        after torch's current stream automatically (alm_stream_wait)."""
        self.vocab = vocab or OmniVocab()
        self.ctx = ctx or _lib.Context(device, stream)
        if workspace_mb:
            self.ctx.set_option('workspace_mb', workspace_mb)
        if share_from is not None:
            assert state_dict is None, 'pass either a state dict or share_from'
            self.ctx.share_weights(share_from.ctx)
        elif state_dict is not None:
            kind = _lib.MODEL_OMNI_KIE if self.vocab.vie_categories else _lib.MODEL_OMNI_SPOT
            self.ctx.load_state_dict(kind, state_dict)
        self.lib = self.ctx.lib
        self._rec_k = 0
        self._rec_beams = (0, 1.0)
        self._rec_loc = False
        self._rec_cs = False
        self.last_rec_candidates = None
        self.last_rec_beams = None
        self.last_rec_locations = None
        self.last_tiles = None  # spot_tiled: the plan, every tile's decode and the merge
        self.last_dense = None  # decode_dense: window per row, grid and saturated windows per page
        self.last_regions = None  # read_regions: the plan, the routing and every chunk's reading

    # nn.Module look-alikes so reference drivers keep working
    def eval(self):
        return self

    def to(self, *_a, **_k):
        return self

    def __call__(self, samples, sequence=None, rec_candidates: int = 0, rec_beams: int = 0, length_penalty: float = 1.0,
                 rec_locations: bool = False, rec_charset: Optional[str] = None):
        return self.forward(samples, sequence, rec_candidates, rec_beams, length_penalty, rec_locations, rec_charset)

    # ---------------------------------------------------------------------------------------- stages
    def encode(self, tensors: torch.Tensor, mask: Optional[torch.Tensor] = None):
        """Swin-B -> FPN -> input_proj (model/omniparser.py:20-31).  Host or CUDA tensors."""
        assert tensors.dim() == 4 and tensors.shape[1] == 3 and tensors.dtype == torch.float32
        t = tensors.contiguous()
        B, _, H, W = t.shape
        mp = None
        self._page_sizes = [(H, W)] * B   # encoded size of every page: the frame of the character locations
        if mask is not None:
            m8 = mask.to(torch.uint8).contiguous()
            if bool(m8.any()):
                self._keep_mask = m8
                mp = m8.data_ptr()
                self._page_sizes = None    # page_sizes_from_mask, when locations are asked for
        self._keep_img = t
        self.ctx.wait_torch(t, mask)  # device inputs: order the context's stream after torch's current stream
        self.ctx.check(self.lib.alm_omni_encode(self.ctx.h, t.data_ptr(), mp, B, H, W))
        self._pages, self._page_hw = B, (H, W)
        return self.memory_shape()

    def encode_pages(self, tensors: torch.Tensor, sizes):
        """Pages of different sizes, each encoded as the reference encodes it alone (``alm_omni_encode_pages``):
        tensors [B, 3, Hc, Wc] (host or CUDA), page b = tensors[b, :, :h_b, :w_b] with sizes[b] = (h_b, w_b).
        The decode methods then give every page its batch-1 result.  Returns ``page_shapes()``."""
        assert tensors.dim() == 4 and tensors.shape[1] == 3 and tensors.dtype == torch.float32
        t = tensors.contiguous()
        B, _, Hc, Wc = t.shape
        if len(sizes) != B:
            raise ValueError(f'{len(sizes)} sizes for {B} pages')
        hs, ws = _size_arrays(sizes)
        self._keep_img = t
        self.ctx.wait_torch(t)
        self.ctx.check(self.lib.alm_omni_encode_pages(self.ctx.h, t.data_ptr(), B, Hc, Wc, hs.ctypes.data,
                                                      ws.ctypes.data))
        self._pages = B
        self._page_sizes = list(zip(hs.tolist(), ws.tolist()))
        self._page_hw = (int(hs[0]), int(ws[0])) if len(set(zip(hs.tolist(), ws.tolist()))) == 1 else None
        return self.page_shapes()

    def page_shapes(self) -> List[tuple]:
        """Memory grid (mh, mw) of every page of the last encode / encode_pages."""
        B = getattr(self, '_pages', 0)
        mh = np.zeros(max(B, 1), dtype=np.int32)
        mw = np.zeros(max(B, 1), dtype=np.int32)
        self.ctx.check(self.lib.alm_omni_page_shapes(self.ctx.h, mh.ctypes.data, mw.ctypes.data))
        return [(int(mh[b]), int(mw[b])) for b in range(B)]

    def memory_shape(self):
        b, h, w = C.c_int(), C.c_int(), C.c_int()
        self.ctx.check(self.lib.alm_omni_memory_shape(self.ctx.h, C.byref(b), C.byref(h), C.byref(w)))
        return b.value, h.value, w.value

    def features(self, level: int) -> torch.Tensor:
        """LN'd Swin stage output, NCHW like ``features[level].tensors`` (backbone/joiner.py:10-18)."""
        B, mh, mw = self.memory_shape()
        H, W = self._page_hw
        hs, ws = (H + 3) // 4, (W + 3) // 4
        for _ in range(level):
            hs, ws = (hs + 1) // 2, (ws + 1) // 2
        out = torch.empty(B, hs, ws, 128 << level, dtype=torch.float32)
        self.ctx.check(self.lib.alm_omni_get_feature(self.ctx.h, level, out.data_ptr(), out.numel()))
        return out.permute(0, 3, 1, 2)

    def memory(self, which: int = 0) -> torch.Tensor:
        """which 0: memory [B,M,512] (input_proj output, flattened); 1: sine position embedding.  After encode_pages
        with pages of different sizes M is the largest page's mh * mw; page b's rows come first, then zeros."""
        shapes = self.page_shapes()
        out = torch.empty(len(shapes), max(h * w for h, w in shapes), 512, dtype=torch.float32)
        self.ctx.check(self.lib.alm_omni_get_memory(self.ctx.h, which, out.data_ptr(), out.numel()))
        return out

    def _check_checkpoint(self, reader: str, kie: bool = False):
        """ValueError unless the checkpoint is of the kind `reader` reads: KIE (kie) or text spotting."""
        if bool(self.vocab.vie_categories) != kie:
            want, got = ('KIE', 'text spotting') if kie else ('text spotting', 'KIE')
            raise ValueError(f'{reader} reads {want} checkpoints; this one is a {got} checkpoint')

    def _device_pages(self, pages):
        """Pages (host numpy / torch or CUDA torch) on the context's device, and their (h, w) sizes."""
        dev = torch.device('cuda', self.ctx.device)
        pages = [(p if isinstance(p, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(p))).to(dev) for p in pages]
        return pages, [(int(p.shape[0]), int(p.shape[1])) for p in pages]

    def _encode_chunk(self, images: NestedTensor, sizes, test_min_size: int, test_max_size: int):
        """A chunk of tiles or pages cut by ``preprocess.omni_tiles`` / ``omni_tiles_at`` (sizes: each image's (h, w)
        before the validation transform) encoded: ``encode`` when the transform gives them one size, ``encode_pages``
        otherwise."""
        from . import preprocess as Pre
        resized, _ = Pre.omni_plan(sizes, test_min_size, test_max_size)
        if len(set(resized)) == 1:
            self.encode(images.tensors)
        else:
            self.encode_pages(images.tensors, resized)

    def _cfg(self, max_instances):
        v = self.vocab
        return _lib.DecodeCfg(v.num_bins, v.pt_eos_index, v.poly_eos_index, v.rec_eos_index, v.pt_sos_index,
                              v.poly_sos_index, v.rec_sos_index, v.recog_pad_index, v.pt_seq_length, v.rec_length, 32,
                              v.vie_categories, max_instances)

    def _set_rec_candidates(self, k: int, beams: int = 0, length_penalty: float = 1.0, locations: bool = False):
        k, beams, lp, locations = check_rec_args(k, beams, length_penalty, locations)
        # the library refuses beams together with candidates or locations: whichever is being turned off goes first
        if k == 0 and self._rec_k:
            self.ctx.check(self.lib.alm_omni_set_rec_candidates(self.ctx.h, 0))
            self._rec_k = 0
        if not locations and self._rec_loc:
            self.ctx.check(self.lib.alm_omni_set_rec_locations(self.ctx.h, 0))
            self._rec_loc = False
        if (beams, lp) != self._rec_beams:
            self.ctx.check(self.lib.alm_omni_set_rec_beams(self.ctx.h, beams, lp))
            self._rec_beams = (beams, lp)
        if k != self._rec_k:
            self.ctx.check(self.lib.alm_omni_set_rec_candidates(self.ctx.h, k))
            self._rec_k = k
        if locations and not self._rec_loc:
            self.ctx.check(self.lib.alm_omni_set_rec_locations(self.ctx.h, 1))
            self._rec_loc = True
        self.last_rec_candidates = None
        self.last_rec_beams = None
        self.last_rec_locations = None

    def _set_rec_charset(self, sets=None, row_set=None):
        """The character sets of the next decode (``alm_omni_set_rec_charset``): sets = ``check_rec_charset``'s
        (allowed, rows) or None (off); row_set (``decode_at`` only) int32 [B, cap] overrides its rows.  Every decode
        method sets them, so a call without rec_charset reads unconstrained."""
        if sets is None:
            if self._rec_cs:
                self.ctx.check(self.lib.alm_omni_set_rec_charset(self.ctx.h, None, 0, 0, None, 0))
                self._rec_cs = False
            return
        allowed = np.ascontiguousarray(sets[0], dtype=np.uint8)
        rows = None if row_set is None else np.ascontiguousarray(row_set, dtype=np.int32)
        self.ctx.check(self.lib.alm_omni_set_rec_charset(self.ctx.h, allowed.ctypes.data, allowed.shape[0],
                                                         allowed.shape[1], None if rows is None else rows.ctypes.data,
                                                         0 if rows is None else rows.size))
        self._rec_cs = True

    def _take_rec_lists(self, rec: np.ndarray):
        """After a decode, the lists switched on by ``_set_rec_candidates``, None for the others:
        last_rec_candidates = (ids int64, probs f32) in the layout of `rec` + [k];
        last_rec_beams = (ids int64, probs f32, scores f32), ids / probs in the layout of `rec` with [W] inserted before
        rec_length, scores [..., max_inst, W];
        last_rec_locations f32, the layout of `rec` + [5] = (cx, cy, sxx, sxy, syy) divided by the page's encoded size
        (w, h) -- cx / w, cy / h, sxx / w^2, sxy / (w h), syy / h^2 -- the normalised frame of poly / num_bins."""
        cand = beams = loc = None
        k, W = self._rec_k, self._rec_beams[0]
        if k:
            ids = np.zeros(rec.shape + (k,), dtype=np.int64)
            probs = np.zeros(ids.shape, dtype=np.float32)
            self.ctx.check(self.lib.alm_omni_get_rec_candidates(self.ctx.h, ids.ctypes.data, probs.ctypes.data,
                                                                ids.size))
            cand = (ids, probs)
        if W:
            ids = np.zeros(rec.shape[:-1] + (W, rec.shape[-1]), dtype=np.int64)
            probs = np.zeros(ids.shape, dtype=np.float32)
            scores = np.zeros(rec.shape[:-1] + (W,), dtype=np.float32)
            self.ctx.check(self.lib.alm_omni_get_rec_beams(self.ctx.h, ids.ctypes.data, probs.ctypes.data,
                                                           scores.ctypes.data, ids.size))
            beams = (ids, probs, scores)
        if self._rec_loc:
            loc = np.zeros(rec.shape + (5,), dtype=np.float32)
            self.ctx.check(self.lib.alm_omni_get_rec_locations(self.ctx.h, loc.ctypes.data, loc.size))
            sizes = self._page_sizes if self._page_sizes is not None else page_sizes_from_mask(self._keep_mask)
            for b, (h, w) in enumerate(sizes):
                loc[b] /= np.array([w, h, w * w, w * h, h * h], dtype=np.float32)
        self.last_rec_candidates, self.last_rec_beams, self.last_rec_locations = cand, beams, loc

    def _prompt(self, pt_prompt) -> torch.Tensor:
        """The point prompt the decode entries take: pt_prompt (default ``vocab.pt_prompt()``) as host int64 [L]."""
        return (pt_prompt if pt_prompt is not None else self.vocab.pt_prompt()).reshape(-1).to(torch.long).cpu() \
            .contiguous()

    def decode(self, pt_prompt: Optional[torch.Tensor] = None, rec_candidates: int = 0, rec_beams: int = 0,
               length_penalty: float = 1.0, rec_locations: bool = False, rec_charset: Optional[str] = None):
        """Greedy pt / poly / rec decoding of every encoded image (model/transformer.py:234-286).
        Returns per-image reference-shaped outputs (None where no point was produced).
        rec_candidates = k > 0 (up to 8): also keep the k most likely characters of every recognition step as
        ``last_rec_candidates = (ids, probs)``, [B, max_inst, rec_length, k] (``slot_candidates`` slices them per
        image); candidate 0 is the returned rec / probs.
        rec_beams = W > 0 (up to 8, not together with rec_candidates): the recognition loop runs a beam search of
        width W (rule: ``alm_omni_set_rec_beams`` in include/alm_ocr.h) and keeps the n-best lists as
        ``last_rec_beams = (ids, probs, scores)``, [B, max_inst, W, rec_length] / [B, max_inst, W] (``slot_beams``
        slices them per image); hypothesis 0 is the returned rec / probs.  length_penalty: alpha of the final
        ranking by score / len^alpha, in [0, 2].
        rec_locations = True (not together with rec_beams): also keep where the last recognition decoder layer looked at
        every step (rule: ``alm_omni_set_rec_locations`` in include/alm_ocr.h) as ``last_rec_locations``,
        [B, max_inst, rec_length, 5] = centroid and covariance (cx, cy, sxx, sxy, syy) normalised by the page's
        encoded size like poly / num_bins (``slot_locations`` slices them per image, ``postprocess.rec_char_boxes``
        turns them into one box per character).
        rec_charset = a string of the vocabulary's characters (rule: DESIGN 4.23, ``alm_omni_set_rec_charset``): every
        recognition step chooses only among them, the unknown class and the two end tokens, so every returned text is
        in the set; probabilities stay those of the unconstrained softmax, so a forced word scores lower.  Candidates,
        beams and locations follow the constrained path.  The setting describes this call only."""
        n_inst, pt, poly, rec, prob = self._decode_arrays(pt_prompt, rec_candidates, rec_beams, length_penalty,
                                                          rec_locations, rec_charset)
        return [_spotting_result(n_inst[b], pt[b], poly[b], rec[b], prob[b]) for b in range(len(n_inst))]

    def _decode_arrays(self, pt_prompt=None, rec_candidates=0, rec_beams=0, length_penalty=1.0, rec_locations=False,
                       rec_charset=None):
        """alm_omni_decode's outputs for every encoded image: n_inst int32 [B], pt int64 [B, max_inst, 2], poly
        [B, max_inst, 32], rec [B, max_inst, rec_length], prob f32 [B, max_inst, rec_length]."""
        v = self.vocab
        B = len(self.page_shapes())
        prompt = self._prompt(pt_prompt)
        maxi = max(1, v.pt_seq_length // 2)
        n_inst = np.zeros(B, dtype=np.int32)
        pt = np.zeros((B, maxi, 2), dtype=np.int64)
        poly = np.zeros((B, maxi, 32), dtype=np.int64)
        rec = np.zeros((B, maxi, v.rec_length), dtype=np.int64)
        prob = np.zeros((B, maxi, v.rec_length), dtype=np.float32)
        cfg = self._cfg(maxi)
        sets = check_rec_charset(rec_charset, v.chars)
        self._set_rec_candidates(rec_candidates, rec_beams, length_penalty, rec_locations)
        self._set_rec_charset(sets)
        self.ctx.check(self.lib.alm_omni_decode(self.ctx.h, prompt.data_ptr(), prompt.numel(), C.byref(cfg),
                                                n_inst.ctypes.data, pt.ctypes.data, poly.ctypes.data, rec.ctypes.data,
                                                prob.ctypes.data))
        self._take_rec_lists(rec)
        return n_inst, pt, poly, rec, prob

    def read_at(self, points, rec_candidates: int = 0, rec_beams: int = 0, length_penalty: float = 1.0,
                rec_locations: bool = False, rec_charset=None):
        """Read the words at caller points of every encoded page: the polygon and recognition loops prompted with
        [x, y, sos] for each point (model/transformer.py:249-284) without the point loop (``alm_omni_decode_at``).
        points: per encoded page an int array [n, 2] of (x, y) bins in [0, num_bins), the frame of ``decode``'s pt
        (``postprocess.point_bins`` converts page pixels, ``postprocess.region_points`` gives a region's point).
        Each point is read as given, in order, with no dedupe; a page with more than max_instances (pt_seq_length // 2)
        points is read in several calls on the same encoded batch and the results are concatenated in point order.
        Returns per page what ``decode`` returns, ``([pt, poly, rec], [probs])`` with pt the given points, or None for
        a page without points.  decode's own points give decode's output bit for bit.  rec_candidates, rec_beams /
        length_penalty and rec_locations: as in ``decode``, the lists [B, rows, ...] with row n the page's point n.
        rec_charset: as in ``decode`` (a string for every point), or per page a sequence of one string or None per
        point (None: that point reads unconstrained); each point reads with its own set.
        KIE checkpoints are refused: their classes come from the point loop."""
        n, pt, poly, rec, prob = self._read_at_arrays(points, rec_candidates, rec_beams, length_penalty, rec_locations,
                                                      rec_charset)
        return [_spotting_result(n[b], pt[b], poly[b], rec[b], prob[b]) for b in range(len(n))]

    def _read_at_arrays(self, points, rec_candidates=0, rec_beams=0, length_penalty=1.0, rec_locations=False,
                        rec_charset=None):
        """alm_omni_decode_at's outputs at the points of every encoded page: count int32 [B], pt int64 [B, N, 2] (the
        given points), poly [B, N, 32], rec [B, N, rec_length], prob f32 [B, N, rec_length], N = max_instances times
        the number of calls."""
        v = self.vocab
        self._check_checkpoint('read_at')
        B = len(self.page_shapes())
        if len(points) != B:
            raise ValueError(f'{len(points)} point lists for {B} encoded pages')
        pts = []
        for b, p in enumerate(points):
            a = np.asarray(p)
            a = a.reshape(0, 2) if a.size == 0 else a
            if a.ndim != 2 or a.shape[1] != 2 or (a.size and a.dtype.kind not in 'iu'):
                raise ValueError(f'page {b}: points must be integer bins [n, 2], got {a.dtype} {a.shape}')
            if a.size and ((a < 0) | (a >= v.num_bins)).any():
                raise ValueError(f'page {b}: bins must be in [0, {v.num_bins})')
            pts.append(a.astype(np.int32))
        counts = np.array([len(a) for a in pts], dtype=np.int32)
        maxi = max(1, v.pt_seq_length // 2)
        calls = max(1, -(-int(counts.max(initial=0)) // maxi))
        cfg = self._cfg(maxi)
        if rec_charset is None or isinstance(rec_charset, str):
            sets, per_point = check_rec_charset(rec_charset, v.chars), None
        else:   # one string or None per point of every page: the pages' rows in page order
            if len(rec_charset) != B:
                raise ValueError(f'rec_charset: {len(rec_charset)} per-point lists for {B} encoded pages')
            for b, cs in enumerate(rec_charset):
                if isinstance(cs, str) or len(cs) != counts[b]:
                    raise ValueError(f'rec_charset[{b}] must hold one string or None per point of page {b}')
            sets = check_rec_charset([s_ for cs in rec_charset for s_ in cs], v.chars, int(counts.sum()))
            per_point = None if sets is None else np.split(sets[1], np.cumsum(counts)[:-1])
        self._set_rec_candidates(rec_candidates, rec_beams, length_penalty, rec_locations)
        outs, lists = [], []
        for k in range(calls):
            xy = np.zeros((B, maxi, 2), dtype=np.int32)
            cnt = np.zeros(B, dtype=np.int32)
            row_set = None if per_point is None else np.zeros((B, maxi), dtype=np.int32)
            for b, a in enumerate(pts):
                part = a[k * maxi:(k + 1) * maxi]
                cnt[b] = len(part)
                xy[b, :len(part)] = part
                if row_set is not None:
                    row_set[b, :len(part)] = per_point[b][k * maxi:(k + 1) * maxi]
            self._set_rec_charset(sets, row_set)
            poly = np.zeros((B, maxi, 32), dtype=np.int64)
            rec = np.zeros((B, maxi, v.rec_length), dtype=np.int64)
            prob = np.zeros((B, maxi, v.rec_length), dtype=np.float32)
            self.ctx.check(self.lib.alm_omni_decode_at(self.ctx.h, xy.ctypes.data, cnt.ctypes.data, maxi, C.byref(cfg),
                                                       poly.ctypes.data, rec.ctypes.data, prob.ctypes.data))
            self._take_rec_lists(rec)
            outs.append((xy.astype(np.int64), poly, rec, prob))
            lists.append((self.last_rec_candidates, self.last_rec_beams, self.last_rec_locations))
        if calls > 1:
            def cat(parts):
                return None if parts[0] is None else (
                    tuple(np.concatenate(a, axis=1) for a in zip(*parts)) if isinstance(parts[0], tuple)
                    else np.concatenate(parts, axis=1))
            self.last_rec_candidates, self.last_rec_beams, self.last_rec_locations = (cat(list(p)) for p in zip(*lists))
        return (counts,) + tuple(np.concatenate(a, axis=1) for a in zip(*outs))

    def decode_prompts(self, prompts: torch.Tensor, rec_candidates: int = 0, rec_beams: int = 0,
                       length_penalty: float = 1.0, rec_locations: bool = False, rec_charset: Optional[str] = None):
        """Several window prompts per encoded image in one batched decode (``alm_omni_decode_prompts``).
        prompts: [P, L] (the same P prompts for every image) or [B, P, L], P <= 16, e.g. rows of
        ``vocab.window_prompt(...)``.  Returns a list over images of lists over prompts; item [b][p] is what the
        reference's batch-1 ``model(image_b, [prompt_{b,p}, poly_sos, rec_sos, size])`` returns:
        ``([pt, poly, rec], [probs])`` or None.  rec_candidates: as in ``decode``, [B, P, max_inst, rec_length, k].
        rec_beams / length_penalty: as in ``decode``, [B, P, max_inst, W, rec_length]; a point shared by several
        prompts of a page carries its n-best list to each of their slots.  rec_locations: as in ``decode``,
        [B, P, max_inst, rec_length, 5]; a shared point carries its locations to each slot.  rec_charset: as in
        ``decode``."""
        v = self.vocab
        B = len(self.page_shapes())
        p = prompts.to(torch.long).cpu()
        if p.dim() == 2:
            p = p.unsqueeze(0).expand(B, -1, -1)
        if p.dim() != 3 or p.shape[0] != B:
            raise ValueError(f'prompts must be [P, L] or [{B}, P, L], got {tuple(prompts.shape)}')
        p = p.contiguous()
        P = p.shape[1]
        maxi = max(1, v.pt_seq_length // 2)
        n_inst = np.zeros((B, P), dtype=np.int32)
        pt = np.zeros((B, P, maxi, 2), dtype=np.int64)
        poly = np.zeros((B, P, maxi, 32), dtype=np.int64)
        rec = np.zeros((B, P, maxi, v.rec_length), dtype=np.int64)
        prob = np.zeros((B, P, maxi, v.rec_length), dtype=np.float32)
        cfg = self._cfg(maxi)
        sets = check_rec_charset(rec_charset, v.chars)
        self._set_rec_candidates(rec_candidates, rec_beams, length_penalty, rec_locations)
        self._set_rec_charset(sets)
        self.ctx.check(self.lib.alm_omni_decode_prompts(self.ctx.h, p.data_ptr(), P, p.shape[2], C.byref(cfg),
                                                        n_inst.ctypes.data, pt.ctypes.data, poly.ctypes.data,
                                                        rec.ctypes.data, prob.ctypes.data))
        self._take_rec_lists(rec)
        return [[_spotting_result(n_inst[b, k], pt[b, k], poly[b, k], rec[b, k], prob[b, k]) for k in range(P)]
                for b in range(B)]

    def decode_dense(self, pt_prompt: Optional[torch.Tensor] = None, grid='auto', iou: float = 0.5,
                     rec_charset: Optional[str] = None):
        """Text spotting of dense pages, with more words than one point sequence holds (``alm_omni_decode_dense``; rule:
        DESIGN 4.16).  grid='auto': every page is read as ``decode`` reads it; a page whose point sequence runs out of
        steps without EOS is read again in the 2 x 2 windows of the training grids, and at 3 x 3 if one of those runs
        out too.  grid=(nx, ny), nx, ny in 1..3: every page is read once in that grid's windows.  A window keeps only
        the points inside it; a word found by two windows (box IoU >= iou in bins) keeps the higher-scoring reading.
        When no page runs out, 'auto' returns exactly what ``decode`` returns.  pt_prompt: as in ``decode``; its box
        must be the whole page.  Returns ``decode``'s per-page results and sets ``last_dense`` = SimpleNamespace(
        window=[int32 [n] per page: the window of each row], grid=int32 [B, 2] (nx, ny) used, saturated=bool [B, 9]
        per window of that grid: its sequence ran out of steps, so the window may have missed words, loops=int32 [n, 4]
        the window point loops and polygon / recognition passes run beyond level 0, as (kind, first page, pages, per
        page)).  rec_charset: as in ``decode``, for every recognition pass."""
        n_inst, pt, poly, rec, prob = self._decode_dense_arrays(pt_prompt, grid, iou, rec_charset)
        return [_spotting_result(n_inst[b], pt[b], poly[b], rec[b], prob[b]) for b in range(len(n_inst))]

    def _decode_dense_arrays(self, pt_prompt=None, grid='auto', iou=0.5, rec_charset=None):
        v = self.vocab
        if v.vie_categories:
            raise ValueError('decode_dense reads text-spotting checkpoints only')
        if isinstance(grid, str):
            if grid != 'auto':
                raise ValueError(f"grid must be 'auto' or (nx, ny) with nx, ny in 1..3, got {grid!r}")
            nx = ny = 0
        else:
            nx, ny = (int(g) for g in grid)
            if not (1 <= nx <= 3 and 1 <= ny <= 3):
                raise ValueError(f"grid must be 'auto' or (nx, ny) with nx, ny in 1..3, got {grid!r}")
        iou = float(iou)
        if not (math.isfinite(iou) and 0 < iou <= 1):
            raise ValueError(f'iou must be in (0, 1], got {iou}')
        B = len(self.page_shapes())
        prompt = self._prompt(pt_prompt)
        maxi = max(1, v.pt_seq_length // 2)
        cap = maxi * (nx * ny if nx else 9)
        n_inst = np.zeros(B, dtype=np.int32)
        pt = np.zeros((B, cap, 2), dtype=np.int64)
        poly = np.zeros((B, cap, 32), dtype=np.int64)
        rec = np.zeros((B, cap, v.rec_length), dtype=np.int64)
        prob = np.zeros((B, cap, v.rec_length), dtype=np.float32)
        window = np.zeros((B, cap), dtype=np.int32)
        grids = np.zeros((B, 2), dtype=np.int32)
        sat = np.zeros((B, 9), dtype=np.uint8)
        cfg = self._cfg(maxi)
        sets = check_rec_charset(rec_charset, v.chars)
        self._set_rec_candidates(0)
        self._set_rec_charset(sets)
        self.ctx.check(self.lib.alm_omni_decode_dense(self.ctx.h, prompt.data_ptr(), prompt.numel(), C.byref(cfg), nx, ny,
                                                      iou, cap, n_inst.ctypes.data, pt.ctypes.data, poly.ctypes.data,
                                                      rec.ctypes.data, prob.ctypes.data, window.ctypes.data,
                                                      grids.ctypes.data, sat.ctypes.data))
        self.last_dense = SimpleNamespace(window=[window[b, :n_inst[b]].copy() for b in range(B)], grid=grids,
                                          saturated=sat.astype(bool), loops=self._dense_loops())
        return n_inst, pt, poly, rec, prob

    def _dense_loops(self):
        """The loops decode_dense ran beyond its level-0 decode (``alm_omni_get_dense_loops``): int32 [n, 4] = (kind,
        first page, pages, per page), kind 0 a window point loop over those pages with `per page` window prompts, kind 1
        a polygon / recognition pass with `per page` rows per page."""
        n = C.c_int32()
        self.ctx.check(self.lib.alm_omni_get_dense_loops(self.ctx.h, None, 0, C.byref(n)))
        out = np.zeros((max(n.value, 1), 4), dtype=np.int32)
        self.ctx.check(self.lib.alm_omni_get_dense_loops(self.ctx.h, out.ctypes.data, out.size, C.byref(n)))
        return out[:n.value].copy()

    def decode_points(self, pt_prompt: Optional[torch.Tensor] = None):
        """`decode_pt_seq` alone (model/transformer.py:102-141) for every encoded image: list of (tokens int64 [n],
        probs f32 [n]) -- the long single-sequence decode of structure heads (BASELINE config 5: 512 tokens)."""
        v = self.vocab
        B = len(self.page_shapes())
        prompt = self._prompt(pt_prompt)
        P = v.pt_seq_length
        n_tok = np.zeros(B, dtype=np.int32)
        toks = np.zeros((B, P), dtype=np.int64)
        prob = np.zeros((B, P), dtype=np.float32)
        cfg = self._cfg(max(1, P // 2))
        self.ctx.check(self.lib.alm_omni_decode_points(self.ctx.h, prompt.data_ptr(), prompt.numel(), C.byref(cfg),
                                                       n_tok.ctypes.data, toks.ctypes.data, prob.ctypes.data))
        return [(torch.from_numpy(toks[b, :n_tok[b]].copy()), torch.from_numpy(prob[b, :n_tok[b]].copy())) for b in range(B)]

    def decode_kie(self, image_sizes, pt_prompt: Optional[torch.Tensor] = None, rec_candidates: int = 0, rec_beams: int = 0,
                   length_penalty: float = 1.0, rec_locations: bool = False, rec_charset: Optional[str] = None):
        """KIE decoding of every encoded image (model/transformer.py:143-217): per image the reference's
        ``[(text, class_name, prob, [[x0,y0,x1,y1], ...]), ...]``.  image_sizes: (h, w) per image (seq[3]).
        rec_candidates: as in ``decode``; the candidates of pair n belong to ``last_kie_raw['rec'][b, n]``.
        rec_beams / length_penalty: as in ``decode``; the n-best list of pair n is ``last_rec_beams[...][b, n]``.
        rec_locations: as in ``decode``; the locations of pair n are ``last_rec_locations[b, n]``.
        rec_charset: as in ``decode``, for every pair's transcription (the point loop and its classes are unchanged)."""
        v = self.vocab
        n_inst, pos, poly, rec, prob, n_tok, toks, tprob = self._decode_kie_arrays(pt_prompt, rec_candidates, rec_beams,
                                                                                  length_penalty, rec_locations,
                                                                                  rec_charset)
        self.last_kie_raw = dict(n_tok=n_tok, tokens=toks, probs=tprob, n_inst=n_inst, inst_pos=pos, poly=poly, rec=rec,
                                 rec_prob=prob)
        results = []
        for b in range(len(n_tok)):
            if n_tok[b] == 0:
                results.append(None)  # transformer.py:240-241
                continue
            h, w = [float(x) for x in image_sizes[b]]
            by_pos = {int(pos[b, n]): n for n in range(int(n_inst[b]))}
            out, words, rects = [], [], []
            i = 0
            while i < n_tok[b]:
                if i in by_pos:  # an (x, y) pair: polygon extent (:163-169) + transcription (:187-203)
                    n = by_pos[i]
                    pts = poly[b, n].reshape(-1, 2)
                    rects.append([w * float(pts[:, 0].min()) / v.num_bins, h * float(pts[:, 1].min()) / v.num_bins,
                                  w * float(pts[:, 0].max()) / v.num_bins, h * float(pts[:, 1].max()) / v.num_bins])
                    words.append(self._kie_word(rec[b, n]))
                    i += 2
                elif toks[b, i] < v.num_bins:
                    i += 1
                else:  # class token closes the entity (:211-215)
                    out.append((' '.join(words), v.classes[int(toks[b, i]) - v.padding_index - 1], float(tprob[b, i]), rects))
                    words, rects = [], []
                    i += 1
            results.append(out)
        return results

    def _kie_word(self, rec_row) -> str:
        """One pair's transcription (transformer.py:187-203): up to pad / rec_eos, skipping pad - 1."""
        v = self.vocab
        chars = []
        for tok in rec_row.tolist():
            if tok == v.recog_pad_index or tok == v.rec_eos_index:
                break
            if tok == v.recog_pad_index - 1:
                continue
            chars.append(v.chars[tok - v.num_bins])
        return ''.join(chars)

    def _decode_kie_arrays(self, pt_prompt=None, rec_candidates=0, rec_beams=0, length_penalty=1.0,
                           rec_locations=False, rec_charset=None):
        """alm_omni_decode_kie's outputs for every encoded image, in _decode_arrays' order with inst_pos in place of
        pt, then the token stream: n_inst int32 [B], inst_pos int32 [B, max_inst], poly int64 [B, max_inst, 32], rec
        [B, max_inst, rec_length], prob f32 [B, max_inst, rec_length], n_tok int32 [B], tokens int64 [B,
        pt_seq_length], token probs f32 [B, pt_seq_length]."""
        v = self.vocab
        assert v.vie_categories > 0 and v.classes is not None and len(v.classes) == v.vie_categories
        B = len(self.page_shapes())
        prompt = self._prompt(pt_prompt)
        maxi, L, P = max(1, v.pt_seq_length // 2), v.rec_length, v.pt_seq_length
        n_tok = np.zeros(B, dtype=np.int32)
        toks = np.zeros((B, P), dtype=np.int64)
        tprob = np.zeros((B, P), dtype=np.float32)
        n_inst = np.zeros(B, dtype=np.int32)
        pos = np.zeros((B, maxi), dtype=np.int32)
        poly = np.zeros((B, maxi, 32), dtype=np.int64)
        rec = np.zeros((B, maxi, L), dtype=np.int64)
        prob = np.zeros((B, maxi, L), dtype=np.float32)
        cfg = self._cfg(maxi)
        sets = check_rec_charset(rec_charset, v.chars)
        self._set_rec_candidates(rec_candidates, rec_beams, length_penalty, rec_locations)
        self._set_rec_charset(sets)
        self.ctx.check(self.lib.alm_omni_decode_kie(self.ctx.h, prompt.data_ptr(), prompt.numel(), C.byref(cfg),
                                                    n_tok.ctypes.data, toks.ctypes.data, tprob.ctypes.data,
                                                    n_inst.ctypes.data, pos.ctypes.data, poly.ctypes.data, rec.ctypes.data,
                                                    prob.ctypes.data))
        self._take_rec_lists(rec)
        return n_inst, pos, poly, rec, prob, n_tok, toks, tprob

    def spot_tiled(self, pages, tile: int = 1200, overlap: int = 256, max_batch: int = 16, margin: float = 4,
                   band: Optional[float] = None, iou: float = 0.5, test_min_size: int = 1200,
                   test_max_size: int = 1920, orientation='upright', whole_page: bool = False,
                   rec_locations: bool = False, rec_candidates: int = 0, rec_beams: int = 0,
                   length_penalty: float = 1.0, rec_charset: Optional[str] = None) -> List[List[dict]]:
        """Text spotting of pages larger than the model's input, read in overlapping tiles (rule: DESIGN 4.11).
        pages: decoded uint8 RGB pages [h, w, 3] (host numpy / torch or CUDA torch).  Every page is cut into the tiles
        of ``preprocess.omni_tile_plan(sizes, tile, overlap)``; each tile goes through the reference's validation
        transform (test_min_size / test_max_size) as an image of its own and gets the reference's batch-1 result.  The
        tiles of all pages are encoded in chunks of at most max_batch (``encode`` when a chunk's tiles have one size,
        ``encode_pages`` otherwise) and decoded; one ``merge_tiles`` call over all pages then drops instances within
        `margin` pixels of an interior tile edge and, of the readings two neighbouring tiles share (bounding-box IoU >=
        iou), keeps the one farther from its tile's interior edges.  band (default overlap / 4) widens each tile's
        core, so a word whose point two tiles place on opposite sides of their seam is still kept once.
        orientation (rule: DESIGN 4.14): 'upright' reads the pages as they are.  int [P] in 0..3 reads page p as
        ``np.rot90(page_p, turns[p])`` (counter-clockwise quarter-turns): tiled, decoded and merged in the turned
        frame, every point and vertex then mapped back to the page.  'auto' first reads every page whole at each of
        the four turns (one tile no smaller than the page), scores each reading by the sum of its instances' 'score'
        and keeps the turn of the largest (the lower turn on a tie; ``orient_select``); a page that fits in one tile
        keeps that reading, a larger one is then read in tiles at the chosen turn.  'mixed' (rule: DESIGN 4.15), for
        pages whose text runs in several directions, reads every page in tiles at all four turns (4 P readings, whose
        tiles are decoded together in chunks of max_batch and merged by one ``merge_tiles`` call), then merges each
        page's four readings with ``merge_turns``: of two words found at different turns whose boxes overlap by IoU >=
        iou, the one with the higher 'score' is kept (the lower turn on a tie).
        Returns per page a list of ``decode_pred_seq`` dicts in pixels of the page as passed in ('pts', 'score',
        'polys', 'rec'), plus 'tile' (index of the tile within its (turned) page, row-major) and 'instance' (its index
        in that tile's decode), in (tile, instance) order; with an orientation given also 'turns', the page's reading
        turn ('mixed': the word's own turn, with 'tile' / 'instance' in that reading's plan, in (turn, tile,
        instance) order).  ``last_tiles`` keeps the plan, every tile's decode and the merge; with an orientation also
        'turns' [P], and for 'auto' 'page_scores' f64 [P, 4] and the probe decodes 'probe'.  For 'mixed' the plan and
        decodes are those of the 4 P readings, 'turns' is [0, 1, 2, 3] * P, 'readings' is the readings' merge and
        'turn_merge' the merge of the turns.
        whole_page (rule: DESIGN 4.17): also read every page larger than one tile whole, at its reading turn ('mixed':
        at each of the four), through the validation transform, with ``decode_dense`` (a page with more words than one
        point sequence holds is read in windows); 'auto' reuses its probe at the chosen turn.  ``merge_whole_page``
        then keeps the whole-page words that every tile cuts, words crossing a seam that no tile saw whole, and drops
        the tile words whose point lies inside one of them.  Such words come with 'tile' -1 and 'instance' their index
        in the whole-page decode, after the page's tile words; ``last_tiles`` gains 'whole' (the whole-page decode
        arrays, one row per page, or per reading for 'mixed') and 'whole_merge'.  A page that fits in one tile is not
        read again and keeps what whole_page=False gives.  Text spotting only.
        rec_locations (rule: DESIGN 4.20): every tile decode, and 'auto''s probes, also keep the character locations
        (``decode``'s rec_locations); each kept word is followed back to its tile instance ('auto': a page that fits in
        one tile, to its probe reading; 'mixed': through the turn merge to its reading's tile) and one ``char_boxes``
        call for all pages gives each word 'chars', ``postprocess.rec_char_boxes``' list (char, centre, cov, box) in
        pixels of the page as passed in.  ``last_tiles`` gains 'loc', every tile's locations.  Not together with
        whole_page: whole-page readings go through ``decode_dense``, which has no locations.
        rec_candidates / rec_beams / length_penalty (rule: DESIGN 4.11): as in ``decode``; every tile decode, and
        'auto''s probes, run with them, and each kept word is followed back to its tile instance as for rec_locations.
        ``last_rec_candidates`` (ids int64, probs f32 [N, rec_length, k]) or ``last_rec_beams`` (ids, probs [N, W,
        rec_length], scores [N, W]) hold the N returned words in result order (page by page, each page's words in
        order), as ``read_regions`` holds its regions; ``last_tiles`` gains 'candidates' or 'beams', every tile
        decode's arrays, indexed by (tile row, instance) like 'rec'.  Candidates leave every word as it is without
        them, candidate 0 being its rec ids and probabilities.  Beams change only 'rec' / 'score', to hypothesis 0:
        the point and polygon loops stay greedy and the tile merge decides on boxes and tile edges, so for 'upright'
        and explicit turns the words, points, polygons, 'tile' and 'instance' are those without beams; 'auto' and
        'mixed' choose on hypothesis 0's score.  Candidates combine with rec_locations; beams do not, and neither
        combines with whole_page (``decode_dense`` offers neither).
        rec_charset (rule: DESIGN 4.23): a string, as in ``decode``; every tile decode, 'auto''s probes and the
        whole-page readings read with it, so every returned text is in the set.  Refusals come before any device
        work."""
        from . import postprocess
        v = self.vocab
        self._check_checkpoint('spot_tiled')
        _check_max_batch(max_batch)
        if rec_locations and whole_page:
            raise ValueError('rec_locations cannot be combined with whole_page: whole-page readings have no locations')
        K, W, lp, rec_locations = check_rec_args(rec_candidates, rec_beams, length_penalty, rec_locations)
        if (K or W) and whole_page:
            raise ValueError('rec_candidates and rec_beams cannot be combined with whole_page: whole-page readings '
                             'have neither')
        check_rec_charset(rec_charset, v.chars)
        mode, turns = _parse_orientation(orientation, len(pages), ('upright', 'auto', 'mixed'), 'page')
        pages, sizes = self._device_pages(pages)
        P = len(sizes)
        margin, band, iou = check_merge_args(margin, overlap / 4 if band is None else band, iou)
        decode = self._tile_decode(K, W, lp, rec_locations, rec_charset)
        extra = {}
        if mode == 'auto':
            turns, extra = self._probe_turns(pages, sizes, tile, overlap, max_batch, test_min_size, test_max_size,
                                             decode)
        # the readings the tiles are cut from: page p at turns[p] (None: upright), or for 'mixed' reading 4 p + k, page
        # p at turn k
        rpages, rsizes, rturns = pages, sizes, turns
        if mode == 'mixed':
            rpages, rsizes = [p for p in pages for _ in range(4)], [s for s in sizes for _ in range(4)]
            rturns = np.tile(np.arange(4, dtype=np.int32), P)
        plan, arrays = self._read_tiles(rpages, rsizes, rturns, extra.get('probe'), tile, overlap, max_batch,
                                        test_min_size, test_max_size, decode)
        n_inst, pt, poly, rec, prob = arrays[:5]
        loc, lists = arrays[5:5 + rec_locations], arrays[5 + rec_locations:]
        m = merge_tiles(self.ctx, rsizes, tile, overlap, plan, n_inst, pt, poly, rec, prob, v.num_bins, margin, band,
                        iou, turns=rturns)
        out, whole = m, None
        if whole_page and any(max(s) > tile for s in sizes):
            if mode == 'auto':  # the probe at the chosen turn is the whole-page reading
                whole = tuple(a[4 * np.arange(P) + turns] for a in extra['probe'])
            else:
                whole = self._read_whole(rpages, rsizes, rturns, tile, max_batch, test_min_size, test_max_size,
                                         lambda: self._decode_dense_arrays(rec_charset=rec_charset))
            out = merge_whole_page(self.ctx, rsizes, tile, overlap, m, *whole, v.num_bins, margin, turns=rturns)
        # the words of every page, each with its reading and its (tile, instance) in the readings' plan
        if mode == 'mixed':
            words = merge_turns(self.ctx, out['count'], out['offset'], out['pts'], out['polys'], out['rec'],
                                out['prob'], v.recog_pad_index, v.rec_eos_index, iou)
            reading = 4 * np.repeat(np.arange(P), words['count']) + words['source'][:, 0]
            source = out['source'][out['offset'][reading] + words['source'][:, 1]].reshape(-1, 2)
        else:
            words, reading, source = out, np.repeat(np.arange(P), out['count']), out['source']
        texts, scores = postprocess.rec_texts(words['rec'], words['prob'], v)
        chars = self._tile_chars(rsizes, plan, rturns, words, source, loc[0]) if rec_locations else None
        first_tile = np.searchsorted(plan[:, 0], np.arange(len(rsizes)))
        results = []
        for p in range(P):
            rows = range(int(words['offset'][p]), int(words['offset'][p]) + int(words['count'][p]))
            results.append([{'pts': [[float(words['pts'][r, 0]), float(words['pts'][r, 1])]], 'score': float(scores[r]),
                             'polys': words['polys'][r].reshape(-1, 2).tolist(), 'rec': texts[r],
                             'tile': _tile_of(source[r, 0], first_tile[reading[r]]), 'instance': int(source[r, 1]),
                             **({} if rturns is None else {'turns': int(rturns[reading[r]])}),
                             **({} if chars is None else {'chars': chars[r]})}
                            for r in rows])
        self.last_tiles = dict(plan=plan, n_inst=n_inst, pt=pt, poly=poly, rec=rec, prob=prob)
        if mode == 'mixed':
            self.last_tiles.update(turns=rturns, readings=m, turn_merge=words)
        else:
            self.last_tiles.update(merged=m)
        if rec_locations:
            self.last_tiles.update(loc=loc[0])
        if whole is not None:
            self.last_tiles.update(whole=whole, whole_merge=out)
        if turns is not None:
            self.last_tiles.update(turns=turns, **extra)
        self._keep_tile_lists(lists, source)
        return results

    def read_regions(self, pages, regions, page_index, kind: str = 'quad', tile: int = 1200, overlap: int = 256,
                     max_batch: int = 16, test_min_size: int = 1200, test_max_size: int = 1920, rec_candidates: int = 0,
                     rec_beams: int = 0, length_penalty: float = 1.0, rec_locations: bool = False,
                     orientation='upright', rec_charset=None) -> List[dict]:
        """Read caller-given regions of raw pages of any size (rule: DESIGN 4.19): OmniParser as the recogniser of
        another detector's regions, each word read in place on the page and returned with its 16-point polygon.
        pages: decoded uint8 RGB pages [h, w, 3] (host numpy / torch or CUDA torch); regions of one kind, in page
        pixels: 'point' [R, 2], 'box' [R, 4] = (x0, y0, x1, y1), 'quad' [R, 4, 2] (DocXChain's corner order) or
        'polygon' [R, 16, 2] (OmniParser's polygons); page_index int [R].
        Each region is read at ``postprocess.region_points`` (the centre rule of training), which must lie on its page.
        A page that fits in one tile is read whole, as the reference reads it.  A larger page is cut into the tiles of
        ``preprocess.omni_tile_plan(sizes, tile, overlap)`` and each region is read in the tile ``route_regions``
        gives: the one containing its bounding box farthest from the tile's interior edges; a region no tile contains
        is read on its page read whole through the validation transform ('tile' -1).  Only the tiles and whole pages
        that hold a region are cut and encoded, in chunks of at most max_batch; each gets ``read_at`` at its regions'
        points (``postprocess.point_bins`` in its own pixels).
        Returns per region, in region order, {'pts', 'score', 'polys', 'rec', 'page', 'tile'}: 'pts' the point the
        decoder was prompted with and 'polys' the 16 vertices, both mapped to page pixels as ``merge_tiles`` maps a
        tile's reading; 'score' / 'rec' as ``decode_pred_seq``; 'tile' the tile's index within its page (row-major).
        ``last_regions`` keeps the plan, the routing (plan index or -1 per region), the points and every chunk's
        tiles / pages and raw arrays.  rec_candidates / rec_beams / length_penalty: as in ``decode``, with
        ``last_rec_candidates`` (ids, probs [R, rec_length, k]) and ``last_rec_beams`` (ids, probs [R, W, rec_length],
        scores [R, W]) in region order.  rec_locations (not together with rec_beams; rule: DESIGN 4.20): every chunk's
        ``read_at`` also keeps the character locations, ``last_rec_locations`` [R, rec_length, 5] in region order (each
        in its tile's or page's frame), and one ``char_boxes`` call gives each region 'chars', ``postprocess.
        rec_char_boxes``' list (char, centre, cov, box) in page pixels.
        orientation (rule: DESIGN 4.21): 'upright' reads every region as the page lies.  int [R] in 0..3 reads region r
        on ``np.rot90(page, turns[r])`` (counter-clockwise quarter-turns), in the tiles of the turned page's plan: its
        point and box are turned into that frame (``turn_points``, ``turn_boxes``) and routed there, and its reading is
        mapped back to the page.  'auto' reads every region at two turns (``region_turn_candidates``: 1 and 3 for a tall
        region, else 0 and 2) and keeps, on the device, the reading with the larger 'score', the lower turn on a tie
        (``select_regions``).  Each distinct (page, turn) reading is cut and encoded as a page of its own (only its tiles
        and whole readings that hold a region).  The dicts gain 'turns', the turn kept, with 'tile' in that reading's
        plan; candidates, beams and 'chars' follow the kept reading.  ``last_regions`` gains 'readings' ((page, turn)
        pairs), 'reading', 'route' and the readings' 'rec' / 'prob' per (region, candidate), 'turns' [R], 'frames' /
        'frame_index' (the frames of ``select_regions``), and for 'auto' 'candidates' [R, 2] and 'scores' f64 [R, 2].
        rec_charset (rule: DESIGN 4.23): a string for every region, as in ``decode``, or a sequence of R strings or None,
        one per region (None: read unconstrained), e.g. digits for an amount field and upper case and digits for a
        plate; 'auto' reads both turns of a region under its set and chooses on the constrained scores.
        Not offered: KIE checkpoints, and any merge or dedupe of overlapping regions -- each region is read as given."""
        from . import postprocess
        from . import preprocess as Pre
        v = self.vocab
        nb, L = v.num_bins, v.rec_length
        self._check_checkpoint('read_regions')
        mb = _check_max_batch(max_batch)
        sizes = [(int(p.shape[0]), int(p.shape[1])) for p in pages]
        centres = postprocess.region_points(regions, kind)
        R = len(centres)
        pi = np.asarray(page_index).reshape(-1)
        if len(pi) != R or (R and (pi.dtype.kind not in 'iu' or pi.min() < 0 or pi.max() >= len(pages))):
            raise ValueError(f'page_index must be {R} integers in 0 .. {len(pages) - 1}')
        pi = pi.astype(np.int64)
        for r in range(R):   # every point on its page (ValueError otherwise)
            postprocess.point_bins(centres[r], sizes[pi[r]], nb)
        mode, cand = _parse_orientation(orientation, R, ('upright', 'auto'), 'region')
        if mode == 'auto':
            cand = region_turn_candidates(sizes, regions, pi, kind)
        else:
            cand = (np.zeros(R, np.int32) if mode == 'upright' else cand).reshape(R, 1)
        K, W = int(rec_candidates), int(rec_beams)
        self._set_rec_candidates(K, W, length_penalty, rec_locations)   # refused before device work
        per_region = rec_charset is not None and not isinstance(rec_charset, str)
        if check_rec_charset(rec_charset, v.chars, R if per_region else None) is None:
            rec_charset, per_region = None, False
        C = cand.shape[1]
        boxes = region_boxes(regions, kind)
        if mode == 'upright':   # every page a reading at turn 0, the plan and routing of the pages as they are
            readings = np.stack([np.arange(len(sizes)), np.zeros(len(sizes), int)], axis=1).astype(np.int32)
            plan = Pre.omni_tile_plan(sizes, tile, overlap)
            route, reading = route_regions(sizes, plan, boxes, pi), pi
        else:
            rp = plan_region_turns(sizes, boxes, pi, cand, tile, overlap)
            readings, plan = rp['readings'], rp['plan']
            route, reading = rp['route'].reshape(-1), rp['reading'].reshape(-1)   # per candidate g = C r + c
        rturns = np.ascontiguousarray(readings[:, 1])
        rsizes = [sizes[p] for p in readings[:, 0]]
        tsizes = Pre.turned_sizes(rsizes, rturns)
        tpts = turn_points(np.repeat(centres, C, axis=0), np.asarray(rsizes, np.float64).reshape(-1, 2)[reading],
                           cand.reshape(-1))
        pages, _ = self._device_pages(pages)
        rpages = [pages[p] for p in readings[:, 0]]   # each page once on the device, listed once per reading
        # the readings' tiles that hold a candidate, then the readings read whole, in chunks of their own kind
        tiles = [('tile', int(t)) for t in np.unique(route[route >= 0])]
        whole = [('whole', int(q)) for q in np.unique(reading[route < 0])]
        RC = R * C
        pt, poly = np.zeros((RC, 2), np.int64), np.zeros((RC, 32), np.int64)
        rec, prob = np.zeros((RC, L), np.int64), np.zeros((RC, L), np.float32)
        cands = (np.zeros((RC, L, K), np.int64), np.zeros((RC, L, K), np.float32)) if K > 0 else None
        beams = (np.zeros((RC, W, L), np.int64), np.zeros((RC, W, L), np.float32), np.zeros((RC, W), np.float32)) \
            if W > 0 else None
        loc = np.zeros((RC, L, 5), np.float32) if rec_locations else None
        chunks = []
        T_whole = max([64] + [max(tsizes[q]) for _, q in whole])
        for chunk in [tiles[i:i + mb] for i in range(0, len(tiles), mb)] + \
                [whole[i:i + mb] for i in range(0, len(whole), mb)]:
            frames, rows = [], []   # (y0, x0, h, w) of each image in its turned page, and its candidates
            for what, i in chunk:
                if what == 'tile':
                    frames.append((int(plan[i, 1]), int(plan[i, 2]), int(plan[i, 3]), int(plan[i, 4])))
                    rows.append(np.nonzero(route == i)[0])
                else:
                    frames.append((0, 0) + tsizes[i])
                    rows.append(np.nonzero((route < 0) & (reading == i))[0])
            idx = [i for _, i in chunk]
            if chunk[0][0] == 'tile':
                nt = Pre.omni_tiles_at(self.ctx, rpages, idx, tile, overlap, test_min_size, test_max_size,
                                       turns=rturns)
            else:
                nt = Pre.omni_tiles(self.ctx, [rpages[i] for i in idx], T_whole, 0, test_min_size, test_max_size,
                                    turns=rturns[idx])
            self._encode_chunk(nt, [f[2:] for f in frames], test_min_size, test_max_size)
            local = [postprocess.point_bins(tpts[r_] - np.array([f[1], f[0]]), f[2:], nb) for f, r_ in zip(frames, rows)]
            cs = [[rec_charset[r_c // C] for r_c in r_] for r_ in rows] if per_region else rec_charset
            n, xy, pl, rc, pb = self._read_at_arrays(local, K, W, length_penalty, rec_locations, cs)
            for j, r_ in enumerate(rows):
                k = len(r_)
                pt[r_], poly[r_], rec[r_], prob[r_] = xy[j, :k], pl[j, :k], rc[j, :k], pb[j, :k]
                for mine, got in ((cands, self.last_rec_candidates), (beams, self.last_rec_beams)):
                    if mine is not None:
                        for a, b in zip(mine, got):
                            a[r_] = b[j, :k]
                if loc is not None:
                    loc[r_] = self.last_rec_locations[j, :k]
            chunks.append(dict(kind=chunk[0][0], index=np.array(idx), n=n, pt=xy, poly=pl, rec=rc, prob=pb))
        # frames: the readings' tiles, then every reading read whole; (H, W, turn) of the reading's upright page
        tl = np.concatenate([plan, [(q, 0, 0) + tsizes[q] for q in range(len(readings))]]).astype(np.int64).reshape(-1, 5)
        hw = np.asarray(rsizes, np.int64).reshape(-1, 2)[tl[:, 0]]
        frames = np.concatenate([hw, rturns[tl[:, 0], None], tl[:, 1:]], axis=1).astype(np.int32)
        fidx = np.where(route >= 0, route, len(plan) + reading).reshape(R, C)
        sel = select_regions(self.ctx, frames, fidx, pt.reshape(R, C, 2), poly.reshape(R, C, 32), rec.reshape(R, C, L),
                             prob.reshape(R, C, L), nb, v.recog_pad_index, v.rec_eos_index)
        g = np.arange(R) * C + sel['kept']   # each region's kept candidate
        texts, scores = postprocess.rec_texts(rec[g], prob[g], v)
        chars = None
        if loc is not None:
            boxes = char_boxes(self.ctx, rsizes, tl, sel['polys'], rec[g], loc[g], fidx.reshape(-1)[g],
                               v.recog_pad_index, v.rec_eos_index, turns=rturns)
            chars = char_dicts(boxes, rec[g], v)
        turns = cand.reshape(-1)[g].astype(np.int32)
        first_tile = np.searchsorted(plan[:, 0], np.arange(len(readings)))
        self.last_rec_candidates = None if cands is None else tuple(a[g] for a in cands)
        self.last_rec_beams = None if beams is None else tuple(a[g] for a in beams)
        self.last_rec_locations = None if loc is None else loc[g]
        if mode == 'upright':   # the pages' own plan and routing
            self.last_regions = dict(plan=plan, route=route, points=centres, chunks=chunks)
        else:
            self.last_regions = dict(plan=plan, route=rp['route'], points=centres, chunks=chunks, readings=readings,
                                     reading=rp['reading'], turns=turns, frames=frames, frame_index=fidx,
                                     rec=rec.reshape(R, C, L), prob=prob.reshape(R, C, L))
        if mode == 'auto':
            self.last_regions.update(candidates=cand, scores=sel['scores'])
        return [{'pts': [sel['pts'][r].tolist()], 'score': float(scores[r]),
                 'polys': sel['polys'][r].reshape(16, 2).tolist(), 'rec': texts[r], 'page': int(pi[r]),
                 'tile': int(route[g[r]] - first_tile[reading[g[r]]]) if route[g[r]] >= 0 else -1,
                 **({} if mode == 'upright' else {'turns': int(turns[r])}),
                 **({} if chars is None else {'chars': chars[r]})} for r in range(R)]

    def kie_tiled(self, pages, tile: int = 1200, overlap: int = 256, max_batch: int = 16, margin: float = 4,
                  band: Optional[float] = None, iou: float = 0.5, test_min_size: int = 1200, test_max_size: int = 1920,
                  orientation='upright', rec_candidates: int = 0, rec_beams: int = 0,
                  rec_locations: bool = False, whole_page: bool = False, rec_charset: Optional[str] = None) -> List[list]:
        """KIE of pages larger than the model's input or turned by quarter-turns, read in overlapping tiles (rule:
        DESIGN 4.18).  pages: decoded uint8 RGB pages [h, w, 3] (host numpy / torch or CUDA torch); the checkpoint must
        be a KIE checkpoint.  Every page is cut into the tiles of ``preprocess.omni_tile_plan(sizes, tile, overlap)``;
        each tile goes through the validation transform (test_min_size / test_max_size) as an image of its own and gets
        the reference's batch-1 KIE decode with the tile's size as orig_size.  Tiles are encoded in chunks of at most
        max_batch.  One ``merge_kie_tiles`` call over all pages then drops entities within `margin` pixels of an
        interior tile edge and, of the readings two neighbouring tiles share (entity box IoU >= iou, whatever their
        classes), keeps the one farther from its tile's interior edges; band (default overlap / 4) widens each tile's
        core for the entity's anchor, the centre of its box.
        orientation: 'upright', or int [P] in 0..3 (page p read as ``np.rot90(page_p, turns[p])``, merged in the
        turned frame and mapped back), or 'auto' (every page read whole at the four turns, ``orient_select`` on the KIE
        readings' (x, y)-pair rows; a page that fits in one tile keeps that reading, a larger one is then read in tiles
        at the chosen turn), as in ``spot_tiled``.
        Returns per page the reference's entity tuples ``(text, class_name, prob, [[x0, y0, x1, y1], ...])`` in pixels
        of the page as passed in, in (tile, entity) order ([] for a page without entities); a page that fits in one
        tile gets ``decode_kie``'s list.  ``last_tiles`` keeps the plan, every tile's decode (n_tok, tokens, probs,
        n_inst, inst_pos, poly, rec, rec_prob) and the merge ('merged': each entity's (tile, entity) source, each word's
        (tile, instance) source, rect and 16-vertex polygon in page pixels, ``decode_pred_seq``'s arithmetic, the input
        of ``group_lines``, ``preprocess.curve_crops`` and ``recognize_polygons``); with an orientation also 'turns',
        and for 'auto' 'page_scores' and the probe decodes 'probe'.
        whole_page (rule: DESIGN 4.22): also read every page larger than one tile whole, at its reading turn, through
        the validation transform, with the KIE decode ('auto' reuses its probe at the chosen turn, with no extra
        decode).  ``merge_kie_whole_page`` then keeps the whole-page entities whose box every tile cuts, entities
        crossing a seam that no tile saw whole, and drops the tile entities whose anchor lies inside one of their
        boxes.  They follow the page's tile entities; ``last_tiles`` gains 'whole' (the whole-page decode arrays, one
        row per page) and 'whole_merge' (its merge; 'merged' stays the tile merge).  A page that fits in one tile is not
        read again and keeps what whole_page=False gives.
        rec_locations (rule: DESIGN 4.20): every tile decode, 'auto''s probes and the whole-page readings also keep
        the character locations; each entity word is followed back to its tile instance or whole-page instance, and one
        ``char_boxes`` call for all pages gives every word ``postprocess.rec_char_boxes``' list (char, centre, cov, box)
        in pixels of the page as passed in.  Each entity tuple then gains a fifth element, that list per word in
        ``rects`` order.  ``last_tiles`` gains 'loc', every tile's locations.  Recognition candidates and beams are not
        offered here.  rec_charset (rule: DESIGN 4.23): a string, as in ``decode_kie``, for every tile decode, probe
        and whole-page reading."""
        v = self.vocab
        self._check_checkpoint('kie_tiled', kie=True)
        if rec_candidates or rec_beams:
            raise ValueError('kie_tiled offers no recognition candidates or beams')
        check_rec_charset(rec_charset, v.chars)
        rec_locations = bool(rec_locations)
        _check_max_batch(max_batch)
        mode, turns = _parse_orientation(orientation, len(pages), ('upright', 'auto'), 'page')
        pages, sizes = self._device_pages(pages)
        P = len(sizes)
        margin, band, iou = check_merge_args(margin, overlap / 4 if band is None else band, iou)
        decode = self._kie_tile_decode(rec_locations, rec_charset)
        extra = {}
        if mode == 'auto':
            turns, extra = self._probe_turns(pages, sizes, tile, overlap, max_batch, test_min_size, test_max_size,
                                             decode)
        plan, arrays = self._read_tiles(pages, sizes, turns, extra.get('probe'), tile, overlap, max_batch,
                                        test_min_size, test_max_size, decode)
        n_inst, pos, poly, rec, prob, n_tok, toks, tprob = arrays[:8]
        m = merge_kie_tiles(self.ctx, sizes, tile, overlap, plan, n_tok, toks, tprob, n_inst, pos, poly, v.num_bins,
                            v.padding_index + 1, v.vie_categories, margin, band, iou, turns=turns)
        out, whole = m, None
        if whole_page and any(max(s) > tile for s in sizes):
            if mode == 'auto':  # the probe at the chosen turn is the whole-page reading
                whole = tuple(a[4 * np.arange(P) + turns] for a in extra['probe'])
            else:
                whole = self._read_whole(pages, sizes, turns, tile, max_batch, test_min_size, test_max_size, decode)
            wn_inst, wpos, wpoly, _, _, wn_tok, wtoks, wtprob = whole[:8]
            out = merge_kie_whole_page(self.ctx, sizes, tile, overlap, m, wn_tok, wtoks, wtprob, wn_inst, wpos, wpoly,
                                       v.num_bins, v.padding_index + 1, v.vie_categories, margin, turns=turns)
        # every entity word's rec row and, with locations, its locations and frame: tile words in the plan's tiles,
        # whole-page words (word_source tile -1) in their page read whole, frame len(plan) + page
        page_of = np.repeat(np.arange(P), out['count'])
        word_page = np.repeat(page_of, out['word_count']).astype(np.int64)
        src = out['word_source'].astype(np.int64).reshape(-1, 2)
        tw = src[:, 0] >= 0
        L = rec.shape[-1]
        wrec = np.zeros((len(src), L), np.int64)
        wrec[tw] = rec[src[tw, 0], src[tw, 1]]
        if whole is not None:
            wrec[~tw] = whole[3][word_page[~tw], src[~tw, 1]]
        chars = None
        if rec_locations:
            from . import preprocess as Pre
            wloc = np.zeros((len(src), L, 5), np.float32)
            wloc[tw] = arrays[8][src[tw, 0], src[tw, 1]]
            if whole is not None:
                wloc[~tw] = whole[8][word_page[~tw], src[~tw, 1]]
            read = sizes if turns is None else Pre.turned_sizes(sizes, turns)
            frames = np.concatenate([plan, [(p, 0, 0) + tuple(read[p]) for p in range(P)]]).astype(np.int64)
            boxes = char_boxes(self.ctx, sizes, frames, out['poly'], wrec, wloc,
                               np.where(tw, src[:, 0], len(plan) + word_page), v.recog_pad_index, v.rec_eos_index,
                               turns=turns)
            chars = char_dicts(boxes, wrec, v)
        results = []
        for p in range(P):
            ents = []
            for r in range(int(out['offset'][p]), int(out['offset'][p]) + int(out['count'][p])):
                ws = range(int(out['word_offset'][r]), int(out['word_offset'][r]) + int(out['word_count'][r]))
                text = ' '.join(self._kie_word(wrec[w]) for w in ws)
                ent = (text, v.classes[int(out['cls'][r])], float(out['prob'][r]), out['rect'][ws].tolist())
                ents.append(ent if chars is None else ent + ([chars[w] for w in ws],))
            results.append(ents)
        self.last_tiles = dict(plan=plan, n_tok=n_tok, tokens=toks, probs=tprob, n_inst=n_inst, inst_pos=pos, poly=poly,
                               rec=rec, rec_prob=prob, merged=m)
        if rec_locations:
            self.last_tiles.update(loc=arrays[8])
        if whole is not None:
            self.last_tiles.update(whole=whole, whole_merge=out)
        if turns is not None:
            self.last_tiles.update(turns=turns, **extra)
        return results

    def _read_tiles(self, pages, sizes, turns, probe, tile, overlap, max_batch, test_min_size, test_max_size, decode):
        """The plan of the pages read at turns (None: upright) and decode's arrays for every tile of it, one row per
        tile.  probe: None, or 'auto''s probe readings (reading 4 p + k, ``_probe_turns``): a page that fits in one tile
        then keeps its probe reading at its turn instead of being read again."""
        from . import preprocess as Pre
        read = sizes if turns is None else Pre.turned_sizes(sizes, turns)
        plan = Pre.omni_tile_plan(read, tile, overlap)
        if probe is None:
            return plan, self._decode_tiles(pages, plan, tile, overlap, turns, max_batch, test_min_size, test_max_size,
                                            decode)
        n_tiles = np.bincount(plan[:, 0], minlength=len(sizes))
        big = [p for p in range(len(sizes)) if max(sizes[p]) > tile]
        if big:
            sub_plan = Pre.omni_tile_plan([read[p] for p in big], tile, overlap)
            sub = self._decode_tiles([pages[p] for p in big], sub_plan, tile, overlap, turns[big], max_batch,
                                     test_min_size, test_max_size, decode)
        parts, j = [], 0
        for p in range(len(sizes)):
            if p in big:
                parts.append(tuple(a[j:j + n_tiles[p]] for a in sub))
                j += n_tiles[p]
            else:  # the page is one tile: its probe reading at the chosen turn is the tiled reading
                r = 4 * p + int(turns[p])
                parts.append(tuple(a[r:r + 1] for a in probe))
        return plan, tuple(np.concatenate(a) for a in zip(*parts))

    def _decode_tiles(self, pages, plan, tile, overlap, turns, max_batch, test_min_size, test_max_size, decode):
        """Every tile of ``plan`` (the pages' plan, turned by turns unless None) encoded in chunks of at most max_batch
        and decoded by decode (``_decode_arrays``, ``_decode_dense_arrays`` or ``_decode_kie_arrays``): its arrays, one
        row per tile."""
        from . import preprocess as Pre
        outs = []
        for first in range(0, len(plan), int(max_batch)):
            count = min(int(max_batch), len(plan) - first)
            nt = Pre.omni_tiles(self.ctx, pages, tile, overlap, test_min_size, test_max_size, first, count, turns=turns)
            self._encode_chunk(nt, [(int(h), int(w)) for h, w in plan[first:first + count, 3:5]], test_min_size,
                               test_max_size)
            outs.append(decode())
        return tuple(np.concatenate(a) for a in zip(*outs))

    def _read_whole(self, pages, sizes, turns, tile, max_batch, test_min_size, test_max_size, decode):
        """Every page larger than one tile read whole at its turn (turns None: upright) as ``_probe_turns`` reads it
        (one tile no smaller than the page, overlap 0, chunks of max_batch), decoded by decode (spot_tiled:
        ``_decode_dense_arrays``, grid 'auto'; kie_tiled: its tile decode) -> decode's arrays, one row per page (zeros,
        so no instance or token, on the other pages)."""
        from . import preprocess as Pre
        P = len(pages)
        big = [p for p in range(P) if max(sizes[p]) > tile]
        tb = None if turns is None else np.ascontiguousarray(np.asarray(turns)[big], np.int32)
        sb = [sizes[p] for p in big]
        T = max(64, max(max(s) for s in sb))
        plan = Pre.omni_tile_plan(sb if tb is None else Pre.turned_sizes(sb, tb), T, 0)
        sub = self._decode_tiles([pages[p] for p in big], plan, T, 0, tb, max_batch, test_min_size, test_max_size,
                                 decode)
        out = tuple(np.zeros((P,) + a.shape[1:], a.dtype) for a in sub)
        for a, b in zip(out, sub):
            a[big] = b
        return out

    def _tile_decode(self, rec_candidates=0, rec_beams=0, length_penalty=1.0, rec_locations=False, rec_charset=None):
        """The decode of spot_tiled's tiles and probes: a function giving ``_decode_arrays``' five arrays, then with
        rec_locations the locations f32 [B, max_inst, rec_length, 5], then with rec_candidates the candidates (ids,
        probs) or with rec_beams the n-best lists (ids, probs, scores), in ``decode``'s layouts; every decode reads
        with rec_charset."""
        def decode():
            out = self._decode_arrays(None, rec_candidates, rec_beams, length_penalty, rec_locations, rec_charset)
            if rec_locations:
                out += (self.last_rec_locations,)
            return out + (self.last_rec_candidates or self.last_rec_beams or ())
        return decode

    def _kie_tile_decode(self, rec_locations=False, rec_charset=None):
        """The decode of kie_tiled's tiles, probes and whole readings: a function giving ``_decode_kie_arrays``' eight
        arrays, then with rec_locations the locations f32 [B, max_inst, rec_length, 5] (``decode_kie``'s layout); every
        decode reads with rec_charset."""
        def decode():
            out = self._decode_kie_arrays(None, 0, 0, 1.0, rec_locations, rec_charset)
            return out + ((self.last_rec_locations,) if rec_locations else ())
        return decode

    def _keep_tile_lists(self, lists, source):
        """After spot_tiled: lists, every tile decode's candidates (ids, probs) or n-best lists (ids, probs, scores),
        one row per tile (empty when neither was asked for), go to last_tiles['candidates'] / ['beams'], and each
        merged row's, followed back to its (tile, instance) = source [N, 2], to last_rec_candidates / last_rec_beams in
        row order; the other is None."""
        s = np.asarray(source, dtype=np.int64).reshape(-1, 2)
        rows = tuple(a[s[:, 0], s[:, 1]] for a in lists) if lists else None
        beams = len(lists) == 3
        self.last_rec_candidates = None if beams else rows
        self.last_rec_beams = rows if beams else None
        if lists:
            self.last_tiles['beams' if beams else 'candidates'] = lists

    def _tile_chars(self, sizes, plan, turns, rows, source, loc) -> List[List[dict]]:
        """'chars' of merged rows (rows: a merge's dict, 'polys' and 'rec' in page pixels; source int [K, 2]: each row's
        (tile, instance) in plan) from the tiles' locations loc [tiles, max_inst, L, 5]: one ``char_boxes`` call."""
        v = self.vocab
        source = np.asarray(source, dtype=np.int64).reshape(-1, 2)
        boxes = char_boxes(self.ctx, sizes, plan, rows['polys'], rows['rec'], loc[source[:, 0], source[:, 1]],
                           source[:, 0], v.recog_pad_index, v.rec_eos_index, turns=turns)
        return char_dicts(boxes, rows['rec'], v)

    def _probe_turns(self, pages, sizes, tile, overlap, max_batch, test_min_size, test_max_size, decode):
        """'auto''s probes: every page read whole at turns 0..3 (reading 4 p + k; one tile no smaller than any page) by
        decode and the choice of orient_select on the readings' instance rows (the first five arrays: n_inst, _, _, rec,
        prob) -> (turns int32 [P], dict(page_scores=f64 [P, 4], probe=the probe decode arrays)).  A tile layout the
        pages cannot be read in (tile, overlap) is refused before the probes run."""
        from . import preprocess as Pre
        Pre.omni_tile_plan(sizes, tile, overlap)
        P = len(pages)
        t4 = np.tile(np.arange(4, dtype=np.int32), P)
        T = max(64, max(max(s) for s in sizes))
        plan = Pre.omni_tile_plan(Pre.turned_sizes([s for s in sizes for _ in range(4)], t4), T, 0)
        probe = self._decode_tiles([p for p in pages for _ in range(4)], plan, T, 0, t4, max_batch, test_min_size,
                                   test_max_size, decode)
        n_inst, _, _, rec, prob = probe[:5]
        turns, scores = orient_select(self.ctx, n_inst.reshape(P, 4), rec.reshape((P, 4) + rec.shape[1:]),
                                      prob.reshape((P, 4) + prob.shape[1:]), self.vocab.recog_pad_index,
                                      self.vocab.rec_eos_index)
        return turns, dict(page_scores=scores, probe=probe)

    def group_lines(self, results, **params) -> List[List[dict]]:
        """The words of every page assembled into text lines in reading order (rule: DESIGN 4.12).  results: per page
        what ``decode_pred_seq`` / ``forward_pages`` + ``decode_pred_seq`` / ``spot_tiled`` return, a list of dicts with
        'polys' [16][2] (and 'rec', 'score'), or None / [] for a page without words.  One ``group_lines`` call on the
        device for all pages; params as there.  Returns per page the list of its lines, top to bottom, each
        dict(words=[indices into that page's list, left to right], polys=[16][2] the line polygon (top boundary left
        to right, then bottom right to left: the input of ``preprocess.curve_crops`` / ``recognize_lines``),
        rec='w0 w1 ...', score=mean of the words' scores)."""
        from . import postprocess
        pages = [r or [] for r in results]
        if not pages:
            return []
        count = np.array([len(r) for r in pages], np.int32)
        offset = (np.cumsum(count) - count).astype(np.int32)
        polys = np.array([d['polys'] for r in pages for d in r], np.float64).reshape(-1, 32)
        return postprocess.line_results(pages, offset, group_lines(self.ctx, polys, count, offset, **params))

    def kie_results_json(self, image_sizes) -> List[Optional[str]]:
        """The text `json.dump(output, f)` stores per image (engine/val.py:38-42) for the last `decode_kie` call, produced
        by the library's C++ entity walk (`alm_post_omni_kie_json`); None where nothing was decoded."""
        from . import postprocess
        raw, v = self.last_kie_raw, self.vocab
        args = SimpleNamespace(chars=v.chars, num_bins=v.num_bins, rec_length=v.rec_length,
                               recog_pad_index=v.recog_pad_index, rec_eos_index=v.rec_eos_index)
        out = []
        for b in range(len(raw['n_tok'])):
            nt, ni = int(raw['n_tok'][b]), int(raw['n_inst'][b])
            if nt == 0:
                out.append(None)
                continue
            out.append(postprocess.kie_json(raw['tokens'][b, :nt], raw['probs'][b, :nt], raw['inst_pos'][b, :ni],
                                            raw['poly'][b, :ni], raw['rec'][b, :ni], image_sizes[b], args, v.classes,
                                            v.padding_index + 1))
        return out

    def decode_logits(self, image: int, kind: str, seq: torch.Tensor) -> torch.Tensor:
        """Teacher-forced ``Transformer.decode`` (model/transformer.py:74-100): seq [n,len] -> [n,len,V]."""
        k = {'pt': 0, 'poly': 1, 'rec': 2}[kind]
        s = seq.to(torch.long).cpu().contiguous()
        V = self.lib.alm_omni_vocab(self.ctx.h)
        out = torch.empty(s.shape[0], s.shape[1], V, dtype=torch.float32)
        self.ctx.check(self.lib.alm_omni_decode_logits(self.ctx.h, image, k, s.data_ptr(), s.shape[0], s.shape[1],
                                                       out.data_ptr()))
        return out

    # ---------------------------------------------------------------------------------------- forward
    def forward(self, samples: NestedTensor, sequence=None, rec_candidates: int = 0, rec_beams: int = 0,
                length_penalty: float = 1.0, rec_locations: bool = False, rec_charset: Optional[str] = None):
        """Reference contract for batch 1 (engine/val.py:22,35): returns
        ``([pt[1,2N], poly[1,32N], rec[1,N,L]], [probs[N,L]])`` or ``None``.
        ``sequence`` = [pt_prompt, poly_prompt, rec_prompt, orig_size]; the poly/rec prompts are the fixed
        sos tokens (val.py:30-31) and are validated, the pt prompt is passed through.
        rec_candidates, rec_beams, length_penalty, rec_locations, rec_charset: as in ``decode`` (the return value keeps
        the reference shape)."""
        outs = self.forward_batch(samples, sequence, rec_candidates, rec_beams, length_penalty, rec_locations,
                                  rec_charset)
        if len(outs) != 1:
            raise ValueError('OmniParser.forward keeps the reference batch-1 contract; use forward_batch for B > 1')
        return outs[0]

    def _pt_prompt(self, sequence):
        if sequence is None:
            return None
        v = self.vocab
        if int(sequence[1].reshape(-1)[0]) != v.poly_sos_index or int(sequence[2].reshape(-1)[0]) != v.rec_sos_index:
            raise ValueError('poly/rec prompts must be the sos tokens of the vocabulary (engine/val.py:30-31)')
        return sequence[0]

    def forward_batch(self, samples: NestedTensor, sequence=None, rec_candidates: int = 0, rec_beams: int = 0,
                      length_penalty: float = 1.0, rec_locations: bool = False,
                      rec_charset: Optional[str] = None) -> List:
        """Padded-batch semantics: every page is encoded on the common canvas with the mask (the reference's
        ``model(samples, seqs)`` for a batch).  forward_pages gives each page its batch-1 result instead."""
        pt_prompt = self._pt_prompt(sequence)
        check_rec_charset(rec_charset, self.vocab.chars)
        self.encode(samples.tensors, samples.mask)
        return self._decode_all(samples.tensors.shape[0], sequence, pt_prompt, rec_candidates, rec_beams, length_penalty,
                                rec_locations, rec_charset)

    def forward_pages(self, samples: NestedTensor, sequence=None, rec_candidates: int = 0, rec_beams: int = 0,
                      length_penalty: float = 1.0, rec_locations: bool = False, dense=None,
                      rec_charset: Optional[str] = None) -> List:
        """A batch of pages of different sizes (e.g. from ``preprocess.omni_pages``): a list over pages of what the
        reference's batch-1 ``model(nested_tensor_from_tensor_list([page_b]), seqs)`` returns, text spotting or KIE.
        The page sizes come from the mask (``page_sizes_from_mask``: each page a top-left rectangle, ValueError
        otherwise).  dense='auto' or a grid (nx, ny): text spotting through ``decode_dense(grid=dense)``, so a page with
        more words than one point sequence holds is read in windows instead of failing (None: ``decode``).  rec_charset:
        as in ``decode``, also with dense."""
        pt_prompt = self._pt_prompt(sequence)
        check_rec_charset(rec_charset, self.vocab.chars)
        if dense is not None and (rec_candidates or rec_beams or rec_locations):
            raise ValueError('dense decoding cannot be combined with rec_candidates, rec_beams or rec_locations')
        sizes = page_sizes_from_mask(samples.mask)
        self.encode_pages(samples.tensors, sizes)
        if dense is not None:
            return self.decode_dense(pt_prompt, grid=dense, rec_charset=rec_charset)
        return self._decode_all(len(sizes), sequence, pt_prompt, rec_candidates, rec_beams, length_penalty, rec_locations,
                                rec_charset)

    def _decode_all(self, B, sequence, pt_prompt, rec_candidates=0, rec_beams=0, length_penalty=1.0, rec_locations=False,
                    rec_charset=None):
        if self.vocab.vie_categories:
            if sequence is None or len(sequence) < 4:
                raise ValueError('KIE needs the original image size as sequence[3] (engine/val.py:33)')
            size = sequence[3]
            sizes = [size] * B if torch.as_tensor(size).dim() == 1 else size
            return self.decode_kie([tuple(float(x) for x in torch.as_tensor(sz).reshape(-1)[:2]) for sz in sizes], pt_prompt,
                                   rec_candidates, rec_beams, length_penalty, rec_locations, rec_charset)
        return self.decode(pt_prompt, rec_candidates, rec_beams, length_penalty, rec_locations, rec_charset)
