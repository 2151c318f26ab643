"""Restatement, in Python doubles, of the recovery of KIE entities that cross tile seams from a whole-page KIE reading
(DESIGN 4.22; include/alm_ocr.h alm_omni_merge_kie_whole_page), on top of oracle/kie_tile_ref.py and oracle/tile_ref.py.
Written from the rule, not from the kernels: a whole entity's box is tested against every tile of its page's plan with
plain double loops (not the kernels' separable per-axis form), and every tile entity's anchor against every kept whole
box of its page.

The rule.
  whole    the walk of the page's whole-page reading (np.rot90(page, k) decoded as one image); word rects the
           reference's image_w * min / num_bins with the turned size, origin 0; the entity box the union of its words'
           rects.
  keep     a whole entity with words whose box every tile of the plan cuts: an edge of the box within margin (<=) of an
           interior edge of the tile, in the tile's frame, edges outside the tile included.
  map      a kept entity's word rects map back corner by corner, min / max re-ordered; its polygons vertex by vertex.
  drop     a tile entity with words whose anchor (the centre of the union of its word rects; none when a coordinate is
           not finite) lies inside the page box of a kept whole entity, edges included.
  output   per page the kept tile entities in input order, then the kept whole entities in entity order."""
from __future__ import annotations

import math

import numpy as np

from oracle import kie_tile_ref as K
from oracle import page_turn_ref as PT
from oracle import tile_ref as R


def cut_by_every_tile(box, th, tw, T, ov, margin):
    """Every tile of the th x tw (turned) page's plan has an edge of box (x0, y0, x1, y1) within margin of one of its
    interior edges, in its own frame."""
    for t in R.tile_grid([(th, tw)], T, ov, 0.0):
        il, ir, it, ib = t['ix'] > 0, t['ix'] < t['nx'] - 1, t['iy'] > 0, t['iy'] < t['ny'] - 1
        cut = False
        for x in (box[0] - t['x0'], box[2] - t['x0']):
            cut = cut or (il and x <= margin) or (ir and t['w'] - x <= margin)
        for y in (box[1] - t['y0'], box[3] - t['y0']):
            cut = cut or (it and y <= margin) or (ib and t['h'] - y <= margin)
        if not cut:
            return False
    return True


def whole_entities(H, W, k, T, ov, margin, num_bins, class_base, n_classes, tokens, probs, inst_pos, poly):
    """One page's whole-page reading -> [(class, prob, [instance, ...], page box or None, kept)]."""
    th, tw = PT.turned_size(H, W, k)
    out = []
    for cls, prob, words in K.walk(tokens, probs, inst_pos, num_bins, class_base, n_classes):
        if not words:
            out.append((cls, prob, words, None, False))
            continue
        rects = [K.word_rect(poly[i], th, tw, num_bins) for i in words]
        box = (min(r[0] for r in rects), min(r[1] for r in rects), max(r[2] for r in rects), max(r[3] for r in rects))
        kept = cut_by_every_tile(box, th, tw, T, ov, margin)
        x0, y0 = PT.map_back(box[0], box[1], k, H, W)
        x1, y1 = PT.map_back(box[2], box[3], k, H, W)
        out.append((cls, prob, words, (min(x0, x1), min(y0, y1), max(x0, x1), max(y0, y1)), kept))
    return out


def anchor(rects):
    """The centre of the union of a tile entity's word rects, or None without words or with a non-finite coordinate."""
    if not len(rects) or not all(math.isfinite(float(c)) for r in rects for c in r):
        return None
    return ((min(float(r[0]) for r in rects) + max(float(r[2]) for r in rects)) * 0.5,
            (min(float(r[1]) for r in rects) + max(float(r[3]) for r in rects)) * 0.5)


def merge(sizes, turns, T, ov, margin, num_bins, class_base, n_classes, tiles, whole):
    """tiles: merge_kie_tiles' dict of the pages; whole: each page's whole-page KIE reading (n_tok, tokens, probs,
    n_inst, inst_pos, poly, one row per page) -> the dict alm_omni_merge_kie_whole_page returns."""
    turns = [0] * len(sizes) if turns is None else [int(k) for k in turns]
    ent = dict(count=[], cls=[], prob=[], word_count=[], source=[])
    word = dict(rect=[], poly=[], word_source=[])
    for p, (H, W) in enumerate(sizes):
        k = turns[p]
        th, tw = PT.turned_size(H, W, k)
        nt, ni = int(whole['n_tok'][p]), int(whole['n_inst'][p])
        wes = whole_entities(H, W, k, T, ov, margin, num_bins, class_base, n_classes, whole['tokens'][p][:nt],
                             whole['probs'][p][:nt], whole['inst_pos'][p][:ni], whole['poly'][p])
        boxes = [e[3] for e in wes if e[4]]
        n = 0
        for r in range(int(tiles['offset'][p]), int(tiles['offset'][p]) + int(tiles['count'][p])):
            ws = range(int(tiles['word_offset'][r]), int(tiles['word_offset'][r]) + int(tiles['word_count'][r]))
            a = anchor([tiles['rect'][w] for w in ws])
            if a is not None and any(b[0] <= a[0] <= b[2] and b[1] <= a[1] <= b[3] for b in boxes):
                continue
            ent['cls'].append(tiles['cls'][r])
            ent['prob'].append(tiles['prob'][r])
            ent['word_count'].append(len(ws))
            ent['source'].append(tiles['source'][r])
            for w in ws:
                word['rect'].append(tiles['rect'][w])
                word['poly'].append(tiles['poly'][w])
                word['word_source'].append(tiles['word_source'][w])
            n += 1
        for e, (cls, prob, words, _, kept) in enumerate(wes):
            if not kept:
                continue
            ent['cls'].append(cls)
            ent['prob'].append(prob)
            ent['word_count'].append(len(words))
            ent['source'].append((-1, e))
            for i in words:
                r = K.word_rect(whole['poly'][p][i], th, tw, num_bins)
                x0, y0 = PT.map_back(r[0], r[1], k, H, W)
                x1, y1 = PT.map_back(r[2], r[3], k, H, W)
                word['rect'].append((min(x0, x1), min(y0, y1), max(x0, x1), max(y0, y1)))
                word['poly'].append([c for j in range(16) for c in PT.map_back(
                    R.coord(whole['poly'][p][i][2 * j], num_bins, tw),
                    R.coord(whole['poly'][p][i][2 * j + 1], num_bins, th), k, H, W)])
                word['word_source'].append((-1, i))
            n += 1
        ent['count'].append(n)
    count = np.array(ent['count'], np.int32)
    wc = np.array(ent['word_count'], np.int32)
    return dict(count=count, offset=(np.cumsum(count) - count).astype(np.int32), cls=np.array(ent['cls'], np.int32),
                prob=np.array(ent['prob'], np.float32), word_offset=(np.cumsum(wc) - wc).astype(np.int32),
                word_count=wc, source=np.array(ent['source'], np.int32).reshape(-1, 2),
                rect=np.array(word['rect'], np.float64).reshape(-1, 4),
                poly=np.array(word['poly'], np.float64).reshape(-1, 32),
                word_source=np.array(word['word_source'], np.int32).reshape(-1, 2))
