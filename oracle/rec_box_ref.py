"""Restatement, in Python doubles, of the character boxes in page pixels of words read in tiles (DESIGN 4.20;
include/alm_ocr.h alm_omni_char_boxes) -- TEST INFRASTRUCTURE ONLY (the product is
advancedliteratemachinery_b200/csrc/rec_box_core.h, run by rec_box_kernel).  Written from the rule: the centre and
covariance of every step in the tile's frame, turned to the page, then ``postprocess.rec_char_boxes``' box on the
word's page polygon.  Every value is a Python float and every operation is the rule's, in its order, so the results are
the device's bits.

  char_box(P, frame, loc)                         one character -> (centre [2], cov [3], box [8])
  char_boxes(polys, rec, loc, frame_index, frames, pad, eos)
                                                  every word -> dict(n_chars, step, centre, cov, box) in the layout of
                                                  alm_omni_char_boxes (slots past n_chars are 0)
"""
from __future__ import annotations

import math

import numpy as np

from oracle.whole_page_ref import map_back


def _centre_line(P):
    """c_i = (P_i + P_{15-i}) / 2 and h_i = |P_i - P_{15-i}|, i = 0..7, of the polygon P (32 floats)."""
    c, hgt = [], []
    for i in range(8):
        j = 15 - i
        c.append(((P[2 * i] + P[2 * j]) / 2.0, (P[2 * i + 1] + P[2 * j + 1]) / 2.0))
        dx, dy = P[2 * i] - P[2 * j], P[2 * i + 1] - P[2 * j + 1]
        hgt.append(math.sqrt(dx * dx + dy * dy))
    return c, hgt


def char_box(P, frame, loc):
    """P: the word's 16 vertices in page pixels (32 floats); frame = (H, W, turn, y0, x0, h, w); loc: (cx, cy, sxx,
    sxy, syy) of the step, normalised by the tile's encoded size."""
    H, W, k, y0, x0, h, w = (int(v) for v in frame)
    cx, cy, sxx, sxy, syy = (float(v) for v in loc)
    mx, my = map_back(k, x0 + cx * float(w), y0 + cy * float(h), float(H), float(W))
    sxx, sxy, syy = sxx * w * w, sxy * w * h, syy * h * h
    if k % 2:
        sxx, sxy, syy = syy, -sxy, sxx
    P = [float(v) for v in P]
    c, hgt = _centre_line(P)
    best, bi, bs = None, 0, 0.0
    for i in range(7):
        sx, sy = c[i + 1][0] - c[i][0], c[i + 1][1] - c[i][1]
        seg2 = sx * sx + sy * sy
        s = 0.0
        if seg2 > 0:
            s = ((mx - c[i][0]) * sx + (my - c[i][1]) * sy) / seg2
            s = 0.0 if s < 0 else (1.0 if s > 1 else s)   # NaN stays NaN
        dx, dy = mx - (c[i][0] + s * sx), my - (c[i][1] + s * sy)
        d = dx * dx + dy * dy
        # np.argmin: the first NaN, else the first minimum
        if best is None or (not math.isnan(best) and (math.isnan(d) or d < best)):
            best, bi, bs = d, i, s
    sx, sy = c[bi + 1][0] - c[bi][0], c[bi + 1][1] - c[bi][1]
    qx, qy = c[bi][0] + bs * sx, c[bi][1] + bs * sy
    if not sx * sx + sy * sy > 0:
        sx, sy = c[7][0] - c[0][0], c[7][1] - c[0][1]
    norm = math.sqrt(sx * sx + sy * sy)
    ux, uy = (sx / norm, sy / norm) if norm > 0 else (1.0, 0.0)
    vx, vy = -uy, ux
    hq = hgt[bi] + bs * (hgt[bi + 1] - hgt[bi])
    var = ux * ux * sxx + 2.0 * ux * uy * sxy + uy * uy * syy
    var = 0.0 if 0.0 > var else var
    a = math.sqrt(3.0) * math.sqrt(var)
    half = hq / 2.0
    box = [qx - a * ux - half * vx, qy - a * uy - half * vy,
           qx + a * ux - half * vx, qy + a * uy - half * vy,
           qx + a * ux + half * vx, qy + a * uy + half * vy,
           qx - a * ux + half * vx, qy - a * uy + half * vy]
    return [mx, my], [sxx, sxy, syy], box


def char_boxes(polys, rec, loc, frame_index, frames, pad, eos):
    """polys [N, 32] (or [N, 16, 2]), rec [N, L], loc [N, L, 5], frame_index [N], frames [F, 7] -> dict(n_chars int32
    [N], step int32 [N, L], centre f64 [N, L, 2], cov f64 [N, L, 3], box f64 [N, L, 8])."""
    polys = np.asarray(polys, dtype=np.float64).reshape(-1, 32)
    rec = np.asarray(rec, dtype=np.int64)
    N, L = rec.shape
    loc = np.asarray(loc, dtype=np.float32).reshape(N, L, 5)
    frames = np.asarray(frames, dtype=np.int64).reshape(-1, 7)
    out = dict(n_chars=np.zeros(N, np.int32), step=np.zeros((N, L), np.int32), centre=np.zeros((N, L, 2)),
               cov=np.zeros((N, L, 3)), box=np.zeros((N, L, 8)))
    for n in range(N):
        P = polys[n].tolist()
        frame = frames[int(frame_index[n])].tolist()
        i = 0
        for j, tok in enumerate(rec[n].tolist()):
            if tok == pad or tok == eos:
                break
            if tok == pad - 1:
                continue
            out['centre'][n, i], out['cov'][n, i], out['box'][n, i] = char_box(P, frame, loc[n, j].tolist())
            out['step'][n, i] = j
            i += 1
        out['n_chars'][n] = i
    return out
