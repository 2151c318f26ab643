"""Caller-given regions read at quarter-turns (DESIGN 4.21): CPU checks of the rule with the kernel's bodies run on the
host (tests/emu/region_turn_emu.cpp) against a numpy restatement -- the score, the tie and NaN rules, the mapping at all
four turns, turn 0 against ``tile_to_page`` -- and of the host helpers: the forward turn of points and boxes, the tall
rule and the routing in the turned frame."""
import ctypes as C

import numpy as np
import pytest

from advancedliteratemachinery_b200 import preprocess as Pre
from advancedliteratemachinery_b200.omniparser import (plan_region_turns, region_boxes, region_turn_candidates,
                                                       tile_to_page, turn_boxes, turn_points)
from tests.support import emu
from tests.test_read_at_cpu import brute_route

NB = 1000
PAD, EOS = 1096, 1099   # OmniVocab's recog_pad_index / rec_eos_index (unknown = PAD - 1)


def bind(lib):
    """Bind tests/emu/region_turn_emu.cpp (host compile of the kernel's bodies)."""
    lib.emu_select_regions.restype = None
    lib.emu_select_regions.argtypes = ([C.c_long, C.c_int, C.c_void_p, C.c_int] + [C.c_void_p] * 5 +
                                       [C.c_int, C.c_int, C.c_int64, C.c_int64] + [C.c_void_p] * 4)


def emu_select(frames, fidx, pt, poly, rec, prob):
    """alm_omni_select_regions' launch on the host -> (kept, scores, pts, polys)"""
    lib = emu('region_turn_emu', bind)
    fidx = np.ascontiguousarray(fidx, np.int32)
    R, Cn = fidx.shape
    frames = np.ascontiguousarray(frames, np.int32).reshape(-1, 7)
    pt, poly, rec = (np.ascontiguousarray(a, np.int64) for a in (pt, poly, rec))
    prob = np.ascontiguousarray(prob, np.float32)
    out = (np.zeros(R, np.int32), np.zeros((R, Cn)), np.zeros((R, 2)), np.zeros((R, 32)))
    lib.emu_select_regions(R, Cn, fidx.ctypes.data, len(frames), frames.ctypes.data, pt.ctypes.data, poly.ctypes.data,
                           rec.ctypes.data, prob.ctypes.data, rec.shape[2], NB, PAD, EOS, *[a.ctypes.data for a in out])
    return out


# ------------------------------------------------------------------------------------------- numpy restatement
def score(rec, prob):
    """decode_pred_seq's 'score' of one row, in double"""
    s, n = 0.0, 0
    for t, p in zip(rec.tolist(), prob.tolist()):
        if t in (PAD, EOS):
            break
        if t == PAD - 1:
            continue
        s += float(np.float32(p))
        n += 1
    return s / (n + 1e-5)


def ranks_above(sb, kb, sa, ka):
    if np.isnan(sb):
        return False
    if np.isnan(sa):
        return True
    return sb > sa if sb != sa else kb < ka


def map_back(k, u, v, H, W):
    return {0: (u, v), 1: (W - v, u), 2: (W - u, H - v), 3: (v, H - u)}[int(k)]


def map_bins(frame, ids):
    """bins [n, 2] of a reading in frame (H, W, k, y0, x0, h, w) -> upright page pixels [n, 2]"""
    H, W, k, y0, x0, h, w = (int(v) for v in frame)
    ids = np.asarray(ids).reshape(-1, 2)
    f = ids.astype(np.float32) / np.float32(NB) * np.array([w, h], np.float32)
    out = []
    for (fx, fy) in f.astype(np.float64):
        out.append(map_back(k, float(x0) + fx, float(y0) + fy, float(H), float(W)))
    return np.array(out, np.float64)


def select_ref(frames, fidx, pt, poly, rec, prob):
    R, Cn = fidx.shape
    kept, scores = np.zeros(R, np.int32), np.zeros((R, Cn))
    pts, polys = np.zeros((R, 2)), np.zeros((R, 32))
    for r in range(R):
        for c in range(Cn):
            scores[r, c] = score(rec[r, c], prob[r, c])
        best = 0
        for c in range(1, Cn):
            if ranks_above(scores[r, c], frames[fidx[r, c]][2], scores[r, best], frames[fidx[r, best]][2]):
                best = c
        kept[r] = best
        f = frames[fidx[r, best]]
        pts[r] = map_bins(f, pt[r, best])[0]
        polys[r] = map_bins(f, poly[r, best]).reshape(32)
    return kept, scores, pts, polys


def random_frames(rng, F):
    """F frames at random turns: pages up to 4 000 px, tiles anywhere inside the turned page (some whole pages)"""
    fr = []
    for i in range(F):
        H, W, k = int(rng.integers(1, 4000)), int(rng.integers(1, 4000)), int(rng.integers(0, 4))
        th, tw = (W, H) if k & 1 else (H, W)
        if i % 4 == 0:
            y0, x0, h, w = 0, 0, th, tw
        else:
            h, w = int(rng.integers(1, th + 1)), int(rng.integers(1, tw + 1))
            y0, x0 = int(rng.integers(0, th - h + 1)), int(rng.integers(0, tw - w + 1))
        fr.append((H, W, k, y0, x0, h, w))
    return np.array(fr, np.int32)


def fabricate(seed, R=300, Cn=2, L=25, F=16):
    rng = np.random.default_rng(seed)
    frames = random_frames(rng, F)
    fidx = rng.integers(0, F, (R, Cn)).astype(np.int32)
    pt = rng.integers(0, NB, (R, Cn, 2))
    poly = rng.integers(0, NB, (R, Cn, 32))
    rec = rng.integers(NB, NB + 96, (R, Cn, L))
    rec[rng.random((R, Cn, L)) < 0.08] = PAD - 1                  # unknown tokens mid-word
    stop = rng.integers(0, L + 1, (R, Cn))                        # ends anywhere, also at step 0 and never
    for r in range(R):
        for c in range(Cn):
            if stop[r, c] < L:
                rec[r, c, stop[r, c]] = PAD if rng.random() < 0.5 else EOS
    prob = rng.random((R, Cn, L)).astype(np.float32)
    # ties: a region read twice with identical rows, at different turns and at the same one
    for r in range(0, R, 7):
        rec[r, 1:], prob[r, 1:] = rec[r, 0], prob[r, 0]
    return frames, fidx, pt, poly, rec, prob


def assert_same(got, want):
    for a, b, what in zip(got, want, ('kept', 'scores', 'pts', 'polys')):
        assert np.array_equal(a, b, equal_nan=True), what


@pytest.mark.parametrize('seed,Cn', [(0, 1), (1, 2), (2, 2), (3, 4)])
def test_emulation_equals_the_rule(seed, Cn):
    data = fabricate(seed, Cn=Cn)
    assert_same(emu_select(*data), select_ref(*data))


def test_long_rows_and_one_step():
    for L in (1, 1021):
        data = fabricate(5, R=40, L=L)
        assert_same(emu_select(*data), select_ref(*data))


def test_ties_go_to_the_lower_turn_then_the_lower_index():
    frames = np.array([(100, 200, 2, 0, 0, 100, 200), (100, 200, 0, 0, 0, 100, 200), (100, 200, 1, 0, 0, 200, 100),
                       (100, 200, 0, 0, 0, 100, 200)], np.int32)
    L = 6
    row = np.array([NB + 3, NB + 4, EOS, 0, 0, 0])
    p = np.array([0.5, 0.25, 0, 0, 0, 0], np.float32)
    fidx = np.array([[0, 1], [2, 0], [1, 3], [1, 2]], np.int32)   # (2, 0), (1, 2), (0, 0), (0, 1)
    R = len(fidx)
    rec, prob = np.broadcast_to(row, (R, 2, L)), np.broadcast_to(p, (R, 2, L))
    pt, poly = np.zeros((R, 2, 2), np.int64), np.zeros((R, 2, 32), np.int64)
    kept, scores, _, _ = emu_select(frames, fidx, pt, poly, rec, prob)
    assert (scores == scores[0, 0]).all()
    assert kept.tolist() == [1, 0, 0, 0]


def test_a_nan_score_is_never_kept_over_a_number():
    frames = np.array([(100, 200, k, 0, 0) + ((200, 100) if k & 1 else (100, 200)) for k in range(4)], np.int32)
    L = 4
    R = 6
    rec = np.full((R, 2, L), NB + 5)
    prob = np.full((R, 2, L), 0.5, np.float32)
    prob[0, 0, 1] = np.nan        # candidate 0 NaN, 1 finite: 1 kept
    prob[1, 1, 2] = np.nan        # candidate 1 NaN: 0 kept
    prob[2, :, 0] = np.nan        # both NaN: candidate 0
    prob[3, 0, 0] = np.inf        # +inf is a number: kept over 0.5
    prob[4, 1, 0] = -np.inf       # -inf still ranks above NaN
    prob[4, 0, 0] = np.nan
    prob[5, 1] = 0.75             # the larger score at the higher turn
    fidx = np.array([[0, 2]] * R, np.int32)
    pt, poly = np.zeros((R, 2, 2), np.int64), np.zeros((R, 2, 32), np.int64)
    got = emu_select(frames, fidx, pt, poly, rec, prob)
    assert got[0].tolist() == [1, 0, 0, 0, 1, 1]
    assert_same(got, select_ref(frames, fidx, pt, poly, rec, prob))


@pytest.mark.parametrize('k', range(4))
def test_mapping_at_every_turn_is_exact_in_double(k):
    rng = np.random.default_rng(10 + k)
    frames = random_frames(rng, 12)
    frames[:, 2] = k
    th, tw = np.where(k & 1, frames[:, 1], frames[:, 0]), np.where(k & 1, frames[:, 0], frames[:, 1])
    frames[:, 5] = np.minimum(frames[:, 5], th - frames[:, 3])
    frames[:, 6] = np.minimum(frames[:, 6], tw - frames[:, 4])
    R = 200
    fidx = rng.integers(0, len(frames), (R, 1)).astype(np.int32)
    pt = rng.integers(0, NB, (R, 1, 2))
    pt[:4] = [[[0, 0]], [[NB - 1, NB - 1]], [[0, NB - 1]], [[NB - 1, 0]]]
    poly = rng.integers(0, NB, (R, 1, 32))
    rec = np.full((R, 1, 3), EOS)
    prob = np.zeros((R, 1, 3), np.float32)
    _, _, pts, polys = emu_select(frames, fidx, pt, poly, rec, prob)
    for r in range(R):
        f = frames[fidx[r, 0]]
        assert np.array_equal(pts[r], map_bins(f, pt[r, 0])[0])
        assert np.array_equal(polys[r], map_bins(f, poly[r, 0]).reshape(32))


def test_turn_zero_with_one_candidate_is_tile_to_page():
    rng = np.random.default_rng(20)
    frames = random_frames(rng, 10)
    frames[:, 2] = 0
    frames[:, 5] = np.minimum(frames[:, 5], frames[:, 0] - frames[:, 3])
    frames[:, 6] = np.minimum(frames[:, 6], frames[:, 1] - frames[:, 4])
    R = 100
    fidx = rng.integers(0, len(frames), (R, 1)).astype(np.int32)
    pt, poly = rng.integers(0, NB, (R, 1, 2)), rng.integers(0, NB, (R, 1, 32))
    rec, prob = np.full((R, 1, 2), NB + 1), np.full((R, 1, 2), 0.5, np.float32)
    kept, _, pts, polys = emu_select(frames, fidx, pt, poly, rec, prob)
    assert not kept.any()
    for r in range(R):
        _, _, _, y0, x0, h, w = frames[fidx[r, 0]]
        assert np.array_equal(pts[r], tile_to_page((y0, x0), (h, w), pt[r, 0], NB)[0])
        assert np.array_equal(polys[r], tile_to_page((y0, x0), (h, w), poly[r, 0].reshape(16, 2), NB).reshape(32))


# ------------------------------------------------------------------------------------------------ host helpers
def test_turn_points_inverts_map_back_on_integers():
    rng = np.random.default_rng(30)
    N = 500
    hw = rng.integers(1, 5000, (N, 2))
    xy = np.stack([rng.integers(0, hw[:, 1] + 1), rng.integers(0, hw[:, 0] + 1)], 1).astype(np.float64)
    k = rng.integers(0, 4, N)
    t = turn_points(xy, hw, k)
    th, tw = np.where(k & 1, hw[:, 1], hw[:, 0]), np.where(k & 1, hw[:, 0], hw[:, 1])
    assert ((t >= 0) & (t <= np.stack([tw, th], 1))).all(), 'a point on the page lands on the turned page'
    for n in range(N):
        assert map_back(k[n], t[n, 0], t[n, 1], float(hw[n, 0]), float(hw[n, 1])) == tuple(xy[n])
    # np.rot90's convention on pixel centres: pixel (x, y) of the page is pixel (x', y') of np.rot90(page, k) with
    # (x' + 0.5, y' + 0.5) the turned centre
    page = np.arange(6 * 9).reshape(6, 9)
    for kk in range(4):
        rot = np.rot90(page, kk)
        for y in range(6):
            for x in range(9):
                u, v = turn_points([[x + 0.5, y + 0.5]], [[6, 9]], [kk])[0]
                assert rot[int(v - 0.5), int(u - 0.5)] == page[y, x]


def test_turn_boxes_are_the_boxes_of_the_turned_corners():
    rng = np.random.default_rng(31)
    N = 300
    hw = rng.integers(50, 3000, (N, 2))
    x = np.sort(rng.integers(0, hw[:, 1:2] + 1, (N, 2)), 1)
    y = np.sort(rng.integers(0, hw[:, :1] + 1, (N, 2)), 1)
    boxes = np.stack([x[:, 0], y[:, 0], x[:, 1], y[:, 1]], 1).astype(np.float64)
    k = rng.integers(0, 4, N)
    got = turn_boxes(boxes, hw, k)
    corners = np.stack([boxes[:, [0, 1]], boxes[:, [2, 1]], boxes[:, [2, 3]], boxes[:, [0, 3]]], 1)
    t = turn_points(corners.reshape(-1, 2), np.repeat(hw, 4, 0), np.repeat(k, 4)).reshape(N, 4, 2)
    assert np.array_equal(got, np.concatenate([t.min(1), t.max(1)], 1))
    assert np.array_equal(turn_boxes(boxes, hw, np.zeros(N, int)), boxes)


def test_tall_rule():
    sizes = [(3000, 2000), (800, 600)]
    boxes = np.array([[10, 10, 30, 40], [10, 10, 30, 39], [0, 0, 100, 20], [5, 5, 5, 5], [30, 40, 10, 10]], float)
    got = region_turn_candidates(sizes, boxes, [0, 0, 1, 1, 0], 'box')
    assert got.tolist() == [[1, 3], [0, 2], [0, 2], [1, 3], [1, 3]]   # 2 h >= 3 w; a zero box is tall
    assert region_turn_candidates(sizes, [[5, 5], [9, 9]], [0, 1], 'point').tolist() == [[0, 2], [0, 2]]
    rng = np.random.default_rng(32)
    R = 200
    c = rng.uniform(100, 500, (R, 1, 2))
    half = rng.uniform(2, 90, (R, 1, 2))
    quads = c + half * np.array([[-1, -1], [1, -1], [1, 1], [-1, 1]])
    pi = rng.integers(0, 2, R)
    cs = Pre.quad_plan(sizes, quads, pi)['sizes'].astype(np.int64)
    want = np.where((2 * cs[:, 1] >= 3 * cs[:, 0])[:, None], [1, 3], [0, 2])
    got = region_turn_candidates(sizes, quads, pi, 'quad')
    assert np.array_equal(got, want) and got.dtype == np.int32 and 0 < (got[:, 0] == 1).sum() < R
    t = np.linspace(0, 1, 8)
    top = np.stack([100 + 20 * t, 100 + 300 * t], 1)            # a tall curved column
    poly = np.concatenate([top, (top + [30, 0])[::-1]])[None]
    cs = Pre.curve_plan(sizes, poly, [0])['sizes'][0]
    assert region_turn_candidates(sizes, poly, [0], 'polygon').tolist() == [[1, 3] if 2 * cs[1] >= 3 * cs[0] else
                                                                            [0, 2]]


@pytest.mark.parametrize('seed', range(4))
def test_routing_in_the_turned_frame_against_brute_force(seed):
    rng = np.random.default_rng(40 + seed)
    sizes = [(int(rng.integers(200, 3600)), int(rng.integers(200, 3600))) for _ in range(3)] + [(900, 700)]
    tile, overlap = int(rng.choice([600, 1200])), int(rng.choice([0, 128, 256]))
    R, Cn = 300, int(rng.choice([1, 2]))
    pi = rng.integers(0, len(sizes), R)
    hw = np.array([sizes[p] for p in pi], np.float64)
    c = np.round(rng.uniform(0, 1, (R, 2)) * hw[:, ::-1])
    half = np.round(rng.uniform(0, 1, (R, 2)) * rng.choice([20, 200, 900], (R, 1)))
    boxes = np.concatenate([np.maximum(c - half, 0), np.minimum(c + half, hw[:, ::-1])], 1)
    turns = rng.integers(0, 4, (R, Cn))
    turns[pi == 3] = 1   # a page read at one turn only
    got = plan_region_turns(sizes, boxes, pi, turns, tile, overlap)
    rd = got['readings']
    assert [tuple(r) for r in rd.tolist()] == sorted(set(zip(pi.tolist() * Cn, turns.T.reshape(-1).tolist())))
    assert np.array_equal(rd[got['reading'], 0], np.repeat(pi[:, None], Cn, 1))
    assert np.array_equal(rd[got['reading'], 1], turns)
    read = Pre.turned_sizes([sizes[p] for p in rd[:, 0]], rd[:, 1])
    assert np.array_equal(got['plan'], Pre.omni_tile_plan(read, tile, overlap))
    for cc in range(Cn):
        tb = turn_boxes(boxes, hw, turns[:, cc])
        want = brute_route(read, got['plan'], tb, got['reading'][:, cc])
        assert np.array_equal(got['route'][:, cc], want), cc
    assert (got['route'] == -1).any() and (got['route'] >= 0).any()


def test_turn_zero_routing_is_the_upright_routing():
    rng = np.random.default_rng(50)
    sizes = [(3508, 2480), (500, 700)]
    R = 200
    pi = rng.integers(0, 2, R)
    hw = np.array([sizes[p] for p in pi], np.float64)
    xy = rng.uniform(0, 1, (R, 2)) * (hw[:, ::-1] - 400)
    boxes = np.concatenate([xy, xy + rng.uniform(10, 400, (R, 2))], 1)
    got = plan_region_turns(sizes, boxes, pi, np.zeros((R, 1), int))
    plan = Pre.omni_tile_plan(sizes)
    assert np.array_equal(got['plan'], plan)
    assert np.array_equal(got['route'][:, 0], brute_route(sizes, plan, region_boxes(boxes, 'box'), pi))
