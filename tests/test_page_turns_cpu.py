"""Pages read turned by quarter-turns (DESIGN 4.14): CPU checks of the turned tile plan, the tile gather, the map-back
and the orientation choice, with the kernels' bodies run on the host (tests/emu/page_turn_emu.cpp) against
oracle/page_turn_ref.py, bit for bit: on np.rot90 itself, on fabricated tile outputs and on
tests/golden/omni_page_turns.npz (the reference run on np.rot90 of a page by oracle/gen_golden_page_turns.py)."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle import page_turn_ref as R
from oracle import tile_ref
from tests.support import assert_same, emu
from tests.test_tiles_cpu import emu_merge, fabricate

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


def bind(lib):
    """Bind tests/emu/page_turn_emu.cpp (host compile of the kernels' bodies)."""
    lib.emu_turned_tiles.restype = C.c_long
    lib.emu_turned_tiles.argtypes = [C.c_void_p] + [C.c_int] * 5 + [C.c_void_p, C.c_long]
    lib.emu_map_back.restype = None
    lib.emu_map_back.argtypes = [C.c_int] + [C.c_double] * 4 + [C.c_void_p, C.c_void_p]
    lib.emu_merge_tiles_turned.restype = C.c_long
    lib.emu_merge_tiles_turned.argtypes = ([C.c_void_p] * 3 + [C.c_int] * 3 + [C.c_void_p] * 5 + [C.c_int] * 3 +
                                           [C.c_double] * 3 + [C.c_void_p] * 7)
    lib.emu_orient_select.restype = None
    lib.emu_orient_select.argtypes = [C.c_int] + [C.c_void_p] * 3 + [C.c_int] * 2 + [C.c_int64] * 2 + [C.c_void_p] * 2


def emu_tiles(page, k, T, ov):
    """tile_gather_kernel on every tile of page read at turn k -> the tiles' bytes, concatenated."""
    lib = emu('page_turn_emu', bind)
    page = np.ascontiguousarray(page, np.uint8)
    H, W = page.shape[:2]
    cap = 4 * (H + T) * (W + T) * 3
    out = np.zeros(cap, np.uint8)
    n = lib.emu_turned_tiles(page.ctypes.data, H, W, k, T, ov, out.ctypes.data, cap)
    assert n >= 0
    return out[:n]


def emu_merge_turned(sizes, turns, T, ov, n_inst, pt, poly, rec, prob, num_bins, margin=4.0, band=None, iou=0.5):
    """alm_omni_merge_tiles_turned's launches on the host -> the dict merge_tiles / page_turn_ref.merge return."""
    lib = emu('page_turn_emu', bind)
    band = ov / 4 if band is None else band
    hs = np.ascontiguousarray([s[0] for s in sizes], np.int32)
    ws = np.ascontiguousarray([s[1] for s in sizes], np.int32)
    ts = np.ascontiguousarray(turns, np.int32)
    n_inst = np.ascontiguousarray(n_inst, np.int32)
    pt, poly, rec = (np.ascontiguousarray(a, np.int64) for a in (pt, poly, rec))
    prob = np.ascontiguousarray(prob, np.float32)
    maxi, L = pt.shape[1], rec.shape[2]
    K = max(int(n_inst.sum()), 1)
    out = dict(count=np.zeros(len(sizes), np.int32), offset=np.zeros(len(sizes), np.int32), pts=np.zeros((K, 2)),
               polys=np.zeros((K, 32)), rec=np.zeros((K, L), np.int64), prob=np.zeros((K, L), np.float32),
               source=np.zeros((K, 2), np.int32))
    n = lib.emu_merge_tiles_turned(hs.ctypes.data, ws.ctypes.data, ts.ctypes.data, len(sizes), T, ov,
                                   n_inst.ctypes.data, pt.ctypes.data, poly.ctypes.data, rec.ctypes.data,
                                   prob.ctypes.data, maxi, L, num_bins, margin, band, iou,
                                   *[out[k].ctypes.data for k in ('count', 'offset', 'pts', 'polys', 'rec', 'prob',
                                                                  'source')])
    for k in ('pts', 'polys', 'rec', 'prob', 'source'):
        out[k] = out[k][:n]
    return out


def emu_select(n_inst, rec, prob, pad, eos):
    """orient_select_kernel on the host -> (turns int32 [P], scores f64 [P, 4])."""
    lib = emu('page_turn_emu', bind)
    n_inst = np.ascontiguousarray(n_inst, np.int32).reshape(-1, 4)
    rec = np.ascontiguousarray(rec, np.int64)
    prob = np.ascontiguousarray(prob, np.float32)
    P = n_inst.shape[0]
    turns, scores = np.zeros(P, np.int32), np.zeros((P, 4))
    lib.emu_orient_select(P, n_inst.ctypes.data, rec.ctypes.data, prob.ctypes.data, rec.shape[2], rec.shape[3], pad,
                          eos, turns.ctypes.data, scores.ctypes.data)
    return turns, scores


def gold():
    return np.load(os.path.join(GOLD, 'omni_page_turns.npz'))


LAYOUTS = ((64, 0), (64, 32), (100, 17), (128, 32))
SIZES = ((1, 1), (7, 5), (63, 129), (131, 97), (200, 65), (65, 200), (300, 221))


def test_turned_plans_are_tile_plans_of_the_turned_sizes():
    """The library's host plan of preprocess.turned_sizes equals tile_ref.plan of np.rot90's shape, every turn."""
    from advancedliteratemachinery_b200 import preprocess as P
    for H, W in SIZES:
        for k in range(4):
            shape = np.rot90(np.zeros((H, W)), k).shape
            assert tuple(P.turned_sizes([(H, W)], [k])[0]) == shape
            for T, ov in LAYOUTS:
                want = np.asarray(tile_ref.plan([shape], T, ov), np.int32).reshape(-1, 5)
                assert np.array_equal(P.omni_tile_plan(P.turned_sizes([(H, W)], [k]), T, ov), want)
                assert R.plan([(H, W)], [k], T, ov) == tile_ref.plan([shape], T, ov)


@pytest.mark.parametrize('k', range(4))
def test_gather_equals_rot90(k):
    """Every tile pixel is the page pixel np.rot90 takes it from, on odd-sized pages smaller and larger than T."""
    rng = np.random.default_rng(k)
    for H, W in SIZES:
        page = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
        for T, ov in LAYOUTS:
            want = np.concatenate([t.reshape(-1) for t in R.tiles([page], [k], T, ov)])
            assert np.array_equal(emu_tiles(page, k, T, ov), want), (H, W, T, ov)


@pytest.mark.parametrize('k', range(4))
def test_map_back_takes_pixel_centres_to_their_source(k):
    """The centre of every turned pixel maps by rule 3 (device body and oracle) to the centre of the page pixel
    np.rot90 took it from."""
    lib = emu('page_turn_emu', bind)
    for H, W in ((7, 5), (4, 9), (1, 3)):
        idx = np.rot90(np.arange(H * W).reshape(H, W), k)
        x, y = C.c_double(), C.c_double()
        for i in range(idx.shape[0]):
            for j in range(idx.shape[1]):
                src_y, src_x = divmod(int(idx[i, j]), W)
                want = (src_x + 0.5, src_y + 0.5)
                lib.emu_map_back(k, j + 0.5, i + 0.5, H, W, C.byref(x), C.byref(y))
                assert (x.value, y.value) == want
                assert R.map_back(j + 0.5, i + 0.5, k, H, W) == want


def test_merge_of_the_fixture_equals_the_oracle():
    """The reference's tiles of np.rot90(page, k), k = 0..3 as four pages: the emulated merge-with-turns equals the
    fixture's oracle merge and the oracle recomputed, bit for bit; the kept rows are those of the upright merge of the
    turned pages, with only the coordinates mapped back."""
    g = gold()
    sizes, turns = [g['page'].shape[:2]] * 4, [0, 1, 2, 3]
    T, ov, nb = int(g['tile']), int(g['overlap']), int(g['num_bins'])
    outs = [g[k] for k in ('n_inst', 'pt', 'poly', 'rec', 'prob')]
    assert np.array_equal(g['plan'], np.asarray(R.plan(sizes, turns, T, ov), np.int32))
    got = emu_merge_turned(sizes, turns, T, ov, *outs, nb)
    assert_same(got, {k: g[f'merged_{k}'] for k in got})
    assert_same(got, R.merge(sizes, turns, T, ov, *outs, nb))
    flat = emu_merge([R.turned_size(*s, k) for s, k in zip(sizes, turns)], T, ov, *outs, nb)
    for k in ('count', 'offset', 'rec', 'prob', 'source'):
        assert np.array_equal(got[k], flat[k]), k
    assert int(got['count'].sum()) > 0


def test_merge_of_fabricated_pages_equals_the_oracle():
    """Fabricated tile outputs of turned pages (several tiles per page, seams in both axes): emulation == oracle bit for
    bit; turn 0 leaves the upright merge untouched."""
    rng = np.random.default_rng(3)
    sizes = [(500, 333), (333, 500), (211, 620), (90, 150)]
    for turns in ([0, 1, 2, 3], [3, 2, 1, 0], [1, 1, 3, 3]):
        turned = [R.turned_size(H, W, k) for (H, W), k in zip(sizes, turns)]
        outs = fabricate(rng, turned, 200, 48, 24, 6, 1000, 12)
        got = emu_merge_turned(sizes, turns, 200, 48, *outs, 1000)
        assert_same(got, R.merge(sizes, turns, 200, 48, *outs, 1000))
        assert int(got['count'].sum()) > 0
    outs = fabricate(rng, sizes, 200, 48, 24, 6, 1000, 12)
    assert_same(emu_merge_turned(sizes, [0] * 4, 200, 48, *outs, 1000), emu_merge(sizes, 200, 48, *outs, 1000))


def test_selection_of_the_fixture_equals_the_oracle_and_the_reference_scores():
    """The fixture's four probe readings: the oracle's instance score is decode_pred_seq's 'score' bit for bit, and the
    emulated choice and page scores equal the oracle's."""
    g = gold()
    pad, eos = int(g['recog_pad_index']), int(g['rec_eos_index'])
    for k in range(4):
        for i in range(int(g['probe_n_inst'][k])):
            assert R.spot_score(g['probe_rec'][k, i], g['probe_prob'][k, i], pad, eos) == g['probe_score'][k, i]
    args = (g['probe_n_inst'][None], g['probe_rec'][None], g['probe_prob'][None], pad, eos)
    turns, scores = emu_select(*args)
    assert turns.tolist() == [int(g['probe_turn'])]
    assert scores.view(np.uint64).tolist() == g['probe_page_scores'][None].view(np.uint64).tolist()
    want = R.choose(*args)
    assert np.array_equal(turns, want[0]) and np.array_equal(scores.view(np.uint64), want[1].view(np.uint64))


def test_selection_equals_the_oracle_on_ties_empty_and_full_readings():
    rng = np.random.default_rng(9)
    P, maxi, L, pad, eos = 40, 7, 9, 1096, 1099
    n_inst = rng.integers(0, maxi + 1, (P, 4)).astype(np.int32)
    n_inst[0] = 0                      # every reading empty: all score 0, turn 0
    n_inst[1] = maxi                   # every reading full
    n_inst[2] = [0, 3, 0, 0]
    rec = rng.choice([pad, eos, pad - 1, 1000, 1001, 1050], (P, 4, maxi, L), p=[.05, .05, .1, .3, .3, .2])
    prob = rng.uniform(0, 1, (P, 4, maxi, L)).astype(np.float32)
    rec[3, 1], prob[3, 1] = rec[3, 3], prob[3, 3]  # a tie between turns 1 and 3 ...
    n_inst[3] = [1, n_inst[3, 3], 0, n_inst[3, 3]]
    rec[3, 0, 0, 0] = pad                          # ... above an empty first instance
    rec[4, :, :, 0] = eos                          # every instance empty: all score 0
    n_inst[4] = maxi
    turns, scores = emu_select(n_inst, rec, prob, pad, eos)
    want_t, want_s = R.choose(n_inst, rec, prob, pad, eos)
    assert np.array_equal(turns, want_t) and np.array_equal(scores.view(np.uint64), want_s.view(np.uint64))
    assert turns[0] == 0 and (scores[0] == 0).all() and turns[4] == 0 and (scores[4] == 0).all()
    assert scores[3, 1] == scores[3, 3] and turns[3] == 1
    assert len(set(turns.tolist())) > 1


def test_argument_errors():
    """Bad turns are refused on the host, before any library call: a wrong length, a turn outside 0..3, a non-integer
    type; orient_select refuses readings that are not four per page."""
    from advancedliteratemachinery_b200 import omniparser as O, preprocess as P
    for bad in ([0, 1], [0, 1, 4], [-1, 0, 0], [0.0, 1.0, 2.0], [[0, 1, 2]]):
        with pytest.raises(ValueError):
            P.check_turns(bad, 3)
    assert P.check_turns(np.array([3, 0, 2], np.int64), 3).dtype == np.int32
    sizes = [(10, 20)]
    outs = [np.zeros(1, np.int32), np.zeros((1, 2, 2)), np.zeros((1, 2, 32)), np.zeros((1, 2, 5)), np.zeros((1, 2, 5))]
    with pytest.raises(ValueError):
        O.merge_tiles(None, sizes, 64, 0, [(0, 0, 0, 20, 10)], *outs, 1000, turns=[4])
    with pytest.raises(ValueError):
        O.merge_tiles(None, sizes, 64, 0, [(0, 0, 0, 20, 10)], *outs, 1000, turns=[1, 1])
    with pytest.raises(ValueError):
        O.orient_select(None, np.zeros((2, 4)), np.zeros((2, 3, 5, 7)), np.zeros((2, 3, 5, 7)), 1, 2)
    with pytest.raises(ValueError):
        O.orient_select(None, np.zeros((2, 4)), np.zeros((2, 4, 5, 7)), np.zeros((2, 4, 5, 6)), 1, 2)
