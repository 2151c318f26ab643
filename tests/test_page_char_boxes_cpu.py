"""Character boxes in page pixels of words read in tiles (DESIGN 4.20): CPU checks with the kernel's bodies run on the
host (tests/emu/rec_box_emu.cpp) against oracle/rec_box_ref.py, bit for bit, on fabricated words and hand-made cases;
the identity frame against ``postprocess.rec_char_boxes``; the turn commuting with the boxes; and the refusals of
``omniparser.char_boxes``."""
import ctypes as C

import numpy as np
import pytest

from oracle import rec_box_ref as R
from oracle.whole_page_ref import map_back
from tests.support import emu

NB = 1000
PAD, EOS = 1096, 1099   # OmniVocab's recog_pad_index / rec_eos_index (unknown = PAD - 1)
KEYS = ('n_chars', 'step', 'centre', 'cov', 'box')


def bind(lib):
    """Bind tests/emu/rec_box_emu.cpp (host compile of the kernel's bodies)."""
    lib.emu_char_boxes.restype = None
    lib.emu_char_boxes.argtypes = ([C.c_long, C.c_int] + [C.c_void_p] * 4 + [C.c_int, C.c_void_p, C.c_int64, C.c_int64] +
                                   [C.c_void_p] * 5)
    lib.emu_valid_frame.restype = C.c_int
    lib.emu_valid_frame.argtypes = [C.c_void_p]


def emu_boxes(polys, rec, loc, frame_index, frames, pad=PAD, eos=EOS):
    """alm_omni_char_boxes' launch on the host -> the dict omniparser.char_boxes / rec_box_ref.char_boxes return."""
    lib = emu('rec_box_emu', bind)
    polys = np.ascontiguousarray(polys, np.float64).reshape(-1, 32)
    rec = np.ascontiguousarray(rec, np.int64)
    N, L = rec.shape
    loc = np.ascontiguousarray(loc, np.float32).reshape(N, L, 5)
    fi = np.ascontiguousarray(frame_index, np.int32)
    frames = np.ascontiguousarray(frames, np.int32).reshape(-1, 7)
    out = dict(n_chars=np.zeros(N, np.int32), step=np.zeros((N, L), np.int32), centre=np.zeros((N, L, 2)),
               cov=np.zeros((N, L, 3)), box=np.zeros((N, L, 8)))
    lib.emu_char_boxes(N, L, polys.ctypes.data, rec.ctypes.data, loc.ctypes.data, fi.ctypes.data, len(frames),
                       frames.ctypes.data, pad, eos, *[out[k].ctypes.data for k in KEYS])
    return out


def assert_same(a, b):
    """Equal in every field, NaN where the other has NaN."""
    for k in KEYS:
        assert np.array_equal(a[k], b[k], equal_nan=a[k].dtype.kind == 'f'), k


def frames_to_tiles(frames):
    """frames [F, 7] -> (sizes [(H, W)] per frame, tiles [F, 5] with page f = frame f, turns [F]): the arguments of
    omniparser.char_boxes that rebuild the same frames."""
    frames = np.asarray(frames).reshape(-1, 7)
    sizes = [(int(f[0]), int(f[1])) for f in frames]
    tiles = np.stack([np.arange(len(frames)), frames[:, 3], frames[:, 4], frames[:, 5], frames[:, 6]], 1)
    return sizes, tiles, frames[:, 2].astype(np.int32)


def fabricate(seed, N=200, L=25, F=12, nan=0.02):
    """N words on F random frames: pages up to 4 000 px at turns 0..3, anisotropic tiles, a third of them on the
    turned page's far border; curved polygons in page pixels, some with repeated centre-line points; ids with unknown
    tokens mid-word and ends anywhere (also at step 0); locations with positive-definite covariances, a few NaN."""
    rng = np.random.default_rng(seed)
    frames = np.zeros((F, 7), np.int32)
    for f in range(F):
        H, W, k = int(rng.integers(64, 4000)), int(rng.integers(64, 4000)), f % 4
        th, tw = (W, H) if k % 2 else (H, W)
        h, w = int(rng.integers(1, th + 1)), int(rng.integers(1, tw + 1))
        y0 = th - h if rng.random() < 0.33 else int(rng.integers(0, th - h + 1))
        x0 = tw - w if rng.random() < 0.33 else int(rng.integers(0, tw - w + 1))
        frames[f] = (H, W, k, y0, x0, h, w)
    fi = rng.integers(0, F, N).astype(np.int32)
    polys = np.zeros((N, 32))
    for n in range(N):
        H, W = frames[fi[n], :2]
        c = rng.uniform([0, 0], [W, H])
        ang = rng.uniform(-np.pi, np.pi)
        d = np.array([np.cos(ang), np.sin(ang)])
        nrm = np.array([-d[1], d[0]])
        t = np.sort(rng.uniform(0, rng.uniform(5, 400), 8))
        if rng.random() < 0.2:
            t[2:4] = t[2]   # zero-length centre-line segments
        bend = rng.normal(0, 3, 8).cumsum()
        half = rng.uniform(0, 40) * (1 + 0.2 * rng.standard_normal(8))
        mid = c + t[:, None] * d + bend[:, None] * nrm
        top, bot = mid - half[:, None] * nrm, mid + half[:, None] * nrm
        polys[n] = np.concatenate([top, bot[::-1]]).reshape(-1)
    rec = rng.integers(NB, NB + 95, (N, L))
    rec[rng.random((N, L)) < 0.1] = PAD - 1
    for n in range(N):
        e = int(rng.integers(0, L + 3))
        if e < L:
            rec[n, e:] = PAD if rng.random() < 0.5 else EOS
            if rng.random() < 0.3:   # whatever follows the stop is ignored
                rec[n, e + 1:] = rng.integers(NB, NB + 95, L - e - 1)
    loc = np.zeros((N, L, 5), np.float32)
    loc[..., :2] = rng.uniform(-0.05, 1.05, (N, L, 2))
    a, b = rng.uniform(1e-5, 2e-2, (N, L)), rng.uniform(1e-5, 2e-2, (N, L))
    r = rng.uniform(-0.99, 0.99, (N, L)) * np.sqrt(a * b)
    loc[..., 2], loc[..., 3], loc[..., 4] = a, r, b
    loc[rng.random((N, L, 5)) < nan] = np.nan
    return polys, rec, loc, fi, frames


def both(*args):
    """The frames are valid and the emulation equals the oracle bit for bit; returns the result."""
    frames = np.ascontiguousarray(args[4], np.int32).reshape(-1, 7)
    assert all(emu('rec_box_emu', bind).emu_valid_frame(f.ctypes.data) for f in frames)
    got = emu_boxes(*args)
    assert_same(got, R.char_boxes(*args, PAD, EOS))
    return got


@pytest.mark.parametrize('seed', range(6))
def test_emulation_equals_oracle_on_fabricated_words(seed):
    polys, rec, loc, fi, frames = fabricate(seed)
    got = both(polys, rec, loc, fi, frames)
    assert set(frames[fi, 2].tolist()) == {0, 1, 2, 3}
    assert (got['n_chars'] == 0).any() and (got['n_chars'] > 10).any()
    assert np.isnan(got['box']).any() and np.isfinite(got['box']).any()


@pytest.mark.parametrize('L', [1, 1021])
def test_emulation_equals_oracle_at_the_rec_length_bounds(L):
    polys, rec, loc, fi, frames = fabricate(10 + L, N=24 if L > 1 else 200, L=L)
    got = both(polys, rec, loc, fi, frames)
    if L > 1:
        assert got['n_chars'].max() > 900


def hand_made_words():
    """First step terminal, unknown tokens mid-word, a zero-height polygon, a polygon whose centre line is one point,
    NaN locations, every turn, tiles at the page's corner and a one-pixel-high tile: (polys, rec, loc, fi, frames)."""
    top = np.stack([np.linspace(100, 170, 8), np.full(8, 50.0)], 1)
    flat = np.concatenate([top, top[::-1]]).reshape(-1)                  # zero height
    dot = np.tile([120.0, 60.0], 16)                                     # every vertex one point
    word = np.concatenate([top, (top + [0, 20])[::-1]]).reshape(-1)
    polys = np.stack([word, word, flat, dot, word, word, word, word])
    L = 6
    rec = np.full((8, L), NB + 3)
    rec[0, 0] = EOS                          # nothing read
    rec[1, [1, 3]] = PAD - 1                 # unknowns skipped: characters are steps 0, 2, 4, 5
    rec[4, 2] = PAD
    loc = np.full((8, L, 5), 0.5, np.float32)
    loc[..., 2:] = [1e-3, 2e-4, 5e-4]
    loc[5, 1, 0] = np.nan
    loc[6, 2, 3] = np.nan
    frames = np.array([(300, 200, k, 0, 0, 64, 64) for k in range(4)] +
                      [(300, 200, 1, 200 - 80, 300 - 50, 80, 50), (300, 200, 0, 300 - 1, 0, 1, 200)], np.int32)
    fi = np.array([0, 1, 2, 3, 4, 5, 0, 1], np.int32)
    return polys, rec, loc, fi, frames


def test_hand_made_words():
    got = both(*hand_made_words())
    assert got['n_chars'].tolist() == [0, 4, 6, 6, 2, 6, 6, 6]
    assert got['step'][1, :4].tolist() == [0, 2, 4, 5] and not got['step'][1, 4:].any()
    assert not got['box'][0].any() and not got['box'][4, 2:].any()
    assert np.isnan(got['centre'][5, 1, 0]) and np.isfinite(got['centre'][5, 0]).all()
    assert np.isnan(got['cov'][6, 2, 1]) and np.isfinite(got['cov'][6, 2, [0, 2]]).all()
    assert np.isfinite(got['box'][2]).all() and np.isfinite(got['box'][3]).all()
    # a zero-height word gives boxes of zero height; a one-point word boxes along +x
    b = got['box'][2, 0].reshape(4, 2)
    assert np.allclose(b[0], b[3]) and np.allclose(b[1], b[2])
    b = got['box'][3, 0].reshape(4, 2)
    assert b[0, 1] == b[1, 1] and b[1, 0] > b[0, 0]


def test_identity_frame_matches_rec_char_boxes():
    from advancedliteratemachinery_b200 import postprocess
    from advancedliteratemachinery_b200.omniparser import OmniVocab
    v = OmniVocab()
    rng = np.random.default_rng(7)
    polys, rec, loc, _, _ = fabricate(7, N=120, nan=0.0)
    for h, w in [(1200, 1200), (905, 1337), (3508, 2480)]:
        ids = rng.integers(0, NB, (len(polys), 32))
        ids[:, 16:] = np.clip(ids[:, 15::-1] + rng.integers(5, 60, (len(polys), 16)), 0, NB - 1)
        P = ids.astype(np.float64).reshape(-1, 16, 2) / NB * np.array([w, h])
        want = postprocess.rec_char_boxes(ids, rec, loc, (h, w), v)
        got = R.char_boxes(P.reshape(-1, 32), rec, loc, np.zeros(len(P), np.int32), [(h, w, 0, 0, 0, h, w)],
                           v.recog_pad_index, v.rec_eos_index)
        for n, chars in enumerate(want):
            assert got['n_chars'][n] == len(chars)
            for i, ch in enumerate(chars):
                assert v.chars[int(rec[n, got['step'][n, i]]) - NB] == ch['char']
                assert np.abs(got['centre'][n, i] - ch['centre']).max() <= 1e-9
                assert np.abs(got['cov'][n, i] - ch['cov'].reshape(-1)[[0, 1, 3]]).max() <= 1e-9
                assert np.abs(got['box'][n, i] - ch['box'].reshape(-1)).max() <= 1e-9


@pytest.mark.parametrize('k', range(4))
def test_the_turn_commutes_with_the_boxes(k):
    """Boxes computed in the turned page's own frame and then mapped back equal the boxes of the mapped polygon read
    in the turned frame, to 1e-9 px."""
    polys, rec, loc, _, _ = fabricate(20 + k, N=80, nan=0.0)
    H, W = 2480, 1754
    th, tw = (W, H) if k % 2 else (H, W)
    tile = (th - 700, tw - 900, 700, 900)   # y0, x0, h, w: at the turned page's far corner
    turned_polys = polys % np.array([tw, th] * 16)
    a = R.char_boxes(turned_polys, rec, loc, np.zeros(80, np.int32), [(th, tw, 0) + tile], PAD, EOS)
    mapped = np.array([map_back(k, x, y, H, W) for x, y in turned_polys.reshape(-1, 2)]).reshape(-1, 32)
    b = R.char_boxes(mapped, rec, loc, np.zeros(80, np.int32), [(H, W, k) + tile], PAD, EOS)
    assert np.array_equal(a['n_chars'], b['n_chars']) and np.array_equal(a['step'], b['step'])
    for n in range(80):
        for i in range(int(a['n_chars'][n])):
            c = map_back(k, *a['centre'][n, i], H, W)
            assert np.abs(np.subtract(c, b['centre'][n, i])).max() <= 1e-9
            sxx, sxy, syy = a['cov'][n, i]
            want = (syy, -sxy, sxx) if k % 2 else (sxx, sxy, syy)
            assert np.abs(np.subtract(want, b['cov'][n, i])).max() <= 1e-9 * max(1.0, abs(sxx) + abs(syy))
            corners = [map_back(k, x, y, H, W) for x, y in a['box'][n, i].reshape(4, 2)]
            assert np.abs(np.subtract(corners, b['box'][n, i].reshape(4, 2))).max() <= 1e-9


def test_wrapper_refuses_bad_shapes_and_frames():
    from advancedliteratemachinery_b200.omniparser import char_boxes
    polys, rec, loc, fi, frames = fabricate(3, N=10)
    sizes, tiles, turns = frames_to_tiles(frames)
    ok = dict(sizes=sizes, tiles=tiles, polys=polys, rec=rec, loc=loc, tile_index=fi, turns=turns)

    def call(**kw):
        a = dict(ok, **kw)
        return char_boxes(None, a['sizes'], a['tiles'], a['polys'], a['rec'], a['loc'], a['tile_index'], PAD, EOS,
                          turns=a['turns'])

    bad = [dict(rec=rec[0]), dict(polys=polys[:, :30]), dict(polys=polys[:9]), dict(loc=loc[:, :, :4]),
           dict(loc=loc[:9]), dict(tile_index=fi[:9]), dict(tile_index=np.full(10, len(tiles))),
           dict(tile_index=np.full(10, -1)), dict(tile_index=fi.astype(np.float64)),
           dict(rec=np.zeros((10, 0), np.int64), loc=np.zeros((10, 0, 5), np.float32)),
           dict(rec=np.full((10, 1022), PAD), loc=np.zeros((10, 1022, 5), np.float32)),
           dict(turns=np.full(len(turns), 4)), dict(turns=turns[:-1])]
    t = tiles.copy(); t[0, 0] = len(sizes); bad.append(dict(tiles=t))             # page out of range
    t = tiles.copy(); t[0, 3] = 0; bad.append(dict(tiles=t))                      # empty tile
    t = tiles.copy(); t[0, 1] = -1; bad.append(dict(tiles=t))                     # before the page
    t = tiles.copy(); t[0, 2] += 1; t[0, 4] = (sizes[0][0] if turns[0] % 2 else sizes[0][1]) - t[0, 2] + 1
    bad.append(dict(tiles=t))                                                     # past the turned page's edge
    bad.append(dict(sizes=[(0, 10)] + sizes[1:]))                                 # empty page
    for kw in bad:
        with pytest.raises(ValueError):
            call(**kw)


def test_wrapper_frame_check_is_the_kernels():
    """omniparser.char_boxes refuses exactly the frames rec_box_core::valid_frame refuses."""
    from advancedliteratemachinery_b200.omniparser import char_boxes
    lib = emu('rec_box_emu', bind)
    rng = np.random.default_rng(11)
    seen = set()
    for _ in range(1000):   # turns outside 0..3 are check_turns' (test above)
        f = np.array([rng.integers(0, 7), rng.integers(0, 7), rng.integers(0, 4), rng.integers(-1, 3),
                      rng.integers(-1, 3), rng.integers(0, 5), rng.integers(0, 5)], np.int32)
        valid = bool(lib.emu_valid_frame(f.ctypes.data))
        sizes, tiles, turns = frames_to_tiles(f[None])
        try:
            char_boxes(None, sizes, tiles, np.zeros((0, 32)), np.zeros((0, 3), np.int64),
                       np.zeros((0, 3, 5), np.float32), np.zeros(0, np.int32), PAD, EOS, turns=turns)
            accepted = True
        except ValueError:
            accepted = False
        assert accepted == valid, f.tolist()
        seen.add(valid)
    assert seen == {True, False}
