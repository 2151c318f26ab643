"""GPU: dense pages read in spatial windows (OmniParserB200.decode_dense, alm_omni_decode_dense,
alm_omni_merge_readings; DESIGN 4.16).  'auto' on a batch where nothing saturates must be decode, launches and bits;
an explicit grid must equal decode_prompts with the same window prompts followed by ownership and the oracle merge; in
a mixed batch the unsaturated pages keep their decode result; the worst case (every window saturated, 16 pages of
1024^2 at the full position table) must decode in a 20 GiB workspace where decode fails; the merge entry must equal
its host emulation in three launches; and every refusal must leave the context usable."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from oracle import dense_ref as D
from tests.support import assert_same, omni_model, release_models
from tests.test_dense_cpu import emu_merge_readings, fabricate

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

ALM_ERR_INVALID = -1  # include/alm_ocr.h
PROB_RTOL = 5e-5  # the poly / rec loops at another batch shape: probabilities differ in the last bits, ids not at all


def model(bias, pt_seq_length=12, workspace_mb=8192):
    """A synthetic checkpoint (seed 0) with pt_eos_bias `bias`; one resident at a time."""
    return omni_model(dict(wseed=0, pt_eos_bias=bias, pt_seq_length=pt_seq_length, rec_length=25),
                      workspace_mb=workspace_mb)


def pages(n, size=64, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(n, 3, size, size, generator=g)


def same_result(a, b, prob_rtol=0.0):
    assert (a is None) == (b is None)
    if a is None:
        return
    for x, y in zip(a[0], b[0]):
        assert torch.equal(x, y)
    if prob_rtol == 0:
        assert torch.equal(a[1][0], b[1][0])
    else:
        np.testing.assert_allclose(a[1][0].numpy(), b[1][0].numpy(), rtol=prob_rtol, atol=0)


def window_oracle(m, outs_prompts, b, nx, ny, iou=0.5):
    """Page b's decode_prompts slots with the (nx, ny) window prompts -> owned rows -> the oracle merge, as a result
    in decode's shape and the window of each row."""
    v = m.vocab
    boxes = D.windows(nx, ny, v.num_bins)
    readings = []
    for w in range(nx * ny):
        r = outs_prompts[b][w]
        rows = []
        if r is not None:
            (pt, poly, rec), (prob,) = r
            pt, poly, rec = pt.numpy().reshape(-1, 2), poly.numpy().reshape(-1, 32), rec.numpy()[0]
            for i in range(pt.shape[0]):
                if D.owns(boxes[w], int(pt[i, 0]), int(pt[i, 1])):
                    rows.append((pt[i], poly[i], rec[i], prob.numpy()[i]))
        readings.append(rows)
    count = np.array([len(r) for r in readings], np.int32)
    offset = (np.cumsum(count) - count).astype(np.int32)
    flat = [x for r in readings for x in r]
    L = v.rec_length
    pts = np.array([x[0] for x in flat], np.float64).reshape(-1, 2)
    polys = np.array([x[1] for x in flat], np.float64).reshape(-1, 32)
    rec = np.array([x[2] for x in flat], np.int64).reshape(-1, L)
    prob = np.array([x[3] for x in flat], np.float32).reshape(-1, L)
    out = D.merge(nx * ny, count, offset, pts, polys, rec, prob, v.recog_pad_index, v.rec_eos_index, iou)
    n = int(out['count'][0])
    if n == 0:
        return None, out['source'][:, 0]
    res = ([torch.from_numpy(out['pts'].astype(np.int64).reshape(1, -1)),
            torch.from_numpy(out['polys'].astype(np.int64).reshape(1, -1)),
            torch.from_numpy(out['rec'][None].copy())], [torch.from_numpy(out['prob'].copy())])
    return res, out['source'][:, 0]


def test_auto_matches_the_reference_fixture(golden_dir):
    """tests/golden/omni_dense.npz (oracle/gen_golden_dense.py, the unmodified reference): level 0 saturates, 2 x 2 has
    windows that end and one that does not, so 'auto' reads the page at 3 x 3; the result is the oracle's merge of the
    reference's owned 3 x 3 rows."""
    import os
    gold = np.load(os.path.join(golden_dir, 'omni_dense.npz'))
    m = model(float(gold['pt_eos_bias'][0]), int(gold['pt_seq_length'][0]))
    g = torch.Generator().manual_seed(int(gold['seed'][0]))
    img = torch.randn(1, 3, *(int(x) for x in gold['canvas']), generator=g)
    m.encode(img.cuda(), torch.zeros(1, *img.shape[2:], dtype=torch.bool).cuda())
    got = m.decode_dense(iou=float(gold['iou'][0]))[0]
    assert m.last_dense.grid[0].tolist() == [3, 3]
    assert m.last_dense.saturated[0].tolist() == gold['sat3'].tolist()
    n = int(gold['merged_count'][0])
    assert got is not None and got[0][0].shape[1] == 2 * n
    (pt, poly, rec), (prob,) = got
    # the fixture clears a 1e-4 top-1 / top-2 gap at every greedy step and every merge decision: ids are bit-exact
    assert np.array_equal(pt.numpy().reshape(-1, 2), gold['merged_pts'].astype(np.int64))
    assert np.array_equal(poly.numpy().reshape(-1, 32), gold['merged_polys'].astype(np.int64))
    assert np.array_equal(rec.numpy()[0], gold['merged_rec'])
    np.testing.assert_allclose(prob.numpy(), gold['merged_prob'], rtol=2e-3, atol=1e-7)
    assert np.array_equal(m.last_dense.window[0], gold['merged_source'][:, 0])


def test_auto_is_decode_when_nothing_saturates():
    m = model(0.45)
    x = pages(4)
    m.encode(x.cuda(), None)
    m.ctx.launch_count(reset=True)
    ref = m.decode()
    n_ref = m.ctx.launch_count(reset=True)
    got = m.decode_dense()
    n_got = m.ctx.launch_count(reset=True)
    assert not m.last_dense.saturated.any()
    assert (m.last_dense.grid == 1).all()
    assert n_got == n_ref
    assert any(r is not None for r in ref)
    for a, b, w in zip(got, ref, m.last_dense.window):
        same_result(a, b)
        assert (w == 0).all()


@pytest.mark.parametrize('grid', [(2, 2), (3, 3), (3, 1), (1, 2)])
def test_explicit_grid_is_decode_prompts_then_ownership_and_the_merge(grid):
    m = model(-1.0)
    v = m.vocab
    x = pages(3, seed=5)
    m.encode(x.cuda(), None)
    nx, ny = grid
    prompts = torch.cat([v.window_prompt()] * (nx * ny))
    for w, box in enumerate(D.windows(nx, ny, v.num_bins)):
        prompts[w, :4] = torch.tensor(box)
    slots = m.decode_prompts(prompts)
    got = m.decode_dense(grid=grid)
    assert (m.last_dense.grid == np.array(grid)).all()
    rows = 0
    for b in range(3):
        want, win = window_oracle(m, slots, b, nx, ny)
        same_result(got[b], want, PROB_RTOL)
        assert np.array_equal(m.last_dense.window[b], win)
        rows += 0 if want is None else want[0][0].shape[1] // 2
    assert rows > 0


def mixed_case(x):
    """The first pt_eos bias of a fixed list under which some but not all of the pages x saturate at level 0 (the
    synthetic checkpoint saturates every page at 0.0 and none at 0.45 with 12 point steps)."""
    for bias in (0.3, 0.2, 0.1, 0.4, 0.05):
        m = model(bias)
        m.encode(x.cuda(), None)
        got = m.decode_dense()
        sat0 = m.last_dense.grid[:, 0] > 1
        if sat0.any() and not sat0.all():
            return m, got, sat0
    pytest.fail('no bias of the list gives a mixed batch')


def test_mixed_batch_rereads_only_the_saturated_pages():
    x = pages(8, seed=9)
    m, got, sat0 = mixed_case(x)
    ref = m.decode()
    for b in range(8):
        if not sat0[b]:
            same_result(got[b], ref[b], PROB_RTOL)
            assert not m.last_dense.saturated[b].any()
        else:
            side = int(m.last_dense.grid[b, 0])
            assert side in (2, 3) and m.last_dense.grid[b, 1] == side
            assert not m.last_dense.saturated[b, side * side:].any()
            if side == 2:
                assert not m.last_dense.saturated[b, :4].any()
    # only the saturated pages are read again: the window point loops cover exactly the pages of each level, each page
    # once per level, and every pass stays within B x max_instances rows
    grids, loops = m.last_dense.grid.copy(), m.last_dense.loops
    for side in (2, 3):
        read = [p for k, i0, n, per in loops if k == 0 and per == side * side for p in range(i0, i0 + n)]
        assert sorted(read) == sorted(np.flatnonzero(grids[:, 0] >= side).tolist()), (side, loops)
    assert set(np.flatnonzero(sat0).tolist()) <= set(p for k, i0, n, _ in loops if k == 0 for p in range(i0, i0 + n))
    maxi = m.vocab.pt_seq_length // 2
    assert all(n * per <= 8 * maxi for k, _, n, per in loops if k == 1)
    # each saturated page read alone gets the grid and the rows it got in the mixed batch
    for b in np.flatnonzero(sat0)[:2]:
        m.encode(x[b:b + 1].cuda(), None)
        one = m.decode_dense()
        assert np.array_equal(m.last_dense.grid[0], grids[b])
        same_ids(one[0], got[b])


def same_ids(a, b):
    assert (a is None) == (b is None)
    if a is not None:
        for x, y in zip(a[0], b[0]):
            assert torch.equal(x, y)


def test_worst_case_every_window_saturates_in_the_bench_workspace():
    m = model(-30.0, pt_seq_length=1024, workspace_mb=20480)
    x = pages(16, size=1024, seed=1)
    m.encode(x.cuda(), None)
    with pytest.raises(RuntimeError):
        m.decode()
    got = m.decode_dense()
    assert (m.last_dense.grid == 3).all()
    assert m.last_dense.saturated.all()
    loops = m.last_dense.loops
    assert [tuple(x) for x in loops if x[0] == 0] == [(0, 0, 16, 4), (0, 0, 16, 9)]   # one batched loop per level
    assert all(n * per <= 16 * 512 for k, _, n, per in loops if k == 1)             # passes within decode's rows
    n = [0 if r is None else r[0][0].shape[1] // 2 for r in got]
    assert 0 < max(n) <= 9 * 509
    assert all(0 <= w.min() and w.max() < 9 for w in m.last_dense.window if len(w))


def test_merge_entry_equals_the_emulation_at_16_pages_x_9_windows():
    from advancedliteratemachinery_b200 import omniparser as O
    m = model(0.45)
    rng = np.random.default_rng(4)
    readings = []
    for p in range(16):
        xy = rng.integers(0, 980, (509, 2))
        for w in range(9):
            j = rng.integers(-2, 3, (509, 4))
            readings.append([(int(a) + j[i, 0], int(b) + j[i, 1], int(a) + 20 + j[i, 2], int(b) + 12 + j[i, 3],
                              float(rng.choice([0.25, 0.5, 1.0]))) for i, (a, b) in enumerate(xy)])
    from tests.test_dense_cpu import rows_of
    rows = rows_of(readings)
    m.ctx.launch_count(reset=True)
    got = O.merge_readings(m.ctx, 9, *rows, m.vocab.recog_pad_index, m.vocab.rec_eos_index)
    assert m.ctx.launch_count(reset=True) == 3
    want = emu_merge_readings(9, *rows, pad=m.vocab.recog_pad_index, eos=m.vocab.rec_eos_index)
    assert_same(got, want)
    assert 0 < int(got['count'].sum()) < int(rows[0].sum())
    # fabricated pages, and the 4-reading case through both entries
    rows = fabricate(rng, 5, 4)
    a = O.merge_readings(m.ctx, 4, *rows, 1096, 1099)
    assert_same(a, O.merge_turns(m.ctx, *rows, 1096, 1099))
    assert_same(a, emu_merge_readings(4, *rows))


def _raw_dense(m, prompt, nx=0, ny=0, iou=0.5, cap=None):
    v = m.vocab
    B = len(m.page_shapes())
    maxi = max(1, v.pt_seq_length // 2)
    cap = maxi * 9 if cap is None else cap
    c1 = max(cap, 1)
    bufs = [np.zeros(B, np.int32), np.zeros((B, c1, 2), np.int64), np.zeros((B, c1, 32), np.int64),
            np.zeros((B, c1, v.rec_length), np.int64), np.zeros((B, c1, v.rec_length), np.float32),
            np.zeros((B, c1), np.int32), np.zeros((B, 2), np.int32), np.zeros((B, 9), np.uint8)]
    p = prompt.reshape(-1).to(torch.long).contiguous()
    return m.lib.alm_omni_decode_dense(m.ctx.h, p.data_ptr(), p.numel(), C.byref(m._cfg(maxi)), nx, ny, iou, cap,
                                       *[b.ctypes.data for b in bufs])


def test_refusals_leave_the_context_usable():
    from advancedliteratemachinery_b200 import OmniParserB200, OmniVocab
    from advancedliteratemachinery_b200 import synthetic as W
    m = model(0.45)
    v = m.vocab
    glob = v.pt_prompt()
    m.encode(pages(2).cuda(), None)
    ok = m.decode_dense()
    cases = [dict(nx=4, ny=1), dict(nx=0, ny=2), dict(nx=1, ny=0), dict(nx=-1, ny=-1), dict(iou=0.0),
             dict(iou=1.5), dict(iou=math.nan), dict(cap=9 * 6 - 1), dict(nx=2, ny=2, cap=4 * 6 - 1)]
    for kw in cases:
        assert _raw_dense(m, glob, **kw) == ALM_ERR_INVALID, kw
        same_result(m.decode_dense()[0], ok[0])
    assert _raw_dense(m, glob, nx=2, ny=2, cap=4 * 6) == 0
    box = glob.clone()
    box[0, 2] = 500
    assert _raw_dense(m, box) == ALM_ERR_INVALID
    same_result(m.decode_dense()[0], ok[0])
    for opt in [dict(rec_candidates=2), dict(rec_beams=2), dict(rec_locations=True)]:
        m._set_rec_candidates(opt.get('rec_candidates', 0), opt.get('rec_beams', 0),
                              locations=opt.get('rec_locations', False))
        assert _raw_dense(m, glob) == ALM_ERR_INVALID, opt
        m._set_rec_candidates(0)
        same_result(m.decode_dense()[0], ok[0])
    with pytest.raises(ValueError):
        m.decode_dense(grid=(4, 4))
    with pytest.raises(ValueError):
        m.decode_dense(iou=0)
    kv = OmniVocab(vie_categories=4, pt_seq_length=9)
    k = OmniParserB200(W.omniparser_state_dict(seed=2, vie_categories=4, pt_eos_bias=-30.0), kv, workspace_mb=1024)
    try:
        k.encode(pages(1).cuda(), None)
        assert _raw_dense(k, kv.pt_prompt()) == ALM_ERR_INVALID   # KIE checkpoint
    finally:
        k.ctx.close()
    same_result(m.decode_dense()[0], ok[0])
