"""GPU: caller character sets of the recognition loop (alm_omni_set_rec_charset / the rec_charset keyword; DESIGN
4.23).

* fixture parity with oracle/gen_golden_charset.py (decode, read_at with per-point sets, decode_kie);
* the full set is no set, bit for bit and launch for launch, through every entry and with candidates, beams and
  locations; turning the setting off restores a context that never had it;
* on synthetic pages under random sets every id and text lies in the set and every step is the argmax over the allowed
  classes of the device's teacher-forced logits; candidates, beams and per-row sets follow the rule;
* the refusals leave the context usable."""
import numpy as np
import pytest
import torch

from tests.support import golden, kw, omni_model, release_models  # noqa: F401

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

ERR_INVALID = -1
NEAR_TIE = 1e-4
DIGITS = '0123456789'
UPPER = 'ABCDEFGHIJKLMNOPQRSTUVWXYZ'


def spot(case='full'):
    from oracle.gen_golden import OMNI_CASES, omni_inputs
    c = OMNI_CASES[case]
    m = omni_model(c)
    img, mask = omni_inputs(c)
    m.encode(img, mask)
    return m, img, mask


def kie():
    from oracle.gen_golden import KIE_CASES, omni_inputs
    c = KIE_CASES['kie']
    m = omni_model(c, kie=True)
    img, mask = omni_inputs(c)
    m.encode(img, mask)
    return m, c


def bits(a):
    a = np.ascontiguousarray(a.numpy() if isinstance(a, torch.Tensor) else a)
    return a.view(np.uint32) if a.dtype == np.float32 else a


def same(a, b, what=''):
    if isinstance(a, dict):
        assert a.keys() == b.keys(), what
        for k in a:
            same(a[k], b[k], f'{what}.{k}')
    elif isinstance(a, (tuple, list)):
        assert len(a) == len(b), what
        for i, (x, y) in enumerate(zip(a, b)):
            same(x, y, f'{what}[{i}]')
    elif isinstance(a, (np.ndarray, torch.Tensor)):
        assert a.shape == b.shape and np.array_equal(bits(a), bits(b)), what
    else:
        assert a == b, what


def counted(m, fn):
    m.ctx.launch_count(reset=True)
    out = fn()
    return out, m.ctx.launch_count()


def allowed_ids(v, text):
    ids = {v.recog_pad_index - 1, v.recog_pad_index, v.rec_eos_index}
    return ids | {v.num_bins + v.chars.index(c) for c in (text or v.chars)}


def text_of(v, row):
    out = []
    for t in row.tolist():
        if t in (v.recog_pad_index, v.rec_eos_index):
            break
        if t != v.recog_pad_index - 1:
            out.append(v.chars[t - v.num_bins])
    return ''.join(out)


# ----------------------------------------------------------------------------------------------- fixture parity
def test_decode_matches_the_fixture_under_each_set():
    gold = golden('omni_charset.npz')
    m, _, _ = spot()
    for name, text in zip(gold['set_names'].tolist(), gold['sets'].tolist()):
        n, pt, _, rec, prob = m._decode_arrays(None, rec_charset=text or None)
        k = int(n[0])
        assert np.array_equal(pt[0, :k], gold['decode_pts']), name
        assert np.array_equal(rec[0, :k], gold[f'decode_{name}_rec']), name
        np.testing.assert_allclose(prob[0, :k], gold[f'decode_{name}_probs'], rtol=2e-3, atol=1e-7)


def test_read_at_with_per_point_sets_matches_the_fixture():
    gold = golden('omni_charset.npz')
    m, _, _ = spot()
    sets = [None if none else t for t, none in zip(gold['at_sets'].tolist(), gold['at_none'].tolist())]
    n, _, _, rec, prob = m._read_at_arrays([gold['at_pts']], rec_charset=[sets])
    assert np.array_equal(rec[0, :4], gold['at_rec'])
    np.testing.assert_allclose(prob[0, :4], gold['at_probs'], rtol=2e-3, atol=1e-7)


def test_decode_kie_matches_the_fixture_under_digits():
    gold = golden('omni_charset.npz')
    m, c = kie()
    n_inst, pos, _, rec, prob, n_tok, toks, _ = m._decode_kie_arrays(None, rec_charset=DIGITS)
    k = int(n_inst[0])
    got_pts = np.stack([toks[0, pos[0, :k]], toks[0, pos[0, :k] + 1]], 1)
    assert np.array_equal(got_pts, gold['kie_pts'])
    assert np.array_equal(rec[0, :k], gold['kie_rec'])
    np.testing.assert_allclose(prob[0, :k], gold['kie_probs'], rtol=2e-3, atol=1e-7)


# ----------------------------------------------------------------------------------------------- full set == no set
def test_full_set_is_no_set_through_every_entry():
    m, img, mask = spot()
    v = m.vocab
    full = v.chars
    extras = [dict(), dict(rec_candidates=5), dict(rec_beams=1), dict(rec_beams=4, length_penalty=0.5),
              dict(rec_locations=True), dict(rec_candidates=3, rec_locations=True)]

    def lists():
        return m.last_rec_candidates, m.last_rec_beams, m.last_rec_locations

    for ex in extras:
        a, na = counted(m, lambda: (m._decode_arrays(None, **ex), lists()))
        b, nb = counted(m, lambda: (m._decode_arrays(None, rec_charset=full, **ex), lists()))
        same(a, b, f'decode {ex}')
        assert na == nb, ex
        pts = [a[0][1][0, :int(a[0][0][0])]]
        a, na = counted(m, lambda: (m._read_at_arrays(pts, **ex), lists()))
        b, nb = counted(m, lambda: (m._read_at_arrays(pts, rec_charset=[[full] * len(pts[0])], **ex), lists()))
        same(a, b, f'read_at {ex}')
        assert na == nb, ex
    prompts = v.pt_prompt().reshape(1, -1).repeat(2, 1)
    a, na = counted(m, lambda: m.decode_prompts(prompts, rec_candidates=2))
    b, nb = counted(m, lambda: m.decode_prompts(prompts, rec_candidates=2, rec_charset=full))
    same(a, b, 'decode_prompts')
    assert na == nb
    # decode_kie
    k, _ = kie()
    a, na = counted(k, lambda: k._decode_kie_arrays(None, rec_beams=2))
    b, nb = counted(k, lambda: k._decode_kie_arrays(None, rec_beams=2, rec_charset=k.vocab.chars))
    same(a, b, 'decode_kie')
    assert na == nb


def test_full_set_is_no_set_for_decode_dense_on_the_dense_fixture():
    gold = golden('omni_dense.npz')
    m = omni_model(dict(wseed=0, pt_eos_bias=float(gold['pt_eos_bias'][0]),
                        pt_seq_length=int(gold['pt_seq_length'][0]), rec_length=25), workspace_mb=8192)
    g = torch.Generator().manual_seed(int(gold['seed'][0]))
    img = torch.randn(1, 3, *(int(x) for x in gold['canvas']), generator=g)
    m.encode(img.cuda(), torch.zeros(1, *img.shape[2:], dtype=torch.bool).cuda())
    a, na = counted(m, lambda: m._decode_dense_arrays(iou=float(gold['iou'][0])))
    b, nb = counted(m, lambda: m._decode_dense_arrays(iou=float(gold['iou'][0]), rec_charset=m.vocab.chars))
    same(a, b, 'decode_dense')
    assert na == nb
    assert m.last_dense.grid[0].tolist() == [3, 3]
    n, _, _, rec, _ = m._decode_dense_arrays(iou=float(gold['iou'][0]), rec_charset=DIGITS)
    ok = allowed_ids(m.vocab, DIGITS)
    assert set(rec[0, :int(n[0])].reshape(-1).tolist()) <= ok


def test_full_set_is_no_set_for_spot_tiled_whole_page_and_read_regions():
    gold = golden('omni_tiles.npz')
    m = omni_model(gold)
    page = gold['page']
    full = m.vocab.chars
    a, na = counted(m, lambda: m.spot_tiled([page], whole_page=True, **kw(gold)))
    b, nb = counted(m, lambda: m.spot_tiled([page], whole_page=True, rec_charset=full, **kw(gold)))
    same(a, b, 'spot_tiled')
    assert na == nb
    pts = np.array([[d['pts'][0][0], d['pts'][0][1]] for d in a[0]], np.float64)
    pi = np.zeros(len(pts), np.int64)
    for orientation in ('upright', 'auto'):
        a, na = counted(m, lambda: m.read_regions([page], pts, pi, kind='point', orientation=orientation,
                                                   rec_candidates=2, **kw(gold)))
        ca = m.last_rec_candidates
        b, nb = counted(m, lambda: m.read_regions([page], pts, pi, kind='point', orientation=orientation,
                                                   rec_candidates=2, rec_charset=[full] * len(pts), **kw(gold)))
        same(a, b, f'read_regions {orientation}')
        same(ca, m.last_rec_candidates, 'read_regions candidates')
        assert na == nb


def test_turning_the_setting_off_restores_a_fresh_context():
    from advancedliteratemachinery_b200 import OmniParserB200
    from oracle.gen_golden import OMNI_CASES, omni_inputs
    c = OMNI_CASES['full']
    owner = omni_model(c)
    img, mask = omni_inputs(c)
    fresh = OmniParserB200(None, owner.vocab, workspace_mb=4096, share_from=owner)
    used = OmniParserB200(None, owner.vocab, workspace_mb=4096, share_from=owner)
    try:
        for mdl in (fresh, used):
            mdl.encode(img, mask)
        used._decode_arrays(None, rec_charset=DIGITS, rec_candidates=3)
        used._read_at_arrays([np.array([[5, 9], [700, 80]])], rec_charset=[[UPPER, None]])
        a, na = counted(fresh, lambda: fresh._decode_arrays(None))
        b, nb = counted(used, lambda: used._decode_arrays(None))
        same(a, b, 'off')
        assert na == nb
    finally:
        fresh.ctx.close()
        used.ctx.close()


# ----------------------------------------------------------------------------------------------- the rule on synthetic pages
def random_sets(v, n, seed):
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        k = int(rng.integers(1, 12))
        out.append(''.join(rng.choice(list(v.chars), k, replace=False)))
    return out


def page_points(m, n, seed):
    rng = np.random.default_rng(seed)
    return rng.integers(0, m.vocab.num_bins, (n, 2)).astype(np.int32)


@pytest.mark.parametrize('seed', [0, 1, 2])
def test_every_step_is_the_argmax_over_the_allowed_set_of_teacher_forced_logits(seed):
    m, _, _ = spot()
    v = m.vocab
    sets = random_sets(v, 4, seed) + [DIGITS, UPPER]
    pts = page_points(m, len(sets), 100 + seed)
    n, _, _, rec, prob = m._read_at_arrays([pts], rec_charset=[sets])
    for i, text in enumerate(sets):
        ok = allowed_ids(v, text)
        assert set(rec[0, i].tolist()) <= ok, (i, text)
        assert set(text_of(v, rec[0, i])) <= set(text)
        seq = torch.cat([torch.tensor([[pts[i, 0], pts[i, 1], v.rec_sos_index]]), torch.from_numpy(rec[0, i:i + 1])], 1)
        lg = m.decode_logits(0, 'rec', seq)[0].double()
        mask = torch.zeros(lg.shape[-1], dtype=torch.bool)
        mask[sorted(ok)] = True
        for t in range(v.rec_length):
            row = lg[2 + t].masked_fill(~mask, float('-inf'))
            top = row.topk(2)
            if float(top.values[0] - top.values[1]) < NEAR_TIE:
                continue
            assert int(top.indices[0]) == int(rec[0, i, t]), (i, t)
            p = torch.softmax(lg[2 + t], -1)[int(rec[0, i, t])]   # not renormalised over the set
            assert abs(float(p) - float(prob[0, i, t])) <= 2e-3 * float(p) + 1e-7, (i, t)


def test_candidates_and_beams_stay_in_the_set():
    m, _, _ = spot()
    v = m.vocab
    ok = allowed_ids(v, DIGITS + '.')
    n, _, _, rec, prob = m._decode_arrays(None, rec_candidates=6, rec_charset=DIGITS + '.')
    ids, probs = m.last_rec_candidates
    k = int(n[0])
    assert np.array_equal(ids[0, :k, :, 0], rec[0, :k]) and np.array_equal(bits(probs[0, :k, :, 0]), bits(prob[0, :k]))
    assert set(ids[0, :k].reshape(-1).tolist()) <= ok
    m._decode_arrays(None, rec_candidates=6, rec_charset='7')   # 4 allowed classes: the other 2 are (-1, 0)
    ids7, probs7 = m.last_rec_candidates
    assert (ids7[0, :k, :, :4] >= 0).all() and (ids7[0, :k, :, 4:] == -1).all() and (probs7[0, :k, :, 4:] == 0).all()
    assert set(ids7[0, :k, :, :4].reshape(-1).tolist()) == allowed_ids(v, '7')
    _, _, _, rec1, prob1 = m._decode_arrays(None, rec_beams=1, rec_charset=DIGITS + '.')
    for i in range(k):   # W = 1 is greedy up to the terminal token
        row = rec[0, i].tolist()
        end = next((j for j, t in enumerate(row) if t in (v.recog_pad_index, v.rec_eos_index)), len(row) - 1)
        assert rec1[0, i, :end + 1].tolist() == row[:end + 1]
        assert np.array_equal(bits(prob1[0, i, :end + 1]), bits(prob[0, i, :end + 1]))
    m._decode_arrays(None, rec_beams=4, rec_charset=DIGITS + '.')
    bids = m.last_rec_beams[0][0, :k]
    assert set(bids[bids >= 0].tolist()) <= ok
    _, _, _, recl, _ = m._decode_arrays(None, rec_locations=True, rec_charset=DIGITS + '.')
    assert np.array_equal(recl, rec)


def test_read_at_per_point_sets_equal_each_set_read_alone():
    """More points than max_instances (4): the row sets are sliced across read_at's calls."""
    m, _, _ = spot()
    v = m.vocab
    pts = page_points(m, 11, 7)
    sets = [DIGITS, UPPER, None, 'xyz', DIGITS, None, UPPER, 'ab', DIGITS, 'q', UPPER]
    n, _, _, rec, prob = m._read_at_arrays([pts], rec_charset=[sets])
    assert rec.shape[1] >= 11
    for text in set(sets):
        rows = [i for i, s in enumerate(sets) if s == text]
        _, _, _, r1, p1 = m._read_at_arrays([pts[rows]], rec_charset=text)
        assert np.array_equal(r1[0, :len(rows)], rec[0, rows]), text
        np.testing.assert_allclose(p1[0, :len(rows)], prob[0, rows], rtol=5e-5, atol=0)
        if text:
            assert all(set(text_of(v, rec[0, i])) <= set(text) for i in rows)


def test_readers_keep_every_text_in_its_set():
    gold = golden('omni_tiles.npz')
    m = omni_model(gold)
    page = gold['page']
    for orientation in ('upright', 'auto', 'mixed'):
        for d in m.spot_tiled([page], orientation=orientation, rec_charset=UPPER, **kw(gold))[0]:
            assert set(d['rec']) <= set(UPPER), orientation
    words = m.spot_tiled([page], **kw(gold))[0]
    pts = np.array([d['pts'][0] for d in words], np.float64)
    sets = [[DIGITS, None, UPPER, 'mN'][i % 4] for i in range(len(pts))]
    for orientation in ('upright', 'auto'):
        got = m.read_regions([page], pts, np.zeros(len(pts), np.int64), kind='point', orientation=orientation,
                             rec_charset=sets, **kw(gold))
        free = m.read_regions([page], pts, np.zeros(len(pts), np.int64), kind='point', orientation=orientation,
                              **kw(gold))
        for g, f, s in zip(got, free, sets):
            if s is None:
                assert g == f, orientation
            else:
                assert set(g['rec']) <= set(s), (orientation, g['rec'], s)
    kg = golden('omni_kie_tiles.npz')
    k = omni_model(kg, kie=True)
    for ent in k.kie_tiled([kg['page']], rec_charset=DIGITS, **kw(kg))[0]:
        assert set(ent[0]) <= set(DIGITS + ' ')


# ----------------------------------------------------------------------------------------------- refusals
def test_refusals_leave_the_context_usable():
    m, _, _ = spot()
    v = m.vocab
    ref = m._decode_arrays(None)
    lib, h = m.lib, m.ctx.h
    one = np.zeros((1, 95), np.uint8)
    one[0, 3] = 1
    empty = np.zeros((2, 95), np.uint8)
    empty[0, 1] = 1
    rows = np.array([0, 1], np.int32)
    assert lib.alm_omni_set_rec_charset(h, empty.ctypes.data, 2, 95, None, 0) == ERR_INVALID   # an empty set
    assert lib.alm_omni_set_rec_charset(h, one.ctypes.data, 1, 95, rows.ctypes.data, 2) == ERR_INVALID  # index 1
    assert lib.alm_omni_set_rec_charset(h, one.ctypes.data, 65537, 95, None, 0) == ERR_INVALID
    assert lib.alm_omni_set_rec_charset(h, None, 1, 95, None, 0) == ERR_INVALID
    assert lib.alm_omni_set_rec_charset(h, one.ctypes.data, 1, 95, rows.ctypes.data, 0) == ERR_INVALID
    # checked by the decode, before any device work
    cfg = m._cfg(max(1, v.pt_seq_length // 2))
    prompt = m._prompt(None)
    out = [np.zeros((1, 64, 2), np.int64), np.zeros((1, 64, 32), np.int64), np.zeros((1, 64, v.rec_length), np.int64)]
    n_inst, prob = np.zeros(1, np.int32), np.zeros((1, 64, v.rec_length), np.float32)
    import ctypes as C

    def decode():
        return lib.alm_omni_decode(h, prompt.data_ptr(), prompt.numel(), C.byref(cfg), n_inst.ctypes.data,
                                   out[0].ctypes.data, out[1].ctypes.data, out[2].ctypes.data, prob.ctypes.data)
    short = np.ones((1, 94), np.uint8)
    assert lib.alm_omni_set_rec_charset(h, short.ctypes.data, 1, 94, None, 0) == 0
    assert decode() == ERR_INVALID                       # n_chars != recog_pad - num_bins - 1
    r = np.zeros(1, np.int32)
    assert lib.alm_omni_set_rec_charset(h, one.ctypes.data, 1, 95, r.ctypes.data, 1) == 0
    assert decode() == ERR_INVALID                       # row sets belong to decode_at
    xy, cnt = np.zeros((1, 4, 2), np.int32), np.ones(1, np.int32)
    poly, rec = np.zeros((1, 4, 32), np.int64), np.zeros((1, 4, v.rec_length), np.int64)
    rp = np.zeros((1, 4, v.rec_length), np.float32)
    assert lib.alm_omni_decode_at(h, xy.ctypes.data, cnt.ctypes.data, 4, C.byref(cfg), poly.ctypes.data,
                                  rec.ctypes.data, rp.ctypes.data) == ERR_INVALID   # n_rows != B * cap
    m._rec_cs = True   # set behind the adapter's back: its next call turns it off
    # Python refusals: before any device work
    with pytest.raises(ValueError):
        m._decode_arrays(None, rec_charset='')
    with pytest.raises(ValueError):
        m._decode_arrays(None, rec_charset='0é')
    with pytest.raises(ValueError):
        m._read_at_arrays([np.zeros((2, 2), np.int32)], rec_charset=[[DIGITS]])
    with pytest.raises(ValueError):
        m.spot_tiled([np.zeros((64, 64, 3), np.uint8)], rec_charset=[DIGITS])
    same(m._decode_arrays(None), ref, 'after the refusals')
