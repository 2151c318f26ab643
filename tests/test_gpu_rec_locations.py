"""GPU: character locations of OmniParser's recognition loop (alm_omni_set_rec_locations / alm_omni_get_rec_locations,
alm_op_rec_locations, the rec_locations keyword of OmniParserB200; DESIGN §4.9).

Op level: the device moments against fp64 moments of the same q and K.  End to end: against the moments of the maps
hooked out of the unmodified reference (tests/golden/omni_rec_maps.npz) -- the ids of every fixture are bit-exact, so
the maps are those of the same greedy steps."""
import os

import numpy as np
import pytest
import torch

from tests.support import omni_model, options, release_models

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

ERR_INVALID, ERR_STATE = -1, -4
CENTRE_TOL = 0.02           # px
COV_REL, COV_ABS = 1e-3, 0.02   # covariance entries: COV_REL * trace + COV_ABS px^2


def _close(got, ref, tag, report=None):
    """got / ref [..., 5] (px): centre within CENTRE_TOL, covariance entries within COV_REL * trace + COV_ABS."""
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    assert np.isfinite(got).all(), tag
    dc = np.abs(got[..., :2] - ref[..., :2]).max()
    tr = ref[..., 2] + ref[..., 4]
    dv = (np.abs(got[..., 2:] - ref[..., 2:]) - (COV_REL * tr[..., None] + COV_ABS)).max()
    if report is not None:
        report[tag] = (float(dc), float(np.abs(got[..., 2:] - ref[..., 2:]).max()))
    assert dc <= CENTRE_TOL and dv <= 0, (tag, dc, dv)


# ----------------------------------------------------------------------------------------------- op level
def _ref_moments(q, k, kpm, key_len, mw, nsplit):
    """fp64 moments of the head-averaged softmax((q_h / 8) K_h^T): q [nimg, Ncap, 512], k [nimg, M, 512]."""
    from oracle.rec_maps_ref import rec_moments
    if nsplit == 1:   # the single-plane kernel sees the bf16 high parts only
        q, k = q.bfloat16(), k.bfloat16()
    q, k = q.double().cpu(), k.double().cpu()
    nimg, Ncap, _ = q.shape
    M = k.shape[1]
    out = np.zeros((nimg, Ncap, 5))
    for i in range(nimg):
        dead = torch.zeros(M, dtype=torch.bool)
        if kpm is not None:
            dead |= kpm[i].cpu().bool()
        dead[key_len[i]:] = True
        s = torch.einsum('nhd,mhd->hnm', q[i].view(Ncap, 8, 64), k[i].view(M, 8, 64)) / 8
        s[:, :, dead] = -float('inf')
        A = torch.softmax(s, -1).mean(0).numpy()                       # [Ncap, M]
        out[i] = rec_moments(A, (M + mw[i] - 1) // mw[i], mw[i])
    return out


def _op(m, q, k, kpm, key_len, mw, q_split):
    nimg, Ncap, _ = q.shape
    out = torch.full((nimg, Ncap, 5), float('nan'), device='cuda')
    kl = None if key_len is None else np.ascontiguousarray(key_len, dtype=np.int32)
    mwa = np.ascontiguousarray(mw, dtype=np.int32)
    m.ctx.check(m.lib.alm_op_rec_locations(m.ctx.h, q.data_ptr(), k.data_ptr(), None if kpm is None else kpm.data_ptr(),
                                           None if kl is None else kl.ctypes.data, mwa.ctypes.data, out.data_ptr(), nimg,
                                           Ncap, k.shape[1], q_split))
    return out.cpu().numpy()


@pytest.fixture(scope='module')
def spot():
    return omni_model(dict(wseed=0, pt_eos_bias=-30.0), workspace_mb=8192)


@pytest.mark.parametrize('nsplit', [3, 1])
@pytest.mark.parametrize('Ncap,q_split', [(1, 0), (64, 1), (70, 1)])
def test_op_against_fp64_moments(spot, nsplit, Ncap, q_split):
    """M = 200 (not a multiple of 64) on a 20-wide grid; image 0: a fully masked 64-key block; image 1: key_len 137
    (NaN beyond it); image 2: a single live key; image 3: scores above 100 on a 13-wide grid."""
    g = torch.Generator(device='cuda').manual_seed(7 + Ncap + nsplit)
    nimg, M = 4, 200
    q = torch.randn(nimg, Ncap, 512, device='cuda', generator=g) * 0.5
    k = torch.randn(nimg, M, 512, device='cuda', generator=g) * 0.5
    q[3] *= 150.0                                                       # |scores| above 100
    kpm = torch.zeros(nimg, M, dtype=torch.uint8, device='cuda')
    kpm[0, 64:128] = 1
    kpm[1, 5] = 1
    key_len = [200, 137, 1, 195]
    mw = [20, 20, 20, 13]
    with options(spot.ctx, nsplit=nsplit):
        got = _op(spot, q, k, kpm, key_len, mw, q_split)
        got2 = _op(spot, q, k, kpm, key_len, mw, q_split)
    assert np.array_equal(got.view(np.uint32), got2.view(np.uint32)), 'not bit-reproducible'
    ref = _ref_moments(q, k, kpm, key_len, mw, nsplit)
    s = torch.einsum('nhd,mhd->hnm', q[3].view(Ncap, 8, 64).double(), k[3].view(M, 8, 64).double()) / 8
    assert float(s.abs().max()) > 100
    np.testing.assert_array_equal(got[2, :, :2], np.broadcast_to([8.0, 8.0], (Ncap, 2)))   # key 0 alone
    np.testing.assert_array_equal(got[2, :, 2:], 0.0)
    report = {}
    _close(got, ref, f'op Ncap={Ncap} nsplit={nsplit}', report)
    print(report)


def test_op_without_key_counts_or_mask(spot):
    g = torch.Generator(device='cuda').manual_seed(3)
    q = torch.randn(2, 16, 512, device='cuda', generator=g)
    k = torch.randn(2, 300, 512, device='cuda', generator=g)
    got = _op(spot, q, k, None, None, [30, 17], 0)
    _close(got, _ref_moments(q, k, None, [300, 300], [30, 17], 3), 'op no mask')


def test_op_rejects_bad_arguments(spot):
    q = torch.zeros(1, 1, 512, device='cuda')
    k = torch.zeros(1, 64, 512, device='cuda')
    out = torch.zeros(1, 1, 5, device='cuda')
    mw = np.array([8], dtype=np.int32)
    lib, h = spot.lib, spot.ctx.h
    assert lib.alm_op_rec_locations(h, q.data_ptr(), k.data_ptr(), None, None, np.array([0], np.int32).ctypes.data,
                                    out.data_ptr(), 1, 1, 64, 0) == ERR_INVALID
    assert lib.alm_op_rec_locations(h, q.data_ptr(), k.data_ptr(), None, np.array([65], np.int32).ctypes.data,
                                    mw.ctypes.data, out.data_ptr(), 1, 1, 64, 0) == ERR_INVALID
    assert lib.alm_op_rec_locations(h, q.cpu().data_ptr(), k.data_ptr(), None, None, mw.ctypes.data, out.data_ptr(), 1,
                                    1, 64, 0) == ERR_INVALID


# ----------------------------------------------------------------------------------------------- end to end
def _seqs(v, canvas):
    return [v.pt_prompt(), torch.tensor([[v.poly_sos_index]]), torch.tensor([[v.rec_sos_index]]), torch.tensor(canvas)]


def _px(loc, size):
    """normalised locations [..., 5] -> px, page size (h, w)"""
    h, w = size
    return np.asarray(loc, np.float64) * np.array([w, h, w * w, w * h, h * h])


@pytest.fixture(scope='module')
def maps_fixture(golden_dir):
    return np.load(os.path.join(golden_dir, 'omni_rec_maps.npz'))


@pytest.mark.parametrize('name', ['full', 'masked', 'oddlen'])
def test_spotting_locations_match_the_reference_maps(spot, name, maps_fixture, golden_dir):
    from advancedliteratemachinery_b200 import NestedTensor
    from oracle.gen_golden import OMNI_CASES, omni_inputs
    case = OMNI_CASES[name]
    v = spot.vocab
    v.pt_seq_length, v.rec_length = case['pt_seq_length'], case['rec_length']
    img, mask = omni_inputs(case)
    size = case.get('image', case['canvas'])
    ref = maps_fixture[f'{name}_moments']
    n = ref.shape[0]
    report, runs = {}, []
    for graphs in (1, 0):
        with options(spot.ctx, use_graphs=graphs):
            out = spot(NestedTensor(img, mask), _seqs(v, case['canvas']), rec_locations=True)
        (pt, poly, rec), _ = out
        assert np.array_equal(rec.numpy()[0], maps_fixture[f'{name}_rec']), name
        loc = spot.last_rec_locations
        assert loc.shape == (1, max(1, v.pt_seq_length // 2), v.rec_length, 5)
        assert not loc[0, n:].any()
        _close(_px(loc[0, :n], size), ref, f'{name} graphs={graphs}', report)
        runs.append(loc)
    assert np.array_equal(runs[0].view(np.uint32), runs[1].view(np.uint32)), 'graphs on / off differ'
    print(report)


def test_kie_locations_match_the_reference_maps(maps_fixture):
    from advancedliteratemachinery_b200 import NestedTensor, OmniParserB200, OmniVocab
    from advancedliteratemachinery_b200 import synthetic as W
    from oracle.gen_golden import KIE_CASES, omni_inputs
    case = KIE_CASES['kie']
    sd = W.omniparser_state_dict(seed=case['wseed'], vie_categories=case['vie'], pt_eos_bias=case['pt_eos_bias'])
    v = OmniVocab(vie_categories=case['vie'], pt_seq_length=case['pt_seq_length'], rec_length=case['rec_length'])
    m = OmniParserB200(sd, v, workspace_mb=8192)
    try:
        img, mask = omni_inputs(case)
        greedy = m(NestedTensor(img, mask), _seqs(v, case['canvas']))
        out = m(NestedTensor(img, mask), _seqs(v, case['canvas']), rec_locations=True, rec_candidates=3)
        assert out == greedy
        raw = m.last_kie_raw
        ref = maps_fixture['kie_moments']
        n = int(raw['n_inst'][0])
        assert n == ref.shape[0] and np.array_equal(raw['rec'][0, :n], maps_fixture['kie_rec'])
        _close(_px(m.last_rec_locations[0, :n], case['canvas']), ref, 'kie')
        assert m.last_rec_candidates is not None
    finally:
        m.ctx.close()


def test_outputs_and_launches_unchanged_by_locations(spot):
    """ids, probabilities, polygons and candidates bit-identical with locations on and off; locations add exactly one
    launch per generated rec step; a get after a decode with locations off is ALM_ERR_STATE."""
    from advancedliteratemachinery_b200 import NestedTensor
    from oracle.gen_golden import OMNI_CASES, omni_inputs
    case = OMNI_CASES['full']
    v = spot.vocab
    v.pt_seq_length, v.rec_length = case['pt_seq_length'], case['rec_length']
    img, mask = omni_inputs(case)

    def run(loc):
        spot(NestedTensor(img, mask), _seqs(v, case['canvas']), rec_candidates=4, rec_locations=loc)  # graphs built
        spot.ctx.launch_count(reset=True)
        out = spot(NestedTensor(img, mask), _seqs(v, case['canvas']), rec_candidates=4, rec_locations=loc)
        return out, spot.ctx.launch_count(), spot.last_rec_candidates, spot.last_rec_locations

    off, n_off, cand_off, loc_off = run(False)
    on, n_on, cand_on, loc_on = run(True)
    assert loc_off is None and loc_on is not None
    for a, b in zip(off[0], on[0]):
        assert torch.equal(a, b)
    assert np.array_equal(off[1][0].numpy().view(np.uint32), on[1][0].numpy().view(np.uint32))
    for a, b in zip(cand_off, cand_on):
        assert np.array_equal(a, b)
    assert n_on - n_off == v.rec_length, (n_on, n_off)
    spot(NestedTensor(img, mask), _seqs(v, case['canvas']))
    buf = np.zeros(loc_on.size, np.float32)
    assert spot.lib.alm_omni_get_rec_locations(spot.ctx.h, buf.ctypes.data, buf.size) == ERR_STATE


def test_prompt_slots_carry_the_locations_of_their_shared_points(spot):
    from advancedliteratemachinery_b200 import NestedTensor
    from oracle.gen_golden import OMNI_CASES, omni_inputs
    case = OMNI_CASES['full']
    v = spot.vocab
    v.pt_seq_length, v.rec_length = case['pt_seq_length'], case['rec_length']
    img, mask = omni_inputs(case)
    spot(NestedTensor(img, mask), _seqs(v, case['canvas']), rec_locations=True)
    single = spot.last_rec_locations
    prompts = torch.cat([v.pt_prompt(), v.pt_prompt()])
    res = spot.decode_prompts(prompts, rec_locations=True)
    loc = spot.last_rec_locations
    assert loc.shape[:2] == (1, 2)
    from advancedliteratemachinery_b200.omniparser import slot_locations
    n = res[0][0][0][0].numel() // 2
    per = slot_locations(np.array([[n, n]]), loc)
    assert np.array_equal(per[0][0], per[0][1]) and np.array_equal(per[0][0], single[0, :n])


def test_beams_and_locations_refuse_each_other(spot):
    lib, h = spot.lib, spot.ctx.h
    spot._set_rec_candidates(0)                      # everything off, whatever earlier tests left on
    assert lib.alm_omni_set_rec_beams(h, 2, 1.0) == 0
    assert lib.alm_omni_set_rec_locations(h, 1) == ERR_INVALID
    assert lib.alm_omni_set_rec_beams(h, 0, 1.0) == 0
    assert lib.alm_omni_set_rec_locations(h, 1) == 0
    assert lib.alm_omni_set_rec_beams(h, 2, 1.0) == ERR_INVALID
    assert lib.alm_omni_set_rec_locations(h, 0) == 0
    spot._rec_loc, spot._rec_beams = False, (0, 1.0)
    with pytest.raises(ValueError):
        spot.decode(rec_beams=2, rec_locations=True)


def test_pages_locations_equal_each_page_alone(spot):
    """forward_pages: every page's locations equal those of the page decoded alone (the same greedy path; the key
    splits of the batch differ, so the sums are compared within the tolerance)."""
    from advancedliteratemachinery_b200 import NestedTensor
    from oracle.gen_golden import OMNI_CASES, omni_inputs
    v = spot.vocab
    v.pt_seq_length, v.rec_length = 8, 25
    pages = [omni_inputs(OMNI_CASES['full'])[0][0], omni_inputs(OMNI_CASES['masked'])[0][0, :, :80, :112]]
    alone = []
    for p in pages:
        out = spot.forward_pages(NestedTensor(p[None].cuda(), torch.zeros(1, *p.shape[1:], dtype=torch.bool).cuda()),
                                 rec_locations=True)
        alone.append((out[0], spot.last_rec_locations[0]))
    t = torch.zeros(2, 3, 96, 128)
    mask = torch.ones(2, 96, 128, dtype=torch.bool)
    for i, p in enumerate(pages):
        t[i, :, :p.shape[1], :p.shape[2]] = p
        mask[i, :p.shape[1], :p.shape[2]] = False
    outs = spot.forward_pages(NestedTensor(t.cuda(), mask.cuda()), rec_locations=True)
    loc = spot.last_rec_locations
    for i, (o, l1) in enumerate(alone):
        assert (o is None) == (outs[i] is None)
        if o is None:
            continue
        assert torch.equal(o[0][2], outs[i][0][2])
        n = o[0][0].numel() // 2
        size = pages[i].shape[1:]
        _close(_px(loc[i, :n], size), _px(l1[:n], size), f'page {i}')


def test_config2_page_locations_match_the_reference(golden_dir, maps_fixture):
    """One 1024 x 1024 page, M = 4 096 keys, 64 instances: on the instances whose ids match the reference fixture the
    moments match; every value is finite and every centroid lies inside the page's grid extent."""
    from advancedliteratemachinery_b200 import NestedTensor, OmniParserB200, OmniVocab
    from oracle.gen_golden import CONFIG2_CASE, config2_page
    from tests.conftest import omni_sd
    case = CONFIG2_CASE
    v = OmniVocab(pt_seq_length=case['pt_seq_length'], rec_length=case['rec_length'])
    m = OmniParserB200(omni_sd(case['wseed'], case['pt_eos_bias']), v, workspace_mb=20480)
    try:
        img, _ = config2_page(case['seed'])
        (pt, poly, rec), _ = m.forward_batch(NestedTensor(img, None), rec_locations=True)[0]
        n = pt.numel() // 2
        loc = _px(m.last_rec_locations[0, :n], (1024, 1024))
        assert np.isfinite(loc).all()
        assert (loc[..., :2] > 0).all() and (loc[..., :2] < 1024).all()
        assert (loc[..., 2] >= 0).all() and (loc[..., 4] >= 0).all()
        ref = maps_fixture['config2_moments']
        same = [i for i in range(min(n, ref.shape[0])) if np.array_equal(rec.numpy()[0, i], maps_fixture['config2_rec'][i])]
        assert len(same) >= 60, len(same)
        report = {}
        _close(loc[same], ref[same], 'config2', report)
        print(report, f'{len(same)} of {n} instances compared')
    finally:
        m.ctx.close()
