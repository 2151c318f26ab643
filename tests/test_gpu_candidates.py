"""GPU: the k most likely characters at every recognition step (alm_mgpstr_topk / MGPSTRB200.recognize_topk,
alm_omni_set_rec_candidates + alm_omni_get_rec_candidates / the rec_candidates keyword of OmniParserB200).

Candidate 0 must be the greedy output bit for bit; the other candidates must be the top-k of the fp64 softmax of the
logits the same model produces (MGP-STR: the forward's own logits; OmniParser: teacher-forced logits on the decoded
path), with the lowest id first on equal probability."""
import numpy as np
import pytest
import torch

from tests.support import close_models, omni_model, options, release_models
from tests.test_pages_cpu import pages_case, pages_page
from tests.test_prompts_cpu import prompt_case, prompt_page

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

ERR_INVALID, ERR_STATE = -1, -4
MAX_NEAR_TIE_FLIPS = 3   # rec steps per fixture allowed to differ from teacher forcing at a judged near-tie
NEAR_TIE = 1e-4          # logit gap below which two classes are a near-tie (the fixtures' greedy gap floor)


# ----------------------------------------------------------------------------------------------- MGP-STR
def _mgp_case(name):
    from oracle.gen_golden import MGP_CASES, MGP_VARIANT_CASES
    from tests.conftest import mgp_sd
    if name == 'b3':
        case = MGP_CASES['b3']
        return mgp_sd(0), case['seed'], case['batch']
    from advancedliteratemachinery_b200 import synthetic as W
    char_only = name == 'charstr'
    dim, depth, heads = W.MGP_VARIANTS['base' if char_only else name]
    seed = MGP_VARIANT_CASES[name]['seed']
    return W.mgpstr_state_dict(seed=seed, dim=dim, depth=depth, heads=heads, char_only=char_only), seed, 2


def _check_against_fp64(logits, ids, probs, k, tag):
    """ids / probs [B, 27, k] against torch.topk of the fp64 softmax of logits [B, 27, V]"""
    p = torch.softmax(logits.double(), -1)
    ref_p, ref_i = torch.topk(p, min(k + 1, p.shape[-1]), dim=-1)   # ties: compared through the gaps below
    gaps = ref_p[..., :-1] - ref_p[..., 1:]
    sep = torch.ones_like(ref_p[..., :k], dtype=torch.bool)
    sep &= torch.cat([torch.ones_like(gaps[..., :1], dtype=torch.bool), gaps[..., :k - 1] > 1e-6], -1)
    if ref_p.shape[-1] > k:
        sep &= gaps[..., :k] > 1e-6
    ids64 = ids.to(torch.int64)
    assert torch.equal(ids64[sep], ref_i[..., :k][sep]), tag
    mine = p.gather(-1, ids64)   # fp64 probability of the chosen ids
    rel = float(((probs.double() - mine).abs() / mine).max())
    print(f'{tag}: max rel prob error vs fp64 {rel:.2e}, {int((~sep).sum())} near-tied positions')
    assert rel < 1e-6, (tag, rel)
    assert (probs[..., 1:] <= probs[..., :-1]).all(), tag


@pytest.mark.parametrize('name', ['b3', 'tiny', 'charstr'])
def test_mgpstr_topk_candidates(name):
    from advancedliteratemachinery_b200 import MGPSTRB200
    sd, seed, B = _mgp_case(name)
    m = MGPSTRB200(sd)
    try:
        char_only = m.info()['n_a3'] == 1
        img = torch.rand(B, 3, 32, 128, generator=torch.Generator().manual_seed(seed))
        for nsplit in (3, 1):
            m.ctx.set_option('nsplit', nsplit)
            ids1, prob1 = m.recognize(img)
            out = m.forward(img, is_eval=True)
            logits = [out[1]] if char_only else out[1:]
            for k in (1, 5, 8):
                ids, probs = m.recognize_topk(img, k)
                assert ids.shape == (3, B, 27, k) and probs.shape == (3, B, 27, k)
                for h, lg in enumerate(logits):
                    tag = f'{name} nsplit={nsplit} k={k} head={h}'
                    assert torch.equal(ids[h, ..., 0], ids1[h]), tag
                    assert torch.equal(probs[h, ..., 0], prob1[h]), tag   # bit for bit
                    _check_against_fp64(lg, ids[h], probs[h], k, tag)
            if char_only:  # planes 1 and 2 are never written
                k = 4
                ids = np.full((3, B, 27, k), -7, dtype=np.int32)
                probs = np.full((3, B, 27, k), -7.0, dtype=np.float32)
                m.ctx.check(m.lib.alm_mgpstr_topk(m.ctx.h, img.data_ptr(), B, k, ids.ctypes.data, probs.ctypes.data))
                assert (ids[1:] == -7).all() and (probs[1:] == -7.0).all()
                assert (ids[0] >= 0).all()
    finally:
        m.ctx.close()


def test_mgpstr_equal_probabilities_put_the_lower_id_first():
    """Two rows of the char head duplicated: their logits tie exactly, and the lower id is listed first."""
    from advancedliteratemachinery_b200 import MGPSTRB200
    from tests.conftest import mgp_sd
    sd = dict(mgp_sd(0))
    img = torch.rand(3, 3, 32, 128, generator=torch.Generator().manual_seed(5))
    m = MGPSTRB200(sd)
    try:
        top = int(torch.mode(m.recognize(img)[0][0].reshape(-1)).values)   # the most frequent top-1 char id
    finally:
        m.ctx.close()
    wk = [k for k in sd if k.endswith('char_head.weight')][0]
    bk = wk[:-len('weight')] + 'bias'
    for twin in (top - 1, top + 1):   # the duplicate below and above the original id
        if not 0 <= twin < sd[wk].shape[0]:
            continue
        sd2 = dict(sd)
        w, b = sd[wk].clone(), sd[bk].clone()
        w[twin], b[twin] = w[top], b[top]
        sd2[wk], sd2[bk] = w, b
        m = MGPSTRB200(sd2)
        try:
            ids, probs = m.recognize_topk(img, 3)
            ids1, prob1 = m.recognize(img)
            hit = ids1[0] == min(top, twin)
            assert hit.any()
            assert (ids[0, ..., 0][hit] == min(top, twin)).all() and (ids[0, ..., 1][hit] == max(top, twin)).all()
            assert torch.equal(probs[0, ..., 0][hit], probs[0, ..., 1][hit])
            assert torch.equal(ids[0, ..., 0], ids1[0]) and torch.equal(probs[0, ..., 0], prob1[0])
        finally:
            m.ctx.close()


# ----------------------------------------------------------------------------------------------- OmniParser
def _allowed(v, V):
    a = torch.zeros(V, dtype=torch.bool)
    a[v.num_bins:v.recog_pad_index + 1] = True
    a[v.rec_eos_index] = True
    return a


def check_teacher_forced(m, image, xy, rec, ids, probs, report):
    """Candidates of the instances of one image (ids / probs [n, L, k], rec [n, L], xy [n, 2]) against the top-k of the
    softmax over logits[:nsoft] of the teacher-forced rec decoder, restricted to the allowed classes."""
    v = m.vocab
    n, L, k = ids.shape
    seq = torch.cat([torch.as_tensor(xy, dtype=torch.long), torch.full((n, 1), v.rec_sos_index),
                     torch.as_tensor(rec[:, :-1], dtype=torch.long)], 1)
    lg = m.decode_logits(image, 'rec', seq)[:, 2:].double()          # [n, L, V]: step i predicts rec[:, i]
    V = lg.shape[-1]
    nsoft = V - v.vie_categories
    p = torch.softmax(lg[..., :nsoft], -1)
    allowed = _allowed(v, nsoft)
    masked = torch.where(allowed, lg[..., :nsoft], torch.tensor(float('-inf'), dtype=torch.float64))
    ref_v, ref_i = torch.topk(masked, k + 1, dim=-1)
    mine = torch.as_tensor(ids)
    ok = torch.equal(mine, ref_i[..., :k])
    if not ok:   # every differing step must be a near-tie of the teacher-forced logits
        bad = (mine != ref_i[..., :k]).any(-1)
        gaps = ref_v[..., :-1] - ref_v[..., 1:]
        near = (gaps < NEAR_TIE).any(-1)
        assert bool(near[bad].all()), 'candidate ids differ from teacher forcing away from a near-tie'
        report['near_tie_steps'] = report.get('near_tie_steps', 0) + int(bad.sum())
    got = torch.as_tensor(probs).double()
    ref = p.gather(-1, mine.clamp(min=0))
    np.testing.assert_allclose(got.numpy(), ref.numpy(), rtol=5e-5, atol=1e-7)


def assert_candidates_head(rec, prob, cand):
    """candidate 0 == rec / rec_prob bit for bit"""
    ids, probs = cand
    assert np.array_equal(ids[..., 0], rec)
    assert np.array_equal(probs[..., 0].view(np.uint32), prob.view(np.uint32))
    assert (probs[..., 1:] <= probs[..., :-1]).all()


def spot_model(wseed, bias):
    return omni_model(dict(wseed=wseed, pt_eos_bias=bias), workspace_mb=8192)


@pytest.mark.parametrize('k', [1, 4])
def test_omni_full_candidates_match_teacher_forcing_and_graphs(k, golden_dir):
    from advancedliteratemachinery_b200 import NestedTensor
    from oracle.gen_golden import OMNI_CASES, omni_inputs
    case = OMNI_CASES['full']
    m = spot_model(case['wseed'], case['pt_eos_bias'])
    v = m.vocab
    v.pt_seq_length, v.rec_length = case['pt_seq_length'], case['rec_length']
    img, mask = omni_inputs(case)
    seqs = [v.pt_prompt(), torch.tensor([[v.poly_sos_index]]), torch.tensor([[v.rec_sos_index]]),
            torch.tensor(case['canvas'])]
    greedy = m(NestedTensor(img, mask), seqs)
    assert m.last_rec_candidates is None
    out = m(NestedTensor(img, mask), seqs, rec_candidates=k)
    (pt, poly, rec), (probs,) = out
    for x, y in zip(greedy[0], out[0]):
        assert torch.equal(x, y)
    assert torch.equal(greedy[1][0], probs)
    ids, cp = m.last_rec_candidates
    n = pt.numel() // 2
    assert ids.shape == (1, v.pt_seq_length // 2, v.rec_length, k)
    assert not ids[0, n:].any() and not cp[0, n:].any()
    assert_candidates_head(rec[0].numpy(), probs.numpy(), (ids[0, :n], cp[0, :n]))
    from advancedliteratemachinery_b200.omniparser import slot_candidates
    (si, sp), = slot_candidates(np.array([n]), ids, cp)
    assert np.array_equal(si, ids[0, :n]) and np.array_equal(sp, cp[0, :n])
    report = {}
    check_teacher_forced(m, 0, pt.reshape(n, 2), rec[0].numpy(), ids[0, :n], cp[0, :n], report)
    assert report.get('near_tie_steps', 0) <= MAX_NEAR_TIE_FLIPS, report
    # the eager decode (no captured graphs) gives the same bits
    with options(m.ctx, use_graphs=0):
        m.encode(img, mask)
        m.decode(rec_candidates=k)
        ids2, cp2 = m.last_rec_candidates
    assert np.array_equal(ids, ids2) and np.array_equal(cp.view(np.uint32), cp2.view(np.uint32))


@pytest.mark.parametrize('k', [1, 4])
def test_omni_kie_candidates_use_the_kie_softmax(k):
    from advancedliteratemachinery_b200 import NestedTensor, OmniParserB200, OmniVocab
    from advancedliteratemachinery_b200 import synthetic as W
    from oracle.gen_golden import KIE_CASES, omni_inputs
    close_models()
    case = KIE_CASES['kie']
    sd = W.omniparser_state_dict(seed=case['wseed'], vie_categories=case['vie'], pt_eos_bias=case['pt_eos_bias'])
    v = OmniVocab(vie_categories=case['vie'], pt_seq_length=case['pt_seq_length'], rec_length=case['rec_length'])
    m = OmniParserB200(sd, v, workspace_mb=8192)
    try:
        img, mask = omni_inputs(case)
        seqs = [v.pt_prompt(), torch.tensor([[v.poly_sos_index]]), torch.tensor([[v.rec_sos_index]]),
                torch.tensor(case['canvas'])]
        greedy = m(NestedTensor(img, mask), seqs)
        raw0 = {a: b.copy() for a, b in m.last_kie_raw.items()}
        out = m(NestedTensor(img, mask), seqs, rec_candidates=k)
        assert out == greedy
        raw = m.last_kie_raw
        for a in raw0:
            assert np.array_equal(raw0[a], raw[a]), a
        ids, cp = m.last_rec_candidates
        n = int(raw['n_inst'][0])
        assert n > 0
        assert_candidates_head(raw['rec'][0, :n], raw['rec_prob'][0, :n], (ids[0, :n], cp[0, :n]))
        toks, pos = raw['tokens'][0], raw['inst_pos'][0, :n]
        xy = np.stack([toks[pos], toks[pos + 1]], 1)
        report = {}
        check_teacher_forced(m, 0, xy, raw['rec'][0, :n], ids[0, :n], cp[0, :n], report)
        assert report.get('near_tie_steps', 0) <= MAX_NEAR_TIE_FLIPS, report
    finally:
        m.ctx.close()


def _prompt_model(gold):
    m = spot_model(int(gold['wseed'][0]), float(gold['pt_eos_bias'][0]))
    m.vocab.pt_seq_length = int(gold['pt_seq_length'][0])
    m.vocab.rec_length = int(gold['rec_length'][0])
    return m


@pytest.mark.parametrize('k', [1, 4])
def test_omni_prompt_slots_carry_their_points_candidates(k, golden_dir):
    from advancedliteratemachinery_b200.omniparser import slot_candidates
    gold = prompt_case(golden_dir)
    m = _prompt_model(gold)
    prompts = torch.from_numpy(gold['prompts'])
    pages = [prompt_page(gold, b) for b in range(2)]
    imgs, masks = torch.cat([p[0] for p in pages]), torch.cat([p[1] for p in pages])
    m.encode(imgs.cuda(), masks.cuda())
    outs = m.decode_prompts(prompts, rec_candidates=k)
    ids, cp = m.last_rec_candidates
    P = prompts.shape[1]
    assert ids.shape[:2] == (2, P) and ids.shape[-1] == k
    n_inst = np.array([[0 if o is None else o[0][0].numel() // 2 for o in page] for page in outs])
    per_slot = slot_candidates(n_inst, ids, cp)
    report = {}
    for b in range(2):
        for p in range(P):
            o = outs[b][p]
            assert (o is None) == (per_slot[b][p] is None)
            if o is None:
                continue
            (pt, _, rec), (probs,) = o
            assert_candidates_head(rec[0].numpy(), probs.numpy(), per_slot[b][p])
            check_teacher_forced(m, b, pt.reshape(-1, 2), rec[0].numpy(), *per_slot[b][p], report)
    assert report.get('near_tie_steps', 0) <= MAX_NEAR_TIE_FLIPS, report
    # each slot == the single-prompt decode of its page (fp32 GEMV vs tensor-core path: probabilities to 5e-5)
    for b in range(2):
        m.encode(imgs[b:b + 1].cuda(), masks[b:b + 1].cuda())
        for p in range(P):
            alone = m.decode(prompts[b, p][None], rec_candidates=k)[0]
            if alone is None:
                assert per_slot[b][p] is None
                continue
            n = alone[0][0].numel() // 2
            ai, ap = m.last_rec_candidates
            assert np.array_equal(ai[0, :n], per_slot[b][p][0]), (b, p)
            np.testing.assert_allclose(ap[0, :n], per_slot[b][p][1], rtol=5e-5, atol=0)


@pytest.mark.parametrize('k', [1, 4])
def test_omni_mixed_pages_candidates_equal_batch1(k, golden_dir):
    from advancedliteratemachinery_b200 import NestedTensor
    gold = pages_case(golden_dir)
    m = spot_model(int(gold['wseed'][0]), float(gold['pt_eos_bias'][0]))
    m.vocab.pt_seq_length = int(gold['pt_seq_length'][0])
    m.vocab.rec_length = int(gold['rec_length'][0])
    order = [0, 3, 1, 4, 2]
    pages = [pages_page(gold, b) for b in order]
    Hc, Wc = max(p.shape[2] for p in pages), max(p.shape[3] for p in pages)
    t = torch.zeros(len(pages), 3, Hc, Wc)
    mask = torch.ones(len(pages), Hc, Wc, dtype=torch.bool)
    for i, p in enumerate(pages):
        t[i, :, :p.shape[2], :p.shape[3]] = p[0]
        mask[i, :p.shape[2], :p.shape[3]] = False
    outs = m.forward_pages(NestedTensor(t.cuda(), mask.cuda()), rec_candidates=k)
    ids, cp = m.last_rec_candidates
    report = {}
    for i, p in enumerate(pages):
        o = outs[i]
        m.encode(p.cuda(), None)
        alone = m.decode(rec_candidates=k)[0]
        assert (o is None) == (alone is None)
        if o is None:
            continue
        n = o[0][0].numel() // 2
        ai, ap = m.last_rec_candidates
        assert np.array_equal(ai[0, :n], ids[i, :n]), i
        np.testing.assert_allclose(ap[0, :n], cp[i, :n], rtol=1e-5, atol=0)
        assert_candidates_head(o[0][2][0].numpy(), o[1][0].numpy(), (ids[i, :n], cp[i, :n]))
        check_teacher_forced(m, 0, o[0][0].reshape(n, 2), o[0][2][0].numpy(), ids[i, :n], cp[i, :n], report)
    assert report.get('near_tie_steps', 0) <= MAX_NEAR_TIE_FLIPS, report


# ----------------------------------------------------------------------------------------------- off means off
def test_without_candidates_nothing_changes():
    from advancedliteratemachinery_b200 import MGPSTRB200, NestedTensor, OmniParserB200
    from oracle.gen_golden import OMNI_CASES, omni_inputs
    from tests.conftest import mgp_sd
    case = OMNI_CASES['full']
    owner = spot_model(case['wseed'], case['pt_eos_bias'])
    v = owner.vocab
    v.pt_seq_length, v.rec_length = case['pt_seq_length'], case['rec_length']
    img, mask = omni_inputs(case)
    seqs = [v.pt_prompt(), torch.tensor([[v.poly_sos_index]]), torch.tensor([[v.rec_sos_index]]),
            torch.tensor(case['canvas'])]

    def run(model):
        model.encode(img, mask)
        model.ctx.launch_count(reset=True)
        out = model.decode(v.pt_prompt())
        return out, model.ctx.launch_count()

    fresh = OmniParserB200(None, v, workspace_mb=8192, share_from=owner)
    used = OmniParserB200(None, v, workspace_mb=8192, share_from=owner)
    try:
        ref, ref_n = run(fresh)
        used(NestedTensor(img, mask), seqs, rec_candidates=4)
        got, got_n = run(used)   # rec_candidates=0: the context is set back to k = 0
        assert got_n == ref_n
        assert used.last_rec_candidates is None
        for a, b in zip(ref, got):
            for x, y in zip(a[0], b[0]):
                assert torch.equal(x, y)
            assert torch.equal(a[1][0], b[1][0])
        assert used.lib.alm_omni_get_rec_candidates(used.ctx.h, np.zeros(1).ctypes.data, np.zeros(1).ctypes.data,
                                                    1) == ERR_STATE
    finally:
        fresh.ctx.close()
        used.ctx.close()
    img = torch.rand(3, 3, 32, 128, generator=torch.Generator().manual_seed(9))
    a, b = MGPSTRB200(mgp_sd(0)), None
    try:
        b = MGPSTRB200(None, share_from=a)
        a.ctx.launch_count(reset=True)
        ra = a.forward(img, is_eval=True)
        na = a.ctx.launch_count()
        b.recognize_topk(img, 5)
        b.ctx.launch_count(reset=True)
        rb = b.forward(img, is_eval=True)
        assert b.ctx.launch_count() == na
        assert torch.equal(a.last_ids, b.last_ids) and torch.equal(a.last_prob, b.last_prob)
        for x, y in zip(ra[1:], rb[1:]):
            assert torch.equal(x, y)
    finally:
        a.ctx.close()
        if b is not None:
            b.ctx.close()


# ----------------------------------------------------------------------------------------------- errors
def test_error_paths():
    from advancedliteratemachinery_b200 import MGPSTRB200
    from oracle.gen_golden import OMNI_CASES, omni_inputs
    from tests.conftest import mgp_sd
    case = OMNI_CASES['full']
    m = spot_model(case['wseed'], case['pt_eos_bias'])
    v = m.vocab
    v.pt_seq_length, v.rec_length = case['pt_seq_length'], case['rec_length']
    lib, h = m.lib, m.ctx.h
    buf_i, buf_p = np.zeros(1 << 16, dtype=np.int64), np.zeros(1 << 16, dtype=np.float32)
    img, mask = omni_inputs(case)
    m.encode(img, mask)
    for bad in (-1, 9):
        assert lib.alm_omni_set_rec_candidates(h, bad) == ERR_INVALID
        with pytest.raises(ValueError):
            m.decode(rec_candidates=bad)
    m.decode()                                            # a decode without candidates
    assert lib.alm_omni_get_rec_candidates(h, buf_i.ctypes.data, buf_p.ctypes.data, buf_i.size) == ERR_STATE
    m.decode(rec_candidates=2)
    need = m.last_rec_candidates[0].size
    assert lib.alm_omni_get_rec_candidates(h, buf_i.ctypes.data, buf_p.ctypes.data, need - 1) == ERR_INVALID
    assert lib.alm_omni_get_rec_candidates(h, None, buf_p.ctypes.data, need) == ERR_INVALID
    assert lib.alm_omni_get_rec_candidates(h, buf_i.ctypes.data, buf_p.ctypes.data, need) == 0
    assert np.array_equal(buf_i[:need], m.last_rec_candidates[0].reshape(-1))
    x = torch.rand(1, 3, 32, 128)
    ids, probs = np.zeros(27 * 3 * 8, dtype=np.int32), np.zeros(27 * 3 * 8, dtype=np.float32)
    assert lib.alm_mgpstr_topk(h, x.data_ptr(), 1, 2, ids.ctypes.data, probs.ctypes.data) == ERR_STATE
    g = MGPSTRB200(mgp_sd(0))
    try:
        for bad in (0, -1, 9):
            assert g.lib.alm_mgpstr_topk(g.ctx.h, x.data_ptr(), 1, bad, ids.ctypes.data, probs.ctypes.data) == ERR_INVALID
            with pytest.raises(ValueError):
                g.recognize_topk(x, bad)
        assert g.lib.alm_mgpstr_topk(g.ctx.h, x.data_ptr(), 1, 8, ids.ctypes.data, probs.ctypes.data) == 0
    finally:
        g.ctx.close()
