"""GPU: recognition beam search (alm_omni_set_rec_beams / alm_omni_get_rec_beams, the rec_beams keyword of
OmniParserB200, alm_op_beam_select, alm_op_self_attention_step_anc).

W = 1 must be the greedy decode bit for bit up to each instance's first terminal token; every returned hypothesis must
be what the same model's teacher-forced logits say it is (step probabilities, score); the n-best list of a page must
not depend on what else is in the batch; the op-level kernels are checked against fp64."""
import math

import numpy as np
import pytest
import torch

from tests.beam_ref import beam_rec
from tests.support import close_models, omni_model, options, release_models
from tests.test_pages_cpu import pages_case, pages_page
from tests.test_prompts_cpu import prompt_case, prompt_page

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

ERR_INVALID, ERR_STATE = -1, -4
NEAR_TIE = 1e-4   # selection / ranking margin below which the oracle's order is not compared


def spot_model(wseed, bias):
    return omni_model(dict(wseed=wseed, pt_eos_bias=bias), workspace_mb=8192)


def _terminal_end(v, row):
    """index after the first rec_eos / recog_pad of a rec row (its length when there is none)"""
    for i, c in enumerate(row.tolist()):
        if c in (v.rec_eos_index, v.recog_pad_index):
            return i + 1
    return len(row)


def _assert_greedy_prefix(v, rec_g, prob_g, rec_b, prob_b, tag):
    """rec [..., L]: the W = 1 decode equals greedy bit for bit up to and including the first terminal token"""
    rg, pg = rec_g.reshape(-1, rec_g.shape[-1]), prob_g.reshape(-1, rec_g.shape[-1])
    rb, pb = rec_b.reshape(rg.shape), prob_b.reshape(rg.shape)
    for i in range(rg.shape[0]):
        e = _terminal_end(v, rg[i])
        assert np.array_equal(rb[i, :e], rg[i, :e]), (tag, i)
        assert np.array_equal(pb[i, :e].view(np.uint32), pg[i, :e].view(np.uint32)), (tag, i)
        assert (rb[i, e:] == v.recog_pad_index).all() and (pb[i, e:] == 0).all(), (tag, i)


def _full_case(m):
    from oracle.gen_golden import OMNI_CASES, omni_inputs
    case = OMNI_CASES['full']
    v = m.vocab
    v.pt_seq_length, v.rec_length = case['pt_seq_length'], case['rec_length']
    return omni_inputs(case)


def _full_model():
    from oracle.gen_golden import OMNI_CASES
    case = OMNI_CASES['full']
    return spot_model(case['wseed'], case['pt_eos_bias'])


def _decode_raw(m, rec_beams=0, rec_candidates=0, length_penalty=1.0):
    """decode() outputs as arrays: n_inst [B], pt [B, maxi, 2], rec / prob [B, maxi, L]"""
    outs = m.decode(rec_candidates=rec_candidates, rec_beams=rec_beams, length_penalty=length_penalty)
    v = m.vocab
    maxi = max(1, v.pt_seq_length // 2)
    B = len(outs)
    n_inst = np.zeros(B, dtype=np.int64)
    pt = np.zeros((B, maxi, 2), dtype=np.int64)
    rec = np.zeros((B, maxi, v.rec_length), dtype=np.int64)
    prob = np.zeros((B, maxi, v.rec_length), dtype=np.float32)
    for b, o in enumerate(outs):
        if o is None:
            continue
        n = o[0][0].numel() // 2
        n_inst[b] = n
        pt[b, :n] = o[0][0].reshape(n, 2).numpy()
        rec[b, :n] = o[0][2][0].numpy()
        prob[b, :n] = o[1][0].numpy()
    return n_inst, pt, rec, prob


# ----------------------------------------------------------------------------------------------- W = 1
@pytest.mark.parametrize('graphs', [1, 0])
def test_width_one_is_greedy_on_the_full_and_masked_fixtures(graphs):
    from oracle.gen_golden import OMNI_CASES, omni_inputs
    for name in ('full', 'masked'):
        case = OMNI_CASES[name]
        m = spot_model(case['wseed'], case['pt_eos_bias'])
        v = m.vocab
        v.pt_seq_length, v.rec_length = case['pt_seq_length'], case['rec_length']
        img, mask = omni_inputs(case)
        with options(m.ctx, use_graphs=graphs):
            m.encode(img, mask)
            n, _, rec, prob = _decode_raw(m)
            assert m.last_rec_beams is None
            n1, _, rec1, prob1 = _decode_raw(m, rec_beams=1)
        assert np.array_equal(n, n1) and n.sum() > 0
        _assert_greedy_prefix(v, rec, prob, rec1, prob1, name)
        ids, bp, sc = m.last_rec_beams
        assert ids.shape == rec.shape[:2] + (1, v.rec_length) and sc.shape == rec.shape[:2] + (1,)
        assert np.array_equal(ids[:, :, 0], rec1) and np.array_equal(bp[:, :, 0], prob1)
        for b in range(len(n)):
            assert not ids[b, n[b]:].any() and not sc[b, n[b]:].any()


def test_width_one_is_greedy_for_kie():
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
        m(NestedTensor(img, mask), seqs)
        raw0 = {a: b.copy() for a, b in m.last_kie_raw.items()}
        m(NestedTensor(img, mask), seqs, rec_beams=1)
        raw = m.last_kie_raw
        n = int(raw['n_inst'][0])
        assert n > 0
        for a in ('n_tok', 'tokens', 'probs', 'n_inst', 'inst_pos', 'poly'):
            assert np.array_equal(raw0[a], raw[a]), a
        _assert_greedy_prefix(v, raw0['rec'][0, :n], raw0['rec_prob'][0, :n], raw['rec'][0, :n], raw['rec_prob'][0, :n],
                              'kie')
        # W = 4 on the KIE softmax: every hypothesis against teacher forcing over logits[:V - vie]
        m(NestedTensor(img, mask), seqs, rec_beams=4)
        raw = m.last_kie_raw
        toks, pos = raw['tokens'][0], raw['inst_pos'][0, :n]
        xy = np.stack([toks[pos], toks[pos + 1]], 1)
        ids, bp, sc = m.last_rec_beams
        _check_hypotheses(m, 0, xy, ids[0, :n], bp[0, :n], sc[0, :n], 1.0)
    finally:
        m.ctx.close()


def test_width_one_is_greedy_for_prompts_and_mixed_pages(golden_dir):
    from advancedliteratemachinery_b200 import NestedTensor
    gold = prompt_case(golden_dir)
    m = spot_model(int(gold['wseed'][0]), float(gold['pt_eos_bias'][0]))
    v = m.vocab
    v.pt_seq_length, v.rec_length = int(gold['pt_seq_length'][0]), int(gold['rec_length'][0])
    prompts = torch.from_numpy(gold['prompts'])
    pages = [prompt_page(gold, b) for b in range(2)]
    imgs, masks = torch.cat([p[0] for p in pages]), torch.cat([p[1] for p in pages])
    m.encode(imgs.cuda(), masks.cuda())

    def flat(outs):
        return [(o[0][2][0].numpy(), o[1][0].numpy()) if o is not None else None for page in outs for o in page]
    g = flat(m.decode_prompts(prompts))
    b1 = flat(m.decode_prompts(prompts, rec_beams=1))
    assert sum(x is not None for x in g) > 0
    for x, y in zip(g, b1):
        assert (x is None) == (y is None)
        if x is not None:
            _assert_greedy_prefix(v, x[0], x[1], y[0], y[1], 'prompts')
    gold = pages_case(golden_dir)
    m = spot_model(int(gold['wseed'][0]), float(gold['pt_eos_bias'][0]))
    v = m.vocab
    v.pt_seq_length, v.rec_length = int(gold['pt_seq_length'][0]), int(gold['rec_length'][0])
    pages = [pages_page(gold, b) for b in (0, 3, 1, 4, 2)]
    Hc, Wc = max(p.shape[2] for p in pages), max(p.shape[3] for p in pages)
    t = torch.zeros(len(pages), 3, Hc, Wc)
    mask = torch.ones(len(pages), Hc, Wc, dtype=torch.bool)
    for i, p in enumerate(pages):
        t[i, :, :p.shape[2], :p.shape[3]] = p[0]
        mask[i, :p.shape[2], :p.shape[3]] = False
    og = m.forward_pages(NestedTensor(t.cuda(), mask.cuda()))
    ob = m.forward_pages(NestedTensor(t.cuda(), mask.cuda()), rec_beams=1)
    for x, y in zip(og, ob):
        assert (x is None) == (y is None)
        if x is not None:
            _assert_greedy_prefix(v, x[0][2][0].numpy(), x[1][0].numpy(), y[0][2][0].numpy(), y[1][0].numpy(), 'pages')


# ----------------------------------------------------------------------------------------------- step 0
@pytest.mark.parametrize('width', [2, 5, 8])
def test_step_zero_takes_the_top_w_classes(width):
    """rec_length 1: the W hypotheses are the step-0 children, ranked by probability: the candidates' top-W"""
    m = _full_model()
    img, mask = _full_case(m)
    v = m.vocab
    v.rec_length = 1
    try:
        m.encode(img, mask)
        m.decode(rec_candidates=width)
        ci, cp = m.last_rec_candidates
        m.decode(rec_beams=width, length_penalty=0.0)
        ids, bp, sc = m.last_rec_beams
    finally:
        v.rec_length = 25
    assert np.array_equal(ids[..., 0], ci[..., 0, :])
    # W > 1 runs the W rows of an instance through the tensor-core decoder path, a single greedy row per image takes the
    # fp32 GEMV path: the logits agree to fp32 rounding, not bit for bit (W = 1 stays on the greedy path: bit for bit)
    np.testing.assert_allclose(bp[..., 0], cp[..., 0, :], rtol=5e-5, atol=0)
    live = ci[..., 0, 0] > 0
    np.testing.assert_allclose(sc[live], np.log(cp[..., 0, :][live].astype(np.float64)), rtol=0, atol=1e-4)


# ----------------------------------------------------------------------------------------------- hypotheses
def _check_hypotheses(m, image, xy, ids, probs, scores, alpha):
    """ids / probs [n, W, L], scores [n, W] of one image against the teacher-forced rec decoder: per-step probability
    = fp64 softmax over logits[:nsoft] of the chosen token; score = sum of their logs up to the terminal token;
    hypotheses distinct and ranked by score / len^alpha."""
    v = m.vocab
    n, Wd, L = ids.shape
    live = np.isfinite(scores) & (ids[..., 0] >= 0)
    seq = torch.cat([torch.as_tensor(np.repeat(xy, Wd, 0), dtype=torch.long),
                     torch.full((n * Wd, 1), v.rec_sos_index),
                     torch.as_tensor(np.where(ids < 0, v.recog_pad_index, ids).reshape(n * Wd, L)[:, :-1])], 1)
    lg = m.decode_logits(image, 'rec', seq)[:, 2:].double()
    nsoft = lg.shape[-1] - v.vie_categories
    p = torch.softmax(lg[..., :nsoft], -1).reshape(n, Wd, L, nsoft).numpy()
    for i in range(n):
        keys, seen = [], set()
        for w in range(Wd):
            if not live[i, w]:
                continue
            e = _terminal_end(v, ids[i, w])
            ref = p[i, w, np.arange(e), ids[i, w, :e]]
            np.testing.assert_allclose(probs[i, w, :e], ref, rtol=1e-4)
            assert (probs[i, w, e:] == 0).all() and (ids[i, w, e:] == v.recog_pad_index).all()
            assert abs(scores[i, w] - float(np.log(ref).sum())) < 1e-3, (i, w)
            hyp = tuple(ids[i, w, :e].tolist())
            assert hyp not in seen, (i, w)
            seen.add(hyp)
            keys.append(scores[i, w] / e ** alpha)
        assert all(keys[r] >= keys[r + 1] - 1e-5 for r in range(len(keys) - 1)), keys


def test_full_fixture_hypotheses_match_teacher_forcing_and_the_cpu_rule():
    from oracle import omniparser_ref as O
    from oracle.gen_golden import OMNI_CASES
    from tests.conftest import omni_sd
    case = OMNI_CASES['full']
    m = _full_model()
    img, mask = _full_case(m)
    sd = omni_sd(case['wseed'], case['pt_eos_bias'])
    mem, pos, kpm, _ = O.encode(img.cpu(), mask.cpu(), sd)
    compared = 0
    for xattn in (0, 2):
        with options(m.ctx, xattn_impl=xattn, nsplit=3):
            m.encode(img, mask)
            for width, alpha in ((2, 0.0), (4, 1.0), (8, 1.0)):
                n_inst, pt, _, _ = _decode_raw(m, rec_beams=width, length_penalty=alpha)
                ids, bp, sc = m.last_rec_beams
                n = int(n_inst[0])
                _check_hypotheses(m, 0, pt[0, :n], ids[0, :n], bp[0, :n], sc[0, :n], alpha)
                if xattn == 0:   # the CPU rule on the oracle's logits: ids bit for bit where no margin is a near-tie
                    rid, rp, rs, _, marg = beam_rec(mem[0], kpm[0], pos[0], sd, torch.as_tensor(pt[0, :n]), width,
                                                    alpha, m.vocab.rec_length)
                    print(f'W={width} alpha={alpha}: margins {marg}')
                    if min(marg.values()) >= NEAR_TIE:
                        assert np.array_equal(ids[0, :n], rid)
                        # 25 steps of GPU vs CPU fp32 log-probabilities, each ~1e-5 apart
                        np.testing.assert_allclose(sc[0, :n], rs, atol=5e-4)
                        np.testing.assert_allclose(bp[0, :n], rp, rtol=5e-5, atol=0)   # GPU vs CPU fp32 logits
                        compared += 1
    print(f'{compared} beam runs compared with the CPU rule id for id')


def test_config2_scale_hypotheses_match_teacher_forcing():
    from advancedliteratemachinery_b200 import OmniParserB200, OmniVocab
    from oracle.gen_golden import CONFIG2_CASE, config2_page
    from tests.conftest import omni_sd
    close_models()
    case = CONFIG2_CASE
    v = OmniVocab(pt_seq_length=case['pt_seq_length'], rec_length=case['rec_length'])
    m = OmniParserB200(omni_sd(case['wseed'], case['pt_eos_bias']), v, workspace_mb=20480)
    try:
        img, mask = config2_page(case['seed'])
        m.encode(img.cuda(), mask.cuda())
        n_inst, pt, rec, prob = _decode_raw(m, rec_beams=4, length_penalty=1.0)
        ids, bp, sc = m.last_rec_beams
        n = int(n_inst[0])
        assert n > 0
        _check_hypotheses(m, 0, pt[0, :n], ids[0, :n], bp[0, :n], sc[0, :n], 1.0)
        # the same page inside a 4-page batch
        g = torch.Generator().manual_seed(77)
        others = torch.randn(3, *img.shape[1:], generator=g)
        m.encode(torch.cat([img, others]).cuda(), torch.cat([mask, mask.expand(3, -1, -1)]).cuda())
        _decode_raw(m, rec_beams=4, length_penalty=1.0)
        ids4, bp4, sc4 = m.last_rec_beams
        assert np.array_equal(ids4[0], ids[0])
        np.testing.assert_allclose(bp4[0], bp[0], rtol=5e-5, atol=0)   # GEMM tiles follow the row count
        np.testing.assert_allclose(sc4[0], sc[0], atol=1e-4)
    finally:
        m.ctx.close()


# ----------------------------------------------------------------------------------------------- invariance
def test_n_best_lists_do_not_depend_on_batch_context_or_graphs():
    from advancedliteratemachinery_b200 import NestedTensor, OmniParserB200
    owner = _full_model()
    img, mask = _full_case(owner)
    v = owner.vocab
    owner.encode(img, mask)
    _decode_raw(owner, rec_beams=4)
    ref = owner.last_rec_beams
    # the page in a batch with two other pages, and through forward_pages
    g = torch.Generator().manual_seed(3)
    others = torch.randn(2, *img.shape[1:], generator=g)
    owner.encode(torch.cat([img.cpu(), others]).cuda(), torch.cat([mask.cpu(), torch.zeros(2, *mask.shape[1:],
                                                                                          dtype=torch.bool)]).cuda())
    _decode_raw(owner, rec_beams=4)
    got = owner.last_rec_beams
    assert np.array_equal(got[0][0], ref[0][0])
    np.testing.assert_allclose(got[1][0], ref[1][0], rtol=5e-5, atol=0)
    h = int((~mask[0].cpu()).any(1).sum()); w = int((~mask[0].cpu()).any(0).sum())
    page = torch.zeros(1, 3, *img.shape[2:])
    page[0, :, :h, :w] = img[0, :, :h, :w].cpu()
    owner.forward_pages(NestedTensor(page.cuda(), mask[:1].cuda()), rec_beams=4)
    fp = owner.last_rec_beams
    owner.encode(page[:, :, :h, :w].cuda(), None)
    _decode_raw(owner, rec_beams=4)
    alone = owner.last_rec_beams
    assert np.array_equal(fp[0], alone[0])
    np.testing.assert_allclose(fp[2], alone[2], atol=1e-4)
    # three contexts over the same weights, graphs on and off
    ctxs = [OmniParserB200(None, v, workspace_mb=8192, share_from=owner) for _ in range(3)]
    try:
        for i, c in enumerate(ctxs):
            c.ctx.set_option('use_graphs', i % 2)
            c.encode(img, mask)
            _decode_raw(c, rec_beams=4)
            assert np.array_equal(c.last_rec_beams[0], ref[0]), i
            assert np.array_equal(c.last_rec_beams[2].view(np.uint32), ref[2].view(np.uint32)), i
    finally:
        for c in ctxs:
            c.ctx.close()


# ----------------------------------------------------------------------------------------------- op level
def _beam_step_ref(logits, score, blen, G, W, nsoft, v, gen_index):
    """one step of the rule in fp64 on fp32 probabilities: (token, parent, prob, score, len) per child row"""
    out = []
    p32 = torch.softmax(torch.as_tensor(logits)[:, :nsoft].float(), -1).numpy()
    allowed = list(range(v.num_bins, v.recog_pad_index + 1)) + [v.rec_eos_index]
    for g in range(G):
        cands = []
        for h in range(W):
            s = 0.0 if gen_index == 0 and h == 0 else (-math.inf if gen_index == 0 else float(score[g * W + h]))
            ln = 0 if gen_index == 0 else int(blen[g * W + h])
            if s == -math.inf:
                continue
            if ln:
                cands.append((s, h, -1, 0.0, 0))
                continue
            for c in allowed:
                pc = float(p32[g * W + h, c])
                if pc > 0:
                    cands.append((s + math.log(pc), h, c, pc, 0))
        cands.sort(key=lambda x: (-x[0], x[1], x[2]))
        for j in range(W):
            if j >= len(cands):
                out.append((v.recog_pad_index, j, 0.0, -math.inf, 0))
                continue
            s, h, c, pc, _ = cands[j]
            if c < 0:
                out.append((v.recog_pad_index, h, 0.0, s, int(blen[g * W + h])))
            else:
                out.append((c, h, pc, s, gen_index + 1 if c in (v.rec_eos_index, v.recog_pad_index) else 0))
    return out


def _op_beam_select(m, logits, score, blen, G, W, nsoft, gen_index):
    import ctypes
    cfg = m._cfg(1)
    d_lg = torch.as_tensor(logits, dtype=torch.float32).cuda().contiguous()
    d_s = torch.as_tensor(score, dtype=torch.float32).cuda().contiguous()
    d_l = torch.as_tensor(blen, dtype=torch.int32).cuda().contiguous()
    tok = torch.zeros(G * W, dtype=torch.int32, device='cuda')
    par = torch.zeros_like(tok)
    prob = torch.zeros(G * W, dtype=torch.float32, device='cuda')
    m.ctx.check(m.lib.alm_op_beam_select(m.ctx.h, d_lg.data_ptr(), G, W, d_lg.shape[1], nsoft, gen_index,
                                         ctypes.byref(cfg), d_s.data_ptr(),
                                         d_l.data_ptr(), tok.data_ptr(), par.data_ptr(), prob.data_ptr()))
    return tok.cpu().numpy(), par.cpu().numpy(), prob.cpu().numpy(), d_s.cpu().numpy(), d_l.cpu().numpy()


def _compare_op(m, logits, score, blen, G, W, nsoft, gen_index, tag):
    v = m.vocab
    tok, par, prob, s_out, l_out = _op_beam_select(m, logits, score, blen, G, W, nsoft, gen_index)
    ref = _beam_step_ref(logits, score, blen, G, W, nsoft, v, gen_index)
    lg64 = torch.as_tensor(logits).double()
    p64 = torch.softmax(lg64[:, :nsoft], -1).numpy()
    for r, (c, h, pc, s, ln) in enumerate(ref):
        assert tok[r] == c and par[r] == h and l_out[r] == ln, (tag, r, (tok[r], par[r], l_out[r]), (c, h, ln))
        if s == -math.inf:
            assert s_out[r] == -np.inf and prob[r] == 0, (tag, r)
            continue
        g = r // W
        if pc > 0:
            exact = p64[g * W + h, c]
            assert abs(prob[r] - exact) <= 4e-6 * exact, (tag, r)   # fp32 expf of the step's softmax
        assert abs(s_out[r] - s) <= 1e-5 * max(1.0, abs(s)), (tag, r, s_out[r], s)


def test_op_beam_select_against_fp64():
    m = _full_model()
    v = m.vocab
    V = 1104
    allowed = list(range(v.num_bins, v.recog_pad_index + 1)) + [v.rec_eos_index]
    rng = np.random.default_rng(0)
    for W, G in ((2, 3), (4, 5), (8, 4)):
        lg = rng.normal(0, 3, (G * W, V)).astype(np.float32)
        score = -rng.random(G * W).astype(np.float32) * 5
        blen = np.zeros(G * W, dtype=np.int32)
        _compare_op(m, lg, score, blen, G, W, V, 0, f'start W={W}')
        # finished and dead parents, a forbidden class holding the row maximum
        blen[1::W] = 3
        score[2::W] = -np.inf if W > 2 else score[2::W]
        lg[:, 5] = 40.0
        _compare_op(m, lg, score, blen, G, W, V, 6, f'mixed W={W}')
        # tied scores: two rows of a group identical (same parent score), equal logits across classes
        lg2 = lg.copy()
        lg2[W * 0 + 1] = lg2[0]
        lg2[:, allowed[3]] = lg2[:, allowed[7]]
        sc2 = score.copy()
        sc2[1] = sc2[0]
        bl2 = np.zeros_like(blen)
        _compare_op(m, lg2, sc2, bl2, G, W, V, 4, f'ties W={W}')
        # zero probabilities (exp underflow) and nsoft < V
        lg3 = lg.copy()
        lg3[:, allowed[::2]] = -200.0
        _compare_op(m, lg3, score, np.zeros_like(blen), G, W, V - 3, 2, f'zero p, nsoft<V W={W}')
    # W = 8 with only 3 allowed classes left after masking: children past the finite candidates are dead
    G, W = 2, 8
    lg = np.full((G * W, V), -1e4, dtype=np.float32)
    lg[:, 0] = 0.0
    lg[:, allowed[:3]] = [1.0, 0.5, 0.25]
    _compare_op(m, lg, np.zeros(G * W, np.float32), np.zeros(G * W, np.int32), G, W, V, 0, 'few classes')


@pytest.mark.parametrize('t', [0, 1, 27])
def test_op_self_attention_step_with_ancestry(t):
    m = _full_model()
    S, Tmax = 12, 30
    g = torch.Generator().manual_seed(t)
    qkv = torch.randn(S, 1536, generator=g)
    kc = torch.full((S, Tmax, 512), float('nan'))
    vc = torch.full((S, Tmax, 512), float('nan'))
    anc = torch.randint(0, S, (S, Tmax), generator=g, dtype=torch.int32)
    kd = torch.randn(S, Tmax, 512, generator=g)
    vd = torch.randn(S, Tmax, 512, generator=g)
    for s in range(S):   # only the rows the ancestry points to hold data
        for j in range(t):
            kc[anc[s, j], j] = kd[anc[s, j], j]
            vc[anc[s, j], j] = vd[anc[s, j], j]
    out = torch.zeros(S, 512)
    d = [x.cuda().contiguous() for x in (qkv, kc, vc, out, anc)]
    for wide in (1, 0):
        with options(m.ctx, sattn_wide=wide):
            m.ctx.check(m.lib.alm_op_self_attention_step_anc(m.ctx.h, d[0].data_ptr(), d[1].data_ptr(), d[2].data_ptr(),
                                                             d[3].data_ptr(), S, t, Tmax, d[4].data_ptr()))
        got = d[3].cpu().double()
        q = qkv[:, :512].double().reshape(S, 8, 64) / 8
        for s in range(S):
            keys = torch.stack([kd[anc[s, j], j] for j in range(t)] + [qkv[s, 512:1024]]).double().reshape(t + 1, 8, 64)
            vals = torch.stack([vd[anc[s, j], j] for j in range(t)] + [qkv[s, 1024:]]).double().reshape(t + 1, 8, 64)
            a = torch.softmax(torch.einsum('hd,thd->ht', q[s], keys), -1)
            ref = torch.einsum('ht,thd->hd', a, vals).reshape(512)
            assert float((got[s] - ref).abs().max()) < 1e-5, (wide, s)
        # row s wrote its own position t
        assert torch.equal(d[1][:, t].cpu(), qkv[:, 512:1024]) and torch.equal(d[2][:, t].cpu(), qkv[:, 1024:])


# ----------------------------------------------------------------------------------------------- errors / off
def test_errors_and_width_zero_restores_greedy():
    from advancedliteratemachinery_b200 import OmniParserB200
    m = _full_model()
    img, mask = _full_case(m)
    v = m.vocab
    lib, h = m.lib, m.ctx.h
    m.encode(img, mask)
    m.decode()   # a decode without beams or candidates: both options off
    for bad in (-1, 9):
        assert lib.alm_omni_set_rec_beams(h, bad, 1.0) == ERR_INVALID
        with pytest.raises(ValueError):
            m.decode(rec_beams=bad)
    for bad in (-0.5, 2.5, float('nan')):
        assert lib.alm_omni_set_rec_beams(h, 2, bad) == ERR_INVALID
    with pytest.raises(ValueError):
        m.decode(rec_beams=2, rec_candidates=2)
    assert lib.alm_omni_set_rec_candidates(h, 3) == 0
    assert lib.alm_omni_set_rec_beams(h, 2, 1.0) == ERR_INVALID    # candidates on
    assert lib.alm_omni_set_rec_candidates(h, 0) == 0
    assert lib.alm_omni_set_rec_beams(h, 2, 1.0) == 0
    assert lib.alm_omni_set_rec_candidates(h, 3) == ERR_INVALID    # beams on
    assert lib.alm_omni_set_rec_beams(h, 0, 1.0) == 0
    m._rec_k, m._rec_beams = 0, (0, 1.0)
    buf_i, buf_p, buf_s = np.zeros(1 << 16, np.int64), np.zeros(1 << 16, np.float32), np.zeros(1 << 16, np.float32)
    m.decode()
    assert lib.alm_omni_get_rec_beams(h, buf_i.ctypes.data, buf_p.ctypes.data, buf_s.ctypes.data, buf_i.size) == ERR_STATE
    m.decode(rec_beams=3)
    need = m.last_rec_beams[0].size
    assert lib.alm_omni_get_rec_beams(h, buf_i.ctypes.data, buf_p.ctypes.data, buf_s.ctypes.data, need - 1) == ERR_INVALID
    assert lib.alm_omni_get_rec_beams(h, None, buf_p.ctypes.data, buf_s.ctypes.data, need) == ERR_INVALID
    assert lib.alm_omni_get_rec_beams(h, buf_i.ctypes.data, buf_p.ctypes.data, None, need) == ERR_INVALID
    assert lib.alm_omni_get_rec_beams(h, buf_i.ctypes.data, buf_p.ctypes.data, buf_s.ctypes.data, need) == 0
    assert np.array_equal(buf_i[:need], m.last_rec_beams[0].reshape(-1))
    assert np.array_equal(buf_s[:need // v.rec_length], m.last_rec_beams[2].reshape(-1))
    # W = 0 after a beam decode: the greedy launches and outputs of a context that never used beams
    fresh = OmniParserB200(None, v, workspace_mb=8192, share_from=m)
    try:
        def run(model):
            model.encode(img, mask)
            model.ctx.launch_count(reset=True)
            out = model.decode()
            return out, model.ctx.launch_count()
        ref, ref_n = run(fresh)
        got, got_n = run(m)
        assert got_n == ref_n and m.last_rec_beams is None
        for a, b in zip(ref, got):
            for x, y in zip(a[0], b[0]):
                assert torch.equal(x, y)
            assert torch.equal(a[1][0], b[1][0])
        assert lib.alm_omni_get_rec_beams(h, buf_i.ctypes.data, buf_p.ctypes.data, buf_s.ctypes.data, buf_i.size) == ERR_STATE
    finally:
        fresh.ctx.close()
