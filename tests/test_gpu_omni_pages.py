"""GPU: pages of different sizes in one batch (alm_omni_encode_pages, OmniParserB200.encode_pages / forward_pages).
Every page must get what the reference returns for that page alone (tests/golden/omni_pages.npz, written from the
unmodified reference one page at a time) and what the library returns for the page encoded alone at B = 1; a batch of
one page size through the new entry must equal alm_omni_encode bit for bit; and the cross-attention kernels with
per-image live-key counts are held to fp64 with NaN in every key beyond a page's count."""
import json

import numpy as np
import pytest
import torch

from tests.support import close_models, omni_model, options, release_models
from tests.test_pages_cpu import pages_case, pages_page

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

ERR_INVALID, ERR_STATE, ERR_UNSUPPORTED = -1, -4, -5
ORDER = [0, 3, 1, 4, 2]   # fixture pages in a batch order that interleaves the sizes (page 0 and 4 share one)
PROB_RTOL = 1e-5


def spot_model(gold):
    return omni_model({k: gold[k][0] for k in ('wseed', 'pt_eos_bias', 'pt_seq_length', 'rec_length')})


def canvas(pages):
    """NestedTensor-layout batch of [1, 3, h, w] pages: NaN outside every page (never read), mask 1 there"""
    Hc, Wc = max(p.shape[2] for p in pages), max(p.shape[3] for p in pages)
    t = torch.full((len(pages), 3, Hc, Wc), float('nan'))
    mask = torch.ones(len(pages), Hc, Wc, dtype=torch.bool)
    for b, p in enumerate(pages):
        t[b, :, :p.shape[2], :p.shape[3]] = p[0]
        mask[b, :p.shape[2], :p.shape[3]] = False
    return t, mask


def fixture_batch(gold):
    pages = [pages_page(gold, b) for b in ORDER]
    return pages, canvas(pages)


def _maxrel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).abs().max() / (b.abs().max() + 1e-30))


def assert_result(a, b, report, key):
    """same ids; probabilities within PROB_RTOL (bit identity recorded in `report`)"""
    assert (a is None) == (b is None), key
    if a is None:
        return
    for x, y in zip(a[0], b[0]):
        assert torch.equal(x, y), key
    np.testing.assert_allclose(a[1][0].numpy(), b[1][0].numpy(), rtol=PROB_RTOL, atol=0, err_msg=key)
    report.setdefault('probs_bit_identical', []).append(bool(torch.equal(a[1][0], b[1][0])))


@pytest.mark.parametrize('impl', [0, 1, 2])
def test_mixed_batch_matches_the_reference_fixture(golden_dir, impl):
    from advancedliteratemachinery_b200 import NestedTensor
    gold = pages_case(golden_dir)
    m = spot_model(gold)
    with options(m.ctx, xattn_impl=impl):   # before the encode: xattn_impl 1 needs its V_c^T
        pages, (t, mask) = fixture_batch(gold)
        outs = m.forward_pages(NestedTensor(t.cuda(), mask.cuda()))
    assert len(outs) == len(ORDER)
    shapes = m.page_shapes()
    mem, pos = m.memory(0), m.memory(1)
    Mmax = max(h * w for h, w in shapes)
    assert mem.shape == (len(ORDER), Mmax, 512)
    for i, b in enumerate(ORDER):
        h, w = (int(x) for x in gold['sizes'][b])
        assert shapes[i] == ((h + 15) // 16, (w + 15) // 16)
        Mb = shapes[i][0] * shapes[i][1]
        ref = torch.from_numpy(gold[f'memory_{b}'])
        assert float((mem[i, :Mb] - ref).norm() / ref.norm()) < 1e-4, b
        np.testing.assert_allclose(pos[i, :Mb].numpy(), gold[f'pos_{b}'], atol=3e-6, rtol=0)
        assert not mem[i, Mb:].any() and not pos[i, Mb:].any()
        if gold['n_inst'][b] == 0:
            assert outs[i] is None, b
            continue
        (pt, poly, rec), (probs,) = outs[i]
        # the fixture clears a 1e-4 top-1 / top-2 gap at every greedy step: ids are bit-exact
        assert np.array_equal(pt.numpy(), gold[f'pt_{b}']), b
        assert np.array_equal(poly.numpy(), gold[f'poly_{b}']), b
        assert np.array_equal(rec.numpy(), gold[f'rec_{b}']), b
        np.testing.assert_allclose(probs.numpy(), gold[f'probs_{b}'], rtol=2e-3, atol=1e-7)
    # no common grid: the single-grid readbacks refuse
    assert m.lib.alm_omni_memory_shape(m.ctx.h, None, None, None) == ERR_STATE
    assert m.lib.alm_omni_get_feature(m.ctx.h, 0, None, 0) == ERR_UNSUPPORTED


def test_each_page_of_a_mixed_batch_equals_the_page_encoded_alone(golden_dir):
    from advancedliteratemachinery_b200 import OmniVocab
    gold = pages_case(golden_dir)
    m = spot_model(gold)
    v = m.vocab
    pages, (t, mask) = fixture_batch(gold)
    sizes = [tuple(p.shape[2:]) for p in pages]
    nb = v.num_bins
    glob = v.window_prompt()[0]
    prompts = torch.stack([glob, torch.tensor([0, 0, nb // 2, nb - 1, nb, nb + len(v.chars), v.pt_sos_index]),
                           v.window_prompt(chars=('a', 'm'))[0]])
    m.encode_pages(t.cuda(), sizes)
    shapes = m.page_shapes()
    mem, pos = m.memory(0), m.memory(1)
    mixed = dict(decode=m.decode(), prompts=m.decode_prompts(prompts), points=m.decode_points())
    seq = torch.cat([v.pt_prompt(), torch.tensor([[5, 7, 300, 400, 999, 0]])], 1)
    logits = [m.decode_logits(i, 'pt', seq) for i in range(len(pages))]
    report = {}
    for i, p in enumerate(pages):
        m.encode(p.cuda(), None)
        assert m.page_shapes() == [shapes[i]]
        Mb = shapes[i][0] * shapes[i][1]
        assert torch.equal(mem[i, :Mb], m.memory(0)[0]) and torch.equal(pos[i, :Mb], m.memory(1)[0]), i
        assert not mem[i, Mb:].any() and not pos[i, Mb:].any()
        assert_result(mixed['decode'][i], m.decode()[0], report, f'decode {i}')
        alone = m.decode_prompts(prompts)[0]
        for k in range(3):
            assert_result(mixed['prompts'][i][k], alone[k], report, f'prompt {i},{k}')
        (tok, prob), = m.decode_points()
        assert torch.equal(mixed['points'][i][0], tok), i
        np.testing.assert_allclose(mixed['points'][i][1].numpy(), prob.numpy(), rtol=PROB_RTOL, atol=0)
        report.setdefault('points_probs_bit_identical', []).append(bool(torch.equal(mixed['points'][i][1], prob)))
        lg = m.decode_logits(0, 'pt', seq)
        err = _maxrel(logits[i], lg)
        assert err <= PROB_RTOL, (i, err)
        report.setdefault('logits_max_rel', []).append(err)
    print('mixed batch vs batch 1:', json.dumps(report))

    # KIE checkpoint: the (x, y, class) point loop and the per-pair polygon / transcription loops
    from advancedliteratemachinery_b200 import OmniParserB200
    from oracle import weights as W
    from oracle.gen_golden import KIE_CASES
    case = KIE_CASES['kie']
    sd = W.omniparser_state_dict(seed=case['wseed'], vie_categories=case['vie'], pt_eos_bias=case['pt_eos_bias'])
    k = OmniParserB200(sd, OmniVocab(vie_categories=case['vie'], pt_seq_length=case['pt_seq_length'],
                                     rec_length=case['rec_length']), workspace_mb=4096)
    try:
        k.encode_pages(t.cuda(), sizes)
        res = k.decode_kie(sizes)
        raw = {key: val.copy() for key, val in k.last_kie_raw.items()}
        assert sum(int(n) for n in raw['n_inst']) > 0, 'the KIE case must decode pairs'
        for i, p in enumerate(pages):
            k.encode(p.cuda(), None)
            alone = k.decode_kie([sizes[i]])
            one = k.last_kie_raw
            nt, ni = int(one['n_tok'][0]), int(one['n_inst'][0])
            assert int(raw['n_tok'][i]) == nt and int(raw['n_inst'][i]) == ni, i
            assert np.array_equal(raw['tokens'][i, :nt], one['tokens'][0, :nt]), i
            assert np.array_equal(raw['inst_pos'][i, :ni], one['inst_pos'][0, :ni]), i
            assert np.array_equal(raw['poly'][i, :ni], one['poly'][0, :ni]), i
            assert np.array_equal(raw['rec'][i, :ni], one['rec'][0, :ni]), i
            np.testing.assert_allclose(raw['probs'][i, :nt], one['probs'][0, :nt], rtol=PROB_RTOL, atol=0)
            assert [(e[0], e[1], e[3]) for e in res[i] or []] == [(e[0], e[1], e[3]) for e in alone[0] or []], i
    finally:
        k.ctx.close()


@pytest.mark.parametrize('crop', [False, True])
def test_one_page_size_through_encode_pages_is_encode_bit_for_bit(golden_dir, crop):
    gold = pages_case(golden_dir)
    m = spot_model(gold)
    pages = [pages_page(gold, 0), pages_page(gold, 4), pages_page(gold, 0)]   # three pages of 96 x 128
    dense = torch.cat(pages)
    t = canvas(pages + [torch.zeros(1, 3, 112, 160)])[0][:3].contiguous() if crop else dense
    shapes = m.encode_pages(t.cuda(), [(96, 128)] * 3)
    assert shapes == [(6, 8)] * 3
    got = dict(mem=m.memory(0), pos=m.memory(1), feat=[m.features(lvl).clone() for lvl in range(4)],
               out=m.decode(), pts=m.decode_points())
    assert m.memory_shape() == (3, 6, 8)
    m.encode(dense.cuda(), None)
    assert torch.equal(got['mem'], m.memory(0)) and torch.equal(got['pos'], m.memory(1))
    for lvl in range(4):
        assert torch.equal(got['feat'][lvl], m.features(lvl)), lvl
    for a, b in zip(got['out'], m.decode()):
        assert (a is None) == (b is None)
        if a is not None:
            assert all(torch.equal(x, y) for x, y in zip(a[0], b[0])) and torch.equal(a[1][0], b[1][0])
    for (ta, pa), (tb, pb) in zip(got['pts'], m.decode_points()):
        assert torch.equal(ta, tb) and torch.equal(pa, pb)


def test_config2_page_inside_a_batch_of_page_sizes(golden_dir):
    """The benchmark page (1024 x 1024, N = 64 instances, pt 128 + 64 x (32 + 25) steps) in one batch with pages of
    1448 x 1024, 1024 x 1448 and 1325 x 1024: its ids equal the page decoded alone, and hold against the reference
    fixture under the judged near-tie protocol of the config-2 test."""
    import os
    from advancedliteratemachinery_b200 import NestedTensor, OmniParserB200, OmniVocab
    from oracle import omniparser_ref as O
    from oracle.gen_golden import CONFIG2_CASE, config2_page
    from tests.conftest import omni_sd
    from tests.test_gpu_omniparser import MAX_NEAR_TIE_FLIPS, _judge_flips
    close_models()
    case = CONFIG2_CASE
    gold = np.load(os.path.join(golden_dir, 'omni_config2_page0.npz'))
    sd = omni_sd(case['wseed'], case['pt_eos_bias'])
    v = OmniVocab(pt_seq_length=case['pt_seq_length'], rec_length=case['rec_length'])
    m = OmniParserB200(sd, v, workspace_mb=20480)
    try:
        img, mask = config2_page(case['seed'])
        g = torch.Generator().manual_seed(77)
        others = [torch.randn(1, 3, h, w, generator=g) for h, w in ((1448, 1024), (1024, 1448), (1325, 1024))]
        pages = [others[0], img, others[1], others[2]]
        t, pmask = canvas(pages)
        outs = m.forward_pages(NestedTensor(t.cuda(), pmask.cuda()))
        shapes = m.page_shapes()
        assert shapes == [(91, 64), (64, 64), (64, 91), (83, 64)]
        alone = m.forward_batch(NestedTensor(img, None))[0]
        n = 64
        got = outs[1]
        for x, y in zip(got[0], alone[0]):
            assert torch.equal(x, y), 'the config-2 page in the batch differs from the page alone'
        (pt, poly, rec), _ = got
        report = dict(equal_to_reference=bool(np.array_equal(pt.numpy(), gold['pt']) and
                                               np.array_equal(poly.numpy(), gold['poly']) and
                                               np.array_equal(rec.numpy(), gold['rec'])))
        if not report['equal_to_reference']:   # every deviation must be a judged reference near-tie
            mem, pos, kpm, _ = O.encode(img, mask, sd)
            gpt = torch.from_numpy(gold['pt'])
            full = {'pt': torch.cat([v.pt_prompt(), gpt], 1),
                    'poly': torch.cat([gpt.reshape(-1, 2), torch.full((n, 1), v.poly_sos_index),
                                       torch.from_numpy(gold['poly']).reshape(n, 32)], 1),
                    'rec': torch.cat([gpt.reshape(-1, 2), torch.full((n, 1), v.rec_sos_index),
                                      torch.from_numpy(gold['rec'])[0]], 1)}
            ref_lg = {kd: O.decode_logits(s, mem[0], kpm[0], pos[0], sd, kd) for kd, s in full.items()}
            m.forward_pages(NestedTensor(t.cuda(), pmask.cuda()))
            our_lg = {kd: m.decode_logits(1, kd, s) for kd, s in full.items()}
            flips = _judge_flips('pt', pt.numpy(), gold['pt'], gold['gap_pt'], ref_lg['pt'], our_lg['pt'], 7,
                                 O.step_candidates)
            if not flips:
                flips += _judge_flips('poly', poly.numpy().reshape(n, 32), gold['poly'].reshape(n, 32), gold['gap_poly'],
                                      ref_lg['poly'], our_lg['poly'], 3, O.step_candidates)
                flips += _judge_flips('rec', rec.numpy()[0], gold['rec'][0], gold['gap_rec'], ref_lg['rec'],
                                      our_lg['rec'], 3, O.step_candidates)
            report['near_tie_flips'] = flips
            assert len(flips) <= MAX_NEAR_TIE_FLIPS, flips
        print('config-2 page in a mixed batch:', json.dumps(report))
        assert all(o is not None for o in outs)
    finally:
        m.ctx.close()


def test_preprocessed_pages_end_to_end(golden_dir):
    """8-bit pages of different aspect ratios -> preprocess.omni_pages (resize, normalise, pad) -> forward_pages equals
    every page preprocessed and forwarded alone."""
    from advancedliteratemachinery_b200 import preprocess
    gold = pages_case(golden_dir)
    m = spot_model(gold)
    g = torch.Generator().manual_seed(5)
    images = [torch.randint(0, 256, (h, w, 3), generator=g, dtype=torch.uint8)
              for h, w in ((60, 80), (90, 50), (70, 70), (45, 80))]
    samples = preprocess.omni_pages(m.ctx, images, 128, 128)
    outs = m.forward_pages(samples)
    resized, _ = preprocess.omni_plan([tuple(im.shape[:2]) for im in images], 128, 128)
    assert m.page_shapes() == [((h + 15) // 16, (w + 15) // 16) for h, w in resized]
    assert len(set(resized)) == len(images)
    report = {}
    for i, im in enumerate(images):
        one = m.forward(preprocess.omni_pages(m.ctx, [im], 128, 128))
        assert_result(outs[i], one, report, f'page {i}')
    assert any(o is not None for o in outs)
    print('preprocessed pages:', json.dumps(report))


# ----------------------------------------------------------------------------------------------- cross-attention op
def _xattn_ref(q, k, v, kpm, img0):
    nimg, ncap = q.shape[0], q.shape[1]
    M = k.shape[1]
    qh = q.double().view(nimg, ncap, 8, 64).transpose(1, 2)
    kh = k[img0:img0 + nimg].double().view(nimg, M, 8, 64).transpose(1, 2)
    vh = v[img0:img0 + nimg].double().view(nimg, M, 8, 64).transpose(1, 2)
    s = (qh / 8) @ kh.transpose(-1, -2)
    s = s.masked_fill(kpm[img0:img0 + nimg, None, None, :].bool(), float('-inf'))
    return (s.softmax(-1) @ vh).transpose(1, 2).reshape(nimg, ncap, 512)


# (xattn_impl, nsplit, q_split, Ncap): 16-row (Ncap <= 16) and 64-row query blocks
OP_CASES = [(0, 3, 0, 5), (0, 1, 0, 16), (0, 3, 1, 65), (0, 1, 1, 17), (2, 3, 0, 1), (2, 1, 0, 16), (2, 3, 1, 65),
            (2, 1, 1, 130)]


@pytest.mark.parametrize('case', OP_CASES, ids=lambda c: 'impl{}-ns{}-{}-N{}'.format(c[0], c[1], 'split' if c[2] else 'f32', c[3]))
@pytest.mark.parametrize('kpm_kind', ['none', 'masked'])
def test_cross_attention_with_key_counts_matches_fp64(case, kpm_kind):
    from advancedliteratemachinery_b200 import _lib
    impl, nsplit, q_split, ncap = case
    M = 1000
    key_len = np.array([M, 1, 63, 64, 65, M, 700], dtype=np.int32)   # image 0 is outside the slice
    total, img0, nimg = len(key_len), 1, len(key_len) - 1
    g = torch.Generator(device='cuda').manual_seed(ncap * 7 + impl)
    q = torch.randn(nimg, ncap, 512, generator=g, device='cuda') * 2
    k = torch.randn(total, M, 512, generator=g, device='cuda') * 2
    v = torch.randn(total, M, 512, generator=g, device='cuda')
    dead = torch.arange(M, device='cuda')[None, :] >= torch.from_numpy(key_len).cuda()[:, None]
    kpm = None
    if kpm_kind == 'masked':   # a padding mask on top of the counts: every third live key of the long images
        kpm = torch.zeros(total, M, dtype=torch.uint8, device='cuda')
        kpm[:, 2::3] = 1
        kpm[key_len < 66] = 0
    ref = _xattn_ref(q, k, v, (dead | (kpm.bool() if kpm is not None else False)).to(torch.uint8), img0)
    tol = 3e-5 if nsplit == 3 else 2e-2
    ctx = _lib.Context(0)
    try:
        ctx.set_option('workspace_mb', 4096)
        ctx.set_option('xattn_impl', impl)
        ctx.set_option('nsplit', nsplit)

        def run(launches):
            out = torch.full((nimg, ncap, 512), float('nan'), device='cuda')
            torch.cuda.synchronize()
            ctx.check(ctx.lib.alm_op_cross_attention_ex(ctx.h, q.data_ptr(), k.data_ptr(), v.data_ptr(),
                                                        None if kpm is None else kpm.data_ptr(), out.data_ptr(), total,
                                                        img0, nimg, ncap, M, 5, q_split, launches, key_len.ctypes.data))
            return out
        got = run(1)
        assert torch.isfinite(got).all(), f'{int((~torch.isfinite(got)).sum())} non-finite outputs'
        err = float((got.double() - ref).abs().max() / ref.abs().max())
        assert err <= tol, err
        again = run(2)   # replay on the same partials / counters
        assert torch.equal(again.view(torch.int32), got.view(torch.int32))
    finally:
        ctx.close()


# ----------------------------------------------------------------------------------------------- errors
def test_error_paths(golden_dir):
    from advancedliteratemachinery_b200 import _lib
    gold = pages_case(golden_dir)
    m = spot_model(gold)
    t = torch.zeros(2, 3, 64, 64)

    def enc(hs, ws, B=2, ctx=m.ctx):
        h, w = np.array(hs, dtype=np.int32), np.array(ws, dtype=np.int32)
        return ctx.lib.alm_omni_encode_pages(ctx.h, t.data_ptr(), B, 64, 64, h.ctypes.data, w.ctypes.data)
    assert enc([64, 64], [64, 64], B=0) == ERR_INVALID
    assert enc([31, 64], [64, 64]) == ERR_INVALID
    assert enc([64, 64], [64, 20]) == ERR_INVALID
    assert enc([65, 64], [64, 64]) == ERR_INVALID
    assert enc([64, 64], [64, 65]) == ERR_INVALID
    assert enc([64, 32], [40, 32]) == 0
    bare = _lib.Context(0)
    try:
        assert enc([64, 64], [64, 64], ctx=bare) == ERR_STATE
        mh = np.zeros(2, dtype=np.int32)
        assert bare.lib.alm_omni_page_shapes(bare.h, mh.ctypes.data, mh.ctypes.data) == ERR_STATE
        # the op entry: counts out of range, and xattn_impl 1 (kpm only)
        q = torch.zeros(2, 1, 512, device='cuda')
        kv = torch.zeros(2, 64, 512, device='cuda')
        out = torch.zeros_like(q)
        for lens, impl, rc in (([64, 0], 0, ERR_INVALID), ([65, 64], 0, ERR_INVALID), ([64, 64], 1, ERR_UNSUPPORTED)):
            bare.set_option('xattn_impl', impl)
            kl = np.array(lens, dtype=np.int32)
            torch.cuda.synchronize()
            assert bare.lib.alm_op_cross_attention_ex(bare.h, q.data_ptr(), kv.data_ptr(), kv.data_ptr(), None,
                                                      out.data_ptr(), 2, 0, 2, 1, 64, 0, 0, 1, kl.ctypes.data) == rc
    finally:
        bare.close()
