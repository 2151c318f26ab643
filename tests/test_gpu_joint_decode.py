"""GPU: the joint polygon + recognition decoder pass, part by part against fp64 and as a whole against the two
single-decoder loops, bit for bit.

While both loops have steps left, rows [0, S) of the joint pass are the polygon sequences and rows [S, 2S) the
recognition sequences; every row's arithmetic must be the single-decoder step's (DESIGN 4.4).  The joint GEMM and the
self-attention step are held to that in tests/test_gpu_polyrec_joint.py.  Here:

* the joint embedding (embed_ln_kernel with a second half: its own tokens, position table and query position) and the
  joint LayerNorm (gather_ln_kernel<4, 512, true>: a per-half affine and query position), through alm_op_embed_ln and
  alm_op_gather_ln_joint, against fp64 and bit for bit against one single launch per half, in the three forms the
  decoder layer runs (n1: ln and ln + qpos planes, n2: ln + qpos planes, n3 / final norm: ln planes), with NaN guards
  after every output;
* the argument checks of both entries;
* whole decodes with the "joint_decode" option on against the same decodes with it off (the two single-decoder loops),
  bit for bit: ids, probabilities, top-k candidates, character locations and KIE output, with CUDA graphs on and off
  and at xattn_impl 0 and 2, on the fixtures, recognition loops of 32, 33 and 40 steps (no tail / the recognition half
  finishing alone), batches in each of the three self-attention regimes of the SM count, one instance per page at
  B >= 33, a dense pass whose polygon / recognition passes start past page 0, and checkpoints whose two halves differ
  where the fixtures' do not (the final norm, the position tables).  Every A/B also checks that the joint pass ran:
  it launches fewer kernels.
"""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests import support
from tests.support import NAN, assert_guard, bits, close_models, ctx, guarded, omni_model, options, release_models
from tests.test_gpu_coschedule import _assert_fixture_ids, _assert_same
from tests.test_gpu_encoder_ops import U32, _assert_split, _ln_tol, _op, _planes, _ptr

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

ERR_INVALID = -1
D = 512
V = 1104
WORKSPACE_MB = 1024


# ----------------------------------------------------------------------------------------------- embed_ln
def _embed_tables(seed):
    """word_emb [V, 512] with row V - 2 offset by 1e3 (its LayerNorm cancels in fp32), two different position tables
    [1024, 512], gamma / beta"""
    g = torch.Generator(device='cuda').manual_seed(seed)
    word = torch.randn(V, D, generator=g, device='cuda')
    word[V - 2] += 1e3
    pos = torch.randn(1024, D, generator=g, device='cuda') * 0.5
    pos2 = torch.randn(1024, D, generator=g, device='cuda') * 0.5 + 0.25
    return word, pos, pos2, torch.randn(D, generator=g, device='cuda'), torch.randn(D, generator=g, device='cuda')


def _embed_tokens(n, t, tstride, seed):
    """int32 [n, tstride]: column t has tokens 0, V - 1, V - 2 (the offset row) and random ids; every other column holds
    other valid ids, so a read of the wrong column gives a wrong row"""
    g = torch.Generator().manual_seed(seed)
    tok = torch.randint(0, V, (n, tstride), generator=g, dtype=torch.int32)
    col = torch.randint(0, V, (n,), generator=g, dtype=torch.int32)
    col[:3] = torch.tensor([0, V - 1, V - 2], dtype=torch.int32)[:n]
    tok[:, t] = col
    other = torch.arange(tstride) != t
    tok[:, other] = (tok[:, other] + (tok[:, other] == col[:, None]).int()) % V
    return tok.cuda()


def _embed(ctx, tok, t, S, word, pos, g, b, S_half=0, tok2=None, pos2=None):
    """alm_op_embed_ln into NaN-guarded outputs -> (x [S, 512], qpos [512], qpos2 [512] or None)"""
    x, xf = guarded(S * D)
    q, qf = guarded(D)
    q2, q2f = guarded(D) if S_half else (None, None)
    ctx.check(_op(ctx, 'alm_op_embed_ln', tok.data_ptr(), tok.stride(0), t, S, S_half, _ptr(tok2),
                  tok2.stride(0) if tok2 is not None else 0, word.data_ptr(), V, pos.data_ptr(), _ptr(pos2),
                  g.data_ptr(), b.data_ptr(), x.data_ptr(), q.data_ptr(), _ptr(q2)))
    assert_guard(xf, S * D)
    assert_guard(qf, D)
    if S_half:
        assert_guard(q2f, D)
    return x.view(S, D), q, q2


def _embed_ref(tok, t, word, pos, g, b):
    rows = word[tok[:, t].long()].double() + pos[t].double()
    return rows, F.layer_norm(rows, (D,), g.double(), b.double(), 1e-5)


def _check_embed_rows(x, rows, ref, g, what):
    # the fp32 sum word + pos is rounded once more than the fp64 one: within the row-sum term of _ln_tol
    tol = _ln_tol(rows, g, ref) + 2 * U32 * rows.abs() * (rows.var(-1, unbiased=False, keepdim=True) + 1e-5).rsqrt() \
        * g.double().abs()
    err = (x.double() - ref).abs()
    assert torch.isfinite(x).all(), what
    assert bool((err <= tol).all()), (what, float((err / tol).max()))
    return float((err / tol).max())


@pytest.mark.parametrize('t', [0, 1, 34, 1023])
@pytest.mark.parametrize('S', [1, 7, 8, 9, 300, 2048])
def test_embed_ln_single_against_fp64(ctx, S, t):
    word, pos, _, g, b = _embed_tables(S + t)
    tok = _embed_tokens(S, t, t + 3, S * 7 + t)   # tstride larger than t + 1
    x, q, _ = _embed(ctx, tok, t, S, word, pos, g, b)
    rows, ref = _embed_ref(tok, t, word, pos, g, b)
    worst = _check_embed_rows(x, rows, ref, g, 'x')
    assert torch.equal(bits(q), bits(pos[t].contiguous())), 'qpos is not pos_emb[t]'
    print(f'[joint] embed_ln S={S} t={t}: worst error / bound {worst:.3f}')


@pytest.mark.parametrize('t', [0, 1, 34, 1023])
@pytest.mark.parametrize('S_half,S', [(13, 26), (8, 16), (300, 600)])
def test_embed_ln_joint_against_fp64_and_two_single_launches(ctx, S_half, S, t):
    """the second half reads its own tokens (another row stride) and position table and writes its own query position;
    S_half 13 splits a CTA of 8 warps, 8 ends one"""
    word, pos, pos2, g, b = _embed_tables(S + t + 1)
    n2 = S - S_half
    tok = _embed_tokens(S_half, t, t + 2, S + t)
    tok2 = _embed_tokens(n2, t, t + 5, S + t + 99)
    x, q, q2 = _embed(ctx, tok, t, S, word, pos, g, b, S_half, tok2, pos2)
    rows1, ref1 = _embed_ref(tok, t, word, pos, g, b)
    rows2, ref2 = _embed_ref(tok2, t, word, pos2, g, b)
    worst = max(_check_embed_rows(x[:S_half], rows1, ref1, g, 'first half'),
                _check_embed_rows(x[S_half:], rows2, ref2, g, 'second half'))
    assert torch.equal(bits(q), bits(pos[t].contiguous())), 'qpos is not pos_emb[t]'
    assert torch.equal(bits(q2), bits(pos2[t].contiguous())), 'qpos2 is not pos_emb2[t]'
    # what the decoder relies on: the joint launch is one single launch per half
    xa, qa, _ = _embed(ctx, tok, t, S_half, word, pos, g, b)
    xb, qb, _ = _embed(ctx, tok2, t, n2, word, pos2, g, b)
    assert torch.equal(bits(x[:S_half]), bits(xa)) and torch.equal(bits(x[S_half:]), bits(xb))
    assert torch.equal(bits(q), bits(qa)) and torch.equal(bits(q2), bits(qb))
    print(f'[joint] embed_ln S_half={S_half} S={S} t={t}: worst error / bound {worst:.3f}')


# ----------------------------------------------------------------------------------------------- joint gather_ln
# the decoder layer's forms: n1 writes the ln planes and the ln + qpos planes, n2 only the ln + qpos planes, n3 and the
# final norm only the ln planes
FORMS = {'n1': ('hi', 'lo', 'hi2', 'lo2'), 'n2': ('hi2', 'lo2'), 'n3': ('hi', 'lo')}


def _gather(ctx, src, rows, outs, gamma, beta, add, rows_half=0, gamma2=None, beta2=None, add2=None):
    """alm_op_gather_ln(_joint) over src [rows, 512] (no map, ld_add 0) -> {output: [rows, 512]}, guards checked"""
    bufs = {}
    for k in outs:
        f32 = k.startswith('f32')
        bufs[k] = guarded(rows * D, torch.float32 if f32 else torch.int16, NAN if f32 else -1)

    def p(k):
        return bufs[k][0].data_ptr() if k in bufs else None
    args = [src.data_ptr(), D, None, 1, D, rows, gamma.data_ptr(), beta.data_ptr(), 1e-5, 0, _ptr(add), 0, p('f32'), D,
            p('hi'), p('lo'), D, p('hi2'), p('lo2'), p('f322')]
    if rows_half:
        ctx.check(_op(ctx, 'alm_op_gather_ln_joint', *args, rows_half, gamma2.data_ptr(), beta2.data_ptr(), _ptr(add2)))
    else:
        ctx.check(_op(ctx, 'alm_op_gather_ln', *args))
    res = {}
    for k, (buf, full) in bufs.items():
        assert_guard(full, buf.numel(), NAN if k.startswith('f32') else -1)
        res[k] = buf.view(rows, D)
    return res


@pytest.mark.parametrize('mean', [0.0, 1e3])
@pytest.mark.parametrize('form', list(FORMS))
@pytest.mark.parametrize('S', [1, 5, 8, 13, 1024])
def test_gather_ln_joint_against_fp64_and_each_half_alone(ctx, S, form, mean):
    rows = 2 * S
    gen = torch.Generator(device='cuda').manual_seed(S * 10 + list(FORMS).index(form) + int(mean))
    src = torch.randn(rows, D, generator=gen, device='cuda') * (1.0 if mean else 3.0) + (mean or 0.5)
    aff = [(torch.randn(D, generator=gen, device='cuda'), torch.randn(D, generator=gen, device='cuda')) for _ in range(2)]
    with_add = 'hi2' in FORMS[form]
    adds = [torch.randn(D, generator=gen, device='cuda') if with_add else None for _ in range(2)]
    twins = ('f32',) * ('hi' in FORMS[form]) + ('f322',) * with_add
    (g1, b1), (g2, b2) = aff
    res = _gather(ctx, src, rows, FORMS[form] + twins, g1, b1, adds[0], S, g2, b2, adds[1])
    worst = 0.0
    for h, (g, b) in enumerate(aff):
        x64 = src[h * S:(h + 1) * S].double()
        ref = F.layer_norm(x64, (D,), g.double(), b.double(), 1e-5)
        tol = _ln_tol(x64, g, ref)
        half = {k: v[h * S:(h + 1) * S] for k, v in res.items()}
        if 'f32' in half:
            err = (half['f32'].double() - ref).abs()
            assert bool((err <= tol).all()), (h, float((err / tol).max()))
            worst = max(worst, float((err / tol).max()))
            _assert_split(half['hi'], half['lo'], half['f32'], f'half {h} ln')
        if with_add:
            ref2 = ref + adds[h].double()
            err = (half['f322'].double() - ref2).abs()
            tol2 = tol + U32 * ref2.abs()
            assert bool((err <= tol2).all()), (h, float((err / tol2).max()))
            worst = max(worst, float((err / tol2).max()))
            _assert_split(half['hi2'], half['lo2'], half['f322'], f'half {h} ln + qpos')
        # bit for bit the single entry on this half alone with its own affine and query position (ld_add 0 too)
        alone = _gather(ctx, src[h * S:], S, FORMS[form] + twins, g, b, adds[h])
        for k in alone:
            assert torch.equal(bits(alone[k]), bits(half[k])), (h, k, 'joint half differs from the single launch')
    # the form exactly as the decoder launches it (no f32 outputs) writes the same planes
    plain = _gather(ctx, src, rows, FORMS[form], g1, b1, adds[0], S, g2, b2, adds[1])
    for k in plain:
        assert torch.equal(plain[k], res[k]), k
    print(f'[joint] gather_ln S={S} {form} mean={mean:g}: worst error / bound {worst:.3f}')


# ----------------------------------------------------------------------------------------------- argument errors
def test_argument_errors_leave_the_context_usable(ctx):
    word, pos, pos2, g, b = _embed_tables(5)
    tok = _embed_tokens(4, 1, 3, 5)
    x, q, q2 = (torch.zeros(8 * D, device='cuda') for _ in range(3))
    P = _ptr

    def embed(t=1, S=8, S_half=4, tok2=tok, p2=pos2, qp2=q2, tok1=tok, tstride=3, tstride2=3):
        return _op(ctx, 'alm_op_embed_ln', P(tok1), tstride, t, S, S_half, P(tok2), tstride2, P(word), V, P(pos), P(p2),
                   P(g), P(b), P(x), P(q), P(qp2))
    assert embed() == 0
    assert embed(S=4, S_half=0, tok2=None, p2=None, qp2=None) == 0
    assert embed(tok2=None) == ERR_INVALID                            # joint form without the second half's pointers
    assert embed(p2=None) == ERR_INVALID
    assert embed(qp2=None) == ERR_INVALID
    assert embed(S=4, S_half=0) == ERR_INVALID                        # single form with them
    assert embed(S_half=8) == ERR_INVALID                             # S_half >= S
    assert embed(S_half=9, S=8) == ERR_INVALID
    assert embed(S_half=-1) == ERR_INVALID
    assert embed(t=1024, tstride=1100, tstride2=1100) == ERR_INVALID  # past the position table
    assert embed(tstride=1) == ERR_INVALID                            # column t outside the row
    assert embed(tstride2=1) == ERR_INVALID
    assert embed(tok1=tok.cpu()) == ERR_INVALID                       # host tokens
    for bad in (-1, V):
        for which in (0, 1):
            tb = tok.clone()
            tb[3, 1] = bad
            kw = dict(tok1=tb) if which == 0 else dict(tok2=tb)
            assert embed(**kw) == ERR_INVALID, (bad, which)       # a token outside [0, V), in either half

    src = torch.zeros(4 * D, device='cuda')
    (hi, _), (lo, _) = _planes(8 * D)
    add, add2 = torch.zeros(D, device='cuda'), torch.zeros(D, device='cuda')

    def joint(nsrc=1, Cs=D, rows=4, rows_half=2, a=add, a2=add2, g2=g):
        return _op(ctx, 'alm_op_gather_ln_joint', P(src), D, None, nsrc, Cs, rows, P(g), P(b), 1e-5, 0, P(a), 0, None, 0,
                   P(hi), P(lo), D, P(hi), P(lo), None, rows_half, P(g2), P(b), P(a2))
    assert joint() == 0
    assert joint(a=None, a2=None) == 0
    assert joint(nsrc=2, Cs=256) == ERR_INVALID                       # one source row per output row
    assert joint(Cs=256) == ERR_INVALID                               # the decoder's 512 only
    assert joint(rows_half=0) == ERR_INVALID
    assert joint(rows_half=4) == ERR_INVALID                          # rows_half >= rows
    assert joint(a2=None) == ERR_INVALID                              # add2 exactly when add
    assert joint(a=None) == ERR_INVALID
    assert joint(g2=None) == ERR_INVALID                              # gamma2 exactly when gamma
    # ld_add 0 (one add row for every output row) is accepted by the single entry too
    assert _op(ctx, 'alm_op_gather_ln', P(src), D, None, 1, D, 4, P(g), P(b), 1e-5, 0, P(add), 0, None, 0, P(hi), P(lo),
               D, P(hi), P(lo), None) == 0

    # the context still computes
    test_embed_ln_joint_against_fp64_and_two_single_launches(ctx, 13, 26, 34)
    test_gather_ln_joint_against_fp64_and_each_half_alone(ctx, 13, 'n1', 1e3)


# ----------------------------------------------------------------------------------------------- whole decodes
def _spot_model(wseed, bias):
    return omni_model(dict(wseed=wseed, pt_eos_bias=bias))


def _decode_launches(m, f):
    m.ctx.launch_count(reset=True)
    out = f()
    return out, m.ctx.launch_count(reset=True)


def joint_ab(m, run, what):
    """run() -> (result, launches of its decodes) with joint_decode 1 and 0, with graphs on and off, at xattn_impl 0 and
    2: bit for bit the same result, and fewer launches with the joint pass (it ran).  Returns the default run's result."""
    base = None
    for graphs in (1, 0):
        for xattn in (0, 2):
            got = {}
            for joint in (1, 0):
                with options(m.ctx, joint_decode=joint, use_graphs=graphs, xattn_impl=xattn):
                    got[joint] = run()
            label = f'{what}: use_graphs {graphs}, xattn_impl {xattn}'
            _assert_same(got[0][0], got[1][0], label + ', joint pass against the single-decoder loops')
            assert got[1][1] < got[0][1], (label, 'the joint pass did not run', got[1][1], got[0][1])
            if base is None:
                base = got[1][0]
    print(f'[joint] {what}: joint pass bit-identical to the single-decoder loops in 4 settings')
    return base


def _spotting_run(m, img, mask, extras=True):
    """encode, then the plain decode and, with extras, the decode with top-3 candidates and character locations"""
    def run():
        m.encode(img, mask)
        out, n = _decode_launches(m, m._decode_arrays)
        res = dict(plain=out)
        if extras:
            ext, n2 = _decode_launches(m, lambda: m._decode_arrays(rec_candidates=3, rec_locations=True))
            res.update(extras=ext, cand=m.last_rec_candidates, loc=m.last_rec_locations)
            n += n2
            m._set_rec_candidates(0)
        return res, n
    return run


def _case(name, golden_dir):
    from oracle.gen_golden import OMNI_CASES, omni_inputs
    case = OMNI_CASES[name]
    gold = np.load(os.path.join(golden_dir, f'omni_{name}.npz'))
    img, mask = omni_inputs(case)
    return case, gold, img, mask


def _set_lengths(m, pt_seq_length, rec_length):
    m.vocab.pt_seq_length, m.vocab.rec_length = pt_seq_length, rec_length


def _result(arrays, b):
    from advancedliteratemachinery_b200.omniparser import _spotting_result
    return _spotting_result(*(a[b] for a in arrays))


@pytest.mark.parametrize('name', ['full', 'masked', 'odd', 'oddlen'])
def test_fixture_decode_joint_equals_single_loops(name, golden_dir):
    case, gold, img, mask = _case(name, golden_dir)
    m = _spot_model(case['wseed'], case['pt_eos_bias'])
    _set_lengths(m, case['pt_seq_length'], case['rec_length'])
    base = joint_ab(m, _spotting_run(m, img, mask), f'omni {name}')
    _assert_fixture_ids(_result(base['plain'], 0), gold, name)
    _assert_fixture_ids(_result(base['extras'], 0), gold, name + ' with candidates and locations')


@pytest.mark.parametrize('rec_length', [32, 33, 40])
def test_recognition_loop_as_long_as_or_longer_than_the_polygon_loop(rec_length, golden_dir):
    """poly_length is 32: at 32 both loops end together, at 33 and 40 the recognition half finishes alone on its half
    of the joint buffers; 40 is the 'longrec' reference fixture"""
    case, gold, img, mask = _case('full', golden_dir)
    m = _spot_model(case['wseed'], case['pt_eos_bias'])
    _set_lengths(m, case['pt_seq_length'], rec_length)
    base = joint_ab(m, _spotting_run(m, img, mask), f'omni full, rec_length {rec_length}')
    if rec_length == 40:
        _, gold, _, _ = _case('longrec', golden_dir)
        _assert_fixture_ids(_result(base['plain'], 0), gold, 'longrec')
    else:   # the recognition ids of the first 25 steps are the 25-step fixture's
        assert np.array_equal(base['plain'][3][0, :, :25], gold['rec'][0])


def _regimes():
    """batches of the 'full' page (4 instances each) whose S = 4 B rows per decoder put the self-attention step in each
    regime of the joint pass's decoder step: both halves and the joint rows on the wide kernel (S <= SMs / 4), one launch per half
    (SMs / 4 < S <= SMs / 2), none on the wide kernel (S > SMs / 2)"""
    sms = support.sms()
    return {'one_wide_launch': (sms // 4) // 4, 'per_half_launches': (sms // 2) // 4, 'one_launch': (sms // 2) // 4 + 1}


@pytest.mark.parametrize('regime', ['one_wide_launch', 'per_half_launches', 'one_launch'])
def test_self_attention_regimes_of_the_sm_count(regime, golden_dir):
    case, gold, img, mask = _case('full', golden_dir)
    B = _regimes()[regime]
    S, sms = 4 * B, support.sms()
    assert {'one_wide_launch': S <= sms / 4, 'per_half_launches': sms / 4 < S <= sms / 2,
            'one_launch': S > sms / 2}[regime], (regime, S, sms)
    m = _spot_model(case['wseed'], case['pt_eos_bias'])
    _set_lengths(m, case['pt_seq_length'], case['rec_length'])
    base = joint_ab(m, _spotting_run(m, img.repeat(B, 1, 1, 1), mask.repeat(B, 1, 1), extras=False),
                    f'omni full x {B} ({regime}, S = {S})')
    for b in range(B):
        _assert_fixture_ids(_result(base['plain'], b), gold, f'page {b}')


def test_one_instance_per_page_at_33_pages(golden_dir):
    """Ncap 1 with B * Ncap > 32: the joint pass's fp32-query cross-attention form"""
    case, gold, img, mask = _case('full', golden_dir)
    m = _spot_model(case['wseed'], case['pt_eos_bias'])
    _set_lengths(m, 2, case['rec_length'])
    B = 33
    base = joint_ab(m, _spotting_run(m, img.repeat(B, 1, 1, 1), mask.repeat(B, 1, 1)), f'omni full x {B}, one instance')
    n_inst = base['plain'][0]
    assert (n_inst == 1).all()
    assert np.array_equal(base['plain'][1][:, 0], np.repeat(gold['pt'].reshape(-1, 2)[:1], B, 0))


def test_pages_of_different_sizes(golden_dir):
    from advancedliteratemachinery_b200 import NestedTensor
    from tests.test_gpu_omni_pages import ORDER, fixture_batch
    from tests.test_pages_cpu import pages_case
    gold = pages_case(golden_dir)
    m = _spot_model(int(gold['wseed'][0]), float(gold['pt_eos_bias'][0]))
    _set_lengths(m, int(gold['pt_seq_length'][0]), int(gold['rec_length'][0]))
    _, (t, mask) = fixture_batch(gold)
    t, mask = t.cuda(), mask.cuda()
    base = joint_ab(m, lambda: _decode_launches(m, lambda: m.forward_pages(NestedTensor(t, mask))), 'omni pages')
    for i, b in enumerate(ORDER):
        if gold['n_inst'][b] == 0:
            assert base[i] is None, b
            continue
        (pt, poly, rec), _ = base[i]
        assert np.array_equal(pt.numpy(), gold[f'pt_{b}']) and np.array_equal(poly.numpy(), gold[f'poly_{b}']) and \
            np.array_equal(rec.numpy(), gold[f'rec_{b}']), b


def test_window_prompts(golden_dir):
    from tests.test_gpu_omni_prompts import check_against_fixture
    from tests.test_prompts_cpu import prompt_case, prompt_page
    gold = prompt_case(golden_dir)
    m = _spot_model(int(gold['wseed'][0]), float(gold['pt_eos_bias'][0]))
    _set_lengths(m, int(gold['pt_seq_length'][0]), int(gold['rec_length'][0]))
    pages = [prompt_page(gold, b) for b in range(2)]
    imgs, masks = torch.cat([p[0] for p in pages]), torch.cat([p[1] for p in pages])
    prompts = torch.from_numpy(gold['prompts'])

    def run():
        m.encode(imgs, masks)
        out, n = _decode_launches(m, lambda: m.decode_prompts(prompts, rec_candidates=2, rec_locations=True))
        return dict(out=out, cand=m.last_rec_candidates, loc=m.last_rec_locations), n

    try:
        base = joint_ab(m, run, 'omni decode_prompts')
    finally:
        m._set_rec_candidates(0)
    m.encode(imgs, masks)
    check_against_fixture(m, gold, base['out'])


def test_kie(golden_dir):
    from advancedliteratemachinery_b200 import NestedTensor
    from oracle.gen_golden import KIE_CASES, omni_inputs
    case = KIE_CASES['kie']
    gold = np.load(os.path.join(golden_dir, 'omni_kie.npz'))
    m = omni_model(case, kie=True)
    img, mask = omni_inputs(case)
    v = m.vocab
    seqs = [v.pt_prompt(), torch.tensor([[v.poly_sos_index]]), torch.tensor([[v.rec_sos_index]]),
            torch.tensor(case['canvas'])]

    def run():
        out, n = _decode_launches(m, lambda: m(NestedTensor(img, mask), seqs, rec_candidates=2))
        return dict(out=out, raw=m.last_kie_raw, cand=m.last_rec_candidates), n

    try:
        base = joint_ab(m, run, 'omni KIE')
    finally:
        m._set_rec_candidates(0)
    assert [r[0] for r in base['out']] == gold['texts'].tolist()
    assert [r[1] for r in base['out']] == gold['classes'].tolist()


def test_dense_pass_starting_past_page_0():
    """decode_dense re-reads only the saturated pages: with a batch where page 0 does not saturate, its polygon /
    recognition passes over the window rows start at img0 != 0"""
    from tests.test_gpu_dense import pages
    x = pages(8, seed=9).cuda()
    for bias in (0.3, 0.2, 0.1, 0.4, 0.05):
        m = _spot_model(0, bias)
        _set_lengths(m, 12, 25)
        m.encode(x, None)
        m.decode_dense()
        if any(k == 1 and i0 > 0 for k, i0, _, _ in m.last_dense.loops):
            break
    else:
        pytest.fail('no bias of the list gives a polygon / recognition pass that starts past page 0')

    def run():
        m.encode(x, None)
        out, n = _decode_launches(m, m._decode_dense_arrays)
        return dict(out=out, loops=m.last_dense.loops, grid=m.last_dense.grid), n

    joint_ab(m, run, f'omni decode_dense (pt_eos_bias {bias})')


def _perturbed_sd(kind):
    """the 'full' checkpoint with the recognition decoder's final norm moved off the shared one, or with the polygon and
    recognition position tables swapped: the two halves of the joint pass then differ where the fixtures' do not"""
    from tests.conftest import omni_sd
    sd = dict(omni_sd(0, -30.0))
    g = torch.Generator().manual_seed(77)
    if kind == 'rec_norm':
        for k in ('transformer.rec_decoder.norm.weight', 'transformer.rec_decoder.norm.bias'):
            sd[k] = sd[k] + 0.1 * torch.randn(sd[k].shape, generator=g)
        assert not torch.equal(sd['transformer.rec_decoder.norm.weight'], sd['transformer.poly_decoder.norm.weight'])
    else:
        p, r = 'transformer.embedding.poly_position_embeddings.weight', 'transformer.embedding.rec_position_embeddings.weight'
        sd[p], sd[r] = sd[r], sd[p]
    return sd


@pytest.mark.parametrize('kind', ['rec_norm', 'swapped_positions'])
def test_checkpoints_whose_halves_differ(kind, golden_dir):
    case, gold, img, mask = _case('full', golden_dir)
    from advancedliteratemachinery_b200 import OmniParserB200, OmniVocab
    close_models()   # one resident model at a time
    m = OmniParserB200(_perturbed_sd(kind), OmniVocab(), workspace_mb=4096)
    try:
        _set_lengths(m, case['pt_seq_length'], 40)
        base = joint_ab(m, _spotting_run(m, img, mask), f'omni full, {kind}, rec_length 40')
    finally:
        m.ctx.close()
    # the change reaches the decode: the probabilities are not the unchanged checkpoint's
    ref = _spot_model(0, -30.0)
    _set_lengths(ref, case['pt_seq_length'], 40)
    ref.encode(img, mask)
    unchanged = ref._decode_arrays()
    assert not np.array_equal(base['plain'][4], unchanged[4]), f'{kind} does not change the decode'
