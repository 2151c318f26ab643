"""GPU: OmniParser's decoder as a whole against an fp64 evaluation of the reference's decoder, fed the device's own
encoder outputs.

`oracle.omniparser_ref.decode_logits` runs in float64 on the memory, position embedding and key mask the device encoded
(`alm_omni_get_memory(0 / 1)`, the page shapes or the batch mask) and on the checkpoint in float64, so the encoder's
error is not part of the comparison (the encoder has its own bit-for-bit replay).  The same call in float32 on the same
inputs is the yardstick: it is what fp32 arithmetic achieves on this decoder, row by row.

Bound, per row (sequence, position), over the V logits of the row, with e32(row) = |f32 - f64|_inf(row):

    max|gpu - f64| <= C * (u / 2^-24) * max(e32(row), 2^-22 * max|f64(row)|),   C = 4

u is the relative error of the operands the device's products see.  At nsplit 3 every tensor-core operand is a bf16
(hi, lo) pair equal to its fp32 value to 2^-17 (DESIGN 2), and the decoder's cross-attention reads its K_c / V_c as such
pairs on the skinny fp32 step as well: u = 2^-17.  At nsplit 1 every operand is rounded once to bf16: u = 2^-9.  The
fp32 restatement perturbs each of its operations by at most 2^-24.  To first order the logits' error is linear in the
perturbations of the operations that feed them, with the same amplification (the row's conditioning) that turns the
fp32 restatement's perturbations into e32; perturbations u / 2^-24 times as large (2^7 at nsplit 3, 2^15 at nsplit 1)
give at most that multiple of its error, and the operations the device keeps in fp32 (LayerNorm, softmax, residuals,
the skinny step's GEMVs) only shrink it.  The 2^-22 term keeps a row whose fp32 restatement happens to round well from
demanding less than a few fp32 ulps of the row's largest logit.  C = 4 covers what one operand's u leaves out of a
product: both operands' errors and, at nsplit 3, the dropped lo * lo term (at most 2.5 u per product, where the fp32
restatement rounds each product once).

Greedy decodes (`forward_batch` at `bench.py`'s settings, `decode_points`, `decode_prompts`, KIE) are teacher-forced in
fp64 on their own ids, one pass per loop: every chosen id must be the fp64 argmax over the step's candidates, or, where
the fp64 top-1 / top-2 gap is at most twice the row's bound, the runner-up (counted and printed).  A logit error
of at most b moves a log-softmax by at most 2 b, so every returned probability p must satisfy
|p - p64| <= p64 * expm1(2 b) + 2^-22 p64 (the last term: the fp32 softmax itself).
"""
import json
import time

import pytest
import torch

from tests.support import options

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

C_BOUND = 4.0
FLOOR = 2.0 ** -22
# u / 2^-24 per nsplit: split pairs carry their fp32 value to 2^-17, single bf16 operands to 2^-9
OPERAND_SCALE = {3: 2.0 ** 7, 1: 2.0 ** 15}
GAP_SCREEN = 1e-2           # rows with a smaller fp64 top-2 gap get their fp32 yardstick (and so their bound) computed

_MODEL = {}
_SD64 = {}


@pytest.fixture(scope='module', autouse=True)
def _file_clock():
    t0 = time.time()
    yield
    print(f'\ntest_gpu_decoder_fp64: {time.time() - t0:.1f} s')
    _close_models()


def _close_models():
    for k in list(_MODEL):
        _MODEL.pop(k).ctx.close()


def _model(key, sd, vocab=None, workspace_mb=8192):
    """One resident OmniParserB200 at a time (the weights are 0.9 GB on the device)."""
    from advancedliteratemachinery_b200 import OmniParserB200, OmniVocab
    if key not in _MODEL:
        _close_models()
        torch.cuda.empty_cache()
        _MODEL[key] = OmniParserB200(sd, vocab or OmniVocab(), workspace_mb=workspace_mb)
    return _MODEL[key]


def _f64(sd):
    if id(sd) not in _SD64:
        _SD64.clear()
        _SD64[id(sd)] = (sd, {k: v.double() if v.is_floating_point() else v for k, v in sd.items()})
    return _SD64[id(sd)][1]


def _spot_sd(wseed=0, bias=-30.0):
    from tests.conftest import omni_sd
    return omni_sd(wseed, bias)


def ref_logits(sd, seq, mem, kpm, pos, kind, with_f32=True):
    """fp64 and fp32 restatements of Transformer.decode on one page's device memory / pos ([M, 512]) and key mask."""
    from oracle import omniparser_ref as O
    f64 = O.decode_logits(seq, mem.double(), kpm, pos.double(), _f64(sd), kind)
    f32 = O.decode_logits(seq, mem.float(), kpm, pos.float(), sd, kind) if with_f32 else None
    return f64, f32


def row_bound(f64, f32, nsplit=3):
    """C * (u / 2^-24) * max(|f32 - f64|_inf, 2^-22 max|f64|) per row."""
    base = torch.maximum((f32.double() - f64).abs().amax(-1), FLOOR * f64.abs().amax(-1))
    return C_BOUND * OPERAND_SCALE[nsplit] * base


def worst_ratio(got, f64, f32, nsplit):
    """max over rows of err / bound; every logit must be finite."""
    assert torch.isfinite(got).all(), 'non-finite logit'
    err = (got.double() - f64).abs().amax(-1)
    return float((err / row_bound(f64, f32, nsplit)).max())


# --------------------------------------------------------------------------------------------- teacher-forced logits
def tf_seqs(v, kind, n, length, seed):
    """n teacher-forced sequences of `length` tokens: the pt prompt then bin pairs; or [x, y, sos] then bins (poly) /
    characters, pad and rec_eos (rec), as the polygon and recognition loops see them."""
    g = torch.Generator().manual_seed(seed)
    nb = v.num_bins
    if kind == 'pt':
        prompt = v.pt_prompt().expand(n, -1)
        return torch.cat([prompt, torch.randint(0, nb, (n, length - prompt.shape[1]), generator=g)], 1)
    xy = torch.randint(0, nb, (n, 2), generator=g)
    sos = v.poly_sos_index if kind == 'poly' else v.rec_sos_index
    body = (torch.randint(0, nb, (n, length - 3), generator=g) if kind == 'poly'
            else torch.randint(nb, v.recog_pad_index + 1, (n, length - 3), generator=g))
    if kind == 'rec':
        body[:, -1] = v.rec_eos_index
    return torch.cat([xy, torch.full((n, 1), sos), body], 1)


def _scaled_q_sd(factor):
    """The spotting checkpoint with the point decoder's self-attention query projections scaled by `factor`: scores
    far above 100, so a wrong running maximum in the self-attention step would overflow or lose the row."""
    sd = dict(_spot_sd())
    for l in range(4):
        p = f'transformer.pt_decoder.layers.{l}.self_attn.'
        w, b = sd[p + 'in_proj_weight'].clone(), sd[p + 'in_proj_bias'].clone()
        w[:512] *= factor
        b[:512] *= factor
        sd[p + 'in_proj_weight'], sd[p + 'in_proj_bias'] = w, b
    return sd


def _fixture_page(name):
    from oracle.gen_golden import OMNI_CASES, omni_inputs
    return omni_inputs(OMNI_CASES[name])


# page: checkpoint (key, state-dict factory), how the page is encoded, and the (kind, length, n_seq) teacher-forced
# cases, each run under every xattn_impl and nsplit listed
TF_PAGES = {
    'odd': dict(ckpt=('w1', lambda: _spot_sd(1)), enc='odd', cases=[('pt', 15, (1, 2, 17, 65)), ('poly', 35, (1, 2, 17, 65)),
                                                                   ('rec', 28, (1, 2, 17, 65))], nsplit=(3, 1)),
    'masked': dict(ckpt=('w0', _spot_sd), enc='masked', cases=[('pt', 15, (1, 2, 17, 65)), ('poly', 35, (1, 2, 17, 65)),
                                                              ('rec', 28, (1, 2, 17, 65))], nsplit=(3, 1)),
    'mixed_last': dict(ckpt=('w0', _spot_sd), enc='mixed', cases=[('pt', 15, (1, 2, 17, 65)), ('poly', 35, (1, 2, 17, 65)),
                                                                 ('rec', 28, (1, 2, 17, 65))], nsplit=(3,)),
    'page1024': dict(ckpt=('w0', _spot_sd), enc=1024, cases=[('pt', 39, (1, 2, 17, 65)), ('poly', 35, (1, 2, 17, 65)),
                                                            ('rec', 28, (1, 2, 17, 65))], nsplit=(3,)),
    # the table form: a 7-token prompt plus 512 tokens, positions 0 .. 518
    'page1920': dict(ckpt=('w0', _spot_sd), enc=1920, cases=[('pt', 519, (1, 2))], nsplit=(3,)),
    # the position table's last row, with self-attention scores far above 100
    'pos1023': dict(ckpt=('q16', lambda: _scaled_q_sd(16.0)), enc='masked', cases=[('pt', 1024, (1, 2))], nsplit=(3,)),
}

MIXED_SIZES = [(640, 512), (200, 300), (480, 352)]


def _encode(m, enc):
    """Encode one page (or the mixed batch) and return (image index, memory [M, 512], pos, key mask [M]) as encoded."""
    from oracle import omniparser_ref as O
    if enc == 'mixed':
        g = torch.Generator().manual_seed(4242)
        Hc, Wc = max(h for h, _ in MIXED_SIZES), max(w for _, w in MIXED_SIZES)
        imgs = torch.zeros(len(MIXED_SIZES), 3, Hc, Wc)
        for b, (h, w) in enumerate(MIXED_SIZES):
            imgs[b, :, :h, :w] = torch.randn(3, h, w, generator=g)
        shapes = m.encode_pages(imgs, MIXED_SIZES)
        b = len(MIXED_SIZES) - 1
        Mb = shapes[b][0] * shapes[b][1]
        assert Mb < max(sh[0] * sh[1] for sh in shapes), 'the last page must not be the largest'
        return b, m.memory(0)[b, :Mb], m.memory(1)[b, :Mb], torch.zeros(Mb, dtype=torch.bool)
    if isinstance(enc, int):
        img = torch.randn(1, 3, enc, enc, generator=torch.Generator().manual_seed(enc))
        mask = torch.zeros(1, enc, enc, dtype=torch.bool)
    else:
        img, mask = _fixture_page(enc)
    _, h, w = m.encode(img, mask)
    kpm = O.level_mask(mask, (h, w)).flatten(1)[0]
    return 0, m.memory(0)[0], m.memory(1)[0], kpm


def _assert_large_self_attention_scores(sd, v):
    """The pos1023 case's premise: the point decoder's first self-attention scores exceed 100 (fp64, CPU)."""
    import torch.nn.functional as F
    from oracle import omniparser_ref as O
    sd = _f64(sd)
    seq = tf_seqs(v, 'pt', 1, 64, seed=1)[0]
    t = 'transformer.'
    pe = sd[t + 'embedding.pt_position_embeddings.weight'][:64]
    x = O._ln(sd[t + 'embedding.word_embeddings.weight'][seq] + pe, sd, t + 'embedding.LayerNorm')
    p = t + 'pt_decoder.layers.0.'
    h = O._ln(x, sd, p + 'norm1') + pe
    w, b = sd[p + 'self_attn.in_proj_weight'], sd[p + 'self_attn.in_proj_bias']
    q = F.linear(h, w[:512], b[:512]).view(64, 8, 64).transpose(0, 1) / 8
    k = F.linear(h, w[512:1024], b[512:1024]).view(64, 8, 64).transpose(0, 1)
    top = float((q @ k.transpose(1, 2)).abs().max())
    assert top > 100, top


@pytest.mark.parametrize('page', list(TF_PAGES))
def test_teacher_forced_logits_against_fp64(page):
    """Teacher-forced logits of every position of pt / poly / rec sequences against fp64, on the skinny fp32 GEMV step
    (n_seq 1) and the tensor-core step with 16- and 64-row query blocks (2, 17, 65), under xattn_impl 0, 1 and 2."""
    t0 = time.time()
    spec = TF_PAGES[page]
    key, sd_fn = spec['ckpt']
    sd = sd_fn()
    m = _model(key, sd, workspace_mb=16384)
    if page == 'pos1023':
        _assert_large_self_attention_scores(sd, m.vocab)
    report, worst = {}, 0.0
    for nsplit in spec['nsplit']:
        # xattn_impl 1 for the encode: the unfused path's V_c^T is built by the encode; 0 and 2 ignore it
        with options(m.ctx, nsplit=nsplit, xattn_impl=1):
            image, mem, pos, kpm = _encode(m, spec['enc'])
            for kind, length, ns in spec['cases']:
                seq = tf_seqs(m.vocab, kind, max(ns), length, seed=length + len(kind))
                f64, f32 = ref_logits(sd, seq, mem, kpm, pos, kind)
                for impl in (0, 1, 2):
                    m.ctx.set_option('xattn_impl', impl)
                    for n in ns:
                        got = m.decode_logits(image, kind, seq[:n])
                        r = worst_ratio(got, f64[:n], f32[:n], nsplit)
                        report[f'{kind} n{n} x{impl} s{nsplit}'] = round(r, 4)
                        worst = max(worst, r)
    print(f'{page}: worst err/bound {worst:.4f} ({time.time() - t0:.1f} s)', json.dumps(report))
    bad = {k: r for k, r in report.items() if r > 1.0}
    assert not bad, bad


# --------------------------------------------------------------------------------------------- greedy decodes
def judge(kind, seq, s0, f64, cands, n_prompt_steps=0, bound_fn=None, tag=''):
    """Every chosen id seq[:, s0 + t] against the fp64 argmax of row s0 - 1 + t over cands(t).  Returns
    (mismatching (seq, t) list, near-tie rows accepted, smallest gap).  bound_fn(rows) -> [len(rows)] bounds, asked for
    only on the sequences of near-tie or mismatching steps."""
    n, T = seq.shape
    steps = T - s0
    V = f64.shape[-1]
    allowed = torch.stack([cands(t + n_prompt_steps, V) for t in range(steps)])
    lg = f64[:, s0 - 1:T - 1].masked_fill(~allowed[None], float('-inf'))
    top = lg.topk(2, -1)
    ids = seq[:, s0:]
    gap = top.values[..., 0] - top.values[..., 1]
    hit = top.indices[..., 0] == ids
    look = (~hit) | (gap < GAP_SCREEN)
    near, flips = [], []
    rows = sorted(set(int(r) for r in look.nonzero()[:, 0])) if bool(look.any()) else []
    if rows:
        b = bound_fn(rows)   # [len(rows), T]
        for i, r in enumerate(rows):
            for t in range(steps):
                bt = float(b[i, s0 - 1 + t])
                if float(gap[r, t]) <= 2 * bt:
                    near.append(dict(kind=kind, seq=r, step=t, gap=float(gap[r, t]), bound=bt, runner_up=not bool(hit[r, t])))
                elif not bool(hit[r, t]):
                    flips.append(dict(kind=kind, seq=r, step=t, gap=float(gap[r, t]), bound=bt))
                if not bool(hit[r, t]):
                    assert int(ids[r, t]) == int(top.indices[r, t, 1]), f'{tag} {kind} seq {r} step {t}: not the top two'
    assert not flips, f'{tag}: ids that are not the fp64 argmax away from a near-tie: {flips[:5]}'
    return near, float(gap.min()) if gap.numel() else float('inf')


def check_probs(got, ids, f64, bound, s0, tag, nsoft=None):
    """Returned probabilities [n, steps] of ids [n, steps] against the fp64 softmax of rows s0 - 1 + t (over the first
    nsoft logits for the KIE polygon / recognition loops), within what a logit error of `bound` (per row) moves them."""
    n, steps = ids.shape
    lg = f64[:, s0 - 1:s0 - 1 + steps]
    if nsoft is not None:
        lg = lg[..., :nsoft]
    p64 = lg.softmax(-1).gather(-1, ids[..., None])[..., 0]
    b = bound[:, s0 - 1:s0 - 1 + steps]
    tol = p64 * torch.expm1(2 * b) + FLOOR * p64
    err = (got.double() - p64).abs()
    worst = float((err / tol).max())
    assert worst <= 1.0, f'{tag}: probability off by {worst:.3g} x its bound'
    return worst


def check_spotting(m, sd, image, mem, kpm, pos, out, tag, prompt=None):
    """One page's greedy output ([pt, poly, rec], [probs]) teacher-forced in fp64: ids and rec probabilities."""
    from oracle import omniparser_ref as O
    v = m.vocab
    (pt, poly, rec), (probs,) = out
    n = pt.numel() // 2
    prompt = v.pt_prompt() if prompt is None else prompt
    full = {'pt': torch.cat([prompt, pt.reshape(1, -1)], 1),
            'poly': torch.cat([pt.reshape(-1, 2), torch.full((n, 1), v.poly_sos_index), poly.reshape(n, 32)], 1),
            'rec': torch.cat([pt.reshape(-1, 2), torch.full((n, 1), v.rec_sos_index), rec.reshape(n, -1)], 1)}
    start = {'pt': prompt.shape[1], 'poly': 3, 'rec': 3}
    near, gaps, pw = [], {}, None
    for kind, seq in full.items():
        f64, _ = ref_logits(sd, seq, mem, kpm, pos, kind, with_f32=False)

        def bound_fn(rows, seq=seq, f64=f64, kind=kind):
            _, f32 = ref_logits(sd, seq[rows], mem, kpm, pos, kind, with_f32=True)
            return row_bound(f64[rows], f32)
        nr, gaps[kind] = judge(kind, seq, start[kind], f64, lambda t, V, k=kind: O.step_candidates(k, t, V),
                               bound_fn=bound_fn, tag=tag)
        near += nr
        if kind == 'rec':
            _, f32 = ref_logits(sd, seq, mem, kpm, pos, kind)
            pw = check_probs(probs, rec.reshape(n, -1), f64, row_bound(f64, f32), 3, tag)
    return dict(instances=n, near_ties=near, min_gap={k: round(g, 6) for k, g in gaps.items()},
                prob_err_over_bound=round(pw, 4))


def _bench_model(ws, pt_len):
    from advancedliteratemachinery_b200 import OmniVocab
    m = _model(('bench', ws), _spot_sd(), OmniVocab(pt_seq_length=pt_len, rec_length=25), workspace_mb=ws)
    m.vocab.pt_seq_length, m.vocab.rec_length = pt_len, 25
    return m


def _batch_pages(name):
    """(pages [B, 3, H, W], pages to check, workspace MB, pt_seq_length).  The 16-page batch is checked in quarters,
    each well within the per-test time limit."""
    from oracle.gen_golden import CONFIG2_CASE, config2_page
    if name.startswith('batch512x768'):
        q = int(name[-1])
        return (torch.randn(16, 3, 512, 768, generator=torch.Generator().manual_seed(768)), list(range(4 * q, 4 * q + 4)),
                20480, 128)
    if name == 'config2':
        s = CONFIG2_CASE['seed']
        return torch.cat([config2_page(s + i)[0] for i in range(16)]), [0, 7, 15], 20480, 128
    if name == 'platypus':   # bench.py's page p: randn seeded 1000 + p
        return torch.cat([torch.randn(1, 3, 896, 896, generator=torch.Generator().manual_seed(1000 + p))
                          for p in range(8)]), [7], 16384, 128
    raise KeyError(name)


@pytest.mark.parametrize('name', [f'batch512x768_{q}' for q in range(4)] + ['config2', 'platypus'])
def test_every_greedy_step_of_batched_decodes_is_the_fp64_argmax(name):
    """forward_batch as bench.py runs it (graphs on, default knobs, the joint polygon + recognition pass): every pt, poly
    and rec step of the checked pages is the fp64 argmax of its candidates, or a judged near-tie; rec_prob within the
    bound."""
    from advancedliteratemachinery_b200 import NestedTensor
    t0 = time.time()
    pages, check, ws, pt_len = _batch_pages(name)
    m = _bench_model(ws, pt_len)
    sd = _spot_sd()
    outs = m.forward_batch(NestedTensor(pages.pin_memory(), None))
    mem, pos = m.memory(0), m.memory(1)
    kpm = torch.zeros(mem.shape[1], dtype=torch.bool)
    report = {}
    for b in check:
        assert outs[b] is not None and outs[b][0][0].numel() == 2 * (pt_len // 2), f'page {b}: the pinned length'
        report[b] = check_spotting(m, sd, b, mem[b], kpm, pos[b], outs[b], f'{name} page {b}')
    n_near = sum(len(r['near_ties']) for r in report.values())
    print(f'{name}: {n_near} near-tie steps accepted ({time.time() - t0:.1f} s)', json.dumps(report))


def test_table_point_sequence_every_step():
    """bench.py's `table` batch: 8 x 1920^2, one 512-token point sequence per page (decode_points); the last page's
    every step against fp64, and its probabilities."""
    from oracle import omniparser_ref as O
    t0 = time.time()
    m = _bench_model(40960, 512)
    pages = torch.cat([torch.randn(1, 3, 1920, 1920, generator=torch.Generator().manual_seed(1000 + p)) for p in range(8)])
    m.encode(pages.pin_memory(), None)
    tok, prob = m.decode_points()[7]
    assert tok.numel() == 512
    mem, pos = m.memory(0)[7], m.memory(1)[7]
    kpm = torch.zeros(mem.shape[0], dtype=torch.bool)
    seq = torch.cat([m.vocab.pt_prompt(), tok.reshape(1, -1)], 1)
    sd = _spot_sd()
    f64, f32 = ref_logits(sd, seq, mem, kpm, pos, 'pt')
    bound = row_bound(f64, f32)
    near, gap = judge('pt', seq, 7, f64, lambda t, V: O.step_candidates('pt', t, V),
                      bound_fn=lambda rows: bound[rows], tag='table page 7')
    pw = check_probs(prob.reshape(1, -1), tok.reshape(1, -1), f64, bound, 7, 'table page 7')
    print(f'table page 7: {len(near)} near-tie steps, min gap {gap:.3g}, prob err/bound {pw:.4f} '
          f'({time.time() - t0:.1f} s)', json.dumps(near))


def test_window_prompts_every_step():
    """decode_prompts with four window prompts on each of two pages: every (page, prompt) slot's steps against fp64 on
    its own prompt."""
    t0 = time.time()
    m = _bench_model(8192, 24)
    v = m.vocab
    g = torch.Generator().manual_seed(31)
    pages = torch.randn(2, 3, 256, 320, generator=g)
    prompts = torch.cat([v.window_prompt(), v.window_prompt((0, 0, 160, 128), (256, 320)),
                         v.window_prompt((100, 60, 320, 256), (256, 320)), v.window_prompt(chars=(v.chars[10], v.chars[40]))])
    m.encode(pages, None)
    outs = m.decode_prompts(prompts)
    mem, pos = m.memory(0), m.memory(1)
    kpm = torch.zeros(mem.shape[1], dtype=torch.bool)
    sd = _spot_sd()
    report, slots = {}, 0
    for b in range(2):
        for p in range(prompts.shape[0]):
            if outs[b][p] is None:
                continue
            slots += 1
            report[f'{b}_{p}'] = check_spotting(m, sd, b, mem[b], kpm, pos[b], outs[b][p], f'prompt {b}/{p}',
                                                prompt=prompts[p:p + 1])
    assert slots >= 4
    print(f'window prompts: {slots} slots ({time.time() - t0:.1f} s)', json.dumps(report))


def test_kie_fixture_every_step():
    """The KIE fixture (x, y, class point loop; polygon and transcription per pair with the class logits left out of the
    softmax): every step against fp64 under the KIE candidate rules, and the point probabilities."""
    from advancedliteratemachinery_b200 import NestedTensor, OmniVocab
    from advancedliteratemachinery_b200 import synthetic as SW
    from oracle import omniparser_ref as O
    from oracle.gen_golden import KIE_CASES, omni_inputs
    t0 = time.time()
    case = KIE_CASES['kie']
    vie = case['vie']
    v = OmniVocab(vie_categories=vie, pt_seq_length=case['pt_seq_length'], rec_length=case['rec_length'])
    sd = SW.omniparser_state_dict(seed=case['wseed'], vie_categories=vie, pt_eos_bias=case['pt_eos_bias'])
    m = _model('kie', sd, v)
    img, mask = omni_inputs(case)
    m(NestedTensor(img, mask), [v.pt_prompt(), torch.tensor([[v.poly_sos_index]]), torch.tensor([[v.rec_sos_index]]),
                               torch.tensor(case['canvas'])])
    raw = m.last_kie_raw
    _, h, w = m.memory_shape()
    mem, pos = m.memory(0)[0], m.memory(1)[0]
    kpm = O.level_mask(mask, (h, w)).flatten(1)[0]
    nt = int(raw['n_tok'][0])
    assert nt > 0
    tok = torch.from_numpy(raw['tokens'][0, :nt]).long()
    seq = torch.cat([v.pt_prompt(), tok[None]], 1)
    nb, eos = v.num_bins, v.pt_eos_index

    def pt_cands(t, V):   # transformer.py:117-123
        a = torch.zeros(V, dtype=torch.bool)
        if t % 3 == 0:
            a[:nb] = True
            a[eos] = True
        elif t % 3 == 1:
            a[:nb] = True
        else:
            a[V - vie:] = True
        return a
    f64, f32 = ref_logits(sd, seq, mem, kpm, pos, 'pt')
    bound = row_bound(f64, f32)
    near, _ = judge('pt', seq, 7, f64, pt_cands, bound_fn=lambda rows: bound[rows], tag='kie')
    pw = check_probs(torch.from_numpy(raw['probs'][0, :nt])[None], tok[None], f64, bound, 7, 'kie pt')
    ni = int(raw['n_inst'][0])
    assert ni > 0
    for n in range(ni):
        i = int(raw['inst_pos'][0, n])
        xy = tok[i:i + 2][None]
        for kind, sos, ids in (('poly', v.poly_sos_index, raw['poly'][0, n]), ('rec', v.rec_sos_index, raw['rec'][0, n])):
            s = torch.cat([xy, torch.tensor([[sos]]), torch.from_numpy(ids).long()[None]], 1)
            f64k, f32k = ref_logits(sd, s, mem, kpm, pos, kind)
            bk = row_bound(f64k, f32k)
            V = f64k.shape[-1]

            def cands(t, V_, kind=kind):   # the class logits are outside the softmax: never candidates
                a = O.step_candidates(kind, t, V_)
                a[V_ - vie:] = False
                return a
            nr, _ = judge(kind, s, 3, f64k, cands, bound_fn=lambda rows, bk=bk: bk[rows], tag=f'kie inst {n}')
            near += nr
            if kind == 'rec':
                check_probs(torch.from_numpy(raw['rec_prob'][0, n])[None], s[:, 3:], f64k, bk, 3, f'kie rec {n}',
                            nsoft=V - vie)
    print(f'kie: {ni} instances, {len(near)} near-tie steps, pt prob err/bound {pw:.4f} ({time.time() - t0:.1f} s)')
