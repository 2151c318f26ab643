"""GPU: the decoder's per-token kernels against plain fp64 references, through their op-level entry points.

The decode tests check these kernels end to end (fixtures, teacher-forced logits) and against each other; a mistake two
variants share passes the second kind of check.  Here every kernel is compared with the same operation in fp64, at the
shapes where its schedule changes and at the edges of its arithmetic:

* cross-attention (xattn.cu, xattn_tma.cu, the single-query kernel): 16- and 64-row query blocks with dead rows, whole
  64-key blocks and whole CTA runs masked (a page padded inside a batch), one live key, the row maximum in the first,
  the last or a masked key, pairs stored by one CTA, pairs merged from several, runs crossing pair boundaries, both
  split schemes, replay on the same partial / counter buffers, and NaN in every cache element the call must not read
  (other decoder layers, other images, V^T's pad columns);
* the self-attention step up to the last position of the table, with scores large enough that a wrong block maximum
  overflows expf;
* the skinny GEMV with every row capacity and K width, N not a multiple of 4, the x / x2 column split and the fused
  LayerNorm + query position (bit for bit against LayerNorm followed by the plain GEMV);
* token selection at the edges of every candidate range, with ties, forbidden maxima and -inf logits.

Every output buffer is followed by a guard region that must come back bit for bit unchanged.  Shapes that depend on the
schedule are derived from the SM count, so the cases hold on any H100.
"""
import ctypes as C

import pytest
import torch

from tests.support import NAN, assert_guard, bits, ctx, guarded, options, sms

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

WORKSPACE_MB = 8192  # the largest cross-attention case builds 3.2 GB of caches
ERR_INVALID, ERR_UNSUPPORTED = -1, -5


def _ptr(t):
    return None if t is None else t.data_ptr()


def _op(ctx, name, *args):
    """Call an entry point once torch's queued work is done: the context runs on its own non-blocking stream (and
    synchronizes it before returning)."""
    torch.cuda.synchronize()
    return getattr(ctx.lib, name)(ctx.h, *args)


# ----------------------------------------------------------------------------------------------- cross-attention
# (xattn_impl, nsplit, xattn_wg, xattn_ctas_per_sm, q_split, Ncap, M, images, mask)
# images: (nimg_total, img0, nimg), or 'wide': npairs >= 2 x SMs (whole pairs inside one CTA's run)
XATTN_CASES = [
    # the point loop's form: fp32 queries, the 16-row kernel (one warp per 16 keys of a block)
    (0, 3, 1, 2, 0, 1, 40, (3, 1, 2), 'right'),
    (0, 3, 1, 2, 0, 5, 255, (3, 1, 2), 'bottom'),
    (0, 3, 1, 2, 0, 16, 4096, (4, 1, 3), 'one'),
    (0, 1, 1, 2, 0, 16, 256, (3, 1, 2), 'none'),
    (0, 3, 1, 1, 0, 1, 14400, (4, 1, 3), 'bottom'),   # the config-5 page
    (0, 3, 1, 3, 0, 5, 64, (3, 1, 2), 'max_masked'),
    (2, 3, 1, 2, 0, 1, 255, (3, 1, 2), 'right'),
    (2, 3, 1, 2, 0, 16, 4096, (4, 1, 3), 'bottom'),
    (2, 1, 1, 2, 0, 5, 40, (3, 1, 2), 'one'),
    (2, 3, 1, 2, 0, 16, 64, (3, 1, 2), 'max_masked'),
    (1, 3, 1, 2, 0, 1, 255, (3, 1, 2), 'bottom'),     # M % 8 != 0: the last key group reaches V^T's pad columns
    (1, 3, 1, 2, 0, 1, 4096, (3, 1, 2), 'one'),
    (1, 1, 1, 2, 0, 1, 40, (3, 1, 2), 'max_masked'),
    (1, 3, 1, 2, 1, 1, 255, (3, 1, 2), 'right'),
    # the poly / rec form: split queries and output planes
    (0, 3, 1, 2, 1, 5, 4096, (3, 1, 2), 'none'),
    (0, 3, 1, 2, 1, 17, 255, (2, 1, 1), 'bottom'),    # fewer key blocks than the grid: every pair split over 4 CTAs
    (0, 3, 2, 2, 1, 17, 255, (2, 1, 1), 'bottom'),
    (0, 3, 1, 1, 1, 65, 256, 'wide', 'right'),        # one CTA stores whole multi-block pairs (gs == 1)
    (0, 3, 1, 1, 1, 64, 256, 'wide', 'bottom'),
    (0, 3, 2, 2, 1, 65, 4096, (4, 1, 3), 'one'),      # runs of ~11 blocks crossing pair boundaries
    (0, 1, 1, 2, 1, 130, 255, (3, 1, 2), 'max_masked'),
    (0, 3, 1, 3, 1, 130, 4096, (3, 1, 2), 'bottom'),
    (2, 3, 1, 2, 1, 17, 255, (2, 1, 1), 'bottom'),
    (2, 3, 1, 2, 1, 65, 4096, (4, 1, 3), 'right'),
    (2, 1, 1, 2, 1, 130, 64, (3, 1, 2), 'one'),
    (2, 3, 1, 2, 1, 64, 256, 'wide', 'none'),
]


def _xattn_id(c):
    impl, ns, wg, cps, qs, ncap, M, imgs, mask = c
    return f'impl{impl}-ns{ns}-wg{wg}-cps{cps}-{"split" if qs else "f32"}-N{ncap}-M{M}-{mask}' + \
        ('-wide' if imgs == 'wide' else f'-img{imgs[1]}x{imgs[2]}')


def _key_mask(kind, total, M):
    """u8 [total, M], 1 = padding key; images of odd index stay unpadded under 'bottom' (pages of a batch differ)"""
    if kind == 'none':
        return None
    m = torch.zeros(total, M, dtype=torch.uint8, device='cuda')
    for i in range(total):
        if kind in ('right', 'max_masked'):
            m[i, M - max(1, (i % 3 + 1) * M // 7):] = 1
        elif kind == 'bottom' and i % 2 == 0:
            live = max(1, (M // 2) // 64 * 64 if M >= 128 else M // 2)   # whole 64-key blocks and CTA runs masked
            m[i, live:] = 1
        elif kind == 'one':
            m[i] = 1
            m[i, (M // 3 + 17 * i) % M] = 0
    return m


def _plant(q, k, kpm, img0, M, score=20.0):
    """Query rows 0, 1, 2 of every image get a key with score `score` (tens above the rest): key 0 (first block), the
    last live key (last live block) and key M-1 (masked under 'right' / 'max_masked')."""
    nimg, ncap = q.shape[0], q.shape[1]
    for i in range(nimg):
        live = (kpm[img0 + i] == 0).nonzero().flatten() if kpm is not None else None
        last = int(live[-1]) if live is not None else M - 1
        for n, key in enumerate((0, last, M - 1)[:ncap]):
            qh = q[i, n].view(8, 64)
            k[img0 + i, key] = (8 * score * qh / (qh * qh).sum(-1, keepdim=True)).flatten()


def _xattn_ref(q, k, v, kpm, img0):
    nimg, ncap = q.shape[0], q.shape[1]
    M = k.shape[1]
    qh = q.double().view(nimg, ncap, 8, 64).transpose(1, 2)
    kh = k[img0:img0 + nimg].double().view(nimg, M, 8, 64).transpose(1, 2)
    vh = v[img0:img0 + nimg].double().view(nimg, M, 8, 64).transpose(1, 2)
    s = (qh / 8) @ kh.transpose(-1, -2)
    if kpm is not None:
        s = s.masked_fill(kpm[img0:img0 + nimg, None, None, :].bool(), float('-inf'))
    return (s.softmax(-1) @ vh).transpose(1, 2).reshape(nimg, ncap, 512)


def _run_xattn(ctx, q, k, v, kpm, img0, M, dl, q_split, launches):
    nimg, ncap = q.shape[0], q.shape[1]
    n = nimg * ncap * 512
    out, full = guarded(n)
    ctx.check(_op(ctx, 'alm_op_cross_attention', q.data_ptr(), k.data_ptr(), v.data_ptr(), _ptr(kpm), out.data_ptr(),
                  k.shape[0], img0, nimg, ncap, M, dl, q_split, launches))
    assert_guard(full, n)
    return out.view(nimg, ncap, 512).clone()


@pytest.mark.parametrize('case', XATTN_CASES, ids=_xattn_id)
def test_cross_attention_matches_fp64(ctx, case):
    impl, nsplit, wg, cps, q_split, ncap, M, imgs, mask = case
    if imgs == 'wide':
        nqb = (ncap + 63) // 64
        nimg = -(-2 * sms() // (8 * nqb)) + 1
        imgs = (nimg + 1, 1, nimg)
    total, img0, nimg = imgs
    assert total * M <= 65536
    g = torch.Generator(device='cuda').manual_seed(M * 131 + ncap)
    q = torch.randn(nimg, ncap, 512, generator=g, device='cuda') * 2      # scores span tens of units
    k = torch.randn(total, M, 512, generator=g, device='cuda') * 2
    v = torch.randn(total, M, 512, generator=g, device='cuda')
    kpm = _key_mask(mask, total, M)
    _plant(q, k, kpm, img0, M)
    ref = _xattn_ref(q, k, v, kpm, img0)
    tol = 3e-5 if nsplit == 3 else 2e-2
    with options(ctx, xattn_impl=impl, nsplit=nsplit, xattn_wg=wg, xattn_ctas_per_sm=cps):
        for dl in (0, 11):
            got = _run_xattn(ctx, q, k, v, kpm, img0, M, dl, q_split, 1)
            assert torch.isfinite(got).all(), f'dl {dl}: {int((~torch.isfinite(got)).sum())} non-finite outputs'
            err = float((got.double() - ref).abs().max() / ref.abs().max())
            assert err <= tol, (dl, err)
        again = _run_xattn(ctx, q, k, v, kpm, img0, M, 11, q_split, 2)   # replay on the same partials / counters
        assert torch.equal(bits(again), bits(got))


def test_cross_attention_argument_errors(ctx):
    q = torch.zeros(2, 17, 512, device='cuda')
    kv = torch.zeros(3, 64, 512, device='cuda')
    out = torch.zeros_like(q)

    def call(**kw):
        a = dict(nimg_total=3, img0=1, nimg=2, Ncap=17, M=64, dl=0, q_split=1, launches=1)
        a.update(kw)
        return _op(ctx, 'alm_op_cross_attention', q.data_ptr(), kv.data_ptr(), kv.data_ptr(), None, out.data_ptr(),
                   a['nimg_total'], a['img0'], a['nimg'], a['Ncap'], a['M'], a['dl'],
                   a['q_split'], a['launches'])
    assert call() == 0
    assert call(img0=2) == ERR_INVALID         # images past nimg_total
    assert call(dl=12) == ERR_INVALID
    assert call(q_split=0) == ERR_INVALID      # fp32 queries are the <= 16-row form
    assert call(launches=0) == ERR_INVALID
    assert call(M=0) == ERR_INVALID
    with options(ctx, xattn_impl=1):
        assert call() == ERR_UNSUPPORTED       # the unfused multi-query path is GEMM + softmax_rows
        assert call(Ncap=1, nimg=1) == 0


# ----------------------------------------------------------------------------------------------- self-attention step
def _s_values():
    last_wide = 4 * sms() // 8                 # the wide kernel serves 8 S <= 4 SMs
    return {'1': 1, '16': 16, 'last_wide': last_wide, 'first_narrow': last_wide + 1, '300': 300}


@pytest.mark.parametrize('wide', [0, 1])
@pytest.mark.parametrize('S_name', ['1', '16', 'last_wide', 'first_narrow', '300'])
def test_self_attention_step_matches_fp64(ctx, S_name, wide):
    S = _s_values()[S_name]
    cases = sorted({(t, tm) for t in (0, 1, 31, 32, 127, 128, 1023) for tm in (t + 1, 1024)})
    with options(ctx, sattn_wide=wide):
        for t, Tmax in cases:
            g = torch.Generator(device='cuda').manual_seed(t * 7 + Tmax + S)
            qkv = torch.randn(S, 1536, generator=g, device='cuda') * 2
            qkv[:, 1024:] /= 2
            K = torch.randn(S, t + 1, 512, generator=g, device='cuda') * 2
            V = torch.randn(S, t + 1, 512, generator=g, device='cuda')
            K[:, t] = qkv[:, 512:1024]
            V[:, t] = qkv[:, 1024:]
            # scores of 150 (at position 100, held by the 3rd warp of the wide kernel, or at t) and -120 at position 0:
            # a block maximum that misses a warp overflows expf
            big = 100 if t >= 100 else t
            qh = qkv[:, :512].view(S, 8, 64)
            unit = (8 * qh / (qh * qh).sum(-1, keepdim=True)).reshape(S, 512)   # q . unit / 8 == 1 in every head
            K[0::3, big] = 150 * unit[0::3]
            if t > 0:
                K[1::3, 0] = -120 * unit[1::3]
            qkv[:, 512:1024] = K[:, t]
            n = S * Tmax * 512
            kc, kfull = guarded(n)
            vc, vfull = guarded(n)
            kc.view(S, Tmax, 512)[:, :t] = K[:, :t]
            vc.view(S, Tmax, 512)[:, :t] = V[:, :t]
            kbefore, vbefore = kc.clone(), vc.clone()
            out, ofull = guarded(S * 512)
            ctx.check(_op(ctx, 'alm_op_self_attention_step', qkv.data_ptr(), kc.data_ptr(), vc.data_ptr(),
                          out.data_ptr(), S, t, Tmax))
            for full in (kfull, vfull):
                assert_guard(full, n)
            for after, before, new in ((kc, kbefore, qkv[:, 512:1024]), (vc, vbefore, qkv[:, 1024:])):
                a, b = after.view(S, Tmax, 512), before.view(S, Tmax, 512)
                assert torch.equal(bits(a[:, t].contiguous()), bits(new.contiguous())), (t, Tmax)
                keep = torch.ones(Tmax, dtype=torch.bool, device='cuda')
                keep[t] = False
                assert torch.equal(bits(a[:, keep].contiguous()), bits(b[:, keep].contiguous())), (t, Tmax)
            assert_guard(ofull, S * 512)
            qd = qkv[:, :512].double().view(S, 8, 64) / 8
            Kd, Vd = K.double().view(S, t + 1, 8, 64), V.double().view(S, t + 1, 8, 64)
            p = torch.einsum('shd,sjhd->shj', qd, Kd).softmax(-1)
            ref = torch.einsum('shj,sjhd->shd', p, Vd).reshape(S, 512)
            got = out.view(S, 512)
            assert torch.isfinite(got).all(), (t, Tmax)
            err = float((got.double() - ref).abs().max() / ref.abs().max())
            assert err <= 1e-5, (t, Tmax, err)


# ----------------------------------------------------------------------------------------------- GEMV
def _gemv(ctx, x, x2, n_split, W, b, resid, M, N, K, act, ln_g=None, ln_b=None, pos=None, pos_split=0):
    out, full = guarded(M * N)
    rc = _op(ctx, 'alm_op_gemv', x.data_ptr(), _ptr(x2), n_split, W.data_ptr(), _ptr(b), _ptr(resid), out.data_ptr(), M,
             N, K, act, _ptr(ln_g), _ptr(ln_b), _ptr(pos), pos_split)
    ctx.check(rc)
    assert_guard(full, M * N)
    return out.view(M, N).clone()


def _split_dot(x, x2, n_split, W):
    """fp64 x . W^T for columns < n_split and x2 . W^T for the rest, and the sums of the terms' magnitudes"""
    W64 = W.double()
    first = torch.arange(W.shape[0], device=W.device)[None, :] < n_split
    dot = torch.where(first, x.double() @ W64.T, x2.double() @ W64.T)
    mag = torch.where(first, x.double().abs() @ W64.abs().T, x2.double().abs() @ W64.abs().T)
    return dot, mag


def _act64(y, act):
    return torch.nn.functional.gelu(y) if act == 1 else (torch.relu(y) if act == 2 else y)


def _assert_close_to_terms(got, ref, mag, what):
    """|got - ref| <= 1e-5 x (sum of the magnitudes of the terms) in every element"""
    assert torch.isfinite(got).all(), what
    ratio = float(((got.double() - ref).abs() / mag).max())
    assert ratio <= 1e-5, (what, ratio)


@pytest.mark.parametrize('K', [64, 512, 1024, 2048])
@pytest.mark.parametrize('M', [1, 8, 9, 16, 17, 32])
def test_gemv_matches_fp64(ctx, M, K):
    g = torch.Generator(device='cuda').manual_seed(M * 10000 + K)
    x = torch.randn(M, K, generator=g, device='cuda')
    x2 = torch.randn(M, K, generator=g, device='cuda') * 3
    for N in (1, 5, 512, 1536, 2048):
        W = torch.randn(N, K, generator=g, device='cuda') / K ** 0.5
        b = torch.randn(N, generator=g, device='cuda')
        resid = torch.randn(M, N, generator=g, device='cuda')
        for act, use_resid, use_x2 in ((0, False, False), (1, True, True), (2, False, True)):
            n_split = 1024 if use_x2 else 1 << 30      # columns >= 1024 read x2: the fused q | k | v projection
            got = _gemv(ctx, x, x2 if use_x2 else None, n_split, W, b, resid if use_resid else None, M, N, K, act)
            ref, mag = _split_dot(x, x2 if use_x2 else x, n_split, W)
            ref, mag = _act64(ref + b.double(), act), mag + b.double().abs()
            if use_resid:
                ref, mag = ref + resid.double(), mag + resid.double().abs()
            _assert_close_to_terms(got, ref, mag, (N, act, use_resid, use_x2))
    if K != 512:
        return
    # fused LayerNorm + query position: bit for bit the unfused pair (LayerNorm, then the GEMV on LN(x) + pos | LN(x))
    gam = torch.randn(512, generator=g, device='cuda')
    bet = torch.randn(512, generator=g, device='cuda')
    pos = torch.randn(512, generator=g, device='cuda')
    xr = x * 4 + 1
    ln = torch.empty_like(xr)
    ctx.check(_op(ctx, 'alm_op_layernorm', xr.data_ptr(), gam.data_ptr(), bet.data_ptr(), 1e-5, ln.data_ptr(), M, 512))
    lnp = ln + pos
    ln64 = torch.nn.functional.layer_norm(xr.double(), (512,), gam.double(), bet.double(), 1e-5)
    for N in (512, 1536, 2048):
        W = torch.randn(N, 512, generator=g, device='cuda') / 512 ** 0.5
        b = torch.randn(N, generator=g, device='cuda')
        for pos_split in (0, 1024, 1 << 30):
            fused = _gemv(ctx, xr, None, 1 << 30, W, b, None, M, N, 512, 2, gam, bet, pos, pos_split)
            plain = _gemv(ctx, lnp, ln, pos_split, W, b, None, M, N, 512, 2)
            assert torch.equal(bits(fused), bits(plain)), (N, pos_split)
            ref, mag = _split_dot(ln64 + pos.double(), ln64, pos_split, W)
            _assert_close_to_terms(fused, torch.relu(ref + b.double()), mag + b.double().abs(), ('ln', N, pos_split))


def test_gemv_argument_errors(ctx):
    x = torch.zeros(40 * 1024, device='cuda')
    W = torch.zeros(8 * 1024, device='cuda')
    g = torch.ones(1024, device='cuda')
    out, full = guarded(40 * 8)

    def call(M, K, ln=False):
        return _op(ctx, 'alm_op_gemv', x.data_ptr(), None, 1 << 30, W.data_ptr(), None, None, out.data_ptr(), M, 8, K,
                   0, _ptr(g if ln else None), _ptr(g if ln else None), None, 0)
    assert call(33, 64) == ERR_INVALID
    assert call(4, 513) == ERR_INVALID
    assert call(4, 700) == ERR_INVALID
    assert call(4, 1024, ln=True) == ERR_INVALID
    assert call(4, 256, ln=True) == ERR_INVALID
    assert torch.isnan(out).all()               # nothing was launched
    assert_guard(full, 40 * 8)


# ----------------------------------------------------------------------------------------------- token selection
NB, RECOG_PAD, PT_EOS, POLY_EOS, REC_EOS, PT_SOS, PADDING = 1000, 1096, 1097, 1098, 1099, 1100, 1103
BASE_V = 1104

# (phase, gen_index, vie, nsoft is V - vie)
HEAD_CASES = [(0, 0, 0, False), (0, 1, 0, False), (0, 6, 0, False), (0, 1001, 0, False), (1, 5, 0, False),
              (2, 9, 0, False)]
for _vie in (4, 29):
    HEAD_CASES += [(0, 3, _vie, False), (0, 4, _vie, False), (0, 302, _vie, False),
                   (1, 2, _vie, True), (1, 2, _vie, False), (2, 4, _vie, True), (2, 4, _vie, False)]


def _candidates(phase, gen_index, vie, V):
    """the ids a step may emit: oracle.omniparser_ref.step_candidates, plus the KIE class slot as greedy_kie states it"""
    from oracle import omniparser_ref as O
    kind = ('pt', 'poly', 'rec')[phase]
    if phase == 0 and vie:
        slot = gen_index % 3
        if slot == 2:
            a = torch.zeros(V, dtype=torch.bool)
            a[V - vie:] = True                       # out[:, :-vie] = 0
            return a
        return O.step_candidates('pt', 0 if slot == 0 else 1, V)   # slot 0: bins + EOS, slot 1: bins
    return O.step_candidates(kind, gen_index, V)


def _head_rows(allowed, nsoft, V, g):
    """logit rows, each planting one situation at the edges of the candidate set"""
    ids = allowed[:nsoft].nonzero().flatten().tolist()
    rows = []

    def base():
        return torch.randn(V, generator=g, dtype=torch.float64).float() * 3

    def plant(pairs):
        r = base()
        top = float(r.max()) + 4
        for j, val in pairs:
            r[j] = top + val
        rows.append(r)
    rows.append(base())
    # the global maximum on a forbidden id
    for f in (PT_SOS, PADDING, RECOG_PAD, PT_EOS, POLY_EOS, REC_EOS, NB - 1, NB, V - 1, V - 5):
        if 0 <= f < nsoft and not allowed[f]:
            plant([(f, 3.0)])
    # the winner at either end of every run of candidates; a forbidden lower id tied with the run's first id
    starts = [j for j in ids if j == 0 or not allowed[j - 1]]
    ends = [j for j in ids if j == V - 1 or not allowed[j + 1]]
    for j in starts + ends:
        plant([(j, 0.0)])
    for j in starts:
        if j > 0:
            plant([(j - 1, 0.0), (j, 0.0)])
    # exact ties between candidates held by neighbouring lanes, different warps and the same thread's next stride
    for j in ids[:1] + ids[len(ids) // 2:len(ids) // 2 + 1]:
        for d in (1, 16, 32, 256):
            if j + d < nsoft and allowed[j + d]:
                plant([(j, 0.0), (j + d, 0.0)])
                plant([(j + d, 0.0), (j, -1e-3)])
    # -inf on forbidden and candidate logits (never on every candidate)
    r = base()
    r[::7] = float('-inf')
    r[ids[0]] = float('-inf')
    r[ids[-1]] = float('-inf')
    if allowed[ids].logical_and(r[ids] > float('-inf')).any():
        rows.append(r)
    return torch.stack(rows)


@pytest.mark.parametrize('case', HEAD_CASES, ids=lambda c: f'ph{c[0]}-gi{c[1]}-vie{c[2]}-{"Vmv" if c[3] else "V"}')
def test_head_select_matches_reference_rule(ctx, case):
    from advancedliteratemachinery_b200 import _lib
    phase, gen_index, vie, soft_cut = case
    V = BASE_V + vie
    nsoft = V - vie if soft_cut else V
    allowed = _candidates(phase, gen_index, vie, V)
    g = torch.Generator().manual_seed(phase * 1000 + gen_index + vie)
    logits = _head_rows(allowed, nsoft, V, g)
    S = logits.shape[0]
    cfg = _lib.DecodeCfg(NB, PT_EOS, POLY_EOS, REC_EOS, PT_SOS, 1101, 1102, RECOG_PAD, 1024, 25, 32, vie, 512)
    token, tfull = guarded(S, torch.int32, -7)
    prob, pfull = guarded(S)
    fin0 = (torch.arange(S) % 4 == 3).int()
    ntok0 = torch.full((S,), 3, dtype=torch.int32)
    fin, ffull = guarded(S, torch.int32, -7)
    ntok, nfull = guarded(S, torch.int32, -7)
    fin.copy_(fin0)
    ntok.copy_(ntok0)
    track = phase == 0        # EOS bookkeeping runs in the point loop
    ld = logits.cuda()
    ctx.check(_op(ctx, 'alm_op_head_select', ld.data_ptr(), S, V, nsoft, phase, gen_index, C.byref(cfg),
                  token.data_ptr(), prob.data_ptr(), fin.data_ptr() if track else None,
                  ntok.data_ptr() if track else None))
    for full, fill in ((tfull, -7), (pfull, NAN), (ffull, -7), (nfull, -7)):
        assert_guard(full, S, fill)
    cand = logits.masked_fill(~allowed, float('-inf'))
    best = cand.max(-1, keepdim=True).values
    want = (cand == best).int().argmax(-1)                  # the lowest id among the maxima
    got = token.cpu().long()
    bad = (got != want).nonzero().flatten().tolist()
    assert not bad, [(r, int(got[r]), int(want[r])) for r in bad[:8]]
    p64 = logits[:, :nsoft].double().softmax(-1).gather(1, want[:, None]).flatten()
    err = float(((prob.cpu().double() - p64).abs() / p64).max())
    assert err <= 1e-5, err
    if track:
        eos = want == PT_EOS
        exp_fin = torch.where(fin0.bool(), fin0, eos.int())
        exp_ntok = torch.where(fin0.bool() | eos, ntok0, torch.full_like(ntok0, gen_index + 1))
        assert torch.equal(fin.cpu(), exp_fin) and torch.equal(ntok.cpu(), exp_ntok)
    else:
        assert torch.equal(fin.cpu(), fin0) and torch.equal(ntok.cpu(), ntok0)
