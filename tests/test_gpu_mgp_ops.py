"""GPU: MGP-STR's own kernels against fp64 and the exact selection rule, through their op-level entry points.

Two kernels run only in MGP-STR, and the end-to-end tests compare only whole logits (1e-3) and ids:

* the fused ViT attention (attn_tc.cu, every block of every crop), through alm_op_attention_ex: the split qkv planes
  and split output planes of the blocks, handed to attention_tc unchanged.  Element by element against
  softmax(q k^T * 64^-0.5) v in fp64, with a bound derived from the split scheme, at every edge of the 64-row query
  blocks, 16-row warp bands, 64-key blocks and 8-key column pairs, for 3 / 6 / 12 / 16 heads and at BASELINE config 3
  (512 crops of 257 tokens, 12 heads);
* the per-row selection that turns every head's logits into ids and probabilities (argmax_prob_kernel /
  row_topk_kernel in mgp.cu), through alm_op_row_select, which runs the forward's own launch code (mgp_row_select).
  Ids against the exact rule bit for bit, with ties across threads and warps, more tied maxima than the list holds,
  k > n, and the real heads' widths inside their padded rows.

Every output buffer is followed by a guard region that must come back bit for bit unchanged, and every input element a
call must not read holds NaN: pad columns, rows after the last crop or row, and the whole lo plane at nsplit 1, where
the model's producers never write it.  Split outputs must be hi = bf16_rn(x), lo = bf16_rn(x - hi) of the fp32 value.
"""
import pytest
import torch

from tests.support import NAN, assert_guard, bits, ctx, guarded, options

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

WORKSPACE_MB = 2048
ERR_INVALID, ERR_UNSUPPORTED = -1, -5
U32 = 2.0 ** -24        # fp32 unit roundoff
UBF = 2.0 ** -8         # bf16 unit roundoff
NAN16 = -1              # 0xffff: a bf16 NaN


def _ptr(t):
    return None if t is None else t.data_ptr()


def _op(ctx, name, *args):
    """Call an entry point once torch's queued work is done (the context runs on its own stream and synchronizes it
    before returning)."""
    torch.cuda.synchronize()
    return getattr(ctx.lib, name)(ctx.h, *args)


def _split(x):
    """fp32 x -> (bf16_rn(x), bf16_rn(x - hi)) as int16 bit tensors"""
    h = x.float().to(torch.bfloat16)
    return h.view(torch.int16), (x.float() - h.float()).to(torch.bfloat16).view(torch.int16)


def _assert_split(hi, lo, x, what=''):
    h, l = _split(x)
    assert torch.equal(hi, h), ('hi', what)
    assert torch.equal(lo, l), ('lo', what)


# ----------------------------------------------------------------------------------------------- ViT attention
KINDS = ('sharp', 'last', 'negative', 'offset')


def _unit(H, gen):
    u = torch.randn(H, 64, generator=gen, device='cuda')
    return u / u.norm(dim=-1, keepdim=True)


def _crop(kind, T, H, gen):
    """fp32 qkv [T, 3 * H * 64] of one crop (q | k | v blocks, head h at columns h * 64 of its block).
    sharp: scores 0.125 q.k of standard deviation 10.  last: every query shares a direction with key T - 1, whose score
    beats the others by about 15 (the lone live key of a ragged last block when T = 1 mod 64).  negative: every live
    score about -30, so a zero-filled key past T that leaked into the softmax would carry nearly all the weight.
    offset: v = 100 + N(0, 1), where a mismatch between the probabilities and their sum shows at 100 times its size."""
    def r(*s):
        return torch.randn(*s, generator=gen, device='cuda')
    q, k, v = r(T, H, 64), r(T, H, 64), r(T, H, 64)
    if kind == 'sharp':
        q, k = q * 10 ** 0.5, k * 10 ** 0.5
    elif kind == 'last':
        u = _unit(H, gen)
        q = q + 3 * u
        k[T - 1] = 40 * u
        v[T - 1] += 5
    elif kind == 'negative':
        u = _unit(H, gen)
        q, k, v = 3 * u + 0.3 * q, -80 * u + 2 * k, v + 2
    else:
        q, k, v = q * 3 ** 0.5, k * 3 ** 0.5, v + 100
    return torch.cat([t.reshape(T, H * 64) for t in (q, k, v)], 1)


def _qkv(B, T, H, seed, kinds=KINDS):
    """fp32 qkv [B * T, 3 D]: crop b is of kind kinds[b % len(kinds)]"""
    gen = torch.Generator(device='cuda').manual_seed(seed)
    return torch.cat([_crop(kinds[b % len(kinds)], T, H, gen) for b in range(B)], 0)


def _planes(x, ld, lo_nan):
    """the split planes of x [R, W] with row stride ld (uint16 buffers): NaN in columns W .. ld-1, in 5 rows after the
    last one, and in the whole lo plane when lo_nan"""
    R, W = x.shape
    hi = torch.full((R + 5, ld), NAN16, dtype=torch.int16, device='cuda')
    lo = torch.full((R + 5, ld), NAN16, dtype=torch.int16, device='cuda')
    h, l = _split(x)
    hi[:R, :W] = h
    if not lo_nan:
        lo[:R, :W] = l
    return hi, lo


def _attn_ref(x, B, T, H, chunk=32):
    """softmax(q k^T * 0.125) v of fp32 qkv x in fp64 on the device, with what the bound needs per query row: the
    standard deviation sd and mean |v| pav of v under the row's probabilities, per output element, and the largest
    A = 0.125 sum_d |q_d k_d| and |s| over the row's keys, per head"""
    D = H * 64
    o, sd, pav = (torch.empty(B * T, D, dtype=torch.float64, device='cuda') for _ in range(3))
    A, Sm = (torch.empty(B * T, H, dtype=torch.float64, device='cuda') for _ in range(2))
    for b0 in range(0, B, chunk):
        n = min(B, b0 + chunk) - b0
        rows = slice(b0 * T, (b0 + n) * T)
        q, k, v = x[rows, :3 * D].double().view(n, T, 3, H, 64).permute(2, 0, 3, 1, 4)     # [n, H, T, 64]

        def put(t):                                                                        # [n, H, T, w] -> [n T, H w]
            return t.transpose(1, 2).reshape(n * T, -1)
        S = (q @ k.transpose(-1, -2)) * 0.125
        P = S.softmax(-1)
        ob = P @ v
        c = v.mean(-2, keepdim=True)
        o[rows] = put(ob)
        sd[rows] = put((P @ (v - c).square() - (ob - c).square()).clamp(min=0).sqrt())
        pav[rows] = put(P @ v.abs())
        A[rows] = put(((q.abs() @ k.abs().transpose(-1, -2)) * 0.125).amax(-1, keepdim=True))
        Sm[rows] = put(S.abs().amax(-1, keepdim=True))
    return dict(o=o, sd=sd, pav=pav, A=A, Sm=Sm, T=T)


def _attn_tol(ref, ns):
    """|got - ref| bound per element.  Each tensor-core product is off by at most e of its magnitude: e = 3 * 2^-16 at
    nsplit 3 (q, k, v and p each held to 2^-16 by their hi + lo pair, and the lo * lo term dropped), and one bf16
    rounding of each operand at nsplit 1 (q and k; p and v).  So a score s_ij moves by at most delta_i = e * A_i, A_i =
    max_j 0.125 sum_d |q_d k_jd|, plus the fp32 accumulation of the products and the fp32 scaling, subtraction and
    exp2 of the online softmax.  Scores moved by at most delta change each probability by a factor within exp(+-2
    delta), hence the output by at most expm1(2 delta) sum_j p_j |v_j - o| <= expm1(2 delta) sd.  P.V adds e per product
    and the fp32 accumulation over T keys, of the running sum and of the division, together at most (e + (2 T + 64) u)
    sum_j p_j |v_j| with the probabilities moved as above."""
    T = ref['T']
    e = 3 * 2.0 ** -16 if ns == 3 else 2 * UBF + UBF ** 2
    delta = ((e + 16 * U32) * ref['A'] + U32 * (4 * ref['Sm'] + 16) + 2.0 ** -21).repeat_interleave(64, 1)
    return (torch.expm1(2 * delta) * ref['sd'] + (e + (2 * T + 64) * U32) * torch.exp(2 * delta) * ref['pav']
            + 2.0 ** -100)


def _run_attn(ctx, hi, lo, B, T, H, ldo, f32=True, with_lo=True):
    """alm_op_attention_ex on planes hi / lo ([rows, ld] int16 views) -> (out f32 or None, out_hi, out_lo), each
    [B T, D]; the columns D .. ldo-1 must stay as prefilled and every guard intact.  Each guard is one 64-row query
    block long, so rows of the last block past T that were written would land in it."""
    D, R = H * 64, B * T
    n, guard = R * ldo, 64 * ldo
    out, ofull = guarded(n, guard=guard) if f32 else (None, None)
    (oh, hfull), (ol, lfull) = (guarded(n, torch.int16, NAN16, guard) for _ in range(2))
    ctx.check(_op(ctx, 'alm_op_attention_ex', hi.data_ptr(), lo.data_ptr() if with_lo else None, hi.stride(0), B, T, H,
                  _ptr(out), oh.data_ptr(), ol.data_ptr(), ldo))
    res = []
    for buf, full, fill in ((out, ofull, NAN), (oh, hfull, NAN16), (ol, lfull, NAN16)):
        if buf is None:
            res.append(None)
            continue
        assert_guard(full, n, fill)
        v = buf.view(R, ldo)
        gap = v[:, D:]
        assert torch.equal(bits(gap), bits(torch.full_like(gap, fill))), 'wrote past the row width'
        res.append(v[:, :D].contiguous())
    return tuple(res)


WORST = {}


def _check_attention(ctx, x, B, T, H, ld, ldo, ref=None, alone=True):
    """every output form of alm_op_attention_ex at nsplit 3 and 1 against the fp64 reference and each other"""
    D = H * 64
    ref = ref or _attn_ref(x, B, T, H)
    for ns in (3, 1):
        with options(ctx, nsplit=ns):
            hi, lo = _planes(x, ld, lo_nan=ns == 1)
            out, oh, ol = _run_attn(ctx, hi, lo, B, T, H, ldo)
            assert torch.isfinite(out).all(), ns
            err = (out.double() - ref['o']).abs()
            tol = _attn_tol(ref, ns)
            ratio = float((err / tol).max())
            WORST[ns] = max(WORST.get(ns, 0.0), ratio)
            print(f'attention B={B} T={T} H={H} nsplit {ns}: worst err / bound {ratio:.3g}')
            assert bool((err <= tol).all()), (ns, ratio, float(err.max()))
            if ns == 3:
                _assert_split(oh, ol, out, 'out')
            else:
                assert torch.equal(oh, _split(out)[0]), 'hi'
                assert bool((ol == NAN16).all()), 'lo plane written at nsplit 1'
            # the model's form: planes only (at nsplit 1 without a lo plane at all)
            _, oh2, ol2 = _run_attn(ctx, hi, lo, B, T, H, ldo, f32=False, with_lo=ns == 3)
            assert torch.equal(oh2, oh) and torch.equal(ol2, ol), ns
            if alone and B > 1:   # the last crop alone (followed by the NaN rows) == the same crop inside the batch
                rows = slice((B - 1) * T, B * T)
                got, _, _ = _run_attn(ctx, hi[rows], lo[rows], 1, T, H, D)
                assert torch.equal(bits(got), bits(out[rows])), ns


# T at every edge of the 64-row query blocks, 16-row warp bands, 64-key blocks and 8-key column pairs, odd and even
ATTN_T = [1, 2, 15, 16, 17, 63, 64, 65, 127, 128, 129, 192, 193, 255, 256, 257, 271, 272]


@pytest.mark.parametrize('T', ATTN_T)
def test_attention_ex_token_edges(ctx, T):
    H = (3, 6, 12, 16)[ATTN_T.index(T) % 4]
    x = _qkv(4, T, H, seed=T * 16 + H)
    _check_attention(ctx, x, 4, T, H, ld=3 * H * 64 + 8, ldo=H * 64 + 8)


@pytest.mark.parametrize('H', [3, 6, 12, 16])
def test_attention_ex_model_widths(ctx, H):
    """tiny / small / base / large at the model's 257 tokens, 8 crops, row strides wider than the data"""
    x = _qkv(8, 257, H, seed=H)
    _check_attention(ctx, x, 8, 257, H, ld=3 * H * 64 + 24, ldo=H * 64 + 16)


def test_attention_ex_config3(ctx):
    """BASELINE config 3: 512 crops of 257 tokens, 12 heads (6 144 x 5 CTAs), at the model's own strides"""
    B, T, H = 512, 257, 12
    x = _qkv(B, T, H, seed=3)
    _check_attention(ctx, x, B, T, H, ld=3 * H * 64, ldo=H * 64, alone=False)
    print(f'attention worst err / bound over this module so far: {WORST}')


@pytest.mark.parametrize('B,T,H', [(2, 257, 3), (1, 50, 1), (3, 130, 2), (1, 272, 1), (40, 257, 12)])
def test_attention_fp32_entry_matches_fp64(ctx, B, T, H):
    """alm_op_attention (fp32 qkv, split inside the call) element by element against fp64, and bit for bit the
    alm_op_attention_ex call on the same planes: 257 tokens, short and ragged sequences, the 272-token maximum, and more
    CTAs than SMs"""
    g = torch.Generator(device='cuda').manual_seed(B * 1000 + T + H)
    D = H * 64
    x = torch.randn(B * T, 3 * D, generator=g, device='cuda')
    x[:, :D] *= 1.5     # sharper softmax than unit-variance scores
    ref = _attn_ref(x, B, T, H)
    for ns, rel in ((3, 3e-5), (1, 2e-2)):
        with options(ctx, nsplit=ns):
            out, ofull = guarded(B * T * D, guard=64 * D)
            ctx.check(_op(ctx, 'alm_op_attention', x.data_ptr(), out.data_ptr(), B, T, H))
            assert_guard(ofull, B * T * D)
            out = out.view(B * T, D)
            err = (out.double() - ref['o']).abs()
            assert bool((err <= _attn_tol(ref, ns)).all()), (ns, float(err.max()))
            assert float(err.max() / ref['o'].abs().max()) < rel, ns     # and within rel of the largest output
            hi, lo = _planes(x, 3 * D, lo_nan=False)
            ex, _, _ = _run_attn(ctx, hi, lo, B, T, H, D)
            assert torch.equal(bits(ex), bits(out)), ns


# ----------------------------------------------------------------------------------------------- row selection
def _select_rows(n, gen):
    """rows of n fp32 logits at the edges of the selection.  Thread t of the 256 reads ids t, t + 256, ...; warp t / 32."""
    def r(s=1.0):
        return torch.randn(n, generator=gen, device='cuda') * s

    def at(ids):
        return sorted({min(j, n - 1) for j in ids})
    rows = [r(3.0), r(0.3), r(30.0)]
    x = r()
    x[0] = x.max() + 1                                              # maximum at id 0
    rows.append(x)
    x = r()
    x[n - 1] = x.max() + 1                                          # at id n - 1, in the last partial slice
    rows.append(x)
    x = r()
    x[at([n - 1, 300, 37, 5, 256, 1])] = x.max() + 1                # equal maxima in different threads and warps
    rows.append(x)
    for a, b in ((3, 40), (40, 3)):                                 # -0.0 and +0.0 as the maximum, either first
        x = -r().abs() - 1
        x[min(a, n - 1)], x[min(b, n - 1)] = -0.0, 0.0
        rows.append(x)
    x = r()
    x[at([n - 1, 2, 3, 31, 32, 100, 255, 256, 257, 511, 700, 1000, 5000, 40000])] = x.max() + 1   # > 8 tied maxima
    rows.append(x)
    for place, size in ((1, 4), (4, 3)):                            # a tie group at candidate 1 and at candidate 4
        x = r() - 10
        top = torch.arange(place, 0, -1, device='cuda', dtype=torch.float32)
        ids = torch.randperm(n, generator=torch.Generator().manual_seed(n + place))[:place + size].tolist()
        for i in range(min(place, n)):
            x[ids[i]] = 20 + float(top[i])
        for j in ids[place:place + size]:
            if j < n:
                x[j] = 20.0
        rows.append(x)
    x = r()                                                         # neighbours one ulp apart, the lower ids lower
    m = x.max() + 1
    m1 = torch.nextafter(m, torch.tensor(-float('inf'), device='cuda'))
    m2 = torch.nextafter(m1, torch.tensor(-float('inf'), device='cuda'))
    x[at([n - 1])], x[at([n // 2])], x[at([0])] = m, m1, m2
    rows.append(x)
    rows.append(-torch.rand(n, generator=gen, device='cuda') * 1e4)  # spread 1e4: most probabilities underflow to +0
    rows.append(torch.full((n,), 0.75, device='cuda'))              # every id tied
    return rows


def _logits(rows, n, ld, gen, special):
    """fp32 [rows, ld] whose columns n .. ld-1 and 3 rows past the end hold NaN: random rows with the special rows at
    the start and at the end"""
    buf = torch.full(((rows + 3) * ld,), NAN, device='cuda')
    x = buf[:rows * ld].view(rows, ld)
    x[:, :n] = torch.randn(rows, n, generator=gen, device='cuda') * 4
    s = torch.stack(special)[:rows]
    x[:s.shape[0], :n] = s
    x[rows - s.shape[0]:, :n] = s.flip(0)
    return x


def _run_select(ctx, x, n, k):
    rows, ld = x.shape[0], x.stride(0)
    per = max(k, 1)
    ids, ifull = guarded(rows * per, torch.int32, -7)
    probs, pfull = guarded(rows * per)
    ctx.check(_op(ctx, 'alm_op_row_select', x.data_ptr(), ld, rows, n, k, ids.data_ptr(), probs.data_ptr()))
    assert_guard(ifull, rows * per, -7)
    assert_guard(pfull, rows * per)
    return ids.view(rows, per), probs.view(rows, per)


def _check_select(ctx, x, n):
    v = x[:, :n]
    # the kernel's order: value descending, lowest id first on equal values; + 0.0 turns -0.0 into +0.0, which the
    # kernel's comparisons treat as equal
    order = torch.sort(-(v + 0.0), dim=-1, stable=True).indices
    x64 = v.double()
    m = x64.amax(-1, keepdim=True)
    p64 = (x64 - m).exp()
    p64 = p64 / p64.sum(-1, keepdim=True)
    # the fp32 bound of test_softmax_rows_matches_fp64: exp of (x - max), the row sum, the division
    tol = p64 * U32 * (2 * (x64 - m).abs() + n / 128 + 16) + 2.0 ** -126

    def close(ids, probs, what):
        g = ids.long()
        err = (probs.double() - p64.gather(1, g)).abs()
        assert bool((err <= tol.gather(1, g)).all()), (what, float((err / tol.gather(1, g)).max()))
    id0, pr0 = _run_select(ctx, x, n, 0)
    assert torch.equal(id0[:, 0].long(), order[:, 0]), 'top-1 ids'
    close(id0, pr0, 'top-1')
    top = v.gather(1, id0.long())
    for k in (1, 2, 5, 8):
        ids, probs = _run_select(ctx, x, n, k)
        kk = min(k, n)
        assert torch.equal(ids[:, :kk].long(), order[:, :kk]), ('ids', k)
        assert bool((ids[:, kk:] == -1).all()) and not bool(bits(probs[:, kk:]).any()), ('past n', k)
        assert torch.equal(ids[:, :1], id0) and torch.equal(bits(probs[:, :1]), bits(pr0)), ('candidate 0', k)
        close(ids[:, :kk], probs[:, :kk], k)
        tied = v.gather(1, ids[:, :kk].long()) == top
        assert torch.equal(bits(probs[:, :kk])[tied], bits(pr0.expand(-1, kk))[tied]), ('tied probability', k)
        assert bool((probs[:, 1:kk] <= probs[:, :kk - 1]).all()), ('not non-increasing', k)


# name: (n, ld, rows); the char / WordPiece / BPE heads in their Vpad rows, and the char head at config 3 (512 x 27)
SELECT_CASES = {
    'n1': (1, 4, 20), 'n7': (7, 9, 20), 'n255': (255, 260, 20), 'n256': (256, 256, 20), 'n257': (257, 264, 20),
    'char': (38, 40, 40), 'wp': (30522, 30528, 24), 'bpe': (50257, 50264, 24), 'char-config3': (38, 40, 512 * 27),
}


@pytest.mark.parametrize('name', list(SELECT_CASES))
def test_row_select_matches_the_exact_rule(ctx, name):
    n, ld, rows = SELECT_CASES[name]
    gen = torch.Generator(device='cuda').manual_seed(n + rows)
    x = _logits(rows, n, ld, gen, _select_rows(n, gen))
    _check_select(ctx, x, n)


# ----------------------------------------------------------------------------------------------- argument errors
def test_argument_errors_leave_the_context_usable(ctx):
    H, T = 1, 4
    x = _qkv(1, T, H, seed=0, kinds=('sharp',))
    hi, lo = _planes(x, 192, lo_nan=False)
    hst = torch.zeros(8 * 192, dtype=torch.int16)
    buf = torch.zeros(1 << 12, dtype=torch.int16, device='cuda')
    out = torch.full((T, 64), NAN, device='cuda')
    P = _ptr

    def attn(q=hi, l=lo, ld=192, o=out, oh=None, ol=None, ldo=64, T=T):
        return _op(ctx, 'alm_op_attention_ex', P(q), P(l), ld, 1, T, H, P(o), P(oh), P(ol), ldo)
    assert attn(q=None) == ERR_INVALID
    assert attn(q=hst) == ERR_INVALID
    assert attn(q=buf[1:]) == ERR_INVALID                    # not 16-byte aligned
    assert attn(o=out.view(-1)[2:]) == ERR_INVALID           # output not 16-byte aligned
    assert attn(ld=184) == ERR_INVALID                       # < 3 H 64
    assert attn(ld=196) == ERR_INVALID                       # not a multiple of 8
    assert attn(ldo=56) == ERR_INVALID                       # < H 64
    assert attn(ldo=68) == ERR_INVALID
    assert attn(o=None) == ERR_INVALID                       # no output
    assert attn(ol=buf) == ERR_INVALID                       # out_lo without out_hi
    assert attn(l=None) == ERR_INVALID                       # nsplit 3 needs the lo plane
    assert attn(T=273) == ERR_UNSUPPORTED
    assert bool(torch.isnan(out).all()), 'written before the error'
    with options(ctx, nsplit=1):
        assert attn(l=None) == 0                             # nsplit 1 reads the hi plane only

    logits = torch.randn(4, 40, device='cuda')
    ids = torch.full((4 * 8,), -7, dtype=torch.int32, device='cuda')
    probs = torch.full((4 * 8,), NAN, device='cuda')

    def sel(lg=logits, ld=40, rows=4, n=38, k=0, i=ids, p=probs):
        return _op(ctx, 'alm_op_row_select', P(lg), ld, rows, n, k, P(i), P(p))
    assert sel(lg=None) == ERR_INVALID
    assert sel(lg=torch.zeros(4, 40)) == ERR_INVALID
    assert sel(i=torch.zeros(32, dtype=torch.int32)) == ERR_INVALID
    assert sel(p=None) == ERR_INVALID
    assert sel(rows=0) == ERR_INVALID
    assert sel(n=0) == ERR_INVALID
    assert sel(n=41) == ERR_INVALID                          # wider than ld
    assert sel(k=9) == ERR_INVALID
    assert sel(k=-1) == ERR_INVALID
    assert bool((ids == -7).all()) and bool(torch.isnan(probs).all()), 'written before the error'

    # the context still computes
    _check_attention(ctx, _qkv(2, 65, 2, seed=1), 2, 65, 2, ld=2 * 3 * 64, ldo=2 * 64)
    gen = torch.Generator(device='cuda').manual_seed(0)
    _check_select(ctx, _logits(30, 38, 40, gen, _select_rows(38, gen)), 38)
