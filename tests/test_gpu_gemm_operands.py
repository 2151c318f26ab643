"""GPU: the input side of the GEMM engine -- operand geometry -- through alm_op_gemm_planes, against fp64, element by
element.

alm_op_gemm builds its own contiguous, zero-padded operands.  The model's batched GEMMs hand the engine something else:
head column slices inside wider rows, batch strides smaller than a row, operands broadcast along either batch dimension,
K tails with never-written pad columns up to ld, hi and lo planes any distance apart.  Here every operand lives in one
uint16 buffer holding both planes, and every bf16 element no (b0, b1, row < rows, k < K) addresses -- pad columns, rows
and gaps between batches, the gap between the planes, a prefix before the operand's first row and a guard after the
buffer -- holds NaN in both planes.  At nsplit 1 the whole lo plane is NaN.  One read of any of them poisons an output.

The reference is fp64 of exactly the products the kernel forms from the planes it is given (tensor cores: hi*hi +
lo*hi + hi*lo at nsplit 3, hi*hi at nsplit 1; the SIMT debug kernel: fp32(hi + lo) squared, or hi*hi).  Every such
product is exact in fp32, so the only error left is fp32 accumulation, and each element must satisfy
    |got - ref| <= n 2^-22 sum|terms|   (n products per element)
carried through alpha, bias, activation and residual with a few ulps of |x| for the epilogue's roundings (and 2e-7
max(1, |x| / 2) for the rational GELU).  The worst err / bound of each case is printed.

The cases: the geometry of every batched call site of both models (MGP-STR's grouped 1x1 convolution, A^3 select, feat
and x_a, the unfused attention's V^T, scores and P.V; OmniParser's K / V cache, V^T and unfused cross-attention
GEMMs), seeded random geometry that reaches both tile widths and both consumer schedules, slices of batched launches
against the same slice run unbatched (bit for bit), and the argument checks of the entry point.  Each runs at nsplit 3
and 1 and at gemm_impl 0 (wgmma) and 1 (SIMT).
"""
import ctypes
import random

import pytest
import torch

from tests import support
from tests.support import ctx, options

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

GUARD = 64
NAN_BF16 = 0x7fc0
NAN_F32 = 0x7fc00000
ALM_ERR_INVALID = -1
U = 2.0 ** -24
T, TP, NTOK, G = 257, 264, 27, 8  # MGP-STR: tokens, their padded row stride, A^3 tokens, conv groups
RUNS = ((3, 0), (3, 1), (1, 0), (1, 1))  # (nsplit, gemm_impl)


def _r8(x):
    return (x + 7) // 8 * 8


def _launch_shape(M, N, nb, sms):
    """(tile width, schedule) the engine picks: gemm.cu's narrow-tile rule and the one-tile-per-CTA test."""
    m_blocks = -(-M // 128)
    narrow = m_blocks * -(-N // 128) * nb < sms // 2 and N > 32
    bn = 32 if narrow else 128
    return bn, 'one tile per CTA' if m_blocks * -(-N // bn) * nb <= sms else 'ping-pong'


class Opd:
    """Geometry of one operand: element (b0, b1, r, k) of a plane sits at off + b0 bs0 + b1 bs1 + r ld + k (a batch
    dimension with extent 1 is broadcast and its stride unused); the lo plane starts `dist` elements after the hi one."""

    def __init__(self, rows, K, ld, nb0=1, nb1=1, bs0=0, bs1=0, off=0, gap=0):
        self.rows, self.K, self.ld, self.nb0, self.nb1, self.bs0, self.bs1, self.off = rows, K, ld, nb0, nb1, bs0, bs1, off
        self.ext = off + (nb0 - 1) * bs0 + (nb1 - 1) * bs1 + (rows - 1) * ld + K
        self.dist = _r8(self.ext) + gap

    def index(self, b0, b1):
        """plane indices [P, rows, K] of batches (b0[p], b1[p])"""
        dev = b0.device
        base = self.off + (b0 if self.nb0 > 1 else 0 * b0) * self.bs0 + (b1 if self.nb1 > 1 else 0 * b1) * self.bs1
        return (base[:, None, None] + torch.arange(self.rows, device=dev)[None, :, None] * self.ld
                + torch.arange(self.K, device=dev)[None, None, :])

    def fill(self, seed):
        """one buffer: [hi plane | gap | lo plane | guard], every element no batch / row / k addresses NaN"""
        g = torch.Generator(device='cuda').manual_seed(seed)
        x = torch.randn(self.ext, generator=g, device='cuda')
        hi = x.to(torch.bfloat16)
        lo = (x - hi.float()).to(torch.bfloat16)
        live = torch.zeros(self.ext, dtype=torch.bool, device='cuda')
        b0 = torch.arange(self.nb0, device='cuda')
        for b1 in range(self.nb1):
            live[self.index(b0, torch.full_like(b0, b1)).reshape(-1)] = True
        buf = torch.full((self.dist + self.ext + GUARD,), NAN_BF16, dtype=torch.int16, device='cuda')
        buf[:self.ext] = torch.where(live, hi.view(torch.int16), NAN_BF16)
        buf[self.dist:self.dist + self.ext] = torch.where(live, lo.view(torch.int16), NAN_BF16)
        self.buf = buf

    def poison_lo(self):
        self.buf[self.dist:self.dist + self.ext] = NAN_BF16

    def desc(self, lo=True, b0=0, b1=0, whole=True):
        """the C descriptor: the whole operand, or (whole=False) its slice (b0, b1) as an unbatched operand"""
        from advancedliteratemachinery_b200 import _lib
        off = self.off
        if not whole:
            off += (b0 if self.nb0 > 1 else 0) * self.bs0 + (b1 if self.nb1 > 1 else 0) * self.bs1
        base = self.buf.data_ptr() + 2 * off
        nb0, nb1, bs0, bs1 = (self.nb0, self.nb1, self.bs0, self.bs1) if whole else (1, 1, 0, 0)
        return _lib.GemmOperand(base, base + 2 * self.dist if lo else None, self.rows, self.K, self.ld, nb0, nb1, bs0,
                                bs1)

    def values(self, b0, b1):
        """(hi, lo) as fp32 [P, rows, K]"""
        i = self.index(b0, b1)
        return (self.buf[i].view(torch.bfloat16).float(), self.buf[self.dist + i].view(torch.bfloat16).float())


class Case:
    """A = a (M rows), B = b (N rows), epilogue e: dict(ldo, obs0, obs1, cg, cgs, bias ('col' | 'row'), bias_bs0,
    resid (ldr, rbs0, rbs1), act, alpha); lo_null: pass no lo plane at nsplit 1"""

    def __init__(self, a, b, e, lo_null=False):
        self.a, self.b, self.e, self.lo_null = a, b, e, lo_null
        self.M, self.N, self.K = a.rows, b.rows, a.K
        self.nb0, self.nb1 = max(a.nb0, b.nb0), max(a.nb1, b.nb1)

    def out_index(self, b0, b1):
        e = self.e
        n = torch.arange(self.N, device=b0.device)
        cn = (n // e['cg']) * e['cgs'] + n % e['cg'] if e.get('cg') else n
        return (b0[:, None, None] * e.get('obs0', 0) + b1[:, None, None] * e.get('obs1', 0)
                + torch.arange(self.M, device=b0.device)[None, :, None] * e['ldo'] + cn[None, None, :])


def _pairs(c):
    """the batches checked against fp64: all of them, or a seeded sample (first and last included) of large launches"""
    nb = c.nb0 * c.nb1
    cap = max(2, min(nb, int(4e7 // ((c.M + c.N) * c.K + 3 * c.M * c.N))))
    ids = list(range(nb)) if cap >= nb else sorted({0, nb - 1, *random.Random(nb).sample(range(nb), cap - 2)})
    ids = torch.tensor(ids, device='cuda')
    return ids % c.nb0, ids // c.nb0


def _setup(c, seed):
    """operand planes, NaN-filled bias / residual buffers and the written mask of the output"""
    c.a.fill(seed)
    c.b.fill(seed + 1)
    e, g = c.e, torch.Generator(device='cuda').manual_seed(seed + 2)
    nbmax = max(c.nb0, c.nb1)
    c.bias = None
    if e.get('bias'):
        n = c.N if e['bias'] == 'col' else c.M
        # room for max(nb0, nb1) batch strides: a kernel that offsets the bias by b1 still reads inside the buffer
        c.bias = torch.full((nbmax * e.get('bias_bs0', 0) + n + GUARD,), float('nan'), device='cuda')
        for b in range(c.nb0 if e.get('bias_bs0', 0) else 1):
            o = b * e.get('bias_bs0', 0)
            c.bias[o:o + n] = torch.randn(n, generator=g, device='cuda')
    c.resid = None
    if e.get('resid'):
        ldr, rbs0, rbs1 = e['resid']
        c.resid = torch.full(((c.nb0 - 1) * rbs0 + (c.nb1 - 1) * rbs1 + c.M * ldr + GUARD,), float('nan'), device='cuda')
        b0 = torch.arange(c.nb0, device='cuda')
        for b1 in range(c.nb1):
            i = (b0[:, None, None] * rbs0 + b1 * rbs1 + torch.arange(c.M, device='cuda')[None, :, None] * ldr
                 + torch.arange(c.N, device='cuda')[None, None, :])
            c.resid[i.reshape(-1)] = torch.randn(i.numel(), generator=g, device='cuda')
    b0 = torch.arange(c.nb0, device='cuda')
    size = int(c.out_index(b0[-1:], torch.tensor([c.nb1 - 1], device='cuda')).max()) + 1 + GUARD  # strides are >= 0
    c.written = torch.zeros(size, dtype=torch.bool, device='cuda')
    for b1 in range(c.nb1):
        c.written[c.out_index(b0, torch.full_like(b0, b1)).reshape(-1)] = True


def _epilogue(c, out_f32, out_hi, out_lo, b0=None, b1=None):
    """the C epilogue: the whole problem, or the unbatched call of slice (b0, b1) writing at offset 0"""
    from advancedliteratemachinery_b200 import _lib
    e = c.e
    whole = b0 is None
    bias_mode = {'col': 1, 'row': 2}.get(e.get('bias'), 0)
    bias = c.bias.data_ptr() + (0 if whole else 4 * b0 * e.get('bias_bs0', 0)) if c.bias is not None else None
    ldr, rbs0, rbs1 = e.get('resid') or (0, 0, 0)
    resid = c.resid.data_ptr() + (0 if whole else 4 * (b0 * rbs0 + b1 * rbs1)) if c.resid is not None else None
    return _lib.GemmEpilogue(out_f32.data_ptr(), out_hi.data_ptr(), out_lo.data_ptr(), e['ldo'],
                             e.get('obs0', 0) if whole else 0, e.get('obs1', 0) if whole else 0, e.get('cg', 0),
                             e.get('cgs', 0), bias, bias_mode, e.get('bias_bs0', 0) if whole else 0, resid, ldr,
                             rbs0 if whole else 0, rbs1 if whole else 0, None, None, e.get('act', 0),
                             e.get('alpha', 1.0))


def _outputs(size):
    return (torch.full((size,), float('nan'), device='cuda'),
            torch.full((size,), NAN_BF16, dtype=torch.int16, device='cuda'),
            torch.full((size,), NAN_BF16, dtype=torch.int16, device='cuda'))


def _call(ctx, a, b, e):
    # the context runs on its own non-blocking stream: the buffers torch filled on its stream must be complete first
    torch.cuda.synchronize()
    return ctx.lib.alm_op_gemm_planes(ctx.h, ctypes.byref(a), ctypes.byref(b), ctypes.byref(e))


def _run(ctx, c, nsplit, impl):
    with options(ctx, nsplit=nsplit, gemm_impl=impl):
        out = _outputs(c.written.numel())
        lo = not (nsplit == 1 and c.lo_null)
        ctx.check(_call(ctx, c.a.desc(lo), c.b.desc(lo), _epilogue(c, *out)))
    return out


def _reference(c, nsplit, impl, b0, b1):
    """(ref, bound) [P, M, N] in fp64 for batches (b0, b1)"""
    ah, al = c.a.values(b0, b1)
    bh, bl = c.b.values(b0, b1)
    mm = lambda x, y: torch.bmm(x.double(), y.double().transpose(1, 2))
    if nsplit == 3 and impl == 0:
        acc = mm(ah, bh) + mm(al, bh) + mm(ah, bl)
        s = mm(ah.abs(), bh.abs()) + mm(al.abs(), bh.abs()) + mm(ah.abs(), bl.abs())
        n = 3 * c.K
    else:
        if nsplit == 3:  # the SIMT kernel re-joins the planes in fp32 before one fma per k
            ah, bh = ah + al, bh + bl
        acc, s, n = mm(ah, bh), mm(ah.abs(), bh.abs()), c.K
    e = c.e
    alpha = e.get('alpha', 1.0)
    x = alpha * acc
    bound = abs(alpha) * n * 2.0 ** -22 * s
    if c.bias is not None:
        if e['bias'] == 'col':
            bv = c.bias[(b0 * e.get('bias_bs0', 0))[:, None] + torch.arange(c.N, device='cuda')][:, None, :]
        else:
            bv = c.bias[(b0 * e.get('bias_bs0', 0))[:, None] + torch.arange(c.M, device='cuda')][:, :, None]
        bound = bound + 4 * U * (x.abs() + bv.double().abs())
        x = x + bv.double()
    else:
        bound = bound + 2 * U * x.abs()
    act = e.get('act', 0)
    if act == 1:
        y = torch.nn.functional.gelu(x)
        bound = 1.13 * bound + 2e-7 * torch.clamp(0.5 * x.abs(), min=1.0) + 4 * U * y.abs()
        x = y
    elif act == 2:
        x = torch.relu(x)
    if c.resid is not None:
        ldr, rbs0, rbs1 = e['resid']
        i = ((b0 * rbs0 + b1 * rbs1)[:, None, None] + torch.arange(c.M, device='cuda')[None, :, None] * ldr
             + torch.arange(c.N, device='cuda')[None, None, :])
        r = c.resid[i].double()
        bound = bound + 2 * U * (x.abs() + r.abs())
        x = x + r
    return x, bound + 2 * U * x.abs()


def _check(c, out, nsplit, impl, label):
    """exact checks of the whole output buffers, then every element of the sampled batches against the bound;
    returns the worst err / bound"""
    f32, hi, lo = out
    w = c.written
    assert bool((f32.view(torch.int32)[~w] == NAN_F32).all()), f'{label}: fp32 element outside the output written'
    assert bool((hi[~w] == NAN_BF16).all()) and bool((lo[~w] == NAN_BF16).all()), \
        f'{label}: bf16 element outside the output written'
    fw = f32[w]
    assert bool(torch.isfinite(fw).all()), f'{label}: {int((~torch.isfinite(fw)).sum())} non-finite outputs'
    h_exp = fw.to(torch.bfloat16)
    assert torch.equal(hi[w], h_exp.view(torch.int16)), f'{label}: hi != bf16_rn(f32)'
    assert torch.equal(lo[w], (fw - h_exp.float()).to(torch.bfloat16).view(torch.int16)), f'{label}: lo != bf16_rn(f32 - hi)'
    b0, b1 = _pairs(c)
    ref, bound = _reference(c, nsplit, impl, b0, b1)
    got = f32[c.out_index(b0, b1)].double()
    ratio = (got - ref).abs() / bound
    bad = ~(ratio <= 1.0)
    if bool(bad.any()):
        p, m, n = (int(v) for v in bad.nonzero()[0])
        raise AssertionError(f'{label}: {int(bad.sum())} elements past the bound, first at batch ({int(b0[p])}, '
                             f'{int(b1[p])}) row {m} column {n}: got {float(got[p, m, n])!r}, fp64 '
                             f'{float(ref[p, m, n])!r}, bound {float(bound[p, m, n]):.3g}')
    return float(ratio.max())


def _run_case(ctx, name, c, seed):
    _setup(c, seed)
    worst = {}
    for nsplit, impl in RUNS:
        if nsplit == 1:
            c.a.poison_lo()
            c.b.poison_lo()
        label = f'{name} nsplit={nsplit} gemm_impl={impl}'
        worst[(nsplit, impl)] = _check(c, _run(ctx, c, nsplit, impl), nsplit, impl, label)
    print(f'[gemm operands] {name}: worst err/bound ' + ', '.join(
        f'nsplit {ns} impl {im}: {r:.3g}' for (ns, im), r in worst.items()))
    return worst


# ------------------------------------------------------------------------------------------ call-site geometry
def _mgp(site, D, B):
    """MGP-STR's batched GEMMs (mgp.cu), built with the call sites' formulas"""
    H, Dg, R = D // 64, D // 8, B * T
    if site == 'conv':  # grouped 1x1 conv: groups are column offsets inside a row, bs0 = Dg < ld
        return Case(Opd(R, Dg, D, nb0=G, bs0=Dg), Opd(Dg, Dg, Dg, nb0=G, bs0=Dg * Dg), dict(ldo=D, obs0=Dg))
    if site == 'select':
        return Case(Opd(NTOK, D, D), Opd(T, D, D, nb1=B, bs1=T * D), dict(ldo=TP, obs1=NTOK * TP))
    if site == 'feat':  # A varies along b0 and is broadcast along b1; B varies along both
        return Case(Opd(Dg, Dg, Dg, nb0=G, bs0=Dg * Dg), Opd(T, Dg, D, nb0=G, bs0=Dg, nb1=B, bs1=T * D),
                    dict(ldo=TP, obs0=Dg * TP, obs1=D * TP))
    if site == 'xa':  # K = 257 inside ld = 264: the pad columns are never written
        return Case(Opd(NTOK, T, TP, nb1=B, bs1=NTOK * TP), Opd(D, T, TP, nb1=B, bs1=D * TP), dict(ldo=D, obs1=NTOK * D))
    if site == 'vt':  # V^T with a row bias on a batched problem
        return Case(Opd(D, D, D), Opd(T, D, D, nb1=B, bs1=T * D), dict(ldo=TP, obs1=D * TP, bias='row'))
    if site == 'scores':  # q and k as head column slices of the packed [T, 2D] projection (k at column D)
        q = Opd(T, 64, 2 * D, nb0=H, bs0=64, nb1=B, bs1=T * 2 * D)
        k = Opd(T, 64, 2 * D, nb0=H, bs0=64, nb1=B, bs1=T * 2 * D, off=D)
        return Case(q, k, dict(ldo=TP, obs0=T * TP, obs1=H * T * TP, alpha=0.125))
    assert site == 'pv'
    return Case(Opd(T, T, TP, nb0=H, bs0=T * TP, nb1=B, bs1=H * T * TP), Opd(64, T, TP, nb0=H, bs0=64 * TP, nb1=B,
                                                                               bs1=D * TP),
                dict(ldo=D, obs0=64, obs1=T * D))


def _omni(site, M, nimg, kvd=3, ncap=1, img0=1, dl=11):
    """OmniParser's batched GEMMs (omni.cu): the K / V caches, V^T and the unfused cross-attention"""
    Mpad = _r8(M)
    if site == 'kv':  # A batched along b1 only, W along b0 only, head-major column groups, per-b0 column bias
        return Case(Opd(M, 512, 512, nb1=nimg, bs1=M * 512), Opd(512, 512, 512, nb0=4 * kvd, bs0=512 * 512),
                    dict(ldo=64, obs0=8 * M * 64, obs1=96 * M * 64, cg=64, cgs=M * 64, bias='col', bias_bs0=512))
    if site == 'vt':
        return Case(Opd(6144, 512, 512), Opd(M, 512, 512, nb1=nimg, bs1=M * 512),
                    dict(ldo=Mpad, obs1=6144 * Mpad, bias='row'))
    if site == 'xscores':  # q head slices against the K cache of images img0.. and decoder layer dl
        return Case(Opd(ncap, 64, 512, nb0=8, bs0=64, nb1=nimg, bs1=ncap * 512),
                    Opd(M, 64, 64, nb0=8, bs0=M * 64, nb1=nimg, bs1=96 * M * 64, off=(img0 * 96 + dl * 8) * M * 64),
                    dict(ldo=Mpad, obs0=ncap * Mpad, obs1=8 * ncap * Mpad, alpha=0.125))
    assert site == 'xpv'  # K = M keys inside ld = Mpad
    return Case(Opd(ncap, M, Mpad, nb0=8, bs0=ncap * Mpad, nb1=nimg, bs1=8 * ncap * Mpad),
                Opd(64, M, Mpad, nb0=8, bs0=64 * Mpad, nb1=nimg, bs1=6144 * Mpad, off=(img0 * 6144 + dl * 512) * Mpad),
                dict(ldo=512, obs0=64, obs1=ncap * 512))


def _call_sites():
    cs = {}
    for site in ('conv', 'select', 'feat', 'xa', 'vt', 'scores', 'pv'):
        for D in (192, 384, 768, 1024):
            for B in (1, 3):
                cs[f'mgp_{site}_D{D}_B{B}'] = lambda site=site, D=D, B=B: _mgp(site, D, B)
    for site in ('xa', 'feat'):  # the batch of MGP-STR-base's throughput configuration
        cs[f'mgp_{site}_D768_B512'] = lambda site=site: _mgp(site, 768, 512)
    for M in (4096, 35):  # a 1024 x 1024 page, and the odd 108 x 76 page
        for kvd in (1, 3):
            cs[f'omni_kv_M{M}_kvd{kvd}'] = lambda M=M, kvd=kvd: _omni('kv', M, 2, kvd=kvd)
        cs[f'omni_vt_M{M}'] = lambda M=M: _omni('vt', M, 2)
        for ncap in (1, 16, 70):
            for site in ('xscores', 'xpv'):
                cs[f'omni_{site}_M{M}_ncap{ncap}'] = lambda site=site, M=M, ncap=ncap: _omni(site, M, 2, ncap=ncap)
    return cs


CALL_SITES = _call_sites()


@pytest.mark.parametrize('name', list(CALL_SITES))
def test_call_site_geometry_matches_fp64(ctx, name):
    _run_case(ctx, name, CALL_SITES[name](), seed=sum(map(ord, name)))


# ------------------------------------------------------------------------------------------ seeded random geometry
N_RANDOM = 60


def _random_case(i, sms):
    r = random.Random(7919 * i + 1)
    M = r.choice((r.randint(1, 64), r.randint(1, 700)))
    N = r.choice((r.randint(1, 64), r.randint(1, 700)))
    K = r.choice((r.randint(1, 64), r.randint(1, 300)))
    nb0, nb1 = r.randint(1, 5), r.randint(1, 5)
    # the first four reach each (tile width, schedule) pair of the engine on this GPU's SM count
    if i == 0:    # 128-wide tiles, ping-pong
        M, N, nb0, nb1 = 700, 700, 4, 5
    elif i == 1:  # 128-wide tiles (N <= 32), one tile per CTA
        M, N, nb0, nb1 = 300, 20, 2, 1
    elif i == 2:  # 32-wide tiles, one tile per CTA
        M, N, nb0, nb1 = 100, 200, 2, 1
    elif i == 3:  # 32-wide tiles, ping-pong: fewer than SMs / 2 128-wide tiles, more than SMs 32-wide ones
        nb0, nb1 = 5, 5
        M, N = 100, 128 * max(1, (sms // 2 - 1) // 25) - r.randint(0, 20)
    ops = []
    for j, rows in enumerate((M, N)):
        ld = _r8(K) + 8 * r.choice((0, 0, 1, 3))
        ext = [1, 1]
        for d, nb in enumerate((nb0, nb1)):
            ext[d] = nb if nb > 1 and ((i < 4 and j == 0) or r.random() < 0.7) else 1
        bs = [0, 0]
        span = rows * ld
        for d in range(2):
            if ext[d] == 1:
                bs[d] = 8 * r.randint(0, 4)  # unused: a broadcast dimension's stride must not matter
                continue
            kind = r.choice(('alias', 'tight', 'loose'))
            if kind == 'alias':   # smaller than a batch: batches overlap (read-only, so legal)
                bs[d] = 8 * r.randint(1, max(1, span // 8 - 1))
            elif kind == 'tight':
                bs[d] = span
            else:
                bs[d] = span + 8 * r.randint(1, 40)
            span = (ext[d] - 1) * bs[d] + span
        ops.append(Opd(rows, K, ld, nb0=ext[0], nb1=ext[1], bs0=bs[0], bs1=bs[1], off=8 * r.randint(0, 4),
                       gap=8 * r.randint(0, 50)))
    a, b = ops
    pnb0, pnb1 = max(a.nb0, b.nb0), max(a.nb1, b.nb1)
    e = dict(act=r.choice((0, 0, 1, 2)), alpha=r.choice((1.0, 1.0, 0.125, -0.75)))
    if r.random() < 0.2 and N > 4:  # head-major column groups
        cg = 4 * r.randint(1, 16)
        e.update(cg=cg, cgs=_r8(M * cg) + 8 * r.randint(0, 3), ldo=cg)
        blk = -(-N // cg) * e['cgs']
    else:
        e['ldo'] = N + r.choice((0, 0, 3, 8 - N % 8 if N % 8 else 0))
        blk = M * e['ldo']
        if r.random() < 0.3:
            e['resid'] = None  # filled below
    pad = r.choice((0, 8))
    if r.random() < 0.5:   # b0 inner, b1 outer
        e['obs0'] = blk + pad
        e['obs1'] = pnb0 * e['obs0'] + pad
    else:                  # b1 inner, b0 outer
        e['obs1'] = blk + pad
        e['obs0'] = pnb1 * e['obs1'] + pad
    bias = r.choice((None, 'col', 'row'))
    if bias:
        e['bias'] = bias
        if pnb0 > 1 and r.random() < 0.7:
            e['bias_bs0'] = 4 * (-(-(N if bias == 'col' else M) // 4) + 1)
    if 'resid' in e:
        ldr = N + r.choice((0, 4))
        e['resid'] = (ldr, M * ldr + 4, pnb0 * (M * ldr + 4) + 8)
    return Case(a, b, e, lo_null=r.random() < 0.5)


@pytest.mark.parametrize('i', range(N_RANDOM))
def test_random_geometry_matches_fp64(ctx, i):
    _run_case(ctx, f'random_{i}', _random_case(i, support.sms()), seed=1000 + i)


def test_random_geometry_reaches_both_tile_widths_and_schedules():
    sms = support.sms()
    seen = set()
    for i in range(N_RANDOM):
        c = _random_case(i, sms)
        seen.add(_launch_shape(c.M, c.N, c.nb0 * c.nb1, sms))
    assert seen == {(w, s) for w in (32, 128) for s in ('ping-pong', 'one tile per CTA')}, seen


# ------------------------------------------------------------------------------------------ slice invariance
SLICES = {
    # N <= 32: 128-wide tiles batched and unbatched; the grouped-conv geometry
    'mgp_conv_D192_B3': lambda: _mgp('conv', 192, 3),
    # 32-wide tiles both ways: 27 x 768 per batch
    'mgp_xa_D768_B3': lambda: _mgp('xa', 768, 3),
    # 128-wide tiles both ways: >= SMs / 2 tiles even unbatched; K = 133, both operands batched along both dims
    'wide_both_batched': lambda: Case(Opd(700, 133, 144, nb0=2, nb1=3, bs0=700 * 144 + 8, bs1=2 * (700 * 144 + 8)),
                                      Opd(1500, 133, 136, nb0=2, nb1=3, bs0=136, bs1=2 * 136 * 1500),
                                      dict(ldo=1504, obs0=700 * 1504, obs1=2 * 700 * 1504, bias='col', bias_bs0=1504,
                                           act=1)),
    # 32-wide tiles both ways, A broadcast along b0 and B along b1, residual strided along both
    'narrow_broadcast': lambda: Case(Opd(100, 77, 80, nb1=3, bs1=100 * 80), Opd(200, 77, 88, nb0=2, bs0=200 * 88),
                                     dict(ldo=200, obs0=100 * 200, obs1=2 * 100 * 200, resid=(208, 100 * 208,
                                                                                                 2 * 100 * 208))),
}


@pytest.mark.parametrize('name', list(SLICES))
def test_slice_of_a_batched_launch_equals_the_unbatched_call(ctx, name):
    c = SLICES[name]()
    sms = support.sms()
    assert _launch_shape(c.M, c.N, c.nb0 * c.nb1, sms)[0] == _launch_shape(c.M, c.N, 1, sms)[0], \
        'the case must give both launches the same tile width'
    _setup(c, seed=sum(map(ord, name)))
    for nsplit, impl in RUNS:
        if nsplit == 1:
            c.a.poison_lo()
            c.b.poison_lo()
        batched = _run(ctx, c, nsplit, impl)
        with options(ctx, nsplit=nsplit, gemm_impl=impl):   # the unbatched calls run at the same settings
            for b0, b1 in {(0, 0), (c.nb0 - 1, c.nb1 - 1), (c.nb0 // 2, c.nb1 - 1)}:
                idx = c.out_index(torch.tensor([b0], device='cuda'), torch.tensor([b1], device='cuda'))[0]
                sub = Case(c.a, c.b, dict(c.e, obs0=0, obs1=0))
                one = _outputs(int(sub.out_index(torch.zeros(1, dtype=torch.long, device='cuda'),
                                                 torch.zeros(1, dtype=torch.long, device='cuda')).max()) + 1 + GUARD)
                ctx.check(_call(ctx, c.a.desc(True, b0, b1, whole=False), c.b.desc(True, b0, b1, whole=False),
                                _epilogue(c, *one, b0=b0, b1=b1)))
                sidx = sub.out_index(torch.zeros(1, dtype=torch.long, device='cuda'),
                                     torch.zeros(1, dtype=torch.long, device='cuda'))[0]
                for k, (x, y) in enumerate(zip(batched, one)):
                    xv = x[idx].view(torch.int32) if k == 0 else x[idx]
                    yv = y[sidx].view(torch.int32) if k == 0 else y[sidx]
                    assert torch.equal(xv, yv), (f'nsplit {nsplit} gemm_impl {impl}: slice ({b0}, {b1}) output '
                                                 f'{("f32", "hi", "lo")[k]} differs from the unbatched call')


# ------------------------------------------------------------------------------------------ argument checks
def test_rejects_operands_the_engine_cannot_address(ctx):
    c = Case(Opd(40, 20, 24, nb0=2, bs0=40 * 24), Opd(50, 20, 32, nb0=2, bs0=50 * 32, gap=16), dict(ldo=56, obs0=40 * 56))
    _setup(c, seed=5)
    out = _outputs(c.written.numel())
    host = (ctypes.c_uint16 * 4096)()
    host_ptr = (ctypes.addressof(host) + 15) // 16 * 16

    def op(o, **kw):
        d = o.desc()
        for k, v in kw.items():
            setattr(d, k, v)
        return d

    a, b = c.a, c.b
    hi, lo = a.buf.data_ptr(), a.buf.data_ptr() + 2 * a.dist
    bad = {
        'null hi': (op(a, hi=None), op(b)),
        'host hi': (op(a, hi=host_ptr), op(b)),
        'host lo': (op(a, lo=host_ptr + 2048), op(b)),
        'hi not 16-byte aligned': (op(a, hi=hi + 2, lo=lo + 2), op(b)),
        'lo not 16-byte aligned': (op(a, lo=lo + 8), op(b)),
        'ld % 8': (op(a, ld=20), op(b)),
        'bs0 % 8': (op(a, bs0=40 * 24 + 4), op(b)),
        'bs1 % 8': (op(a), op(b, bs1=12)),
        'lo before hi': (op(a, hi=lo, lo=hi), op(b)),
        'lo == hi': (op(a, lo=hi), op(b)),
        'ld < K': (op(a, ld=16), op(b)),
        'extents do not broadcast': (op(a, nb0=3), op(b)),
        'b1 extents do not broadcast': (op(a, nb1=2, bs1=8), op(b, nb1=3, bs1=8)),
    }
    with options(ctx, nsplit=3):
        for what, (x, y) in bad.items():
            assert _call(ctx, x, y, _epilogue(c, *out)) == ALM_ERR_INVALID, what
        assert _call(ctx, op(a, lo=None), op(b), _epilogue(c, *out)) == ALM_ERR_INVALID, 'no lo plane at nsplit 3'
        assert ctx.lib.alm_op_gemm_planes(ctx.h, None, ctypes.byref(op(b)), ctypes.byref(_epilogue(c, *out))) == \
            ALM_ERR_INVALID
        e = _epilogue(c, *out)
        e.out_f32 = host_ptr
        assert _call(ctx, op(a), op(b), e) == ALM_ERR_INVALID, 'host output'
        e = _epilogue(c, *out)
        e.out_f32 = e.out_hi = e.out_lo = None
        assert _call(ctx, op(a), op(b), e) == ALM_ERR_INVALID, 'no output'
        # nothing was written, and the context still runs a valid call afterwards
        for t in out:
            assert bool((t.view(torch.int32) == NAN_F32).all()) if t.dtype == torch.float32 else bool((t == NAN_BF16).all())
        _check(c, _run(ctx, c, 3, 0), 3, 0, 'after the rejections')
        c.a.poison_lo()
        c.b.poison_lo()
        c.lo_null = True  # nsplit 1 runs without lo planes
        _check(c, _run(ctx, c, 1, 0), 1, 0, 'nsplit 1 without lo planes')
