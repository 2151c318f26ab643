"""GPU: MGP-STR's forward replayed op by op through the op-level entry points, bit for bit against the model.

Every kernel MGP-STR runs is held to fp64 on its own, on random operands (test_gpu_gemm_operands.py,
test_gpu_gemm_epilogue.py, test_gpu_gemm_capped.py, test_gpu_encoder_ops.py, test_gpu_mgp_ops.py).  Here the forward
is rebuilt from those entry points alone -- alm_op_patch_im2col, alm_op_gemm_planes, alm_op_gather_ln,
alm_op_attention_ex, alm_op_softmax_rows and alm_op_row_select -- in the reference's op order (oracle/mgpstr_ref.py:
the reference's modules/mgp_str.py:64-91, the timm-0.4.12 Block the ViT inherits, modules/token_learner.py:21-33).
The kernels are deterministic, so the replay must give MGPSTRB200.forward(is_eval=True)'s three A^3 maps and three logit
tensors, and recognize_topk's ids and probabilities, bit for bit.  The op tests then cover the model: each op is
held to fp64, and the match shows that mgp_forward (csrc/mgp.cu) runs exactly those ops on exactly those buffers.

Only layout conventions come from the library: token-major rows, T = 257 tokens padded to TP = 264 for the A^3 maps and
the feature-major operands, and [N, Kpad] weight planes (hi = bf16_rn(w), lo = bf16_rn(w - hi), K zero-padded to a
multiple of 8, the packed [3D, D] qkv as stored).

Poisoning: every buffer the replay allocates holds NaN until its producer writes it, and is followed by a guard that
must still hold NaN once its consumers have run.  At nsplit 1 no producer is handed a lo plane, so every lo plane stays
NaN: a consumer that read one would turn the replay into NaN where the model, whose producers may write lo planes,
stays finite.  The pad columns T .. TP-1 of the A^3 maps and of feat^T are never written by anything.

fp64 (crops 0, 1, 255, 256, 510 and 511 at B = 512, every crop at small B): every op of the replay also writes its
fp32 value, which is checked against fp64 of that op on the replay's own inputs with the op tests' bounds -- GEMMs
|got - ref| <= n 2^-22 sum|terms| over the products the kernel forms from its planes (carried through alpha, bias, GELU
and residual as in test_gpu_gemm_operands.py), attention _attn_tol, LayerNorm and row softmax as in
test_gpu_encoder_ops.py, the selection as in test_gpu_mgp_ops.py -- and every split output must be hi = bf16_rn(x),
lo = bf16_rn(x - hi) (hi only at nsplit 1).  The worst err / bound of every op kind and block is printed.
"""
import ctypes

import pytest
import torch
import torch.nn.functional as F

from tests.support import options
from tests.test_gpu_mgp_ops import _attn_ref, _attn_tol, _check_select

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

T, TP, NTOK, NPATCH, G = 257, 264, 27, 256, 8   # tokens, their padded stride, A^3 tokens, patches, conv groups
GUARD = 256                                     # elements after every buffer (a multiple of 8: planes stay aligned)
NAN16 = -1                                      # 0xffff: a bf16 NaN
NAN_F32 = 0x7fc00000
U32 = 2.0 ** -24
K_TOP = 5


# ----------------------------------------------------------------------------------------------- checkpoints
def _checkpoint(name):
    """-> (state dict, batch, crops checked against fp64 or None for all)"""
    from advancedliteratemachinery_b200 import synthetic as S
    from tests.conftest import mgp_sd
    if name.startswith('base'):
        B = int(name[len('base-B'):])
        return mgp_sd(0), B, ([0, 1, 255, 256, 510, 511] if B == 512 else None)
    if name in ('tiny', 'small', 'large'):
        dim, depth, heads = S.MGP_VARIANTS[name]
        return S.mgpstr_state_dict(seed=5, dim=dim, depth=depth, heads=heads), 2, None
    if name == 'charstr':
        return S.mgpstr_state_dict(seed=6, char_only=True), 2, None
    assert name in ('depth1', 'depth2')
    return S.mgpstr_state_dict(seed=7, depth=int(name[-1])), 3, None


class _Lin:
    """a weight [N, K] as upload_split lays it out: hi / lo int16 planes [N, Kpad] in one buffer, lo after hi"""

    def __init__(self, w, b=None, Kpad=None):
        w = w.reshape(w.shape[0], -1).float().cuda()
        N, K = w.shape
        Kp = Kpad or (K + 7) // 8 * 8
        buf = torch.zeros(2, N, Kp, dtype=torch.int16, device='cuda')
        hi = w.to(torch.bfloat16)
        buf[0, :, :K] = hi.view(torch.int16)
        buf[1, :, :K] = (w - hi.float()).to(torch.bfloat16).view(torch.int16)
        self.hi, self.lo, self.N, self.K = buf[0], buf[1], N, Kp
        self.b = b.float().cuda().contiguous() if b is not None else None

    def rows(self, r0, r1):
        """rows r0 .. r1-1 as a weight of their own (the unfused path's q|k and v views of the packed qkv)"""
        v = _Lin.__new__(_Lin)
        v.hi, v.lo, v.N, v.K = self.hi[r0:r1], self.lo[r0:r1], r1 - r0, self.K
        v.b = self.b[r0:r1] if self.b is not None else None
        return v


class _Weights:
    def __init__(self, sd):
        sd = {k[len('module.mgp_str.'):] if k.startswith('module.mgp_str.') else k: v for k, v in sd.items()}
        dev = lambda k: sd[k].float().cuda().contiguous()
        lin = lambda p, **kw: _Lin(sd[p + '.weight'], sd.get(p + '.bias'), **kw)
        ln = lambda p: (dev(p + '.weight'), dev(p + '.bias'))
        self.D = sd['pos_embed'].shape[2]
        self.H = self.D // 64
        self.patch = lin('patch_embed.proj', Kpad=64)
        self.cls = dev('cls_token').reshape(-1)
        self.pos = dev('pos_embed').reshape(T, self.D)
        self.blocks = []
        b = 0
        while f'blocks.{b}.norm1.weight' in sd:
            p = f'blocks.{b}.'
            self.blocks.append(dict(n1=ln(p + 'norm1'), n2=ln(p + 'norm2'), qkv=lin(p + 'attn.qkv'),
                                    proj=lin(p + 'attn.proj'), fc1=lin(p + 'mlp.fc1'), fc2=lin(p + 'mlp.fc2')))
            b += 1
        names = ('char', 'bpe', 'wp') if 'bpe_tokenLearner.token_norm.weight' in sd else ('char',)
        self.a3 = []
        for a in names:
            p = a + '_tokenLearner.'
            # CHAR-STR reads its logits through timm's `head` (modules/char_str.py:70)
            self.a3.append(dict(token_norm=ln(p + 'token_norm'), norm=ln(p + 'norm'), w0=lin(p + 'tokenLearner.0'),
                                w1=lin(p + 'tokenLearner.1'), feat=lin(p + 'feat'),
                                head=lin('head' if len(names) == 1 else a + '_head')))


_CACHE = {}


def _model(name):
    """(MGPSTRB200, _Weights, B, crops) of a checkpoint; one kept at a time"""
    if name not in _CACHE:
        from advancedliteratemachinery_b200 import MGPSTRB200
        _close_all()
        sd, B, crops = _checkpoint(name)
        _CACHE[name] = (MGPSTRB200(sd), _Weights(sd), B, crops)
    return _CACHE[name]


def _close_all():
    """close the cached model's context and hand torch's cached blocks back, so that the next context's workspace
    (24 GB by default) finds room"""
    for k in list(_CACHE):
        _CACHE.pop(k)[0].ctx.close()
    torch.cuda.empty_cache()


@pytest.fixture(scope='module', autouse=True)
def _close_models():
    yield
    _close_all()
    for kind, r in sorted(WORST.items()):
        print(f'[mgp replay] {kind}: worst err / bound over the module {r:.3g}')


def _image(B, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(B, 3, 32, 128, generator=g).cuda()


# ----------------------------------------------------------------------------------------------- buffers
class _Pool:
    """device buffers of one stage of the replay, NaN until written, each followed by GUARD NaN elements"""

    def __init__(self):
        self.fulls = []

    def f32(self, n):
        full = torch.full((n + GUARD,), float('nan'), device='cuda')
        self.fulls.append((full, n))
        return full[:n]

    def i32(self, n):
        full = torch.full((n + GUARD,), -7, dtype=torch.int32, device='cuda')
        self.fulls.append((full, n))
        return full[:n]

    def planes(self, n):
        d = (n + GUARD + 7) // 8 * 8
        full = torch.full((2 * d,), NAN16, dtype=torch.int16, device='cuda')
        self.fulls += [(full[:d], n), (full[d:], n)]
        return full[:n], full[d:d + n]

    def done(self):
        """every guard intact; the buffers are released"""
        for full, n in self.fulls:
            g = full[n:]
            want = {torch.float32: NAN_F32, torch.int32: -7, torch.int16: NAN16}[g.dtype]
            bits = g.view(torch.int32) if g.dtype == torch.float32 else g
            assert bool((bits == want).all()), 'a write past the end of a buffer'
        self.fulls = []


def _p(t):
    return None if t is None else t.data_ptr()


def _opd(hi, lo, rows, K, ld, nb0=1, bs0=0, nb1=1, bs1=0):
    from advancedliteratemachinery_b200 import _lib
    return _lib.GemmOperand(hi.data_ptr(), _p(lo), rows, K, ld, nb0, nb1, bs0, bs1)


def _wop(w):
    return _opd(w.hi, w.lo, w.N, w.K, w.K)


def _epi(f32=None, hi=None, lo=None, ldo=0, obs0=0, obs1=0, bias=None, bias_mode=0, resid=None, ldr=0, out_map=None,
         resid_map=None, act=0, alpha=1.0):
    from advancedliteratemachinery_b200 import _lib
    return _lib.GemmEpilogue(_p(f32), _p(hi), _p(lo), ldo, obs0, obs1, 0, 0, _p(bias), bias_mode if bias is not None
                             else 0, 0, _p(resid), ldr, 0, 0, _p(out_map), _p(resid_map), act, alpha)


# ----------------------------------------------------------------------------------------------- fp64 checks
def _bf(x):
    return x.view(torch.bfloat16).double()


WORST = {}


class _Checker:
    """fp64 of every op of the replay on its own inputs, for the token rows of the checked crops"""

    def __init__(self, ns, crops, label):
        self.ns, self.label = ns, label
        self.crops = torch.tensor(crops, device='cuda')
        self.worst = {}

    def rows(self, per):
        return (self.crops[:, None] * per + torch.arange(per, device='cuda')).flatten()

    def _record(self, kind, where, err, bound):
        ratio = float((err / bound).max())
        bad = ~(err <= bound)
        assert not bool(bad.any()), (f'{self.label} {kind} ({where}): {int(bad.sum())} elements past the bound, worst '
                                     f'err / bound {ratio:.3g}')
        key = (kind, where)
        self.worst[key] = max(self.worst.get(key, 0.0), ratio)
        WORST[kind] = max(WORST.get(kind, 0.0), ratio)

    def split(self, kind, where, f32, hi, lo):
        """the planes of the fp32 values f32 (same shape): hi = bf16_rn(x), lo = bf16_rn(x - hi); lo NaN at nsplit 1"""
        assert bool(torch.isfinite(f32).all()), f'{self.label} {kind} ({where}): non-finite fp32 output'
        h = f32.to(torch.bfloat16)
        assert torch.equal(hi, h.view(torch.int16)), f'{self.label} {kind} ({where}): hi != bf16_rn(x)'
        if self.ns == 3:
            assert torch.equal(lo, (f32 - h.float()).to(torch.bfloat16).view(torch.int16)), \
                f'{self.label} {kind} ({where}): lo != bf16_rn(x - hi)'
        else:
            assert bool((lo == NAN16).all()), f'{self.label} {kind} ({where}): a lo plane written at nsplit 1'

    def gemm(self, kind, where, a, b, got, alpha=1.0, bias=None, act=0, resid=None):
        """a = (hi, lo) int16 [P, M, K], b = (hi, lo) [P, N, K]: the planes the kernel reads; got fp32 [P, M, N]; bias /
        resid broadcast to it.  The bound of test_gpu_gemm_operands.py: n 2^-22 sum|terms| over the n products each
        element sums, then a few ulps per epilogue rounding (2e-7 max(1, |x| / 2) for the rational GELU)."""
        ah, bh = _bf(a[0]), _bf(b[0])
        mm = lambda x, y: torch.matmul(x, y.transpose(-1, -2))
        K = a[0].shape[-1]
        if self.ns == 3:
            al, bl = _bf(a[1]), _bf(b[1])
            acc = mm(ah, bh) + mm(al, bh) + mm(ah, bl)
            s = mm(ah.abs(), bh.abs()) + mm(al.abs(), bh.abs()) + mm(ah.abs(), bl.abs())
            n = 3 * K
        else:
            acc, s, n = mm(ah, bh), mm(ah.abs(), bh.abs()), K
        x = alpha * acc
        bound = abs(alpha) * n * 2.0 ** -22 * s
        if bias is not None:
            bv = bias.double()
            bound = bound + 4 * U32 * (x.abs() + bv.abs())
            x = x + bv
        else:
            bound = bound + 2 * U32 * x.abs()
        if act == 1:
            y = F.gelu(x)
            bound = 1.13 * bound + 2e-7 * torch.clamp(0.5 * x.abs(), min=1.0) + 4 * U32 * y.abs()
            x = y
        if resid is not None:
            r = resid.double()
            bound = bound + 2 * U32 * (x.abs() + r.abs())
            x = x + r
        bound = bound + 2 * U32 * x.abs()
        self._record(kind, where, (got.double() - x).abs(), bound)

    def ln(self, kind, where, x, gamma, beta, eps, got):
        """fp32 LayerNorm of rows x: test_gpu_encoder_ops.py's bound, with this LayerNorm's eps"""
        x64 = x.double()
        ref = F.layer_norm(x64, (x.shape[-1],), gamma.double(), beta.double(), eps)
        mean = x64.mean(-1, keepdim=True)
        rstd = (x64.var(-1, unbiased=False, keepdim=True) + eps).rsqrt()
        tol = 1e-5 + 2.0 ** -20 * ref.abs() + 32 * U32 * mean.abs() * rstd * gamma.double().abs()
        self._record(kind, where, (got.double() - ref).abs(), tol)

    def softmax(self, kind, where, s, got):
        """row softmax of fp32 rows s: test_gpu_encoder_ops.py's bound"""
        x = s.double()
        ref = x.softmax(-1)
        m = x.max(-1, keepdim=True).values
        rel = U32 * (2 * (x - m).abs() + x.shape[-1] / 128 + 16)
        self._record(kind, where, (got.double() - ref).abs(), ref * rel + 2.0 ** -126)

    def attention(self, where, qkv, nb, H, got):
        """qkv fp32 [nb T, 3D] of the checked crops (the values the planes split), got fp32 [nb T, D]"""
        ref = _attn_ref(qkv, nb, T, H)
        self._record('attention', where, (got.double() - ref['o']).abs(), _attn_tol(ref, self.ns))

    def report(self):
        kinds = {}
        for (kind, where), r in self.worst.items():
            kinds.setdefault(kind, []).append((r, where))
        for kind, rs in kinds.items():
            r, where = max(rs)
            per = ', '.join(f'{w}: {x:.3g}' for x, w in rs) if len(rs) > 1 else ''
            print(f'[{self.label}] {kind}: worst err / bound {r:.3g} ({where})' + (f'; {per}' if per else ''))


# ----------------------------------------------------------------------------------------------- the replay
def _replay(ctx, w, img, ns, impl, chk=None):
    """The forward from op entry points under the context's nsplit (ns) -> dict(attn, logits, ids, probs, ids_k,
    probs_k, launches): per A^3 head the maps [B, 27, 257], logits [B, 27, V], top-1 ids / probs [B, 27] and the
    K_TOP candidates [B, 27, K_TOP]; launches: what the replay launched, the extra K_TOP selections not counted.
    impl: the ViT attention of attn_impl 0 (fused kernel) or 1 (GEMMs + row softmax).  chk: a _Checker, which makes
    every producer also write its fp32 value and checks every op on the checked crops."""
    B = img.shape[0]
    D, H = w.D, w.H
    R, Dg = B * T, D // 8
    lib, h = ctx.lib, ctx.h

    def call(name, *args):
        torch.cuda.synchronize()    # the context runs on its own stream
        ctx.check(getattr(lib, name)(h, *args))

    def gemm(a, b, e):
        torch.cuda.synchronize()
        ctx.check(lib.alm_op_gemm_planes(h, ctypes.byref(a), ctypes.byref(b), ctypes.byref(e)))

    def out_planes(pool, n):
        """(hi, lo, lo handed to the producer, fp32 twin or None)"""
        hi, lo = pool.planes(n)
        return hi, lo, lo if ns == 3 else None, pool.f32(n) if chk else None

    def layernorm(src, rows, gb, eps, pool, where, kind):
        hi, lo, lo_w, f = out_planes(pool, rows * D)
        call('alm_op_gather_ln', src.data_ptr(), D, None, 1, D, rows, gb[0].data_ptr(), gb[1].data_ptr(), eps, 0, None,
             0, _p(f), D, hi.data_ptr(), _p(lo_w), D, None, None, None)
        if chk:
            r = chk.rows(T if rows == R else NTOK)
            chk.ln(kind, where, src.view(rows, D)[r], gb[0], gb[1], eps, f.view(rows, D)[r])
            chk.split(kind, where, f.view(rows, D)[r], hi.view(rows, D)[r], lo.view(rows, D)[r])
        return hi, lo

    def linear(a, l, rows, pool, where, kind, out_x=None, act=0):
        """rows of the planes a x l^T + bias (timm's Linear): to split planes -> (hi, lo, fp32 twin or None), or
        (out_x) added in place to x"""
        if out_x is None:
            hi, lo, lo_w, f = out_planes(pool, rows * l.N)
            e = _epi(f, hi, lo_w, ldo=l.N, bias=l.b, bias_mode=1, act=act)
            before = None
        else:
            e = _epi(out_x, ldo=l.N, bias=l.b, bias_mode=1, resid=out_x, ldr=l.N)
            r = chk.rows(T) if chk else None
            before = out_x.view(rows, l.N)[r].clone() if chk else None
        gemm(_opd(a[0], a[1], rows, l.K, l.K), _wop(l), e)
        if chk:
            r = chk.rows(T if rows == R else NTOK)
            av = tuple(p.view(rows, l.K)[r][None] for p in a[:2])
            got = (f if out_x is None else out_x).view(rows, l.N)[r]
            chk.gemm(kind, where, av, (l.hi[None], l.lo[None]), got[None], bias=l.b, act=act,
                     resid=None if before is None else before[None])
            if out_x is None:
                chk.split(kind, where, got, hi.view(rows, l.N)[r], lo.view(rows, l.N)[r])
        return None if out_x is not None else (hi, lo, f)

    top = _Pool()
    # ---- patch embed + cls + pos (mgp_str.py:66-70): the 4 x 4 / stride-4 conv as im2col + GEMM, K 48 padded to 64
    pool = _Pool()
    a_hi, a_lo = pool.planes(B * NPATCH * 64)
    call('alm_op_patch_im2col', img.data_ptr(), B, 32, 128, None, B, 32, 128, a_hi.data_ptr(),
         _p(a_lo if ns == 3 else None))
    x = top.f32(R * D)
    r = torch.arange(B * NPATCH, device='cuda', dtype=torch.int32)
    omap = ((r // NPATCH) * T + 1 + r % NPATCH).int()   # patch p of crop b -> token row b 257 + 1 + p
    rmap = (1 + r % NPATCH).int()                        # ... whose position embedding is pos row 1 + p
    x.view(B, T, D)[:, 0] = w.cls + w.pos[0]             # the cls token row: one fp32 add
    gemm(_opd(a_hi, a_lo, B * NPATCH, 64, 64), _wop(w.patch),
         _epi(x, ldo=D, bias=w.patch.b, bias_mode=1, resid=w.pos, ldr=D, out_map=omap, resid_map=rmap))
    if chk:
        nc = len(chk.crops)
        pr = chk.rows(NPATCH)
        ref = img[chk.crops].view(nc, 3, 8, 4, 32, 4).permute(0, 2, 4, 1, 3, 5).reshape(nc * NPATCH, 48)
        ref = torch.cat([ref, torch.zeros(nc * NPATCH, 16, device='cuda')], 1)
        chk.split('im2col', 'patches', ref, a_hi.view(-1, 64)[pr], a_lo.view(-1, 64)[pr])   # exact
        xr = x.view(B, T, D)[chk.crops]
        assert torch.equal(xr[:, 0].view(torch.int32), (w.cls + w.pos[0]).expand(nc, D).view(torch.int32))
        chk.gemm('patch GEMM', 'patches', (a_hi.view(-1, 64)[pr][None], a_lo.view(-1, 64)[pr][None]),
                 (w.patch.hi[None], w.patch.lo[None]), xr[:, 1:].reshape(1, -1, D), bias=w.patch.b,
                 resid=w.pos[1:].repeat(nc, 1)[None])
    pool.done()

    # ---- ViT blocks (timm 0.4.12 Block: x + attn(norm1(x)), x + mlp(norm2(x)); LayerNorm eps 1e-6)
    for i, blk in enumerate(w.blocks):
        where = f'block {i}'
        pool = _Pool()
        ln = layernorm(x, R, blk['n1'], 1e-6, pool, where, 'LayerNorm')
        o_hi, o_lo, o_lo_w, o_f = out_planes(pool, R * D)
        if impl == 0:   # the packed qkv projection, then softmax(q k^T * 64^-0.5) v in one kernel
            qkv = linear(ln, blk['qkv'], R, pool, where, 'qkv GEMM')
            call('alm_op_attention_ex', qkv[0].data_ptr(), qkv[1].data_ptr(), 3 * D, B, T, H, _p(o_f), o_hi.data_ptr(),
                 _p(o_lo_w), D)
            if chk:     # on the fp32 qkv the planes are the split of (checked in linear)
                tr = chk.rows(T)
                chk.attention(where, qkv[2].view(R, 3 * D)[tr], len(chk.crops), H, o_f.view(R, D)[tr])
                chk.split('attention', where, o_f.view(R, D)[tr], o_hi.view(R, D)[tr], o_lo.view(R, D)[tr])
        else:           # q|k and V^T GEMMs, scores, row softmax, P.V
            qk = linear(ln, blk['qkv'].rows(0, 2 * D), R, pool, where, 'q|k GEMM')
            wv = blk['qkv'].rows(2 * D, 3 * D)
            vt_hi, vt_lo, vt_lo_w, vt_f = out_planes(pool, B * D * TP)
            gemm(_wop(wv), _opd(ln[0], ln[1], T, D, D, nb1=B, bs1=T * D),
                 _epi(vt_f, vt_hi, vt_lo_w, ldo=TP, obs1=D * TP, bias=wv.b, bias_mode=2))
            S = pool.f32(B * H * T * TP)
            q = _opd(qk[0], qk[1], T, 64, 2 * D, nb0=H, bs0=64, nb1=B, bs1=T * 2 * D)
            k = _opd(qk[0][D:], qk[1][D:], T, 64, 2 * D, nb0=H, bs0=64, nb1=B, bs1=T * 2 * D)
            gemm(q, k, _epi(S, ldo=TP, obs0=T * TP, obs1=H * T * TP, alpha=0.125))
            P_hi, P_lo, P_lo_w, P_f = out_planes(pool, B * H * T * TP)
            call('alm_op_softmax_rows', S.data_ptr(), TP, B * H * T, T, None, 1, 0, _p(P_f), P_hi.data_ptr(),
                 _p(P_lo_w), TP)
            p = _opd(P_hi, P_lo, T, T, TP, nb0=H, bs0=T * TP, nb1=B, bs1=H * T * TP)
            v = _opd(vt_hi, vt_lo, 64, T, TP, nb0=H, bs0=64 * TP, nb1=B, bs1=D * TP)
            gemm(p, v, _epi(o_f, o_hi, o_lo_w, ldo=D, obs0=64, obs1=T * D))
            if chk:
                _check_unfused(chk, where, ln, wv, (vt_hi, vt_lo, vt_f), qk, S, (P_hi, P_lo, P_f), (o_hi, o_lo, o_f),
                               B, D, H)
        linear((o_hi, o_lo), blk['proj'], R, pool, where, 'proj GEMM + residual', out_x=x)
        ln = layernorm(x, R, blk['n2'], 1e-6, pool, where, 'LayerNorm')
        hid = linear(ln, blk['fc1'], R, pool, where, 'fc1 GEMM + GELU', act=1)
        linear(hid, blk['fc2'], R, pool, where, 'fc2 GEMM + residual', out_x=x)
        pool.done()

    # ---- A^3 modules (token_learner.py:21-33) and their heads (mgp_str.py:79-91); LayerNorm eps 1e-5
    out = dict(attn=[], logits=[], ids=[], probs=[], ids_k=[], probs_k=[])
    extra = 0
    for a, m in enumerate(w.a3):
        where = ('char', 'bpe', 'wp')[a]
        pool = _Pool()
        tn = layernorm(x, R, m['token_norm'], 1e-5, pool, where, 'A3 LayerNorm')
        # tokenLearner[0]: the grouped 1 x 1 conv, group g a [R, Dg] x [Dg, Dg]^T GEMM at column g Dg
        s0_hi, s0_lo, s0_lo_w, s0_f = out_planes(pool, R * D)
        gemm(_opd(tn[0], tn[1], R, Dg, D, nb0=G, bs0=Dg), _opd(m['w0'].hi, m['w0'].lo, Dg, Dg, Dg, nb0=G, bs0=Dg * Dg),
             _epi(s0_f, s0_hi, s0_lo_w, ldo=D, obs0=Dg))
        # tokenLearner[1]: selected^T[b, s, t] = W1[s] . s0[b, t], token-major maps of stride TP
        sel = pool.f32(B * NTOK * TP)
        gemm(_wop(m['w1']), _opd(s0_hi, s0_lo, T, D, D, nb1=B, bs1=T * D), _epi(sel, ldo=TP, obs1=NTOK * TP))
        attn = pool.f32(B * NTOK * TP)
        Pa_hi, Pa_lo = pool.planes(B * NTOK * TP)
        call('alm_op_softmax_rows', sel.data_ptr(), TP, B * NTOK, T, None, 1, 0, attn.data_ptr(), Pa_hi.data_ptr(),
             _p(Pa_lo if ns == 3 else None), TP)
        # feat: the grouped 1 x 1 conv again, written feature-major: feat^T[b, g Dg + f, t]
        ft_hi, ft_lo, ft_lo_w, ft_f = out_planes(pool, B * D * TP)
        gemm(_opd(m['feat'].hi, m['feat'].lo, Dg, Dg, Dg, nb0=G, bs0=Dg * Dg),
             _opd(tn[0], tn[1], T, Dg, D, nb0=G, bs0=Dg, nb1=B, bs1=T * D),
             _epi(ft_f, ft_hi, ft_lo_w, ldo=TP, obs0=Dg * TP, obs1=D * TP))
        # x_a[b] = selected[b] (27 x 257) . feat[b] (257 x D): K = 257 inside the stride 264
        xa = pool.f32(B * NTOK * D)
        gemm(_opd(Pa_hi, Pa_lo, NTOK, T, TP, nb1=B, bs1=NTOK * TP), _opd(ft_hi, ft_lo, D, T, TP, nb1=B, bs1=D * TP),
             _epi(xa, ldo=D, obs1=NTOK * D))
        xn = layernorm(xa, B * NTOK, m['norm'], 1e-5, pool, where, 'A3 LayerNorm')
        hd = m['head']
        Vpad = (hd.N + 7) // 8 * 8
        logits = pool.f32(B * NTOK * Vpad)
        gemm(_opd(xn[0], xn[1], B * NTOK, D, D), _wop(hd), _epi(logits, ldo=Vpad, bias=hd.b, bias_mode=1))
        if chk:
            _check_a3(chk, where, tn, (s0_hi, s0_lo, s0_f), m, sel, attn, (Pa_hi, Pa_lo), (ft_hi, ft_lo, ft_f), xa, xn,
                      logits, B, D, Vpad)
        # demo.py:36-60: the top-1 id and its softmax probability; then the K_TOP candidates
        ids, probs = pool.i32(B * NTOK), pool.f32(B * NTOK)
        call('alm_op_row_select', logits.data_ptr(), Vpad, B * NTOK, hd.N, 0, ids.data_ptr(), probs.data_ptr())
        ids_k, probs_k = pool.i32(B * NTOK * K_TOP), pool.f32(B * NTOK * K_TOP)
        call('alm_op_row_select', logits.data_ptr(), Vpad, B * NTOK, hd.N, K_TOP, ids_k.data_ptr(), probs_k.data_ptr())
        extra += 1
        out['attn'].append(attn.view(B, NTOK, TP)[:, :, :T])
        out['logits'].append(logits.view(B, NTOK, Vpad)[:, :, :hd.N])
        out['ids'].append(ids.view(B, NTOK))
        out['probs'].append(probs.view(B, NTOK))
        out['ids_k'].append(ids_k.view(B, NTOK, K_TOP))
        out['probs_k'].append(probs_k.view(B, NTOK, K_TOP))
        pool.done()
    top.done()
    out['extra_launches'] = extra
    return out


def _check_unfused(chk, where, ln, wv, vt, qk, S, P, o, B, D, H):
    """V^T, scores, row softmax and P.V of the checked crops against fp64"""
    c = chk.crops
    nc = len(c)
    tr = chk.rows(T)
    lnv = tuple(p.view(B, T, D)[c] for p in ln)                                          # [nc, T, D]
    vt_f = vt[2].view(B, D, TP)[c][:, :, :T]
    chk.gemm('V^T GEMM', where, (wv.hi[None], wv.lo[None]), lnv, vt_f, bias=wv.b[None, :, None])
    chk.split('V^T GEMM', where, vt_f, vt[0].view(B, D, TP)[c][:, :, :T], vt[1].view(B, D, TP)[c][:, :, :T])
    assert bool((vt[0].view(B, D, TP)[:, :, T:] == NAN16).all()), 'V^T pad columns written'

    def heads(p, off):   # [nc, T, 2D] plane -> [nc H, T, 64] at column offset off
        return p.view(B, T, 2 * D)[c][:, :, off:off + D].reshape(nc, T, H, 64).transpose(1, 2).reshape(nc * H, T, 64)
    qv = tuple(heads(p, 0) for p in qk[:2])
    kv = tuple(heads(p, D) for p in qk[:2])
    Sv = S.view(B, H, T, TP)[c][:, :, :, :T].reshape(nc * H, T, T)
    chk.gemm('scores GEMM', where, qv, kv, Sv, alpha=0.125)
    Pf = P[2].view(B, H, T, TP)[c][:, :, :, :T]
    chk.softmax('row softmax', where, Sv.reshape(nc, H, T, T), Pf)
    chk.split('row softmax', where, Pf, P[0].view(B, H, T, TP)[c][:, :, :, :T], P[1].view(B, H, T, TP)[c][:, :, :, :T])
    pv = tuple(p.view(B, H, T, TP)[c][:, :, :, :T].reshape(nc * H, T, T) for p in P[:2])
    vv = tuple(p.view(B, D, TP)[c][:, :, :T].reshape(nc * H, 64, T) for p in vt[:2])
    of = o[2].view(B, T, H, 64)[c].transpose(1, 2).reshape(nc * H, T, 64)
    chk.gemm('P.V GEMM', where, pv, vv, of)
    chk.split('P.V GEMM', where, o[2].view(B * T, D)[tr], o[0].view(B * T, D)[tr], o[1].view(B * T, D)[tr])


def _check_a3(chk, where, tn, s0, m, sel, attn, Pa, ft, xa, xn, logits, B, D, Vpad):
    """the A^3 module and head of the checked crops against fp64"""
    c = chk.crops
    nc = len(c)
    Dg = D // 8
    tr = chk.rows(T)

    def groups(p):       # [R, D] plane -> [nc, G, T, Dg]
        return p.view(B, T, G, Dg)[c].transpose(1, 2)
    w0 = tuple(p.view(G, Dg, Dg)[None] for p in (m['w0'].hi, m['w0'].lo))
    s0f = s0[2].view(B, T, G, Dg)[c].transpose(1, 2)
    chk.gemm('A3 grouped conv GEMM', where, tuple(groups(p) for p in tn), w0, s0f)
    chk.split('A3 grouped conv GEMM', where, s0[2].view(B * T, D)[tr], s0[0].view(B * T, D)[tr],
              s0[1].view(B * T, D)[tr])
    selv = sel.view(B, NTOK, TP)[c][:, :, :T]
    chk.gemm('A3 select GEMM', where, (m['w1'].hi[None], m['w1'].lo[None]), tuple(p.view(B, T, D)[c] for p in s0[:2]),
             selv)
    av = attn.view(B, NTOK, TP)[c][:, :, :T]
    chk.softmax('A3 row softmax', where, selv, av)
    chk.split('A3 row softmax', where, av, Pa[0].view(B, NTOK, TP)[c][:, :, :T], Pa[1].view(B, NTOK, TP)[c][:, :, :T])
    for buf, fill in ((attn, NAN_F32), (sel, NAN_F32)):
        assert bool((buf.view(B, NTOK, TP)[:, :, T:].view(torch.int32) == fill).all()), 'A3 map pad columns written'
    wf = tuple(p.view(G, Dg, Dg)[None] for p in (m['feat'].hi, m['feat'].lo))
    ftf = ft[2].view(B, G, Dg, TP)[c][..., :T]
    chk.gemm('A3 feat GEMM', where, wf, tuple(groups(p) for p in tn), ftf)
    chk.split('A3 feat GEMM', where, ftf, ft[0].view(B, G, Dg, TP)[c][..., :T], ft[1].view(B, G, Dg, TP)[c][..., :T])
    assert bool((ft[0].view(B, D, TP)[:, :, T:] == NAN16).all()), 'feat^T pad columns written'
    chk.gemm('A3 x_a GEMM', where, tuple(p.view(B, NTOK, TP)[c][:, :, :T] for p in Pa),
             tuple(p.view(B, D, TP)[c][:, :, :T] for p in ft[:2]), xa.view(B, NTOK, D)[c])
    hd = m['head']
    ar = chk.rows(NTOK)
    chk.gemm('head GEMM', where, tuple(p.view(B * NTOK, D)[ar][None] for p in xn), (hd.hi[None], hd.lo[None]),
             logits.view(B * NTOK, Vpad)[ar][:, :hd.N][None], bias=hd.b)


# ----------------------------------------------------------------------------------------------- the model
def _forward(m, img):
    """MGPSTRB200.forward(is_eval=True) and recognize_topk(K_TOP) -> (dict of device tensors, launches of the forward).
    A batch of another size runs first, so that the workspace holds its activations where this batch's buffers go: a
    forward that read anything it did not write in this call (the A^3 pad columns, a dropped lo plane) would read
    finite garbage rather than a fresh allocation's zeros."""
    ctx = m.ctx
    m.recognize(_image(img.shape[0] + 3, seed=1))
    ctx.launch_count(reset=True)
    res = m.forward(img, is_eval=True)
    launches = ctx.launch_count(reset=True)
    ids, probs = m.last_ids.clone(), m.last_prob.clone()
    ids_k, probs_k = m.recognize_topk(img, K_TOP)
    assert ctx.launch_count(reset=True) == launches, 'recognize_topk launches what the forward launches'
    n = len(res[0])
    return dict(attn=list(res[0]), logits=[t for t in res[1:1 + n]], ids=list(ids[:n]), probs=list(probs[:n]),
                ids_k=list(ids_k[:n]), probs_k=list(probs_k[:n])), launches


def _assert_same_bits(got, want, label):
    for key in ('attn', 'logits', 'ids', 'probs', 'ids_k', 'probs_k'):
        assert len(got[key]) == len(want[key]), (label, key)
        for a, (g, w) in enumerate(zip(got[key], want[key])):
            w = w.cuda()
            assert g.shape == w.shape, (label, key, a)
            gb = g.contiguous().view(torch.int32)
            wb = w.contiguous().view(torch.int32)
            if not torch.equal(gb, wb):
                diff = (gb != wb)
                first = [int(i) for i in diff.nonzero()[0]]
                raise AssertionError(f'{label}: {key} of head {a} differs from the model in {int(diff.sum())} of '
                                     f'{diff.numel()} elements, first at {first}: replay {float(g[tuple(first)])!r}, '
                                     f'model {float(w[tuple(first)])!r}')


CASES = ['depth1', 'depth2', 'base-B1', 'base-B3', 'base-B512', 'tiny', 'small', 'large', 'charstr']
RUNS = [(3, 0), (3, 1), (1, 0), (1, 1)]   # (nsplit, attn_impl)


@pytest.mark.parametrize('case,ns,impl', [(c, ns, impl) for c in CASES for ns, impl in RUNS])
def test_replay_is_the_forward_bit_for_bit(case, ns, impl):
    """The replay in the model's op order gives the forward's maps, logits, ids and probabilities bit for bit, launches
    what the forward launches but its two index / cls kernels, and every op of it is within its fp64 bound on the
    checked crops."""
    m, w, B, crops = _model(case)
    ctx = m.ctx
    img = _image(B, seed=len(case) * 100 + B)
    label = f'{case} nsplit {ns} attn_impl {impl}'
    with options(ctx, nsplit=ns, attn_impl=impl):
        want, launches = _forward(m, img)
        chk = _Checker(ns, crops if crops is not None else list(range(B)), label)
        ctx.launch_count(reset=True)
        got = _replay(ctx, w, img, ns, impl, chk)
        replayed = ctx.launch_count(reset=True) - got['extra_launches']
        # the forward's own index maps (mgp_patch_maps_kernel) and cls rows (mgp_cls_kernel) are built in torch here
        assert replayed == launches - 2, (label, replayed, launches)
        _assert_same_bits(got, want, label)
        chk.report()
        # the selection of the checked rows against the exact rule and the fp32 softmax bound
        rows = chk.rows(NTOK)
        for a, lg in enumerate(got['logits']):
            V = lg.shape[-1]
            Vpad = (V + 7) // 8 * 8
            sel = torch.full((len(rows), Vpad), float('nan'), device='cuda')
            sel[:, :V] = lg.reshape(-1, V)[rows]
            _check_select(ctx, sel, V)


def test_single_pass_forward_leaves_the_context_splitting():
    """On one context: the forward at nsplit 1 (which drops every lo plane inside it), then the replay and the forward
    at nsplit 3.  The replay runs through the same context, so a single-pass flag left set after the forward would
    drop the lo planes of the replay's producers, and its nsplit 3 consumers would read NaN.  Both runs in the model's
    own output forms (no fp32 twins)."""
    m, w, B, _ = _model('base-B3')
    ctx = m.ctx
    img = _image(B, seed=11)
    with options(ctx, nsplit=1, attn_impl=0):
        single, _ = _forward(m, img)
        got1 = _replay(ctx, w, img, 1, 0)
        _assert_same_bits(got1, single, 'nsplit 1, model form')
    with options(ctx, nsplit=3, attn_impl=0):
        got3 = _replay(ctx, w, img, 3, 0)
        split, _ = _forward(m, img)
        _assert_same_bits(got3, split, 'nsplit 3 after a forward at nsplit 1')
        assert not torch.equal(got3['logits'][0], got1['logits'][0]), 'nsplit 3 and 1 must differ'
