"""GPU: OmniParser's encoder replayed op by op through the op-level entry points, bit for bit against the model.

Every kernel the encoder runs is held to fp64 on its own, on random operands (test_gpu_encoder_ops.py and the
test_gpu_gemm_*.py files).  The end-to-end tests compare whole stage outputs norm-wise, which lets through a fault that
touches few elements: one block's GEMM handed the wrong plane, the wrong window map or LayerNorm eps in one block, a
scatter that misses the pad rows of odd grids, a page's memory rows in another page's slot.  Here encode_group
(csrc/omni.cu) is rebuilt from those entry points alone, in its order -- alm_op_patch_im2col, alm_op_gemm_planes,
alm_op_gather_ln, alm_op_swin_map, alm_op_window_attention_planes, alm_op_fpn_assemble and alm_op_sine_pos -- and the
kernels are deterministic, so alm_omni_get_feature(0..3), alm_omni_get_memory(0) and (1) must equal the replay's stage
outputs, input_proj output and position embedding bit for bit; after alm_omni_encode_pages, every page's memory and pos
rows, with +0.0 rows after each page's mh * mw and the page shapes of each page's own grid.

Only layout conventions come from the library: token-major rows, [N, Kpad] weight planes (hi = bf16_rn(w), lo =
bf16_rn(w - hi)) with the patch embedding's K padded from 48 to 64, the qkv q rows and q bias multiplied by WATTN_QSCALE
in fp32 before the split (the scale folded at load time), the FPN and merge reductions without bias.

Poisoning: every buffer of the replay holds NaN until its producer writes it and is followed by a NaN guard that must
survive.  Producers write their lo planes at every nsplit, as the encoder's do.  At nsplit 1 no GEMM is handed a lo
operand, since the engine then reads only hi planes (csrc/gemm.cu: gemm); the window attention is handed the lo plane
its qkv GEMM wrote, since both of its kernels read it at every nsplit -- the encoder's real behaviour at nsplit 1.

fp64: every op also writes its fp32 value, which is checked against fp64 of that op on the replay's own inputs with
the op tests' bounds -- GEMMs n 2^-22 sum|terms| over the products the kernel forms from its planes, gather + LayerNorm,
FPN assembly and sine position embedding as in test_gpu_encoder_ops.py, window attention _wattn_tol on the planes'
values -- and every split output must be hi = bf16_rn(x), lo = bf16_rn(x - hi).  The first and last page of each call
are checked; on the 640 x 480 page only the windows of the first and last window row and column and the tokens within 7
of the grid's border.  The worst err / bound of every op kind is printed.
"""
import ctypes

import pytest
import torch

from tests.support import options
from tests.test_gpu_encoder_ops import _fpn_err_tol, _joined, _stage_grids, _wattn_tol
from tests.test_gpu_mgp_replay import _Checker, _epi, _Lin, _opd, _Pool
from tests.test_gpu_omniparser import window_attention_ref64

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

DEPTHS, HEADS = (2, 2, 18, 2), (4, 8, 16, 32)
WATTN_QSCALE = 0.17677669529663687      # 32^-0.5 in fp32 (swin_transformer.py:130)
EPS = 1e-5                              # every LayerNorm of the encoder
SINE_TOL = 3e-6                         # test_sine_pos_matches_oracle's bound
WSEED, EOS_BIAS = 0, -30.0              # the checkpoint of the 'masked' fixture case


# ----------------------------------------------------------------------------------------------- weights
class _Weights:
    def __init__(self, sd):
        bb = 'backbone.0.'
        dev = lambda k: sd[k].float().cuda().contiguous()
        ln = lambda p: (dev(p + '.weight'), dev(p + '.bias'))
        lin = lambda p, bias=True, **kw: _Lin(sd[p + '.weight'], sd[p + '.bias'] if bias else None, **kw)
        qs = torch.tensor(WATTN_QSCALE, dtype=torch.float32)
        self.patch = lin(bb + 'patch_embed.proj', Kpad=64)
        self.patch_norm = ln(bb + 'patch_embed.norm')
        self.stages = []
        for s in range(4):
            C = 128 << s
            blocks = []
            for b in range(DEPTHS[s]):
                p = f'{bb}layers.{s}.blocks.{b}.'
                wq, bq = sd[p + 'attn.qkv.weight'].float().clone(), sd[p + 'attn.qkv.bias'].float().clone()
                wq[:C] *= qs
                bq[:C] *= qs
                blocks.append(dict(n1=ln(p + 'norm1'), n2=ln(p + 'norm2'), qkv=_Lin(wq, bq), proj=lin(p + 'attn.proj'),
                                   fc1=lin(p + 'mlp.fc1'), fc2=lin(p + 'mlp.fc2'),
                                   tab=dev(p + 'attn.relative_position_bias_table')))
            st = dict(blocks=blocks, out_norm=ln(f'{bb}norm{s}'))
            if s < 3:
                st['merge_norm'] = ln(f'{bb}layers.{s}.downsample.norm')
                st['merge_red'] = lin(f'{bb}layers.{s}.downsample.reduction', bias=False)
            self.stages.append(st)
        self.fpn = [lin(f'fpn.fpn_in.{i}', bias=False) for i in range(4)]   # fpn_in.0 reads stage 3
        self.inproj = lin('input_proj')


_MODEL = {}


def _model():
    """(OmniParserB200, _Weights): one resident model for the module"""
    if not _MODEL:
        from advancedliteratemachinery_b200 import OmniParserB200, OmniVocab
        from tests.conftest import omni_sd
        sd = omni_sd(WSEED, EOS_BIAS)
        _MODEL['m'] = (OmniParserB200(sd, OmniVocab(), workspace_mb=8192), _Weights(sd))
    return _MODEL['m']


WORST = {}


@pytest.fixture(scope='module', autouse=True)
def _close_model():
    yield
    if _MODEL:
        _MODEL.pop('m')[0].ctx.close()
        torch.cuda.empty_cache()
    for kind, r in sorted(WORST.items()):
        print(f'[omni replay] {kind}: worst err / bound over the module {r:.3g}')


# ----------------------------------------------------------------------------------------------- fp64 checks
class _EncChecker(_Checker):
    """the MGP replay's checker over the rows of the checked pages (border: only near the grid's edges)"""

    def __init__(self, ns, label, border):
        super().__init__(ns, [0], label)
        self.border = border
        self.pages = [0]

    def _record(self, kind, where, err, bound):
        super()._record(kind, where, err, bound)
        WORST[kind] = max(WORST.get(kind, 0.0), self.worst[(kind, where)])

    def split(self, kind, where, f32, hi, lo):
        """the encoder's producers write both planes at every nsplit"""
        ns, self.ns = self.ns, 3
        try:
            super().split(kind, where, f32, hi, lo)
        finally:
            self.ns = ns

    def _edge(self, H, W, band):
        y, x = torch.meshgrid(torch.arange(H, device='cuda'), torch.arange(W, device='cuda'), indexing='ij')
        keep = (y < band) | (y >= H - band) | (x < band) | (x >= W - band) if self.border else torch.ones_like(y).bool()
        return (y * W + x)[keep]

    def tok_rows(self, H, W):
        """token rows b (H W) + y W + x of the checked pages"""
        local = self._edge(H, W, 7)
        return torch.cat([b * H * W + local for b in self.pages])

    def win_local(self, nWh, nWw):
        """window rows w 49 + t within one page, of the checked windows"""
        w = self._edge(nWh, nWw, 1)
        return (w[:, None] * 49 + torch.arange(49, device='cuda')).flatten()

    def win_rows(self, nWh, nWw):
        local = self.win_local(nWh, nWw)
        return torch.cat([b * nWh * nWw * 49 + local for b in self.pages])


def _bits(t):
    return t.contiguous().view(torch.int32)


# ----------------------------------------------------------------------------------------------- the replay
class _Replay:
    """encode_group from op entry points under the context's nsplit (ns), every op checked by chk"""

    def __init__(self, ctx, w, ns, chk):
        self.ctx, self.w, self.ns, self.chk = ctx, w, ns, chk

    def call(self, name, *args):
        torch.cuda.synchronize()    # the context runs on its own stream
        self.ctx.check(getattr(self.ctx.lib, name)(self.ctx.h, *args))

    def lo(self, t):
        return t if self.ns == 3 else None

    def linear(self, pool, a, rows, l, kind, where, sel, out=None, act=0, resid=None, out_map=None, resid_map=None):
        """rows of the planes a times l^T (+ bias, GELU): to new split planes -> (hi, lo), or (out) to fp32 rows of out,
        through out_map / resid_map, plus resid.  sel: the checked rows of a."""
        chk, N = self.chk, l.N
        s = sel
        orow = s if out_map is None else out_map.long()[s]
        s, orow = s[orow >= 0], orow[orow >= 0]
        rrow = orow if resid_map is None else resid_map.long()[s]
        before = None if resid is None else resid.view(-1, N)[rrow]       # a copy: resid may be out (in place)
        if out is None:
            hi, lo = pool.planes(rows * N)
            f = pool.f32(rows * N)
            e = _epi(f, hi, lo, ldo=N, bias=l.b, bias_mode=1, act=act)
        else:
            e = _epi(out, ldo=N, bias=l.b, bias_mode=1, resid=resid, ldr=N if resid is not None else 0,
                     out_map=out_map, resid_map=resid_map, act=act)
        a_op = _opd(a[0], self.lo(a[1]), rows, l.K, l.K)
        w_op = _opd(l.hi, self.lo(l.lo), l.N, l.K, l.K)
        torch.cuda.synchronize()
        self.ctx.check(self.ctx.lib.alm_op_gemm_planes(self.ctx.h, ctypes.byref(a_op), ctypes.byref(w_op),
                                                       ctypes.byref(e)))
        got = (f if out is None else out).view(-1, N)[orow]
        chk.gemm(kind, where, tuple(p.view(rows, l.K)[s][None] for p in a), (l.hi[None], l.lo[None]), got[None],
                 bias=l.b, act=act, resid=None if before is None else before[None])
        if out is None:
            chk.split(kind, where, got, hi.view(rows, N)[orow], lo.view(rows, N)[orow])
            return hi, lo
        return None

    def layernorm(self, pool, src, Cs, rows, gb, kind, where, sel, map_=None, nsrc=1, zero_missing=0, f32=None,
                  split=True):
        """alm_op_gather_ln of rows of src (width Cs) -> (hi, lo) or None; f32: the fp32 output, else a twin"""
        chk, C = self.chk, nsrc * Cs
        hi, lo = pool.planes(rows * C) if split else (None, None)
        f = f32 if f32 is not None else pool.f32(rows * C)
        self.call('alm_op_gather_ln', src.data_ptr(), Cs, None if map_ is None else map_.data_ptr(), nsrc, Cs, rows,
                  gb[0].data_ptr(), gb[1].data_ptr(), EPS, zero_missing, None, 0, f.data_ptr(), C,
                  None if hi is None else hi.data_ptr(), None if lo is None else lo.data_ptr(), C, None, None, None)
        srows = src.view(-1, Cs)
        if map_ is None:
            xin = srows[sel]
            dead = torch.zeros(len(sel), dtype=torch.bool, device='cuda')
        else:
            m = map_.long().view(rows, nsrc)[sel]
            xin = torch.where((m >= 0)[..., None], srows[m.clamp(min=0)], 0.0).reshape(len(sel), C)
            dead = (m < 0).all(-1) if zero_missing else torch.zeros(len(sel), dtype=torch.bool, device='cuda')
        fv = f.view(rows, C)[sel]
        chk.ln(kind, where, xin[~dead], gb[0], gb[1], EPS, fv[~dead])
        assert not bool(_bits(fv[dead]).any()), f'{chk.label} {kind} ({where}): a pad row is not +0'
        if split:
            chk.split(kind, where, fv, hi.view(rows, C)[sel], lo.view(rows, C)[sel])
            return hi, lo
        return None

    def encode_group(self, img, n_canvas, Hc, Wc, slots, B, H, W, memory, mem_map):
        """one size group of B pages H x W, canvas slots `slots` (int32 device or None) of img [n_canvas, 3, Hc, Wc];
        input_proj rows to memory through mem_map (None: in order) -> the four stage outputs (fp32 token rows)"""
        w, chk = self.w, self.chk
        chk.pages = sorted({0, B - 1})
        grids = _stage_grids(H, W)
        top = _Pool()
        # ---- patch embed: im2col -> GEMM (+bias) -> LayerNorm
        pool = _Pool()
        H0, W0 = grids[0]
        rows = B * H0 * W0
        a = pool.planes(rows * 64)
        self.call('alm_op_patch_im2col', img.data_ptr(), n_canvas, Hc, Wc, None if slots is None else slots.data_ptr(),
                  B, H, W, a[0].data_ptr(), a[1].data_ptr())
        tr = chk.tok_rows(H0, W0)
        self._check_im2col(img, slots, H, W, a)
        tmp = pool.f32(rows * 128)
        self.linear(pool, a, rows, w.patch, 'patch GEMM', 'patch embed', tr, out=tmp)
        x = top.f32(rows * 128)
        self.layernorm(pool, tmp, 128, rows, w.patch_norm, 'LayerNorm', 'patch embed', tr, f32=x, split=False)
        pool.done()

        feats, feat_split = [], []
        for s in range(4):
            C, heads = 128 << s, HEADS[s]
            Hs, Ws = grids[s]
            nWh, nWw = -(-Hs // 7), -(-Ws // 7)
            rowsP, rows = B * nWh * nWw * 49, B * Hs * Ws
            tr, wr = chk.tok_rows(Hs, Ws), chk.win_rows(nWh, nWw)
            pool = _Pool()
            maps = []
            for shift in (0, 3):
                mp = pool.i32(rowsP)
                self.call('alm_op_swin_map', 0, B, Hs, Ws, shift, mp.data_ptr())
                maps.append(mp)
            for bi, blk in enumerate(w.stages[s]['blocks']):
                where = f'stage {s} block {bi}'
                shift = 3 if bi & 1 else 0
                mp = maps[bi & 1]
                ln = self.layernorm(pool, x, C, rowsP, blk['n1'], 'LayerNorm', where, wr, map_=mp, zero_missing=1)
                qkv = self.linear(pool, ln, rowsP, blk['qkv'], 'qkv GEMM', where, wr)
                att = self.window_attention(pool, qkv, blk['tab'], B, nWh, nWw, C, heads, shift, where)
                self.linear(pool, att, rowsP, blk['proj'], 'proj GEMM + residual', where, wr, out=x, resid=x,
                            out_map=mp)
                ln = self.layernorm(pool, x, C, rows, blk['n2'], 'LayerNorm', where, tr)
                hid = self.linear(pool, ln, rows, blk['fc1'], 'fc1 GEMM + GELU', where, tr, act=1)
                self.linear(pool, hid, rows, blk['fc2'], 'fc2 GEMM + residual', where, tr, out=x, resid=x)
            pool.done()
            # the stage's output norm: the fp32 feature and the FPN's split operand
            feat = top.f32(rows * C)
            feat_split.append(self.layernorm(top, x, C, rows, w.stages[s]['out_norm'], 'LayerNorm', f'stage {s} out',
                                             tr, f32=feat))
            feats.append(feat)
            if s < 3:   # PatchMerging: 2 x 2 gather -> LayerNorm(4C) -> reduction 4C -> 2C
                H2, W2 = grids[s + 1]
                rows2 = B * H2 * W2
                tr2 = chk.tok_rows(H2, W2)
                pool = _Pool()
                mm = pool.i32(rows2 * 4)
                self.call('alm_op_swin_map', 1, B, Hs, Ws, 0, mm.data_ptr())
                ma = self.layernorm(pool, x, C, rows2, w.stages[s]['merge_norm'], 'LayerNorm', f'merge {s}', tr2,
                                    map_=mm, nsrc=4)
                x = top.f32(rows2 * 2 * C)
                self.linear(pool, ma, rows2, w.stages[s]['merge_red'], 'merge GEMM', f'merge {s}', tr2, out=x)
                pool.done()

        # ---- FPN from p5 down: p_s = c_s' + nearest(p_{s+1}), fp32
        p = [None] * 4
        for s in range(3, -1, -1):
            Hs, Ws = grids[s]
            rows = B * Hs * Ws
            p[s] = top.f32(rows * 256)
            tr = chk.tok_rows(Hs, Ws)
            if s == 3:
                self.linear(top, feat_split[s], rows, w.fpn[3 - s], 'FPN GEMM', 'p5', tr, out=p[s])
            else:
                up = top.i32(rows)
                self.call('alm_op_swin_map', 2, B, Hs, Ws, 0, up.data_ptr())
                self.linear(top, feat_split[s], rows, w.fpn[3 - s], 'FPN GEMM', f'p{s + 2}', tr, out=p[s],
                            resid=p[s + 1], resid_map=up)
        # ---- the stride-2 concat and input_proj, scattered to the memory rows
        mh, mw = grids[2]
        BM = B * mh * mw
        cat = top.planes(BM * 1024)
        self.call('alm_op_fpn_assemble', *[t.data_ptr() for t in p], B, H, W, cat[0].data_ptr(), cat[1].data_ptr())
        pg = chk.pages
        levels = [p[s].view(B, *grids[s], 256)[pg] for s in range(4)]
        sub = [t.view(B, mh * mw * 1024)[pg].flatten() for t in cat]
        for err, tol in _fpn_err_tol(sub[0], sub[1], levels, grids):    # p3's columns: its exact split
            chk._record('FPN assembly', 'fpn', err, tol)
        mr = torch.cat([b * mh * mw + torch.arange(mh * mw, device='cuda') for b in pg])
        self.linear(top, cat, BM, w.inproj, 'input_proj GEMM', 'memory', mr, out=memory, out_map=mem_map)
        top.done()
        return feats

    def window_attention(self, pool, qkv, tab, B, nWh, nWw, C, heads, shift, where):
        chk = self.chk
        rowsP = B * nWh * nWw * 49
        hi, lo = pool.planes(rowsP * C)
        f = pool.f32(rowsP * C)
        self.call('alm_op_window_attention_planes', qkv[0].data_ptr(), qkv[1].data_ptr(), tab.data_ptr(), f.data_ptr(),
                  hi.data_ptr(), lo.data_ptr(), B, nWh, nWw, C, heads, shift)
        per = nWh * nWw * 49
        local = chk.win_local(nWh, nWw)
        for b in chk.pages:
            r = slice(b * per, (b + 1) * per)
            q = _joined(qkv[0].view(rowsP, 3 * C)[r], qkv[1].view(rowsP, 3 * C)[r])
            ref = window_attention_ref64(q, tab, 1, nWh, nWw, heads, shift, scale=1.0)[local]
            tol = _wattn_tol(q, heads, 1, nWh, nWw, scale=1.0)[local]
            got = f.view(rowsP, C)[r][local]
            chk._record('window attention', where, (got.double() - ref).abs(), tol)
            chk.split('window attention', where, got, hi.view(rowsP, C)[r][local], lo.view(rowsP, C)[r][local])
        return hi, lo

    def _check_im2col(self, img, slots, H, W, a):
        """the patch rows of the checked pages: the exact split of the zero-padded 4 x 4 patches, K 48 padded to 64"""
        from oracle import omniparser_ref as O
        pg = self.chk.pages
        idx = slots.long()[pg] if slots is not None else torch.tensor(pg, device='cuda')
        Hp, Wp = -(-H // 4), -(-W // 4)
        pad = O.patch_pad(img[idx][:, :, :H, :W])
        ref = pad.reshape(len(pg), 3, Hp, 4, Wp, 4).permute(0, 2, 4, 1, 3, 5).reshape(-1, 48)
        ref = torch.cat([ref, torch.zeros(ref.shape[0], 16, device='cuda')], 1)
        rows = torch.cat([b * Hp * Wp + torch.arange(Hp * Wp, device='cuda') for b in pg])
        self.chk.split('im2col', 'patches', ref, a[0].view(-1, 64)[rows], a[1].view(-1, 64)[rows])

    def sine_pos(self, mask, B, H, W, mh, mw, pos, where):
        """alm_op_sine_pos into pos [B mh mw, 512] against the oracle"""
        from oracle import omniparser_ref as O
        kpm = torch.full((B * mh * mw + 256,), 7, dtype=torch.uint8, device='cuda')
        self.call('alm_op_sine_pos', None if mask is None else mask.data_ptr(), B, H, W, mh, mw, pos.data_ptr(),
                  kpm.data_ptr())
        assert bool((kpm[B * mh * mw:] == 7).all()), 'kpm written past its end'
        m = torch.zeros(B, H, W, dtype=torch.bool) if mask is None else mask.bool().cpu()
        lm = O.level_mask(m, (mh, mw))
        ref = O.position_embedding_sine(lm).reshape(-1, 512).double()
        assert torch.equal(kpm[:B * mh * mw].cpu(), lm.flatten().to(torch.uint8))
        err = (pos.view(-1, 512).cpu().double() - ref).abs()
        self.chk._record('sine position', where, err, torch.full_like(err, SINE_TOL))


# ----------------------------------------------------------------------------------------------- cases
def _canvas(B, Hc, Wc, sizes, seed):
    """pages of random pixels at the top left of each slot, NaN elsewhere (nothing outside a page may be read)"""
    g = torch.Generator().manual_seed(seed)
    img = torch.full((B, 3, Hc, Wc), float('nan'))
    for b, (h, w) in enumerate(sizes):
        img[b, :, :h, :w] = torch.randn(3, h, w, generator=g)
    return img.cuda()


def _case(name):
    """-> (img, mask or None, page sizes or None): alm_omni_encode(img, mask) or alm_omni_encode_pages(img, sizes)"""
    if name == 'odd':
        return _canvas(2, 100, 164, [(100, 164)] * 2, 1), None, None
    if name == 'masked':
        from oracle.gen_golden import OMNI_CASES, omni_inputs
        img, mask = omni_inputs(OMNI_CASES['masked'])
        return img.cuda(), mask.cuda(), None
    if name == 'page':
        return _canvas(1, 640, 480, [(640, 480)], 3), None, None
    assert name == 'mixed'
    sizes = [(96, 128), (160, 72), (96, 128)]
    return _canvas(3, 160, 128, sizes, 4), None, sizes


def _assert_same_bits(got, want, label):
    gb, wb = _bits(got), _bits(want)
    assert gb.shape == wb.shape, (label, gb.shape, wb.shape)
    if not torch.equal(gb, wb):
        diff = gb != wb
        first = [int(i) for i in diff.nonzero()[0]]
        raise AssertionError(f'{label}: differs from the model in {int(diff.sum())} of {diff.numel()} elements, first '
                             f'at {first}: replay {float(got[tuple(first)])!r}, model {float(want[tuple(first)])!r}')


def _run_single(m, rp, img, mask, label):
    """alm_omni_encode against the replay of its one size group"""
    B, _, H, W = img.shape
    grids = _stage_grids(H, W)
    mh, mw = grids[2]
    m.encode(img, mask)
    mask8 = mask.to(torch.uint8).contiguous() if mask is not None and bool(mask.any()) else None
    top = _Pool()
    memory = top.f32(B * mh * mw * 512)
    feats = rp.encode_group(img, B, H, W, None, B, H, W, memory, None)
    for s, f in enumerate(feats):
        want = m.features(s).permute(0, 2, 3, 1).contiguous().cuda()
        _assert_same_bits(f.view(B, *grids[s], 128 << s), want, f'{label}: stage {s} feature')
    _assert_same_bits(memory.view(B, mh * mw, 512), m.memory(0).cuda(), f'{label}: memory')
    pos = top.f32(B * mh * mw * 512)
    rp.sine_pos(mask8, B, H, W, mh, mw, pos, 'memory')
    _assert_same_bits(pos.view(B, mh * mw, 512), m.memory(1).cuda(), f'{label}: pos')
    top.done()


def _run_pages(m, rp, img, sizes, label):
    """alm_omni_encode_pages against the replay of its size groups, in order of first appearance"""
    B, _, Hc, Wc = img.shape
    shapes = m.encode_pages(img, sizes)
    grid = [_stage_grids(h, w)[2] for h, w in sizes]
    assert shapes == grid, (label, shapes, grid)
    M = max(h * w for h, w in grid)
    top = _Pool()
    memory = top.f32(B * M * 512)
    pos = {}
    for size in dict.fromkeys(sizes):
        slots = [b for b in range(B) if sizes[b] == size]
        h, w = size
        mh, mw = _stage_grids(h, w)[2]
        Mg = mh * mw
        d_slots = torch.tensor(slots, dtype=torch.int32, device='cuda')
        mem_map = torch.tensor([s * M + r for s in slots for r in range(Mg)], dtype=torch.int32, device='cuda')
        rp.encode_group(img, B, Hc, Wc, d_slots, len(slots), h, w, memory, mem_map)
        pos[size] = top.f32(Mg * 512)
        rp.sine_pos(None, 1, h, w, mh, mw, pos[size], f'pos {h} x {w}')
    want_mem, want_pos = m.memory(0).cuda(), m.memory(1).cuda()
    mem = memory.view(B, M, 512)
    for b, (mh, mw) in enumerate(grid):
        Mg = mh * mw
        _assert_same_bits(mem[b, :Mg], want_mem[b, :Mg], f'{label}: memory of page {b}')
        _assert_same_bits(pos[sizes[b]].view(Mg, 512), want_pos[b, :Mg], f'{label}: pos of page {b}')
        assert bool(torch.isnan(mem[b, Mg:]).all()), f'{label}: the replay wrote memory rows past page {b}\'s keys'
        for t, what in ((want_mem, 'memory'), (want_pos, 'pos')):
            assert not bool(_bits(t[b, Mg:]).any()), f'{label}: {what} rows past page {b}\'s keys are not +0.0'
    top.done()


CASES = ['odd', 'masked', 'page', 'mixed']
RUNS = [(c, ns, 3) for c in CASES for ns in (3, 1)] + [(c, ns, 0) for c in ('odd', 'mixed') for ns in (3, 1)]


@pytest.mark.parametrize('case,ns,impl', RUNS)
def test_replay_is_the_encoder_bit_for_bit(case, ns, impl):
    """The replay in encode_group's op order gives the model's stage features, memory and position embedding bit for
    bit, and every op of it is within its fp64 bound on the checked rows."""
    m, w = _model()
    ctx = m.ctx
    img, mask, sizes = _case(case)
    label = f'{case} nsplit {ns} wattn_impl {impl}'
    chk = _EncChecker(ns, label, border=case == 'page')
    with options(ctx, nsplit=ns, wattn_impl=impl):
        rp = _Replay(ctx, w, ns, chk)
        if sizes is None:
            _run_single(m, rp, img, mask, label)
        else:
            _run_pages(m, rp, img, sizes, label)
        chk.report()
