"""GPU: the encoder's non-GEMM kernels against plain fp64 and exact references, through their op-level entry points.

Every page and every MGP-STR crop runs through these kernels (kernels.cu, the top of omni_kernels.cu, wattn_ms.cu).  The
end-to-end tests compare whole stage outputs with a norm-wise tolerance, which can hide a wrong edge window, pad row or
interpolation tap.  Here each kernel is compared element by element with the same operation restated from the oracle
(oracle/omniparser_ref.py), at the shapes the benchmark's pages produce and at the edges of its index arithmetic:

* the window / merge / nearest row maps, exactly, on grids of every residue mod 7 and mod 2 and the stage grids of real
  pages;
* gather + LayerNorm + split through those maps at the Swin widths, zero pad rows, the memory + pos form, the 192-wide
  ViT instantiation, rows with a large mean, and source rows wider than the gathered width;
* the patch im2col with canvas slots, odd sizes and unaligned rows; the FPN assembly with bilinear taps at both
  borders; the sine position embedding with masks up to the shared-memory bound; the row softmax with masks;
* the Swin window-attention core with sharp scores and the shift mask, at every head count and across the persistent
  kernel's schedule, on fp32 qkv and on the encoder's own operand: the split planes of a q already scaled by 32^-0.5.

Every output buffer is followed by a guard region that must come back bit for bit unchanged, and input memory the call
must not read holds NaN.  Wherever a kernel writes a split pair it must be hi = bf16_rn(x), lo = bf16_rn(x - hi) of the
fp32 value it writes (or would write).  Shapes that depend on the schedule are derived from the SM count.
"""
import pytest
import torch
import torch.nn.functional as F

from tests.support import NAN, assert_guard, bits, ctx, guarded, options, sms

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

WORKSPACE_MB = 4096
ERR_INVALID, ERR_UNSUPPORTED = -1, -5
U32 = 2.0 ** -24        # fp32 unit roundoff


def _ptr(t):
    return None if t is None else t.data_ptr()


def _op(ctx, name, *args):
    """Call an entry point once torch's queued work is done (the context runs on its own stream and synchronizes it
    before returning)."""
    torch.cuda.synchronize()
    return getattr(ctx.lib, name)(ctx.h, *args)


def _planes(n):
    """a bf16 (hi, lo) output pair as int16 bit buffers prefilled with 0xffff (a NaN), each with a guard"""
    return guarded(n, torch.int16, -1), guarded(n, torch.int16, -1)


def _assert_split(hi, lo, x, what=''):
    """hi == bf16_rn(x) and lo == bf16_rn(x - hi), bit for bit (hi, lo int16 bit views; x fp32)"""
    h = x.float().to(torch.bfloat16)
    assert torch.equal(hi, h.view(torch.int16)), ('hi', what)
    assert torch.equal(lo, (x.float() - h.float()).to(torch.bfloat16).view(torch.int16)), ('lo', what)


def _joined(hi, lo):
    return hi.view(torch.bfloat16).double() + lo.view(torch.bfloat16).double()


def _nan_rows(rows, ld, C, extra=3):
    """fp32 [rows, ld] device matrix (a view of a buffer with `extra` more rows) whose columns C..ld-1 and the rows past
    the end hold NaN; the caller fills [:, :C]"""
    buf = torch.full(((rows + extra) * ld,), NAN, device='cuda')
    return buf[:rows * ld].view(rows, ld)


def _stage_grids(H, W):
    """token grids of the four Swin stages of an H x W page (the encoder's stage_grid)"""
    hs, ws, out = -(-H // 4), -(-W // 4), []
    for _ in range(4):
        out.append((hs, ws))
        hs, ws = (hs + 1) // 2, (ws + 1) // 2
    return out


PAGES = {'config2': (1024, 1024), 'config5': (1920, 1920), 'odd': (108, 76)}


# ----------------------------------------------------------------------------------------------- row maps
def _index(B, H, W):
    return torch.arange(B * H * W, dtype=torch.int64).view(B, H, W, 1)


def _window_map_ref(B, H, W, shift):
    """LN1 -> zero pad -> roll -> window partition (swin_transformer.py:213-229) applied to row indices (-1 = pad)"""
    from oracle import omniparser_ref as O
    x = F.pad(_index(B, H, W), (0, 0, 0, (7 - W % 7) % 7, 0, (7 - H % 7) % 7), value=-1)
    if shift:
        x = torch.roll(x, shifts=(-shift, -shift), dims=(1, 2))
    return O.window_partition(x).flatten()


def _merge_map_ref(B, H, W):
    from oracle import omniparser_ref as O
    return O.merge_concat(_index(B, H, W), value=-1).flatten()


def _nearest_map_ref(B, H, W):
    """F.interpolate(mode='nearest') of the (ceil(H/2), ceil(W/2)) grid's row indices up to (H, W), in float32 like the
    oracle's FPN (indices < 2^24 are exact)"""
    Hs, Ws = (H + 1) // 2, (W + 1) // 2
    src = torch.arange(B * Hs * Ws, dtype=torch.float32).view(B, 1, Hs, Ws)
    return F.interpolate(src, size=(H, W), mode='nearest').long().flatten()


def _swin_map(ctx, kind, B, H, W, shift):
    n = {0: B * -(-H // 7) * -(-W // 7) * 49, 1: B * ((H + 1) // 2) * ((W + 1) // 2) * 4, 2: B * H * W}[kind]
    m, full = guarded(n, torch.int32, -7)
    ctx.check(_op(ctx, 'alm_op_swin_map', kind, B, H, W, shift, m.data_ptr()))
    assert_guard(full, n, -7)
    return m


def _check_maps(ctx, B, H, W):
    for shift in (0, 3):
        got = _swin_map(ctx, 0, B, H, W, shift).cpu().long()
        assert torch.equal(got, _window_map_ref(B, H, W, shift)), ('window', B, H, W, shift)
    assert torch.equal(_swin_map(ctx, 1, B, H, W, 0).cpu().long(), _merge_map_ref(B, H, W)), ('merge', B, H, W)
    assert torch.equal(_swin_map(ctx, 2, B, H, W, 0).cpu().long(), _nearest_map_ref(B, H, W)), ('nearest', B, H, W)


def test_swin_maps_small_grids(ctx):
    """every residue of H mod 7 and mod 2 against a spread of widths, grids smaller than a window, 1-wide strips, B > 1"""
    grids = [(1, 1, 1), (1, 3, 4), (1, 7, 7), (1, 1, 13), (1, 13, 1), (3, 1, 1)]
    grids += [(2, H, W) for H in range(1, 15) for W in (1, 2, 5, 7, 8, 13, 16)]
    for B, H, W in grids:
        _check_maps(ctx, B, H, W)


@pytest.mark.parametrize('page', list(PAGES))
def test_swin_maps_page_grids(ctx, page):
    for H, W in _stage_grids(*PAGES[page]):
        _check_maps(ctx, 2 if page == 'odd' else 1, H, W)


# ----------------------------------------------------------------------------------------------- gather + LayerNorm
OUTS = ('f32', 'hi', 'lo', 'hi2', 'lo2', 'f322')


def _run_gather(ctx, src, map_, nsrc, Cs, rows, gamma=None, beta=None, zero_missing=0, add=None,
                outs=OUTS, ldo_f32=None, ldo_bf=None):
    """alm_op_gather_ln on src [*, lds] -> {output name: [rows, C] tensor}; the output columns C..ld-1 must stay as
    prefilled and every guard intact"""
    C = nsrc * Cs
    ldo_f32, ldo_bf = ldo_f32 or C, ldo_bf or C
    bufs = {}
    for name in outs:
        f32 = name.startswith('f32')
        bufs[name] = guarded(rows * (ldo_f32 if f32 else ldo_bf), torch.float32 if f32 else torch.int16,
                              NAN if f32 else -1)

    def p(k):
        return bufs[k][0].data_ptr() if k in bufs else None
    ctx.check(_op(ctx, 'alm_op_gather_ln', src.data_ptr(), src.stride(0), _ptr(map_), nsrc, Cs, rows, _ptr(gamma),
                  _ptr(beta), 1e-5, zero_missing, _ptr(add), add.stride(0) if add is not None else 0, p('f32'), ldo_f32,
                  p('hi'), p('lo'), ldo_bf, p('hi2'), p('lo2'), p('f322')))
    res = {}
    for k, (buf, full) in bufs.items():
        fill = NAN if k.startswith('f32') else -1
        assert_guard(full, buf.numel(), fill)
        v = buf.view(rows, -1)
        if v.shape[1] > C:
            gap = v[:, C:]
            assert torch.equal(bits(gap), bits(torch.full_like(gap, fill))), (k, 'wrote past the row width')
        res[k] = v[:, :C].contiguous()
    return res


def _ln_tol(rows64, gamma, ref):
    """|got - ref| bound of the fp32 LayerNorm: 1e-5 absolute plus 2^-20 relative (rounding of the normalised values and
    of the fp32 variance sum), plus the rounding of the fp32 row sum.  The row sum over C values (sequential per lane,
    then a 5-level shuffle tree) is within 32 ulp of the row mean, so a row of mean m shifts every normalised value by up
    to 32 * 2^-24 * |m| * rstd * |gamma|: this is the fp32 input quantisation term, 0.002 for a mean of 1e3 and unit
    spread, against the one-pass variance's error there of order 1."""
    mean = rows64.mean(-1, keepdim=True)
    rstd = (rows64.var(-1, unbiased=False, keepdim=True) + 1e-5).rsqrt()
    return 1e-5 + 2.0 ** -20 * ref.abs() + 32 * U32 * mean.abs() * rstd * gamma.double().abs()


def _check_gather(ctx, res, ref, tol, args, kwargs, dead=None):
    """fp32 outputs against ref within tol; every split pair is the split of its fp32 twin; dead rows are +0 in every
    output; the split-only call writes the same bits"""
    f32 = res['f32']
    assert torch.isfinite(f32).all()
    err = (f32.double() - ref).abs()
    assert bool((err <= tol).all()), float((err / tol).max())
    _assert_split(res['hi'], res['lo'], f32, 'out')
    if 'f322' in res:
        _assert_split(res['hi2'], res['lo2'], res['f322'], 'out2')
    if dead is not None and bool(dead.any()):
        for k, v in res.items():
            assert not bool(bits(v[dead]).any()), (k, 'a pad row is not +0')
    split_only = _run_gather(ctx, *args, **kwargs, outs=('hi', 'lo'))
    assert torch.equal(split_only['hi'], res['hi']) and torch.equal(split_only['lo'], res['lo'])


def _src(rows, C, gen, scale=3.0, shift=1.0, pad=4):
    """rows x C values in a [rows, C + pad] matrix: NaN in the gap columns and in rows past the end"""
    x = _nan_rows(rows, C + pad, C)
    x[:, :C] = torch.randn(rows, C, generator=gen, device='cuda') * scale + shift
    return x


def _affine(C, gen):
    return torch.randn(C, generator=gen, device='cuda'), torch.randn(C, generator=gen, device='cuda')


# Swin stage widths 128 .. 1024 through the window partition, grids whose residues mod 7 leave pad rows
@pytest.mark.parametrize('shift', [0, 3])
@pytest.mark.parametrize('C,grid', [(128, (2, 23, 30)), (256, (1, 13, 19)), (512, (2, 9, 8)), (1024, (1, 4, 5))])
def test_gather_ln_window_partition(ctx, C, grid, shift):
    from oracle import omniparser_ref as O
    B, H, W = grid
    gen = torch.Generator(device='cuda').manual_seed(C + shift)
    x = _src(B * H * W, C, gen)
    g, b = _affine(C, gen)
    wmap = _swin_map(ctx, 0, B, H, W, shift)
    rows = wmap.numel()
    args = (x, wmap, 1, C, rows)
    kw = dict(gamma=g, beta=b, zero_missing=1)
    res = _run_gather(ctx, *args, **kw)
    x64 = x[:, :C].double()
    ln = F.layer_norm(x64, (C,), g.double(), b.double(), 1e-5).view(B, H, W, C)
    ln = F.pad(ln, (0, 0, 0, (7 - W % 7) % 7, 0, (7 - H % 7) % 7))
    if shift:
        ln = torch.roll(ln, shifts=(-shift, -shift), dims=(1, 2))
    ref = O.window_partition(ln).reshape(rows, C)
    dead = (wmap < 0).bool()
    gathered = torch.where(dead[:, None], torch.zeros_like(ref), x64[wmap.long().clamp(min=0)])
    tol = _ln_tol(gathered, g, ref)
    assert int(dead.sum()) == rows - B * H * W
    _check_gather(ctx, res, ref, tol, args, kw, dead)


# PatchMerging's 2 x 2 concat: 4C = 512, 1024, 2048, odd grids (the missing half of a pair is a zero in the LayerNorm)
@pytest.mark.parametrize('C,grid', [(128, (2, 13, 9)), (256, (1, 14, 11)), (512, (2, 7, 5))])
def test_gather_ln_patch_merge(ctx, C, grid):
    from oracle import omniparser_ref as O
    B, H, W = grid
    gen = torch.Generator(device='cuda').manual_seed(C + 1)
    x = _src(B * H * W, C, gen)
    g, b = _affine(4 * C, gen)
    mmap = _swin_map(ctx, 1, B, H, W, 0)
    rows = mmap.numel() // 4
    args = (x, mmap, 4, C, rows)
    kw = dict(gamma=g, beta=b)
    res = _run_gather(ctx, *args, **kw)
    cat = O.merge_concat(x[:, :C].double().view(B, H, W, C)).reshape(rows, 4 * C)
    ref = F.layer_norm(cat, (4 * C,), g.double(), b.double(), 1e-5)
    _check_gather(ctx, res, ref, _ln_tol(cat, g, ref), args, kw)


def test_gather_ln_memory_plus_pos(ctx):
    """the cross-attention operands: memory and memory + pos, no LayerNorm; the fp32 outputs are exact"""
    gen = torch.Generator(device='cuda').manual_seed(11)
    rows, C = 1001, 512
    mem = _src(rows, C, gen, pad=4)
    pos = _src(rows, C, gen, pad=8)
    args = (mem, None, 1, C, rows)
    kw = dict(add=pos, ldo_f32=C + 4, ldo_bf=C + 8)
    res = _run_gather(ctx, *args, **kw)
    m32, p32 = mem[:, :C], pos[:, :C]
    assert torch.equal(bits(res['f32']), bits(m32.contiguous()))
    assert torch.equal(bits(res['f322']), bits((m32 + p32).contiguous()))
    _assert_split(res['hi'], res['lo'], m32, 'memory')
    _assert_split(res['hi2'], res['lo2'], m32 + p32, 'memory + pos')
    enc = _run_gather(ctx, *args, add=pos, outs=('hi', 'lo', 'hi2', 'lo2'))   # the encoder's form: split pairs only
    for k in ('hi', 'lo', 'hi2', 'lo2'):
        assert torch.equal(enc[k], res[k]), k


@pytest.mark.parametrize('C,rows,mean', [(192, 777, 1.0), (128, 9, 1.0), (512, 300, 1e3), (1024, 300, 1e3),
                                         (2048, 300, 1e3), (192, 300, 1e3)])
def test_gather_ln_rows(ctx, C, rows, mean):
    """plain rows (map NULL): the 192-wide ViT instantiation, and rows of mean 1e3 with unit spread, where a one-pass
    variance E[x^2] - mean^2 cancels catastrophically in fp32"""
    gen = torch.Generator(device='cuda').manual_seed(C + rows)
    x = _src(rows, C, gen, scale=1.0 if mean > 1 else 3.0, shift=mean, pad=8)
    g, b = _affine(C, gen)
    args = (x, None, 1, C, rows)
    kw = dict(gamma=g, beta=b)
    res = _run_gather(ctx, *args, **kw)
    x64 = x[:, :C].double()
    ref = F.layer_norm(x64, (C,), g.double(), b.double(), 1e-5)
    _check_gather(ctx, res, ref, _ln_tol(x64, g, ref), args, kw)


# ----------------------------------------------------------------------------------------------- patch im2col
# (B, H, W, Hc, Wc, canvas slots, slot of each image or None): H, W = 1, 2, 3 mod 4 with Wc != W (rows not 16-byte
# aligned), one unused slot; MGP-STR's 32 x 128 crops at B = 512
IM2COL_CASES = {
    'r1': (3, 33, 45, 35, 47, 4, [2, 0, 3]),
    'r2': (2, 34, 47, 34, 49, 3, [1, 2]),
    'r3': (2, 35, 46, 38, 51, 3, [2, 0]),
    'mgpstr': (512, 32, 128, 32, 128, 512, None),
}


@pytest.mark.parametrize('name', list(IM2COL_CASES))
def test_patch_im2col_exact(ctx, name):
    from oracle import omniparser_ref as O
    B, H, W, Hc, Wc, n_canvas, slots = IM2COL_CASES[name]
    gen = torch.Generator(device='cuda').manual_seed(H * W)
    canvas, _ = guarded(n_canvas * 3 * Hc * Wc)
    canvas = canvas.view(n_canvas, 3, Hc, Wc)
    order = slots if slots is not None else list(range(B))
    for s in order:     # NaN everywhere outside each image's H x W, and in the unused slot
        canvas[s, :, :H, :W] = torch.randn(3, H, W, generator=gen, device='cuda')
    d_slots = torch.tensor(slots, dtype=torch.int32, device='cuda') if slots is not None else None
    Hp, Wp = -(-H // 4), -(-W // 4)
    n = B * Hp * Wp * 64
    img = O.patch_pad(canvas[order][:, :, :H, :W])
    ref = img.view(B, 3, Hp, 4, Wp, 4).permute(0, 2, 4, 1, 3, 5).reshape(B * Hp * Wp, 48)
    ref = torch.cat([ref, torch.zeros(B * Hp * Wp, 16, device='cuda')], 1).flatten()
    for with_lo in (True, False):
        (hi, hfull), (lo, lfull) = _planes(n)
        ctx.check(_op(ctx, 'alm_op_patch_im2col', canvas.data_ptr(), n_canvas, Hc, Wc, _ptr(d_slots), B, H, W,
                      hi.data_ptr(), lo.data_ptr() if with_lo else None))
        assert_guard(hfull, n, -1)
        assert_guard(lfull, n, -1)
        if with_lo:
            _assert_split(hi, lo, ref, name)
        else:
            assert torch.equal(hi, ref.to(torch.bfloat16).view(torch.int16))
            assert bool((lo == -1).all()), 'lo written without a lo plane'


# ----------------------------------------------------------------------------------------------- FPN assembly
# pages whose stage grids are odd at every level (68 x 900: 17/9/5/3 x 225/113/57/29), 100 x 900, and the benchmark's
FPN_PAGES = [(2, 68, 900), (2, 100, 900), (1, 1024, 1024), (1, 1920, 1920)]


@pytest.mark.parametrize('B,H,W', FPN_PAGES)
def test_fpn_assemble_matches_fp64(ctx, B, H, W):
    grids = _stage_grids(H, W)
    gen = torch.Generator(device='cuda').manual_seed(H + W)
    levels = []
    for hs, ws in grids:
        buf, _ = guarded(B * hs * ws * 256)     # NaN past the end of every level
        buf.copy_(torch.randn(B * hs * ws * 256, generator=gen, device='cuda'))
        levels.append(buf.view(B, hs, ws, 256))
    mh, mw = grids[2]
    n = B * mh * mw * 1024
    (hi, hfull), (lo, lfull) = _planes(n)
    ctx.check(_op(ctx, 'alm_op_fpn_assemble', *[p.data_ptr() for p in levels], B, H, W, hi.data_ptr(), lo.data_ptr()))
    assert_guard(hfull, n, -1)
    assert_guard(lfull, n, -1)
    for s, (err, tol) in enumerate(_fpn_err_tol(hi, lo, levels, grids)):
        assert bool((err <= tol).all()), (s, float(err.max()))


def _fpn_err_tol(hi, lo, levels, grids):
    """the split pair hi / lo (int16, [rows * 1024]) of alm_op_fpn_assemble on levels [B, hs, ws, 256] (grids: their
    (hs, ws)) against fp64: p3's columns must be its exact split; -> (|got - ref|, bound) of the bilinear levels p2, p4
    and p5"""
    from oracle import omniparser_ref as O
    # fpn.py:38-44 in fp64, then the stride-2 1 x 1 input_proj's sampling of pixels (2i, 2j)
    cat = O.fpn_concat(*[p.double().permute(0, 3, 1, 2) for p in levels])[:, :, ::2, ::2]
    ref = cat.permute(0, 2, 3, 1).reshape(-1, 1024)
    hi, lo = hi.reshape(-1, 1024), lo.reshape(-1, 1024)
    # p3: exact copies
    _assert_split(hi[:, 256:512].contiguous(), lo[:, 256:512].contiguous(), levels[1][:, ::2, ::2].reshape(-1, 256), 'p3')
    # bilinear levels: the kernel computes the source coordinate scale * (dst + 0.5) - 0.5 in fp32 (3 roundings, each
    # <= 2^-24 * in), so a tap may move by 3 * 2^-24 * in along each axis, changing the value by that times
    # 2 * max|p|; plus 16 ulp of max|p| for the fp32 lerp and 2^-16 relative for the split pair (hi + lo)
    got = _joined(hi, lo)
    out = []
    for s, c0 in ((0, 0), (2, 512), (3, 768)):
        hs, ws = grids[s]
        pmax = float(levels[s].abs().max())
        tol = pmax * U32 * (6 * (hs + ws) + 16) + 2.0 ** -16 * ref[:, c0:c0 + 256].abs()
        out.append(((got[:, c0:c0 + 256] - ref[:, c0:c0 + 256]).abs(), tol))
    return out


# ----------------------------------------------------------------------------------------------- sine position embedding
def _sine_masks(kind, B, H, W, gen):
    if kind == 'none':
        return None
    m = torch.zeros(B, H, W, dtype=torch.uint8)
    m[1, :, 1:] = 1                                     # one live pixel wide
    if B > 3:
        m[2, H * 5 // 8:, :] = 1                        # live 5/8 x 3/7 of the page
        m[2, :, W * 3 // 7:] = 1
    m[-1] = (torch.rand(H, W, generator=gen) < 0.3).to(torch.uint8)   # not a rectangle: columns of different heights
    return m


def _sine_pos(ctx, mask, B, H, W, h, w):
    n = B * h * w
    pos, pfull = guarded(n * 512)
    kpm, kfull = guarded(n, torch.uint8, 7)
    d_mask = mask.cuda() if mask is not None else None
    rc = _op(ctx, 'alm_op_sine_pos', _ptr(d_mask), B, H, W, h, w, pos.data_ptr(), kpm.data_ptr())
    assert_guard(pfull, n * 512)
    assert_guard(kfull, n, 7)
    return rc, pos, kpm


@pytest.mark.parametrize('B,H,W,h,w,kind', [(2, 1920, 1920, 120, 120, 'none'), (4, 1920, 1920, 120, 120, 'masks'),
                                             (3, 640, 640, 160, 160, 'masks'), (3, 61, 45, 9, 7, 'masks')])
def test_sine_pos_matches_oracle(ctx, B, H, W, h, w, kind):
    """position_embedding_sine(level_mask(mask)) of the oracle; 160 x 160 is the largest grid whose two fp32 cumulative
    sums fit the kernel's 200 KB of shared memory"""
    from oracle import omniparser_ref as O
    gen = torch.Generator().manual_seed(h * w + B)
    mask = _sine_masks(kind, B, H, W, gen)
    rc, pos, kpm = _sine_pos(ctx, mask, B, H, W, h, w)
    ctx.check(rc)
    m = O.level_mask((mask if mask is not None else torch.zeros(B, H, W, dtype=torch.uint8)).bool(), (h, w))
    ref = O.position_embedding_sine(m).reshape(-1, 512)
    assert torch.equal(kpm.cpu(), m.flatten().to(torch.uint8))
    got = pos.view(-1, 512).cpu()
    # both are fp32 with the same operations up to the sin / cos implementation and powf's last bit of dim_t
    err = float((got - ref).abs().max())
    assert err <= 3e-6, err


def test_sine_pos_rejects_grids_past_shared_memory(ctx):
    rc, pos, kpm = _sine_pos(ctx, None, 1, 644, 640, 161, 160)
    assert rc == ERR_UNSUPPORTED
    assert bool(torch.isnan(pos).all()) and bool((kpm == 7).all()), 'written before the error'
    # the context stays usable
    from oracle import omniparser_ref as O
    rc, pos, kpm = _sine_pos(ctx, None, 1, 64, 64, 4, 4)
    ctx.check(rc)
    ref = O.position_embedding_sine(torch.zeros(1, 4, 4, dtype=torch.bool)).reshape(-1, 512)
    assert float((pos.view(-1, 512).cpu() - ref).abs().max()) <= 3e-6


# ----------------------------------------------------------------------------------------------- row softmax
@pytest.mark.parametrize('masked', [False, True])
@pytest.mark.parametrize('n', [1, 27, 257, 4096, 14400])
def test_softmax_rows_matches_fp64(ctx, n, masked):
    """MGP-STR's A^3 maps (no mask) and the decoder's unfused cross-attention (kpm per image, rows_per_mask = 8 Ncap)"""
    ncap, nimg = 3, 3
    rpm = 8 * ncap
    rows = rpm * nimg
    gen = torch.Generator(device='cuda').manual_seed(n + masked)
    lds, ldo = n + 5, n + 3
    s = _nan_rows(rows, lds, n)
    s[:, :n] = torch.randn(rows, n, generator=gen, device='cuda') * 8       # scores span tens of units
    kpm = None
    if masked:
        kpm = torch.zeros(nimg, n, dtype=torch.uint8, device='cuda')
        if n > 1:
            kpm[0, n - max(1, n // 3):] = 1                                   # right-hand columns
            kpm[1] = (torch.rand(n, generator=gen, device='cuda') < 0.5).to(torch.uint8)
            kpm[1, n // 2] = 0
            kpm[2] = 1                                                        # one live column
            kpm[2, (n * 2) // 3] = 0
            for i in range(2):                                                # the row maximum in a masked column
                j = int(kpm[i].nonzero()[0])
                s[i * rpm:(i + 1) * rpm, j] = s[:, :n].max() + 30
    out, ofull = guarded(rows * ldo)
    (hi, hfull), (lo, lfull) = _planes(rows * ldo)

    def run(f32, hi_, lo_):
        ctx.check(_op(ctx, 'alm_op_softmax_rows', s.data_ptr(), lds, rows, n, _ptr(kpm), rpm, n, _ptr(f32), _ptr(hi_),
                      _ptr(lo_), ldo))
    run(out, hi, lo)
    for full, fill in ((ofull, NAN), (hfull, -1), (lfull, -1)):
        assert_guard(full, rows * ldo, fill)
    o, h, l = out.view(rows, ldo), hi.view(rows, ldo), lo.view(rows, ldo)
    assert bool(torch.isnan(o[:, n:]).all()) and bool((h[:, n:] == -1).all()) and bool((l[:, n:] == -1).all()), \
        'columns n..ldo-1 written'
    x = s[:, :n].double()
    if kpm is not None:
        x = x.masked_fill(kpm.repeat_interleave(rpm, 0).bool(), float('-inf'))
    ref = x.softmax(-1)
    got = o[:, :n]
    assert torch.isfinite(got).all()
    # fp32: exp of (s - max) with its rounding of 2^-24 |s - max| relative, the row sum over n / 128 terms per thread
    # plus a 7-level tree, the division
    m = x.max(-1, keepdim=True).values
    rel = U32 * (2 * (x - m).abs().nan_to_num(posinf=0.0) + n / 128 + 16)
    err = (got.double() - ref).abs()
    assert bool((err <= ref * rel + 2.0 ** -126).all()), float((err / (ref * rel + 2.0 ** -126)).max())
    if kpm is not None:
        assert not bool(bits(got)[ref == 0].any()), 'a masked column is not +0'
    _assert_split(h[:, :n].contiguous(), l[:, :n].contiguous(), got, 'P')
    (hi2, _), (lo2, _) = _planes(rows * ldo)
    run(None, hi2, lo2)
    assert torch.equal(hi2, hi) and torch.equal(lo2, lo)


# ----------------------------------------------------------------------------------------------- window attention
def _nslots(heads, n_win):
    return max(1, min(n_win, sms() // (heads // 2)))


def _ring(ns, B, nWh):
    """a layout of B x nWh x nWw >= 3 ns windows that is not a multiple of ns: every persistent CTA's 3-stage ring
    wraps at least once and the slots end unevenly"""
    nWw = -(-3 * ns // (B * nWh))
    while (B * nWh * nWw) % ns == 0:
        nWw += 1
    return B, nWh, nWw


# heads -> (shift, layout from the persistent kernel's slot count ns = SMs / (heads / 2))
WATTN_EX_CASES = {
    'h32-below-nslots': (32, 3, lambda ns: (1, 1, max(1, ns - 3))),
    'h32-ring-nWw1': (32, 3, lambda ns: (1, 3 * ns + 5, 1)),
    'h16-ring-batch': (16, 3, lambda ns: (4 * ns + 3, 1, 1)),
    'h8-ring-B2': (8, 3, lambda ns: _ring(ns, 2, 2)),
    'h4-ring-B2': (4, 3, lambda ns: _ring(ns, 2, 8)),
    'h4-config5-stage0': (4, 3, lambda ns: (1, 69, 69)),     # the 1920 x 1920 page: 480 x 480 tokens
    'h32-shift0': (32, 0, lambda ns: _ring(ns, 1, 2)),
}


def _wattn_inputs(B, nWh, nWw, heads, shift, seed):
    """qkv [rows, 3C] with scores q.k * 32^-0.5 of standard deviation 10; in every window with more than one shift
    region, query 0 gets a raw score of 50 (the largest by far) on a key of another region, so a lost -100 mask moves
    its output by O(1)"""
    from oracle import omniparser_ref as O
    C = heads * 32
    gen = torch.Generator(device='cuda').manual_seed(seed)
    nW = B * nWh * nWw
    rows = nW * 49
    buf, _ = guarded(rows * 3 * C)            # NaN past the last row
    qkv = buf.view(rows, 3 * C)
    qkv.copy_(torch.randn(rows, 3 * C, generator=gen, device='cuda'))
    qkv[:, :2 * C] *= 10 ** 0.5
    tab = torch.randn(169, heads, generator=gen, device='cuda') * 0.5
    if shift:
        mask = O.shift_mask(nWh * 7, nWw * 7)                  # [nWh * nWw, 49, 49], -100 across regions
        w = qkv.view(B, nWh * nWw, 49, 3, heads, 32)
        for wi in (mask[:, 0, :] != 0).any(-1).nonzero().flatten().tolist():
            j = int((mask[wi, 0] != 0).nonzero()[0])
            q0 = w[:, wi, 0, 0]                                # [B, heads, 32]
            w[:, wi, j, 1] = q0 * (50 / (q0 * q0).sum(-1, keepdim=True) / 32 ** -0.5)
    return qkv, tab


def _wattn_tol(qkv, heads, B, nWh, nWw, scale=32 ** -0.5):
    """|got - ref| bound per element for the three-term split (hi*hi + lo*hi + hi*lo of operands held to 2^-16 relative):
    each product is off by at most e = 3 * 2^-16 of its magnitude, so a score s_ij by e * A_ij, A_ij = sum_d
    |q_d k_d| * scale, which moves the output o_i by at most e * max_j A_ij * max_j |v_j - o_i| <= e * A_i * 2 V;
    P.V adds e * V (V = max |v| of the window and head).  fp32 softmax terms are orders of magnitude below these.
    scale 1: q already scaled (the encoder's qkv planes)."""
    e = 3 * 2.0 ** -16
    q, k, v = qkv.double().view(-1, 49, 3, heads, 32).permute(2, 0, 3, 1, 4)
    A = ((q.abs() * scale) @ k.abs().transpose(-1, -2)).amax(-1)              # [nW, heads, 49]
    V = v.abs().amax((-1, -2))                                               # [nW, heads]
    t = e * (2 * A * V[..., None] + V[..., None])
    return t.transpose(1, 2).unsqueeze(-1).expand(-1, 49, heads, 32).reshape(qkv.shape[0], heads * 32)


def _run_wattn(ctx, qkv, tab, B, nWh, nWw, heads, shift, f32=True):
    rows, C = qkv.shape[0], heads * 32
    n = rows * C
    out, ofull = guarded(n)
    (hi, hfull), (lo, lfull) = _planes(n)
    ctx.check(_op(ctx, 'alm_op_window_attention_ex', qkv.data_ptr(), tab.data_ptr(), out.data_ptr() if f32 else None,
                  hi.data_ptr(), lo.data_ptr(), B, nWh, nWw, C, heads, shift))
    for full, fill in ((ofull, NAN), (hfull, -1), (lfull, -1)):
        assert_guard(full, n, fill)
    if not f32:
        assert bool(torch.isnan(out).all()), 'fp32 output written without one'
    return out.view(rows, C), hi, lo


WATTN_QSCALE = 0.17677669529663687     # 32^-0.5 in fp32, folded into the encoder's q rows at load time


def _qkv_planes(qkv, C):
    """the encoder's qkv operand: q columns times WATTN_QSCALE in fp32, then split -> (hi, lo) int16 planes, each
    followed by a guard"""
    x = qkv.clone()
    x[:, :C] *= torch.tensor(WATTN_QSCALE, dtype=torch.float32, device=x.device)
    h = x.to(torch.bfloat16)
    planes = []
    for p in (h, (x - h.float()).to(torch.bfloat16)):
        buf, _ = guarded(x.numel(), torch.int16, -1)
        buf.copy_(p.view(torch.int16).flatten())
        planes.append(buf)
    return planes


def _run_wattn_planes(ctx, planes, tab, B, nWh, nWw, heads, shift, f32=True):
    rows, C = planes[0].numel() // (3 * heads * 32), heads * 32
    n = rows * C
    out, ofull = guarded(n)
    (hi, hfull), (lo, lfull) = _planes(n)
    ctx.check(_op(ctx, 'alm_op_window_attention_planes', planes[0].data_ptr(), planes[1].data_ptr(), tab.data_ptr(),
                  out.data_ptr() if f32 else None, hi.data_ptr(), lo.data_ptr(), B, nWh, nWw, C, heads, shift))
    for full, fill in ((ofull, NAN), (hfull, -1), (lfull, -1)):
        assert_guard(full, n, fill)
    if not f32:
        assert bool(torch.isnan(out).all()), 'fp32 output written without one'
    return out.view(rows, C), hi, lo


def _check_wattn(ctx, B, nWh, nWw, heads, shift, seed):
    """alm_op_window_attention_ex on fp32 qkv, and alm_op_window_attention_planes on the planes of the pre-scaled
    q (against fp64 of the planes' own values hi + lo, no further scaling), under every wattn_impl"""
    from tests.test_gpu_omniparser import window_attention_ref64
    qkv, tab = _wattn_inputs(B, nWh, nWw, heads, shift, seed)
    ref = window_attention_ref64(qkv, tab, B, nWh, nWw, heads, shift)
    tol = _wattn_tol(qkv, heads, B, nWh, nWw)
    planes = _qkv_planes(qkv, heads * 32)
    joined = _joined(*planes).view(qkv.shape)
    ref_p = window_attention_ref64(joined, tab, B, nWh, nWw, heads, shift, scale=1.0)
    tol_p = _wattn_tol(joined, heads, B, nWh, nWw, scale=1.0)
    for impl in (0, 1, 3):
        with options(ctx, wattn_impl=impl):
            out, hi, lo = _run_wattn(ctx, qkv, tab, B, nWh, nWw, heads, shift)
            assert torch.isfinite(out).all(), impl
            err = (out.double() - ref).abs()
            assert bool((err <= tol).all()), (impl, float((err / tol).max()), float(err.max()))
            _assert_split(hi, lo, out.flatten(), f'impl {impl}')
            _, hi2, lo2 = _run_wattn(ctx, qkv, tab, B, nWh, nWw, heads, shift, f32=False)   # the encoder's form
            assert torch.equal(hi2, hi) and torch.equal(lo2, lo), impl
            out, hi, lo = _run_wattn_planes(ctx, planes, tab, B, nWh, nWw, heads, shift)
            assert torch.isfinite(out).all(), ('planes', impl)
            err = (out.double() - ref_p).abs()
            assert bool((err <= tol_p).all()), ('planes', impl, float((err / tol_p).max()), float(err.max()))
            _assert_split(hi, lo, out.flatten(), f'planes, impl {impl}')
            _, hi2, lo2 = _run_wattn_planes(ctx, planes, tab, B, nWh, nWw, heads, shift, f32=False)
            assert torch.equal(hi2, hi) and torch.equal(lo2, lo), ('planes', impl)


@pytest.mark.parametrize('name', list(WATTN_EX_CASES))
def test_window_attention_ex_matches_fp64(ctx, name):
    heads, shift, layout = WATTN_EX_CASES[name]
    B, nWh, nWw = layout(_nslots(heads, 1 << 30))
    n_win, ns = B * nWh * nWw, _nslots(heads, B * nWh * nWw)
    if 'ring' in name:
        assert n_win >= 3 * ns and n_win % ns != 0, (n_win, ns)
    if 'below' in name:
        assert n_win < sms() // (heads // 2)
    _check_wattn(ctx, B, nWh, nWw, heads, shift, seed=n_win + heads)


def _core_cases():
    from tests.test_gpu_omniparser import WATTN_CORE_CASES
    return WATTN_CORE_CASES


@pytest.mark.parametrize('B,nWh,nWw,heads,shift', _core_cases())
def test_window_attention_ex_core_cases_sharp(ctx, B, nWh, nWw, heads, shift):
    """test_window_attention_core's layouts with sharp scores, every output form"""
    _check_wattn(ctx, B, nWh, nWw, heads, shift, seed=B * 1000 + nWh * 100 + nWw * 10 + heads)


# ----------------------------------------------------------------------------------------------- argument errors
def test_argument_errors_leave_the_context_usable(ctx):
    d = torch.zeros(1 << 16, device='cuda')
    hst = torch.zeros(1 << 16)
    (hi, _), (lo, _) = _planes(1 << 16)
    i32 = torch.zeros(1 << 14, dtype=torch.int32, device='cuda')
    u8 = torch.zeros(1 << 14, dtype=torch.uint8, device='cuda')
    P = _ptr

    def gather(src=d, Cs=128, nsrc=1, out=d):
        return _op(ctx, 'alm_op_gather_ln', P(src), 2048, None, nsrc, Cs, 4, None, None, 1e-5, 0, None, 0, P(out), 2048,
                   None, None, 0, None, None, None)
    assert gather() == 0
    assert gather(src=None) == ERR_INVALID
    assert gather(src=hst) == ERR_INVALID
    assert gather(out=hst) == ERR_INVALID
    assert gather(out=None) == ERR_INVALID                    # no output
    assert gather(Cs=100) == ERR_INVALID                      # not a multiple of 128 (or 192)
    assert gather(Cs=640) == ERR_UNSUPPORTED                  # no instantiation for 5 x 128
    assert gather(Cs=128, nsrc=5) == ERR_UNSUPPORTED

    def smap(m=i32, kind=0, shift=3):
        return _op(ctx, 'alm_op_swin_map', kind, 1, 9, 9, shift, P(m))
    assert smap() == 0
    assert smap(m=None) == ERR_INVALID
    assert smap(m=hst) == ERR_INVALID
    assert smap(kind=3) == ERR_INVALID
    assert smap(kind=1) == ERR_INVALID                        # merge has no shift
    assert smap(shift=7) == ERR_INVALID

    slots = torch.tensor([1, 0], dtype=torch.int32, device='cuda')

    def im2col(img=d, s=slots, out=hi, n_canvas=2, H=16):
        return _op(ctx, 'alm_op_patch_im2col', P(img), n_canvas, 16, 16, P(s), 2, H, 16, P(out), None)
    assert im2col() == 0
    assert im2col(img=None) == ERR_INVALID
    assert im2col(img=hst) == ERR_INVALID
    assert im2col(out=None) == ERR_INVALID
    assert im2col(n_canvas=1) == ERR_INVALID                  # slot 1 is off the canvas
    assert im2col(s=None, n_canvas=1) == ERR_INVALID          # image 1 is off the canvas
    assert im2col(H=17) == ERR_INVALID                        # taller than the canvas

    def fpn(p3=d, out=hi):
        return _op(ctx, 'alm_op_fpn_assemble', P(d), P(p3), P(d), P(d), 1, 32, 32, P(out), None)
    assert fpn() == 0
    assert fpn(p3=None) == ERR_INVALID
    assert fpn(p3=hst) == ERR_INVALID
    assert fpn(out=None) == ERR_INVALID

    def sine(pos=d, kpm=u8, mask=None):
        return _op(ctx, 'alm_op_sine_pos', P(mask), 1, 32, 32, 4, 4, P(pos), P(kpm))
    assert sine() == 0
    assert sine(pos=None) == ERR_INVALID
    assert sine(kpm=torch.zeros(16, dtype=torch.uint8)) == ERR_INVALID
    assert sine(mask=torch.zeros(1024, dtype=torch.uint8)) == ERR_INVALID

    def softmax(s=d, out=d, kpm=None, rpm=1, n=64):
        return _op(ctx, 'alm_op_softmax_rows', P(s), 64, 8, n, P(kpm), rpm, 64, P(out), None, None, 64)
    assert softmax() == 0
    assert softmax(s=None) == ERR_INVALID
    assert softmax(out=hst) == ERR_INVALID
    assert softmax(out=None) == ERR_INVALID
    assert softmax(n=65) == ERR_INVALID                       # wider than lds / ldo
    assert softmax(kpm=u8, rpm=0) == ERR_INVALID

    tab = torch.zeros(169 * 4, device='cuda')

    def wattn(qkv=d, out=d, C=128, heads=4):
        return _op(ctx, 'alm_op_window_attention_ex', P(qkv), P(tab), P(out), None, None, 1, 1, 1, C, heads, 3)
    assert wattn() == 0
    assert wattn(qkv=None) == ERR_INVALID
    assert wattn(qkv=hst) == ERR_INVALID
    assert wattn(out=None) == ERR_INVALID                     # no output at all
    assert wattn(C=100) == ERR_UNSUPPORTED                    # head_dim 32 only
    assert _op(ctx, 'alm_op_window_attention', P(d), P(tab), None, 1, 1, 1, 128, 4, 3) == ERR_INVALID

    (qh, _), (ql, _) = _planes(49 * 3 * 128)
    (oh, _), (ol, _) = _planes(49 * 128)
    out = torch.full((49 * 128,), NAN, device='cuda')

    def planes(qkv_hi=qh, qkv_lo=ql, t=tab, f32=out, hi_=oh, lo_=ol, B=1, nWh=1, nWw=1, C=128, heads=4, shift=3):
        return _op(ctx, 'alm_op_window_attention_planes', P(qkv_hi), P(qkv_lo), P(t), P(f32), P(hi_), P(lo_), B, nWh,
                   nWw, C, heads, shift)
    for kw in (dict(qkv_hi=None), dict(qkv_lo=None), dict(t=None), dict(f32=None, hi_=None, lo_=None),
               dict(hi_=None),                                          # out_lo needs out_hi
               dict(qkv_hi=torch.zeros(49 * 3 * 128, dtype=torch.int16)), dict(t=hst), dict(f32=hst),
               dict(qkv_hi=qh[1:]), dict(qkv_lo=ql[4:]), dict(f32=out[1:]), dict(hi_=oh[1:]),   # misaligned
               dict(B=0), dict(nWh=0), dict(nWw=-1), dict(heads=0), dict(shift=-1), dict(shift=7)):
        assert planes(**kw) == ERR_INVALID, kw
    assert planes(C=100) == ERR_UNSUPPORTED                   # head_dim 32 only
    assert planes(C=256) == ERR_UNSUPPORTED
    assert bool(torch.isnan(out).all()) and bool((oh == -1).all()) and bool((ol == -1).all()), 'written before an error'
    qh.zero_()
    ql.zero_()
    assert planes() == 0
    assert bool((out == 0).all())

    # the context still computes
    _check_maps(ctx, 2, 11, 5)
