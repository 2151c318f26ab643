"""GPU: the GEMM engine under `small_grid_cap`, against fp64 and bit for bit against the uncapped launch.

`small_grid_cap` n (and the encoder / decoder caps, which reach the same launch code) sends a GEMM with at most 2 x SMs
tiles to n CTAs, so each CTA walks up to ceil(tiles / n) tiles.  That reaches schedules the full grid never runs: 32-column
tiles with dozens of tiles per CTA (uncapped, a CTA has at most two of them), the ping-pong loop for the few-tile decoder
GEMMs that run cooperatively when uncapped, consumer 1 stepping its stage / phase over long runs of the other consumer's
k-blocks, and the epilogue's per-tile row and column tables rewritten on every tile.

A tile's arithmetic does not depend on the CTA or consumer that computes it (same k order, same MMA sequence per 64-row
half), so every capped result must be bit-identical to the uncapped one, which is held to fp64 with the per-element
bound of test_gpu_gemm_operands.py (|got - ref| <= n 2^-22 sum|terms|), NaN in every operand element no row / k
addresses and in every output element the call must not write.  Shapes are derived from the SM count so that the cap
applies (tiles <= 2 x SMs).  The caps: 1, 2, 3, 7, SMs - 1 and at or above the tile count (which must act as no cap).

The cases: k_blocks below, at and several times the pipeline depth with every residue mod the depth, at both tile widths
and nsplit 3 / 1; the decoder's per-token shapes (M = 1 ... 130 against its 512 / 1536 / 2048-wide linears); column and
row bias, column-group scatter, residual, row maps with dropped rows and the in-place residual.  Split outputs are
checked on every call (hi == bf16_rn(f32), lo == bf16_rn(f32 - hi)).
"""
import pytest
import torch

from tests import support
from tests.support import ctx, options
from tests.test_gpu_gemm_operands import (GUARD, NAN_F32, Case, Opd, _call, _check, _epilogue, _launch_shape,
                                          _outputs, _r8, _run, _setup)

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

# SmemLayout in gemm.cu: the operand-stage budget of a CTA (227 KB less the barrier block, alignment slack and the
# epilogue's per-warp buffers), and the deepest ring the kernel builds
STAGE_BUDGET = 227 * 1024 - 1024 - 1024 - 8 * (16 * 32 + 32 * 4 + 128) * 4
MAX_STAGES = 16
WORST = {}  # (tile width, nsplit) -> worst err / bound


@pytest.fixture(scope='module', autouse=True)
def _report():
    yield
    print('[gemm capped] worst err/bound: ' + ', '.join(
        f'{bn}-column tiles nsplit {ns}: {r:.3g}' for (bn, ns), r in sorted(WORST.items())))


def _stages(M, bn, nsplit):
    """pipeline depth launch_wgmma picks: as many stages of (A tile, B tile) x planes as fit, at most 16"""
    planes = 2 if nsplit == 3 else 1
    stage = planes * min(128, _r8(M)) * 64 * 2 + planes * bn * 64 * 2
    return min(MAX_STAGES, STAGE_BUDGET // stage)


def _tiles(M, N, bn, nb=1):
    return -(-M // 128) * -(-N // bn) * nb


def _caps(tiles, sms):
    return sorted({1, 2, 3, 7, sms - 1, tiles, 4 * sms})


def _n_local(tiles, cap):
    """tiles per CTA of a launch capped at `cap` CTAs"""
    grid = min(tiles, cap)
    return [len(range(b, tiles, grid)) for b in range(grid)]


def _kbs(stages):
    """k-block counts: 1, around the ring depth, and one for every residue mod the depth at >= 3 turns of the ring"""
    return sorted({1, stages - 1, stages, stages + 1} | {3 * stages + r for r in range(stages)} - {0})


def _bits(out):
    return [t.view(torch.int32) if t.dtype == torch.float32 else t for t in out]


def _assert_same(base, got, label):
    for k, (x, y) in enumerate(zip(_bits(base), _bits(got))):
        if not torch.equal(x, y):
            raise AssertionError(f'{label}: {int((x != y).sum())} {("f32", "hi", "lo")[k]} elements differ from the '
                                 f'uncapped call')


def _record(c, nsplit, worst):
    bn = _launch_shape(c.M, c.N, c.nb0 * c.nb1, support.sms())[0]
    WORST[(bn, nsplit)] = max(WORST.get((bn, nsplit), 0.0), worst)


def _capped(ctx, name, c, nsplit, seed, caps=None):
    """c uncapped against fp64, then under every cap bit for bit against the uncapped outputs; returns the worst
    err / bound"""
    sms = support.sms()
    tiles = _tiles(c.M, c.N, _launch_shape(c.M, c.N, c.nb0 * c.nb1, sms)[0], c.nb0 * c.nb1)
    assert tiles <= 2 * sms, f'{name}: {tiles} tiles, the cap applies to <= {2 * sms}'
    _setup(c, seed)
    if nsplit == 1:
        c.a.poison_lo()
        c.b.poison_lo()
    with options(ctx, small_grid_cap=0):
        base = _run(ctx, c, nsplit, 0)
    worst = _check(c, base, nsplit, 0, f'{name} nsplit {nsplit} uncapped')
    for cap in caps or _caps(tiles, sms):
        with options(ctx, small_grid_cap=cap):
            _assert_same(base, _run(ctx, c, nsplit, 0), f'{name} nsplit {nsplit} small_grid_cap {cap}')
    _record(c, nsplit, worst)
    return worst


# ------------------------------------------------------------------------------------------ shapes
def _narrow_shape(sms):
    """3 row blocks (tail of 44 rows inside half 0) x 21 column blocks of 32 (9 columns in the last): 63 tiles"""
    M, N = 300, 32 * 20 + 9
    assert _launch_shape(M, N, 1, sms)[0] == 32
    return M, N


def _wide_shape(sms):
    """11 row blocks (tail of 100 rows inside half 1) x n 128-column blocks (88 columns in the last), 2 x SMs tiles"""
    M, nb = 128 * 10 + 100, (2 * sms) // 11
    N = 128 * nb - 40
    assert _launch_shape(M, N, 1, sms)[0] == 128
    return M, N


SHAPES = {'narrow': _narrow_shape, 'wide': _wide_shape}


def test_the_cases_reach_every_schedule_property():
    """odd and even tile counts per CTA, grids where some CTAs have one tile more, cooperative and ping-pong launches,
    and every residue of k_blocks mod the ring depth"""
    sms = support.sms()
    for width, shape in SHAPES.items():
        M, N = shape(sms)
        bn = 32 if width == 'narrow' else 128
        tiles = _tiles(M, N, bn)
        counts = [_n_local(tiles, cap) for cap in _caps(tiles, sms)]
        assert any(max(n) > 20 for n in counts), width
        assert {n % 2 for nl in counts for n in nl} == {0, 1}, width
        assert any(len(set(nl)) > 1 for nl in counts), f'{width}: no grid with uneven tiles per CTA'
        assert any(set(nl) == {1} for nl in counts) and any(max(nl) > 1 for nl in counts), width
        for nsplit in (3, 1):
            s = _stages(M, bn, nsplit)
            kbs = _kbs(s)
            assert {k % s for k in kbs if k >= 3 * s} == set(range(s)) and min(kbs) < s < max(kbs), (width, nsplit)


@pytest.mark.parametrize('nsplit', [3, 1])
@pytest.mark.parametrize('width', list(SHAPES))
def test_k_blocks_around_the_ring_depth(ctx, width, nsplit):
    """every residue of k_blocks mod the stage count: consumer 1's skip over the other consumer's tiles must land on
    the right stage and phase after many tiles"""
    M, N = SHAPES[width](support.sms())
    bn = 32 if width == 'narrow' else 128
    for kb in _kbs(_stages(M, bn, nsplit)):
        K = 64 * kb - (24 if kb % 2 == 0 else 0)  # K tails on the even counts
        c = Case(Opd(M, K, _r8(K)), Opd(N, K, _r8(K) + 8), dict(ldo=_r8(N) + 8, bias='col', act=kb % 3))
        worst = _capped(ctx, f'{width} M {M} N {N} K {K}', c, nsplit, seed=kb)
        print(f'[gemm capped] {width} K {K} nsplit {nsplit}: worst err/bound {worst:.3g}')


# the decoder's per-token linears with more than 32 live sequences (omni.cu decoder_step): q / k / v / output
# projections (N = 512, residual), the packed projections (N = 1536), the MLP (N = 2048 with ReLU, then K = 2048)
DECODER = {'n512_k512_resid': (512, 512, dict(bias='col', resid=True)),
           'n1536_k512': (1536, 512, dict(bias='col')),
           'n2048_k512_relu': (2048, 512, dict(bias='col', act=2)),
           'n512_k2048_resid': (512, 2048, dict(bias='col', resid=True))}


@pytest.mark.parametrize('nsplit', [3, 1])
@pytest.mark.parametrize('name', list(DECODER))
def test_decoder_token_shapes(ctx, name, nsplit):
    """M = 1 ... 130 rows: tails inside half 0, inside half 1, exactly 64 and 128, and a second row block.  Uncapped
    these run cooperatively (one tile per CTA); every cap runs them ping-pong."""
    N, K, extra = DECODER[name]
    sms = support.sms()
    worst = 0.0
    for M in range(1, 131):
        e = dict(ldo=N, **{k: v for k, v in extra.items() if k != 'resid'})
        if extra.get('resid'):
            e['resid'] = (N, 0, 0)
        c = Case(Opd(M, K, K), Opd(N, K, K), e)
        tiles = _tiles(M, N, _launch_shape(M, N, 1, sms)[0])
        worst = max(worst, _capped(ctx, f'{name} M {M}', c, nsplit, seed=M, caps=sorted({1, 2, 3, 7, sms - 1, tiles})))
    print(f'[gemm capped] decoder {name} nsplit {nsplit}: worst err/bound {worst:.3g}')


def _epilogue_cases(sms):
    (Mn, Nn), (Mw, Nw) = _narrow_shape(sms), _wide_shape(sms)
    cases = {}
    for width, M, N in (('narrow', Mn, Nn), ('wide', Mw, Nw)):
        K = 136
        cases[f'{width}_row_bias_relu'] = lambda M=M, N=N, K=K: Case(Opd(M, K, K), Opd(N, K, K + 8),
                                                                        dict(ldo=N + 3, bias='row', act=2))
        cases[f'{width}_col_group'] = lambda M=M, N=N, K=K: Case(Opd(M, K, K), Opd(N, K, K),
                                                                 dict(ldo=64, cg=64, cgs=_r8(M * 64) + 8, bias='col'))
        cases[f'{width}_resid_alpha'] = lambda M=M, N=N, K=K: Case(Opd(M, K, K), Opd(N, K, K),
                                                                   dict(ldo=_r8(N), resid=(_r8(N) + 4, 0, 0),
                                                                        alpha=-0.75, act=1))
    # a batched problem: tiles run through several batches on one CTA (output, bias and residual batch offsets)
    M, N, K = 100, 200, 72
    cases['narrow_batched'] = lambda: Case(Opd(M, K, K, nb0=3, bs0=M * K), Opd(N, K, K, nb1=2, bs1=N * K),
                                           dict(ldo=N, obs0=M * N, obs1=3 * M * N, bias='col', bias_bs0=N,
                                                resid=(N, M * N, 3 * M * N)))
    return cases


EPILOGUES = list(_epilogue_cases(132))  # the names only: they do not depend on the SM count


@pytest.mark.parametrize('nsplit', [3, 1])
@pytest.mark.parametrize('name', EPILOGUES)
def test_epilogue_tables_refreshed_on_every_tile(ctx, name, nsplit):
    c = _epilogue_cases(support.sms())[name]()
    worst = _capped(ctx, name, c, nsplit, seed=sum(map(ord, name)))
    print(f'[gemm capped] {name} nsplit {nsplit}: worst err/bound {worst:.3g}')


@pytest.mark.parametrize('nsplit', [3, 1])
@pytest.mark.parametrize('width', list(SHAPES))
def test_row_maps_and_in_place_residual(ctx, width, nsplit):
    """Row maps (a permutation with dropped rows, residual rows read through their own map) and the in-place residual
    (out_f32 == resid): under every cap, bit for bit the plain call with the rows moved / the residual copied."""
    sms = support.sms()
    M, N = SHAPES[width](sms)
    K, ld = 100, _r8(N)
    c = Case(Opd(M, K, _r8(K)), Opd(N, K, _r8(K)), dict(ldo=ld, bias='col', resid=(ld, 0, 0), act=1))
    _setup(c, seed=11)
    if nsplit == 1:
        c.a.poison_lo()
        c.b.poison_lo()
    g = torch.Generator(device='cuda').manual_seed(12)
    out_map = torch.randperm(M, generator=g, device='cuda').to(torch.int32)
    out_map[torch.randperm(M, generator=g, device='cuda')[:M // 5]] = -1
    extra = 9  # the mapped residual has more rows than the problem
    resid_map = torch.randperm(M + extra, generator=g, device='cuda')[:M].to(torch.int32)
    big = torch.full(((M + extra) * ld + GUARD,), float('nan'), device='cuda')
    big[:(M + extra) * ld].view(M + extra, ld)[:, :N] = torch.randn(M + extra, N, generator=g, device='cuda')
    c.resid[:M * ld].view(M, ld)[:, :N] = big[:(M + extra) * ld].view(M + extra, ld)[resid_map.long(), :N]
    keep = out_map >= 0
    rows = torch.arange(M, device='cuda')[keep]
    col = torch.arange(N, device='cuda')
    src = (rows[:, None] * ld + col).reshape(-1)
    dst = (out_map[keep].long()[:, None] * ld + col).reshape(-1)
    tiles = _tiles(M, N, 32 if width == 'narrow' else 128)
    with options(ctx, small_grid_cap=0):
        base = _run(ctx, c, nsplit, 0)
    worst = _check(c, base, nsplit, 0, f'{width} plain')
    for cap in [0] + _caps(tiles, sms):
        with options(ctx, nsplit=nsplit, small_grid_cap=cap):
            # row maps
            out = _outputs(c.written.numel())
            e = _epilogue(c, *out)
            e.resid, e.out_map, e.resid_map = big.data_ptr(), out_map.data_ptr(), resid_map.data_ptr()
            ctx.check(_call(ctx, c.a.desc(), c.b.desc(), e))
            want = _outputs(c.written.numel())
            for w, b in zip(want, base):
                w[dst] = b[src]
            _assert_same(want, out, f'{width} nsplit {nsplit} row maps, small_grid_cap {cap}')
            # in place: the residual buffer is the fp32 output
            x = c.resid.clone()
            out = _outputs(c.written.numel())
            e = _epilogue(c, x, out[1], out[2])
            e.resid = x.data_ptr()
            ctx.check(_call(ctx, c.a.desc(), c.b.desc(), e))
            n = base[0].numel()
            assert bool((x[n:].view(torch.int32) == NAN_F32).all()), f'{width}: in-place write past the output'
            _assert_same(base, (x[:n], out[1], out[2]), f'{width} nsplit {nsplit} in-place residual, small_grid_cap {cap}')
    _record(c, nsplit, worst)
    print(f'[gemm capped] {width} row maps / in place nsplit {nsplit}: worst err/bound {worst:.3g}')
