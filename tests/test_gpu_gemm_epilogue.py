"""GPU: every feature of the GEMM engine's fused epilogue through alm_op_gemm, against fp64.

Each case runs at nsplit 3 and 1 with the tolerances of test_gpu_gemm_pingpong.py, plus exact checks: every output
buffer starts as NaN with a guard region after it, and each element the call must not write (dropped rows, pad columns,
gaps between column groups and batches, the guard) must come back bit for bit.  When fp32 and split outputs are both
requested, hi == bf16_rn(f32) and lo == bf16_rn(f32 - hi) element for element.

The cases cover both consumer schedules (ping-pong with several tiles per CTA, and one tile per CTA) at both tile
widths, M tails inside either 64-row half, N a multiple of 32 / of 8 only / with N % 4 != 0 / odd, output rows that are
not 16-byte addressable (per-element stores), GELU / ReLU / none, alpha != 1, row bias and batched column bias, residual
with and without resid_map and in place, out_map with dropped rows, and the head-major column-group scatter in a
batched problem.
"""
import pytest
import torch

from tests.support import ctx, options, sms

torch.set_grad_enabled(False)

GUARD = 67
WORKSPACE_MB = 4096
NAN_BF16 = 0x7fc0
ALM_ERR_INVALID = -1


# name: dict(M, N, K, batch, w_batch, act, alpha, bias ('none' | 'col' | 'row'), resid ('none' | 'plain' | 'map' |
# 'inplace'), out_map, col_group, out ('f32' | 'split' | 'both'), ldo (None: N))
def _cases():
    s = sms()
    return {
        # ping-pong, 128-column tiles, M tail in half 1, N a multiple of 8 only (last chunk partly past N)
        'pingpong_gelu_both': dict(M=(2 * s + 3) * 128 + 70, N=280, K=64, act=1, bias='col', out='both'),
        # ping-pong, M tail in half 0, N a multiple of 32, permuted and dropped rows, mapped residual, alpha
        'pingpong_resid_map': dict(M=(3 * s) * 128 + 40, N=192, K=96, alpha=0.5, resid='map', out_map=True,
                                   ldo=200, out='f32'),
        # ping-pong, in-place residual (fc2 / proj form)
        'pingpong_inplace': dict(M=(2 * s + 1) * 128 + 100, N=128, K=128, bias='col', resid='inplace', out='f32'),
        # one 32-column tile per CTA, odd N, ldo not a multiple of 8 (per-element stores), ReLU, row bias, split only
        'coop_narrow_row_bias': dict(M=300, N=77, K=64, act=2, alpha=1.25, bias='row', out='split'),
        # one 128-column tile per CTA, M tail in half 1, N % 4 == 2, GELU, both outputs
        'coop_wide_gelu': dict(M=(s // 16 + 1) * 128 - 20, N=8 * 128 - 2, K=64, act=1, bias='col', ldo=8 * 128,
                               out='both'),
        # head-major column groups with gaps between groups, batched column bias, several tiles per CTA
        'col_group_batched': dict(M=2990, N=512, K=64, batch=3, bias='col', col_group=64, out='split'),
        # 32-column tiles, up to 2 per CTA, shared weights over a batch, odd N, K padded to 8, fp32 rows not 16-byte
        # addressable (per-element column-bias loads)
        'narrow_shared_w': dict(M=1000, N=333, K=40, batch=2, w_batch=1, act=0, bias='col', out='f32'),
        # 32-column tiles with residual and both outputs on 16-byte rows
        'narrow_resid_both': dict(M=1000, N=1000, K=64, act=1, bias='col', resid='plain', out='both'),
    }


CASES = ['pingpong_gelu_both', 'pingpong_resid_map', 'pingpong_inplace', 'coop_narrow_row_bias', 'coop_wide_gelu',
         'col_group_batched', 'narrow_shared_w', 'narrow_resid_both']


def _bf16_rn(x):
    return x.float().to(torch.bfloat16)


def _run_case(ctx, c, nsplit):
    M, N, K = c['M'], c['N'], c['K']
    batch = c.get('batch', 1)
    w_batch = c.get('w_batch', batch)
    act, alpha = c.get('act', 0), c.get('alpha', 1.0)
    bias_kind, resid_kind, out_kind = c.get('bias', 'none'), c.get('resid', 'none'), c['out']
    cg = c.get('col_group', 0)
    g = torch.Generator().manual_seed(M * 7 + N * 3 + K + batch)
    A = torch.randn(batch, M, K, generator=g)
    W = torch.randn(w_batch, N, K, generator=g) / K ** 0.5
    acc = torch.einsum('bmk,bnk->bmn', A.double(), W.double().expand(batch, N, K))

    # output geometry
    if cg:
        ldo, cstride = cg, (M + 3) * cg                    # rows M .. M + 2 of every group block are gaps
        obs0 = (N // cg) * cstride + 64                    # and 64 elements between batches
    else:
        ldo, cstride = c.get('ldo') or N, 0
        obs0 = M * ldo + (8 if batch > 1 else 0)
    orow = torch.arange(M)
    if c.get('out_map'):
        perm = torch.randperm(M, generator=g)
        orow = perm.clone()
        orow[torch.arange(M) % 7 == 3] = -1                # dropped rows
    live = orow >= 0
    n = torch.arange(N)
    cn = (n // cg) * cstride + n % cg if cg else n
    idx = (torch.arange(batch)[:, None, None] * obs0 + orow.clamp(min=0)[None, :, None] * ldo + cn[None, None, :])
    idx_live = idx[:, live, :]
    size = max(int(idx_live.max()) + 1, batch * obs0) + GUARD

    # reference
    x = alpha * acc
    bias = None
    bias_mode, bias_bs0 = 0, 0
    if bias_kind == 'col':
        bias_bs0 = N + 4 if batch > 1 else 0
        bias = torch.randn(max(batch, 1) * (N + 4), generator=g)
        bview = torch.stack([bias[b * bias_bs0:b * bias_bs0 + N] for b in range(batch)])
        x = x + bview.double()[:, None, :]
        bias_mode = 1
    elif bias_kind == 'row':
        bias = torch.randn(M, generator=g)
        x = x + bias.double()[None, :, None]
        bias_mode = 2
    if act == 1:
        x = torch.nn.functional.gelu(x)
    elif act == 2:
        x = torch.relu(x)

    resid = resid_map = None
    ldr, rbs0 = 0, 0
    if resid_kind in ('plain', 'map'):
        ldr = N + 4
        rrows = M + 5
        resid = torch.randn(batch, rrows, ldr, generator=g)
        rbs0 = rrows * ldr
        rrow = orow.clamp(min=0)
        if resid_kind == 'map':
            rrow = torch.randint(0, rrows, (M,), generator=g)
            resid_map = rrow.to(torch.int32)
        x = x + resid[:, rrow, :N].double()

    out_f32 = out_hi = out_lo = None
    if out_kind in ('f32', 'both'):
        out_f32 = torch.full((size,), float('nan'), device='cuda')
    if out_kind in ('split', 'both'):
        out_hi = torch.full((size,), NAN_BF16, dtype=torch.int16, device='cuda')
        out_lo = torch.full((size,), NAN_BF16, dtype=torch.int16, device='cuda')
    resid_d = None
    if resid_kind == 'inplace':
        # out_f32 is the residual: every written element holds its residual before the call
        base = torch.randn(batch, M, N, generator=g)
        flat = out_f32.cpu()
        flat[idx_live.reshape(-1)] = base[:, live, :].reshape(-1)
        out_f32.copy_(flat)
        x = x + base.double()
        resid_d, ldr, rbs0 = out_f32, ldo, obs0
    elif resid is not None:
        resid_d = resid.cuda()

    def ptr(t):
        return None if t is None else t.data_ptr()

    Ad, Wd = A.cuda(), W.cuda()
    bias_d = bias.cuda() if bias is not None else None
    rmap_d = resid_map.cuda() if resid_map is not None else None
    omap_d = orow.to(torch.int32).cuda() if c.get('out_map') else None
    with options(ctx, nsplit=nsplit):
        ctx.check(ctx.lib.alm_op_gemm(ctx.h, Ad.data_ptr(), Wd.data_ptr(), M, N, K, batch, w_batch, ptr(out_f32),
                                      ptr(out_hi), ptr(out_lo), ldo, obs0, ptr(bias_d), bias_mode, bias_bs0, alpha, act,
                                      ptr(resid_d), ldr, rbs0, ptr(rmap_d), ptr(omap_d), cg, cstride))
    ref = x[:, live, :]
    written = torch.zeros(size, dtype=torch.bool)
    written[idx_live.reshape(-1)] = True
    got = {}
    if out_f32 is not None:
        f = out_f32.cpu()
        assert torch.equal(f[~written].view(torch.int32), torch.full((int((~written).sum()),), float('nan')).view(torch.int32)), \
            'fp32 output: an element outside the live rows / columns was written'
        got['f32'] = f[idx_live]
    if out_hi is not None:
        hi, lo = out_hi.cpu(), out_lo.cpu()
        for name, t in (('hi', hi), ('lo', lo)):
            assert bool((t[~written] == NAN_BF16).all()), f'{name} output: an element outside the live rows / columns was written'
        hi_v, lo_v = hi[idx_live].view(torch.bfloat16), lo[idx_live].view(torch.bfloat16)
        got['split'] = hi_v.float() + lo_v.float()
        if out_f32 is not None:
            f = got['f32']
            h_exp = _bf16_rn(f)
            assert torch.equal(hi_v.view(torch.int16), h_exp.view(torch.int16)), 'hi != bf16_rn(f32)'
            assert torch.equal(lo_v.view(torch.int16), _bf16_rn(f - h_exp.float()).view(torch.int16)), \
                'lo != bf16_rn(f32 - hi)'
    return ref, got


@pytest.mark.gpu
@pytest.mark.parametrize('name', CASES)
def test_gemm_epilogue_matches_fp64(ctx, name):
    c = _cases()[name]
    for nsplit, tol in ((3, 2e-5), (1, 6e-3)):
        ref, got = _run_case(ctx, c, nsplit)
        for kind, v in got.items():
            v = v.double()
            assert torch.isfinite(v).all(), (nsplit, kind)
            rows_err = ((v - ref).norm(dim=2) / (ref.norm(dim=2) + 1e-30)).amax(dim=0)
            assert float(rows_err.max()) < 10 * tol, (nsplit, kind, int(rows_err.argmax()))
            assert float((v - ref).norm() / ref.norm()) < tol, (nsplit, kind)


@pytest.mark.gpu
def test_gemm_epilogue_rejects_what_the_engine_cannot_run(ctx):
    M, N, K = 64, 128, 32
    A = torch.randn(2, M, K, device='cuda')
    W = torch.randn(2, N, K, device='cuda')
    out = torch.zeros(2 * M * N, device='cuda')
    resid = torch.zeros(2 * M * N, device='cuda')
    omap = torch.arange(M, dtype=torch.int32, device='cuda')
    lib, h = ctx.lib, ctx.h
    # no output
    assert lib.alm_op_gemm(h, A.data_ptr(), W.data_ptr(), M, N, K, 1, 1, None, None, None, N, 0, None, 0, 0, 1.0, 0,
                           None, 0, 0, None, None, 0, 0) == ALM_ERR_INVALID
    # row maps on a batched problem
    assert lib.alm_op_gemm(h, A.data_ptr(), W.data_ptr(), M, N, K, 2, 2, out.data_ptr(), None, None, N, M * N, None, 0,
                           0, 1.0, 0, None, 0, 0, None, omap.data_ptr(), 0, 0) == ALM_ERR_INVALID
    # column groups with a residual, and groups that are not 4k columns wide
    assert lib.alm_op_gemm(h, A.data_ptr(), W.data_ptr(), M, N, K, 1, 1, out.data_ptr(), None, None, 64, M * N, None, 0,
                           0, 1.0, 0, resid.data_ptr(), N, 0, None, None, 64, M * 64) == ALM_ERR_INVALID
    assert lib.alm_op_gemm(h, A.data_ptr(), W.data_ptr(), M, N, K, 1, 1, out.data_ptr(), None, None, 62, M * N, None, 0,
                           0, 1.0, 0, None, 0, 0, None, None, 62, M * 64) == ALM_ERR_INVALID
    # a weight batch that neither matches nor broadcasts
    assert lib.alm_op_gemm(h, A.data_ptr(), W.data_ptr(), M, N, K, 2, 3, out.data_ptr(), None, None, N, M * N, None, 0,
                           0, 1.0, 0, None, 0, 0, None, None, 0, 0) == ALM_ERR_INVALID


def test_alm_op_gemm_is_declared_and_bound():
    import os
    import re
    from advancedliteratemachinery_b200 import _lib
    header = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'include', 'alm_ocr.h')).read()
    assert re.search(r'ALM_API\s+int\s+alm_op_gemm\s*\(', header)
    assert len(_lib.SIGNATURES['alm_op_gemm'][1]) == 25
