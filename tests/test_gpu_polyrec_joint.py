"""GPU: the joint polygon + recognition decoder pass runs every linear of a layer as ONE GEMM over both decoders' rows
(a batch dimension of 2: A rows [0, S) and [S, 2S), the decoders' weights one slab apart, bias and residual per batch).
Each half of that launch must be bit for bit the single-decoder launch on that half: same products, same accumulation
order, same epilogue.  The joint launch has twice the tiles, so at the decoder's shapes it can take the other tile
width (1 024 rows x N = 1 024: 32-wide column tiles alone, 128-wide jointly); the cases below cross that boundary.

Checked through alm_op_gemm_planes, at nsplit 3 (the decoder's) and 1, on the shapes of the decoder layer (q|k, v,
out projections, FFN, the three head layers at V = 1 104) and on row counts of smaller batches.  The self-attention
step, launched once over both halves, is checked the same way against one launch per half
(alm_op_self_attention_step).  The cross-attention runs once per decoder in the joint pass, as before.
"""
import ctypes

import pytest
import torch

from tests.support import ctx, options

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

BIAS_COL, ACT_NONE, ACT_RELU = 1, 0, 2

# (rows per decoder S, N, K, activation, residual, split output)
SHAPES = [
    (1024, 1024, 512, ACT_NONE, False, False),  # self-attention q|k (tile width changes when joined)
    (1024, 512, 512, ACT_NONE, False, False),   # self-attention v, cross-attention q
    (1024, 512, 512, ACT_NONE, True, False),    # out projections + residual
    (1024, 2048, 512, ACT_RELU, False, True),   # linear1 -> split planes
    (1024, 512, 2048, ACT_NONE, True, False),   # linear2 + residual
    (1024, 1104, 512, ACT_NONE, False, False),  # vocabulary head
    (1024, 512, 512, ACT_RELU, False, True),    # head layers 0 / 1
    (192, 1024, 512, ACT_NONE, False, False),
    (40, 512, 512, ACT_NONE, True, False),
    (300, 2048, 512, ACT_RELU, False, True),
]


def _planes(x):
    """fp32 [R, K] -> bf16 [2, R * K]: hi then lo plane of the split"""
    hi = x.to(torch.bfloat16)
    lo = (x - hi.float()).to(torch.bfloat16)
    return torch.stack([hi.flatten(), lo.flatten()]).contiguous()


def _op(planes, off, rows, K, nb0=1, bs0=0):
    from advancedliteratemachinery_b200 import _lib
    o = _lib.GemmOperand()
    o.hi = planes[0].data_ptr() + 2 * off
    o.lo = planes[1].data_ptr() + 2 * off
    o.rows, o.K, o.ld, o.nb0, o.nb1, o.bs0, o.bs1 = rows, K, K, nb0, 1, bs0, 0
    return o


def _call(ctx, a, b, e):
    torch.cuda.synchronize()
    ctx.check(ctx.lib.alm_op_gemm_planes(ctx.h, ctypes.byref(a), ctypes.byref(b), ctypes.byref(e)))


@pytest.mark.parametrize('nsplit', [3, 1])
@pytest.mark.parametrize('shape', SHAPES, ids=lambda s: 'S%d_N%d_K%d_act%d%s%s' % (s[0], s[1], s[2], s[3],
                                                                                  '_resid' if s[4] else '',
                                                                                  '_split' if s[5] else ''))
def test_joint_linear_is_two_single_linears(ctx, shape, nsplit):
    from advancedliteratemachinery_b200 import _lib
    S, N, K, act, resid, split = shape
    g = torch.Generator().manual_seed(S * 7 + N * 3 + K)
    A = _planes(torch.randn(2 * S, K, generator=g)).cuda()
    W = _planes(torch.randn(2 * N, K, generator=g) * K ** -0.5).cuda()
    bias = torch.randn(2 * N, generator=g).cuda()
    res = torch.randn(2 * S, N, generator=g).cuda() if resid else None

    def run(batched):
        out = torch.full((2 * S, N), float('nan'), device='cuda')
        planes = torch.zeros(2, 2 * S * N, dtype=torch.bfloat16, device='cuda') if split else None

        def epi(h, obs0):
            e = _lib.GemmEpilogue()
            e.out_f32 = out.data_ptr() + 4 * h * S * N
            if split:
                e.out_hi = planes[0].data_ptr() + 2 * h * S * N
                e.out_lo = planes[1].data_ptr() + 2 * h * S * N
            e.ldo, e.obs0 = N, obs0
            e.bias, e.bias_mode, e.bias_bs0 = bias.data_ptr() + 4 * h * N, BIAS_COL, N if obs0 else 0
            if resid:
                e.resid, e.ldr, e.rbs0 = res.data_ptr() + 4 * h * S * N, N, S * N if obs0 else 0
            e.act, e.alpha = act, 1.0
            return e

        if batched:
            _call(ctx, _op(A, 0, S, K, 2, S * K), _op(W, 0, N, K, 2, N * K), epi(0, S * N))
        else:
            for h in range(2):
                _call(ctx, _op(A, h * S * K, S, K), _op(W, h * N * K, N, K), epi(h, 0))
        torch.cuda.synchronize()
        return out, planes

    with options(ctx, nsplit=nsplit):
        joint, joint_planes = run(True)
        single, single_planes = run(False)
    assert not torch.isnan(single).any()
    assert torch.equal(joint.view(torch.int32), single.view(torch.int32)), 'joint GEMM differs from the two single GEMMs'
    if split:
        assert torch.equal(joint_planes.view(torch.int16), single_planes.view(torch.int16))


def _wide(S, sms):
    return S * 8 <= 4 * sms  # the decoder's choice of the CTA-per-(sequence, head) kernel (sattn_wide on)


@pytest.mark.parametrize('t', [0, 13, 34])
@pytest.mark.parametrize('S', [1024, 512, 100])
def test_joint_self_attention_step_is_two_half_steps(ctx, S, t):
    """The joint pass runs the self-attention step once over both halves (2S sequences, both halves' caches at one
    Tmax) when each half alone takes the same kernel; every sequence's output and cache row must be what a launch over
    its half alone gives."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert _wide(S, sms) == _wide(2 * S, sms), 'the joint pass launches per half at this S'
    Tmax = 35
    g = torch.Generator().manual_seed(S + t)
    qkv = torch.randn(2 * S, 1536, generator=g).cuda()
    kc0 = torch.randn(2 * S, Tmax, 512, generator=g).cuda()
    vc0 = torch.randn(2 * S, Tmax, 512, generator=g).cuda()

    def step(rows):
        kc, vc = kc0.clone(), vc0.clone()
        out = torch.full((2 * S, 512), float('nan'), device='cuda')
        torch.cuda.synchronize()
        for r0 in rows:
            n = 2 * S if len(rows) == 1 else S
            ctx.check(ctx.lib.alm_op_self_attention_step(ctx.h, ctypes.c_void_p(qkv[r0].data_ptr()),
                                                         ctypes.c_void_p(kc[r0].data_ptr()),
                                                         ctypes.c_void_p(vc[r0].data_ptr()),
                                                         ctypes.c_void_p(out[r0].data_ptr()), n, t, Tmax))
        torch.cuda.synchronize()
        return out, kc, vc

    joint = step([0])
    halves = step([0, S])
    assert not torch.isnan(halves[0]).any()
    for a, b in zip(joint, halves):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))
