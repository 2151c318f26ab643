"""GPU: the two consumer schedules of the GEMM engine on problems that give CTAs several tiles or exactly one, against
fp64.

The op shapes of test_gpu_omniparser.py never give a CTA more than one tile, so the second consumer warpgroup never runs
a tile of its own there.  These shapes have more tiles than 2 x SMs with 3 or 4 tiles per CTA, M tails inside the second
64-row half and past it (the half that multiplies half 0's rows and stores nothing), a batched problem, narrow 32-column
tiles with up to 2 tiles per CTA, and launches whose CTAs all have one tile (the cooperative split) at both tile widths.
The column-group scatter epilogue is reached through alm_op_gemm (test_gpu_gemm_epilogue.py), and with the model's
cross-attention K / V cache geometry (a batched problem with many tiles per CTA at page scale) through
alm_op_gemm_planes (test_gpu_gemm_operands.py).
"""
import pytest
import torch

from tests.support import ctx, options

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)


WORKSPACE_MB = 4096


def _shapes():
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    m_blocks = (7 * sms + 7) // 8                  # x 2 column blocks x batch 2 = 3.5 tiles per CTA
    n128 = (sms // 2 - 1) // 5                      # 5 x n128 tiles of 128 columns < SMs / 2: 32-column tiles
    return [((m_blocks - 1) * 128 + 100, 200, 192, 1, 2),   # GELU, tail rows 64..99 of the last block, N tail
            ((3 * sms + 1) * 128 + 40, 128, 64, 0, 1),        # 3 or 4 tiles per CTA, one k-block, half 1 past M
            (4 * 128 + 40, n128 * 128 - 8, 320, 2, 1),        # 32-column tiles, 1 or 2 per CTA, ReLU
            (356, 600, 320, 2, 1),                            # 32-column tiles, one per CTA: cooperative
            (9 * 128 + 98, 10 * 128, 256, 1, 1)]              # 128-column tiles, one per CTA: cooperative


@pytest.mark.parametrize('case', range(5))
def test_gemm_schedules_match_fp64(ctx, case):
    M, N, K, act, batch = _shapes()[case]
    g = torch.Generator().manual_seed(M + N + K)
    A = torch.randn(batch, M, K, generator=g)
    Wt = torch.randn(batch, N, K, generator=g) / K ** 0.5
    b = torch.randn(N, generator=g)
    ref = torch.einsum('bmk,bnk->bmn', A.double(), Wt.double()) + b.double()
    ref = torch.nn.functional.gelu(ref) if act == 1 else (torch.relu(ref) if act == 2 else ref)
    Ad, Wd, bd = A.cuda(), Wt.cuda(), b.cuda()
    for nsplit, tol in ((3, 2e-5), (1, 6e-3)):
        with options(ctx, nsplit=nsplit):
            out = torch.full((batch, M, N), float('nan'), device='cuda')
            ctx.check(ctx.lib.alm_op_linear(ctx.h, Ad.data_ptr(), Wd.data_ptr(), bd.data_ptr(), out.data_ptr(), M, N, K,
                                            act, batch))
            got = out.cpu().double()
        rows_err = ((got - ref).norm(dim=2) / (ref.norm(dim=2) + 1e-30)).amax(dim=0)   # worst batch per row
        assert torch.isfinite(got).all(), nsplit
        assert float(rows_err.max()) < 10 * tol, (nsplit, int(rows_err.argmax()))
        assert float((got - ref).norm() / ref.norm()) < tol, nsplit
