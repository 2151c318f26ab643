"""GPU: perspective crops of detected text regions (alm_pre_quad_crops) and recognition straight from the pages
(MGPSTRB200.recognize_regions).  Bar: bit for bit against the reference fixture, the host emulation of the kernels
and the existing crop + recognise path."""
import numpy as np
import pytest
import torch

from tests.support import emu
from tests.test_quad_crops_cpu import bind, emu_quad_crops, quad_fixture, text_regions

pytestmark = pytest.mark.gpu
ALM_ERR_INVALID = -1


@pytest.mark.parametrize('on_device', [False, True])
def test_quad_crops_equal_fixture(on_device):
    from advancedliteratemachinery_b200 import _lib, preprocess as P
    z, pages, _, out = quad_fixture()
    ctx = _lib.Context(0)
    ims = [torch.from_numpy(p).cuda() for p in pages] if on_device else pages
    got = P.quad_crops(ctx, ims, z['quads'], z['page_index'])
    assert torch.equal(got.cpu().view(torch.int32), out.view(torch.int32))
    ctx.close()


def test_thousand_regions_equal_host_emulation():
    """16 pages of 1024 x 1024, 64 regions each: every output bit equals the host run of the kernel bodies."""
    from advancedliteratemachinery_b200 import _lib, preprocess as P
    pages, quads, pidx = text_regions(seed=7)
    _, _, ref = emu_quad_crops(emu('quad_emu', bind), pages, quads, pidx)
    ctx = _lib.Context(0)
    got = P.quad_crops(ctx, [torch.from_numpy(p).cuda() for p in pages], quads, pidx)
    assert np.array_equal(got.cpu().numpy().view(np.uint32), ref.view(np.uint32))
    ctx.close()


def test_launch_count_does_not_grow_with_regions():
    from advancedliteratemachinery_b200 import _lib, preprocess as P
    pages, quads, pidx = text_regions(seed=3)
    dev = [torch.from_numpy(p).cuda() for p in pages]
    ctx = _lib.Context(0)
    counts = []
    for R in (1, 64, 1024):
        ctx.launch_count(reset=True)
        P.quad_crops(ctx, dev, quads[:R], pidx[:R])
        counts.append(ctx.launch_count())
    assert counts[0] == counts[1] == counts[2] == 3, counts
    ctx.close()


@pytest.mark.parametrize('nsplit', [3, 1])
def test_recognize_regions_equals_crop_then_recognize(nsplit):
    from advancedliteratemachinery_b200 import MGPSTRB200, preprocess as P
    from tests.conftest import mgp_sd
    z, pages, crops, _ = quad_fixture()
    m = MGPSTRB200(mgp_sd(0))
    m.ctx.set_option('nsplit', nsplit)
    ref_ids, ref_prob = m.recognize(P.mgp_crops(m.ctx, crops))
    ids, prob = m.recognize_regions(pages, z['quads'], z['page_index'])
    assert torch.equal(ids, ref_ids) and torch.equal(prob.view(torch.int32), ref_prob.view(torch.int32))
    ids, prob = m.recognize_regions(pages, z['quads'], z['page_index'], max_batch=7)  # chunked
    assert torch.equal(ids, ref_ids) and torch.equal(prob.view(torch.int32), ref_prob.view(torch.int32))
    ref_ids, ref_prob = m.recognize_topk(P.mgp_crops(m.ctx, crops), 4)
    ids, prob = m.recognize_regions(pages, z['quads'], z['page_index'], k=4, max_batch=16)
    assert torch.equal(ids, ref_ids) and torch.equal(prob.view(torch.int32), ref_prob.view(torch.int32))
    ids, prob = m.recognize_regions(pages, np.zeros((0, 4, 2)), [])
    assert ids.shape == (3, 0, 27)
    m.ctx.close()


def test_error_paths_leave_the_context_usable():
    from advancedliteratemachinery_b200 import _lib, preprocess as P
    z, pages, _, out = quad_fixture()
    ctx = _lib.Context(0)
    q = z['quads'][:2].copy()
    bad_nan = q.copy()
    bad_nan[1, 2, 0] = np.nan
    huge = np.array([[[0, 0], [200000, 0], [200000, 50000], [0, 50000]]], np.float32)  # 30 GB crop
    cases = [(q, [0, 3], {}), (q, [-1, 0], {}), (bad_nan, [0, 0], {}), (q, [0, 0], {'imgH': 0}),
             (q, [0, 0], {'imgW': 0}), (huge, [0], {})]
    for quads, pidx, kw in cases:
        with pytest.raises(_lib.AlmError) as e:
            P.quad_crops(ctx, pages, quads, pidx, **kw)
        assert e.value.code == ALM_ERR_INVALID, (pidx, kw)
    assert 'region 0' in ctx.lib.alm_last_error(ctx.h).decode()  # the arena overflow names the region
    assert P.quad_crops(ctx, pages, np.zeros((0, 4, 2)), []).shape == (0, 3, 32, 128)
    got = P.quad_crops(ctx, pages, z['quads'], z['page_index'])
    assert torch.equal(got.cpu().view(torch.int32), out.view(torch.int32))
    ctx.close()
