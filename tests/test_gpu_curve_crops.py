"""GPU: curved text rectified along the Bezier curves of its 16-point polygon (alm_pre_curve_crops) and recognition
straight from the pages (MGPSTRB200.recognize_polygons).  Bar: bit for bit against the reference fixture, the host
emulation of the kernels and the existing crop + recognise path; the quad path untouched."""
import numpy as np
import pytest
import torch

from tests.support import emu
from tests.test_curve_crops_cpu import bind, curve_fixture, curve_regions, emu_curve_crops
from tests.test_quad_crops_cpu import quad_fixture

pytestmark = pytest.mark.gpu
ALM_ERR_INVALID = -1


@pytest.mark.parametrize('on_device', [False, True])
def test_curve_crops_equal_fixture(on_device):
    from advancedliteratemachinery_b200 import _lib, preprocess as P
    z, pages, _, out = curve_fixture()
    ctx = _lib.Context(0)
    ims = [torch.from_numpy(p).cuda() for p in pages] if on_device else pages
    got = P.curve_crops(ctx, ims, z['polys'], z['page_index'])
    assert torch.equal(got.cpu().view(torch.int32), out.view(torch.int32))
    ctx.close()


def test_thousand_curved_regions_equal_host_emulation():
    """16 pages of 1024 x 1024, 64 curved regions each: every output bit equals the host run of the kernel bodies."""
    from advancedliteratemachinery_b200 import _lib, preprocess as P
    pages, polys, pidx = curve_regions(seed=7)
    _, _, ref = emu_curve_crops(emu('curve_emu', bind), pages, polys, pidx)
    ctx = _lib.Context(0)
    got = P.curve_crops(ctx, [torch.from_numpy(p).cuda() for p in pages], polys, pidx)
    assert np.array_equal(got.cpu().numpy().view(np.uint32), ref.view(np.uint32))
    ctx.close()


def test_launch_count_does_not_grow_with_regions():
    from advancedliteratemachinery_b200 import _lib, preprocess as P
    pages, polys, pidx = curve_regions(seed=3)
    dev = [torch.from_numpy(p).cuda() for p in pages]
    ctx = _lib.Context(0)
    counts = []
    for R in (1, 64, 1024):
        ctx.launch_count(reset=True)
        P.curve_crops(ctx, dev, polys[:R], pidx[:R])
        counts.append(ctx.launch_count())
    assert counts[0] == counts[1] == counts[2] == 3, counts
    ctx.close()


@pytest.mark.parametrize('nsplit', [3, 1])
def test_recognize_polygons_equals_crop_then_recognize(nsplit):
    from advancedliteratemachinery_b200 import MGPSTRB200, preprocess as P
    from tests.conftest import mgp_sd
    z, pages, crops, _ = curve_fixture()
    m = MGPSTRB200(mgp_sd(0))
    m.ctx.set_option('nsplit', nsplit)
    ref_ids, ref_prob = m.recognize(P.mgp_crops(m.ctx, crops))
    ids, prob = m.recognize_polygons(pages, z['polys'], z['page_index'])
    assert torch.equal(ids, ref_ids) and torch.equal(prob.view(torch.int32), ref_prob.view(torch.int32))
    ids, prob = m.recognize_polygons(pages, z['polys'].reshape(-1, 32), z['page_index'], max_batch=7)  # chunked
    assert torch.equal(ids, ref_ids) and torch.equal(prob.view(torch.int32), ref_prob.view(torch.int32))
    dicts = [{'polys': p.tolist()} for p in z['polys']]  # decode_pred_seq results
    ref_ids, ref_prob = m.recognize_topk(P.mgp_crops(m.ctx, crops), 4)
    ids, prob = m.recognize_polygons(pages, dicts, z['page_index'], k=4, max_batch=16)
    assert torch.equal(ids, ref_ids) and torch.equal(prob.view(torch.int32), ref_prob.view(torch.int32))
    ids, prob = m.recognize_polygons(pages, np.zeros((0, 16, 2)), [])
    assert ids.shape == (3, 0, 27)
    m.ctx.close()


def test_error_paths_leave_the_context_usable():
    from advancedliteratemachinery_b200 import _lib, preprocess as P
    z, pages, _, out = curve_fixture()
    ctx = _lib.Context(0)
    ctx.set_option('workspace_mb', 1024)  # below one crop at the largest size cv2.remap allows (3.2 GB)
    p = z['polys'][:2].copy()
    bad_nan = p.copy()
    bad_nan[1, 5, 0] = np.nan
    far = p + np.float32(1.1e6)
    xs = np.linspace(0, 30000, 8)
    huge = np.concatenate([np.stack([xs, np.zeros(8)], 1), np.stack([xs[::-1], np.full(8, 30000.0)], 1)])[None]
    cases = [(p, [0, 9], {}), (p, [-1, 0], {}), (bad_nan, [0, 0], {}), (far, [0, 0], {}), (p, [0, 0], {'imgH': 0}),
             (p, [0, 0], {'imgW': 0}), (huge.astype(np.float32), [0], {})]  # the last: a 2.7 GB crop, too large
    for polys, pidx, kw in cases:
        with pytest.raises(_lib.AlmError) as e:
            P.curve_crops(ctx, pages, polys, pidx, **kw)
        assert e.value.code == ALM_ERR_INVALID, (pidx, kw)
    assert 'region 0' in ctx.lib.alm_last_error(ctx.h).decode()  # the arena overflow names the region
    assert P.curve_crops(ctx, pages, np.zeros((0, 16, 2)), []).shape == (0, 3, 32, 128)
    got = P.curve_crops(ctx, pages, z['polys'], z['page_index'])
    assert torch.equal(got.cpu().view(torch.int32), out.view(torch.int32))
    ctx.close()


def test_quad_crops_unchanged_around_curve_crops():
    """Quad crops on the same context before and after curve crops stay bit-identical to the quad fixture."""
    from advancedliteratemachinery_b200 import _lib, preprocess as P
    zq, qpages, _, qout = quad_fixture()
    zc, cpages, _, cout = curve_fixture()
    ctx = _lib.Context(0)
    before = P.quad_crops(ctx, qpages, zq['quads'], zq['page_index'])
    curved = P.curve_crops(ctx, cpages, zc['polys'], zc['page_index'])
    after = P.quad_crops(ctx, qpages, zq['quads'], zq['page_index'])
    for got, want in ((before, qout), (curved, cout), (after, qout)):
        assert torch.equal(got.cpu().view(torch.int32), want.view(torch.int32))
    ctx.close()
