"""GPU: spotted words grouped into text lines (alm_omni_group_lines, omniparser.group_lines,
OmniParserB200.group_lines).  The device must equal tests/golden/omni_groups.npz (oracle/group_ref.py on synthetic
layouts) and the host build of the same bodies (tests/emu/group_emu.cpp) exactly, line polygons bit for bit; it must
be reproducible run to run, take the same number of launches whatever the counts, refuse bad arguments before any
device work, chain after spot_tiled without changing it, and hand its line polygons over to preprocess.curve_crops."""
import numpy as np
import pytest
import torch

from tests.support import assert_same, ctx, emu, golden
from tests.test_groups_cpu import bind

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

OUTPUTS = ('n_lines', 'line_offset', 'line_first', 'line_words', 'order', 'line_of', 'rank_of', 'line_polys')
PARAMS = ('cos_tol', 'height_ratio', 'max_offset', 'max_overlap', 'max_gap')
NAMES = ['paragraph', 'paragraph_rot7', 'paragraph_rot30', 'columns_3h', 'columns_1h', 'heading', 'arc', 'circle',
         'interleave', 'mutual', 'overlap', 'ties', 'degenerate', 'single', 'empty', 'all', 'tiles']
ALM_ERR_INVALID = -1


@pytest.fixture(scope='module')
def gold():
    return golden('omni_groups.npz')


def emu_group(polys, count, offset, **params):
    """alm_omni_group_lines' five launches as host code (tests/emu/group_emu.cpp) -> the dict group_lines returns."""
    from advancedliteratemachinery_b200.omniparser import check_group_args
    lib = emu('group_emu', bind)
    prm = check_group_args(**params)
    polys = np.ascontiguousarray(polys, np.float64).reshape(-1, 32)
    count, offset = np.ascontiguousarray(count, np.int32), np.ascontiguousarray(offset, np.int32)
    N, P = len(polys), len(count)
    out = dict(n_lines=np.zeros(P, np.int32), line_offset=np.zeros(P, np.int32), line_first=np.zeros(N, np.int32),
               line_words=np.zeros(N, np.int32), order=np.zeros(N, np.int32), line_of=np.zeros(N, np.int32),
               rank_of=np.zeros(N, np.int32), line_polys=np.zeros((N, 32)))
    K = lib.emu_group_lines(P, count.ctypes.data, offset.ctypes.data, polys.ctypes.data, *[prm[k] for k in PARAMS],
                            *[out[k].ctypes.data for k in OUTPUTS])
    for k in ('line_first', 'line_words', 'line_polys'):
        out[k] = out[k][:K]
    return out


def pages_call(pages):
    count = np.array([len(p) for p in pages], np.int32)
    return np.concatenate(pages), count, (np.cumsum(count) - count).astype(np.int32)


@pytest.mark.parametrize('name', NAMES)
def test_device_equals_the_golden(ctx, gold, name):
    from advancedliteratemachinery_b200.omniparser import group_lines
    got = group_lines(ctx, gold[f'{name}_polys'], gold[f'{name}_count'], gold[f'{name}_offset'],
                      **dict(zip(PARAMS, gold[f'{name}_params'].tolist())))
    assert_same(got, {k: gold[f'{name}_{k}'] for k in OUTPUTS})


def test_device_equals_the_emulation_at_scale_and_is_reproducible(ctx):
    """One page of 4096 words; 16 pages of unequal counts, three of them empty; under the proposed parameters and
    under others.  Two runs of the same call give the same bits."""
    from advancedliteratemachinery_b200.omniparser import group_lines
    from oracle.gen_golden_groups import random_page
    rng = np.random.default_rng(17)
    big = pages_call([random_page(rng, 4096)])
    counts = [700, 0, 1, 129, 128, 0, 1500, 40, 2, 511, 0, 300, 64, 127, 1000, 33]
    many = pages_call([random_page(rng, n) if n else np.zeros((0, 32)) for n in counts])
    for call in (big, many):
        for prm in ({}, dict(cos_tol=0.7, height_ratio=0.3, max_offset=0.8, max_overlap=1.0, max_gap=2.5)):
            got = group_lines(ctx, *call, **prm)
            assert_same(got, emu_group(*call, **prm))
            assert_same(got, group_lines(ctx, *call, **prm))
            assert 0 < int(got['n_lines'].sum()) < len(call[0]) // 2
    assert group_lines(ctx, *many)['n_lines'][[1, 5, 10]].tolist() == [0, 0, 0]


def test_the_launch_count_does_not_depend_on_the_counts(ctx):
    from advancedliteratemachinery_b200.omniparser import group_lines
    from oracle.gen_golden_groups import random_page
    rng = np.random.default_rng(2)
    launches = []
    for pages in ([random_page(rng, 1)], [random_page(rng, 4096)], [random_page(rng, 300)] * 7):
        ctx.launch_count(reset=True)
        group_lines(ctx, *pages_call(pages))
        launches.append(ctx.launch_count())
    assert launches == [5, 5, 5]
    ctx.launch_count(reset=True)
    assert group_lines(ctx, np.zeros((0, 32)), [0, 0], [0, 0])['n_lines'].tolist() == [0, 0]
    assert ctx.launch_count() == 0


def test_invalid_arguments_are_named_and_leave_the_context_usable(ctx, gold):
    """Every refusal is ALM_ERR_INVALID with the argument's name in the message, and the very next valid call on the
    same context is correct."""
    from advancedliteratemachinery_b200.omniparser import GROUP_DEFAULTS, group_lines
    polys = np.ascontiguousarray(gold['all_polys'])
    N = len(polys)
    want = {k: gold[f'all_{k}'] for k in OUTPUTS}
    prm = dict(zip(PARAMS, gold['all_params'].tolist()))

    def call(**over):
        a = dict(n_pages=len(gold['all_count']), page_count=gold['all_count'].copy(), page_offset=gold['all_offset'].copy(),
                 polys=polys, cap=N, **GROUP_DEFAULTS)
        a.update({k: np.zeros(N * (32 if k == 'line_polys' else 1), np.float64 if k == 'line_polys' else np.int32)
                  for k in OUTPUTS})
        a.update(over)
        ptr = {k: (None if a[k] is None else a[k].ctypes.data) for k in ('page_count', 'page_offset', 'polys') + OUTPUTS}
        rc = ctx.lib.alm_omni_group_lines(ctx.h, a['n_pages'], ptr['page_count'], ptr['page_offset'], ptr['polys'],
                                          *[a[k] for k in PARAMS], *[ptr[k] for k in OUTPUTS], a['cap'])
        return rc, ctx.lib.alm_last_error(ctx.h).decode()

    def edited(key, index, value):
        v = gold[f'all_{key}'].copy()
        v[index] = value
        return v

    bad = [('n_pages', dict(n_pages=0)), ('page_count', dict(page_count=None)), ('page_offset', dict(page_offset=None)),
           ('page_count', dict(page_count=edited('count', 2, -1))),
           ('page_offset', dict(page_offset=edited('offset', 3, int(gold['all_offset'][3]) - 1))),
           ('page_offset', dict(page_offset=edited('offset', 13, N))),
           ('page_offset', dict(page_offset=edited('offset', 1, -5))),
           ('polys', dict(polys=None)), ('cap', dict(cap=N - 1)),
           ('cos_tol', dict(cos_tol=1.01)), ('cos_tol', dict(cos_tol=float('nan'))),
           ('height_ratio', dict(height_ratio=-0.01)), ('height_ratio', dict(height_ratio=1.5)),
           ('max_offset', dict(max_offset=-1.0)), ('max_overlap', dict(max_overlap=float('inf'))),
           ('max_gap', dict(max_gap=float('nan')))] + [(k, {k: None}) for k in OUTPUTS]
    for name, over in bad:
        rc, msg = call(**over)
        assert rc == ALM_ERR_INVALID and name in msg, (name, rc, msg)
        assert_same(group_lines(ctx, polys, gold['all_count'], gold['all_offset'], **prm), want)
    assert call()[0] == 0


def test_grouping_chains_after_spot_tiled_and_leaves_it_unchanged():
    """spot_tiled on the tiles fixture's page, then group_lines: the oracle applied to the same merged polygons; the
    spotting result is what it was, before and after."""
    from advancedliteratemachinery_b200 import OmniParserB200, OmniVocab
    from advancedliteratemachinery_b200.omniparser import group_lines
    from oracle import group_ref as R
    from tests.conftest import omni_sd
    t = golden('omni_tiles.npz')
    m = OmniParserB200(omni_sd(int(t['wseed']), float(t['pt_eos_bias'])),
                       OmniVocab(pt_seq_length=int(t['pt_seq_length']), rec_length=int(t['rec_length'])), workspace_mb=4096)
    try:
        kw = dict(tile=int(t['tile']), overlap=int(t['overlap']), test_min_size=int(t['test_min_size']),
                  test_max_size=int(t['test_max_size']))
        small = np.random.default_rng(5).integers(0, 256, (100, 90, 3), dtype=np.uint8)
        res = m.spot_tiled([t['page'], small], **kw)
        before = repr(res)
        mg = m.last_tiles['merged']
        assert np.array_equal(mg['polys'][:int(mg['count'][0])], t['merged_polys'])
        for prm in ({}, dict(cos_tol=-1.0, height_ratio=0.0, max_offset=50.0, max_overlap=50.0, max_gap=50.0)):
            want = R.group_lines(mg['polys'], mg['count'], mg['offset'], **prm)
            assert_same(group_lines(m.ctx, mg['polys'], mg['count'], mg['offset'], **prm), want)
            lines = m.group_lines(res, **prm)
            assert [len(p) for p in lines] == want['n_lines'].tolist()
            for p, page in enumerate(lines):
                assert sorted(i for ln in page for i in ln['words']) == list(range(len(res[p])))
                for ln in page:
                    assert ln['rec'] == ' '.join(res[p][i]['rec'] for i in ln['words'])
                    assert ln['score'] == sum(res[p][i]['score'] for i in ln['words']) / len(ln['words'])
            l0 = int(want['line_offset'][1])
            assert lines[1][0]['polys'] == want['line_polys'][l0].reshape(16, 2).tolist()
        assert len(want['line_words']) < len(mg['polys'])   # the loose parameters join words of this page
        assert repr(res) == before and repr(m.spot_tiled([t['page'], small], **kw)) == before
        assert m.group_lines([None, []]) == [[], []]
    finally:
        m.ctx.close()


def test_line_polygons_feed_curve_crops(ctx, gold):
    """The hand-over to recognize_lines: the paragraph's (also the rotated one's and the arc's) line polygons go
    through preprocess.curve_crops, one crop per line, finite."""
    from advancedliteratemachinery_b200 import preprocess as P
    page = np.random.default_rng(1).integers(0, 256, (800, 1800, 3), dtype=np.uint8)
    for name in ('paragraph', 'paragraph_rot7', 'arc'):
        lp = gold[f'{name}_line_polys']
        crops = P.curve_crops(ctx, [page], lp.reshape(-1, 16, 2), np.zeros(len(lp), np.int32))
        assert crops.shape == (len(lp), 3, 32, 128)
        assert bool(torch.isfinite(crops).all()) and float(crops.max()) <= 1.0 and float(crops.std()) > 0.01
