"""Spotted words grouped into text lines: CPU checks of the grouping kernels' bodies run on the host
(tests/emu/group_emu.cpp) against oracle/group_ref.py, bit for bit, on tests/golden/omni_groups.npz (synthetic layouts
by oracle/gen_golden_groups.py) and on random pages; the lines the named fixtures must give, spelled out here; the
structural properties of any grouping; and the host-side Python (line_results, argument validation)."""
import ctypes as C
import math
import os

import numpy as np
import pytest

from tests.support import assert_same, emu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
OUTPUTS = ('n_lines', 'line_offset', 'line_first', 'line_words', 'order', 'line_of', 'rank_of', 'line_polys')
PARAMS = ('cos_tol', 'height_ratio', 'max_offset', 'max_overlap', 'max_gap')


def bind(lib):
    """Bind tests/emu/group_emu.cpp (host compile of the grouping kernels' bodies)."""
    lib.emu_group_lines.restype = C.c_long
    lib.emu_group_lines.argtypes = [C.c_int] + [C.c_void_p] * 3 + [C.c_double] * 5 + [C.c_void_p] * 8


def emu_group(polys, count, offset, **params):
    """alm_omni_group_lines' five launches on the host -> the dict group_lines / group_ref.group_lines return."""
    from oracle import group_ref as R
    lib = emu('group_emu', bind)
    prm = dict(R.DEFAULTS, **params)
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


def gold():
    return np.load(os.path.join(GOLD, 'omni_groups.npz'))


def gold_case(g, name):
    return (g[f'{name}_polys'], g[f'{name}_count'], g[f'{name}_offset']), dict(zip(PARAMS, g[f'{name}_params'].tolist()))


def lines_of(res, page=0):
    """The lines of one page as lists of word rows."""
    first, n = int(res['line_offset'][page]), int(res['n_lines'][page])
    return [res['order'][res['line_first'][l]:res['line_first'][l] + res['line_words'][l]].tolist()
            for l in range(first, first + n)]


def test_golden_has_every_fixture():
    assert gold()['names'].tolist() == [
        'paragraph', 'paragraph_rot7', 'paragraph_rot30', 'columns_3h', 'columns_1h', 'heading', 'arc', 'circle',
        'interleave', 'mutual', 'overlap', 'ties', 'degenerate', 'single', 'empty', 'all', 'tiles']


@pytest.mark.parametrize('name', ['paragraph', 'paragraph_rot7', 'paragraph_rot30', 'columns_3h', 'columns_1h',
                                  'heading', 'arc', 'circle', 'interleave', 'mutual', 'overlap', 'ties', 'degenerate',
                                  'single', 'empty', 'all', 'tiles'])
def test_emulation_equals_the_golden(name):
    g = gold()
    args, prm = gold_case(g, name)
    assert_same(emu_group(*args, **prm), {k: g[f'{name}_{k}'] for k in OUTPUTS})


def test_regenerating_the_golden_reproduces_the_file():
    from oracle import gen_golden_groups as G
    g, new = gold(), G.golden()
    assert sorted(g.files) == sorted(new)
    for k in new:
        a, b = g[k], np.asarray(new[k])
        assert a.dtype == b.dtype and a.shape == b.shape, k
        assert a.tobytes() == b.tobytes(), k


def check_structure(polys, count, offset, res, prm):
    """Every word in exactly one line, ranks 0 .. len - 1 once each, order a permutation of each page's rows, every
    consecutive pair of a line a successor candidate, line polygon ends = the end words' corners."""
    from oracle import group_ref as R
    N = len(polys)
    assert sorted(res['order'].tolist()) == list(range(N))
    assert int(res['line_words'].sum()) == N and (res['line_words'] >= 1).all()
    assert res['line_offset'].tolist() == (np.cumsum(res['n_lines']) - res['n_lines']).tolist()
    for p in range(len(count)):
        rows = res['order'][offset[p]:offset[p] + count[p]]
        assert sorted(rows.tolist()) == list(range(offset[p], offset[p] + count[p]))
        heads = []
        for l, words in enumerate(lines_of(res, p), int(res['line_offset'][p])):
            assert res['line_of'][words].tolist() == [l] * len(words)
            assert res['rank_of'][words].tolist() == list(range(len(words)))
            fr = [R.frame([float(v) for v in polys[w]]) for w in words]
            for a, b in zip(fr, fr[1:]):
                assert R.candidate(a, b, prm) is not None
            heads.append((fr[0]['L'][1], fr[0]['L'][0], words[0]))
            lp, a, b = res['line_polys'][l], polys[words[0]], polys[words[-1]]
            if fr[0]['ok']:
                ends = np.concatenate([a[0:2], b[14:16], b[16:18], a[30:32]])
                assert np.array_equal(lp[[0, 1, 14, 15, 16, 17, 30, 31]], ends)
            else:
                assert len(words) == 1 and lp.tobytes() == a.tobytes()
        assert heads == sorted(heads)


def test_random_pages_emulation_equals_the_oracle_and_is_well_formed():
    """200 random pages (1 to 600 words, any rotation, heights 8 to 60 px, displaced / duplicated / non-finite words),
    some grouped several pages per call and with other parameters."""
    from oracle import gen_golden_groups as G
    from oracle import group_ref as R
    rng = np.random.default_rng(3)
    pages = [G.random_page(rng, int(n)) for n in np.concatenate([[1, 2, 600], rng.integers(1, 600, 197)])]
    at = words = joined = 0
    while at < len(pages):
        k = int(rng.integers(1, 5))
        chunk = pages[at:at + k] + ([np.zeros((0, 32))] if at % 3 == 0 else [])
        at += k
        count = np.array([len(p) for p in chunk], np.int32)
        offset = (np.cumsum(count) - count).astype(np.int32)
        polys = np.concatenate(chunk)
        prm = {} if at % 2 else dict(cos_tol=float(rng.uniform(0.5, 1)), height_ratio=float(rng.uniform(0, 1)),
                                     max_offset=float(rng.uniform(0, 1)), max_overlap=float(rng.uniform(0, 1)),
                                     max_gap=float(rng.uniform(0, 3)))
        res = emu_group(polys, count, offset, **prm)
        assert_same(res, R.group_lines(polys, count, offset, **prm))
        check_structure(polys, count, offset, res, dict(R.DEFAULTS, **prm))
        if not prm:
            words += len(polys)
            joined += len(polys) - int(res['n_lines'].sum())
    assert joined > words // 2   # under the proposed parameters most words of these pages continue a line


def partition(res, page=0):
    return sorted(sorted(ln) for ln in lines_of(res, page))


def by_truth(truth, merge=lambda t: t):
    groups = {}
    for i, t in enumerate(truth.tolist()):
        groups.setdefault(merge(t), []).append(i)
    return sorted(groups.values())


def centre_x(polys, rows):
    return [float(polys[r].reshape(16, 2)[:, 0].mean()) for r in rows]


def test_named_fixtures_give_the_lines_they_were_laid_out_on():
    """The expected lines, from the layout and not from the oracle, so the golden cannot encode a wrong rule."""
    g = gold()
    res = {n: {k: g[f'{n}_{k}'] for k in OUTPUTS} for n in g['names'].tolist()}
    # paragraphs, also rotated: the 12 rows, top to bottom, each left to right
    for name, deg in (('paragraph', 0.0), ('paragraph_rot7', 7.0), ('paragraph_rot30', 30.0)):
        lines, truth = lines_of(res[name]), g[f'{name}_truth']
        assert [sorted(set(truth[ln].tolist())) for ln in lines] == [[r] for r in range(12)]
        assert partition(res[name]) == by_truth(truth)
        c, s = math.cos(math.radians(deg)), math.sin(math.radians(deg))
        for ln in lines:   # left to right along the text direction
            along = [float((g[f'{name}_polys'][w].reshape(16, 2) @ [c, s]).mean()) for w in ln]
            assert along == sorted(along)
    # a 3 h gutter is never crossed; a 1 h gutter is: the rows run through both columns
    assert partition(res['columns_3h']) == by_truth(g['columns_3h_truth'])
    assert partition(res['columns_1h']) == by_truth(g['columns_1h_truth'], lambda t: t // 2)
    for ln in lines_of(res['columns_1h']):
        x = centre_x(g['columns_1h_polys'], ln)
        assert len(ln) == 6 and x == sorted(x)
    # the heading, the footnote number behind it and the body rows are apart, in that order
    truth = g['heading_truth']
    assert [sorted(set(truth[ln].tolist())) for ln in lines_of(res['heading'])] == [[0], [1], [2], [3], [4]]
    assert partition(res['heading']) == by_truth(truth)
    # the arc is one line, left to right; its polygon is curved: the middle of the top boundary lies above its ends
    (ln,) = lines_of(res['arc'])
    x = centre_x(g['arc_polys'], ln)
    assert len(ln) == 9 and x == sorted(x)
    lp = res['arc']['line_polys'][0].reshape(16, 2)
    assert lp[3, 1] < min(lp[0, 1], lp[7, 1]) - 100 and lp[12, 1] < min(lp[8, 1], lp[15, 1]) - 100
    assert np.all(np.diff(lp[:8, 0]) > 0) and np.all(np.diff(lp[8:, 0]) < 0)
    # the circle is one line that starts at row 0 and runs clockwise: the generator put row k at position pos[k]
    pos = [5, 9, 0, 3, 11, 7, 1, 8, 4, 10, 2, 6]
    assert lines_of(res['circle']) == [[pos.index((pos[0] + t) % 12) for t in range(12)]]
    # two lines 1.2 h apart whose words interleave in x stay apart
    assert lines_of(res['interleave']) == [[0, 2, 4, 6, 8], [1, 3, 5, 7, 9]]
    # C is the best successor of A and of B and joins B; A's line ends, its other candidate E stays alone
    assert lines_of(res['mutual']) == [[1, 2, 3], [0], [4]]
    # gap 0 and an overlap of 0.3 h join, an overlap of 0.7 h does not
    assert lines_of(res['overlap']) == [[0, 1, 2], [3, 4]]
    # equal keys: the lower row wins as successor and as predecessor
    assert lines_of(res['ties']) == [[0, 1], [2], [3]]
    # degenerate words are lines of their own and keep their polygon; the row around them is one line
    assert sorted(lines_of(res['degenerate'])) == [[0, 2, 5], [1], [3], [4]]
    assert lines_of(res['degenerate'])[-1] == [4]   # the NaN word comes last
    assert lines_of(res['single']) == [[0]] and res['empty']['n_lines'].tolist() == [0]
    # all pages in one call: every page as on its own (the circle closes under the call's wider cos_tol)
    names = [n for n in g['names'].tolist() if n not in ('all', 'tiles')]
    off = g['all_offset']
    for p, n in enumerate(names):
        want = lines_of(res[n])
        assert [[w - int(off[p]) for w in ln] for ln in lines_of(res['all'], p)] == want, n


def test_parameters_move_the_fixtures_they_pin():
    g = gold()

    def regroup(name, **prm):
        return lines_of(emu_group(g[f'{name}_polys'], g[f'{name}_count'], g[f'{name}_offset'], **prm))
    assert len(regroup('circle')) == 12                                    # 30 degrees between neighbours > 15
    assert len(regroup('columns_3h', max_gap=4.0)) == 8
    assert len(regroup('columns_1h', max_gap=0.8)) == 16
    assert len(regroup('heading', height_ratio=0.3)) == 4                  # the footnote number joins the heading
    assert len(regroup('interleave', max_offset=1.3)) == 1
    assert regroup('overlap', max_overlap=0.8) == [[0, 1, 2, 3, 4]]
    assert regroup('overlap', max_overlap=0.2) == [[0, 1], [2], [3, 4]]


def test_line_results_joins_and_scores():
    from advancedliteratemachinery_b200 import postprocess as Post
    g = gold()
    groups = {k: g[f'mutual_{k}'] for k in OUTPUTS}
    words = [{'rec': t, 'score': s, 'polys': g['mutual_polys'][i].reshape(16, 2).tolist()}
             for i, (t, s) in enumerate(zip('ABCDE', (0.5, 0.25, 0.75, 0.5, 1.0)))]
    (lines,) = Post.line_results([words], [0], groups)
    assert [ln['words'] for ln in lines] == [[1, 2, 3], [0], [4]]
    assert [ln['rec'] for ln in lines] == ['B C D', 'A', 'E']
    assert [ln['score'] for ln in lines] == [0.5, 0.5, 1.0]
    assert lines[0]['polys'] == g['mutual_line_polys'][0].reshape(16, 2).tolist()
    # two pages, the second one's rows start at 5; a page without words has no lines
    both = {k: g[f'all_{k}'] for k in OUTPUTS}
    pages = [[{'rec': str(i)} for i in range(int(c))] for c in g['all_count']]
    out = Post.line_results(pages, g['all_offset'], both)
    assert [len(o) for o in out] == g['all_n_lines'].tolist() and out[14] == []
    assert sorted(i for ln in out[3] for i in ln['words']) == list(range(int(g['all_count'][3])))


def test_wrapper_refuses_bad_arguments_before_any_call():
    from advancedliteratemachinery_b200 import omniparser as O
    polys = np.zeros((3, 32))
    for bad in (dict(cos_tol=1.5), dict(cos_tol=float('nan')), dict(height_ratio=-0.1), dict(height_ratio=2),
                dict(max_offset=-1), dict(max_overlap=float('inf')), dict(max_gap=float('nan')), dict(max_gaps=1)):
        with pytest.raises(ValueError):
            O.group_lines(None, polys, [3], [0], **bad)
    with pytest.raises(ValueError):
        O.group_lines(None, polys, [2], [0])
    with pytest.raises(ValueError):
        O.group_lines(None, polys, [3], [0, 0])
    assert O.check_group_args(max_gap=2)['max_gap'] == 2.0 and O.check_group_args()['cos_tol'] == math.cos(math.radians(15))
