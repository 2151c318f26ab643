"""CPU: caller character sets of the recognition loop (DESIGN 4.23) -- the sets and row sets check_rec_charset builds for
alm_omni_set_rec_charset, its refusals, and the restated reference loop (oracle/charset_ref.py) against
tests/golden/omni_charset.npz."""
import numpy as np
import pytest
import torch

from advancedliteratemachinery_b200.omniparser import DEFAULT_CHARS, check_rec_charset
from tests.support import golden

torch.set_grad_enabled(False)
CH = DEFAULT_CHARS


def test_a_string_is_one_set_for_every_row():
    allowed, rows = check_rec_charset('0123456789', CH)
    assert allowed.shape == (1, 95) and allowed.dtype == np.uint8 and rows is None
    assert ''.join(c for c, a in zip(CH, allowed[0]) if a) == '0123456789'
    assert check_rec_charset(None, CH) is None
    allowed, rows = check_rec_charset(CH, CH)   # the full set
    assert allowed.all()


def test_identical_sets_share_one_entry_in_first_appearance_order():
    allowed, rows = check_rec_charset(['12', 'AB', '21', 'AB', '1122', 'x'], CH, 6)
    assert allowed.shape == (3, 95)
    assert rows.dtype == np.int32 and rows.tolist() == [0, 1, 0, 1, 0, 2]
    names = [''.join(c for c, a in zip(CH, row) if a) for row in allowed]
    assert names == ['12', 'AB', 'x']


def test_none_rows_read_with_the_full_set_and_all_none_is_no_set():
    allowed, rows = check_rec_charset([None, '7', None], CH, 3)
    assert rows.tolist() == [0, 1, 0] and allowed[0].all() and allowed[1].sum() == 1
    assert check_rec_charset([None, None], CH, 2) is None
    assert check_rec_charset([], CH, 0) is None


@pytest.mark.parametrize('bad, rows, match', [
    ('', None, 'non-empty'),
    ('12é', None, 'outside the vocabulary'),
    ('\n', None, 'outside the vocabulary'),
    (['12'], None, 'non-empty string'),        # a sequence where one string is taken
    (7, None, 'non-empty string'),
    (['12', '3'], 3, 'one string or None per row'),
    (['12', ''], 2, r'rec_charset\[1\]'),
    (['12', 5], 2, r'rec_charset\[1\]'),
    (['1', 'ü'], 2, 'outside the vocabulary'),
])
def test_refusals(bad, rows, match):
    with pytest.raises(ValueError, match=match):
        check_rec_charset(bad, CH, rows)


def test_set_count_cap():
    from advancedliteratemachinery_b200 import _lib
    assert _lib.MAX_CHARSETS == 65536
    many = [CH[i % 95] + CH[(i // 95) % 95] + CH[(i // 9025) % 95] for i in range(3)]
    assert check_rec_charset(many, CH, 3)[0].shape == (3, 95)


def test_header_states_the_cap():
    import os
    here = os.path.dirname(os.path.abspath(__file__))
    with open(os.path.join(here, '..', 'include', 'alm_ocr.h')) as f:
        assert '#define ALM_MAX_CHARSETS 65536' in f.read()


def test_oracle_against_the_fixture():
    """The restated loop under digits, and with the full set, reproduces the fixture (ids exactly, probabilities to
    fp32 round-off); every returned text lies in its set."""
    from oracle import charset_ref as R
    from oracle import omniparser_ref as O
    from oracle import weights as W
    from oracle.gen_golden import OMNI_CASES, omni_inputs
    gold = golden('omni_charset.npz')
    case = OMNI_CASES['full']
    sd = W.omniparser_state_dict(seed=case['wseed'], pt_eos_bias=case['pt_eos_bias'])
    img, mask = omni_inputs(case)
    mem, pos, kpm, _ = O.encode(img, mask, sd)
    pts = torch.from_numpy(gold['decode_pts'])
    for name in ('digits', 'full'):
        text = dict(zip(gold['set_names'].tolist(), gold['sets'].tolist()))[name] or None
        cs = R.charset_mask(text).expand(len(pts), -1)
        rec, probs, gaps = R.rec_loop(mem[0], kpm[0], pos[0], sd, pts, case['rec_length'], cs)
        assert np.array_equal(rec.numpy(), gold[f'decode_{name}_rec']), name
        np.testing.assert_allclose(probs.numpy(), gold[f'decode_{name}_probs'], rtol=1e-5, atol=1e-7)
        assert float(gaps.min()) >= 1e-4
        if text:
            assert set(''.join(R.rec_text(r) for r in rec)) <= set(text)
    for key in ('decode_digits', 'decode_upper', 'decode_three', 'at', 'kie'):
        assert float(gold[f'{key}_min_gap']) >= 1e-4, key
    for r, (t, none) in zip(gold['at_rec'], zip(gold['at_sets'].tolist(), gold['at_none'].tolist())):
        if not none:
            assert set(R.rec_text(r)) <= set(t)


def test_allowed_classes_keep_unknown_pad_and_end():
    from oracle import charset_ref as R
    from oracle import weights as W
    V = W.REC_EOS + 5
    a = R.allowed_classes(V, R.charset_mask('0').reshape(1, -1))[0]
    assert a[W.NUM_BINS + W.CHARS.index('0')] and a[W.RECOG_PAD - 1] and a[W.RECOG_PAD] and a[W.REC_EOS]
    assert int(a.sum()) == 4
