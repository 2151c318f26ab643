"""Caller character sets in the recognition loop -> tests/golden/omni_charset.npz.

TEST INFRASTRUCTURE ONLY -- runs on the CPU in the build container.

    python -m oracle.gen_golden_charset

oracle/charset_ref.rec_loop restates the reference's greedy recognition loop (model/transformer.py:266-283; KIE
:171-186) with the set's mask applied after the reference's own zeroing.  Cases, on the synthetic checkpoints and pages
of oracle/gen_golden:
  * decode_*   the 'full' page's decoded points read under digits, upper case, a three-character set and the full set;
  * at_*       four points of the 'full' page read at once, each with its own set (one of them unconstrained);
  * kie_*      the KIE page's (x, y) pairs under digits.
Every greedy step must clear gen_golden.GAP_FLOOR within its allowed set.  The restatement under the full set must
equal the unconstrained restatement (oracle/omniparser_ref), and, where the reference checkout is present, the
reference's own loops on the same points (oracle/gen_golden_points).
"""
from __future__ import annotations

import os
import tempfile

import numpy as np
import torch

from oracle.gen_golden import GAP_FLOOR, GOLD, KIE_CASES, OMNI_CASES, REF, omni_inputs

SETS = {'digits': '0123456789', 'upper': 'ABCDEFGHIJKLMNOPQRSTUVWXYZ', 'three': 'oaU', 'full': None}
AT_SETS = ['0123456789', None, 'ABCDEFGHIJKLMNOPQRSTUVWXYZ0123456789', '.,-/0123456789']


def _check_gaps(what, gaps):
    g = float(gaps.min())
    assert g >= GAP_FLOOR, (what, g, 'near-tie within the allowed set: pick another set or point')
    return g


def gen_charset():
    from oracle import charset_ref as R
    from oracle import omniparser_ref as O
    from oracle import weights as W
    gold = {}
    # ---- decode: the 'full' page's own points under each set
    case = OMNI_CASES['full']
    sd = W.omniparser_state_dict(seed=case['wseed'], pt_eos_bias=case['pt_eos_bias'])
    img, mask = omni_inputs(case)
    mem, pos, kpm, _ = O.encode(img, mask, sd)
    res = O.greedy_text_spotting(mem[0], kpm[0], pos[0], sd, O.default_prompts(True)[0], case['pt_seq_length'],
                                 case['rec_length'])
    pts = res[0][0].reshape(-1, 2)
    n = pts.shape[0]
    for name, text in SETS.items():
        cs = R.charset_mask(text).expand(n, -1)
        rec, probs, gaps = R.rec_loop(mem[0], kpm[0], pos[0], sd, pts, case['rec_length'], cs)
        g = _check_gaps(f'decode_{name}', gaps)
        if text is None:   # the full set is the unconstrained loop, bit for bit
            assert torch.equal(rec, res[0][2][0]) and torch.equal(probs, res[1][0]), 'full set != no set'
        else:
            assert all(c in text for c in ''.join(R.rec_text(r) for r in rec)), name
        gold.update({f'decode_{name}_rec': rec.numpy(), f'decode_{name}_probs': probs.numpy(),
                     f'decode_{name}_min_gap': np.array(g)})
        print(f'omni_charset decode {name}: {[R.rec_text(r) for r in rec]}  smallest gap {g:.2e}')
    gold['decode_pts'] = pts.numpy()
    gold['sets'] = np.array([SETS[k] or '' for k in SETS])
    gold['set_names'] = np.array(list(SETS))
    # ---- read_at: four points, each with its own set
    apts = torch.tensor([(120, 340), (880, 610), (455, 95), (610, 900)], dtype=torch.long)
    cs = torch.stack([R.charset_mask(t) for t in AT_SETS])
    rec, probs, gaps = R.rec_loop(mem[0], kpm[0], pos[0], sd, apts, case['rec_length'], cs)
    g = _check_gaps('at', gaps)
    free, free_p, _ = R.rec_loop(mem[0], kpm[0], pos[0], sd, apts, case['rec_length'])
    assert torch.equal(rec[1], free[1]) and torch.equal(probs[1], free_p[1]), 'the unconstrained point differs'
    if os.path.isdir(REF):   # the reference's own polygon and recognition loops at the same points
        from oracle.gen_golden_points import _model, _read_at
        import sys
        from oracle.gen_golden import SHIM
        sys.path[:0] = [SHIM, os.path.join(REF, 'OmniParser')]
        tmp = tempfile.mktemp(suffix='.pth')
        torch.save({'model': {}}, tmp)
        model, _ = _model(case, tmp)
        _, _, ref_rec, ref_probs = _read_at(model, img, mask, apts.numpy().tolist(), case)
        os.remove(tmp)
        assert torch.equal(ref_rec[0], free), 'the restatement without a set != the reference'
        assert float((ref_probs - free_p).abs().max()) < 1e-5
        print('omni_charset: the unconstrained restatement equals the reference at the read_at points')
    gold.update(at_pts=apts.numpy(), at_sets=np.array([t or '' for t in AT_SETS]),
                at_none=np.array([t is None for t in AT_SETS]), at_rec=rec.numpy(), at_probs=probs.numpy(),
                at_min_gap=np.array(g))
    print(f'omni_charset at: {[R.rec_text(r) for r in rec]}  smallest gap {g:.2e}')
    # ---- KIE: the page's (x, y) pairs under digits
    kc = KIE_CASES['kie']
    sd = W.omniparser_state_dict(seed=kc['wseed'], vie_categories=kc['vie'], pt_eos_bias=kc['pt_eos_bias'])
    img, mask = omni_inputs(kc)
    mem, pos, kpm, _ = O.encode(img, mask, sd)
    from advancedliteratemachinery_b200.omniparser import CLASSES_SROIE
    _, (pt_seq, _) = O.greedy_kie(mem[0], kpm[0], pos[0], sd, O.default_prompts(True)[0], kc['pt_seq_length'],
                                  kc['rec_length'], kc['vie'], torch.tensor(kc['canvas']), CLASSES_SROIE)
    pairs, i = [], 0   # the reference's walk (transformer.py:148-210)
    while i < len(pt_seq):
        if pt_seq[i] < W.NUM_BINS and i + 1 < len(pt_seq) and pt_seq[i + 1] < W.NUM_BINS:
            pairs.append((int(pt_seq[i]), int(pt_seq[i + 1])))
            i += 2
        else:
            i += 1
    kpts = torch.tensor(pairs, dtype=torch.long).reshape(-1, 2)
    assert len(pairs) > 0
    cs = R.charset_mask(SETS['digits']).expand(len(pairs), -1)
    rec, probs, gaps = R.rec_loop(mem[0], kpm[0], pos[0], sd, kpts, kc['rec_length'], cs, vie=kc['vie'])
    g = _check_gaps('kie', gaps)
    gold.update(kie_pts=kpts.numpy(), kie_rec=rec.numpy(), kie_probs=probs.numpy(), kie_min_gap=np.array(g))
    print(f'omni_charset kie: {[R.rec_text(r) for r in rec]}  smallest gap {g:.2e}')
    np.savez_compressed(os.path.join(GOLD, 'omni_charset.npz'), **gold)
    print('omni_charset: ok')


if __name__ == '__main__':
    torch.set_grad_enabled(False)
    gen_charset()
