"""Cost of caller character sets in the recognition loop (DESIGN 4.23), against the same call without a set, measured
alternately in one process.

    python tools/bench_charset.py [--repeats 7] [--out DIR]

  decode: 16 synthetic 1024 x 1024 pages (synthetic checkpoint seed 0, pt_eos suppressed: 128 point steps = 64
    instances per page, 25 recognition steps), decode() vs decode(rec_charset=digits) -- wall ms and the polygon +
    recognition loops' device ms (alm_omni_last_timing);
  read_regions: 8 synthetic A4 pages at 300 dpi (2480 x 3508), 200 word quads each, read_regions() vs read_regions with
    one set per region (digits, upper case and digits, '.,-/' and digits, None in turn) -- wall ms.
Medians over the repeats; the two variants alternate within every repeat.  The card name and power limit are read in
the same run.  Needs an sm_90 GPU and the built library.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, 'tools'))

DIGITS = '0123456789'


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else 'unknown'


def wall(f):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = f()
    torch.cuda.synchronize()
    return out, (time.perf_counter() - t0) * 1e3


def bench_decode(repeats):
    import torch
    from advancedliteratemachinery_b200 import OmniParserB200, OmniVocab
    from advancedliteratemachinery_b200 import synthetic as W
    m = OmniParserB200(W.omniparser_state_dict(seed=0, pt_eos_bias=-30.0), OmniVocab(pt_seq_length=128, rec_length=25),
                       workspace_mb=24576)
    try:
        pages = [torch.randn(1, 3, 1024, 1024, generator=torch.Generator().manual_seed(1000 + i)) for i in range(16)]
        m.encode(torch.cat(pages).cuda(), None)

        def run(cs):
            out, t = wall(lambda: m._decode_arrays(None, rec_charset=cs))
            return out, t, m.ctx.omni_last_timing()['poly_rec_loops_ms']

        run(None), run(DIGITS)   # warm-up: graphs captured
        a, b = [], []
        for _ in range(repeats):
            a.append(run(None))
            b.append(run(DIGITS))
        med = lambda xs: round(statistics.median(xs), 3)  # noqa: E731
        n, _, _, rec, _ = b[-1][0]
        v = m.vocab
        ok = {v.recog_pad_index - 1, v.recog_pad_index, v.rec_eos_index} | {v.num_bins + v.chars.index(c) for c in DIGITS}
        inside = all(set(rec[i, :n[i]].reshape(-1).tolist()) <= ok for i in range(len(n)))
        return dict(workload='decode_16x1024sq', instances=int(n.sum()), decode_ms=med(r[1] for r in a),
                    decode_digits_ms=med(r[1] for r in b), polyrec_ms=med(r[2] for r in a),
                    polyrec_digits_ms=med(r[2] for r in b), ids_in_set=inside)
    finally:
        m.ctx.close()


def bench_regions(repeats, n_pages=8, words=200):
    import torch
    from advancedliteratemachinery_b200 import OmniParserB200, OmniVocab
    from advancedliteratemachinery_b200 import synthetic as W
    from bench_read_at import a4_quads
    m = OmniParserB200(W.omniparser_state_dict(seed=0, pt_eos_bias=-30.0), OmniVocab(rec_length=25), workspace_mb=24576)
    try:
        rng = np.random.default_rng(7)
        pages = [torch.from_numpy(rng.integers(0, 256, (3508, 2480, 3), dtype=np.uint8)).cuda() for _ in range(n_pages)]
        quads = np.concatenate([a4_quads(rng, words) for _ in range(n_pages)])
        pi = np.repeat(np.arange(n_pages), words)
        sets = [[DIGITS, 'ABCDEFGHIJKLMNOPQRSTUVWXYZ' + DIGITS, '.,-/' + DIGITS, None][i % 4] for i in range(len(quads))]
        free = lambda: m.read_regions(pages, quads, pi, kind='quad')  # noqa: E731
        per = lambda: m.read_regions(pages, quads, pi, kind='quad', rec_charset=sets)  # noqa: E731
        wall(free), wall(per)
        a, b = [], []
        for _ in range(repeats):
            a.append(wall(free))
            b.append(wall(per))
        got = b[-1][0]
        inside = all(s is None or set(d['rec']) <= set(s) for d, s in zip(got, sets))
        med = lambda xs: round(statistics.median(xs), 2)  # noqa: E731
        return dict(workload='read_regions_8xA4_200', regions=len(quads), read_regions_ms=med(r[1] for r in a),
                    read_regions_sets_ms=med(r[1] for r in b), texts_in_set=inside)
    finally:
        m.ctx.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--repeats', type=int, default=7)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    import torch
    torch.set_grad_enabled(False)
    rows = [dict(card=card())]
    print(json.dumps(rows[0]), flush=True)
    for f in (bench_decode, bench_regions):
        rows.append(f(args.repeats))
        print(json.dumps(rows[-1]), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'bench_charset.json'), 'w') as fh:
            json.dump(rows, fh, indent=1)


if __name__ == '__main__':
    main()
