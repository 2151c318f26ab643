"""Caller-given regions read at quarter-turns (read_regions(orientation=...)), measured.

    python tools/bench_region_turns.py [--a4 8] [--words 200] [--repeats 5] [--out DIR]

read_regions on --a4 synthetic A4 pages at 300 dpi (2480 x 3508) with --words word-sized integer boxes each, three ways:
'upright', every region at one explicit turn (turn 2: the page read upside down, the same tiles as upright), and
'auto' (every region read at two turns, the better reading kept on the device).  Wall ms per call (page upload, tile
cutting, encoding, decoding, the selection) and words per second, medians of alternating repeats, with the tiles and
whole readings each call encoded.  Also the wall time of alm_omni_select_regions alone on 'auto''s candidate rows.
The card name and power limit are read in the same run.  Needs an sm_90 GPU and the built library.
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


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else 'unknown'


def a4_boxes(rng, words):
    """word-sized integer boxes on a 2480 x 3508 page"""
    w, h = rng.integers(80, 400, words), rng.integers(30, 60, words)
    x, y = rng.integers(60, 2480 - 60 - w), rng.integers(60, 3508 - 60 - h)
    return np.stack([x, y, x + w, y + h], 1).astype(np.float64)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--a4', type=int, default=8)
    ap.add_argument('--words', type=int, default=200)
    ap.add_argument('--repeats', type=int, default=5)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    import torch
    from advancedliteratemachinery_b200 import OmniParserB200, OmniVocab
    from advancedliteratemachinery_b200 import synthetic as W
    from advancedliteratemachinery_b200.omniparser import select_regions
    assert torch.cuda.is_available(), 'needs an H100'
    m = OmniParserB200(W.omniparser_state_dict(seed=0, pt_eos_bias=-30.0), OmniVocab(pt_seq_length=128, rec_length=25),
                       workspace_mb=24576)
    rng = np.random.default_rng(7)
    pages = [torch.from_numpy(rng.integers(0, 256, (3508, 2480, 3), dtype=np.uint8)).cuda() for _ in range(args.a4)]
    boxes = np.concatenate([a4_boxes(rng, args.words) for _ in range(args.a4)])
    pi = np.repeat(np.arange(args.a4), args.words)
    R = len(boxes)
    modes = {'upright': 'upright', 'turn2': np.full(R, 2), 'auto': 'auto'}

    def run(o):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        m.read_regions(pages, boxes, pi, kind='box', orientation=o)
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3

    for o in modes.values():   # warm-up: every shape seen once
        run(o)
    times = {k: [] for k in modes}
    encoded = {}
    for _ in range(args.repeats):
        for k, o in modes.items():
            times[k].append(run(o))
            encoded[k] = {kind: int(sum(len(c['index']) for c in m.last_regions['chunks'] if c['kind'] == kind))
                          for kind in ('tile', 'whole')}
    lr = m.last_regions   # 'auto', the last call
    sel = (lr['frames'], lr['frame_index'], np.zeros((R, 2, 2), np.int64), np.zeros((R, 2, 32), np.int64), lr['rec'],
           lr['prob'], m.vocab.num_bins, m.vocab.recog_pad_index, m.vocab.rec_eos_index)
    select_regions(m.ctx, *sel)
    st = []
    for _ in range(args.repeats):
        t0 = time.perf_counter()
        select_regions(m.ctx, *sel)
        st.append((time.perf_counter() - t0) * 1e3)
    result = dict(card=card(), pages=args.a4, page='2480x3508 (A4, 300 dpi)', regions=R, kind='box')
    for k in modes:
        ms = statistics.median(times[k])
        result[k] = dict(ms=round(ms, 1), words_per_s=round(R / (ms / 1e3), 1), tiles_read=encoded[k]['tile'],
                         whole_readings=encoded[k]['whole'])
    result['auto_over_upright'] = round(result['auto']['ms'] / result['upright']['ms'], 3)
    result['select_regions_ms'] = round(statistics.median(st), 3)
    print(json.dumps(result))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'bench_region_turns.json'), 'w') as f:
            json.dump(result, f, indent=1)


if __name__ == '__main__':
    main()
