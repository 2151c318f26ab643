"""Cost of character boxes in page pixels (OmniParserB200.spot_tiled(rec_locations=True), omniparser.char_boxes;
DESIGN 4.20).

python tools/bench_page_char_boxes.py [--repeats 3] [--out DIR]

Workloads, the config-2 checkpoint and decode of bench.py (synthetic weights, seed 0, pt_eos suppressed, pt_seq_length
128: 64 instances per tile), as tools/bench_whole_page.py:
  A4     8 synthetic A4 pages at 300 dpi (2 480 x 3 508 uint8, host numpy), tile 1 200, overlap 256, 'upright', with
         and without rec_locations;
  boxes  4 000 words of rec_length 25 on one A4 page read whole (the identity frame, so both give the same boxes),
         fabricated as tests/test_page_char_boxes_cpu.py does: the entry (one launch with its copies) against
         postprocess.rec_char_boxes, the host loop it replaces for the one-image paths; and the entry alone on
         16 pages x 4 096 words.
Every variant is timed host clock to device synchronise, the variants of a workload alternating within each repeat;
medians and (min, max) over `--repeats`.  The GPU name and power limit are read in the same run.  How well the
attention locates real characters is not measured here: a synthetic checkpoint says nothing about it.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--repeats', type=int, default=3)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'the benchmark measures the GPU path'
    from advancedliteratemachinery_b200 import OmniParserB200, OmniVocab, postprocess
    from advancedliteratemachinery_b200.omniparser import char_boxes
    from oracle import weights as W
    from tests.test_page_char_boxes_cpu import fabricate, frames_to_tiles
    torch.set_grad_enabled(False)
    gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                         text=True).stdout.strip().splitlines()[0]
    v = OmniVocab(pt_seq_length=128, rec_length=25)
    m = OmniParserB200(W.omniparser_state_dict(seed=0, pt_eos_bias=-30.0), v)
    rng = np.random.default_rng(0)
    a4 = [rng.integers(0, 256, (3508, 2480, 3), dtype=np.uint8) for _ in range(8)]
    # 4 000 words on one A4 page read whole: polygons as bins (rec_char_boxes' input) and as page pixels (the entry's)
    h, w = 3508, 2480
    _, rec, loc, _, _ = fabricate(1, N=4000, nan=0.0)
    ids = rng.integers(0, v.num_bins, (4000, 32))
    polys = ids.astype(np.float64).reshape(-1, 16, 2) / v.num_bins * np.array([w, h])
    zero = np.zeros(4000, np.int32)
    big = fabricate(2, N=16 * 4096, F=16 * 12, nan=0.0)
    big_sizes, big_tiles, big_turns = frames_to_tiles(big[4])
    pad, eos = v.recog_pad_index, v.rec_eos_index
    workloads = {
        'A4': {'off': lambda: m.spot_tiled(a4, 1200, 256),
               'rec_locations': lambda: m.spot_tiled(a4, 1200, 256, rec_locations=True)},
        'boxes': {'entry': lambda: char_boxes(m.ctx, [(h, w)], [(0, 0, 0, h, w)], polys.reshape(-1, 32), rec, loc,
                                              zero, pad, eos),
                  'rec_char_boxes': lambda: postprocess.rec_char_boxes(ids, rec, loc, (h, w), v)},
        'boxes_16x4096': {'entry': lambda: char_boxes(m.ctx, big_sizes, big_tiles, big[0], big[1], big[2], big[3],
                                                      pad, eos, turns=big_turns)},
    }
    res = {'gpu': gpu, 'repeats': args.repeats}
    stat = lambda x: {'median': float(np.median(x)), 'min': float(np.min(x)), 'max': float(np.max(x))}
    for name, variants in workloads.items():
        counts = {}
        for k, fn in variants.items():  # warm every shape
            out = fn()
            # characters for the boxes, words for the pages
            counts[k] = int(out['n_chars'].sum()) if isinstance(out, dict) else sum(len(r) for r in out)
        times = {k: [] for k in variants}
        for _ in range(args.repeats):
            for k, fn in variants.items():
                times[k].append(timed(fn))
        first = float(np.median(times[next(iter(variants))]))
        res[name] = {'seconds': {k: stat(t) for k, t in times.items()},
                     'ratio_to_first': {k: float(np.median(t)) / first for k, t in times.items()},
                     'counts': counts}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'bench_page_char_boxes.json'), 'w') as f:
            f.write(line + '\n')
    m.ctx.close()


if __name__ == '__main__':
    main()
