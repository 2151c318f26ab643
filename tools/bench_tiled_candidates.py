"""Cost of recognition candidates and beams on pages read in tiles (OmniParserB200.spot_tiled(rec_candidates=,
rec_beams=); DESIGN 4.11).

python tools/bench_tiled_candidates.py [--repeats 3] [--out DIR]

Workload, the config-2 checkpoint and decode of bench.py (synthetic weights, seed 0, pt_eos suppressed, pt_seq_length
128: 64 instances per tile), as tools/bench_page_char_boxes.py: 8 synthetic A4 pages at 300 dpi (2 480 x 3 508 uint8,
host numpy), tile 1 200, overlap 256, 'upright' (96 tiles), read by spot_tiled() alone, with rec_candidates=8 and with
rec_beams=4.  Every variant is timed host clock to device synchronise, the variants alternating within each repeat;
medians and (min, max) over `--repeats`.  The GPU name and power limit are read in the same run.  The warm-up outputs
also say whether the candidates left every word as it was and whether the beams kept every point, polygon and tile.
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
    from advancedliteratemachinery_b200 import OmniParserB200, OmniVocab
    from oracle import weights as W
    torch.set_grad_enabled(False)
    gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                         text=True).stdout.strip().splitlines()[0]
    m = OmniParserB200(W.omniparser_state_dict(seed=0, pt_eos_bias=-30.0), OmniVocab(pt_seq_length=128, rec_length=25))
    rng = np.random.default_rng(0)
    a4 = [rng.integers(0, 256, (3508, 2480, 3), dtype=np.uint8) for _ in range(8)]
    variants = {'spot_tiled': lambda: m.spot_tiled(a4, 1200, 256),
                'rec_candidates=8': lambda: m.spot_tiled(a4, 1200, 256, rec_candidates=8),
                'rec_beams=4': lambda: m.spot_tiled(a4, 1200, 256, rec_beams=4)}
    outs = {k: fn() for k, fn in variants.items()}   # warm every shape
    geometry = lambda res: [[{k: v for k, v in d.items() if k not in ('rec', 'score')} for d in r] for r in res]
    times = {k: [] for k in variants}
    for _ in range(args.repeats):
        for k, fn in variants.items():
            times[k].append(timed(fn))
    stat = lambda x: {'median': float(np.median(x)), 'min': float(np.min(x)), 'max': float(np.max(x))}
    first = float(np.median(times['spot_tiled']))
    res = {'gpu': gpu, 'repeats': args.repeats, 'pages': len(a4), 'tiles': int(len(m.last_tiles['plan'])),
           'seconds': {k: stat(t) for k, t in times.items()},
           'ratio_to_spot_tiled': {k: float(np.median(t)) / first for k, t in times.items()},
           'words': {k: sum(len(r) for r in o) for k, o in outs.items()},
           'candidates_same_words': outs['rec_candidates=8'] == outs['spot_tiled'],
           'beams_same_geometry': geometry(outs['rec_beams=4']) == geometry(outs['spot_tiled'])}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'bench_tiled_candidates.json'), 'w') as f:
            f.write(line + '\n')
    m.ctx.close()


if __name__ == '__main__':
    main()
