"""KIE entities across tile seams and character boxes for entity words (DESIGN 4.22): what kie_tiled's whole_page and
rec_locations options cost.

    python tools/bench_kie_whole_page.py [--reps 3] [--out bench_out/bench_kie_whole_page.json]

Workloads, each with a synthetic KIE checkpoint (advancedliteratemachinery_b200/synthetic.py, SROIE classes, pt_eos
suppressed so every tile and page decodes the full point sequence):
  receipts  8 synthetic receipts of 945 x 3000 (80 mm at 300 dpi): one tile wide, three tiles tall
  a4        8 A4 pages at 300 dpi (2480 x 3508): 12 tiles each
Variants, alternated rep by rep in one process: kie_tiled (tile 1200, overlap 256, max_batch 16) with
  off        neither option (the path kie_tiled had before them)
  whole      whole_page=True: every page also read whole and merged by merge_kie_whole_page
  loc        rec_locations=True: every decode keeps locations, one char_boxes call
  whole_loc  both
Also the merge alone at scale, 16 pages x 12 tiles of fabricated tile entities and whole readings: the device call (host
clock over 20 calls, each ending in a synchronise) against the host build (tests/emu/kie_whole_page_emu.cpp).  Times
are medians of wall-clock seconds around work that ends in a device synchronise.  The card's name and power limit are
read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

T, OV, PT_SEQ = 1200, 256, 60
VARIANTS = dict(off={}, whole=dict(whole_page=True), loc=dict(rec_locations=True),
                whole_loc=dict(whole_page=True, rec_locations=True))


def pages(kind, n, seed):
    rng = np.random.default_rng(seed)
    h, w = (3000, 945) if kind == 'receipts' else (3508, 2480)
    return [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for _ in range(n)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'the benchmark measures the GPU'
    torch.set_grad_enabled(False)
    from advancedliteratemachinery_b200 import OmniParserB200, OmniVocab
    from advancedliteratemachinery_b200 import synthetic as W
    from advancedliteratemachinery_b200.omniparser import merge_kie_tiles, merge_kie_whole_page
    from oracle import page_turn_ref as PT
    from tests.test_kie_tiles_cpu import fabricate
    from tests.test_kie_whole_page_cpu import emu_whole, fabricate_whole
    card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                          text=True).stdout.strip()
    v = OmniVocab(vie_categories=4, pt_seq_length=PT_SEQ, rec_length=25)
    m = OmniParserB200(W.omniparser_state_dict(seed=2, vie_categories=4, pt_eos_bias=-30.0), v, workspace_mb=40960)
    res = dict(card=card, pt_seq_length=PT_SEQ)
    for kind in ('receipts', 'a4'):
        pp = pages(kind, 8, 1 if kind == 'receipts' else 2)
        counts = {}
        for name, opt in VARIANTS.items():   # warm-up, and what each variant returns
            ents = m.kie_tiled(pp, tile=T, overlap=OV, **opt)
            counts[name] = dict(entities=sum(len(e) for e in ents),
                                whole_kept=int((m.last_tiles['whole_merge']['source'][:, 0] < 0).sum())
                                if 'whole_merge' in m.last_tiles else 0)
        off = m.kie_tiled(pp, tile=T, overlap=OV)
        assert [[e[:4] for e in p] for p in m.kie_tiled(pp, tile=T, overlap=OV, rec_locations=True)] == off
        times = {k: [] for k in VARIANTS}
        for _ in range(a.reps):
            for name, opt in VARIANTS.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                m.kie_tiled(pp, tile=T, overlap=OV, **opt)
                torch.cuda.synchronize()
                times[name].append(time.perf_counter() - t0)
        res[kind] = dict(pages=8, size=list(pp[0].shape[:2]), counts=counts,
                         **{f'{k}_s': float(np.median(t)) for k, t in times.items()},
                         **{f'{k}_all_s': t for k, t in times.items()})
        print(kind, json.dumps(res[kind]), flush=True)
    # the merge alone at scale
    rng = np.random.default_rng(12)
    sizes = [(3508, 2480)] * 16
    raw = fabricate(rng, sizes, T, OV, None, n_ent=60, max_tok=1024, max_inst=400)
    plan = PT.plan(sizes, [0] * 16, T, OV)
    keys = ('n_tok', 'tokens', 'probs', 'n_inst', 'inst_pos', 'poly')
    tiles = merge_kie_tiles(m.ctx, sizes, T, OV, plan, *[raw[k] for k in keys], 1000, v.padding_index + 1, 4)
    whole = fabricate_whole(rng, sizes, T, OV, [0] * 16, n_ent=200)
    args = (m.ctx, sizes, T, OV, tiles, *[whole[k] for k in keys], 1000, v.padding_index + 1, 4)
    out = merge_kie_whole_page(*args)
    dev = []
    for _ in range(5):  # each call ends in a synchronise of the library's stream
        t0 = time.perf_counter()
        for _ in range(20):
            merge_kie_whole_page(*args)
        dev.append((time.perf_counter() - t0) * 1e3 / 20)
    hst = []
    for _ in range(5):
        t0 = time.perf_counter()
        emu_whole(sizes, T, OV, tiles, whole, class_base=v.padding_index + 1)
        hst.append((time.perf_counter() - t0) * 1e3)
    res['merge_16x12'] = dict(tile_entities=int(len(tiles['cls'])), whole_tokens=int(whole['n_tok'].sum()),
                              kept=int(out['count'].sum()), whole_kept=int((out['source'][:, 0] < 0).sum()),
                              device_ms=float(np.median(dev)), host_build_ms=float(np.median(hst)))
    print('merge', json.dumps(res['merge_16x12']), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or '.', exist_ok=True)
        with open(a.out, 'w') as f:
            json.dump(res, f, indent=1)
    m.ctx.close()


if __name__ == '__main__':
    main()
