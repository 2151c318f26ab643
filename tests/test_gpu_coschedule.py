"""GPU: both models under every co-scheduling knob, bit for bit against the default schedule.

The knobs let several contexts and streams share one H100: `enc_grid_cap` / `dec_grid_cap` bound the GEMM grids of
alm_omni_encode* / of the decode loops, `small_grid_cap` those of every GEMM with at most 2 x SMs tiles,
`decode_streams` 1 runs the polygon and recognition loops serially on one stream, and `decode_priority` 1 moves the
decode loops to internal high-priority streams forked from and joined back to the caller's stream.  None of them may
change a bit: a tile's arithmetic does not depend on the grid (tests/test_gpu_gemm_capped.py holds the engine to that
against fp64), and the stream settings only change ordering.  Each setting, with CUDA graphs on and off, must give the
default run's ids, probabilities, teacher-forced logits, encoder memory, recognition extras and MGP-STR logits; the
default run itself meets its fixture's bar (bit-exact ids against tests/golden/omni_*.npz and mgp_*.npz).

Also: a 1024 x 1024 page encoded with one CTA per GEMM (hundreds of tiles per CTA), the in-flight form the benchmark
times (3 OmniParser and 2 MGP-STR contexts sharing weights, each on its own stream with its own knobs, run
concurrently), and the scope of the settings: after an encode under `enc_grid_cap` and a decode refused after the
high-priority streams were entered, the context runs on the caller's stream again, sees device inputs written there,
and gives a fresh context's bits.
"""
import os
import threading
import time

import numpy as np
import pytest
import torch

from tests.support import omni_model, options, release_models

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)


def _settings():
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return {'default': {}, 'enc_grid_cap=1': dict(enc_grid_cap=1), 'enc_grid_cap=7': dict(enc_grid_cap=7),
            f'enc_grid_cap={sms // 2}': dict(enc_grid_cap=sms // 2), 'dec_grid_cap=1': dict(dec_grid_cap=1),
            'dec_grid_cap=5': dict(dec_grid_cap=5), 'small_grid_cap=1': dict(small_grid_cap=1),
            'small_grid_cap=3': dict(small_grid_cap=3), 'decode_streams=1': dict(decode_streams=1),
            'decode_priority=1': dict(decode_priority=1),
            'all': dict(enc_grid_cap=7, dec_grid_cap=5, small_grid_cap=3, decode_streams=1, decode_priority=1)}


def omni_for(wseed, pt_eos_bias, vie=0):
    """one resident OmniParserB200 per synthetic checkpoint"""
    return omni_model(dict(wseed=wseed, pt_eos_bias=pt_eos_bias, vie=vie), kie=bool(vie))


def _flat(x):
    """every array / tensor / scalar of a nested result as bytes (dtype and shape included)"""
    if x is None:
        return [b'None']
    if isinstance(x, dict):
        return [y for k in sorted(x) for y in [k.encode()] + _flat(x[k])]
    if isinstance(x, (list, tuple)):
        return [b'['] + [y for v in x for y in _flat(v)] + [b']']
    if isinstance(x, torch.Tensor):
        x = x.cpu().numpy()
    if isinstance(x, np.ndarray):
        return [f'{x.dtype}{x.shape}'.encode() + np.ascontiguousarray(x).tobytes()]
    return [repr(x).encode()]


def _assert_same(base, got, label):
    a, b = _flat(base), _flat(got)
    assert len(a) == len(b), f'{label}: the result has a different structure'
    bad = [i for i, (x, y) in enumerate(zip(a, b)) if x != y]
    assert not bad, f'{label}: {len(bad)} of {len(a)} result arrays differ from the default run (first: item {bad[0]})'


def sweep(ctx, run, what):
    """run() under the default options, then under every setting with graphs on and off: bit for bit the default"""
    base = run()
    n = 0
    for graphs in (1, 0):
        for name, opts in _settings().items():
            if name == 'default' and graphs:
                continue
            with options(ctx, use_graphs=graphs, **opts):
                _assert_same(base, run(), f'{what}: {name}, use_graphs {graphs}')
            n += 1
    print(f'[coschedule] {what}: {n} settings bit-identical to the default')
    return base


# ------------------------------------------------------------------------------------------ OmniParser paths
def _fixture_spotting(name, golden_dir):
    from advancedliteratemachinery_b200.omniparser import _spotting_result
    from oracle.gen_golden import OMNI_CASES, omni_inputs
    case = OMNI_CASES[name]
    gold = np.load(os.path.join(golden_dir, f'omni_{name}.npz'))
    m = omni_for(case['wseed'], case['pt_eos_bias'])
    m.vocab.pt_seq_length, m.vocab.rec_length = case['pt_seq_length'], case['rec_length']
    img, mask = omni_inputs(case)
    return case, gold, m, img, mask, _spotting_result


def _assert_fixture_ids(out, gold, label=''):
    assert out is not None, label
    (pt, poly, rec), (probs,) = out
    assert np.array_equal(pt.numpy(), gold['pt']), f'{label} pt ids differ from the reference'
    assert np.array_equal(poly.numpy(), gold['poly']), f'{label} poly ids differ from the reference'
    assert np.array_equal(rec.numpy(), gold['rec']), f'{label} rec ids differ from the reference'
    np.testing.assert_allclose(probs.numpy(), gold['probs'], rtol=2e-3, atol=1e-7)


@pytest.mark.parametrize('name', ['full', 'masked', 'odd'])
def test_spotting_fixture_under_every_knob(name, golden_dir):
    case, gold, m, img, mask, result = _fixture_spotting(name, golden_dir)
    v = m.vocab
    gpt = torch.from_numpy(gold['pt'])
    n = gpt.numel() // 2
    seq_pt = torch.cat([v.pt_prompt(), gpt], 1)
    seq_rec = torch.cat([gpt.reshape(-1, 2), torch.full((n, 1), v.rec_sos_index), torch.from_numpy(gold['rec'])[0]], 1)

    def run():
        m.encode(img, mask)
        return dict(memory=m.memory(0), decode=m._decode_arrays(), tf_pt=m.decode_logits(0, 'pt', seq_pt),
                    tf_rec=m.decode_logits(0, 'rec', seq_rec))

    base = sweep(m.ctx, run, f'omni {name}')
    _assert_fixture_ids(result(*(a[0] for a in base['decode'])), gold, name)


@pytest.mark.parametrize('extra', ['rec_candidates', 'rec_beams', 'rec_locations'])
def test_recognition_extras_under_every_knob(extra, golden_dir):
    """the extras that add per-step kernels (top-k, beam selection with ancestry, cross-attention locations)"""
    case, gold, m, img, mask, _ = _fixture_spotting('full', golden_dir)
    kw = {'rec_candidates': dict(rec_candidates=3), 'rec_beams': dict(rec_beams=3),
          'rec_locations': dict(rec_locations=True)}[extra]

    def run():
        m.encode(img, mask)
        out = m.decode(**kw)
        return dict(out=out, cand=m.last_rec_candidates, beams=m.last_rec_beams, loc=m.last_rec_locations)

    try:
        base = sweep(m.ctx, run, f'omni full {extra}')
    finally:
        m.decode()  # extras off again
    if extra != 'rec_beams':  # candidate 0 and the located greedy run are the greedy decode
        _assert_fixture_ids(base['out'][0], gold, extra)


def test_pages_fixture_under_every_knob(golden_dir):
    from advancedliteratemachinery_b200 import NestedTensor
    from tests.test_gpu_omni_pages import ORDER, fixture_batch
    from tests.test_pages_cpu import pages_case
    gold = pages_case(golden_dir)
    m = omni_for(int(gold['wseed'][0]), float(gold['pt_eos_bias'][0]))
    m.vocab.pt_seq_length, m.vocab.rec_length = int(gold['pt_seq_length'][0]), int(gold['rec_length'][0])
    _, (t, mask) = fixture_batch(gold)
    t, mask = t.cuda(), mask.cuda()

    def run():
        out = m.forward_pages(NestedTensor(t, mask))
        return dict(out=out, memory=m.memory(0))

    base = sweep(m.ctx, run, 'omni forward_pages')
    for i, b in enumerate(ORDER):
        if gold['n_inst'][b] == 0:
            assert base['out'][i] is None, b
            continue
        (pt, poly, rec), _ = base['out'][i]
        assert np.array_equal(pt.numpy(), gold[f'pt_{b}']) and np.array_equal(poly.numpy(), gold[f'poly_{b}']) and \
            np.array_equal(rec.numpy(), gold[f'rec_{b}']), b


def test_window_prompts_fixture_under_every_knob(golden_dir):
    from tests.test_gpu_omni_prompts import check_against_fixture
    from tests.test_prompts_cpu import prompt_case, prompt_page
    gold = prompt_case(golden_dir)
    m = omni_for(int(gold['wseed'][0]), float(gold['pt_eos_bias'][0]))
    m.vocab.pt_seq_length, m.vocab.rec_length = int(gold['pt_seq_length'][0]), int(gold['rec_length'][0])
    pages = [prompt_page(gold, b) for b in range(2)]
    imgs, masks = torch.cat([p[0] for p in pages]), torch.cat([p[1] for p in pages])
    prompts = torch.from_numpy(gold['prompts'])

    def run():
        m.encode(imgs, masks)
        return dict(out=m.decode_prompts(prompts), memory=m.memory(0))

    base = sweep(m.ctx, run, 'omni decode_prompts')
    m.encode(imgs, masks)
    check_against_fixture(m, gold, base['out'])


def test_kie_fixture_under_every_knob(golden_dir):
    from advancedliteratemachinery_b200 import NestedTensor
    from oracle.gen_golden import KIE_CASES, omni_inputs
    case = KIE_CASES['kie']
    gold = np.load(os.path.join(golden_dir, 'omni_kie.npz'))
    m = omni_for(case['wseed'], case['pt_eos_bias'], vie=case['vie'])
    v = m.vocab
    v.pt_seq_length, v.rec_length = case['pt_seq_length'], case['rec_length']
    img, mask = omni_inputs(case)
    seqs = [v.pt_prompt(), torch.tensor([[v.poly_sos_index]]), torch.tensor([[v.rec_sos_index]]),
            torch.tensor(case['canvas'])]

    def run():
        out = m(NestedTensor(img, mask), seqs)
        return dict(out=out, raw=m.last_kie_raw, memory=m.memory(0))

    base = sweep(m.ctx, run, 'omni KIE')
    assert [r[0] for r in base['out']] == gold['texts'].tolist()
    raw = base['raw']
    assert np.array_equal(raw['tokens'][0, :raw['n_tok'][0]], gold['pt_seq'])


def test_page_encoded_with_one_cta_per_gemm():
    """1024 x 1024 page with every encoder GEMM on one CTA: hundreds of tiles per CTA through the ping-pong loop.
    Memory bit for bit the full grid's."""
    m = omni_for(0, -30.0)
    img = torch.randn(1, 3, 1024, 1024, generator=torch.Generator().manual_seed(1000)).cuda()
    m.encode(img)
    base = m.memory(0)
    with options(m.ctx, enc_grid_cap=1):
        t = time.time()
        m.encode(img)
        got = m.memory(0)
        print(f'[coschedule] 1024 x 1024 encode at enc_grid_cap 1: {time.time() - t:.2f} s')
    assert torch.equal(got.view(torch.int32), base.view(torch.int32))


# ------------------------------------------------------------------------------------------ MGP-STR
@pytest.mark.parametrize('name', ['b1', 'b3'])
def test_mgpstr_fixture_under_every_knob(name, golden_dir):
    """B = 1 makes most ViT GEMMs narrow (32-column tiles), B = 3 mixes both widths; every one has <= 2 x SMs tiles"""
    from advancedliteratemachinery_b200 import MGPSTRB200
    from oracle.gen_golden import MGP_CASES
    from tests.conftest import mgp_sd
    case = MGP_CASES[name]
    gold = np.load(os.path.join(golden_dir, f'mgp_{name}.npz'))
    img = torch.rand(case['batch'], 3, 32, 128, generator=torch.Generator().manual_seed(case['seed']))
    m = MGPSTRB200(mgp_sd(0))
    try:
        def run():
            out = m(img, is_eval=True)
            return dict(out=out, ids=m.last_ids, prob=m.last_prob, topk=m.recognize_topk(img, 3))

        base = sweep(m.ctx, run, f'mgp {name}')
    finally:
        m.ctx.close()
    ids = base['ids']
    assert np.array_equal(ids[0].numpy(), gold['char'].argmax(-1))
    assert np.array_equal(ids[1].to(torch.int64).numpy(), gold['bpe_ids'])
    assert np.array_equal(ids[2].to(torch.int64).numpy(), gold['wp_ids'])


# ------------------------------------------------------------------------------------------ in flight
def test_contexts_in_flight_with_their_own_knobs():
    """3 OmniParser and 2 MGP-STR contexts sharing weights, each on its own stream with different knobs, two rounds
    each from their own host threads with nothing synchronising them: each context gives its single-context bits"""
    from advancedliteratemachinery_b200 import MGPSTRB200, NestedTensor, OmniParserB200
    from tests.conftest import mgp_sd
    owner = omni_for(0, -30.0)
    owner.vocab.pt_seq_length, owner.vocab.rec_length = 8, 25
    g = torch.Generator().manual_seed(44)
    pages = torch.randn(2, 3, 96, 128, generator=g)
    crops = torch.rand(3, 3, 32, 128, generator=g)
    streams = [torch.cuda.Stream() for _ in range(5)]
    omni = [OmniParserB200(None, owner.vocab, stream=streams[j].cuda_stream, workspace_mb=2048, share_from=owner)
            for j in range(3)]
    mgp = [MGPSTRB200(mgp_sd(0), stream=streams[3].cuda_stream)]
    mgp.append(MGPSTRB200(None, stream=streams[4].cuda_stream, share_from=mgp[0]))
    knobs = [dict(), dict(enc_grid_cap=7, dec_grid_cap=5, decode_priority=1),
             dict(enc_grid_cap=1, small_grid_cap=3, decode_streams=1, use_graphs=0),
             dict(small_grid_cap=1), dict(small_grid_cap=3)]

    def work(j):
        if j < 3:
            return omni[j].forward_batch(NestedTensor(pages, None)), omni[j].memory(0)
        out = mgp[j - 3](crops, is_eval=True)
        return out, mgp[j - 3].last_ids.clone()

    try:
        single = []
        for j in range(5):
            single.append(work(j))
        for j in range(5):
            for k, v in knobs[j].items():
                (omni + mgp)[j].ctx.set_option(k, v)
        results = [[None, None] for _ in range(5)]
        errors = []

        def thread(j):
            try:
                for r in range(2):
                    results[j][r] = work(j)
            except BaseException as e:  # reported below, after every thread has ended
                errors.append((j, e))

        ts = [threading.Thread(target=thread, args=(j,)) for j in range(5)]
        for t in ts:
            t.start()
        for t in ts:
            t.join()
        assert not errors, errors
        for j in range(5):
            for r in range(2):
                _assert_same(single[j], results[j][r], f'context {j} ({knobs[j]}) round {r}')
    finally:
        for x in omni + mgp:
            x.ctx.close()


# ------------------------------------------------------------------------------------------ scope of the settings
def test_settings_end_with_the_call_and_the_caller_stream_is_restored(golden_dir):
    """A context on the caller's stream S: encode under enc_grid_cap, then a decode refused after the decode loops
    moved to the high-priority streams (the point sequence runs into the end of the position table).  Afterwards a
    device input written on S by a kernel that is still running when the call is made must be read after it (the
    context enqueues on S again), and the results equal a fresh context's bit for bit."""
    from advancedliteratemachinery_b200 import AlmError, NestedTensor, OmniParserB200, OmniVocab
    from oracle.gen_golden import OMNI_CASES, omni_inputs
    owner = omni_for(0, -30.0)
    S = torch.cuda.Stream()
    v = OmniVocab(pt_seq_length=8, rec_length=25)
    m = OmniParserB200(None, v, stream=S.cuda_stream, workspace_mb=2048, share_from=owner)
    fresh = OmniParserB200(None, v, workspace_mb=2048, share_from=owner)
    g = torch.Generator().manual_seed(45)
    page = torch.randn(1, 3, 96, 128, generator=g)
    try:
        want = fresh.forward_batch(NestedTensor(page, None))
        want_mem = fresh.memory(0)
        for k, v in dict(enc_grid_cap=7, dec_grid_cap=5, decode_priority=1).items():
            m.ctx.set_option(k, v)
        img, mask = omni_inputs(OMNI_CASES['oddlen'])
        m.vocab.pt_seq_length = 1024
        with pytest.raises(AlmError, match='position table'):
            m.forward_batch(NestedTensor(img, mask))
        m.vocab.pt_seq_length = 8
        # written on S behind a long kernel, handed to the library without alm_stream_wait
        dev = torch.zeros(1, 3, 96, 128, device='cuda')
        src = page.cuda()
        torch.cuda.synchronize()
        with torch.cuda.stream(S):
            torch.cuda._sleep(200_000_000)
            dev.copy_(src)
        m.ctx.check(m.lib.alm_omni_encode(m.ctx.h, dev.data_ptr(), None, 1, 96, 128))
        assert torch.equal(m.memory(0).view(torch.int32), want_mem.view(torch.int32)), \
            'the encode did not run on the caller stream after the refused decode'
        _assert_same(want, m.decode(), 'decode after the refused one')
        # and through the adapter, with the input written on torch's current stream
        big = torch.randn(32, 1024, 1024, device='cuda')
        for _ in range(8):
            big = big @ big.transpose(1, 2) * 1e-3
        dev2 = (page.pin_memory().cuda(non_blocking=True) + big.mean() * 0).contiguous()
        _assert_same(want, m.forward_batch(NestedTensor(dev2, None)), 'forward after the refused decode')
        _assert_same(want_mem, m.memory(0), 'memory after the refused decode')
    finally:
        m.ctx.close()
        fresh.ctx.close()
