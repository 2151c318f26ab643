"""GPU: several window prompts per page in one batched decode (alm_omni_decode_prompts, OmniParserB200.decode_prompts).
Every (page, prompt) slot must give what the reference's batch-1 call with that prompt gives (tests/golden/omni_prompts.npz,
written from the unmodified reference) and what alm_omni_decode gives for that page and prompt alone."""
import ctypes as C

import numpy as np
import pytest
import torch

from tests.support import close_models, omni_model, options, release_models
from tests.test_prompts_cpu import prompt_case, prompt_page

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

LOGIT_REL_TOL = 1e-3
ALM_ERR_INVALID, ALM_ERR_OOM, ALM_ERR_STATE = -1, -3, -4



def _maxrel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).abs().max() / (b.abs().max() + 1e-30))


def fixture_model(gold, workspace_mb=8192):
    """One resident OmniParserB200 on the fixture's checkpoint, decode lengths of the fixture."""
    return omni_model({k: gold[k][0] for k in ('wseed', 'pt_eos_bias', 'pt_seq_length', 'rec_length')},
                      workspace_mb=workspace_mb)


def fixture_pages(gold):
    pages = [prompt_page(gold, b) for b in range(2)]
    return torch.cat([p[0] for p in pages]), torch.cat([p[1] for p in pages])


def assert_slot_equal(a, b, prob_rtol):
    assert (a is None) == (b is None)
    if a is None:
        return
    for x, y in zip(a[0], b[0]):
        assert torch.equal(x, y)
    if prob_rtol == 0:
        assert torch.equal(a[1][0], b[1][0])
    else:
        np.testing.assert_allclose(a[1][0].numpy(), b[1][0].numpy(), rtol=prob_rtol, atol=0)


def check_against_fixture(m, gold, outs):
    prompts = torch.from_numpy(gold['prompts'])
    for b in range(2):
        for p in range(4):
            key, out = f'{b}_{p}', outs[b][p]
            if gold['n_inst'][b, p] == 0:
                assert out is None, key  # transformer.py:240-241
                continue
            assert out is not None, key
            (pt, poly, rec), (probs,) = out
            # the fixture clears a 1e-4 top-1 / top-2 gap at every greedy step: ids are bit-exact
            assert np.array_equal(pt.numpy(), gold[f'pt_{key}']), key
            assert np.array_equal(poly.numpy(), gold[f'poly_{key}']), key
            assert np.array_equal(rec.numpy(), gold[f'rec_{key}']), key
            np.testing.assert_allclose(probs.numpy(), gold[f'probs_{key}'], rtol=2e-3, atol=1e-7)
            lg = m.decode_logits(b, 'pt', torch.cat([prompts[b, p][None], torch.from_numpy(gold[f'pt_{key}'])], 1))
            n_prompt = prompts.shape[2]
            assert _maxrel(lg[0, n_prompt - 1:], torch.from_numpy(gold[f'tf_pt_{key}'])) < LOGIT_REL_TOL, key


def test_window_prompts_match_the_reference_fixture(golden_dir):
    gold = prompt_case(golden_dir)
    m = fixture_model(gold)
    imgs, masks = fixture_pages(gold)
    m.encode(imgs.cuda(), masks.cuda())
    outs = m.decode_prompts(torch.from_numpy(gold['prompts']))
    check_against_fixture(m, gold, outs)
    # the duplicated prompt of each page gets the same result as its twin
    prompts = gold['prompts']
    for b in range(2):
        for p in range(4):
            for q in range(p):
                if np.array_equal(prompts[b, p], prompts[b, q]):
                    assert_slot_equal(outs[b][p], outs[b][q], 0)


def test_each_slot_equals_the_single_prompt_decode_of_its_page(golden_dir):
    gold = prompt_case(golden_dir)
    m = fixture_model(gold)
    prompts = torch.from_numpy(gold['prompts'])
    imgs, masks = fixture_pages(gold)
    m.encode(imgs.cuda(), masks.cuda())
    batched = m.decode_prompts(prompts)
    for b in range(2):
        m.encode(imgs[b:b + 1].cuda(), masks[b:b + 1].cuda())
        for p in range(4):
            alone = m.decode(prompts[b, p][None])[0]
            # a point decoded alone runs the poly / rec loops on the fp32 GEMV path, in the batch (several distinct
            # points per page) on the split-bf16 tensor-core GEMMs: probabilities differ in the last bits (1.4e-5
            # relative measured on an H100), ids not at all
            assert_slot_equal(batched[b][p], alone, 5e-5)
    # P = 1 through the new entry is alm_omni_decode, bit for bit
    m.encode(imgs.cuda(), masks.cuda())
    for p in range(4):
        one = prompts[0, p][None]
        ref = m.decode(one)
        new = m.decode_prompts(one)
        for b in range(2):
            assert_slot_equal(new[b][0], ref[b], 0)


def test_more_than_32_slots_leave_the_skinny_path_and_stay_batch_invariant(golden_dir):
    """9 pages x 4 prompts = 36 point sequences: the pt loop runs its linears on the tensor-core GEMMs and the fused
    cross-attention on split bf16 queries.  Every slot must equal the same slot of a 2-page call (8 sequences, skinny)."""
    gold = prompt_case(golden_dir)
    m = fixture_model(gold)
    m.vocab.pt_seq_length = 6
    prompts = torch.from_numpy(gold['prompts'][0])
    g = torch.Generator().manual_seed(23)
    imgs = torch.randn(9, 3, 64, 96, generator=g)
    m.encode(imgs.cuda(), None)
    big = m.decode_prompts(prompts)
    assert sum(o is not None for page in big for o in page) > 0
    for lo in (0, 7):
        m.encode(imgs[lo:lo + 2].contiguous().cuda(), None)
        small = m.decode_prompts(prompts)
        for k in range(2):
            for p in range(4):
                a, b = big[lo + k][p], small[k][p]
                assert (a is None) == (b is None)
                if a is not None:
                    for x, y in zip(a[0], b[0]):
                        assert torch.equal(x, y)


@pytest.mark.parametrize('impl', [2, 1])
def test_window_prompts_under_the_other_cross_attention_kernels(impl, golden_dir):
    """xattn_impl 2 (TMA-fed fused kernel, fp32 queries with 4 rows per image on the skinny pt path) and xattn_impl 1
    (unfused score GEMM + softmax + P.V GEMM; the pt loop takes the tensor-core path) give the fixture's results."""
    gold = prompt_case(golden_dir)
    m = fixture_model(gold)
    imgs, masks = fixture_pages(gold)
    with options(m.ctx, xattn_impl=impl):
        m.encode(imgs.cuda(), masks.cuda())   # xattn_impl 1 needs its V_c^T built by the encode
        check_against_fixture(m, gold, m.decode_prompts(torch.from_numpy(gold['prompts'])))


def _raw_decode_prompts(m, prompts, P, n_prompt, max_instances=None):
    v = m.vocab
    maxi = max(1, v.pt_seq_length // 2) if max_instances is None else max_instances
    B = max(1, prompts.numel() // max(1, P * n_prompt))
    n_inst = np.zeros((B, max(P, 1)), dtype=np.int32)
    pt = np.zeros((B, max(P, 1), maxi, 2), dtype=np.int64)
    poly = np.zeros((B, max(P, 1), maxi, 32), dtype=np.int64)
    rec = np.zeros((B, max(P, 1), maxi, v.rec_length), dtype=np.int64)
    prob = np.zeros((B, max(P, 1), maxi, v.rec_length), dtype=np.float32)
    p = prompts.to(torch.long).contiguous()
    return m.lib.alm_omni_decode_prompts(m.ctx.h, p.data_ptr(), P, n_prompt, C.byref(m._cfg(maxi)), n_inst.ctypes.data,
                                         pt.ctypes.data, poly.ctypes.data, rec.ctypes.data, prob.ctypes.data)


def test_error_paths(golden_dir):
    from advancedliteratemachinery_b200 import OmniParserB200, OmniVocab
    from advancedliteratemachinery_b200 import synthetic as W
    gold = prompt_case(golden_dir)
    m = fixture_model(gold, workspace_mb=1024)
    v = m.vocab
    glob = v.pt_prompt()
    try:
        assert _raw_decode_prompts(m, glob.repeat(2, 1), 2, 7) == ALM_ERR_STATE   # before any encode
        imgs, masks = fixture_pages(gold)
        m.encode(imgs.cuda(), masks.cuda())
        two = glob.repeat(2, 1, 1)                                                # [B=2, P=1, 7]
        assert _raw_decode_prompts(m, two, 0, 7) == ALM_ERR_INVALID
        assert _raw_decode_prompts(m, glob.repeat(2, 17, 1), 17, 7) == ALM_ERR_INVALID
        assert _raw_decode_prompts(m, glob.repeat(2, 1, 3)[..., :17], 1, 17) == ALM_ERR_INVALID
        bad = two.clone()
        bad[1, 0, 2] = -1
        assert _raw_decode_prompts(m, bad, 1, 7) == ALM_ERR_INVALID
        bad[1, 0, 2] = m.lib.alm_omni_vocab(m.ctx.h)
        assert _raw_decode_prompts(m, bad, 1, 7) == ALM_ERR_INVALID
        assert _raw_decode_prompts(m, two, 1, 7, max_instances=v.pt_seq_length // 2 - 1) == ALM_ERR_INVALID
        assert _raw_decode_prompts(m, two, 1, 7) == 0
        # 4 pages x 16 prompts at a full position table: 64 sequences x 16 MB of self-attention caches > a 1 GB workspace
        m.encode(torch.cat([imgs, imgs]).cuda(), torch.cat([masks, masks]).cuda())
        v.pt_seq_length = 1024
        assert _raw_decode_prompts(m, glob.repeat(4, 16, 1), 16, 7) == ALM_ERR_OOM
        v.pt_seq_length = int(gold['pt_seq_length'][0])
        m.encode(imgs.cuda(), masks.cuda())
        assert _raw_decode_prompts(m, two, 1, 7) == 0                             # the context stays usable
        with options(m.ctx, kv_decoders=1):
            m.encode(imgs.cuda(), masks.cuda())
            assert _raw_decode_prompts(m, two, 1, 7) == ALM_ERR_STATE
    finally:
        close_models()
    kv = OmniVocab(vie_categories=4, pt_seq_length=9)
    k = OmniParserB200(W.omniparser_state_dict(seed=2, vie_categories=4, pt_eos_bias=-30.0), kv, workspace_mb=1024)
    try:
        k.encode(imgs[:1].cuda(), None)
        assert _raw_decode_prompts(k, kv.pt_prompt().reshape(1, 1, 7), 1, 7) == ALM_ERR_INVALID   # KIE checkpoint
    finally:
        k.ctx.close()
