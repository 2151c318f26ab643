"""GPU parity: MGP-STR CUDA path (through the C ABI) vs the CPU oracle and the reference fixtures.
Tolerance (north_star): logits within 1e-3 relative; top-1 ids identical to the reference's argmax."""
import os

import numpy as np
import pytest
import torch

from tests.support import mgp_model, options, release_models

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)


@pytest.fixture(scope='module')
def model():
    return mgp_model()


def _maxrel(a, b):
    return float((a.double() - b.double()).abs().max() / b.double().abs().max())


@pytest.mark.parametrize('name', ['b1', 'b3'])
def test_forward_matches_reference_fixture(model, name, golden_dir):
    from oracle.gen_golden import MGP_CASES
    case = MGP_CASES[name]
    gold = np.load(os.path.join(golden_dir, f'mgp_{name}.npz'))
    g = torch.Generator().manual_seed(case['seed'])
    img = torch.rand(case['batch'], 3, 32, 128, generator=g)
    attns, char, bpe, wp = model(img, is_eval=True)          # host tensor: H2D inside the C ABI
    assert _maxrel(char, torch.from_numpy(gold['char'])) < 1e-3
    np.testing.assert_allclose(attns[0].numpy(), gold['char_attn'], atol=2e-5, rtol=1e-3)
    np.testing.assert_allclose(attns[1].reshape(-1)[::5].numpy(), gold['bpe_attn_s'], atol=2e-5, rtol=1e-3)
    np.testing.assert_allclose(attns[2].reshape(-1)[::5].numpy(), gold['wp_attn_s'], atol=2e-5, rtol=1e-3)
    for k, (nm, lg) in enumerate((('char', char), ('bpe', bpe), ('wp', wp))):
        ids = model.last_ids[k].to(torch.int64)
        assert torch.equal(ids, lg.argmax(-1)), 'fused argmax disagrees with the logits it came from'
        if nm == 'char':
            assert np.array_equal(ids.numpy(), gold['char'].argmax(-1))
            continue
        ref_s = torch.from_numpy(gold[nm + '_s'])
        assert _maxrel(lg.reshape(-1)[::997], ref_s) < 1e-3
        assert np.array_equal(ids.numpy(), gold[nm + '_ids']), nm
        np.testing.assert_allclose(model.last_prob[k].numpy(), gold[nm + '_prob'], rtol=2e-3)


def test_matches_oracle_on_a_fresh_batch_and_is_batch_invariant(model):
    from oracle import mgpstr_ref as M
    from tests.conftest import mgp_sd
    g = torch.Generator().manual_seed(77)
    img = torch.rand(5, 3, 32, 128, generator=g)
    ref = M.forward(img, mgp_sd(0))
    out = model(img.cuda(), is_eval=True)                     # device tensor: no staging copy
    for a, b in zip(out[1:], ref[1:]):
        assert _maxrel(a, b) < 1e-3
    single = model(img[2:3].contiguous(), is_eval=True)
    assert torch.equal(single[1][0], out[1][2])               # same crop alone == inside the batch (bitwise)


def test_ids_only_call_skips_the_big_logit_copies(model):
    g = torch.Generator().manual_seed(3)
    img = torch.rand(4, 3, 32, 128, generator=g)
    full = model.forward(img, is_eval=True)
    ids_full = model.last_ids.clone()
    model.forward(img, is_eval=True, want_logits=False)
    assert torch.equal(ids_full, model.last_ids)
    assert full[2] is not None


@pytest.mark.parametrize('name', ['tiny', 'small', 'large', 'charstr'])
def test_variants_match_reference_fixtures(name, golden_dir):
    """The other released sizes (tiny 192x3 heads, small 384x6, large 1024x16, depth 24) and the char-only CHAR-STR:
    geometry is derived from the checkpoint tensors; fixtures come from the reference classes."""
    from advancedliteratemachinery_b200 import MGPSTRB200
    from advancedliteratemachinery_b200 import synthetic as W
    from oracle.gen_golden import MGP_VARIANT_CASES
    case = MGP_VARIANT_CASES[name]
    gold = np.load(os.path.join(golden_dir, f'mgp_{name}.npz'))
    char_only = name == 'charstr'
    dim, depth, heads = W.MGP_VARIANTS['base' if char_only else name]
    sd = W.mgpstr_state_dict(seed=case['seed'], dim=dim, depth=depth, heads=heads, char_only=char_only)
    m = MGPSTRB200(sd)
    try:
        inf = m.info()
        assert (inf['dim'], inf['depth'], inf['heads'], inf['n_a3']) == (dim, depth, heads, 1 if char_only else 3)
        g = torch.Generator().manual_seed(case['seed'])
        img = torch.rand(2, 3, 32, 128, generator=g)
        out = m(img, is_eval=True)
        assert _maxrel(out[1], torch.from_numpy(gold['char'])) < 1e-3
        np.testing.assert_allclose(out[0][0].numpy(), gold['char_attn'], atol=2e-5, rtol=1e-3)
        assert np.array_equal(m.last_ids[0].numpy(), gold['char'].argmax(-1))
        if char_only:
            assert len(out) == 2 and len(out[0]) == 1
        else:
            for k, nm in ((1, 'bpe'), (2, 'wp')):
                assert _maxrel(out[1 + k].reshape(-1)[::997], torch.from_numpy(gold[nm + '_s'])) < 1e-3
                assert np.array_equal(m.last_ids[k].to(torch.int64).numpy(), gold[nm + '_ids']), nm
    finally:
        m.ctx.close()


def test_config3_batch_512_rows_equal_small_batches_and_the_oracle(model):
    """BASELINE config 3 geometry: B = 512 crops in one call (131 584 token rows).  Every crop's ids equal the ids of the
    same crop in a 4-crop call (batch invariance at scale), 6 crops spread over the batch match the CPU oracle's logits,
    and the single-pass bf16 mode (the config's stated dtype) is reported with its own id flip rate."""
    from oracle import mgpstr_ref as M
    from tests.conftest import mgp_sd
    g = torch.Generator().manual_seed(512)
    img = torch.rand(512, 3, 32, 128, generator=g)
    model.forward(img.cuda(), is_eval=True, want_logits=False)
    ids_big = model.last_ids.clone()
    pick = [0, 1, 2, 3, 255, 256, 509, 510, 511]
    for lo in (0, 252, 508):
        model.forward(img[lo:lo + 4].contiguous(), is_eval=True, want_logits=False)
        assert torch.equal(model.last_ids, ids_big[:, lo:lo + 4]), f'crops {lo}..{lo + 3}'
    sel = torch.tensor([0, 100, 255, 256, 400, 511])
    ref = M.forward(img[sel], mgp_sd(0))
    for k in range(3):
        assert torch.equal(ids_big[k, sel].to(torch.int64), ref[1 + k].argmax(-1)), k
    out = model(img[sel].contiguous(), is_eval=True)
    for a, b in zip(out[1:], ref[1:]):
        assert _maxrel(a, b) < 1e-3
    with options(model.ctx, nsplit=1):
        model.forward(img.cuda(), is_eval=True, want_logits=False)
        flips = float((model.last_ids != ids_big).float().mean())
        print(f'single-pass bf16 at B=512: {flips * 100:.2f} % of the 3 x 512 x 27 ids differ from the split (fp32-class) mode')
        assert flips < 0.25


def test_fused_attention_model_path_matches_fixture_and_unfused_path(golden_dir):
    """MGP-STR forward with attn_impl 0 (fused attention kernel + packed qkv GEMM) vs the reference fixture and vs the
    unfused path (attn_impl 1) on the same weights."""
    from advancedliteratemachinery_b200 import MGPSTRB200
    from oracle.gen_golden import MGP_CASES
    from tests.conftest import mgp_sd
    gold = np.load(os.path.join(golden_dir, 'mgp_b3.npz'))
    g = torch.Generator().manual_seed(MGP_CASES['b3']['seed'])
    img = torch.rand(3, 3, 32, 128, generator=g)
    m = MGPSTRB200(mgp_sd(0))
    try:
        outs = {}
        for impl in (0, 1):
            m.ctx.set_option('attn_impl', impl)
            outs[impl] = m(img, is_eval=True)
            assert _maxrel(outs[impl][1], torch.from_numpy(gold['char'])) < 1e-3, impl
            assert np.array_equal(m.last_ids[1].to(torch.int64).numpy(), gold['bpe_ids']), impl
            assert np.array_equal(m.last_ids[2].to(torch.int64).numpy(), gold['wp_ids']), impl
        assert _maxrel(outs[0][1], outs[1][1]) < 1e-4
    finally:
        m.ctx.close()
