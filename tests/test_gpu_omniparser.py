"""GPU parity: OmniParser CUDA path (through the C ABI) vs the CPU oracle and the committed reference
fixtures.  Tolerances (north_star): logits within 1e-3 relative, argmax token ids identical.

Protocol for ids (SURVEY.md section 7, "parity vs precision"): the small fixtures are generated free of near-ties and
must match bit for bit.  At benchmark scale (3 776 greedy steps per page) random synthetic weights do produce steps whose
reference top-1/top-2 gap is at the level of fp32 accumulation-order noise; there a mismatch is tolerated only if the
reference gap at that step is below 10x the measured logit error AND the CUDA path picked the reference runner-up, every
such flip is printed, and the count is bounded (MAX_NEAR_TIE_FLIPS).  Teacher-forced logits are always checked.
"""
import os

import numpy as np
import pytest
import torch

from tests.support import close_models, ctx, omni_model, options, release_models

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

LOGIT_REL_TOL = 1e-3
# the op tests need little; the library default (24 GB), held for the whole module, would leave no room for the three
# 20 GB contexts of the config-2 test on an 80 GB card
WORKSPACE_MB = 4096


def _rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _maxrel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).abs().max() / (b.abs().max() + 1e-30))


def model_for(wseed, pt_eos_bias):
    """One resident OmniParserB200 per synthetic checkpoint (weights are 0.9 GB on the device)."""
    return omni_model(dict(wseed=wseed, pt_eos_bias=pt_eos_bias), workspace_mb=8192)


# ----------------------------------------------------------------------------------------------- ops
@pytest.mark.parametrize('M,N,K,act,batch', [(128, 128, 64, 0, 1), (300, 200, 96, 1, 1), (77, 1104, 512, 2, 1),
                                             (49, 27, 96, 0, 3), (1000, 130, 2048, 0, 2), (257, 257, 64, 0, 4)])
def test_linear_tcgen05_matches_fp64(ctx, M, N, K, act, batch):
    g = torch.Generator().manual_seed(M + N + K)
    A = torch.randn(batch, M, K, generator=g)
    Wt = torch.randn(batch, N, K, generator=g) / K ** 0.5
    b = torch.randn(N, generator=g)
    ref = torch.einsum('bmk,bnk->bmn', A.double(), Wt.double()) + b.double()
    ref = torch.nn.functional.gelu(ref) if act == 1 else (torch.relu(ref) if act == 2 else ref)
    Ad, Wd, bd = A.cuda(), Wt.cuda(), b.cuda()
    for nsplit, tol in ((3, 2e-5), (1, 6e-3)):
        for impl in (0, 1):  # tensor-core kernel and the SIMT debug kernel must agree with fp64
            with options(ctx, nsplit=nsplit, gemm_impl=impl):
                out = torch.full((batch, M, N), float('nan'), device='cuda')
                ctx.check(ctx.lib.alm_op_linear(ctx.h, Ad.data_ptr(), Wd.data_ptr(), bd.data_ptr(), out.data_ptr(), M,
                                                N, K, act, batch))
                assert _rel(out.cpu(), ref) < tol, (nsplit, impl)


# Swin stages and merges (128 .. 2048), MGP-STR tiny / small / base / large (192 is its own gather_ln_kernel<2, 192>
# instantiation); 1 and 9 rows leave most of the 8-rows-per-CTA grid's last CTA idle
@pytest.mark.parametrize('C', [128, 192, 256, 384, 512, 768, 1024, 2048])
def test_layernorm(ctx, C):
    g, b = torch.randn(C), torch.randn(C)
    gd, bd = g.cuda(), b.cuda()
    for rows in (1, 9, 777):
        x = torch.randn(rows, C) * 3 + 1
        ref = torch.nn.functional.layer_norm(x.double(), (C,), g.double(), b.double(), 1e-5)
        xd = x.cuda()
        y = torch.full((rows * C + 1024,), float('nan'), device='cuda')
        torch.cuda.synchronize()  # the context's stream does not wait for torch's
        ctx.check(ctx.lib.alm_op_layernorm(ctx.h, xd.data_ptr(), gd.data_ptr(), bd.data_ptr(), 1e-5, y.data_ptr(), rows, C))
        assert torch.isnan(y[rows * C:]).all(), (rows, 'write past the output')
        assert float((y[:rows * C].view(rows, C).cpu().double() - ref).abs().max()) < 1e-5, rows


def window_attention_ref64(qkv, tab, B, nWh, nWw, heads, shift, scale=32 ** -0.5):
    """swin_transformer.py:127-148 without the projections, in fp64 on qkv's device: scale-then-dot, relative-position
    bias, -100 shift mask, softmax, PV.  qkv [B*nWh*nWw*49, 3C] window-major, tab [169, heads] -> [rows, C].  scale 1:
    q already scaled (the encoder's qkv planes)."""
    from oracle import omniparser_ref as O
    from oracle.weights import relative_position_index
    rows = qkv.shape[0]
    q, k, v = qkv.double().view(-1, 49, 3, heads, 32).permute(2, 0, 3, 1, 4)
    attn = (q * scale) @ k.transpose(-2, -1)
    idx = relative_position_index().view(-1).to(qkv.device)
    attn = attn + tab.double()[idx].view(49, 49, -1).permute(2, 0, 1).unsqueeze(0)
    if shift:
        mask = O.shift_mask(nWh * 7, nWw * 7).to(qkv.device, torch.float64)
        attn = (attn.view(B, nWh * nWw, heads, 49, 49) + mask.unsqueeze(1).unsqueeze(0)).view(-1, heads, 49, 49)
    return (attn.softmax(-1) @ v).transpose(1, 2).reshape(rows, heads * 32)


# (B, nWh, nWw, heads, shift); tests/test_gpu_encoder_ops.py runs these through alm_op_window_attention_ex as well
WATTN_CORE_CASES = [(1, 1, 1, 4, 0), (2, 2, 3, 4, 3), (1, 3, 2, 16, 3), (3, 5, 3, 8, 3), (7, 9, 10, 4, 0)]


@pytest.mark.parametrize('B,nWh,nWw,heads,shift', WATTN_CORE_CASES)
def test_window_attention_core(ctx, B, nWh, nWw, heads, shift):
    """swin_transformer.py:127-148 without the projections: scale-then-dot, bias, -100 shift mask, softmax, PV."""
    C = heads * 32
    g = torch.Generator().manual_seed(7)
    rows = B * nWh * nWw * 49
    qkv = torch.randn(rows, 3 * C, generator=g)
    tab = torch.randn(169, heads, generator=g) * 0.5
    ref = window_attention_ref64(qkv, tab, B, nWh, nWw, heads, shift)
    qd, td = qkv.cuda(), tab.cuda()
    # mma.sync kernel, fp32 SIMT debug kernel, persistent TMA-fed mma.sync kernel over head pairs
    for impl, tol in ((0, 5e-5), (1, 5e-6), (3, 5e-5)):
        with options(ctx, wattn_impl=impl):
            out = torch.full((rows, C), float('nan'), device='cuda')
            ctx.check(ctx.lib.alm_op_window_attention(ctx.h, qd.data_ptr(), td.data_ptr(), out.data_ptr(), B, nWh, nWw,
                                                      C, heads, shift))
            assert float((out.cpu() - ref).abs().max()) < tol, impl


# ----------------------------------------------------------------------------------------------- model
CASES = ['full', 'masked', 'odd', 'eos', 'oddlen', 'empty', 'longrec']


@pytest.mark.parametrize('name', CASES)
def test_encoder_matches_oracle_and_reference_fixture(name, golden_dir):
    from oracle import omniparser_ref as O
    from oracle.gen_golden import OMNI_CASES, omni_inputs
    from tests.conftest import omni_sd
    case = OMNI_CASES[name]
    gold = np.load(os.path.join(golden_dir, f'omni_{name}.npz'))
    m = model_for(case['wseed'], case['pt_eos_bias'])
    img, mask = omni_inputs(case)
    B, h, w = m.encode(img.cuda(), mask.cuda())
    assert (h, w) == tuple(gold['hw'])
    sd = omni_sd(case['wseed'], case['pt_eos_bias'])
    feats = O.swin_backbone(img, sd)
    for lvl in range(4):
        f = m.features(lvl).permute(0, 2, 3, 1)
        assert _rel(f, feats[lvl]) < 1e-4, f'stage {lvl}'
        np.testing.assert_allclose(f.reshape(-1)[::7].numpy(), gold[f'feat{lvl}_s'], atol=5e-4, rtol=0)
    mem = m.memory(0)[0]
    assert _rel(mem, torch.from_numpy(gold['memory'])) < 1e-4
    np.testing.assert_allclose(m.memory(1)[0].numpy(), gold['pos'], atol=3e-6, rtol=0)


@pytest.mark.parametrize('name', CASES)
def test_decode_matches_reference_fixture(name, golden_dir):
    from oracle.gen_golden import OMNI_CASES, omni_inputs
    case = OMNI_CASES[name]
    gold = np.load(os.path.join(golden_dir, f'omni_{name}.npz'))
    m = model_for(case['wseed'], case['pt_eos_bias'])
    m.vocab.pt_seq_length = case['pt_seq_length']
    m.vocab.rec_length = case['rec_length']
    img, mask = omni_inputs(case)
    from advancedliteratemachinery_b200 import NestedTensor
    v = m.vocab
    seqs = [v.pt_prompt(), torch.tensor([[v.poly_sos_index]]), torch.tensor([[v.rec_sos_index]]),
            torch.tensor(case['canvas'])]
    out = m(NestedTensor(img, mask), seqs)   # host tensors: H2D happens inside the C ABI
    if gold['none'][0]:
        assert out is None  # transformer.py:240-241
        return
    (pt, poly, rec), (probs,) = out
    # teacher-forced logits on the REFERENCE ids (no cascade), within the north_star tolerance
    gpt = torch.from_numpy(gold['pt'])
    n = gpt.numel() // 2
    L = case['rec_length']
    lg = m.decode_logits(0, 'pt', torch.cat([v.pt_prompt(), gpt], 1))
    ref = torch.from_numpy(gold['tf_pt'])
    err_pt = _maxrel(lg[0, 6:], ref)
    assert err_pt < LOGIT_REL_TOL and _rel(lg[0, 6:], ref) < LOGIT_REL_TOL
    poly_full = torch.cat([gpt.reshape(-1, 2), torch.full((n, 1), v.poly_sos_index),
                           torch.from_numpy(gold['poly']).reshape(n, 32)], 1)
    lg = m.decode_logits(0, 'poly', poly_full)
    assert _maxrel(lg[:, [2, 17, 33]], torch.from_numpy(gold['tf_poly'])) < LOGIT_REL_TOL
    rec_full = torch.cat([gpt.reshape(-1, 2), torch.full((n, 1), v.rec_sos_index), torch.from_numpy(gold['rec'])[0]], 1)
    lg = m.decode_logits(0, 'rec', rec_full)
    assert _maxrel(lg[:, [2, 2 + L // 2, 2 + L - 1]], torch.from_numpy(gold['tf_rec'])) < LOGIT_REL_TOL
    # greedy ids: BIT-EXACT.  The fixtures are generated with a near-tie floor (oracle/gen_golden.py GAP_FLOOR: every
    # greedy step of the reference has a top-1/top-2 logit gap >= 1e-4, ~7x the CUDA path's measured logit error), so
    # there is no near-tie excuse here; the near-tie protocol only exists in the page-scale test below, where it counts,
    # prints and bounds the flips.
    assert float(gold['min_gap'].min()) >= 1e-4
    assert np.array_equal(pt.numpy(), gold['pt']), 'pt ids differ from the reference'
    assert np.array_equal(poly.numpy(), gold['poly']), 'poly ids differ from the reference'
    assert np.array_equal(rec.numpy(), gold['rec']), 'rec ids differ from the reference'
    np.testing.assert_allclose(probs.numpy(), gold['probs'], rtol=2e-3, atol=1e-7)
    # the post-processing contract (utils/misc.py:164-185) on our ids gives the reference strings
    from oracle import omniparser_ref as O
    texts, confs = O.decode_rec_strings(rec[0], probs)
    assert texts == gold['texts'].tolist()


def test_batch_of_independent_pages_keeps_batch1_semantics(golden_dir):
    """B=3 different pages in one call == three batch-1 reference runs (F6): per-image instance counts,
    per-image EOS, shared-size canvas."""
    from advancedliteratemachinery_b200 import NestedTensor
    from oracle.gen_golden import OMNI_CASES, omni_inputs
    names = ['eos', 'oddlen', 'empty']  # same 64x64 canvas, same checkpoint seed, different eos bias...
    # ...so use one checkpoint (bias 0.45) and compare with the oracle run on it for each page
    from oracle import omniparser_ref as O
    from tests.conftest import omni_sd
    sd = omni_sd(0, 0.45)
    m = model_for(0, 0.45)
    m.vocab.pt_seq_length = 12
    m.vocab.rec_length = 25
    imgs = torch.cat([omni_inputs(OMNI_CASES[n])[0] for n in names])
    masks = torch.cat([omni_inputs(OMNI_CASES[n])[1] for n in names])
    outs = m.forward_batch(NestedTensor(imgs.cuda(), masks.cuda()))
    mem, pos, kpm, _ = O.encode(imgs, masks, sd)
    counts = []
    for b in range(3):
        ref = O.greedy_text_spotting(mem[b], kpm[b], pos[b], sd, m.vocab.pt_prompt(), 12, 25)
        if ref is None:
            assert outs[b] is None
            counts.append(0)
            continue
        (pt, poly, rec), (probs,) = outs[b]
        assert torch.equal(pt, ref[0][0]) and torch.equal(poly, ref[0][1]) and torch.equal(rec, ref[0][2])
        counts.append(pt.numel() // 2)
    assert len(set(counts)) > 1, 'the batch should mix different instance counts'


def test_determinism_and_batch_invariance_at_page_scale():
    """Size-independent properties at a real page size (2 x 512x768): same input twice -> identical ids and
    bit-identical memory; a page decoded alone == the same page inside a batch."""
    m = model_for(0, 0.45)
    m.vocab.pt_seq_length = 6
    g = torch.Generator().manual_seed(5)
    imgs = torch.randn(2, 3, 512, 768, generator=g).cuda()
    from advancedliteratemachinery_b200 import NestedTensor
    m.encode(imgs, None)
    mem1 = m.memory(0)
    out1 = m.decode()
    m.encode(imgs, None)
    mem2 = m.memory(0)
    out2 = m.decode()
    assert torch.equal(mem1, mem2)
    m.encode(imgs[1:2].contiguous(), None)
    mem_single = m.memory(0)
    out_single = m.decode()
    assert torch.equal(mem_single[0], mem1[1])
    for a, b in ((out1[0], out2[0]), (out1[1], out2[1]), (out1[1], out_single[0])):
        assert (a is None) == (b is None)
        if a is not None:
            for x, y in zip(a[0], b[0]):
                assert torch.equal(x, y)


def test_single_pass_bf16_mode_is_close_but_not_the_parity_mode(golden_dir):
    """nsplit=1 (plain bf16 operands): reported separately -- logits within 5e-2 relative, not 1e-3."""
    from oracle.gen_golden import OMNI_CASES, omni_inputs
    case = OMNI_CASES['full']
    gold = np.load(os.path.join(golden_dir, 'omni_full.npz'))
    m = model_for(case['wseed'], case['pt_eos_bias'])
    with options(m.ctx, nsplit=1):
        img, mask = omni_inputs(case)
        m.encode(img, mask)
        r = _rel(m.memory(0)[0], torch.from_numpy(gold['memory']))
        assert 1e-4 < r < 5e-2, r


def test_error_paths():
    from advancedliteratemachinery_b200 import AlmError, _lib
    c = _lib.Context(0)
    with pytest.raises(AlmError):   # encode before load
        c.check(c.lib.alm_omni_encode(c.h, torch.zeros(1, 3, 64, 64).data_ptr(), None, 1, 64, 64))
    with pytest.raises(AlmError):   # missing tensors
        c.load_state_dict(_lib.MODEL_OMNI_SPOT, {'backbone.0.patch_embed.proj.weight': torch.zeros(128, 3, 4, 4)})
    with pytest.raises(AlmError):
        c.set_option('nsplit', 2)
    c.close()


def test_kie_decode_matches_reference_fixture(golden_dir):
    """--infer_vie branch (transformer.py:143-217): (x, y, class) point loop, per-pair polygon + transcription
    with the class logits excluded from the softmax, entity grouping."""
    from advancedliteratemachinery_b200 import NestedTensor, OmniParserB200, OmniVocab
    from advancedliteratemachinery_b200 import synthetic as W
    from oracle.gen_golden import KIE_CASES, omni_inputs
    case = KIE_CASES['kie']
    gold = np.load(os.path.join(golden_dir, 'omni_kie.npz'))
    close_models()
    sd = W.omniparser_state_dict(seed=case['wseed'], vie_categories=case['vie'], pt_eos_bias=case['pt_eos_bias'])
    v = OmniVocab(vie_categories=case['vie'], pt_seq_length=case['pt_seq_length'], rec_length=case['rec_length'])
    m = OmniParserB200(sd, v, workspace_mb=8192)
    img, mask = omni_inputs(case)
    seqs = [v.pt_prompt(), torch.tensor([[v.poly_sos_index]]), torch.tensor([[v.rec_sos_index]]), torch.tensor(case['canvas'])]
    out = m(NestedTensor(img, mask), seqs)
    assert [r[0] for r in out] == gold['texts'].tolist()
    assert [r[1] for r in out] == gold['classes'].tolist()
    np.testing.assert_allclose(np.array([r[2] for r in out]), gold['probs'], rtol=2e-3)
    np.testing.assert_allclose(np.array([r[3] for r in out]), gold['rects'])
    raw = m.last_kie_raw
    assert np.array_equal(raw['tokens'][0, :raw['n_tok'][0]], gold['pt_seq'])
    np.testing.assert_allclose(raw['probs'][0, :raw['n_tok'][0]], gold['pt_probs'][:raw['n_tok'][0]], rtol=2e-3)
    # the C++ entity walk (alm_post_omni_kie_json) on the same raw outputs == the adapter's list
    import json
    js = m.kie_results_json([case['canvas']])
    assert json.loads(js[0]) == [[r[0], r[1], r[2], r[3]] for r in out]
    m.ctx.close()


def test_full_size_page_encoder_matches_oracle():
    """BASELINE config-2 geometry (1024x1024: every Swin stage zero-padded to x7, 4096 memory tokens): the
    encoder + FPN + input_proj output of one page against the CPU oracle."""
    from oracle import omniparser_ref as O
    from tests.conftest import omni_sd
    sd = omni_sd(0, 0.45)
    m = model_for(0, 0.45)
    g = torch.Generator().manual_seed(1000)
    img = torch.randn(1, 3, 1024, 1024, generator=g)
    mask = torch.zeros(1, 1024, 1024, dtype=torch.bool)
    mem, pos, kpm, hw = O.encode(img, mask, sd)
    assert m.encode(img.cuda(), None) == (1, 64, 64) and hw == (64, 64)
    assert _rel(m.memory(0), mem) < 1e-4
    assert float((m.memory(1) - pos).abs().max()) < 5e-6


def test_fused_cross_attention_matches_gemm_path_and_oracle():
    """The flash-style fused cross-attention (xattn.cu) against the unfused paths (score GEMM + softmax + P.V GEMM;
    fp32 single-query kernel) and the oracle: 70 sequences of one image (two 64-query blocks, 58 dead rows), 10 and 1
    sequences (the 16-row variant the pt loop uses), M = 15 x 17 = 255 keys (ragged last key block, Mpad = 256, two key
    splits), right-hand columns masked."""
    from oracle import omniparser_ref as O
    from tests.conftest import omni_sd
    sd = omni_sd(0, 0.45)
    m = model_for(0, 0.45)
    v = m.vocab
    g = torch.Generator().manual_seed(77)
    img = torch.randn(1, 3, 240, 272, generator=g)
    mask = torch.zeros(1, 240, 272, dtype=torch.bool)
    mask[:, :, 224:] = True
    img[mask[:, None].expand_as(img)] = 0
    n_seq, L = 70, 5
    seq = torch.cat([torch.randint(0, v.num_bins, (n_seq, 2), generator=g), torch.full((n_seq, 1), v.rec_sos_index),
                     torch.randint(v.num_bins, v.recog_pad_index, (n_seq, L - 3), generator=g)], 1)
    m.encode(img, mask)
    _, mh, mw = m.memory_shape()
    assert mh * mw == 255
    mem_o, pos_o, kpm_o, _ = O.encode(img, mask, sd)
    assert bool(kpm_o[0].any()) and not bool(kpm_o[0].all())
    ref = O.decode_logits(seq[:8], mem_o[0], kpm_o[0], pos_o[0], sd, 'rec')
    lg = {0: {}, 1: {}}
    for impl in (1, 0):  # the unfused path needs its feature-major V_c^T built by the encode
        with options(m.ctx, xattn_impl=impl):
            m.encode(img, mask)
            for n in (70, 10, 1):
                lg[impl][n] = m.decode_logits(0, 'rec', seq[:n])
    for n in (70, 10, 1):
        assert torch.isfinite(lg[0][n]).all()
        assert _maxrel(lg[0][n], lg[1][n]) < 2e-5, (n, _maxrel(lg[0][n], lg[1][n]))
        k = min(n, 8)
        assert _maxrel(lg[0][n][:k], ref[:k]) < LOGIT_REL_TOL
        assert _rel(lg[0][n][:k], ref[:k]) < 1e-4
        # the two self-attention step kernels (CTA per (sequence, head) for few sequences / warp per pair) and the
        # fused kernel's 2 vs 3 CTAs per SM schedules agree as well
        with options(m.ctx, sattn_wide=0, xattn_ctas_per_sm=3):
            alt = m.decode_logits(0, 'rec', seq[:n])
        assert _maxrel(lg[0][n], alt) < 2e-5, (n, _maxrel(lg[0][n], alt))


def test_fused_cross_attention_8warp_variant_matches():
    """`xattn_wg` 2 (8 warps: four 16-row tiles x two key groups per 64-key block) == the 4-warp kernel, on the same
    ragged / masked / split case as above and on a batch of two images."""
    m = model_for(0, 0.45)
    v = m.vocab
    g = torch.Generator().manual_seed(78)
    img = torch.randn(2, 3, 240, 272, generator=g)
    mask = torch.zeros(2, 240, 272, dtype=torch.bool)
    mask[1, :, 224:] = True
    img[mask[:, None].expand_as(img)] = 0
    n_seq, L = 70, 5
    seq = torch.cat([torch.randint(0, v.num_bins, (n_seq, 2), generator=g), torch.full((n_seq, 1), v.rec_sos_index),
                     torch.randint(v.num_bins, v.recog_pad_index, (n_seq, L - 3), generator=g)], 1)
    m.encode(img, mask)
    for image in (0, 1):
        for n in (70, 33):
            ref = m.decode_logits(image, 'rec', seq[:n])
            with options(m.ctx, xattn_wg=2):
                alt = m.decode_logits(image, 'rec', seq[:n])
            assert torch.isfinite(alt).all()
            assert _maxrel(alt, ref) < 2e-5, (image, n, _maxrel(alt, ref))


def test_more_than_32_pages_leave_the_skinny_path_and_stay_batch_invariant():
    """34 pages per call: the pt loop has more than 32 live sequences, so its linears run on the tensor-core GEMM
    path and the 16-row fused cross-attention takes fp32 queries / writes split outputs.  Every page must decode to
    the same ids as in a 2-page call (pages are independent)."""
    from advancedliteratemachinery_b200 import NestedTensor
    m = model_for(0, 0.45)
    m.vocab.pt_seq_length = 6
    m.vocab.rec_length = 25
    g = torch.Generator().manual_seed(21)
    imgs = torch.randn(34, 3, 64, 96, generator=g)
    big = m.forward_batch(NestedTensor(imgs.cuda(), None))
    for lo in (0, 32):
        small = m.forward_batch(NestedTensor(imgs[lo:lo + 2].contiguous().cuda(), None))
        for k in range(2):
            a, b = big[lo + k], small[k]
            assert (a is None) == (b is None)
            if a is not None:
                for x, y in zip(a[0], b[0]):
                    assert torch.equal(x, y)


@pytest.mark.parametrize('impl', [2])
def test_tma_cross_attention_variant_matches_the_default_kernel(impl):
    """`xattn_impl` 2 (csrc/xattn_tma.cu: mma.sync with a TMA ring) against the default fused kernel: 70 / 33 sequences,
    10 and 1 (the pt case), ragged key range (M = 255: partial last key block), masked keys, two images, then a whole
    greedy decode."""
    from advancedliteratemachinery_b200 import NestedTensor
    m = model_for(0, 0.45)
    v = m.vocab
    g = torch.Generator().manual_seed(79)
    img = torch.randn(2, 3, 240, 272, generator=g)
    mask = torch.zeros(2, 240, 272, dtype=torch.bool)
    mask[1, :, 224:] = True
    img[mask[:, None].expand_as(img)] = 0
    seq = torch.cat([torch.randint(0, v.num_bins, (70, 2), generator=g), torch.full((70, 1), v.rec_sos_index),
                     torch.randint(v.num_bins, v.recog_pad_index, (70, 2), generator=g)], 1)
    m.encode(img, mask)
    for image in (0, 1):
        for n in (70, 33, 10, 1):
            with options(m.ctx, xattn_impl=0):
                ref = m.decode_logits(image, 'rec', seq[:n])
            with options(m.ctx, xattn_impl=impl):
                alt = m.decode_logits(image, 'rec', seq[:n])
            assert torch.isfinite(alt).all()
            assert _maxrel(alt, ref) < 2e-5, (image, n, _maxrel(alt, ref))
    m.vocab.pt_seq_length = 6
    with options(m.ctx, xattn_impl=0):
        a = m.forward_batch(NestedTensor(img.cuda(), mask.cuda()))
    with options(m.ctx, xattn_impl=impl):
        b = m.forward_batch(NestedTensor(img.cuda(), mask.cuda()))
    for x, y in zip(a, b):
        assert (x is None) == (y is None)
        if x is not None:
            for p, q in zip(x[0], y[0]):
                assert torch.equal(p, q)


def test_config5_geometry_largest_page_and_long_point_sequence():
    """BASELINE config-5 geometry: one 1920 x 1920 page (M = 120 x 120 = 14 400 memory tokens, 225 key blocks per
    (image, head)) through the encoder against the CPU oracle, then a long point sequence (the `table` use: many
    tokens after the 7-token prompt) whose teacher-forced logits must match the oracle at the north_star tolerance."""
    from oracle import omniparser_ref as O
    from tests.conftest import omni_sd
    sd = omni_sd(0, -30.0)
    m = model_for(0, -30.0)
    v = m.vocab
    g = torch.Generator().manual_seed(1920)
    img = torch.randn(1, 3, 1920, 1920, generator=g)
    mask = torch.zeros(1, 1920, 1920, dtype=torch.bool)
    mem, pos, kpm, hw = O.encode(img, mask, sd)
    assert m.encode(img.cuda(), None) == (1, 120, 120) and hw == (120, 120)
    assert _rel(m.memory(0), mem) < 1e-4
    seq = torch.cat([v.pt_prompt(), torch.randint(0, v.num_bins, (1, 40), generator=g)], 1)
    lg = m.decode_logits(0, 'pt', seq)
    ref = O.decode_logits(seq, mem[0], kpm[0], pos[0], sd, 'pt')
    assert _maxrel(lg, ref) < LOGIT_REL_TOL and _rel(lg, ref) < 1e-4
    m.vocab.pt_seq_length = 64
    out = m.decode()
    assert out[0] is not None and out[0][0][0].numel() == 64      # eos is pinned off: the full sequence is produced


# ----------------------------------------------------------------------------------------------- benchmark scale
MAX_NEAR_TIE_FLIPS = 3   # sequences (of 129 per page) allowed to leave the reference at a judged near-tie


def _first_diffs(got, gold):
    """[(row, first differing step)] for two [rows, steps] id arrays."""
    out = []
    for r in range(gold.shape[0]):
        d = np.nonzero(got[r] != gold[r])[0]
        if d.size:
            out.append((r, int(d[0])))
    return out


def _judge_flips(kind, got, gold, gaps, ref_logits, our_logits, start, cands):
    """Every sequence whose ids leave the reference must do so at a reference near-tie: gap < 10 x the measured logit
    error at that position, and the id picked is the reference runner-up.  Returns printable flip records."""
    flips = []
    for r, t in _first_diffs(got, gold):
        pos = start - 1 + t
        err = float((our_logits[r, pos] - ref_logits[r, pos]).abs().max())
        lg = ref_logits[r, pos].masked_fill(~cands(kind, t, ref_logits.shape[-1]), float('-inf'))
        top = lg.topk(2)
        gap = float(top.values[0] - top.values[1])
        assert abs(gap - float(gaps[r, t])) < 1e-4, 'oracle gap differs from the fixture gap'
        assert gap < 10 * max(err, 1e-6), f'{kind} seq {r} step {t}: reference gap {gap:.2e} vs logit error {err:.2e} -- a real mismatch'
        assert int(got[r, t]) == int(top.indices[1]), f'{kind} seq {r} step {t}: not the reference runner-up'
        flips.append(dict(kind=kind, seq=r, step=t, ref_gap=gap, logit_err=err))
    return flips


def test_config2_scale_decode_matches_the_reference(golden_dir):
    """BASELINE config 2 at full scale, against the UNMODIFIED reference's output on the same page (fixture
    omni_config2_page0.npz: oracle/gen_golden.py config2, 164 s of CPU for the no-cache loops): one 1024x1024 page,
    M = 4096 memory tokens, N = 64 instances, pt 128 + 64 x (32 poly + 25 rec) greedy steps, CUDA graphs on.
      (a) teacher-forced logits of ALL 129 sequences (pt, 64 poly, 64 rec; every position) vs the CPU oracle <= 1e-3;
      (b) greedy ids vs the reference ids: identical, or judged near-tie flips, counted, printed and bounded;
      (c) the same page inside a 16-page batch, decoded by 3 contexts in flight that share one set of weights, gives
          the same ids in every context (batch / concurrency invariance at the benchmark's own configuration)."""
    import json
    import threading
    from advancedliteratemachinery_b200 import NestedTensor, OmniParserB200, OmniVocab
    from oracle import omniparser_ref as O
    from oracle.gen_golden import CONFIG2_CASE, config2_page
    from tests.conftest import omni_sd
    case = CONFIG2_CASE
    gold = np.load(os.path.join(golden_dir, 'omni_config2_page0.npz'))
    sd = omni_sd(case['wseed'], case['pt_eos_bias'])
    close_models()
    v = OmniVocab(pt_seq_length=case['pt_seq_length'], rec_length=case['rec_length'])
    m = OmniParserB200(sd, v, workspace_mb=20480)
    img, mask = config2_page(case['seed'])
    out = m.forward_batch(NestedTensor(img, None))[0]
    (pt, poly, rec), (probs,) = out
    n = 64
    assert pt.numel() == 2 * n and poly.numel() == 32 * n and tuple(rec.shape) == (1, n, 25)
    gpt, gpoly, grec = torch.from_numpy(gold['pt']), torch.from_numpy(gold['poly']), torch.from_numpy(gold['rec'])

    # ---- (a) teacher-forced logits on the REFERENCE ids: CUDA path vs CPU oracle, all sequences, all positions
    mem, pos, kpm, _ = O.encode(img, mask, sd)
    full = {'pt': torch.cat([v.pt_prompt(), gpt], 1),
            'poly': torch.cat([gpt.reshape(-1, 2), torch.full((n, 1), v.poly_sos_index), gpoly.reshape(n, 32)], 1),
            'rec': torch.cat([gpt.reshape(-1, 2), torch.full((n, 1), v.rec_sos_index), grec[0]], 1)}
    ref_lg, our_lg, worst = {}, {}, {}
    for kind, seq in full.items():
        ref_lg[kind] = O.decode_logits(seq, mem[0], kpm[0], pos[0], sd, kind)
        our_lg[kind] = m.decode_logits(0, kind, seq)
        worst[kind] = _maxrel(our_lg[kind], ref_lg[kind])
        assert worst[kind] < LOGIT_REL_TOL and _rel(our_lg[kind], ref_lg[kind]) < LOGIT_REL_TOL, (kind, worst[kind])

    # ---- (b) greedy ids vs the reference
    def flips_vs_reference(o):
        (pt_, poly_, rec_), (probs_,) = o
        assert pt_.numel() == 2 * n
        fl = _judge_flips('pt', pt_.numpy(), gold['pt'], gold['gap_pt'], ref_lg['pt'], our_lg['pt'], 7, O.step_candidates)
        if not fl:  # same instance set: every polygon / transcription row is comparable
            fl += _judge_flips('poly', poly_.numpy().reshape(n, 32), gold['poly'].reshape(n, 32), gold['gap_poly'],
                               ref_lg['poly'], our_lg['poly'], 3, O.step_candidates)
            fl += _judge_flips('rec', rec_.numpy()[0], gold['rec'][0], gold['gap_rec'], ref_lg['rec'], our_lg['rec'], 3,
                               O.step_candidates)
            if np.array_equal(rec_.numpy(), gold['rec']):
                np.testing.assert_allclose(probs_.numpy(), gold['probs'], rtol=2e-3, atol=1e-7)
        return fl

    flips = flips_vs_reference(out)
    report = dict(logit_max_rel=worst, near_tie_flips=flips, sequences=2 * n + 1, greedy_steps=128 + n * 57,
                  smallest_reference_gap=float(min(gold['gap_pt'].min(), gold['gap_poly'].min(), gold['gap_rec'].min())))
    print('config-2 page parity:', json.dumps(report))
    assert len(flips) <= MAX_NEAR_TIE_FLIPS, flips

    # ---- (c) 16-page batch, 3 contexts in flight sharing one set of weights (bench.py's omni workload: 3 x 20 GB of
    #      workspace on an 80 GB card), graphs on
    pages = torch.cat([config2_page(case['seed'] + i)[0] for i in range(16)]).pin_memory()
    torch.cuda.empty_cache()   # blocks cached by the earlier tests of this process would not leave room for the workspaces
    models = [m] + [OmniParserB200(None, v, workspace_mb=20480, share_from=m) for _ in range(2)]
    results = [None] * len(models)

    def work(j):
        for _ in range(2):  # second round replays the captured graphs
            results[j] = models[j].forward_batch(NestedTensor(pages, None))
    ts = [threading.Thread(target=work, args=(j,)) for j in range(len(models))]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert all(r is not None and len(r) == 16 for r in results)
    for j in range(1, len(models)):   # the concurrent contexts agree bit for bit on all 16 pages
        for k in range(16):
            for x, y in zip(results[j][k][0], results[0][k][0]):
                assert torch.equal(x, y), f'context {j} page {k} differs from context 0'
    # page 0 inside the batch vs the reference (the key-range split of the fused attention depends on the batch size,
    # so "alone" and "in a batch" may round differently: each is held to the reference separately)
    batch_flips = flips_vs_reference(results[0][0])
    report['near_tie_flips_in_batch'] = batch_flips
    report['batch_page0_equals_page_alone'] = all(torch.equal(x, y) for x, y in zip(results[0][0][0], out[0]))
    print('config-2 batch parity:', json.dumps(report))
    assert len(batch_flips) <= MAX_NEAR_TIE_FLIPS, batch_flips
    for mm in models[1:]:
        mm.ctx.close()
    m.ctx.close()


def test_default_vocab_runs_and_position_table_exhaustion_is_an_error():
    """OmniVocab() defaults (pt_seq_length 1024, 7-token prompt: 1030 > the 1024-row position table): the reference runs
    this configuration because EOS ends the loop early (transformer.py:126); it only fails if step 1018 is reached."""
    from advancedliteratemachinery_b200 import AlmError, NestedTensor, OmniVocab
    from oracle import omniparser_ref as O
    from oracle.gen_golden import OMNI_CASES, omni_inputs
    from tests.conftest import omni_sd
    case = OMNI_CASES['eos']
    m = model_for(case['wseed'], case['pt_eos_bias'])
    keep = (m.vocab.pt_seq_length, m.vocab.rec_length)
    try:
        dv = OmniVocab()
        assert dv.pt_seq_length == 1024
        m.vocab.pt_seq_length, m.vocab.rec_length = dv.pt_seq_length, dv.rec_length
        img, mask = omni_inputs(case)
        out = m.forward_batch(NestedTensor(img, mask))[0]
        sd = omni_sd(case['wseed'], case['pt_eos_bias'])
        mem, pos, kpm, _ = O.encode(img, mask, sd)
        ref = O.greedy_text_spotting(mem[0], kpm[0], pos[0], sd, dv.pt_prompt(), 1024, 25)
        for x, y in zip(out[0], ref[0]):
            assert torch.equal(x, y)
    finally:
        m.vocab.pt_seq_length, m.vocab.rec_length = keep
    m2 = model_for(0, -30.0)   # pt_eos suppressed: the loop runs into the end of the position table
    keep = m2.vocab.pt_seq_length
    try:
        m2.vocab.pt_seq_length = 1024
        img, mask = omni_inputs(OMNI_CASES['oddlen'])
        with pytest.raises(AlmError, match='position table'):
            m2.forward_batch(NestedTensor(img, mask))
    finally:
        m2.vocab.pt_seq_length = keep


def test_shared_weights_contexts_and_stream_ordered_device_inputs():
    """alm_share_weights: a second context over the same device weights decodes identically, and keeps working after the
    owner context is freed (the slabs are ref-counted).  Device inputs produced on torch's current stream right before
    the call are ordered by alm_stream_wait inside the adapter."""
    from advancedliteratemachinery_b200 import NestedTensor, OmniParserB200, OmniVocab
    from tests.conftest import omni_sd
    close_models()
    free0 = torch.cuda.mem_get_info()[0]
    v = OmniVocab(pt_seq_length=6)
    owner = OmniParserB200(omni_sd(0, 0.45), v, workspace_mb=4096)
    used_one = free0 - torch.cuda.mem_get_info()[0]          # the converted weights (arenas are allocated on first use)
    second = OmniParserB200(None, v, workspace_mb=4096, share_from=owner)
    used_two = free0 - torch.cuda.mem_get_info()[0]
    assert used_one > (500 << 20) and used_two - used_one < (64 << 20), 'the second context must not copy the weights'
    g = torch.Generator().manual_seed(33)
    host = torch.randn(2, 3, 96, 128, generator=g)
    a = owner.forward_batch(NestedTensor(host, None))
    # device input written by async torch work on the current stream immediately before the call
    big = torch.randn(64, 1024, 1024, device='cuda')
    for _ in range(8):
        big = big @ big.transpose(1, 2) * 1e-3   # keeps the torch stream busy
    dev = (host.pin_memory().cuda(non_blocking=True) + big.mean() * 0).contiguous()
    b = second.forward_batch(NestedTensor(dev, None))
    for x, y in zip(a, b):
        assert (x is None) == (y is None)
        if x is not None:
            for s, t in zip(x[0], y[0]):
                assert torch.equal(s, t)
    owner.ctx.close()
    c = second.forward_batch(NestedTensor(host, None))
    for x, y in zip(a, c):
        if x is not None:
            for s, t in zip(x[0], y[0]):
                assert torch.equal(s, t)
    second.ctx.close()


def test_comm_entry_points_single_rank():
    """alm_comm_* with a one-rank NCCL communicator: id, init, weight broadcast (in place, values unchanged), gather."""
    from advancedliteratemachinery_b200 import NestedTensor
    m = model_for(0, 0.45)
    m.vocab.pt_seq_length = 6
    g = torch.Generator().manual_seed(3)
    img = torch.randn(1, 3, 64, 96, generator=g)
    before = m.forward_batch(NestedTensor(img, None))
    uid = m.ctx.comm_unique_id()
    assert len(uid) == 128
    m.ctx.comm_init(uid, 0, 1)
    m.ctx.broadcast_weights(0)
    after = m.forward_batch(NestedTensor(img, None))
    for x, y in zip(before, after):
        assert (x is None) == (y is None)
        if x is not None:
            for s, t in zip(x[0], y[0]):
                assert torch.equal(s, t)
    from advancedliteratemachinery_b200.dist import gather_sequences
    back = gather_sequences(after, m.vocab, ctx=m.ctx)
    assert len(back) == 1 and (back[0] is None) == (after[0] is None)
    if after[0] is not None:
        for s, t in zip(after[0][0], back[0][0]):
            assert torch.equal(s, t)


def test_points_only_decode_equals_the_point_loop_of_the_full_decode():
    """alm_omni_decode_points (decode_pt_seq alone, transformer.py:102-141) == the pt output of the full decode, for a
    batch mixing an early-EOS page, an odd-length page and a page without points."""
    from advancedliteratemachinery_b200 import NestedTensor
    from oracle.gen_golden import OMNI_CASES, omni_inputs
    m = model_for(0, 0.45)
    m.vocab.pt_seq_length = 12
    m.vocab.rec_length = 25
    names = ['eos', 'oddlen', 'empty']
    imgs = torch.cat([omni_inputs(OMNI_CASES[n])[0] for n in names])
    masks = torch.cat([omni_inputs(OMNI_CASES[n])[1] for n in names])
    outs = m.forward_batch(NestedTensor(imgs, masks))
    m.encode(imgs, masks)
    pts = m.decode_points()
    assert len(pts) == 3
    for o, (tok, prob) in zip(outs, pts):
        if o is None:
            assert tok.numel() == 0
        else:
            assert torch.equal(o[0][0].reshape(-1), tok) and prob.numel() == tok.numel()
            assert float(prob.min()) > 0 and float(prob.max()) <= 1


def test_ln_fused_gemv_point_loop_is_bit_identical():
    """`fuse_ln_gemv` 1 runs every pre-LayerNorm of the point loop inside the GEMV that consumes it (same arithmetic,
    same summation order): teacher-forced pt logits and greedy ids must equal the unfused path bit for bit."""
    from advancedliteratemachinery_b200 import NestedTensor
    m = model_for(0, 0.45)
    m.vocab.pt_seq_length = 12
    m.vocab.rec_length = 25
    g = torch.Generator().manual_seed(91)
    imgs = torch.randn(3, 3, 128, 160, generator=g)
    seq = torch.cat([m.vocab.pt_prompt(), torch.randint(0, 1000, (1, 9), generator=g)], 1)
    res = {}
    for f in (0, 1):
        with options(m.ctx, fuse_ln_gemv=f):
            outs = m.forward_batch(NestedTensor(imgs, None))
            res[f] = (outs, m.decode_logits(1, 'pt', seq))
    assert torch.equal(res[0][1], res[1][1])
    for a, b in zip(res[0][0], res[1][0]):
        assert (a is None) == (b is None)
        if a is not None:
            for x, y in zip(a[0], b[0]):
                assert torch.equal(x, y)
