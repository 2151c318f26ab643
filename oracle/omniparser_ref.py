"""CPU fp32 restatement of the OmniParser inference forward -- TEST INFRASTRUCTURE ONLY.

This is the parity oracle for the CUDA path (tests/, __graft_entry__.smoke(), bench.py's
cpu_baseline / --impl reference leg).  The product never imports it.

It restates, op for op and in the same arithmetic order, the reference graph selected by the
shipped flags ``--tfm_pre_norm --use_fpn --use_char_window_prompt`` (OCR/OmniParser/test.sh:8-14).
Citations are relative to /root/reference/OCR/OmniParser/.  ``oracle/gen_golden.py`` pins it
against the unmodified reference modules (run in the build container, where /root/reference
exists) and writes the fixtures in tests/golden/ that the GPU box checks against.

Parity status: pinned against the reference's own modules on synthetic checkpoints
(oracle/weights.py); the reference has no golden vectors of its own (SURVEY.md section 4).
"""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn.functional as F

from . import weights as W

WS = W.WINDOW


# ------------------------------------------------------------------------------------------------
# Swin-B backbone (model/backbone/swin_transformer.py)
# ------------------------------------------------------------------------------------------------
def window_partition(x, ws=WS):  # swin_transformer.py:39-51
    B, H, Wd, C = x.shape
    x = x.view(B, H // ws, ws, Wd // ws, ws, C)
    return x.permute(0, 1, 3, 2, 4, 5).contiguous().view(-1, ws, ws, C)


def window_reverse(windows, H, Wd, ws=WS):  # swin_transformer.py:54-68
    B = int(windows.shape[0] / (H * Wd / ws / ws))
    x = windows.view(B, H // ws, Wd // ws, ws, ws, -1)
    return x.permute(0, 1, 3, 2, 4, 5).contiguous().view(B, H, Wd, -1)


def shift_mask(H, Wd, ws=WS):  # swin_transformer.py:368-387
    shift = ws // 2
    Hp = int(np.ceil(H / ws)) * ws
    Wp = int(np.ceil(Wd / ws)) * ws
    img_mask = torch.zeros((1, Hp, Wp, 1))
    cnt = 0
    for h in (slice(0, -ws), slice(-ws, -shift), slice(-shift, None)):
        for w in (slice(0, -ws), slice(-ws, -shift), slice(-shift, None)):
            img_mask[:, h, w, :] = cnt
            cnt += 1
    mw = window_partition(img_mask).view(-1, ws * ws)
    am = mw.unsqueeze(1) - mw.unsqueeze(2)
    return am.masked_fill(am != 0, -100.0).masked_fill(am == 0, 0.0)


def window_attention(x, sd, p, heads, mask):  # swin_transformer.py:119-151
    B_, N, C = x.shape
    qkv = F.linear(x, sd[p + 'qkv.weight'], sd[p + 'qkv.bias'])
    qkv = qkv.reshape(B_, N, 3, heads, C // heads).permute(2, 0, 3, 1, 4)
    q, k, v = qkv[0], qkv[1], qkv[2]
    q = q * ((C // heads) ** -0.5)
    attn = q @ k.transpose(-2, -1)
    idx = W.relative_position_index().view(-1)
    bias = sd[p + 'relative_position_bias_table'][idx].view(N, N, -1).permute(2, 0, 1).contiguous()
    attn = attn + bias.unsqueeze(0)
    if mask is not None:
        nW = mask.shape[0]
        attn = attn.view(B_ // nW, nW, heads, N, N) + mask.unsqueeze(1).unsqueeze(0)
        attn = attn.view(-1, heads, N, N)
    attn = attn.softmax(dim=-1)
    x = (attn @ v).transpose(1, 2).reshape(B_, N, C)
    return F.linear(x, sd[p + 'proj.weight'], sd[p + 'proj.bias'])


def swin_block(x, H, Wd, sd, p, heads, shift, mask):  # swin_transformer.py:196-253
    B, L, C = x.shape
    shortcut = x
    x = F.layer_norm(x, (C,), sd[p + 'norm1.weight'], sd[p + 'norm1.bias'], 1e-5).view(B, H, Wd, C)
    pad_r = (WS - Wd % WS) % WS
    pad_b = (WS - H % WS) % WS
    x = F.pad(x, (0, 0, 0, pad_r, 0, pad_b))  # zero pad AFTER norm1: pad tokens are live keys
    Hp, Wp = x.shape[1], x.shape[2]
    if shift > 0:
        x = torch.roll(x, shifts=(-shift, -shift), dims=(1, 2))
    xw = window_partition(x).view(-1, WS * WS, C)
    aw = window_attention(xw, sd, p + 'attn.', heads, mask if shift > 0 else None)
    x = window_reverse(aw.view(-1, WS, WS, C), Hp, Wp)
    if shift > 0:
        x = torch.roll(x, shifts=(shift, shift), dims=(1, 2))
    x = x[:, :H, :Wd, :].contiguous().view(B, H * Wd, C)
    x = shortcut + x
    y = F.layer_norm(x, (C,), sd[p + 'norm2.weight'], sd[p + 'norm2.bias'], 1e-5)
    y = F.linear(y, sd[p + 'mlp.fc1.weight'], sd[p + 'mlp.fc1.bias'])
    y = F.gelu(y)  # exact erf GELU (nn.GELU default)
    y = F.linear(y, sd[p + 'mlp.fc2.weight'], sd[p + 'mlp.fc2.bias'])
    return x + y


def merge_concat(x, value=0):  # swin_transformer.py:279-291: [B,H,W,C] -> [B,ceil(H/2),ceil(W/2),4C]
    H, Wd = x.shape[1], x.shape[2]
    if H % 2 == 1 or Wd % 2 == 1:
        x = F.pad(x, (0, 0, 0, Wd % 2, 0, H % 2), value=value)
    return torch.cat([x[:, 0::2, 0::2], x[:, 1::2, 0::2], x[:, 0::2, 1::2], x[:, 1::2, 1::2]], -1)


def patch_merging(x, H, Wd, sd, p):  # swin_transformer.py:269-296
    B, L, C = x.shape
    x = merge_concat(x.view(B, H, Wd, C))
    x = x.view(B, -1, 4 * C)
    x = F.layer_norm(x, (4 * C,), sd[p + 'norm.weight'], sd[p + 'norm.bias'], 1e-5)
    return F.linear(x, sd[p + 'reduction.weight'])


def patch_pad(img):  # patch_embed's padding (swin_transformer.py:427-443): zero pad [B,3,H,W] to whole 4x4 patches
    _, _, H, Wd = img.shape
    if Wd % 4:
        img = F.pad(img, (0, 4 - Wd % 4))
    if H % 4:
        img = F.pad(img, (0, 0, 0, 4 - H % 4))
    return img


def patch_embed(img, sd, p):  # swin_transformer.py:427-443
    img = patch_pad(img)
    x = F.conv2d(img, sd[p + 'proj.weight'], sd[p + 'proj.bias'], stride=4)
    Wh, Ww = x.shape[2], x.shape[3]
    x = x.flatten(2).transpose(1, 2)
    x = F.layer_norm(x, (x.shape[-1],), sd[p + 'norm.weight'], sd[p + 'norm.bias'], 1e-5)
    return x, Wh, Ww


def swin_backbone(img, sd, prefix='backbone.0.', return_raw=False):
    """SwinTransformer.forward (swin_transformer.py:597-625) -> 4 NHWC feature maps (LN'd)."""
    x, H, Wd = patch_embed(img, sd, prefix + 'patch_embed.')
    outs, raws = [], []
    for s, (depth, heads) in enumerate(zip(W.SWIN_DEPTHS, W.SWIN_HEADS)):
        mask = shift_mask(H, Wd)
        for b in range(depth):
            x = swin_block(x, H, Wd, sd, f'{prefix}layers.{s}.blocks.{b}.', heads,
                           0 if b % 2 == 0 else WS // 2, mask)
        C = x.shape[-1]
        raws.append(x)
        o = F.layer_norm(x, (C,), sd[f'{prefix}norm{s}.weight'], sd[f'{prefix}norm{s}.bias'], 1e-5)
        outs.append(o.view(-1, H, Wd, C))
        if s < 3:
            x = patch_merging(x, H, Wd, sd, f'{prefix}layers.{s}.downsample.')
            H, Wd = (H + 1) // 2, (Wd + 1) // 2
    return (outs, raws) if return_raw else outs


# ------------------------------------------------------------------------------------------------
# neck: mask resize, sine position embedding, FPN, input_proj
# ------------------------------------------------------------------------------------------------
def level_mask(mask, size):  # swin_transformer.py:622 (nearest, legacy index rule)
    return F.interpolate(mask[None].float(), size=size).to(torch.bool)[0]


def position_embedding_sine(mask, num_pos_feats=256, temperature=10000):  # position_embedding.py:24-44
    not_mask = ~mask
    y_embed = not_mask.cumsum(1, dtype=torch.float32)
    x_embed = not_mask.cumsum(2, dtype=torch.float32)
    eps, scale = 1e-6, 2 * math.pi
    y_embed = y_embed / (y_embed[:, -1:, :] + eps) * scale
    x_embed = x_embed / (x_embed[:, :, -1:] + eps) * scale
    dim_t = torch.arange(num_pos_feats, dtype=torch.float32)
    dim_t = temperature ** (2 * (dim_t // 2) / num_pos_feats)
    pos_x = x_embed[:, :, :, None] / dim_t
    pos_y = y_embed[:, :, :, None] / dim_t
    pos_x = torch.stack((pos_x[:, :, :, 0::2].sin(), pos_x[:, :, :, 1::2].cos()), dim=4).flatten(3)
    pos_y = torch.stack((pos_y[:, :, :, 0::2].sin(), pos_y[:, :, :, 1::2].cos()), dim=4).flatten(3)
    return torch.cat((pos_y, pos_x), dim=3)  # NHWC [B,h,w,512]  (reference permutes to NCHW)


def fpn(feats_nhwc, sd):  # fpn.py:21-45 ; inputs/outputs NCHW inside, like the reference
    c2, c3, c4, c5 = [f.permute(0, 3, 1, 2).contiguous() for f in feats_nhwc]
    p5 = F.conv2d(c5, sd['fpn.fpn_in.0.weight'])
    p4 = F.conv2d(c4, sd['fpn.fpn_in.1.weight']) + F.interpolate(p5, size=c4.shape[2:], mode='nearest')
    p3 = F.conv2d(c3, sd['fpn.fpn_in.2.weight']) + F.interpolate(p4, size=c3.shape[2:], mode='nearest')
    p2 = F.conv2d(c2, sd['fpn.fpn_in.3.weight']) + F.interpolate(p3, size=c2.shape[2:], mode='nearest')
    return fpn_concat(p2, p3, p4, p5)


def fpn_concat(p2, p3, p4, p5):  # fpn.py:38-44: NCHW levels -> bilinear to p3's grid, concatenated
    size = p3.shape[2:]
    p2 = F.interpolate(p2, size=size, mode='bilinear')
    p4 = F.interpolate(p4, size=size, mode='bilinear')
    p5 = F.interpolate(p5, size=size, mode='bilinear')
    return torch.cat((p2, p3, p4, p5), dim=1)


def encode(img, mask, sd):
    """backbone -> FPN -> input_proj (omniparser.py:19-31).

    img [B,3,H,W] f32 (normalised), mask [B,H,W] bool (True = pad).
    Returns memory [B,M,512], pos [B,M,512], key-padding mask [B,M] (bool), (h, w).
    """
    feats = swin_backbone(img, sd)
    src = F.conv2d(fpn(feats, sd), sd['input_proj.weight'], sd['input_proj.bias'], stride=2)
    h, w = feats[2].shape[1], feats[2].shape[2]
    assert src.shape[2:] == (h, w), (src.shape, h, w)
    m = level_mask(mask, (h, w))
    pos = position_embedding_sine(m)
    memory = src.flatten(2).permute(0, 2, 1).contiguous()
    return memory, pos.reshape(pos.shape[0], h * w, -1).contiguous(), m.flatten(1), (h, w)


# ------------------------------------------------------------------------------------------------
# decoder (model/transformer.py) -- executed exactly like the reference: no KV cache, the whole
# prefix is re-run every step and the image memory is repeated per sequence.
# ------------------------------------------------------------------------------------------------
def _mha(query, key, value, sd, p, attn_mask=None, key_padding_mask=None, nhead=8):
    """nn.MultiheadAttention slow path as executed by torch 2.x with need_weights=True
    (torch/nn/functional.py multi_head_attention_forward): q scaled BEFORE q@k^T, float masks added.
    Tensors are [L, B, E] like the reference."""
    L, B, E = query.shape
    S = key.shape[0]
    hd = E // nhead
    w, b = sd[p + 'in_proj_weight'], sd[p + 'in_proj_bias']
    q = F.linear(query, w[:E], b[:E])
    k = F.linear(key, w[E:2 * E], b[E:2 * E])
    v = F.linear(value, w[2 * E:], b[2 * E:])
    q = q.view(L, B * nhead, hd).transpose(0, 1)
    k = k.view(S, B * nhead, hd).transpose(0, 1)
    v = v.view(S, B * nhead, hd).transpose(0, 1)
    mask = attn_mask
    if key_padding_mask is not None:
        kpm = torch.zeros(key_padding_mask.shape, dtype=q.dtype).masked_fill(key_padding_mask, float('-inf'))
        kpm = kpm.view(B, 1, 1, S).expand(-1, nhead, -1, -1).reshape(B * nhead, 1, S)
        mask = kpm if mask is None else mask + kpm
    q = q * (1.0 / math.sqrt(hd))
    attn = torch.baddbmm(mask, q, k.transpose(-2, -1)) if mask is not None else torch.bmm(q, k.transpose(-2, -1))
    attn = attn.softmax(dim=-1)
    out = torch.bmm(attn, v).transpose(0, 1).contiguous().view(L * B, E)
    out = F.linear(out, sd[p + 'out_proj.weight'], sd[p + 'out_proj.bias'])
    return out.view(L, B, E)


def _ln(x, sd, p):
    return F.layer_norm(x, (x.shape[-1],), sd[p + '.weight'], sd[p + '.bias'], 1e-5)


def decoder_layer_pre(tgt, memory, sd, p, tgt_mask, mem_kpm, pos, query_pos):  # transformer.py:430-454
    t2 = _ln(tgt, sd, p + 'norm1')
    q = k = t2 + query_pos
    tgt = tgt + _mha(q, k, t2, sd, p + 'self_attn.', attn_mask=tgt_mask)
    t2 = _ln(tgt, sd, p + 'norm2')
    tgt = tgt + _mha(t2 + query_pos, memory + pos, memory, sd, p + 'multihead_attn.', key_padding_mask=mem_kpm)
    t2 = _ln(tgt, sd, p + 'norm3')
    t2 = F.linear(F.relu(F.linear(t2, sd[p + 'linear1.weight'], sd[p + 'linear1.bias'])),
                  sd[p + 'linear2.weight'], sd[p + 'linear2.bias'])
    return tgt + t2


def causal_mask(sz, dtype=torch.float32):  # transformer.py:331-337
    m = (torch.triu(torch.ones(sz, sz)) == 1).transpose(0, 1)
    return m.to(dtype).masked_fill(m == 0, float('-inf')).masked_fill(m == 1, 0.0)


def decode_logits(seq, memory, mem_kpm, pos, sd, kind):
    """Transformer.decode (transformer.py:74-100) for ONE image: seq int64 [Bs, t] ->
    logits [Bs, t, V].  memory/pos [M,512], mem_kpm [M] bool; repeated per sequence like :88-96.  Runs in the dtype of
    memory and the state dict (float64 for the tests' high-precision reference)."""
    t = 'transformer.'
    Bs, T = seq.shape
    emb = sd[t + 'embedding.word_embeddings.weight'][seq]          # transformer.py:313
    pe = sd[t + f'embedding.{kind}_position_embeddings.weight'][:T]  # :315-320
    pe = pe.unsqueeze(0).repeat(Bs, 1, 1)
    x = _ln(emb + pe, sd, t + 'embedding.LayerNorm')               # :324-325
    tgt = x.permute(1, 0, 2)
    qpos = pe.permute(1, 0, 2)
    mem = memory[:, None, :].repeat(1, Bs, 1)
    ps = pos[:, None, :].repeat(1, Bs, 1)
    kpm = mem_kpm[None, :].repeat(Bs, 1)
    tm = causal_mask(T, x.dtype)
    for l in range(W.DEC_LAYERS):
        tgt = decoder_layer_pre(tgt, mem, sd, f'{t}{kind}_decoder.layers.{l}.', tm, kpm, ps, qpos)
    tgt = _ln(tgt, sd, f'{t}{kind}_decoder.norm')                  # shared final LN, :369-370
    h = tgt.transpose(0, 1)
    q = f'{t}{kind}_pred_layer.layers.'
    h = F.relu(F.linear(h, sd[q + '0.weight'], sd[q + '0.bias']))  # block/mlp.py:11-13
    h = F.relu(F.linear(h, sd[q + '1.weight'], sd[q + '1.bias']))
    return F.linear(h, sd[q + '2.weight'], sd[q + '2.bias'])


def default_prompts(use_char_window_prompt=True):  # engine/val.py:25-31
    if use_char_window_prompt:
        pt = [0, 0, W.NUM_BINS - 1, W.NUM_BINS - 1, W.NUM_BINS, W.NUM_BINS + len(W.CHARS), W.PT_SOS]
    else:
        pt = [0, 0, W.NUM_BINS - 1, W.NUM_BINS - 1, W.PT_SOS]
    return (torch.tensor([pt], dtype=torch.long), torch.tensor([[W.POLY_SOS]], dtype=torch.long),
            torch.tensor([[W.REC_SOS]], dtype=torch.long))


def greedy_text_spotting(memory, mem_kpm, pos, sd, pt_prompt, pt_seq_length, rec_length=25,
                         return_logits=False):
    """Transformer.forward eval branch for text spotting (transformer.py:234-286) for ONE image.

    Returns None when no point is produced (:240-241), else
    ``([pt[1,2N], poly[1,32N], rec[1,N,rec_length]] int64, [rec_probs[N,rec_length]])`` and, when
    ``return_logits``, the per-step last-position logits of the three loops.
    """
    nb, eos = W.NUM_BINS, W.PT_EOS
    n_prompt = pt_prompt.shape[1]
    logs = {'pt': [], 'poly': [], 'rec': []}
    pt_seq = pt_prompt
    for i in range(pt_seq_length):                                  # decode_pt_seq, :102-141
        lg = decode_logits(pt_seq, memory, mem_kpm, pos, sd, 'pt')[:, -1, :]
        logs['pt'].append(lg)
        out = lg.softmax(-1)
        if i % 2 == 0:
            out[:, nb:eos] = 0
            out[:, eos + 1:] = 0
        else:
            out = out[:, :nb]
        _, extra = out.topk(dim=-1, k=1)
        if extra[0] == eos:
            break
        pt_seq = torch.cat([pt_seq, extra], dim=-1)
    pt_seq = pt_seq[:, n_prompt:]
    if pt_seq.shape[1] % 2 != 0:
        pt_seq = pt_seq[:, :-1]
    pt_seq = pt_seq[0]
    if pt_seq.numel() == 0:
        return (None, logs) if return_logits else None
    pt_seq = pt_seq.reshape(-1, 2)
    n = pt_seq.shape[0]
    poly_seq = torch.cat((pt_seq, torch.full((n, 1), W.POLY_SOS, dtype=torch.long)), dim=-1)
    for _ in range(32):                                             # :254-263
        lg = decode_logits(poly_seq, memory, mem_kpm, pos, sd, 'poly')[:, -1, :]
        logs['poly'].append(lg)
        out = lg.softmax(-1)[:, :nb]
        _, extra = out.topk(dim=-1, k=1)
        poly_seq = torch.cat([poly_seq, extra], dim=-1)
    poly_seq = poly_seq[:, 3:35]
    rec_seq = torch.cat((pt_seq, torch.full((n, 1), W.REC_SOS, dtype=torch.long)), dim=-1)
    rec_probs = []
    for _ in range(rec_length):                                     # :270-282
        lg = decode_logits(rec_seq, memory, mem_kpm, pos, sd, 'rec')[:, -1, :]
        logs['rec'].append(lg)
        out = lg.softmax(-1)
        out[:, :nb] = 0
        out[:, W.PT_EOS] = 0
        out[:, W.POLY_EOS] = 0
        out[:, W.REC_EOS + 1:] = 0
        prob, extra = out.topk(dim=-1, k=1)
        rec_seq = torch.cat([rec_seq, extra], dim=-1)
        rec_probs.append(prob)
    rec_seq = rec_seq[:, 3:].unsqueeze(0)
    res = ([pt_seq.reshape(1, -1), poly_seq.reshape(1, -1), rec_seq], [torch.cat(rec_probs, dim=-1)])
    return (res, logs) if return_logits else res


def greedy_min_gaps(logs):
    """Smallest top-1 / top-2 LOGIT gap among the candidates each greedy step may pick (pt: bins, + pt_eos on even
    steps; poly: bins; rec: chars, pad and rec_eos -- transformer.py:110-123,257-259,274-278) for the per-step logits
    returned by ``greedy_text_spotting(..., return_logits=True)``.  A fixture whose gaps are all far above the CUDA
    path's logit error (~1e-5) admits no near-tie excuse: its ids must match bit for bit."""
    nb = W.NUM_BINS
    out = {}
    for kind, steps in logs.items():
        g = float('inf')
        for i, lg in enumerate(steps):
            a = torch.zeros(lg.shape[-1], dtype=torch.bool)
            if kind == 'pt':
                a[:nb] = True
                if i % 2 == 0:
                    a[W.PT_EOS] = True
            elif kind == 'poly':
                a[:nb] = True
            else:
                a[nb:W.PT_EOS] = True
                a[W.REC_EOS] = True
            top = lg.masked_fill(~a, float('-inf')).topk(2, dim=-1).values
            g = min(g, float((top[:, 0] - top[:, 1]).min()))
        out[kind] = g
    return out


def step_candidates(kind, step, V):
    """Ids a greedy step may emit (transformer.py:110-123,257-259,274-278); text spotting."""
    a = torch.zeros(V, dtype=torch.bool)
    nb = W.NUM_BINS
    if kind == 'pt':
        a[:nb] = True
        if step % 2 == 0:
            a[W.PT_EOS] = True
    elif kind == 'poly':
        a[:nb] = True
    else:
        a[nb:W.PT_EOS] = True
        a[W.REC_EOS] = True
    return a


def teacher_forced_gaps(memory, mem_kpm, pos, sd, pt_prompt, pt, poly, rec):
    """One teacher-forced pass per loop over given greedy outputs (pt [1,2N], poly [1,32N], rec [1,N,L]): for every
    generated token the top-1 / top-2 gap among the step's candidates, and whether the restatement's argmax equals the
    given id everywhere.  Because prefix states are invariant under the causal mask (SURVEY F5) this reproduces the
    no-cache greedy loops step for step.  Returns {kind: (gaps [n_seq, steps], all_equal)}."""
    n = pt.numel() // 2
    n_prompt = pt_prompt.shape[1]
    full = {'pt': torch.cat([pt_prompt, pt.reshape(1, -1)], 1),
            'poly': torch.cat([pt.reshape(-1, 2), torch.full((n, 1), W.POLY_SOS, dtype=torch.long), poly.reshape(n, -1)], 1),
            'rec': torch.cat([pt.reshape(-1, 2), torch.full((n, 1), W.REC_SOS, dtype=torch.long), rec.reshape(n, -1)], 1)}
    start = {'pt': n_prompt, 'poly': 3, 'rec': 3}
    out = {}
    for kind, seq in full.items():
        lg = decode_logits(seq, memory, mem_kpm, pos, sd, kind)
        s0 = start[kind]
        steps = seq.shape[1] - s0
        gaps = torch.zeros(seq.shape[0], steps)
        ok = True
        for t in range(steps):
            a = step_candidates(kind, t, lg.shape[-1])
            top = lg[:, s0 - 1 + t].masked_fill(~a, float('-inf')).topk(2, dim=-1)
            gaps[:, t] = top.values[:, 0] - top.values[:, 1]
            ok = ok and bool((top.indices[:, 0] == seq[:, s0 + t]).all())
        out[kind] = (gaps, ok)
    return out


def greedy_kie(memory, mem_kpm, pos, sd, pt_prompt, pt_seq_length, rec_length, vie, image_size, classes):
    """KIE eval branch for ONE image: decode_pt_seq with infer_vie (transformer.py:102-141, :117-123) followed by
    decode_vie_pt_poly_rec_seq (:143-217).  Returns None when no token is produced, else the reference's
    ``[(text, class_name, prob, [[x0,y0,x1,y1], ...]), ...]``; second value = raw (pt_seq, pt_probs)."""
    nb, eos = W.NUM_BINS, W.PT_EOS
    n_prompt = pt_prompt.shape[1]
    pt_seq, pt_probs = pt_prompt, []
    for i in range(pt_seq_length):
        out = decode_logits(pt_seq, memory, mem_kpm, pos, sd, 'pt')[:, -1, :].softmax(-1)
        if i % 3 == 0:
            out[:, nb:eos] = 0
            out[:, eos + 1:] = 0
        elif i % 3 == 1:
            out = out[:, :nb]
        else:
            out[:, :-vie] = 0
        prob, extra = out.topk(dim=-1, k=1)
        if extra[0] == eos:
            break
        pt_seq = torch.cat([pt_seq, extra], dim=-1)
        pt_probs.append(prob)
    pt_seq = pt_seq[:, n_prompt:]
    if pt_seq.shape[1] % 2 != 0:
        pt_seq = pt_seq[:, :-1]
    pt_seq = pt_seq[0]
    if pt_seq.numel() == 0:
        return None, (pt_seq, pt_probs)
    image_h, image_w = image_size
    result, tmp_recog, tmp_rect = [], [], []
    i = 0
    while i < len(pt_seq):
        if pt_seq[i].item() < nb:
            if i + 1 <= len(pt_seq) - 1 and pt_seq[i + 1].item() < nb:
                poly_seq = torch.cat((pt_seq[i:i + 2].unsqueeze(0), torch.tensor([[W.POLY_SOS]])), dim=-1)
                for _ in range(32):
                    lg = decode_logits(poly_seq, memory, mem_kpm, pos, sd, 'poly')[:, -1, :-vie]
                    _, extra = lg.softmax(-1)[:, :nb].topk(dim=-1, k=1)
                    poly_seq = torch.cat([poly_seq, extra], dim=-1)
                pts = poly_seq[0, 3:35].reshape(-1, 2)
                rect = [image_w * pts[:, 0].min().item() / nb, image_h * pts[:, 1].min().item() / nb,
                        image_w * pts[:, 0].max().item() / nb, image_h * pts[:, 1].max().item() / nb]
                rec_seq = torch.cat((pt_seq[i:i + 2].unsqueeze(0), torch.tensor([[W.REC_SOS]])), dim=-1)
                for _ in range(rec_length):
                    out = decode_logits(rec_seq, memory, mem_kpm, pos, sd, 'rec')[:, -1, :-vie].softmax(-1)
                    out[:, :nb] = 0
                    out[:, W.PT_EOS] = 0
                    out[:, W.POLY_EOS] = 0
                    out[:, W.REC_EOS + 1:] = 0
                    _, extra = out.topk(dim=-1, k=1)
                    rec_seq = torch.cat([rec_seq, extra], dim=-1)
                recog = []
                for tok in rec_seq[0, 3:].tolist():
                    if tok == W.RECOG_PAD or tok == W.REC_EOS:
                        break
                    if tok == W.RECOG_PAD - 1:
                        continue
                    recog.append(W.CHARS[tok - nb])
                tmp_recog.append(''.join(recog))
                tmp_rect.append(rect)
                i += 2
            else:
                i += 1
        else:
            result.append((' '.join(tmp_recog), classes[pt_seq[i].item() - W.PADDING - 1], pt_probs[i].item(), tmp_rect))
            i += 1
            tmp_recog, tmp_rect = [], []
    return result, (pt_seq, pt_probs)


def forward(img, mask, sd, pt_seq_length, rec_length=25, use_char_window_prompt=True):
    """OmniParser.forward (omniparser.py:19-32) for a batch of independent batch-1 problems
    (the reference only supports batch 1, engine/val.py:22).  Returns a list per image."""
    memory, pos, kpm, _ = encode(img, mask, sd)
    pt_prompt, _, _ = default_prompts(use_char_window_prompt)
    return [greedy_text_spotting(memory[b], kpm[b], pos[b], sd, pt_prompt, pt_seq_length, rec_length)
            for b in range(img.shape[0])]


# ------------------------------------------------------------------------------------------------
# post-processing (engine/val.py:70-100, utils/misc.py:147-189)
# ------------------------------------------------------------------------------------------------
def decode_rec_strings(rec_seq, rec_probs):
    """ids [N,L] + probs [N,L] -> (strings, confidences) following utils/misc.py:164-185."""
    texts, confs = [], []
    for ids, pr in zip(rec_seq.tolist(), rec_probs.tolist()):
        chars, ps = [], []
        for tok, p in zip(ids, pr):
            if tok == W.RECOG_PAD or tok == W.REC_EOS:
                break
            if tok == W.RECOG_PAD - 1:
                continue
            chars.append(W.CHARS[tok - W.NUM_BINS])
            ps.append(p)
        texts.append(''.join(chars))
        confs.append(sum(ps) / (len(ps) + 1e-5))
    return texts, confs
