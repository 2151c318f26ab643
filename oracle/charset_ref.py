"""Caller character sets in the recognition loop (DESIGN 4.23): a restatement of the reference's greedy recognition
loop (model/transformer.py:266-283; the KIE loop at :171-186) with the set's mask applied after the reference's own
zeroing of the non-character classes.  The reference convention is softmax, then mask, then top-1: the probability of
a chosen class stays its probability under the unconstrained softmax.
"""
from __future__ import annotations

import torch

from oracle import omniparser_ref as O
from oracle import weights as W


def charset_mask(text, chars=W.CHARS) -> torch.Tensor:
    """bool [len(chars)]: chars[i] in text (None: every character)."""
    return torch.tensor([text is None or c in text for c in chars], dtype=torch.bool)


def allowed_classes(V: int, cs: torch.Tensor) -> torch.Tensor:
    """bool [n, V]: the classes a constrained rec step may choose for each row's character mask cs [n, len(CHARS)] --
    the characters of the set, the unknown class RECOG_PAD - 1, RECOG_PAD and REC_EOS."""
    nb, n = W.NUM_BINS, cs.shape[0]
    a = torch.zeros(n, V, dtype=torch.bool)
    a[:, nb:W.PT_EOS] = True            # characters, unknown, pad (transformer.py:274-278)
    a[:, W.REC_EOS] = True
    a[:, nb:nb + len(W.CHARS)] &= cs
    return a


def rec_loop(memory, mem_kpm, pos, sd, pts, rec_length, cs=None, vie=0):
    """The greedy recognition loop from [x, y, rec_sos] for each point of pts int64 [n, 2], each row restricted to
    its characters cs bool [n, len(CHARS)] (None: no set).  vie > 0: the KIE loop, softmax over logits[:-vie].
    Returns (rec int64 [n, rec_length], probs f32 [n, rec_length], gaps f32 [n, rec_length]: the top-1 / top-2 logit
    gap among each step's allowed classes)."""
    nb, n = W.NUM_BINS, pts.shape[0]
    rec_seq = torch.cat((pts, torch.full((n, 1), W.REC_SOS, dtype=torch.long)), dim=-1)
    probs, gaps = [], []
    for _ in range(rec_length):
        lg = O.decode_logits(rec_seq, memory, mem_kpm, pos, sd, 'rec')[:, -1, :]
        if vie:
            lg = lg[:, :-vie]
        out = lg.softmax(-1)
        out[:, :nb] = 0                  # the reference's zeroing (transformer.py:274-278)
        out[:, W.PT_EOS] = 0
        out[:, W.POLY_EOS] = 0
        out[:, W.REC_EOS + 1:] = 0
        if cs is not None:               # then the caller's set: characters outside it
            out[:, nb:nb + len(W.CHARS)] = out[:, nb:nb + len(W.CHARS)].masked_fill(~cs, 0)
        prob, extra = out.topk(dim=-1, k=1)
        a = allowed_classes(lg.shape[-1], cs if cs is not None else torch.ones(n, len(W.CHARS), dtype=torch.bool))
        top = lg.masked_fill(~a, float('-inf')).topk(2, dim=-1)
        assert torch.equal(top.indices[:, :1], extra), 'softmax-then-mask and masked argmax disagree'
        gaps.append(top.values[:, 0] - top.values[:, 1])
        rec_seq = torch.cat([rec_seq, extra], dim=-1)
        probs.append(prob)
    return rec_seq[:, 3:], torch.cat(probs, dim=-1), torch.stack(gaps, dim=-1)


def rec_text(ids) -> str:
    """decode_seq's text of one rec row (transformer.py:187-203): up to pad / rec_eos, the unknown class dropped."""
    out = []
    for t in ids:
        t = int(t)
        if t == W.RECOG_PAD or t == W.REC_EOS:
            break
        if t != W.RECOG_PAD - 1:
            out.append(W.CHARS[t - W.NUM_BINS])
    return ''.join(out)
