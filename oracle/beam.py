"""Oracle (test infrastructure): CTC prefix beam search without a language model — PARITY UNPINNED.

The reference delegates ``ctc_beam_search`` to the external, un-vendored, absent ``paddlespeech_ctcdecoders`` SWIG/C++
library (masr/decoders/swig_wrapper.py:1,35-64; call sites masr/decoders/beam_search_decoder.py:45-56,75-91; version
unpinned: ``pip install paddlespeech_ctcdecoders -U``, docs/beam_search.md:5) plus a 2.8 GB KenLM file fetched at run
time (:19-25).  Neither the library, its source nor the LM exist in /root/reference or in this image, and no reference
test pins its results, so this restatement follows the algorithm's *public definition* (DeepSpeech2-style prefix beam
search, SURVEY.md Appendix D) with the parameters MASR passes (beam_size=300, cutoff_prob=0.99, cutoff_top_n=40,
blank_id=0, configs/conformer.yml:74-88) and scorer=None.  It is validated against itself (beam=1 on one-hot posteriors ==
greedy, score monotonicity, exact agreement with the CUDA implementation) and against a float64 CTC forward: where no live
prefix is pruned, every beam entry's score equals the forward of its prefix to 2.0e-7 (tests/test_gpu_beam_contract.py).

Definition used (log domain, natural log):
  per frame  : candidates = the tokens, sorted by probability (descending, ties by lower id), of the shortest prefix of
               that order whose cumulative mass >= cutoff_prob, capped at cutoff_top_n;  logp_c = log(p_c)
  per prefix : p_b (ends in blank), p_nb (ends in non-blank); root: p_b = 0, p_nb = -inf; score = p_b (+) p_nb
               blank c         : p_b'(l)   (+)= score(l) + logp_c
               c == last(l)    : p_nb'(l)  (+)= p_nb(l) + logp_c ;  p_nb'(l+c) (+)= p_b(l) + logp_c
               otherwise       : p_nb'(l+c) (+)= score(l) + logp_c
  prune      : keep the beam_size best prefixes by score' (ties: earlier-created prefix first)
  result     : prefixes best-first as (score, token ids); MASR takes element 0 (beam_search_decoder.py:56).
The library's early-exit heuristic (`min_cutoff`) is an optimisation and is not modelled.
"""
from __future__ import annotations

import math
from typing import Dict, List, Sequence, Tuple

import numpy as np

NEG_INF = -float("inf")


# ---- log-sum-exp in a SPECIFIED sequence of IEEE float32 operations --------------------------------------------------------
# A pruned beam search over hundreds of frames amplifies a 1-ulp difference in any score into a different beam (near-tied
# hypotheses swap ranks at the pruning boundary), so "the GPU kernel equals this restatement" is only testable if both evaluate
# log(exp(a) + exp(b)) with the SAME rounding at every step.  libm's / CUDA's expf, log1pf differ in the last bit, so the
# function is defined here operation by operation (one correctly rounded float32 +, -, *, / or round-to-nearest-even per
# line; no fused multiply-add) and csrc/beam.cu evaluates exactly this sequence with __fmul_rn / __fadd_rn / __fdiv_rn.
# Accuracy against float64 (tests/test_gpu_beam_contract.py): exp32_det 4 ulp and log1p32_det 3.2 ulp relative, logaddexp32
# 1 ulp of 1 + |result| — irrelevant for the search; determinism is the point.
_F = np.float32
_LOG2E, _LN2_HI, _LN2_LO = _F(1.4426950408889634), _F(0.693145751953125), _F(1.42860682030941723212e-6)
_EXP_C = [_F(1.0 / 720.0), _F(1.0 / 120.0), _F(1.0 / 24.0), _F(1.0 / 6.0), _F(0.5), _F(1.0), _F(1.0)]
_ATANH_C = [_F(2.0 / 17.0), _F(2.0 / 15.0), _F(2.0 / 13.0), _F(2.0 / 11.0), _F(2.0 / 9.0), _F(2.0 / 7.0), _F(2.0 / 5.0), _F(2.0 / 3.0), _F(2.0)]


def exp32_det(d: np.float32) -> np.float32:
    """exp(d) for d <= 0: n = rint(d log2 e); r = d - n ln2 (two-step); degree-6 Horner; scale by 2^n."""
    d = _F(d)
    if d < _F(-87.0):
        return _F(0.0)
    n = np.rint(_F(d * _LOG2E))
    r = _F(d - _F(n * _LN2_HI))
    r = _F(r - _F(n * _LN2_LO))
    p = _EXP_C[0]
    for c in _EXP_C[1:]:
        p = _F(_F(p * r) + c)
    return _F(p * np.ldexp(_F(1.0), int(n)))


def log1p32_det(u: np.float32) -> np.float32:
    """log(1 + u) for 0 <= u <= 1 as 2 atanh(u / (2 + u)): s = u / (2 + u); z = s s; s * P(z), P of degree 8 in z."""
    u = _F(u)
    s = _F(u / _F(_F(2.0) + u))
    z = _F(s * s)
    p = _ATANH_C[0]
    for c in _ATANH_C[1:]:
        p = _F(_F(p * z) + c)
    return _F(s * p)


def logaddexp32(a: np.float32, b: np.float32) -> np.float32:
    """float32 log-sum-exp exactly as the CUDA kernel evaluates it: max + log1p_det(exp_det(min - max))."""
    a, b = _F(a), _F(b)
    if a == NEG_INF:
        return b
    if b == NEG_INF:
        return a
    hi, lo = (a, b) if a >= b else (b, a)
    return _F(hi + log1p32_det(exp32_det(_F(lo - hi))))


def prune_frame(p: np.ndarray, cutoff_prob: float, cutoff_top_n: int) -> List[Tuple[int, np.float32]]:
    """-> [(token id, float32 probability)] kept for this frame, best first."""
    order = np.lexsort((np.arange(p.shape[0]), -p.astype(np.float64)))       # prob descending, id ascending on ties
    keep, cum = [], np.float32(0.0)
    for idx in order[:cutoff_top_n]:
        keep.append((int(idx), np.float32(p[idx])))
        cum = np.float32(cum + np.float32(p[idx]))
        if cum >= np.float32(cutoff_prob):
            break
    return keep


def prefix_beam_search(probs: np.ndarray, beam_size: int = 300, cutoff_prob: float = 0.99, cutoff_top_n: int = 40,
                       blank: int = 0, nbest: int = 1, cands_per_frame=None):
    """probs [T, V] float32 posteriors -> list of (score float, token id list), best first.
    ``cands_per_frame`` (optional): per frame the already pruned candidate list [(token id, float32 log-probability)] — e.g.
    the output of the CUDA top-k kernel — so that the SEARCH can be compared bit for bit (``probs`` is then only used for T)."""
    # a prefix is identified by a node id in a trie: node -> (parent node, last token); root = 0
    parent, last = [-1], [-1]
    child: Dict[Tuple[int, int], int] = {}
    beam = [(0, np.float32(0.0), np.float32(NEG_INF))]                       # (node, p_b, p_nb), best first
    for t in range(probs.shape[0]):
        if cands_per_frame is not None:
            cands = [(int(c), np.float32(lp)) for c, lp in cands_per_frame[t]]
        else:
            cands = [(c, np.float32(math.log(float(pc)))) for c, pc in prune_frame(probs[t], cutoff_prob, cutoff_top_n)
                     if pc > 0]
        new_b: Dict[int, np.float32] = {}
        new_nb: Dict[int, np.float32] = {}
        order: List[int] = []                                                # creation / first-touch order for tie-breaks

        def touch(node):
            if node not in new_b:
                new_b[node], new_nb[node] = np.float32(NEG_INF), np.float32(NEG_INF)
                order.append(node)

        for node, pb, pnb in beam:                                           # existing prefixes keep their rank order
            touch(node)
        for node, pb, pnb in beam:
            score = logaddexp32(pb, pnb)
            for c, lp in cands:
                if c == blank:
                    new_b[node] = logaddexp32(new_b[node], np.float32(score + lp))
                    continue
                if c == last[node]:
                    new_nb[node] = logaddexp32(new_nb[node], np.float32(pnb + lp))
                    add = np.float32(pb + lp) if pb != NEG_INF else np.float32(NEG_INF)
                else:
                    add = np.float32(score + lp)
                if add == NEG_INF:
                    continue
                key = (node, c)
                ch = child.get(key)
                if ch is None:
                    ch = len(parent)
                    parent.append(node)
                    last.append(c)
                    child[key] = ch
                touch(ch)
                new_nb[ch] = logaddexp32(new_nb[ch], add)
        scored = []
        for rank, node in enumerate(order):
            s = logaddexp32(new_b[node], new_nb[node])
            if s != NEG_INF:
                scored.append((-float(s), rank, node))
        scored.sort()
        beam = [(node, new_b[node], new_nb[node]) for _, _, node in scored[:beam_size]]
    out = []
    for node, pb, pnb in beam[:nbest]:
        toks = []
        n = node
        while n > 0:
            toks.append(last[n])
            n = parent[n]
        out.append((float(logaddexp32(pb, pnb)), toks[::-1]))
    return out
