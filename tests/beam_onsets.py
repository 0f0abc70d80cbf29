"""Token onsets of the CPU restatements of the prefix beam search (oracle/beam.py, oracle/lm.py, oracle/word_lm.py), stated
from their definition and nothing else: a token's onset is the first frame t after whose selection the prefix ending in
that token was in the beam.  The restatements themselves are used unchanged: the beam after frame t is what they return
with nbest = beam_size over frames [0, t] (plain and character LM: one run per frame, O(T^2), so keep T and the beam
small), or the beam ``WordLmSearch`` holds after t + 1 one-frame pushes (word LM).  A prefix is identified by its tokens,
which is what a trie node stands for, so a prefix that leaves the beam and comes back keeps its first onset."""
from typing import Dict, List, Sequence, Tuple

import numpy as np

from oracle import beam as obeam, lm as olm, word_lm as owl


def beams(mode: str, frames, blps=None, beam: int = 16, lm=None, vocab=None, alpha: float = 0.0,
          beta: float = 0.0) -> Tuple[List[List[Tuple[int, ...]]], List[int]]:
    """-> (per frame t the prefixes of the post-selection beam, rank order; the reported best prefix after the last frame).
    ``mode``: "plain" (no LM), "char" (``lm`` an ``oracle.lm.ArpaLM``) or "word" (``lm`` an ``oracle.word_lm.WordLM``)."""
    T, out = len(frames), []
    if mode == "word":
        s = owl.WordLmSearch(lm, alpha, beta, beam)
        for t in range(T):
            s.push(frames[t:t + 1], blps[t:t + 1])
            out.append([tuple(s.toks_of[n]) for n, _, _ in s.beam])
        r = s.result(1)
        return out, (list(r[0][2]) if r else [])
    for t in range(1, T + 1):
        if mode == "plain":
            res = [toks for _, toks in obeam.prefix_beam_search(np.zeros((t, 1)), beam_size=beam, nbest=beam,
                                                                  cands_per_frame=frames[:t])]
        else:
            res = [toks for _, _, toks in olm.prefix_beam_search_lm(np.zeros((t, 1)), lm, vocab, alpha, beta, beam_size=beam,
                                                                     nbest=beam, cands_per_frame=frames[:t],
                                                                     blank_logp_per_frame=blps[:t])]
        out.append([tuple(x) for x in res])
    return out, (list(out[-1][0]) if out and out[-1] else [])


def first_frames(per_frame: Sequence[Sequence[Tuple[int, ...]]]) -> Dict[Tuple[int, ...], int]:
    """prefix -> the first frame it was in the beam."""
    first: Dict[Tuple[int, ...], int] = {}
    for t, bm in enumerate(per_frame):
        for p in bm:
            first.setdefault(p, t)
    return first


def onsets(per_frame, toks: Sequence[int]) -> List[int]:
    """The onset frame of every token of ``toks`` (a prefix that was in the beam, so all its prefixes were too)."""
    first = first_frames(per_frame)
    return [first[tuple(toks[:i + 1])] for i in range(len(toks))]


def best_onsets(mode: str, frames, blps=None, beam: int = 16, lm=None, vocab=None, alpha: float = 0.0,
                beta: float = 0.0) -> Tuple[List[int], List[int]]:
    """The restatement's reported prefix and its tokens' onsets."""
    per_frame, best = beams(mode, frames, blps, beam, lm, vocab, alpha, beta)
    return best, onsets(per_frame, best)
