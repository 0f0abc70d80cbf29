"""Oracle (test infrastructure): hotword biasing of the CTC prefix beam search, restated over strings.

A hotword is a token sequence.  The credit of a prefix is a function of its tokens, computed by stepping a state that is
the current match (a tuple of tokens that prefixes some hotword) — with no automaton arrays: a node is any prefix of a
hotword (set membership), a child is a node one token longer, fail(n) the longest proper suffix of n that is a node,
ta(n) the longest prefix of n (n included) that is a whole hotword, tail(n) the longest suffix of what follows ta(n) in n
that is a node (the state the matcher reaches from the root on those tokens), acc(n) = float32(w) * len(n).

One step from state s by token c (bank: float32, from 0):
    cur = s; loop: cur + (c,) a node -> nxt = it; cur = () -> nxt = (); ta(cur) -> bank += acc(ta(cur)), cur = tail(cur);
    else cur = fail(cur).   delta = (bank + acc(nxt)) - acc(s);  next = () if no hotword extends nxt else nxt.
fin(s) = the bank of the same loop with a token that extends nothing; the read-out of a state is fin(s) - acc(s).

In the search (``prefix_beam_search_hot``, ``WordLmSearchHot``): every extension by a non-blank token with a finite base
adds delta after the LM terms, ((base + alpha lnP) + beta) + delta; stay transitions and the min_cutoff test see no
credit; the entry reported is the best by (fused (+ word read-out)) + read-out, and its reported score is that minus C,
C = (the float32 left-to-right sum of its tokens' deltas) + its read-out.  With no hotwords both equal oracle.lm /
oracle.word_lm exactly.  Every + and * is one float32 rounding."""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from oracle.beam import NEG_INF, logaddexp32, prune_frame
from oracle.word_lm import AFTER_SPACE, ROOT, WordLmSearch

_F = np.float32


class HotwordMatcher:
    """The credit rule of a list of hotwords (token tuples) at ``w`` per token."""

    def __init__(self, hotwords: Sequence[Sequence[int]], w: float):
        self.words = {tuple(h) for h in hotwords}
        self.nodes = {h[:i] for h in self.words for i in range(len(h) + 1)}
        self.w = _F(w)

    def acc(self, n) -> np.float32:
        return _F(self.w * _F(len(n)))

    def leaf(self, n) -> bool:
        return not any(len(m) == len(n) + 1 and m[:len(n)] == n for m in self.nodes)

    def fail(self, n):
        for i in range(1, len(n) + 1):
            if n[i:] in self.nodes:
                return n[i:]
        return ()

    def ta(self, n):
        for i in range(len(n), 0, -1):
            if n[:i] in self.words:
                return n[:i]
        return None

    def tail(self, n):
        rest = n[len(self.ta(n)):]
        for i in range(len(rest) + 1):
            if rest[i:] in self.nodes:
                return rest[i:]
        return ()

    def _walk(self, s, c):
        bank, cur = _F(0.0), s
        while True:
            if c is not None and cur + (c,) in self.nodes:
                return bank, cur + (c,)
            if cur == ():
                return bank, ()
            t = self.ta(cur)
            if t is not None:
                bank = _F(bank + self.acc(t))
                cur = self.tail(cur)
            else:
                cur = self.fail(cur)

    def step(self, s, c):
        """-> (delta, next state)."""
        bank, nxt = self._walk(s, c)
        delta = _F(_F(bank + self.acc(nxt)) - self.acc(s))
        return delta, (() if self.leaf(nxt) else nxt)

    def readout(self, s) -> np.float32:
        return _F(self._walk(s, None)[0] - self.acc(s))

    def credit(self, toks) -> Tuple[np.float32, tuple]:
        """C of a token sequence: the float32 in-order sum of its deltas plus the read-out of the state it ends in."""
        c, s = _F(0.0), ()
        for t in toks:
            d, s = self.step(s, t)
            c = _F(c + d)
        return _F(c + self.readout(s)), s


def prefix_beam_search_hot(probs, lm, vocab, alpha: float = 0.0, beta: float = 0.0, beam_size: int = 300,
                           cutoff_prob: float = 0.99, cutoff_top_n: int = 40, blank: int = 0, nbest: int = 1,
                           cands_per_frame=None, blank_logp_per_frame=None, min_cutoff: bool = True,
                           hotwords: Optional[HotwordMatcher] = None):
    """``oracle.lm.prefix_beam_search_lm`` (``lm`` None or an ArpaLM) with hotword credit -> list of (fused score without
    credit, approx, token ids), best first by the selection score."""
    alpha, beta = _F(alpha), _F(beta)
    H = hotwords
    parent, last = [-1], [-1]
    child: Dict[Tuple[int, int], int] = {}
    toks_of: List[Tuple[int, ...]] = [()]
    hs: List[tuple] = [()]
    lnp_memo: Dict[Tuple[int, int], np.float32] = {}

    def lnp_ext(node, c):
        key = (node, c)
        if key not in lnp_memo:
            lnp_memo[key] = lm.lnp(lm.window([vocab[t] for t in toks_of[node]]), vocab[c])
        return lnp_memo[key]

    T = len(cands_per_frame) if cands_per_frame is not None else probs.shape[0]
    beam = [(0, _F(0.0), _F(NEG_INF))]
    for t in range(T):
        if cands_per_frame is not None:
            cands = [(int(c), _F(lp)) for c, lp in cands_per_frame[t]]
        else:
            cands = [(c, _F(math.log(float(pc)))) for c, pc in prune_frame(probs[t], cutoff_prob, cutoff_top_n) if pc > 0]
        cut = _F(NEG_INF)
        if lm is not None and min_cutoff and len(beam) == beam_size:
            blp = _F(blank_logp_per_frame[t]) if blank_logp_per_frame is not None else _F(math.log(float(probs[t, blank])))
            worst = logaddexp32(beam[-1][1], beam[-1][2])
            cut = _F(_F(worst + blp) - max(_F(0.0), beta))
        new_b: Dict[int, np.float32] = {}
        new_nb: Dict[int, np.float32] = {}
        order: List[int] = []

        def touch(node):
            if node not in new_b:
                new_b[node], new_nb[node] = _F(NEG_INF), _F(NEG_INF)
                order.append(node)

        for node, pb, pnb in beam:
            touch(node)
        for node, pb, pnb in beam:
            score = logaddexp32(pb, pnb)
            for c, lp in cands:
                if _F(lp + score) < cut:
                    continue
                if c == blank:
                    new_b[node] = logaddexp32(new_b[node], _F(score + lp))
                    continue
                if c == last[node]:
                    new_nb[node] = logaddexp32(new_nb[node], _F(pnb + lp))
                    add = _F(pb + lp) if pb != NEG_INF else _F(NEG_INF)
                else:
                    add = _F(score + lp)
                if add == NEG_INF:
                    continue
                if lm is not None:
                    add = _F(_F(add + _F(alpha * lnp_ext(node, c))) + beta)
                if H is not None:
                    add = _F(add + H.step(hs[node], c)[0])
                key = (node, c)
                ch = child.get(key)
                if ch is None:
                    ch = len(parent)
                    parent.append(node)
                    last.append(c)
                    toks_of.append(toks_of[node] + (c,))
                    hs.append(H.step(hs[node], c)[1] if H is not None else ())
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
    adj = []
    for rank, (node, pb, pnb) in enumerate(beam):
        s = logaddexp32(pb, pnb)
        if H is not None:
            s = _F(s + H.readout(hs[node]))
        adj.append((-float(s), rank, node, s))
    adj.sort(key=lambda e: (e[0], e[1]))
    out = []
    for _, _, node, s in adj[:nbest]:
        toks = list(toks_of[node])
        score = s if H is None else _F(s - H.credit(toks)[0])
        approx = score
        if lm is not None:
            S = lm.sentence_lnp([vocab[c] for c in toks])
            approx = _F(_F(score - _F(_F(len(toks)) * beta)) - _F(alpha * S))
        out.append((float(score), float(approx), toks))
    return out


class WordLmSearchHot(WordLmSearch):
    """``oracle.word_lm.WordLmSearch`` with hotword credit (``hotwords``: a HotwordMatcher or None)."""

    def __init__(self, wlm, alpha, beta, beam_size: int = 300, blank: int = 0, min_cutoff: bool = True,
                 hotwords: Optional[HotwordMatcher] = None):
        super().__init__(wlm, alpha, beta, beam_size, blank, min_cutoff)
        self.H = hotwords
        self.hs: List[tuple] = [()]

    def push(self, cands_per_frame, blank_logp_per_frame):
        w, lex, space, blank, H = self.w, self.w.lex, self.w.space, self.blank, self.H
        alpha, beta = self.alpha, self.beta
        for cands, blp in zip(cands_per_frame, blank_logp_per_frame):
            cands = [(int(c), _F(lp)) for c, lp in cands]
            beam = self.beam
            cut = _F(NEG_INF)
            if self.min_cutoff and len(beam) == self.beam_size:
                worst = logaddexp32(beam[-1][1], beam[-1][2])
                cut = _F(_F(worst + _F(blp)) - max(_F(0.0), beta))
            new_b: Dict[int, np.float32] = {}
            new_nb: Dict[int, np.float32] = {}
            order: List[int] = []

            def touch(node):
                if node not in new_b:
                    new_b[node], new_nb[node] = _F(NEG_INF), _F(NEG_INF)
                    order.append(node)

            for node, pb, pnb in beam:
                touch(node)
            for node, pb, pnb in beam:
                score = logaddexp32(pb, pnb)
                for c, lp in cands:
                    if _F(lp + score) < cut:
                        continue
                    if c == blank:
                        new_b[node] = logaddexp32(new_b[node], _F(score + lp))
                        continue
                    if c == self.last[node]:
                        new_nb[node] = logaddexp32(new_nb[node], _F(pnb + lp))
                        add = _F(pb + lp) if pb != NEG_INF else _F(NEG_INF)
                    else:
                        add = _F(score + lp)
                    key = (node, c)
                    ch = self.child.get(key)
                    st = self.lexs[node]
                    if ch is None:
                        if st == AFTER_SPACE:
                            self.lexs[node] = ROOT
                            self.attempts += 1
                            continue
                        if c == space:
                            if st == ROOT or lex.word[st] < 0:
                                continue
                            nst = AFTER_SPACE
                        else:
                            nst = lex.child[st].get(c)
                            if nst is None:
                                continue
                    if add == NEG_INF:
                        continue
                    if c == space:
                        word = lex.words[lex.word[st]]
                        lnp = w.lnp(w.window(self.words_of[node]), word)
                        add = _F(_F(add + _F(alpha * lnp)) + beta)
                    if H is not None:
                        add = _F(add + H.step(self.hs[node], c)[0])
                    if ch is None:
                        ch = len(self.parent)
                        self.parent.append(node)
                        self.last.append(c)
                        self.toks_of.append(self.toks_of[node] + (c,))
                        self.words_of.append(self.words_of[node] + ((lex.words[lex.word[st]],) if c == space else ()))
                        self.lexs.append(nst)
                        self.hs.append(H.step(self.hs[node], c)[1] if H is not None else ())
                        self.child[key] = ch
                    touch(ch)
                    new_nb[ch] = logaddexp32(new_nb[ch], add)
            scored = []
            for rank, node in enumerate(order):
                s = logaddexp32(new_b[node], new_nb[node])
                if s != NEG_INF:
                    scored.append((-float(s), rank, node))
            scored.sort()
            self.beam = [(node, new_b[node], new_nb[node]) for _, _, node in scored[:self.beam_size]]
        return self

    def result(self, nbest: int = 1):
        """-> [(score after the word read-out, without credit, approx, token ids)], best first by the selection score."""
        H = self.H
        adj = []
        for rank, (node, pb, pnb) in enumerate(self.beam):
            s = logaddexp32(pb, pnb)
            bonus = self.readout_bonus(node)
            if bonus is not None:
                s = _F(s + bonus)
            if H is not None:
                s = _F(s + H.readout(self.hs[node]))
            adj.append((-float(s), rank, node, s))
        adj.sort(key=lambda e: (e[0], e[1]))
        out = []
        for _, _, node, s in adj[:nbest]:
            toks = list(self.toks_of[node])
            if H is not None:
                s = _F(s - H.credit(toks)[0])
            S = self.w.sentence_lnp(self.w.split(toks))
            approx = _F(_F(s - _F(_F(len(toks)) * self.beta)) - _F(self.alpha * S))
            out.append((float(s), float(approx), toks))
        return out
