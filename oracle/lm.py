"""Oracle (test infrastructure): a character-based ARPA n-gram LM and its shallow fusion into the CTC prefix beam search —
PARITY UNPINNED.

The reference scores beam extensions with the external ``paddlespeech_ctcdecoders`` ``Scorer`` over a KenLM file
(masr/decoders/swig_wrapper.py:4-18, beam_search_decoder.py:28-32,47).  Neither the library nor KenLM exist here, so this
module restates that library's public algorithm for a CHARACTER-based scorer, made deterministic in float32 exactly like
``oracle.beam.prefix_beam_search`` (which it extends; with no LM that function is the search, unchanged) so that the CUDA
kernels (csrc/lm.cu, csrc/beam.cu) can equal it bit for bit.

Tables: every ARPA log10 value v (probabilities and backoffs) is kept as float32(double(v) * ln 10).

lnP(c | h) — standard backoff, in this float32 order.  The window h is the last N-1 tokens of the prefix, left-padded with
``<s>`` (``make_ngram``); N is the ARPA's max order.  If any word of the window or the predicted word is not an LM unigram,
or is ``<unk>``, lnP = -1000 (the reference's OOV_SCORE — a previously emitted OOV character poisons the next N-1
extensions).  Otherwise acc = 0; for L = N-1 .. 0: if (h[-L:], c) is an n-gram return acc + p (one rounding); else if
L >= 1 and h[-L:] is an n-gram, acc += bo(h[-L:]).  This equals KenLM's state-based scoring for ARPA files in which only
n-grams that prefix a longer n-gram carry a backoff (what lmplz writes, and what masr_b200.synth writes).

Fused search (``prefix_beam_search_lm``), on top of the no-LM definition of oracle/beam.py:
  extension ℓ -> ℓ+c (c non-blank; the character-based scorer fires on every extension):
      base = score(ℓ) + lp_c, or p_b(ℓ) + lp_c when c == last(ℓ);  add = (base + alpha * lnP(c | ℓ)) + beta
  stay transitions (blank, repeat) get no LM term.
  min_cutoff: when the beam is full (nbeam == beam_size), min_cutoff = (score(worst) + ln p_blank(t)) - max(0, beta), where
      p_blank(t) is the frame's full softmax probability of blank; a (prefix, candidate) pair with lp_c + score(ℓ) <
      min_cutoff contributes nothing (no blank, repeat or extension transition) — the reference's `break` over its
      score-sorted prefixes, stated per pair.  So alpha = beta = 0 still differs from the no-LM search unless the cut is off.
  ranking, pruning, tie-breaks, node identity: exactly as oracle/beam.py, on the fused score.
  reported: approx = (score - float32(len) * beta) - alpha * S, S = the float32 in-order sum of lnP over the sentence
      <s>^(N-1) + tokens + </s>, or <s>^N + </s> for an empty prefix (``get_sent_log_prob``).  Without an LM approx == score.
Every + and * above is one float32 rounding; alpha and beta are float32.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from oracle.beam import NEG_INF, logaddexp32, prune_frame

_F = np.float32
LN10 = math.log(10.0)
OOV_SCORE = _F(-1000.0)
MAX_ORDER = 6
BOS, EOS, UNK = "<s>", "</s>", "<unk>"


class ArpaError(ValueError):
    pass


def to_ln(v: float) -> np.float32:
    return _F(float(v) * LN10)


class ArpaLM:
    """A parsed ARPA file: ``ngrams[n]`` maps a tuple of n words to (ln p, ln backoff) as float32."""

    def __init__(self, order: int, counts: List[int], ngrams: Dict[int, Dict[Tuple[str, ...], Tuple[np.float32, np.float32]]]):
        self.order, self.counts, self.ngrams = order, counts, ngrams
        self.unigrams = {w[0] for w in ngrams[1]}

    @property
    def is_character_based(self) -> bool:
        """Every unigram except <s>, </s>, <unk> is one code point (the reference Scorer's test)."""
        return all(len(w) == 1 for w in self.unigrams if w not in (BOS, EOS, UNK))

    @property
    def dict_size(self) -> int:
        return len(self.unigrams)

    def in_vocab(self, w: str) -> bool:
        return w in self.unigrams and w != UNK

    def lnp(self, ctx: Sequence[str], w: str) -> np.float32:
        """lnP(w | ctx); ctx = exactly N-1 words (already padded with <s>)."""
        assert len(ctx) == self.order - 1
        if not self.in_vocab(w) or not all(self.in_vocab(x) for x in ctx):
            return OOV_SCORE
        acc = _F(0.0)
        for L in range(self.order - 1, -1, -1):
            h = tuple(ctx[len(ctx) - L:]) if L else ()
            e = self.ngrams[L + 1].get(h + (w,))
            if e is not None:
                return _F(acc + e[0])
            if L >= 1:
                b = self.ngrams[L].get(h)
                if b is not None:
                    acc = _F(acc + b[1])
        return OOV_SCORE

    def window(self, words: Sequence[str]) -> List[str]:
        """The last N-1 words of ``words``, left-padded with <s> (``make_ngram``)."""
        n1 = self.order - 1
        w = list(words[max(0, len(words) - n1):]) if n1 else []
        return [BOS] * (n1 - len(w)) + w

    def sentence_lnp(self, words: Sequence[str]) -> np.float32:
        """``get_sent_log_prob``: float32 in-order sum of lnP over <s>^(N-1) + words + </s> (<s>^N + </s> when empty)."""
        N = self.order
        sent = [BOS] * N if not words else [BOS] * (N - 1) + list(words)
        sent.append(EOS)
        s = _F(0.0)
        for i in range(len(sent) - N + 1):
            s = _F(s + self.lnp(sent[i:i + N - 1], sent[i + N - 1]))
        return s


def read_arpa(path: str) -> ArpaLM:
    """Plain-text ARPA -> ArpaLM.  Raises ArpaError on a missing \\data\\ section, count or section mismatches, a missing
    <s> or </s>, an order above 6, or a malformed line — the same cases csrc/lm.cu rejects."""
    with open(path, "rb") as f:
        head = f.read(8)
    if head.startswith(b"mmap lm"):
        raise ArpaError(f"{path}: a KenLM binary, not an ARPA file")
    with open(path, encoding="utf-8") as f:
        lines = [ln.strip() for ln in f]
    i = 0
    while i < len(lines) and lines[i] != "\\data\\":
        i += 1
    if i == len(lines):
        raise ArpaError("missing \\data\\ section")
    i += 1
    counts: List[int] = []
    while i < len(lines) and lines[i].startswith("ngram "):
        try:
            k, c = lines[i][6:].split("=")
            k, c = int(k), int(c)
        except ValueError:
            raise ArpaError(f"malformed line {i + 1}: {lines[i]!r}")
        if k != len(counts) + 1 or c < 0:
            raise ArpaError(f"count mismatch: line {i + 1}: {lines[i]!r}")
        counts.append(c)
        i += 1
    if not counts:
        raise ArpaError("\\data\\ section declares no n-gram counts")
    order = len(counts)
    if order > MAX_ORDER:
        raise ArpaError(f"order {order} > {MAX_ORDER} is not supported")
    ngrams: Dict[int, Dict[Tuple[str, ...], Tuple[np.float32, np.float32]]] = {}
    for n in range(1, order + 1):
        while i < len(lines) and lines[i] == "":
            i += 1
        if i == len(lines) or lines[i] != f"\\{n}-grams:":
            raise ArpaError(f"section mismatch: expected \\{n}-grams:")
        i += 1
        table, nread = {}, 0
        while i < len(lines) and lines[i] != "" and not lines[i].startswith("\\"):
            f = lines[i].split()
            if len(f) not in (n + 1, n + 2):
                raise ArpaError(f"malformed line {i + 1}: {lines[i]!r}")
            try:
                p = to_ln(float(f[0]))
                bo = to_ln(float(f[n + 1])) if len(f) == n + 2 else _F(0.0)
            except ValueError:
                raise ArpaError(f"malformed line {i + 1}: {lines[i]!r}")
            table[tuple(f[1:n + 1])] = (p, bo)           # (a repeated n-gram: the last wins)
            nread += 1
            i += 1
        if nread != counts[n - 1]:
            raise ArpaError(f"count mismatch: \\{n}-grams: has {nread} entries, \\data\\ says {counts[n - 1]}")
        ngrams[n] = table
    while i < len(lines) and lines[i] == "":
        i += 1
    if i == len(lines) or lines[i] != "\\end\\":
        raise ArpaError("section mismatch: expected \\end\\")
    lm = ArpaLM(order, counts, ngrams)
    for w in (BOS, EOS):
        if w not in lm.unigrams:
            raise ArpaError(f"{w} is not a unigram")
    return lm


def prefix_beam_search_lm(probs: np.ndarray, lm: Optional[ArpaLM], vocab: Sequence[str], alpha: float = 0.0, beta: float = 0.0,
                          beam_size: int = 300, cutoff_prob: float = 0.99, cutoff_top_n: int = 40, blank: int = 0,
                          nbest: int = 1, cands_per_frame=None, blank_logp_per_frame=None, min_cutoff: bool = True):
    """``oracle.beam.prefix_beam_search`` with shallow fusion of ``lm`` (see the module docstring) ->
    list of (fused score, approx, token ids), best first.  ``lm=None`` is the no-LM search (approx == score).
    ``blank_logp_per_frame`` (optional): ln p_blank per frame, e.g. from the CUDA top-k kernel; else log(probs[t, blank]).
    ``min_cutoff=False`` switches the early cut off (to compare with the no-LM search at alpha = beta = 0)."""
    alpha, beta = _F(alpha), _F(beta)
    parent, last = [-1], [-1]
    child: Dict[Tuple[int, int], int] = {}
    toks_of: List[Tuple[int, ...]] = [()]
    lnp_memo: Dict[Tuple[int, int], np.float32] = {}

    def lnp_ext(node, c):
        key = (node, c)
        if key not in lnp_memo:
            lnp_memo[key] = lm.lnp(lm.window([vocab[t] for t in toks_of[node]]), vocab[c])
        return lnp_memo[key]

    beam = [(0, _F(0.0), _F(NEG_INF))]
    for t in range(probs.shape[0]):
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
                key = (node, c)
                ch = child.get(key)
                if ch is None:
                    ch = len(parent)
                    parent.append(node)
                    last.append(c)
                    toks_of.append(toks_of[node] + (c,))
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
        score = logaddexp32(pb, pnb)
        toks = list(toks_of[node])
        approx = score
        if lm is not None:
            S = lm.sentence_lnp([vocab[c] for c in toks])
            approx = _F(_F(score - _F(_F(len(toks)) * beta)) - _F(alpha * S))
        out.append((float(score), float(approx), toks))
    return out
