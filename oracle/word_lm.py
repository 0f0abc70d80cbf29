"""Oracle (test infrastructure): a WORD-based ARPA n-gram LM with the reference decoder's lexicon constraint, fused into
the CTC prefix beam search — PARITY UNPINNED.

English models (configs/english_example.yml: ``metrics_type: wer``, a ``<space>`` token) run ``ctc_beam_search`` with a
word KenLM through the external ``paddlespeech_ctcdecoders`` ``Scorer``, which then (a) scores the LM once per completed
word and (b) limits every hypothesis to words the LM knows through an OpenFST dictionary built from the LM's unigrams.
The library is absent, so this module restates those rules deterministically in float32 on top of oracle/lm.py (the ARPA
reader and the backoff rule; the character and no-LM searches are untouched) so that csrc/lm.cu and csrc/beam.cu can
equal it bit for bit.

Word mode: the ARPA file is not character-based (``ArpaLM.is_character_based``) and the model vocabulary has the token
``<space>`` (TextFeaturizer writes ' ' as ``<space>``).  Rejected with ArpaError (as by masr_word_lm_load_arpa): a
character-based file, a vocabulary without ``<space>``, an order above 5, or more than 2^24 - 1 declared unigrams (word ids
are 24 bits; 5 of them fill the 128-bit n-gram key) — plus every case ``read_arpa`` rejects.

Lexicon: every LM unigram except <s>, </s>, <unk> whose code points are each a model token (exact spelling, no case
folding); unspellable words are left out.  ``dict_size`` = the number of lexicon words (the library's get_dict_size()).
Word ids: lexicon words 0 .. dict_size-1 in unigram file order (first occurrence), <s> = dict_size, </s> = dict_size + 1.
The lexicon is a trie over token ids, nodes numbered in insertion order (words in id order, root = 0); with each word
followed by ``<space>`` it accepts the language of the library's determinised, minimised FST, state for state in
accept / reject and finality.  lnP(w | h) is oracle/lm.py's backoff rule where a word is in vocabulary iff it is a
lexicon word, <s> or </s> (else -1000).

Lexicon state of a prefix (kept with its trie node): a lexicon node (the letters since its last <space>), AFTER_SPACE
(final, no outgoing arcs), or ROOT (the lexicon root, after a reset).  The root prefix starts at ROOT.

Search, per frame, on top of ``oracle.lm.prefix_beam_search_lm`` (min_cutoff, stay transitions, ranking, pruning,
tie-breaks and node identity unchanged):
  attempt     every non-blank (prefix l, candidate c) pair that passes min_cutoff, repeats included even when p_b(l) = -inf
              (the library calls get_path_trie before it looks at log_prob_b_prev).
  acceptance  the child (l, c) exists -> accept.  Else from a lexicon node n: a letter c if n has that child; <space> if
              n is a word end and not the root.  From AFTER_SPACE: the FIRST attempt (in candidate order) is rejected and
              resets the prefix's state to ROOT, once and for the rest of the utterance (get_path_trie's
              ``is_final && reset`` branch).  A rejected extension contributes nothing.
  scoring     c == <space>: add = (base + alpha * lnP(w | h)) + beta, w = the word just completed, h = the N-1 words
              before it, <s>-padded.  Any other extension: add = base (no LM term and NO beta: beta sits inside the
              library's ``if (c == space_id || is_character_based)`` block).
  read-out    after the last frame (and at every streaming read-out, on the side: the carried state never sees it), every
              beam entry that is non-empty and does not end in <space> gets + (alpha * lnP(last word | h) + beta); a trailing
              partial word that is not a word end has lnP = -1000.  Best = max adjusted score, ties in beam rank order;
              approx = (score' - float32(len) * beta) - alpha * S, len = tokens including spaces, S = sentence_lnp over the
              words split on <space> (a trailing partial word counts as a word).
Known deviation, not emulated: the library deletes a childless pruned trie node and would apply a reset again to that
prefix if it were created anew later; here a node, and its reset, persist for the utterance.
Every + and * is one float32 rounding; alpha and beta are float32.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from oracle.beam import NEG_INF, logaddexp32
from oracle.lm import BOS, EOS, OOV_SCORE, UNK, ArpaError, ArpaLM, read_arpa

_F = np.float32
SPACE = "<space>"
MAX_WORD_ORDER = 5
WORD_ID_BITS = 24
MAX_WORD_IDS = (1 << WORD_ID_BITS) - 1          # ids 0 .. 2^24 - 2; 2^24 - 1 marks an out-of-vocabulary word
ROOT, AFTER_SPACE = 0, -1


def declared_counts(path: str) -> List[int]:
    """The n-gram counts of the \\data\\ section (for the width check, which comes before the n-gram sections are read)."""
    out: List[int] = []
    with open(path, encoding="utf-8", errors="replace") as f:
        for ln in f:
            s = ln.strip()
            if s == "\\data\\":
                out = []
                continue
            if s.startswith("ngram ") and "=" in s:
                try:
                    out.append(int(s[6:].split("=")[1]))
                except ValueError:
                    return out
            elif out and s:
                break
    return out


class Lexicon:
    """The trie of spellable LM words: ``child[n]`` token -> node, ``word[n]`` word id ending at n (or -1)."""

    def __init__(self, lm: ArpaLM, vocab: Sequence[str], unigram_order: Sequence[str]):
        tok = {}
        for i, t in enumerate(vocab):
            tok.setdefault(t, i)
        self.words: List[str] = []
        self.word_id: Dict[str, int] = {}
        self.child: List[Dict[int, int]] = [dict()]
        self.word: List[int] = [-1]
        for w in unigram_order:
            if w in (BOS, EOS, UNK) or w in self.word_id:
                continue
            ids = [tok.get(ch) for ch in w]
            if any(i is None for i in ids):
                continue                                     # unspellable: not in the lexicon
            wid = len(self.words)
            self.words.append(w)
            self.word_id[w] = wid
            n = ROOT
            for i in ids:
                nxt = self.child[n].get(i)
                if nxt is None:
                    nxt = len(self.child)
                    self.child[n][i] = nxt
                    self.child.append(dict())
                    self.word.append(-1)
                n = nxt
            self.word[n] = wid
        self.bos, self.eos = len(self.words), len(self.words) + 1

    @property
    def dict_size(self) -> int:
        return len(self.words)

    def csr(self):
        """(off [nodes+1], tok [arcs], nxt [arcs], word [nodes]): each node's arcs in ascending token order."""
        off, tok, nxt = [0], [], []
        for d in self.child:
            for t in sorted(d):
                tok.append(t)
                nxt.append(d[t])
            off.append(len(tok))
        return off, tok, nxt, list(self.word)


class WordLM:
    """A word ARPA LM against a model vocabulary: ``lm`` (oracle.lm.ArpaLM), ``lex`` (Lexicon), ``space`` (token id)."""

    def __init__(self, path: str, vocab: Sequence[str]):
        counts = declared_counts(path)
        if counts and counts[0] > MAX_WORD_IDS:
            raise ArpaError(f"{counts[0]} unigrams exceed the {WORD_ID_BITS}-bit word ids of the word LM tables")
        if len(counts) > MAX_WORD_ORDER:
            raise ArpaError(f"word LM order {len(counts)} > {MAX_WORD_ORDER} is not supported")
        self.lm = read_arpa(path)
        if self.lm.is_character_based:
            raise ArpaError(f"{path} is a character-based LM, not a word LM")
        if SPACE not in vocab:
            raise ArpaError(f"the vocabulary has no {SPACE} token: a word LM needs one")
        self.space = list(vocab).index(SPACE)
        self.vocab = list(vocab)
        with open(path, encoding="utf-8") as f:
            lines = [ln.strip() for ln in f]
        i = lines.index("\\1-grams:") + 1
        order: List[str] = []
        while i < len(lines) and lines[i] != "" and not lines[i].startswith("\\"):
            order.append(lines[i].split()[1])
            i += 1
        self.lex = Lexicon(self.lm, vocab, order)
        self.order = self.lm.order

    @property
    def dict_size(self) -> int:
        return self.lex.dict_size

    def in_vocab(self, w: str) -> bool:
        return w in self.lex.word_id or w in (BOS, EOS)

    def lnp(self, ctx: Sequence[str], w: str) -> np.float32:
        if not self.in_vocab(w) or not all(self.in_vocab(x) for x in ctx):
            return OOV_SCORE
        return self.lm.lnp(ctx, w)

    def window(self, words: Sequence[str]) -> List[str]:
        return self.lm.window(words)

    def sentence_lnp(self, words: Sequence[str]) -> np.float32:
        N = self.order
        sent = [BOS] * N if not words else [BOS] * (N - 1) + list(words)
        sent.append(EOS)
        s = _F(0.0)
        for i in range(len(sent) - N + 1):
            s = _F(s + self.lnp(sent[i:i + N - 1], sent[i + N - 1]))
        return s

    def split(self, toks: Sequence[int]) -> List[str]:
        """Token ids -> words split on <space> (a trailing partial word included, empty pieces dropped)."""
        words, cur = [], []
        for t in toks:
            if t == self.space:
                if cur:
                    words.append("".join(cur))
                cur = []
            else:
                cur.append(self.vocab[t])
        if cur:
            words.append("".join(cur))
        return words


class WordLmSearch:
    """The fused search as a stream: ``push`` frames (candidate lists and ln p_blank per frame), ``result`` reads out."""

    def __init__(self, wlm: WordLM, alpha: float, beta: float, beam_size: int = 300, blank: int = 0, min_cutoff: bool = True):
        self.w, self.alpha, self.beta = wlm, _F(alpha), _F(beta)
        self.beam_size, self.blank, self.min_cutoff = beam_size, blank, min_cutoff
        self.parent, self.last = [-1], [-1]
        self.child: Dict[Tuple[int, int], int] = {}
        self.toks_of: List[Tuple[int, ...]] = [()]
        self.words_of: List[Tuple[str, ...]] = [()]       # completed words of the prefix
        self.lexs: List[int] = [ROOT]                      # lexicon state, per trie node (a reset persists with the node)
        self.beam = [(0, _F(0.0), _F(NEG_INF))]
        self.attempts = 0                                  # (for tests) attempts that reset a prefix

    def push(self, cands_per_frame, blank_logp_per_frame):
        w, lex, space, blank = self.w, self.w.lex, self.w.space, self.blank
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
                    # the attempt (get_path_trie)
                    key = (node, c)
                    ch = self.child.get(key)
                    st = self.lexs[node]
                    if ch is None:
                        if st == AFTER_SPACE:
                            self.lexs[node] = ROOT                 # first attempt after <space>: rejected, resets once
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
                    if ch is None:
                        ch = len(self.parent)
                        self.parent.append(node)
                        self.last.append(c)
                        self.toks_of.append(self.toks_of[node] + (c,))
                        self.words_of.append(self.words_of[node] + ((lex.words[lex.word[st]],) if c == space else ()))
                        self.lexs.append(nst)
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

    def readout_bonus(self, node) -> Optional[np.float32]:
        """alpha * lnP(last word | h) + beta for a non-empty prefix not ending in <space>, else None."""
        if node == 0 or self.last[node] == self.w.space:
            return None
        st = self.lexs[node]
        lex = self.w.lex
        word = lex.words[lex.word[st]] if st >= 0 and lex.word[st] >= 0 else None
        lnp = self.w.lnp(self.w.window(self.words_of[node]), word) if word is not None else OOV_SCORE
        return _F(_F(self.alpha * lnp) + self.beta)

    def result(self, nbest: int = 1):
        """-> [(score after the read-out term, approx, token ids)], best first (ties in beam rank order)."""
        adj = []
        for rank, (node, pb, pnb) in enumerate(self.beam):
            s = logaddexp32(pb, pnb)
            bonus = self.readout_bonus(node)
            if bonus is not None:
                s = _F(s + bonus)
            adj.append((-float(s), rank, node, s))
        adj.sort(key=lambda e: (e[0], e[1]))
        out = []
        for _, _, node, s in adj[:nbest]:
            toks = list(self.toks_of[node])
            S = self.w.sentence_lnp(self.w.split(toks))
            approx = _F(_F(s - _F(_F(len(toks)) * self.beta)) - _F(self.alpha * S))
            out.append((float(s), float(approx), toks))
        return out


def prefix_beam_search_wordlm(wlm: WordLM, cands_per_frame, blank_logp_per_frame, alpha: float = 0.0, beta: float = 0.0,
                              beam_size: int = 300, blank: int = 0, nbest: int = 1, min_cutoff: bool = True):
    """The whole-utterance search on given per-frame candidates [(token id, float32 ln p)] and ln p_blank per frame ->
    list of (score after the read-out term, approx, token ids), best first."""
    s = WordLmSearch(wlm, alpha, beta, beam_size, blank, min_cutoff)
    return s.push(cands_per_frame, blank_logp_per_frame).result(nbest)


def prune_candidates(probs: np.ndarray, cutoff_prob: float = 0.99, cutoff_top_n: int = 40):
    """Per-frame candidate lists and ln p_blank from posteriors, as ``prefix_beam_search_lm`` derives them."""
    from oracle.beam import prune_frame
    cands = [[(c, _F(math.log(float(pc)))) for c, pc in prune_frame(p, cutoff_prob, cutoff_top_n) if pc > 0] for p in probs]
    blp = [_F(math.log(float(p[0]))) if p[0] > 0 else _F(NEG_INF) for p in probs]
    return cands, blp
