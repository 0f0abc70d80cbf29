"""Hotword (contextual) biasing for the GPU CTC prefix beam search: the user's hotwords as an Aho-Corasick automaton over
model tokens, built here with numpy and searched by csrc/beam.cu (the ``*_hot`` entry points).  Semantics:
oracle/hotwords.py, which restates the same rule over strings.

Each hotword is one token per character (``' '`` is ``<space>`` when the vocabulary has it).  A prefix earns ``score``
per token of every whole hotword it contains, by a longest-match rule: nested hotwords ("北京" and "北京大学") both work,
a match abandoned part-way keeps the credit of any whole hotword inside it, and a match left unfinished at the end of
the search earns nothing.  The search ranks and selects with the credit; the score it reports excludes it.

``HotwordGraph`` is one list of hotwords; ``HotwordBuffer`` is one device buffer with a fixed number of fixed-size
regions, each holding one graph (a stream pool: one region per slot plus one for the pool default), so that a slot's
graph can be replaced without moving any other slot's nodes."""
from __future__ import annotations

import math
from collections import deque
from typing import Dict, Iterable, List, Optional, Sequence, Tuple

import numpy as np

from . import _lib

MAX_TOKENS = 32                          # tokens per hotword: the kernel's automaton walk is bounded by it
SPACE = "<space>"
_F = np.float32
_FIELDS = ("arc_off", "arc_tok", "arc_next", "fail", "tail", "leaf", "acc", "ta_acc", "fin")


def tokenize(hotwords: Iterable[str], vocab: Sequence[str], blank: int = 0) -> List[Tuple[int, ...]]:
    """Hotwords -> their token sequences, duplicates merged (first occurrence order).  Raises ValueError naming the
    hotword (and the character) for an empty hotword, a character outside the vocabulary or mapping to the blank, and a
    hotword longer than MAX_TOKENS tokens."""
    index: Dict[str, int] = {}
    for i, v in enumerate(vocab):
        index.setdefault(v, i)
    space = index.get(SPACE)
    out, seen = [], set()
    for hw in hotwords:
        if not isinstance(hw, str):
            raise ValueError(f"hotword {hw!r} is not a string")
        if hw == "":
            raise ValueError("hotword '' is empty")
        toks = []
        for ch in hw:
            t = space if ch == " " and space is not None else index.get(ch)
            if t is None:
                raise ValueError(f"hotword {hw!r}: character {ch!r} is not in the vocabulary")
            if t == blank:
                raise ValueError(f"hotword {hw!r}: character {ch!r} is the blank token")
            toks.append(t)
        if len(toks) > MAX_TOKENS:
            raise ValueError(f"hotword {hw!r} has {len(toks)} tokens, more than {MAX_TOKENS}")
        key = tuple(toks)
        if key not in seen:
            seen.add(key)
            out.append(key)
    return out


def check_score(score) -> np.float32:
    """The credit per token, float32: finite and >= 0, else ValueError."""
    w = _F(score)
    if not math.isfinite(float(w)) or w < 0:
        raise ValueError(f"hotword_score {score!r} must be finite and >= 0")
    return w


class HotwordGraph:
    """``hotwords`` (strings) against ``vocab`` with ``score`` per token.  Attributes: ``hotwords`` (merged, in order),
    ``tokens`` (their token sequences), ``score`` (float32), ``nodes``, and the automaton as numpy arrays over local node
    ids (root 0, breadth-first, children by ascending token): ``arc_off`` [nodes + 1], ``arc_tok`` / ``arc_next`` [arcs],
    ``fail``, ``tail`` (-1: no whole hotword in the match), ``leaf``, ``acc``, ``ta_acc``, ``fin`` [nodes] — the fields
    of ``masr_hotword_graph`` (include/masr_b200.h).  ``tables(device)`` uploads it once per device."""

    def __init__(self, hotwords: Iterable[str], vocab: Sequence[str], score: float = 1.5, blank: int = 0):
        hotwords = list(hotwords)
        self.tokens = tokenize(hotwords, vocab, blank)
        self.score = check_score(score)
        merged, seen = [], set()
        for hw in hotwords:
            key = tokenize([hw], vocab, blank)[0]
            if key not in seen:
                seen.add(key)
                merged.append(hw)
        self.hotwords = merged
        self._build()
        self._dev: Dict[str, "HotwordBuffer"] = {}

    def _build(self):
        children: List[Dict[int, int]] = [{}]
        depth, parent_tok = [0], [-1]
        for key in self.tokens:                                   # the trie (insertion ids, renumbered below)
            n = 0
            for t in key:
                if t not in children[n]:
                    children[n][t] = len(children)
                    children.append({})
                    depth.append(depth[n] + 1)
                    parent_tok.append(t)
                n = children[n][t]
        order, q = [], deque([0])                                 # breadth-first, children by ascending token
        while q:
            n = q.popleft()
            order.append(n)
            q.extend(children[n][t] for t in sorted(children[n]))
        new = {old: i for i, old in enumerate(order)}
        N = len(order)
        kids = [{t: new[c] for t, c in sorted(children[old].items())} for old in order]
        dep = np.array([depth[old] for old in order], np.int64)
        terminal = np.zeros(N, bool)
        par = np.full(N, -1, np.int64)
        for i in range(N):
            for c in kids[i].values():
                par[c] = i
        for key in self.tokens:
            n = 0
            for t in key:
                n = kids[n][t]
            terminal[n] = True

        def goto(state, t):                                       # the Aho-Corasick transition (fail is set for shallower)
            while state != 0 and t not in kids[state]:
                state = fail[state]
            return kids[state].get(t, 0)

        fail = np.zeros(N, np.int64)
        toks_of: List[Tuple[int, ...]] = [()] * N
        for i in range(1, N):                                     # breadth-first: parents before children
            p = int(par[i])
            t = next(tt for tt, c in kids[p].items() if c == i)
            toks_of[i] = toks_of[p] + (t,)
            fail[i] = 0 if p == 0 else goto(int(fail[p]), t)
        w = self.score
        acc = (w * dep.astype(np.float32)).astype(np.float32)      # float32(w) * depth, one rounding
        ta = np.full(N, -1, np.int64)
        for i in range(1, N):
            ta[i] = i if terminal[i] else ta[par[i]]
        tail = np.full(N, -1, np.int64)
        for i in range(1, N):
            if ta[i] >= 0:
                s = 0
                for t in toks_of[i][int(dep[ta[i]]):]:
                    s = goto(s, t)
                tail[i] = s
        ta_acc = np.where(ta >= 0, acc[np.maximum(ta, 0)], _F(0)).astype(np.float32)
        fin = np.zeros(N, np.float32)
        for i in range(1, N):                                     # the loop of a token that extends nothing
            bank, cur = _F(0), i
            while cur != 0:
                if tail[cur] >= 0:
                    bank = _F(bank + ta_acc[cur])
                    cur = int(tail[cur])
                else:
                    cur = int(fail[cur])
            fin[i] = bank
        arc_off = np.zeros(N + 1, np.int32)
        arc_tok, arc_next = [], []
        for i in range(N):
            arc_off[i] = len(arc_tok)
            for t, c in kids[i].items():
                arc_tok.append(t)
                arc_next.append(c)
        arc_off[N] = len(arc_tok)
        self.nodes = N
        self.arc_off, self.arc_tok, self.arc_next = arc_off, np.array(arc_tok, np.int32), np.array(arc_next, np.int32)
        self.fail, self.tail = fail.astype(np.int32), tail.astype(np.int32)
        self.leaf = np.array([0 if kids[i] else 1 for i in range(N)], np.int32)
        self.leaf[0] = 0
        self.acc, self.ta_acc, self.fin = acc, ta_acc, fin

    def tables(self, device) -> _lib.HotwordGraph:
        """The ``masr_hotword_graph`` of this graph's copy on ``device`` (uploaded on first use, then reused; root 0)."""
        import torch
        key = str(torch.device(device))
        if key not in self._dev:
            buf = HotwordBuffer(device, 1, self.nodes)
            buf.put(0, self)
            self._dev[key] = buf
        return self._dev[key].tables(device)


class HotwordBuffer:
    """One device buffer of ``regions`` regions of up to ``max_nodes`` nodes each (stride ``max_nodes + 1``, so each
    region ends in an unused node that closes its last node's arc range).  ``put(r, graph)`` copies a graph into region r
    (its node ids shifted to the region's), ``root(r)`` is that graph's root node.  ``bytes_per_node``: the device memory
    one node of capacity takes."""

    bytes_per_node = 4 * (len(_FIELDS) + 1)      # nine int/float fields, the arc arrays sized like the nodes

    def __init__(self, device, regions: int, max_nodes: int):
        import torch
        if max_nodes < 1:
            raise ValueError(f"max_nodes {max_nodes} must be >= 1")
        self.device, self.regions, self.max_nodes = torch.device(device), int(regions), int(max_nodes)
        self.stride = self.max_nodes + 1
        n = self.regions * self.stride
        i32, f32 = torch.int32, torch.float32
        self.arr = {f: torch.zeros(n + (1 if f == "arc_off" else 0), device=self.device,
                                   dtype=f32 if f in ("acc", "ta_acc", "fin") else i32) for f in _FIELDS}
        self.arr["arc_off"].copy_(torch.arange(n + 1, dtype=i32).div(self.stride, rounding_mode="floor") * self.stride)
        self._t = _lib.HotwordGraph(*(self.arr[f].data_ptr() for f in _FIELDS), n)

    def root(self, region: int) -> int:
        return int(region) * self.stride

    def put(self, region: int, g: HotwordGraph):
        """Copy ``g`` into ``region`` (host to device, on the current stream; never during a graph capture)."""
        import torch
        if g.nodes > self.max_nodes:
            raise ValueError(f"the hotword graph has {g.nodes} nodes, more than the {self.max_nodes} per slot this pool "
                             f"was built with (max_hotword_nodes)")
        base, S = self.root(region), self.stride
        loc_end = int(g.arc_off[g.nodes])
        arc_off = np.full(S, base + loc_end, np.int32)
        arc_off[:g.nodes] = base + g.arc_off[:g.nodes]
        pad_i = lambda a, fill=0: np.r_[a, np.full(S - len(a), fill, a.dtype)]
        shift = lambda a: np.where(a >= 0, a + base, -1).astype(np.int32)
        host = {"arc_off": arc_off, "arc_tok": pad_i(g.arc_tok), "arc_next": pad_i((g.arc_next + base).astype(np.int32)),
                "fail": pad_i((g.fail + base).astype(np.int32)), "tail": pad_i(shift(g.tail), -1), "leaf": pad_i(g.leaf),
                "acc": pad_i(g.acc), "ta_acc": pad_i(g.ta_acc), "fin": pad_i(g.fin)}
        for f in _FIELDS:
            self.arr[f][base:base + S].copy_(torch.from_numpy(np.ascontiguousarray(host[f])))

    def tables(self, device=None) -> _lib.HotwordGraph:
        return self._t


def outside_lexicon(g: HotwordGraph, vocab: Sequence[str], wlm) -> List[str]:
    """The words of ``g``'s hotwords (split on ``<space>``) that a word LM's lexicon (``lm.WordLM``) does not hold: the
    search can never produce a hotword that uses one of them."""
    space = wlm.space
    out = []
    for toks in g.tokens:
        words, cur = [], []
        for t in toks + (space,):
            if t != space:
                cur.append(t)
            elif cur:
                words.append(cur)
                cur = []
        for w in words:
            n = 0
            for t in w:
                lo, hi = int(wlm.lex_off[n]), int(wlm.lex_off[n + 1])
                i = lo + int(np.searchsorted(wlm.lex_tok[lo:hi], t))
                n = int(wlm.lex_next[i]) if i < hi and wlm.lex_tok[i] == t else -1
                if n < 0:
                    break
            if n < 0 or wlm.lex_word[n] < 0:
                s = "".join(vocab[t] for t in w)
                if s not in out:
                    out.append(s)
    return out


def graph_or_none(hotwords, vocab: Sequence[str], score: float = 1.5, blank: int = 0) -> Optional[HotwordGraph]:
    """None for no hotwords (None or an empty list), a HotwordGraph for a list of strings, the graph itself for one."""
    if hotwords is None or isinstance(hotwords, HotwordGraph):
        return hotwords
    hotwords = list(hotwords)
    return HotwordGraph(hotwords, vocab, score, blank) if hotwords else None
