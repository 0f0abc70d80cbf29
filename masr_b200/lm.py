"""Character and word n-gram language models (plain-text ARPA) for the GPU prefix beam search — the reference's
``Scorer(alpha, beta, language_model_path, vocab_list)`` (masr/decoders/swig_wrapper.py:4-18, beam_search_decoder.py:28-37)
for a character-based LM (``CharLM``) and for a word-based LM with its lexicon constraint (``WordLM``).  The file is parsed
by the library's C++ loader (csrc/lm.cu); the packed tables are uploaded once per device into torch-allocated buffers and
shared read-only by every search.  Semantics: oracle/lm.py, oracle/word_lm.py."""
from __future__ import annotations

import ctypes as C
import os
import time
from typing import Dict, List, Sequence

import numpy as np

from . import _lib

KENLM_MAGIC = b"mmap lm"


def sniff(path: str) -> str:
    """What ``path`` holds, judged by content: 'missing', 'kenlm_binary' (starts with ``mmap lm``), 'arpa' (a ``\\data\\``
    line before the first n-gram section) or 'unknown'."""
    if not path or not os.path.isfile(path):
        return "missing"
    with open(path, "rb") as f:
        head = f.read(1 << 16)
    if head.startswith(KENLM_MAGIC):
        return "kenlm_binary"
    for line in head.split(b"\n"):
        s = line.strip()
        if s == b"\\data\\":
            return "arpa"
        if s.startswith(b"\\"):
            break
    return "unknown"


class CharLM:
    """An ARPA LM against a model vocabulary.  ``order``, ``is_character_based``, ``dict_size`` are the reference
    Scorer's ``get_max_order()``, ``is_character_based()``, ``get_dict_size()`` (dict_size = the ARPA's unigram count);
    ``read_counts`` / ``kept_counts`` per order (n-grams containing a word outside the model vocabulary are dropped: no
    query reaches them); ``table_bytes``; ``load_seconds`` (host CPU time of the parse + table build)."""

    def __init__(self, path: str, vocab_list: Sequence[str]):
        lib = _lib.load()
        self.path, self.vocab_size = path, len(vocab_list)
        vocab = "\n".join(vocab_list).encode("utf-8")
        h = C.c_void_p()
        t0 = time.process_time()
        _lib.check(lib.masr_lm_load_arpa(C.c_char_p(os.fsencode(path)), C.c_char_p(vocab), len(vocab_list), C.byref(h)),
                   "masr_lm_load_arpa")
        try:
            info = (C.c_int64 * 32)()
            _lib.call("masr_lm_info", h, info)
            self.order = int(info[_lib.LM_INFO_ORDER])
            self.is_character_based = bool(info[_lib.LM_INFO_CHAR_BASED])
            self.dict_size = int(info[_lib.LM_INFO_DICT_SIZE])
            self.read_counts = [int(info[_lib.LM_INFO_READ + n]) for n in range(self.order)]
            self.kept_counts = [int(info[_lib.LM_INFO_KEPT + n]) for n in range(self.order)]
            self.slots = [int(info[_lib.LM_INFO_SLOTS + n]) for n in range(self.order)]
            self.table_bytes = int(info[_lib.LM_INFO_TABLE_BYTES])
            self.keys = np.empty(int(info[_lib.LM_INFO_KEY_WORDS]), np.uint32)
            self.vals = np.empty(int(info[_lib.LM_INFO_VAL_FLOATS]), np.float32)
            self.tok2lm = np.empty(self.vocab_size, np.int32)
            self._layout = _lib.LmTables()
            _lib.call("masr_lm_export", h, self.keys.ctypes.data, self.vals.ctypes.data, self.tok2lm.ctypes.data,
                      C.byref(self._layout))
        finally:
            lib.masr_lm_free(h)
        self.load_seconds = time.process_time() - t0
        self._dev: Dict[str, tuple] = {}

    BEAM = "masr_ctc_prefix_beam_lm"        # the fused search's entry points: BEAM, BEAM + "_stream" / "_pool" / "_state_size"

    def describe(self) -> str:
        return f"is_character_based = {self.is_character_based}, max_order = {self.order}, dict_size = {self.dict_size}"

    def tables(self, device) -> _lib.LmTables:
        """The ``masr_lm_tables`` of this LM's copy on ``device`` (uploaded on first use, then reused read-only)."""
        import torch
        dev = torch.device(device)
        key = str(dev)
        if key not in self._dev:
            keys = torch.from_numpy(self.keys.view(np.int32)).to(dev)
            vals = torch.from_numpy(self.vals).to(dev)
            tok = torch.from_numpy(self.tok2lm).to(dev)
            t = _lib.LmTables.from_buffer_copy(self._layout)
            t.keys, t.vals, t.tok2lm = keys.data_ptr(), vals.data_ptr(), tok.data_ptr()
            self._dev[key] = (t, keys, vals, tok)
        return self._dev[key][0]

    def score(self, ctx, word, device="cuda"):
        """lnP(word | ctx) for a batch of queries on the GPU (``masr_lm_score_f32``): ctx [Q, order-1] and word [Q] are
        model token ids, -1 = <s>, -2 = </s>.  -> float32 numpy [Q]."""
        import torch
        dev = torch.device(device)
        t = self.tables(dev)
        w = torch.as_tensor(np.asarray(word, np.int32)).to(dev)
        c = torch.as_tensor(np.asarray(ctx, np.int32).reshape(len(w), max(0, self.order - 1))).to(dev).contiguous()
        out = torch.empty(len(w), device=dev, dtype=torch.float32)
        _lib.call("masr_lm_score_f32", C.byref(t), c.data_ptr() if c.numel() else None, w.data_ptr(), len(w), out.data_ptr(),
                  torch.cuda.current_stream(dev).cuda_stream)
        return out.cpu().numpy()


class WordLM:
    """A word-based ARPA LM against a model vocabulary that has ``<space>``: the reference Scorer for a word LM, which
    scores a word once, when the ``<space>`` after it is emitted, and limits every hypothesis to the words of a lexicon
    built from the LM's unigrams (the library's OpenFST dictionary).  The same surface as ``CharLM`` (``order``,
    ``is_character_based`` (False), ``dict_size`` (lexicon words, the library's get_dict_size()), ``describe()``,
    ``tables(device)``, ``score()``) plus the lexicon: ``lex_off`` / ``lex_tok`` / ``lex_next`` (each node's arcs,
    ascending by token), ``lex_word`` (word id ending at a node or -1), ``space`` (the <space> token id).  Word ids:
    lexicon words 0 .. dict_size-1 in unigram file order, <s> = dict_size, </s> = dict_size + 1.  Semantics:
    oracle/word_lm.py.  Raises ``MasrB200Error`` for what ``masr_word_lm_load_arpa`` rejects (a character-based file, a
    vocabulary without ``<space>``, an order above 5, more than 2^24 - 1 unigrams, ...)."""

    BEAM = "masr_ctc_prefix_beam_wordlm"

    def __init__(self, path: str, vocab_list: Sequence[str]):
        lib = _lib.load()
        self.path, self.vocab_size = path, len(vocab_list)
        vocab = "\n".join(vocab_list).encode("utf-8")
        h = C.c_void_p()
        t0 = time.process_time()
        _lib.check(lib.masr_word_lm_load_arpa(C.c_char_p(os.fsencode(path)), C.c_char_p(vocab), len(vocab_list), C.byref(h)),
                   "masr_word_lm_load_arpa")
        try:
            info = (C.c_int64 * 32)()
            _lib.call("masr_word_lm_info", h, info)
            self.order = int(info[_lib.LM_INFO_ORDER])
            self.is_character_based = False
            self.dict_size = int(info[_lib.LM_INFO_DICT_SIZE])
            self.read_counts = [int(info[_lib.LM_INFO_READ + n]) for n in range(self.order)]
            self.kept_counts = [int(info[_lib.LM_INFO_KEPT + n]) for n in range(self.order)]
            self.slots = [int(info[_lib.LM_INFO_SLOTS + n]) for n in range(self.order)]
            self.table_bytes = int(info[_lib.LM_INFO_TABLE_BYTES])
            self.space = int(info[_lib.WORD_LM_INFO_SPACE])
            nodes, arcs = int(info[_lib.WORD_LM_INFO_NODES]), int(info[_lib.WORD_LM_INFO_ARCS])
            self.keys = np.empty(int(info[_lib.LM_INFO_KEY_WORDS]), np.uint32)
            self.vals = np.empty(int(info[_lib.LM_INFO_VAL_FLOATS]), np.float32)
            self.lex_off = np.empty(nodes + 1, np.int32)
            self.lex_tok = np.empty(max(1, arcs), np.int32)
            self.lex_next = np.empty(max(1, arcs), np.int32)
            self.lex_word = np.empty(nodes, np.int32)
            self._layout = _lib.WordLmTables()
            _lib.call("masr_word_lm_export", h, self.keys.ctypes.data, self.vals.ctypes.data, self.lex_off.ctypes.data,
                      self.lex_tok.ctypes.data, self.lex_next.ctypes.data, self.lex_word.ctypes.data, C.byref(self._layout))
            self.lex_tok, self.lex_next = self.lex_tok[:arcs], self.lex_next[:arcs]
        finally:
            lib.masr_lm_free(h)
        self.load_seconds = time.process_time() - t0
        self._dev: Dict[str, tuple] = {}

    def describe(self) -> str:
        return f"is_character_based = {self.is_character_based}, max_order = {self.order}, dict_size = {self.dict_size}"

    def tables(self, device) -> _lib.WordLmTables:
        """The ``masr_word_lm_tables`` of this LM's copy on ``device`` (uploaded on first use, then reused read-only)."""
        import torch
        dev = torch.device(device)
        key = str(dev)
        if key not in self._dev:
            bufs = [torch.from_numpy(a).to(dev) for a in (self.keys.view(np.int32), self.vals, self.lex_off,
                                                           np.r_[self.lex_tok, 0].astype(np.int32),
                                                           np.r_[self.lex_next, 0].astype(np.int32), self.lex_word)]
            t = _lib.WordLmTables.from_buffer_copy(self._layout)
            t.keys, t.vals, t.lex_off, t.lex_tok, t.lex_next, t.lex_word = (b.data_ptr() for b in bufs)
            self._dev[key] = (t, bufs)
        return self._dev[key][0]

    def score(self, ctx, word, device="cuda"):
        """lnP(word | ctx) for a batch of queries on the GPU (``masr_word_lm_score_f32``): ctx [Q, order-1] and word [Q]
        are word ids (-1 = out of vocabulary).  -> float32 numpy [Q]."""
        import torch
        dev = torch.device(device)
        t = self.tables(dev)
        w = torch.as_tensor(np.asarray(word, np.int32)).to(dev)
        c = torch.as_tensor(np.asarray(ctx, np.int32).reshape(len(w), max(0, self.order - 1))).to(dev).contiguous()
        out = torch.empty(len(w), device=dev, dtype=torch.float32)
        _lib.call("masr_word_lm_score_f32", C.byref(t), c.data_ptr() if c.numel() else None, w.data_ptr(), len(w),
                  out.data_ptr(), torch.cuda.current_stream(dev).cuda_stream)
        return out.cpu().numpy()

