"""The GPU CTC prefix beam search (csrc/beam.cu) from the host: its device buffers and its two launches, for each of its
three forms — one-shot (a batch of whole utterances), streaming (one stream fed chunk by chunk) and pool (every slot of a
stream pool, launched inside the pool's CUDA graph) — without an LM, with a character LM or with a word LM, each with or
without hotwords.  Which entry point, which argument order and which buffers go with a (form, LM kind, hotwords) is decided
here and nowhere else."""
from __future__ import annotations

import ctypes as C
import weakref

import numpy as np
import torch

from ._lib import call

BK_MAX = 40                                  # candidates per frame: the largest cutoff_top_n the top-k kernel takes
ONE_SHOT, STREAM, POOL = "", "_stream", "_pool"      # the forms, named by their entry points' suffix


def check_n_best(n_best, beam_size: int) -> int:
    """``n_best`` as an int in 1..beam_size, else a ValueError."""
    if isinstance(n_best, bool) or not isinstance(n_best, (int, np.integer)):
        raise ValueError(f"n_best must be an integer, got {n_best!r}")
    if not 1 <= int(n_best) <= int(beam_size):
        raise ValueError(f"n_best={n_best} out of range (1..beam_size={beam_size})")
    return int(n_best)


class BeamSearch:
    """One search's device buffers on ``device``.  ``topk`` launches the top-k kernel and ``search`` the prefix beam kernel,
    both through ``eng._k`` of the engine passed in: two calls, so that a caller can put an event between them and run
    ``search`` on another stream.  The search keeps no reference to the engine and only a weak one to the LM (whoever
    launches it keeps the LM alive: the caller, or StreamBeam / PoolBeam), so an engine that keeps a search for reuse is
    still freed as soon as it is dropped, and so is an LM its caller drops.

    ``form``: ONE_SHOT, STREAM or POOL.  ``slots``: utterances (one CTA each); ``rows``: CTC-head rows the top-k kernel
    writes (``cand_id`` / ``cand_lp`` [rows, BK_MAX], ``cand_n`` and, with an LM, ``blank_lp`` [rows]); ``max_frames``: the
    most frames one slot searches (since its start or reset), which sizes its trie and its row of ``out_tok``.  ``lm``:
    None, a ``lm.CharLM`` or a ``lm.WordLM``, fused with weight ``alpha`` and insertion bonus ``beta``.
    The trie per slot is ``masr_ctc_prefix_beam_workspace(1, max_frames)`` (ONE_SHOT, STREAM), or 5 (max_frames *
    beam_size + 1) for POOL, whose kernel never clears a slot's hash: it starts empty here and whoever resets a slot empties
    its range again.  STREAM and POOL keep the beam of every slot in ``state_i`` / ``state_f``; POOL starts slot b afresh
    while ``fresh[b]`` != 0.
    Results: ``out_tok`` [slots, max_frames] and ``out`` [3, slots] = (``score``, ``count`` as int32 bits, fused score):
    ``score`` is what the search reports (approx_ctc with an LM), ``fused`` the score the beam was ranked by (``score``
    itself without an LM).  ``frames`` reads out the onset frame of each reported token.
    ``hot``: None, or hotwords (a ``hotwords.HotwordGraph``, or for POOL a ``hotwords.HotwordBuffer``) searched by the
    ``*_hot`` entry points; ``slot_root`` [slots] (device int32) is each slot's root node in it (-1: no hotwords for that
    slot), all 0 (the graph's root) unless given.  Scores are reported without the hotword credit."""

    def __init__(self, device, form: str, slots: int, rows: int, max_frames: int, beam_size: int = 300,
                 cutoff_prob: float = 0.99, cutoff_top_n: int = 40, lm=None, alpha: float = 0.0, beta: float = 0.0,
                 hot=None, slot_root: torch.Tensor = None):
        self.device, self.form, self.slots, self.max_frames = torch.device(device), form, int(slots), int(max_frames)
        self.beam, self.cutoff, self.top_n = int(beam_size), float(cutoff_prob), int(cutoff_top_n)
        self._lm, self.alpha, self.beta = None if lm is None else weakref.ref(lm), float(alpha), float(beta)
        self.hot = hot
        base = ("masr_ctc_prefix_beam" if lm is None else lm.BEAM) + ("" if hot is None else "_hot")
        self.name = base + form
        dev, i32, f32, S = self.device, torch.int32, torch.float32, self.slots
        pool_n, trie_n = C.c_int64(0), C.c_int64(0)
        call("masr_ctc_prefix_beam_workspace", S, self.max_frames, C.byref(pool_n), C.byref(trie_n))
        self.trie_cap = 5 * (self.max_frames * self.beam + 1) if form == POOL else trie_n.value
        self.cand_id = torch.zeros(rows, BK_MAX, device=dev, dtype=i32)
        self.cand_lp = torch.zeros(rows, BK_MAX, device=dev, dtype=f32)
        self.cand_n = torch.zeros(rows, device=dev, dtype=i32)
        self.blank_lp = None if lm is None else torch.zeros(rows, device=dev, dtype=f32)
        if lm is not None:
            lm.tables(dev)                                 # (uploaded here, never inside a graph capture)
        self.slot_root = None
        if hot is not None:
            hot.tables(dev)
            self.slot_root = torch.zeros(S, device=dev, dtype=i32) if slot_root is None else slot_root
        self.scratch = torch.empty(pool_n.value, device=dev, dtype=f32)
        if form == POOL:
            self.trie_par = torch.full((S * self.trie_cap,), -1, device=dev, dtype=i32)
        else:
            self.trie_par = torch.empty(S * self.trie_cap, device=dev, dtype=i32)
        self.trie_tok = torch.empty(S * self.trie_cap, device=dev, dtype=i32)
        self.state_i = self.state_f = None
        if form != ONE_SHOT:
            si, sf = C.c_int64(0), C.c_int64(0)
            call(base + "_state_size", C.byref(si), C.byref(sf))
            self.state_i = torch.zeros(S, si.value, device=dev, dtype=i32)
            self.state_f = torch.zeros(S, sf.value, device=dev, dtype=f32)
        self.fresh = torch.ones(S, device=dev, dtype=i32) if form == POOL else None
        self.out_tok = torch.zeros(S, self.max_frames, device=dev, dtype=i32)
        self.out = torch.zeros(3, S, device=dev, dtype=f32)
        self.score, self.count = self.out[0], self.out[1].view(i32)
        self.fused = self.out[0] if lm is None else self.out[2]
        self.out_frame = None
        self.nb_tok = None                                 # N-best buffers: allocated by the first ``nbest``

    @property
    def lm(self):
        """The LM this search fuses (None without one, or once its owner has dropped it)."""
        return None if self._lm is None else self._lm()

    def fits(self, slots: int, frames: int, beam_size, cutoff_prob, cutoff_top_n, lm, alpha, beta, hot=None) -> bool:
        """Whether this search has room for ``slots`` utterances of ``frames`` frames and was built with these settings."""
        return (self.slots >= slots and self.max_frames >= frames and (self._lm is None) == (lm is None) and self.lm is lm
                and self.hot is hot
                and (self.beam, self.cutoff, self.top_n, self.alpha, self.beta)
                == (int(beam_size), float(cutoff_prob), int(cutoff_top_n), float(alpha), float(beta)))

    def topk(self, eng, logits: torch.Tensor, ld: int, rows: int):
        """The candidates (and with an LM ln p_blank) of ``rows`` CTC-head rows of ``logits`` (row stride ``ld``)."""
        cands = (self.cand_id.data_ptr(), self.cand_lp.data_ptr(), self.cand_n.data_ptr())
        head = (logits.data_ptr(), ld, rows, eng.V, self.top_n, self.cutoff)
        if self._lm is None:
            eng._k("ctc_topk", "masr_ctc_topk_f32", *head, *cands)
        else:
            eng._k("ctc_topk", "masr_ctc_topk_blank_f32", *head, 0, *cands, self.blank_lp.data_ptr())

    def search(self, eng, lens: int, B: int, bstride: int, resume: int = 0):
        """The prefix beam search of slots 0..B-1 over candidate rows b * bstride + t, t < lens[b] (``lens``: the address
        of a device int32 [B]).  ``resume`` (STREAM): 0 starts the stream at the root, else it continues from its state.
        Host arguments only, no allocation or synchronisation: a POOL search can be captured into a CUDA graph."""
        cands = (self.cand_id.data_ptr(), self.cand_lp.data_ptr(), self.cand_n.data_ptr())
        if self._lm is None:
            blank, fusion, scores = (), (), (self.score.data_ptr(),)
        else:                        # the kernel writes the fused score to out_score and approx_ctc to out_approx
            blank, fusion = (self.blank_lp.data_ptr(),), (C.byref(self.lm.tables(self.device)), self.alpha, self.beta)
            scores = (self.fused.data_ptr(), self.score.data_ptr())
        state = ()
        if self.form != ONE_SHOT:
            state = (self.state_i.data_ptr(), self.state_f.data_ptr(),
                     self.fresh.data_ptr() if self.form == POOL else int(resume))
        hot = () if self.hot is None else (C.byref(self.hot.tables(self.device)), self.slot_root.data_ptr())
        eng._k("prefix_beam", self.name, *cands, *blank, bstride, lens, B, self.beam, 0, *fusion, self.scratch.data_ptr(),
               self.trie_par.data_ptr(), self.trie_tok.data_ptr(), self.trie_cap, *state, self.out_tok.data_ptr(),
               self.max_frames, self.count.data_ptr(), *scores, *hot)

    def frames(self, eng, B: int) -> torch.Tensor:
        """The onset frame of every token that slots 0..B-1 reported in their last search -> ``out_frame`` [slots,
        max_frames] int32 (row b valid up to ``count[b]``), frames counted since each slot's (fresh) start.  One launch
        after ``search``, on the same stream, and never inside a graph capture: the buffer is allocated on first use."""
        if self.out_frame is None:
            self.out_frame = torch.zeros(self.slots, self.max_frames, device=self.device, dtype=torch.int32)
        eng._k("beam_frames", "masr_ctc_prefix_beam_frames", self.trie_par.data_ptr(), self.trie_tok.data_ptr(), self.trie_cap,
               self.out_tok.data_ptr(), self.max_frames, self.count.data_ptr(), B, self.out_frame.data_ptr(),
               self.max_frames)
        return self.out_frame

    def nbest(self, eng, B: int, n: int):
        """The ``n`` best hypotheses of slots 0..B-1 from the beam the last ``search`` left (STREAM and POOL only) ->
        device tensors (tokens [slots, n, max_frames], count [slots, n], score [slots, n], fused [slots, n], hypotheses
        [slots]): hypothesis h of slot b, h < hypotheses[b], ranked as the search ranks its result, so h = 0 is its
        ``out_tok`` / ``count`` / ``score`` / ``fused``; ``score`` is approx_ctc with an LM, and need not decrease down the
        list then (the list is ordered by ``fused``).  A POOL slot that is still fresh reports 0.  One launch after ``search``, on the
        same stream, never inside a graph capture: the buffers are allocated on first use (and again for a larger n)."""
        if self.form == ONE_SHOT:
            raise ValueError("the N-best read-out needs the beam the streaming or pool form keeps")
        if not 1 <= int(n) <= self.beam:
            raise ValueError(f"n={n} out of range (1..{self.beam})")
        n = int(n)
        if self.nb_tok is None or self.nb_tok.shape[1] < n:
            dev = self.device
            self.nb_tok = torch.zeros(self.slots, n, self.max_frames, device=dev, dtype=torch.int32)
            self.nb_out = torch.zeros(3, self.slots, n, device=dev, dtype=torch.float32)
            self.nb_n = torch.zeros(self.slots, device=dev, dtype=torch.int32)
        tok, out = self.nb_tok.view(-1)[:self.slots * n * self.max_frames], self.nb_out.view(3, -1)[:, :self.slots * n]
        score, count = out[0], out[1].view(torch.int32)
        if self._lm is None:
            fusion, scores = (), (score.data_ptr(),)
        else:                        # as search: the fused score to out_score, approx_ctc to out_approx
            fusion, scores = (C.byref(self.lm.tables(self.device)), self.alpha, self.beta), (out[2].data_ptr(), score.data_ptr())
        hot = () if self.hot is None else (C.byref(self.hot.tables(self.device)), self.slot_root.data_ptr())
        base = self.name[:-len(self.form)]
        eng._k("beam_nbest", base + "_nbest", self.trie_par.data_ptr(), self.trie_tok.data_ptr(), self.trie_cap,
               self.state_i.data_ptr(), self.state_f.data_ptr(), self.fresh.data_ptr() if self.form == POOL else None, B, n,
               *fusion, tok.data_ptr(), self.max_frames, count.data_ptr(), *scores, self.nb_n.data_ptr(), *hot)
        S = self.slots
        fused = score if self._lm is None else out[2]
        return (tok.view(S, n, self.max_frames), count.view(S, n), score.view(S, n), fused.view(S, n), self.nb_n)
