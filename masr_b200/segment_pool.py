"""Live streams of any length: every slot of a ``StreamPool`` cut into utterances by the streaming silero VAD on the GPU.

A ``StreamPool`` slot is one ever-growing ``predict_stream`` utterance, bounded by the pool's ``max_frames`` (3000
encoder frames = 2 minutes by default), and every pushed sample goes through the encoder whether anyone speaks or not.
``SegmentingStreamPool`` runs the reference's ``VADPredictor.stream_vad`` (vad_predictor.py:177-213) on every slot
(``GpuSileroVAD.slots``: one encoder and one recurrence launch per push for all slots) and decodes each detected
utterance as a fresh ``predict_stream`` on the slot, finalised at the VAD's end event: what ``predict_long`` does for a
file, done live.  Silence between utterances is never fed to the recogniser.

The rules, per slot (``SegmentPlanner``; W = ``window_size_samples``, pad = ``speech_pad_samples``, all in 16 kHz
samples counted since the slot's last reset):

* every complete window of W samples is one ``stream_vad`` step (``stream_vad_step``) with ``current_sample`` = the end
  of that window;
* a ``start`` event opens a segment at ``s = max(current_sample - pad, end of the previous segment, 0)``;
* an ``end`` event closes it at ``e = min(temp_end + pad, current_sample)``;
* after each push an open segment is fed as far as ``current_sample``, or ``min(current_sample, temp_end + pad)`` while a
  silence is pending, so no fed sample ever lies after the segment's end; the remainder up to ``e`` goes with
  ``is_end=True`` and the recogniser's slot is reset;
* a segment that would outgrow the pool (``max_segment_samples``) is closed at exactly that many samples; while the VAD is
  still triggered a new segment opens at the same sample;
* the end of the stream (``push(..., is_end=True)`` or ``finish``) closes an open segment at the last received sample.

Each piece is pushed through ``StreamPool.push`` (slots grouped by ``is_end`` as ``serve.StreamSessions`` does), so a
segment's result is ``predict_stream`` over exactly its pieces, on a fresh stream.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Tuple

import numpy as np

from .audio import pcm_bytes_to_float32, samples_to_float32
from .engine import FRAME_LEN, FRAME_SHIFT
from .resample import MODEL_RATE
from .stream_pool import StreamSlotError
from .vad import StreamVADState, stream_vad_step


def max_segment_samples(frame_limit: Optional[int]) -> Optional[int]:
    """The longest segment (in samples) whose ``predict_stream`` stays within ``frame_limit`` encoder frames.

    n samples give F = 1 + (n - 400) // 160 fbank frames (none below 400).  ``predict_stream`` runs them in 67-frame
    windows at a stride of 64 (the final push with a 7-frame minimum), each window giving ``subsampled_len`` of its frames,
    and these sum to ``subsampled_len(F) = ((F - 1) // 2 - 1) // 2`` encoder frames whatever the pieces were.  That is at
    most L iff F <= 4 L + 6, i.e. n <= 400 + 160 (4 L + 5) + 159 = 640 L + 1359 (1,921,359 samples, 120.08 s, at the
    default L = 3000).  None: no limit."""
    if frame_limit is None:
        return None
    return FRAME_LEN + FRAME_SHIFT * (4 * int(frame_limit) + 5) + FRAME_SHIFT - 1


class SegmentPlanner:
    """The host rules of one slot (module docstring): window probabilities in, ASR pieces out.  Pure bookkeeping, no GPU.

    ``windows(probs)`` steps the VAD over one push's complete windows and returns the pieces to push, in order, as
    ``(a, b, is_end)`` sample ranges; ``finish(received)`` closes an open segment at ``received``.  ``segments`` lists
    every closed ``(start, end)``; ``open`` is the open segment's start (or None)."""

    OPTIONS = ("threshold", "min_silence_duration_ms", "speech_pad_ms")       # the GpuSileroVAD keywords it uses

    def __init__(self, window: int, max_samples: Optional[int], threshold: float = 0.5, min_silence_duration_ms: int = 100,
                 speech_pad_ms: int = 30, sampling_rate: int = MODEL_RATE):
        self.W, self.max_samples, self.sr = int(window), max_samples, int(sampling_rate)
        self.threshold, self.min_silence_duration_ms, self.speech_pad_ms = threshold, min_silence_duration_ms, speech_pad_ms
        self.pad = self.sr * speech_pad_ms / 1000                       # float, as the reference computes it
        self.reset()

    def reset(self):
        self.st = StreamVADState()
        self.open: Optional[int] = None
        self.fed = 0                     # the open segment has been fed [open, fed)
        self.last_end = 0
        self.segments: List[Tuple[int, int]] = []

    def feed_limit(self) -> int:
        """How far an open segment may be fed now: no later than any end the VAD can still announce for it."""
        st = self.st
        return st.current_sample if not st.temp_end else min(st.current_sample, int(st.temp_end + self.pad))

    def keep_from(self) -> int:
        """The earliest sample any later piece can start at (the host ring of the slot keeps everything from here)."""
        if self.open is not None:
            return self.fed
        # a later start is at least the end of the next window minus the pad
        return max(self.last_end, int(self.st.current_sample + self.W - self.pad), 0)

    def _feed_to(self, x: int, final: bool, out: list):
        while self.max_samples is not None and x - self.open > self.max_samples:       # forced cut
            cut = self.open + self.max_samples
            out.append((self.fed, cut, True))
            self.segments.append((self.open, cut))
            self.open = self.fed = self.last_end = cut
        if final:
            out.append((self.fed, x, True))
            self.segments.append((self.open, x))
            self.open, self.fed, self.last_end = None, x, x
        elif x > self.fed:
            out.append((self.fed, x, False))
            self.fed = x

    def windows(self, probs) -> List[Tuple[int, int, bool]]:
        out: list = []
        st = self.st
        for p in probs:
            st.current_sample += self.W
            ev = stream_vad_step(st, float(p), self.sr, self.threshold, self.min_silence_duration_ms, self.speech_pad_ms)
            if ev is None:
                continue
            if "start" in ev:
                self.open = self.fed = max(ev["start"], self.last_end, 0)
            elif self.open is not None:
                self._feed_to(min(ev["end"], st.current_sample), True, out)
        if self.open is not None:
            self._feed_to(self.feed_limit(), False, out)
        return out

    def finish(self, received: int) -> List[Tuple[int, int, bool]]:
        out: list = []
        if self.open is not None:
            self._feed_to(max(int(received), self.fed), True, out)
        return out


class SegmentingStreamPool:
    """``StreamPool`` slots segmented by the streaming GPU silero VAD (module docstring for the rules).

    ``push(audio, is_end=False)`` -> per pushed slot ``{'segments': [{'start', 'end', 'text', 'score'}, ...] (closed
    during this push), 'partial': {'start', 'text', 'score'} | None (the open segment's latest result), 'speech': bool}``.
    With a pool made with ``timestamps=True`` segments and partials also carry ``'tokens'`` (+ ``'words'``), timed in
    seconds since the slot's stream started, and with a pool made with ``n_best`` they carry ``'n_best'`` (the
    segment's or partial's best hypotheses, ``[{'text', 'score'}, ...]``, entry 0 its own text and score).
    ``is_end`` (one bool or ``{slot: bool}``) ends a slot's stream: its open segment closes at the last received sample and
    the slot starts a new stream (with an empty transcript) on its next push.  ``transcript(slot)`` joins the closed
    segments as ``predict_long`` does.  Per-slot errors (undecodable input, a rate other than 16 kHz, a failure of the slot's recognition) fail only
    that slot, as ``StreamPool.push`` does: it is reset, its exception lands in ``last_errors`` and ``on_error`` decides
    between raising ``StreamSlotError`` and returning the healthy slots' results."""

    def __init__(self, pool, vad):
        """``pool``: a ``StreamPool``; ``vad``: a ``GpuSileroVAD`` (its keyword options are the VAD's)."""
        self.pool, self.vad, self.S = pool, vad, pool.S
        self.W = int(vad.kw["window_size_samples"])
        cap, max_len = pool.pool.frame_bounds()
        limits = [v for v in (cap, None if max_len is None else max_len - 1) if v is not None]
        self.max_samples = max_segment_samples(min(limits) if limits else None)
        self.vad_slots = vad.slots(self.S)
        kw = {k: vad.kw[k] for k in SegmentPlanner.OPTIONS}
        self.planners = [SegmentPlanner(self.W, self.max_samples, **kw) for _ in range(self.S)]
        self.last_probs: Dict[int, np.ndarray] = {}           # the VAD's window probabilities of the last push
        self.last_errors: Dict[int, Exception] = {}
        # per slot: samples from ring_base on (what later pieces can still need), samples received, the open segment's
        # latest result, the closed segments, whether the stream has ended
        self.ring: List[np.ndarray] = [np.zeros(0, np.float32)] * self.S
        self.ring_base, self.received = [0] * self.S, [0] * self.S
        self.partial: List[Optional[dict]] = [None] * self.S
        self.closed: List[List[dict]] = [[] for _ in range(self.S)]
        self.ended = [False] * self.S

    def _clear(self, slots):
        for s in slots:
            self.pool.reset_stream(s)
            self.vad_slots.reset(s)
            self.planners[s].reset()
            self.ring[s], self.ring_base[s], self.received[s] = np.zeros(0, np.float32), 0, 0
            self.partial[s], self.closed[s], self.ended[s] = None, [], False

    def reset_stream(self, slot: int):
        """Start ``slot`` over: VAD state, recogniser stream and transcript."""
        self._clear([slot])

    def set_hotwords(self, slot: int, hotwords):
        """``StreamPool.set_hotwords`` for ``slot``'s stream: legal while the slot has received no audio since its reset.
        The list holds for every utterance the VAD cuts from the stream (the per-utterance resets keep it)."""
        if self.received[slot] != 0:
            raise ValueError(f"slot {slot} has received audio since its reset: set its hotwords right after a reset")
        self.pool.set_hotwords(slot, hotwords)

    def transcript(self, slot: int) -> dict:
        """The closed segments of the slot's stream joined as ``predict_long`` joins its segments: '，' between non-empty
        texts, the mean score rounded to 2 (0 without segments)."""
        texts, scores = "", []
        for r in self.closed[slot]:
            if r["text"] != "":
                texts = texts + "，" + r["text"]
            scores.append(r["score"])
        if texts[:1] == "，":
            texts = texts[1:]
        return {"text": texts, "score": round(sum(scores) / len(scores), 2) if scores else 0}

    def finish(self, slot: int, on_error: str = "raise"):
        """End the slot's stream (``push({slot: empty}, is_end=True)``)."""
        return self.push({slot: np.zeros(0, np.float32)}, is_end=True, on_error=on_error)

    def push(self, audio: Dict[int, object], is_end=False, channels: int = 1, samp_width: int = 2, on_error: str = "raise",
             sample_rate=MODEL_RATE):
        self.last_errors = errors = {}
        ends = {s: bool(is_end.get(s, False) if isinstance(is_end, dict) else is_end) for s in audio}
        new = {}
        for s in sorted(audio):
            if not 0 <= s < self.S:
                raise IndexError(f"slot {s} out of range (0..{self.S - 1})")
            a = audio[s]
            try:
                rate = int(sample_rate.get(s, MODEL_RATE) if isinstance(sample_rate, dict) else sample_rate)
                if rate != MODEL_RATE:
                    raise ValueError(f"masr_b200: the segmenting stream pool takes {MODEL_RATE} Hz audio only (got {rate} Hz)")
                new[s] = samples_to_float32(a) if isinstance(a, np.ndarray) else pcm_bytes_to_float32(a, channels, samp_width)
            except Exception as e:                    # this slot only; its state is untouched
                errors[s] = e
        for s in new:
            if self.ended[s]:                         # the first push after an ended stream starts a new one
                self._clear([s])
        probs = self.vad_slots.advance(new) if new else {}
        self.last_probs = probs
        plans: Dict[int, list] = {}
        for s, x in new.items():
            if len(x):
                self.ring[s] = np.concatenate([self.ring[s], x]) if len(self.ring[s]) else np.array(x, np.float32)
            self.received[s] += len(x)
            pl = self.planners[s]
            plans[s] = pl.windows(probs[s]) + (pl.finish(self.received[s]) if ends[s] else [])
        seg_out: Dict[int, List[dict]] = {s: [] for s in new}
        failed = set()
        rounds = max((len(v) for v in plans.values()), default=0)
        for r in range(rounds):
            grp = {False: {}, True: {}}
            for s, pieces in plans.items():
                if r < len(pieces) and s not in failed:
                    a, b, end = pieces[r]
                    grp[end][s] = (a, b)
            for end in (False, True):
                if not grp[end]:
                    continue
                pieces = {s: self.ring[s][a - self.ring_base[s]:b - self.ring_base[s]] for s, (a, b) in grp[end].items()}
                for s in grp[end]:                    # the recogniser's stream starts at the segment's start
                    pl = self.planners[s]
                    k = len(self.closed[s])
                    self.pool.t0[s] = (pl.segments[k][0] if k < len(pl.segments) else pl.open) / MODEL_RATE
                res = self.pool.push(pieces, is_end=end, on_error="return")
                for s, e in self.pool.last_errors.items():
                    errors[s] = e
                    failed.add(s)
                for s, (a, b) in grp[end].items():
                    if s in failed:
                        continue
                    got = res.get(s)
                    if end:
                        seg_start = self.planners[s].segments[len(self.closed[s])][0]
                        text, score = (got["text"], got["score"]) if got is not None else ("", 0.0)
                        rec = {"start": seg_start, "end": b, "text": text, "score": score}
                        if self.pool.timestamps:
                            rec.update({k: v for k, v in got.items() if k in ("tokens", "words")} if got is not None
                                       else {"tokens": []})
                        if self.pool.n_best is not None:
                            rec["n_best"] = got["n_best"] if got is not None else [{"text": "", "score": 0.0}]
                        self.closed[s].append(rec)
                        seg_out[s].append(rec)
                        self.partial[s] = None
                        self.pool.reset_stream(s)
                    elif got is not None:
                        self.partial[s] = {"start": self.planners[s].open, "text": got["text"], "score": got["score"]}
                        self.partial[s].update({k: got[k] for k in ("tokens", "words", "n_best") if k in got})
        for s in failed:                              # the slot's stream is abandoned: start it over
            self._clear([s])
        out: Dict[int, dict] = {}
        for s in new:
            if s in failed:
                continue
            pl = self.planners[s]
            if ends[s]:
                self.ended[s] = True
                self.vad_slots.reset(s)
            else:
                keep = min(pl.keep_from(), self.received[s])
                drop = keep - self.ring_base[s]
                if drop > 0:
                    self.ring[s] = self.ring[s][drop:].copy()
                    self.ring_base[s] = keep
            out[s] = {"segments": seg_out[s], "partial": self.partial[s], "speech": bool(pl.st.triggered) and not ends[s]}
        if errors and on_error == "raise":
            raise StreamSlotError(errors, out)
        return out
