"""Token and word times of a transcript: the one place that knows the frame clock of each engine and turns CTC frame spans
into ``{'token', 'start', 'end'}`` and ``{'word', 'start', 'end'}`` lists (DESIGN.md §2, timestamps).

Frame clock: encoder output frame t starts at t * dt seconds, dt = 10 ms feature frames times the engine's output stride
(4 for Conformer, Squeezeformer and DeepSpeech2, 8 for EfficientConformer); no receptive-field centring.  A span [s, e)
of frames is reported as start s * dt, end e * dt, both rounded to the millisecond.

Spans come from the decoder:
  greedy  each emitted token is one run of equal non-blank argmax ids: start = its first frame, end = its last frame + 1;
  beam    a token's frame is the onset of its prefix-trie node, the first frame after whose selection the prefix ending in
          that token was in the beam (csrc/beam.cu, masr_ctc_prefix_beam_frames): start = onset, end = onset + 1.  The
          search does not track where a token's run ends, so a beam token's end says nothing about its duration.
Words (vocabularies with ``<space>``): tokens split on ``<space>``; a word runs from its first letter's start to its last
letter's end."""
from __future__ import annotations

from typing import List, Sequence, Tuple

import numpy as np

SPACE = "<space>"
FEATURE_SHIFT_S = 0.01                     # one 10 ms fbank frame


def frame_seconds(eng) -> float:
    """dt of ``eng``'s encoder output frames, in seconds."""
    from .engine import EfficientConformerEngine
    return FEATURE_SHIFT_S * (8 if isinstance(eng, EfficientConformerEngine) else 4)


def greedy_spans(ids: Sequence[int], blank: int = 0) -> Tuple[List[int], List[int], List[int]]:
    """Per-frame argmax ids -> (tokens, start frames, end frames): one token per run of equal non-blank ids."""
    ids = np.asarray(ids, dtype=np.int64).reshape(-1)
    if ids.size == 0:
        return [], [], []
    cut = np.flatnonzero(np.diff(ids)) + 1                     # first frame of every run but the first
    starts = np.concatenate(([0], cut))
    ends = np.concatenate((cut, [ids.size]))
    keep = ids[starts] != blank
    return ids[starts][keep].tolist(), starts[keep].tolist(), ends[keep].tolist()


def beam_spans(onsets: Sequence[int]) -> Tuple[List[int], List[int]]:
    """Onset frames of a beam result's tokens -> (start frames, end frames)."""
    starts = [int(f) for f in onsets]
    return starts, [f + 1 for f in starts]


def token_times(tokens: Sequence[int], starts: Sequence[int], ends: Sequence[int], vocab: Sequence[str], dt: float,
                offset: float = 0.0) -> List[dict]:
    """Frame spans -> ``[{'token', 'start', 'end'}]`` in seconds, shifted by ``offset`` seconds."""
    return [{'token': vocab[t], 'start': round(offset + s * dt, 3), 'end': round(offset + e * dt, 3)}
            for t, s, e in zip(tokens, starts, ends)]


def word_times(tokens: Sequence[dict]) -> List[dict]:
    """``token_times`` output -> ``[{'word', 'start', 'end'}]``, split on ``<space>`` tokens."""
    words, cur = [], []
    for tok in list(tokens) + [{'token': SPACE}]:
        if tok['token'] != SPACE:
            cur.append(tok)
        elif cur:
            words.append({'word': ''.join(c['token'] for c in cur), 'start': cur[0]['start'], 'end': cur[-1]['end']})
            cur = []
    return words


def attach(result: dict, tokens: Sequence[int], starts: Sequence[int], ends: Sequence[int], vocab: Sequence[str], dt: float,
           offset: float = 0.0) -> dict:
    """Add ``'tokens'`` (and ``'words'`` when ``vocab`` has ``<space>``) to ``result`` and return it."""
    result['tokens'] = token_times(tokens, starts, ends, vocab, dt, offset)
    if SPACE in vocab:
        result['words'] = word_times(result['tokens'])
    return result


def greedy_result(result: dict, ids: Sequence[int], vocab: Sequence[str], dt: float, offset: float = 0.0) -> dict:
    """``attach`` the greedy spans of per-frame ids ``ids``."""
    return attach(result, *greedy_spans(ids), vocab, dt, offset)


def beam_result(result: dict, tokens: Sequence[int], onsets: Sequence[int], vocab: Sequence[str], dt: float,
                offset: float = 0.0) -> dict:
    """``attach`` the spans of a beam result's tokens and their onset frames."""
    return attach(result, tokens, *beam_spans(onsets), vocab, dt, offset)


def sentences(segments: Sequence[Tuple[int, int]], results: Sequence[dict], sample_rate: int) -> List[dict]:
    """``predict_long``'s ``'sentences'``: per VAD segment (start, end sample) whose result has non-empty text, ``{'text',
    'score', 'start', 'end', 'tokens'}`` (+ ``'words'``) with the segment's bounds in seconds; ``results`` are timed with
    their segment's start as the offset, so their token times are already absolute."""
    out = []
    for (s0, s1), r in zip(segments, results):
        if r['text'] != '':
            out.append(dict(r, start=round(s0 / sample_rate, 3), end=round(s1 / sample_rate, 3)))
    return out
