"""CPU: the streaming VAD's host rules.

* ``GpuSileroVAD.stream_vad`` / ``__call__`` / ``reset_states`` / ``_validate_input`` with the network replaced by a
  script, against the reference's own code over the same scripts (tests/golden/stream_vad_golden.json);
* the segmenting pool's piece schedule (``SegmentPlanner``) on scripted tracks, and its capacity
  (``max_segment_samples``) against ``predict_stream``'s chunk arithmetic.
"""
import json
import os

import numpy as np
import pytest

from masr_b200 import vad
from masr_b200.engine import num_frames, subsampled_len
from masr_b200.predict import CACHED_FEATURE_NUM, DECODING_WINDOW, chunk_starts
from masr_b200.segment_pool import SegmentPlanner, max_segment_samples

with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "stream_vad_golden.json"), encoding="utf-8") as f:
    GOLDEN = json.load(f)
DEFAULTS = dict(threshold=0.5, min_silence_duration_ms=100, speech_pad_ms=30)


class ScriptedVAD(vad.GpuSileroVAD):
    """The network replaced by a script: every row gets the next probability; the state is a count of the calls since
    the last reset (what the golden's session stand-in feeds as h)."""

    def __init__(self, probs, **kw):
        vad.ProbabilityVAD.__init__(self, None, **kw)
        self.it, self.fed = iter(probs), []
        self._init_stream_state()

    def _run_windows(self, x, sr):
        self._slots = self._slots or [0]
        self.fed.append([list(x.shape), float(self._slots[0])])
        self._slots[0] += 1
        return np.full((x.shape[0], 1), next(self.it), np.float32)


def test_stream_vad_equals_the_reference():
    """Including the reference's reset on the first call after reset_states, which clears the first window's
    current_sample (a start announced at -pad)."""
    for case in GOLDEN["streams"]:
        probs = GOLDEN["tracks"][case["track"]]
        v = ScriptedVAD(probs, window_size_samples=case["window"], **case["kw"])
        got = [v.stream_vad(np.zeros(case["window"], np.float32), 16000, case["return_seconds"]) for _ in probs]
        assert got == case["events"], case
    assert ScriptedVAD([0.9]).stream_vad(np.zeros(100, np.float32), 16000) is None      # shorter than a window


def test_call_validation_and_carried_state_rules():
    calls = GOLDEN["calls"]
    v = ScriptedVAD([c["out"][0][0] for c in calls if "out" in c])
    for c in calls:
        if "error" in c:
            with pytest.raises(ValueError) as e:
                v(np.zeros(c["shape"], np.float32), c["sr"])
            assert str(e.value) == c["error"]
            continue
        assert v(np.zeros(c["shape"], np.float32), c["sr"]).tolist() == c["out"]
        assert v.fed[-1] == c["fed"]          # x[::step] on [B, W] keeps every step-th row; resets as the reference
    with pytest.raises(ValueError, match="Too many dimensions"):
        v(np.zeros((1, 1, 512), np.float32), 16000)


# ---- the segmenting pool's piece schedule ------------------------------------------------------------------------------
def _track(rng, n):
    """Sticky speech / silence runs with some windows anywhere in [0, 1)."""
    out = []
    while len(out) < n:
        k = int(rng.integers(1, 40))
        base = rng.uniform(0.5, 1.0, k) if rng.random() < 0.5 else rng.uniform(0.0, 0.5, k)
        out.extend(np.where(rng.random(k) < 0.15, rng.uniform(0.0, 1.0, k), base).tolist())
    return out[:n]


def _plan(probs, W, pushes, max_samples, kw):
    """Drive a SegmentPlanner as the pool does; each push of n samples completes some windows; the stream ends."""
    pl, received, done, pieces = SegmentPlanner(W, max_samples, **kw), 0, 0, []
    for n in pushes:
        received += n
        pieces += pl.windows(probs[done:received // W])
        done = received // W
    return pl, pieces + pl.finish(received), received


def _want_segments(probs, W, received, max_samples, kw):
    """The documented rules applied directly: start at max(current_sample - pad, previous end, 0), end at
    min(temp_end + pad, current_sample) or at the end of the stream, forced cuts of exactly max_samples."""
    st, pad, out, cur, last = vad.StreamVADState(), 16000 * kw["speech_pad_ms"] / 1000, [], None, 0
    for p in probs[:received // W]:
        st.current_sample += W
        ev = vad.stream_vad_step(st, p, 16000, kw["threshold"], kw["min_silence_duration_ms"], kw["speech_pad_ms"])
        if ev and "start" in ev:
            cur = max(int(st.current_sample - pad), last, 0)
        elif ev:
            last = min(ev["end"], st.current_sample)
            out.append((cur, last))
    if st.triggered:
        out.append((cur, received))
    cut = []
    for s, e in out:
        while max_samples is not None and e - s > max_samples:
            cut.append((s, s + max_samples))
            s += max_samples
        cut.append((s, e))
    return cut


@pytest.mark.parametrize("W", [512, 1536])
@pytest.mark.parametrize("kw", [DEFAULTS, dict(threshold=0.6, min_silence_duration_ms=300, speech_pad_ms=100),
                                dict(threshold=0.3, min_silence_duration_ms=50, speech_pad_ms=0)])
def test_piece_schedule_on_scripted_tracks(W, kw):
    rng = np.random.default_rng(W + kw["speech_pad_ms"])
    for trial in range(40):
        probs = _track(rng, 400)
        total = len(probs) * W + int(rng.integers(0, W))
        cuts = np.sort(rng.integers(0, total, int(rng.integers(1, 40))))
        max_samples = [None, 20000, 6 * W + 7][trial % 3]
        pl, pieces, received = _plan(probs, W, np.diff(np.r_[0, cuts, total]).tolist(), max_samples, kw)
        assert pl.segments == _want_segments(probs, W, received, max_samples, kw)
        # segments never overlap; each one's pieces are consecutive from its start and the last (is_end) stops at its
        # end: concatenated they are exactly samples[s:e], and no fed sample lies after the end
        at = 0
        for s, e in pl.segments:
            assert at <= s < e
            at = s
            while True:
                a, b, end = pieces.pop(0)
                assert a == at and b <= e
                at = b
                if end:
                    break
            assert at == e
        assert not pieces


def test_a_pending_silence_is_held_back_and_the_forced_cut_fires_at_the_capacity():
    W = 512
    pl = SegmentPlanner(W, None, **DEFAULTS)
    assert pl.windows([0.9] * 4 + [0.1] * 3) == [(W - 480, 5 * W + 480, False)]     # fed up to temp_end + pad only
    assert pl.windows([0.1, 0.1]) == [(5 * W + 480, 5 * W + 480, True)] and pl.segments == [(W - 480, 5 * W + 480)]
    cap = max_segment_samples(200)
    pl, _, received = _plan([0.9] * 700, W, [8000] * 44 + [800], cap, DEFAULTS)
    assert [e - s for s, e in pl.segments[:-1]] == [cap] * (len(pl.segments) - 1) and len(pl.segments) > 2
    assert pl.segments[0][0] == W - 480 and pl.segments[-1][1] == received


def _frames_fed(pieces):
    """Encoder frames predict_stream produces for consecutive pieces (the last with is_end): its fbank frame grid,
    67-frame windows at stride 64 and the 3 carried frames (predict.py:303-330)."""
    total = cached = n = out = 0
    for i, k in enumerate(pieces):
        n += k
        cached, total = cached + num_frames(n) - total, num_frames(n)
        starts = chunk_starts(cached, i == len(pieces) - 1)
        for c in starts:
            out += subsampled_len(min(c + DECODING_WINDOW, cached) - c)
        if starts:
            cached -= min(starts[-1] + DECODING_WINDOW, cached) - CACHED_FEATURE_NUM
    return out


@pytest.mark.parametrize("L", [1, 7, 200, 3000])
def test_capacity_is_the_largest_segment_within_the_frame_limit(L):
    n_max = max_segment_samples(L)
    assert max_segment_samples(3000) == 1921359 and max_segment_samples(None) is None
    rng = np.random.default_rng(L)
    for n in (n_max - 1, n_max, n_max + 1, n_max + 160):
        for trial in range(5):
            cuts = np.sort(rng.integers(0, n, int(rng.integers(0, 12)))) if trial else np.zeros(0, np.int64)
            f = _frames_fed(np.diff(np.r_[0, cuts, n]).tolist())
            assert f == subsampled_len(num_frames(n)) and (f <= L) == (n <= n_max), (n, n_max, f)
