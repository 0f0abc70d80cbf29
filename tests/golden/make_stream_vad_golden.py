"""Freeze the reference's streaming VAD (``VADPredictor.stream_vad`` / ``reset_states`` / ``__call__`` /
``_validate_input``, masr/infer_utils/vad_predictor.py:54-104, 177-213) over scripted speech-probability tracks ->
stream_vad_golden.json.  The onnxruntime session is replaced by a script that returns the next probability and
``h + 1`` (so ``h`` counts the calls since the last reset): the reference's own ``__call__`` runs, with its input
validation and reset rules.  Needs neither onnxruntime nor the model file; run with the reference tree present.
"""
import json
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
HERE = os.path.dirname(os.path.abspath(__file__))

from oracle import ref_shims  # noqa: E402

TRACKS = {
    "speech_at_first_window": [0.9, 0.8, 0.7] + [0.1] * 7,
    # default min silence 1600 samples: 4 silent windows of 512 keep the segment, 5 close it
    "silence_just_under": [0.1, 0.9, 0.9, 0.2, 0.2, 0.2, 0.2, 0.9, 0.9] + [0.1] * 6,
    "silence_just_over": [0.1, 0.9, 0.9, 0.2, 0.2, 0.2, 0.2, 0.2, 0.9, 0.9] + [0.1] * 6,
    # at or above threshold while a silence is pending clears it; between the thresholds does not
    "retrigger_pending": [0.0, 0.6, 0.2, 0.2, 0.5, 0.2, 0.2, 0.2, 0.4] + [0.2] * 7,
    "exact_thresholds": [0.5, 0.35, 0.35, 0.3499, 0.2, 0.2, 0.2, 0.2, 0.2, 0.6, 0.45, 0.45] + [0.0] * 8,
    "random_sticky": [float(v) for v in np.round(np.clip(np.repeat(np.random.default_rng(11).random(20), 4), 0, 1), 2)],
}
OPTIONS = [{}, {"threshold": 0.6, "min_silence_duration_ms": 300, "speech_pad_ms": 100},
           {"threshold": 0.3, "min_silence_duration_ms": 50, "speech_pad_ms": 0}]
CALLS = [((512,), 16000), ((1, 512), 16000), ((3, 512), 32000), ((2, 512), 16000), ((4, 1024), 48000),
         ((2, 1024), 16000), ((1, 512), 16000), ((1, 1536), 16000), ((1, 256), 16000), ((1, 512), 22050),
         ((1, 512), 16000), ((5, 512), 16000)]


class _Session:
    def __init__(self, probs):
        self.it, self.fed = iter(probs), []

    def run(self, _, feeds):
        self.fed.append((list(feeds["input"].shape), float(feeds["h"].reshape(-1)[0])))
        return np.full((feeds["input"].shape[0], 1), next(self.it), np.float32), feeds["h"] + 1, feeds["c"] + 1


def _vad(VADPredictor, kw, W, probs):
    v = object.__new__(VADPredictor)
    v.threshold, v.min_speech_duration_ms, v.window_size_samples = kw.get("threshold", 0.5), 250, W
    v.min_silence_duration_ms, v.speech_pad_ms = kw.get("min_silence_duration_ms", 100), kw.get("speech_pad_ms", 30)
    v.sample_rates, v.session = [8000, 16000], _Session(probs)
    VADPredictor.reset_states(v)
    return v


def gen():
    ref_shims.install()
    sys.modules.setdefault("onnxruntime", types.ModuleType("onnxruntime"))
    from masr.infer_utils.vad_predictor import VADPredictor
    streams = []
    for name, probs in TRACKS.items():
        for i, kw in enumerate(OPTIONS):
            for W, secs in ((512, False), (1536, i == 0)):
                v = _vad(VADPredictor, kw, W, probs)
                events = [v.stream_vad(np.zeros(W, np.float32), 16000, return_seconds=secs) for _ in probs]
                streams.append({"track": name, "kw": kw, "window": W, "return_seconds": secs, "events": events})
    calls = []
    v = _vad(VADPredictor, {}, 512, [0.25 + 0.01 * i for i in range(len(CALLS))])
    for shape, sr in CALLS:
        try:
            out = v(np.zeros(shape, np.float32), sr)
            calls.append({"shape": list(shape), "sr": sr, "out": out.tolist(), "fed": v.session.fed[-1]})
        except ValueError as e:
            calls.append({"shape": list(shape), "sr": sr, "error": str(e)})
    with open(os.path.join(HERE, "stream_vad_golden.json"), "w", encoding="utf-8") as f:
        json.dump({"tracks": TRACKS, "streams": streams, "calls": calls}, f, separators=(",", ":"))


if __name__ == "__main__":
    gen()
