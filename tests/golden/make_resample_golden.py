"""Freeze ``predictor_golden_resample.json``: the UNMODIFIED reference ``MASRPredictor`` (conformer.yml, ctc_greedy, CPU,
synthetic weights of ``masr_b200.synth``; built by ``oracle.ref_shims.build_real_predictor``) on audio at other sample
rates than 16 kHz.

resampy is not installed, so a ``resampy`` module whose ``resample`` is ``oracle.resample.resample`` is put into
``sys.modules`` before the reference is imported.  The golden therefore pins the reference's CONTROL FLOW around
resampling (which calls resample, on which samples, labelled with which rate — including the streaming quirk that the
16 kHz remainder is resampled again as if it were at the new chunk's rate); the resampling arithmetic itself is pinned
only to the restatement in ``oracle/resample.py``.

    python tests/golden/make_resample_golden.py        # build container only (needs the reference tree)
"""
import json
import os
import sys
import tempfile
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
HERE = os.path.dirname(os.path.abspath(__file__))

from oracle import ref_shims  # noqa: E402
from oracle import resample as oracle_resample  # noqa: E402

CALLS = []


def _resample(x, sr_orig, sr_new, filter="kaiser_best", **kw):
    assert filter == "kaiser_best" and not kw
    CALLS.append((int(len(x)), int(sr_orig), int(sr_new)))
    return oracle_resample.resample(np.asarray(x, np.float32), sr_orig, sr_new)


sys.modules["resampy"] = types.SimpleNamespace(resample=_resample)

from masr_b200 import synth  # noqa: E402

WHOLE = [(8000, 40, 2.3), (22050, 41, 1.9), (44100, 42, 2.1), (48000, 43, 2.6)]     # (rate, audio seed, seconds)
STREAMS = [(48000, 44, 4.2, 24000), (8000, 45, 3.7, 4000)]                          # (rate, audio seed, seconds, push)
LONG = (48000, 46, 9.0)                                                               # (rate, audio seed, seconds)
# the scripted VAD's segments, in 16 kHz samples of the resampled recording
LONG_STAMPS = [{"start": 4000, "end": 36000}, {"start": 52000, "end": 100000}, {"start": 110000, "end": 140000}]


def make_audio(seed, n):
    return synth.speechlike_audio(seed, n)


class ScriptedVAD:
    """Stands in for the silero VAD: fixed segments, and a record of what it was given."""

    def __init__(self, stamps):
        self.stamps, self.seen = stamps, []

    def get_speech_timestamps(self, samples, sampling_rate):
        self.seen.append((int(len(samples)), int(sampling_rate)))
        return [dict(s) for s in self.stamps]


def result(r):
    return None if r is None else {"text": r["text"], "score": float(r["score"])}


def main():
    with tempfile.TemporaryDirectory() as tmp:
        pred = ref_shims.build_real_predictor(tmp, streaming=True, wseed=0)
        data = {"wseed": 0, "whole": [], "streams": [], "long": None}
        for sr, seed, secs in WHOLE:
            x = make_audio(seed, int(sr * secs))
            del CALLS[:]
            r = pred.predict(audio_data=x.copy(), sample_rate=sr)
            assert CALLS == [(len(x), sr, 16000)], CALLS
            data["whole"].append({"rate": sr, "aseed": seed, "samples": len(x), "result": result(r)})
            print("whole", sr, r)
        for sr, seed, secs, push in STREAMS:
            x = make_audio(seed, int(sr * secs))
            pcm = (np.clip(x, -1, 1) * 32767).astype("<i2")
            pred.reset_stream()
            del CALLS[:]
            pushes = []
            for s in range(0, len(pcm), push):
                r = pred.predict_stream(audio_data=pcm[s:s + push].tobytes(), is_end=s + push >= len(pcm), sample_rate=sr)
                pushes.append(result(r))
            data["streams"].append({"rate": sr, "aseed": seed, "samples": len(x), "push": push, "pushes": pushes,
                                    "resample_calls": [list(c) for c in CALLS]})
            print("stream", sr, [c[0] for c in CALLS], pushes[-1])
        pred.reset_stream()
        sr, seed, secs = LONG
        x = make_audio(seed, int(sr * secs))
        vadp = ScriptedVAD(LONG_STAMPS)
        pred.vad_predictor = vadp
        del CALLS[:]
        r = pred.predict_long(audio_data=x.copy(), sample_rate=sr)
        assert CALLS[0] == (len(x), sr, 16000) and len(CALLS) == 1, CALLS
        data["long"] = {"rate": sr, "aseed": seed, "samples": len(x), "stamps": LONG_STAMPS, "vad_saw": list(vadp.seen[0]),
                        "result": result(r)}
        print("long", r, vadp.seen)
    with open(os.path.join(HERE, "predictor_golden_resample.json"), "w", encoding="utf-8") as f:
        json.dump(data, f, ensure_ascii=False, indent=1)


if __name__ == "__main__":
    main()
