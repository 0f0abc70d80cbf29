"""CPU: the resampling restatement (oracle/resample.py, resampy's kaiser_best loop) — its table, its length rule, its
signal properties, its vectorised loop against the literal per-output loop, and the oracle chain (resample -> fbank ->
Conformer -> greedy) against the reference predictor's outputs frozen in predictor_golden_resample.json."""
import json
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN, synth_weights
from masr_b200 import resample as product
from masr_b200 import synth
from oracle import conformer as oc, ctc as octc, fbank as ob
from oracle import resample as orr

SCORE_TOL = 1e-3


def literal_resample(x, sr_orig, sr_new=16000):
    """resampy's interpolation loop written out per output sample and per tap (slow; small inputs only)."""
    ratio = float(sr_new) / sr_orig
    n_out = int(len(x) * sr_new / sr_orig)
    win = orr.kaiser_best_table() * ratio if ratio < 1 else orr.kaiser_best_table()
    delta = np.diff(win, append=win[-1])
    nwin, scale = len(win), min(1.0, ratio)
    step = int(scale * 512)
    t_out = np.arange(n_out) * (1.0 / ratio)
    y = np.zeros(n_out, np.float32)
    for t in range(n_out):
        n = int(t_out[t])
        frac = scale * (t_out[t] - n)
        for right in (False, True):
            if right:
                frac = scale - frac
            idx = frac * 512
            off = int(idx)
            eta = idx - off
            taps = min(len(x) - n - 1, (nwin - off) // step) if right else min(n + 1, (nwin - off) // step)
            for i in range(taps):
                w = win[off + i * step] + eta * delta[off + i * step]
                xi = x[n + i + 1] if right else x[n - i]
                y[t] = np.float32(np.float64(y[t]) + w * np.float64(xi))
    return y


def sine(sr, f, amp, seconds=1.0):
    t = np.arange(int(sr * seconds)) / sr
    return (amp * np.sin(2 * np.pi * f * t)).astype(np.float32)


def test_table():
    w = orr.kaiser_best_table()
    assert w.shape == (32769,) and w.dtype == np.float64
    assert w[0] == orr.ROLLOFF == 0.9475937167399596
    assert 0 < w[-1] < 1e-7                                      # the Kaiser window's tail
    assert np.array_equal(product.kaiser_best_table().view(np.int64), w.view(np.int64))


def test_length_rule_and_too_short_error():
    for n in (1, 2):
        with pytest.raises(ValueError, match=f"Input signal length={n} is too small to resample from 48000->16000"):
            orr.resample(np.zeros(n, np.float32), 48000)
        with pytest.raises(ValueError, match="too small"):
            product.output_length(n, 48000)
    assert len(orr.resample(np.ones(3, np.float32), 48000)) == 1 == product.output_length(3, 48000)
    for n, sr in [(48000, 44100), (12345, 22050), (7, 11025), (1, 8000), (160000, 96000)]:
        assert product.output_length(n, sr) == int(n * 16000 / sr) == len(orr.resample(np.zeros(n, np.float32), sr))
    assert product.output_length(1234, 16000) == 1234 and product.output_length(0, 16000) == 0
    assert not product.needs_resampling(None) and not product.needs_resampling([16000, 16000])
    assert product.needs_resampling([16000, 8000])


@pytest.mark.parametrize("sr,n", [(48000, 3), (48000, 700), (8000, 300), (44100, 900), (22050, 500), (96000, 1500),
                                  (11025, 64)])
def test_vectorised_oracle_equals_literal_loop(sr, n):
    x = (np.random.default_rng(sr + n).standard_normal(n) * 0.3).astype(np.float32)
    assert np.array_equal(orr.resample(x, sr).view(np.int32), literal_resample(x, sr).view(np.int32))


def test_signal_properties():
    # upsampling 8 -> 16 kHz: a 1 kHz sine comes back to float32 accuracy away from the truncated ends
    y = orr.resample(sine(8000, 1000, 0.5), 8000)
    assert np.abs(y - sine(16000, 1000, 0.5)[:len(y)])[800:-800].max() < 2e-7
    # 48 -> 16 kHz: index_step = int(512 / 3) = 170 samples the filter slightly off its design spacing (resampy's own
    # behaviour), so the passband gain is off by ~3e-3
    y = orr.resample(sine(48000, 1000, 0.5), 48000)
    err = np.abs(y - sine(16000, 1000, 0.5)[:len(y)])[800:-800].max()
    assert 1e-3 < err < 2e-3
    # an 11 kHz tone is above the new Nyquist frequency: the filter removes it
    y = orr.resample(sine(48000, 11000, 0.5), 48000)
    assert np.abs(y[800:-800]).max() < 2e-4


@pytest.fixture(scope="module")
def golden():
    with open(os.path.join(GOLDEN, "predictor_golden_resample.json"), encoding="utf-8") as f:
        return json.load(f)


def _greedy(samples16, sd, cfg, vocab):
    feat = torch.from_numpy(ob.featurize(samples16.copy()))
    with torch.no_grad():
        probs = oc.get_encoder_out(sd, cfg, feat[None])[0].numpy()
    score, text, _ = octc.greedy_decode(probs, vocab)
    return text, score


def test_oracle_chain_reproduces_reference_golden(golden):
    sd = synth.to_torch(synth_weights(golden["wseed"]))
    cfg, vocab = oc.ConformerConfig(), synth.vocabulary()
    for case in golden["whole"]:
        x = synth.speechlike_audio(case["aseed"], case["samples"])
        text, score = _greedy(orr.resample(x, case["rate"]), sd, cfg, vocab)
        assert text == case["result"]["text"] and abs(score - case["result"]["score"]) < SCORE_TOL, case["rate"]
    lg = golden["long"]
    y = orr.resample(synth.speechlike_audio(lg["aseed"], lg["samples"]), lg["rate"])
    assert lg["vad_saw"] == [len(y), 16000]
    texts, scores = [], []
    for st in lg["stamps"]:
        text, score = _greedy(y[st["start"]:st["end"]], sd, cfg, vocab)
        if text:
            texts.append(text)
        scores.append(score)
    assert "，".join(texts) == lg["result"]["text"]
    assert abs(round(sum(scores) / len(scores), 2) - lg["result"]["score"]) <= 0.011
    # the streaming quirk: from the second push on, the 16 kHz remainder is resampled again with the new chunk
    s48 = golden["streams"][0]
    assert s48["rate"] == 48000 and s48["resample_calls"][1] == [24320, 48000, 16000]
