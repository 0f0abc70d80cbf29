"""H100: the silero VAD kernels (csrc/vad.cu) against the float64 interpreter of the model's own graph
(oracle/silero_vad.py), stage by stage and end to end, and ``predict_long`` with the model file against the same
recognition driven by the interpreter's probabilities.

Tolerances (fp32 kernels against float64; the largest errors measured on an H100 in brackets):
* layer-1 gate inputs: every stage before them is a short fp32 dot product (256-tap STFT, at most 516 terms in the
  first 1x1 convs) on values of order 1-10, and the gate inputs reach |x| ~ 40; fp32 rounding of ~1e-6 relative per
  stage over about ten stages gives ~1e-5, so |err| <= 2e-4 * (1 + |ref|) [3.3e-5];
* recurrence from identical gate inputs: 64- and 128-term fp32 dot products per gate and a contracting LSTM (|f| < 1)
  keep the state error near fp32 rounding, and the sigmoid of the decoder has slope <= 1/4: 2e-6 per window [1.3e-7];
* end to end: the gate-input error passes through the recurrence, which damps it, so 1e-4 per window [1.3e-6 on a few
  seconds, 1.1e-5 over 18,750 recurrent steps, with no growth from the first tenth of the recording to the last].
"""
import ctypes
import os

import numpy as np
import pytest
import torch

from conftest import make_audio
from masr_b200 import _lib, vad
from oracle import silero_vad as sv

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not os.path.exists(sv.MODEL_PATH),
                                 reason="oracle/_ref/silero_vad.onnx is fetched by build() from the reference tree")]

GATE_TOL, REC_TOL, PROB_TOL = 2e-4, 2e-6, 1e-4
PERM = np.concatenate([np.arange(64) + 64 * k for k in (0, 2, 3, 1)])     # ONNX i, o, f, c -> kernel i, f, g, o


@pytest.fixture(scope="module")
def graph():
    return sv.load()


@pytest.fixture(scope="module")
def vads():
    return {W: vad.GpuSileroVAD(sv.MODEL_PATH, device="cuda:0", window_size_samples=W) for W in (512, 1024, 1536)}


def _inputs():
    return {
        "silence": np.zeros(16000 * 2, np.float32),
        "noise": make_audio("noise", 21, 16000 * 3, 0.5),
        "speech": make_audio("speech", 22, 16000 * 4),
        "ragged": make_audio("speech", 23, 16000 * 3 + 1001),     # not a multiple of any window size
    }


@pytest.mark.parametrize("W", [512, 1024, 1536])
def test_encoder_matches_the_interpreter_gate_inputs(graph, vads, W):
    (W1, _, b1), _ = sv.lstm_weights(graph)
    for name, a in _inputs().items():
        _, kept = sv.speech_probs(graph, a, window=W, keep=(sv.LSTM_INPUT,))
        want = np.concatenate([k[sv.LSTM_INPUT][:, 0] @ W1.T + b1 for k in kept])[:, PERM]
        got = vads[W].encode(a).cpu().numpy().astype(np.float64)
        assert got.shape == want.shape == (len(kept) * (W // 512), 256)
        err = np.abs(got - want) / (1.0 + np.abs(want))
        print(f"encoder W={W} {name}: max scaled err {err.max():.3e}, max |ref| {np.abs(want).max():.2f}")
        assert err.max() <= GATE_TOL, (name, err.max())


@pytest.mark.parametrize("W", [512, 1536])
def test_recurrence_matches_float64(graph, vads, W):
    v = vads[W]
    a = make_audio("speech", 31, 16000 * 20 + 77)
    gx = v.encode(a)
    got = v.recur(gx).cpu().numpy()
    # lstm_f64 reads gates in ONNX order: undo the kernel's permutation on the kernel's own gate inputs
    gx64 = gx.cpu().numpy().astype(np.float64)[:, np.argsort(PERM)]
    want = sv.lstm_f64(gx64, sv.lstm_weights(graph), W // 512, graph.inits["model.decoder.decoder.1.weight"].reshape(64),
                       float(graph.inits["model.decoder.decoder.1.bias"][0]))
    err = np.abs(got - want).max()
    print(f"recurrence W={W}: {len(gx)} steps, max err {err:.3e}")
    assert got.shape == want.shape and err <= REC_TOL


@pytest.mark.parametrize("W", [512, 1024, 1536])
def test_window_probabilities_match_the_interpreter(graph, vads, W):
    for name, a in _inputs().items():
        want, _ = sv.speech_probs(graph, a, window=W)
        got = np.array(vads[W].window_probs(a, 16000))
        err = np.abs(got - want).max()
        print(f"probs W={W} {name}: {len(want)} windows, max err {err:.3e}, range [{want.min():.3f}, {want.max():.3f}]")
        assert got.shape == want.shape and err <= PROB_TOL, (name, err)


def test_ten_minute_recording_stays_within_tolerance(graph, vads):
    """18,750 recurrent steps (6,250 windows of 1536 samples): the fp32 state does not drift from float64."""
    rng = np.random.default_rng(5)
    parts = []
    while sum(len(p) for p in parts) < 16000 * 600:
        kind = "speech" if rng.random() < 0.6 else "noise"
        parts.append(make_audio(kind, int(rng.integers(1 << 30)), int(rng.integers(16000, 16000 * 8)),
                                float(rng.uniform(0.05, 1.0))))
    a = np.concatenate(parts)[:16000 * 600]
    want, _ = sv.speech_probs(graph, a, window=1536)
    got = np.array(vads[1536].window_probs(a, 16000))
    err = np.abs(got - want)
    first, last = err[:len(err) // 10].max(), err[-len(err) // 10:].max()
    print(f"10 min W=1536: {len(want)} windows, max err {err.max():.3e} (first tenth {first:.3e}, last tenth {last:.3e})")
    assert len(want) * 3 >= 18000 and err.max() <= PROB_TOL


def _composite():
    parts = [make_audio("speech", 500 + i, n) for i, n in enumerate((16000 * 6, 16000 * 9 + 300, 16000 * 4))]
    gap = (np.random.default_rng(0).standard_normal(16000 * 3) * 1e-4).astype(np.float32)
    return np.concatenate([gap, parts[0], gap, parts[1], gap, parts[2], gap])


def test_timestamps_equal_the_state_machine_on_oracle_probs(graph, vads):
    a = _composite()
    want_p, _ = sv.speech_probs(graph, a)
    # the comparison is exact only when no probability sits within the kernels' tolerance of a threshold
    assert np.min(np.minimum(np.abs(want_p - 0.5), np.abs(want_p - 0.35))) > PROB_TOL
    want = vad.speech_timestamps_from_probs(list(want_p), len(a), 16000)
    assert len(want) == 3
    assert vads[512].get_speech_timestamps(a, 16000) == want
    # a multiple of 16 kHz is decimated first, as the reference's _validate_input does
    a48 = np.repeat(a, 3)
    assert vads[512].get_speech_timestamps(a48, 48000) == vad.speech_timestamps_from_probs(list(want_p), len(a48), 48000)


def test_predict_long_with_the_model_file_equals_oracle_probabilities(tmp_path, graph):
    from conftest import synth_weights
    from masr_b200 import synth
    from masr_b200.predict import MASRPredictor
    mp, vp = str(tmp_path / "m.pt"), str(tmp_path / "vocabulary.txt")
    torch.save(synth.to_torch(synth_weights(0)), mp)
    synth.write_vocabulary(vp)
    cfg = {"use_model": "conformer", "streaming": True, "decoder": "ctc_greedy",
           "preprocess_conf": {"feature_method": "fbank", "n_mels": 80, "sample_rate": 16000, "use_dB_normalization": True, "target_dB": -20},
           "dataset_conf": {"dataset_vocab": vp}}
    a = _composite()
    probs, _ = sv.speech_probs(graph, a)
    pred = MASRPredictor(configs=cfg, model_path=mp, use_gpu=True)
    got = pred.predict_long(a, vad_model_path=sv.MODEL_PATH)
    assert isinstance(pred.vad_predictor, vad.GpuSileroVAD)
    want = pred.predict_long(a, vad_predictor=vad.ProbabilityVAD(lambda x, sr: probs))
    assert got == want and want["text"] != ""


def test_sample_rates_and_windows(vads):
    with pytest.raises(ValueError, match="16 kHz"):
        vads[512].get_speech_timestamps(np.zeros(8000, np.float32), 8000)
    with pytest.raises(ValueError, match="Supported sampling rates"):
        vads[512].get_speech_timestamps(np.zeros(8000, np.float32), 22050)
    with pytest.raises(ValueError, match="512, 1024 or 1536"):
        vad.GpuSileroVAD(sv.MODEL_PATH, window_size_samples=768)
    assert vads[512].get_speech_timestamps(np.zeros(0, np.float32), 16000) == []


def test_kernel_error_paths(vads):
    v = vads[512]
    w = v.weights
    x = torch.zeros(4096, device="cuda:0")
    gx = torch.zeros(8, 256, device="cuda:0")
    out = torch.zeros(8, device="cuda:0")
    enc = lambda *a: _lib.call("masr_silero_vad_encode_f32", *a)
    rec = lambda *a: _lib.call("masr_silero_vad_recur_f32", *a)
    with pytest.raises(_lib.MasrB200Error, match="null pointer"):
        enc(None, 4096, 512, w["basis"].data_ptr(), w["enc"].data_ptr(), gx.data_ptr(), None)
    with pytest.raises(_lib.MasrB200Error, match="not one of 512, 1024, 1536"):
        enc(x.data_ptr(), 4096, 256, w["basis"].data_ptr(), w["enc"].data_ptr(), gx.data_ptr(), None)
    with pytest.raises(_lib.MasrB200Error, match="empty"):
        enc(x.data_ptr(), 0, 512, w["basis"].data_ptr(), w["enc"].data_ptr(), gx.data_ptr(), None)
    with pytest.raises(_lib.MasrB200Error, match="null pointer"):
        rec(gx.data_ptr(), 8, 512, None, out.data_ptr(), out.data_ptr(), None)
    with pytest.raises(_lib.MasrB200Error, match="not one of 512, 1024, 1536"):
        rec(gx.data_ptr(), 8, 2048, w["rec"].data_ptr(), out.data_ptr(), out.data_ptr(), None)
    with pytest.raises(_lib.MasrB200Error, match="empty"):
        rec(gx.data_ptr(), 0, 512, w["rec"].data_ptr(), out.data_ptr(), out.data_ptr(), None)
    with pytest.raises(_lib.MasrB200Error, match="null pointer"):
        _lib.call("masr_silero_vad_layout", None)
    sizes = (ctypes.c_int64 * 4)()
    _lib.call("masr_silero_vad_layout", sizes)
    assert sizes[3] == 256
    torch.cuda.synchronize()
