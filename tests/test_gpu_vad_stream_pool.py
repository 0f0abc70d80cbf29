"""H100: the slot-batched, resumable silero recurrence (``masr_silero_vad_recur_slots_f32``), the streaming VAD API of
``GpuSileroVAD`` and the ``SegmentingStreamPool`` built on them.

* the slots kernel with one slot and a zero state is the whole-recording kernel bit for bit, and a window's gate inputs
  do not depend on the encoder tile it lands in, so a stream pushed in ragged pieces gets the probabilities of one pass
  bit for bit (idle slots untouched, reset slots restart from zero);
* probabilities with carried states against the float64 interpreter fed the same h / c (``PROB_TOL`` as in
  test_gpu_silero_vad.py); ``__call__`` over [B, W] equals B independent streams; ``stream_vad`` events equal the
  restated state machine on the GPU's probabilities;
* the segmenting pool's boundaries equal the host rules replayed on the GPU probabilities, and each segment's result is
  a fresh ``predict_stream`` over the same pieces (the text exactly, greedy and beam with a character LM; the score
  within 1e-3, the bound StreamPool has against predict_stream);
  a long stream is force-cut at the derived capacity and never raises; one slot's malformed message fails that slot only.
"""
import os

import numpy as np
import pytest
import torch

from conftest import make_audio, synth_weights
from masr_b200 import synth, vad
from masr_b200.segment_pool import SegmentingStreamPool, SegmentPlanner, max_segment_samples
from masr_b200.stream_pool import StreamPool, StreamSlotError
from oracle import silero_vad as sv

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not os.path.exists(sv.MODEL_PATH),
                                 reason="oracle/_ref/silero_vad.onnx is fetched by build() from the reference tree")]

PROB_TOL = 1e-4
PUSH = 8000                                                    # 0.5 s pieces


@pytest.fixture(scope="module")
def vads():
    return {W: vad.GpuSileroVAD(sv.MODEL_PATH, device="cuda:0", window_size_samples=W) for W in (512, 1024, 1536)}


def _inputs():
    return {
        "silence": np.zeros(16000 * 2, np.float32),
        "noise": make_audio("noise", 21, 16000 * 3, 0.5),
        "speech": make_audio("speech", 22, 16000 * 4),
        "ragged": make_audio("speech", 23, 16000 * 3 + 1001),
    }


@pytest.mark.parametrize("W", [512, 1024, 1536])
def test_slots_kernel_with_one_zero_slot_is_the_whole_recording_kernel(vads, W):
    v = vads[W]
    for name, a in _inputs().items():
        gx = v.encode(a)
        n = gx.shape[0] // (W // 512)
        want = v.recur(gx)
        state = torch.zeros(1, 4, 64, device="cuda:0")
        got = v.recur_slots(gx, [0, n], state)
        assert torch.equal(got, want), name
        assert state.abs().sum() > 0


def test_slots_kernel_error_paths(vads):
    from masr_b200 import _lib
    w, gx, state = vads[512].weights["rec"], torch.zeros(8, 256, device="cuda:0"), torch.zeros(1, 4, 64, device="cuda:0")
    off, out = torch.tensor([0, 8], dtype=torch.int32, device="cuda:0"), torch.zeros(8, device="cuda:0")
    for off_p, n, W, msg in ((None, 1, 512, "null pointer"), (off.data_ptr(), 1, 768, "not one of 512, 1024, 1536"),
                             (off.data_ptr(), 0, 512, "n_slots")):
        with pytest.raises(_lib.MasrB200Error, match=msg):
            _lib.call("masr_silero_vad_recur_slots_f32", gx.data_ptr(), off_p, n, W, w.data_ptr(), state.data_ptr(),
                      out.data_ptr(), out.data_ptr(), None)
    assert not state.any()


@pytest.mark.parametrize("W", [512, 1536])
def test_gate_inputs_do_not_depend_on_the_tile(vads, W):
    v = vads[W]
    a = make_audio("speech", 40, W * 37)
    base = v.encode(a)
    T = W // 512
    for k in range(1, 7):                                      # shift the windows through every tile position
        pre = make_audio("noise", 41 + k, W * k)
        got = v.encode(np.concatenate([pre, a]))[k * T:]
        assert torch.equal(got, base), k


def _whole(v, a):
    W = v.kw["window_size_samples"]
    n = len(a) // W
    return v.recur(v.encode(a[:n * W])).cpu().numpy() if n else np.zeros(0, np.float32)


@pytest.mark.parametrize("S", [1, 7, 64, 200])
def test_ragged_pushes_equal_one_pass(vads, S):
    v = vads[512]
    rng = np.random.default_rng(S)
    lens = rng.integers(300, 16000 * 3, S)
    streams = [make_audio("speech" if i % 3 else "noise", 100 + i, int(n)) for i, n in enumerate(lens)]
    slots = v.slots(S)
    got = [[] for _ in range(S)]
    at = [0] * S
    while any(at[s] < lens[s] for s in range(S)):
        msg = {}
        for s in range(S):
            if at[s] >= lens[s] or rng.random() < 0.2:
                continue                                       # idle this push
            k = int(rng.choice([0, 100, 511, 512, 513, 3000, 9000]))
            msg[s] = streams[s][at[s]:at[s] + k]
            at[s] += k
        before = slots.state.clone()
        out = slots.advance(msg)
        moved = set()
        for s, p in out.items():
            got[s].append(p)
            if len(p):
                moved.add(s)
        for s in range(S):                                     # a slot without a complete window keeps its state bytes
            if s not in moved:
                assert torch.equal(slots.state[s].view(torch.int32), before[s].view(torch.int32)), s
    for s in range(S):
        g = np.concatenate(got[s]) if got[s] else np.zeros(0, np.float32)
        assert np.array_equal(g, _whole(v, streams[s])), s
    # a reset slot restarts from zero
    slots.reset(0)
    assert not slots.state[0].any() and len(slots.carry[0]) == 0
    assert np.array_equal(slots.advance({0: streams[0]})[0], _whole(v, streams[0]))


def test_carried_states_against_float64(vads):
    v = vads[512]
    graph = sv.load()
    streams = [make_audio("speech", 60 + i, 16000 * 2 + 333 * i) for i in range(3)]
    slots = v.slots(3)
    got = [[] for _ in range(3)]
    for lo in range(0, 16000 * 2 + 666, 5000):
        out = slots.advance({i: a[lo:lo + 5000] for i, a in enumerate(streams)})
        for i in range(3):
            got[i].append(out[i])
    for i, a in enumerate(streams):
        n = len(a) // 512
        want, _ = sv.speech_probs(graph, a[:n * 512])          # the interpreter carries h / c across windows
        g = np.concatenate(got[i])
        err = np.abs(g - want).max()
        print(f"stream {i}: {n} windows, max err {err:.3e}")
        assert g.shape == want.shape and err <= PROB_TOL


def test_call_rows_are_independent_streams_and_stream_vad_events(vads):
    v = vads[512]
    B, steps = 5, 40
    audio = [make_audio("speech" if i % 2 else "noise", 70 + i, 512 * steps) for i in range(B)]
    v.reset_states()
    batched = [v(np.stack([a[512 * t:512 * (t + 1)] for a in audio]), 16000) for t in range(steps)]
    assert batched[0].shape == (B, 1)
    singles = [vad.GpuSileroVAD(sv.MODEL_PATH, device="cuda:0") for _ in range(B)]
    for i, s in enumerate(singles):
        col = np.array([s(audio[i][512 * t:512 * (t + 1)], 16000)[0, 0] for t in range(steps)])
        assert np.array_equal(col, np.array([b[i, 0] for b in batched])), i
    # stream_vad over a speech / silence / speech stream: events equal the state machine on the GPU's probabilities
    a = np.concatenate([np.zeros(8000, np.float32), make_audio("speech", 80, 16000 * 2), np.zeros(16000, np.float32),
                        make_audio("speech", 81, 16000)])
    v.reset_states()
    events = [v.stream_vad(a[i:i + 512], 16000) for i in range(0, len(a) - 511, 512)]
    st, want = vad.StreamVADState(), []
    for i, p in enumerate(_whole(vads[512], a)):
        st.current_sample += 512 if i else 0                  # the reference's first call resets current_sample
        want.append(vad.stream_vad_step(st, float(p), 16000))
    assert events == want and any(e and "start" in e for e in events) and any(e and "end" in e for e in events)


# ---------------------------------------------------------------------------------------------------------------------
# the segmenting pool
def _predictor(tmp, use_model, lm_path=None):
    from masr_b200.predict import MASRPredictor
    sd = {"conformer": lambda: synth_weights(0), "deepspeech2": lambda: synth.deepspeech2_state_dict(0, streaming=True),
          "squeezeformer": lambda: synth.squeezeformer_state_dict(0, streaming=True),
          "efficient_conformer": lambda: synth.efficient_conformer_state_dict(0)}[use_model]()
    mp, vp = str(tmp / f"{use_model}.pt"), str(tmp / "vocabulary.txt")
    torch.save(synth.to_torch(sd), mp)
    synth.write_vocabulary(vp)
    cfg = {"use_model": use_model, "streaming": True, "decoder": "ctc_greedy" if lm_path is None else "ctc_beam_search",
           "preprocess_conf": {"feature_method": "fbank", "n_mels": 80, "sample_rate": 16000, "use_dB_normalization": True,
                               "target_dB": -20},
           "dataset_conf": {"dataset_vocab": vp},
           "ctc_beam_search_decoder_conf": {"alpha": 0.5, "beta": 2.0, "beam_size": 16, "cutoff_prob": 0.99, "cutoff_top_n": 40,
                                            "language_model_path": lm_path}}
    return MASRPredictor(configs=cfg, model_path=mp, use_gpu=True)


def _streams(n=8):
    """zeros / speech / zeros / speech / zeros per slot (synthetic speech), of different lengths."""
    z = lambda n: np.zeros(n, np.float32)
    return [np.concatenate([z(4000 + 1000 * i), make_audio("speech", 200 + i, 16000 * (2 + i % 3)), z(16000 + 2000 * (i % 3)),
                            make_audio("speech", 300 + i, 16000 * (1 + i % 2) + 777 * i), z(3000 * (i % 4))]) for i in range(n)]


def _drive(sp, streams, bad=None):
    """0.5 s pushes, each slot ending (is_end) with its last piece -> per slot the pushed sizes, the VAD probabilities and
    the closed segments, and per push the errors.  ``bad``: (push, slot) that gets a malformed PCM message instead."""
    S = len(streams)
    sizes, probs, segs, errs = [[] for _ in range(S)], [[] for _ in range(S)], [[] for _ in range(S)], []
    for k in range(max((len(a) + PUSH - 1) // PUSH for a in streams)):
        msg = {s: a[k * PUSH:(k + 1) * PUSH] for s, a in enumerate(streams) if k * PUSH < len(a)}
        ends = {s: (k + 1) * PUSH >= len(streams[s]) for s in msg}
        if bad is not None and bad[0] == k:
            msg[bad[1]] = b"\x01\x02\x03"
        out = sp.push(msg, is_end=ends, on_error="return")
        errs.append(dict(sp.last_errors))
        for s, r in out.items():
            sizes[s].append(len(msg[s]))
            probs[s].append(sp.last_probs[s])
            segs[s].extend(r["segments"])
            assert r["speech"] == (sp.planners[s].st.triggered and not ends[s])
    return sizes, probs, segs, errs


def _check_pool(pred, sp, streams, sizes, probs, segs):
    """Per slot: the host rules replayed on the GPU probabilities give the same segments, and each segment's result is
    a fresh predict_stream over exactly its pieces: the text exactly, the score within 1e-3 (the bound StreamPool has
    against predict_stream: its batched chunk GEMMs round differently from the one-stream ones)."""
    for s, a in enumerate(streams):
        pl, pieces = SegmentPlanner(sp.W, sp.max_samples, **{k: sp.vad.kw[k] for k in SegmentPlanner.OPTIONS}), []
        for i, p in enumerate(probs[s]):
            pieces += pl.windows(p) + (pl.finish(sum(sizes[s])) if i == len(probs[s]) - 1 else [])
        assert [(g["start"], g["end"]) for g in segs[s]] == pl.segments, s
        for g in segs[s]:
            pred.reset_stream()
            while True:
                lo, hi, end = pieces.pop(0)
                r = pred.predict_stream(a[lo:hi], is_end=end)
                if end:
                    break
            want = ("", 0.0) if r is None else (r["text"], r["score"])
            assert g["text"] == want[0] and abs(g["score"] - want[1]) < 1e-3, (s, g, want)
        scores = [g["score"] for g in segs[s]]
        assert sp.transcript(s) == {"text": "，".join(g["text"] for g in segs[s] if g["text"]),
                                    "score": round(sum(scores) / len(scores), 2) if scores else 0}
    pred.reset_stream()


@pytest.mark.parametrize("use_model, lm", [("conformer", False), ("deepspeech2", False), ("squeezeformer", False),
                                           ("efficient_conformer", False), ("conformer", True)])
def test_segmenting_pool_equals_predict_stream_per_segment(tmp_path, use_model, lm):
    lm_path = None
    if lm:                                                     # beam search with a character LM
        lm_path = str(tmp_path / "o3.arpa")
        synth.character_lm_arpa(lm_path, seed=3, order=3, n_chars=4200, n_sentences=600)
    pred = _predictor(tmp_path, use_model, lm_path)
    assert (pred.lm is not None) == lm
    sp = pred.create_stream_pool(8, vad_model_path=sv.MODEL_PATH)
    assert isinstance(sp, SegmentingStreamPool)
    streams = _streams()
    sizes, probs, segs, errs = _drive(sp, streams)
    assert not any(errs)
    assert all(len(x) >= 1 for x in segs) and sum(len(x) >= 2 for x in segs) >= 6, [len(x) for x in segs]
    _check_pool(pred, sp, streams, sizes, probs, segs)


def test_unbounded_stream_is_force_cut_and_never_raises(tmp_path):
    pred = _predictor(tmp_path, "conformer")
    sp = pred.create_stream_pool(2, max_frames=200, vad_model_path=sv.MODEL_PATH)
    cap = max_segment_samples(200)
    assert sp.max_samples == cap
    streams = [make_audio("speech", 90, 16000 * 30), make_audio("speech", 91, 16000 * 12)]   # continuous speech
    sizes, probs, segs, errs = _drive(sp, streams)
    assert not any(errs) and sum(g["end"] - g["start"] == cap for g in segs[0]) >= 3
    _check_pool(pred, sp, streams, sizes, probs, segs)
    # a 10-minute mixed stream runs to the end
    rng = np.random.default_rng(7)
    parts = []
    while sum(len(p) for p in parts) < 16000 * 600:
        n = int(rng.integers(16000, 16000 * 25))
        parts.append(np.zeros(n, np.float32) if rng.random() < 1 / 3 else make_audio("speech", int(rng.integers(1 << 30)), n))
    sp.reset_stream(0)
    _, _, segs, errs = _drive(sp, [np.concatenate(parts)[:16000 * 600]])
    assert not any(errs) and len(segs[0]) > 10 and all(g["end"] - g["start"] <= cap for g in segs[0])


def test_malformed_message_fails_only_its_slot_and_defaults_are_unchanged(tmp_path):
    pred = _predictor(tmp_path, "conformer")
    assert type(pred.create_stream_pool(3)) is StreamPool
    assert pred.create_stream_pool(1, vad_model_path=sv.MODEL_PATH, vad_options={"threshold": 0.6}).vad.threshold == 0.6
    streams = _streams(4)
    _, _, want, _ = _drive(pred.create_stream_pool(4, vad_model_path=sv.MODEL_PATH), streams)
    sp = pred.create_stream_pool(4, vad_model_path=sv.MODEL_PATH)
    _, _, got, errs = _drive(sp, streams, bad=(3, 2))
    assert set(errs[3]) == {2} and not any(e for i, e in enumerate(errs) if i != 3)
    assert [got[s] for s in (0, 1, 3)] == [want[s] for s in (0, 1, 3)]
    with pytest.raises(StreamSlotError) as e:
        sp.push({0: streams[0][:PUSH], 1: b"\x01"})
    assert set(e.value.errors) == {1} and 0 in e.value.results
    with pytest.raises(StreamSlotError):
        sp.push({0: streams[0][:PUSH]}, sample_rate=8000)
