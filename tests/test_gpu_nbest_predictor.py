"""GPU (-m gpu): ``n_best`` through MASRPredictor for Conformer, Squeezeformer, EfficientConformer and DeepSpeech2 —
``predict`` / ``predict_batch`` against oracle/beam.py's ``nbest=`` on the candidates the GPU searched (texts and float32
scores bit for bit), ``predict_stream`` after every push against the oracle over the frames seen so far, stream-pool
slots (with and without the VAD segmenting pool) against the oracle on the pool's own candidates and entry 0 against
their results; results without ``n_best`` equal those of a call that never asked for it."""
import os

import numpy as np
import pytest
import torch

from masr_b200.text import ids_to_text
from oracle import hotwords as oh

pytestmark = pytest.mark.gpu
F = np.float32
BEAM = 16
FAMILIES = ["conformer", "squeezeformer", "efficient_conformer", "deepspeech2"]


def _predictor(tmp, use_model, lm_path=""):
    from conftest import synth_weights
    from masr_b200 import synth
    from masr_b200.predict import MASRPredictor
    sd = {"conformer": lambda: synth_weights(0), "deepspeech2": lambda: synth.deepspeech2_state_dict(0, streaming=True),
          "squeezeformer": lambda: synth.squeezeformer_state_dict(0, streaming=True),
          "efficient_conformer": lambda: synth.efficient_conformer_state_dict(0)}[use_model]()
    mp, vp = str(tmp / f"{use_model}.pt"), str(tmp / "vocabulary.txt")
    torch.save(synth.to_torch(sd), mp)
    synth.write_vocabulary(vp)
    cfg = {"use_model": use_model, "streaming": True, "decoder": "ctc_beam_search",
           "preprocess_conf": {"feature_method": "fbank", "n_mels": 80, "sample_rate": 16000, "use_dB_normalization": True,
                               "target_dB": -20},
           "dataset_conf": {"dataset_vocab": vp},
           "ctc_beam_search_decoder_conf": {"alpha": 0.5, "beta": 2.0, "beam_size": BEAM, "cutoff_prob": 0.99,
                                            "cutoff_top_n": 40, "language_model_path": lm_path}}
    return MASRPredictor(configs=cfg, model_path=mp, use_gpu=True)


def _oracle(cands, n, vocab):
    res = oh.prefix_beam_search_hot(None, None, None, beam_size=BEAM, cands_per_frame=cands, nbest=n)
    return [{"text": ids_to_text(t, vocab), "score": F(s)} for s, _, t in res]


def _f32(entries):
    return [{"text": e["text"], "score": F(e["score"])} for e in entries]


def _check_result(r, n):
    assert 1 <= len(r["n_best"]) <= n
    assert r["n_best"][0] == {"text": r["text"], "score": r["score"]}


@pytest.mark.parametrize("use_model", FAMILIES)
def test_predict_and_batch_n_best(tmp_path, use_model):
    from conftest import make_audio
    from masr_b200 import synth
    vocab = synth.vocabulary()
    pred = _predictor(tmp_path, use_model)
    eng = pred.predictor
    x1, x2 = make_audio("speech", 91, 16000 * 2), make_audio("speech", 92, 16000 * 3)
    plain = pred.predict(audio_data=x1.copy())
    plain_b = pred.predict_batch([x1.copy(), x2.copy()])
    for n in (1, 5, BEAM):
        one = pred.predict(audio_data=x1.copy(), n_best=n)
        _check_result(one, n)
        assert {k: one[k] for k in ("text", "score")} == plain
        if n > 1:
            assert _f32(one["n_best"]) == _oracle(eng.last_beam_candidates()[0], n, vocab)
    assert len(one["n_best"]) > 1
    batch = pred.predict_batch([x1.copy(), x2.copy()], n_best=5)
    ws, T, B = eng._last_beam
    for b in range(2):
        _check_result(batch[b], 5)
        assert {k: batch[b][k] for k in ("text", "score")} == plain_b[b]
        T_b = int(ws["tlens"][b].item())
        assert _f32(batch[b]["n_best"]) == _oracle(eng.last_beam_candidates()[b][:T_b], 5, vocab), b
    # without n_best: the one-shot path again, results unchanged
    assert pred.predict(audio_data=x1.copy()) == plain and pred.predict_batch([x1.copy(), x2.copy()]) == plain_b
    silent = pred.predict(audio_data=np.zeros(800, np.float32), n_best=3)          # no encoder frames
    assert silent["n_best"] == [{"text": silent["text"], "score": silent["score"]}]


def test_predict_n_best_with_char_lm(tmp_path):
    """With a character LM: entry 0 is the result (approx_ctc), the list is at most n long, results without n_best are
    unchanged (the oracle comparison with an LM is made at kernel level, tests/test_gpu_nbest.py)."""
    from conftest import make_audio
    from masr_b200 import synth
    lm_path = str(tmp_path / "o3.arpa")
    synth.character_lm_arpa(lm_path, seed=3, order=3, n_chars=4200, n_sentences=600)
    pred = _predictor(tmp_path, "conformer", lm_path)
    assert pred.lm is not None
    x = make_audio("speech", 93, 16000 * 2)
    plain = pred.predict(audio_data=x.copy())
    r = pred.predict(audio_data=x.copy(), n_best=8)
    _check_result(r, 8)
    assert {k: r[k] for k in ("text", "score")} == plain and pred.predict(audio_data=x.copy()) == plain


class _StreamRecorder:
    """Every candidate row the predictor's StreamBeam searched since the last reset."""

    def __init__(self, monkeypatch):
        from masr_b200.engine import StreamBeam
        self.cands = []
        orig = StreamBeam.push
        rec = self

        def push(sb, logits, rows, n_best=None):
            out = orig(sb, logits, rows, n_best)
            ids, lp, n = sb.cand_id.cpu().numpy(), sb.cand_lp.cpu().numpy(), sb.cand_n.cpu().numpy()
            rec.cands += [[(int(ids[t, k]), lp[t, k]) for k in range(n[t])] for t in range(rows)]
            return out

        monkeypatch.setattr(StreamBeam, "push", push)


@pytest.mark.parametrize("use_model", FAMILIES)
def test_predict_stream_and_pool_n_best(tmp_path, monkeypatch, use_model):
    from conftest import make_audio
    from masr_b200 import synth
    from test_gpu_stream_pool_beam import _Recorder
    vocab = synth.vocabulary()
    pred = _predictor(tmp_path, use_model)
    rec = _StreamRecorder(monkeypatch)
    pcm = (np.clip(make_audio("speech", 94, 16000 * 3), -1, 1) * 32767).astype("<i2")
    pushes = [(pcm[i:i + 8000].tobytes(), i + 8000 >= len(pcm)) for i in range(0, len(pcm), 8000)]
    pred.reset_stream()
    plain = [pred.predict_stream(audio_data=b, is_end=e) for b, e in pushes]
    pred.reset_stream()
    rec.cands = []
    want, seen = [], 0
    for (b, e), p in zip(pushes, plain):
        r = pred.predict_stream(audio_data=b, is_end=e, n_best=4)
        assert (r is None) == (p is None)
        if r is None:
            continue
        _check_result(r, 4)
        assert {k: r[k] for k in ("text", "score")} == p
        assert _f32(r["n_best"]) == _oracle(rec.cands, 4, vocab)
        want.append(r)
        seen += 1
    assert seen and any(len(r["n_best"]) > 1 for r in want)
    pred.reset_stream()
    # the stream pool: slot 1 carries the stream, slot 0 stays idle, slot 2 gets a different one
    pool = pred.create_stream_pool(3, max_frames=400, n_best=4)
    prec = _Recorder(pool)
    other = (np.clip(make_audio("speech", 95, 16000 * 2), -1, 1) * 32767).astype("<i2")
    got = []
    for k, (b, e) in enumerate(pushes):
        msg = {1: b}
        if k * 8000 < len(other):
            msg[2] = other[k * 8000:(k + 1) * 8000].tobytes()
        out = pool.push(msg, is_end=e)
        for s, r in out.items():
            if r is None:
                continue
            _check_result(r, 4)
            assert _f32(r["n_best"]) == _oracle(prec.cands[s], 4, vocab), (k, s)
        if out[1] is not None:
            got.append(out[1])
    assert len(got) == len(want)
    for r, w in zip(got, want):                                  # the pool's batched encoder rounds differently
        assert r["text"] == w["text"] and abs(r["score"] - w["score"]) < 1e-3
    plain_pool = pred.create_stream_pool(1, max_frames=400)
    r = [plain_pool.push({0: b}, is_end=e)[0] for b, e in pushes]
    assert all(x is None or "n_best" not in x for x in r)


def test_segmenting_pool_carries_n_best(tmp_path):
    from conftest import make_audio
    from oracle import silero_vad as sv
    if not os.path.exists(sv.MODEL_PATH):
        pytest.skip("oracle/_ref/silero_vad.onnx is fetched by build() from the reference tree")
    pred = _predictor(tmp_path, "conformer")
    z = np.zeros(8000, np.float32)
    a = np.concatenate([z, make_audio("speech", 96, 16000 * 2), np.zeros(20000, np.float32),
                        make_audio("speech", 97, 16000 * 2), z])
    sp = pred.create_stream_pool(2, vad_model_path=sv.MODEL_PATH, n_best=3)
    plain = pred.create_stream_pool(2, vad_model_path=sv.MODEL_PATH)
    segs, partials, segs_p = [], [], []
    for i in range(0, len(a), 8000):
        end = i + 8000 >= len(a)
        r = sp.push({0: a[i:i + 8000]}, is_end=end)[0]
        rp = plain.push({0: a[i:i + 8000]}, is_end=end)[0]
        segs += r["segments"]
        segs_p += rp["segments"]
        if r["partial"] is not None:
            partials.append(r["partial"])
            assert "n_best" not in (rp["partial"] or {})
    assert segs and partials
    for g in segs + partials:
        _check_result(g, 3)
    assert [{k: g[k] for k in ("start", "end", "text", "score")} for g in segs] == segs_p
