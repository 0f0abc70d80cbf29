"""GPU (-m gpu): hotwords through MASRPredictor on a synthetic Conformer — predict, predict_batch and predict_long with a
per-call list against oracle/hotwords.py on the candidates the GPU searched, ``hotwords=[]`` byte-identical to no
argument, predict_stream with the predictor's list, and create_stream_pool slots with the default list, none and their
own list (kept across a reset), each against the oracle on the pool's own candidates and against predict_stream of a
predictor built with that list."""
import numpy as np
import pytest
import torch

from masr_b200.text import ids_to_text
from oracle import hotwords as oh

pytestmark = pytest.mark.gpu
F = np.float32
BEAM = 64


def make_predictor(tmp, hotwords=None, decoder="ctc_beam_search"):
    from conftest import synth_weights
    from masr_b200 import synth
    from masr_b200.predict import MASRPredictor
    mp, vp = str(tmp / "m.pt"), str(tmp / "vocabulary.txt")
    torch.save(synth.to_torch(synth_weights(0)), mp)
    synth.write_vocabulary(vp)
    cfg = {"use_model": "conformer", "streaming": True, "decoder": decoder,
           "preprocess_conf": {"feature_method": "fbank", "n_mels": 80, "sample_rate": 16000, "use_dB_normalization": True,
                               "target_dB": -20},
           "dataset_conf": {"dataset_vocab": vp},
           "ctc_beam_search_decoder_conf": {"beam_size": BEAM, "cutoff_prob": 0.99, "cutoff_top_n": 40,
                                            "language_model_path": ""}}
    return MASRPredictor(configs=cfg, model_path=mp, use_gpu=True, hotwords=hotwords)


class _Stamps:
    def __init__(self, stamps):
        self.stamps = stamps

    def get_speech_timestamps(self, samples, sr):
        return [dict(s) for s in self.stamps]


def restate(eng, b, H):
    """The oracle search of row b of the last one-shot search, on the candidates the GPU searched."""
    ws, T, B = eng._last_beam
    T_b = int(ws["tlens"][b].item())
    cands = eng.last_beam_candidates()[b][:T_b]
    (score, _, toks), = oh.prefix_beam_search_hot(None, None, None, beam_size=BEAM, cands_per_frame=cands, hotwords=H)
    return toks, F(score)


def hotwords_from(eng, vocab):
    """Two-token runs of tokens the model puts among its candidates (so the credit competes inside the beam)."""
    seen = [c for fr in eng.last_beam_candidates()[0] for c, _ in fr if c not in (0, 1) and vocab[c] != "<space>"]
    uniq = list(dict.fromkeys(seen))
    return [vocab[uniq[i]] + vocab[uniq[i + 1]] for i in range(0, min(len(uniq) - 1, 12), 2)] + [vocab[uniq[0]]]


def test_predictor_hotwords_equal_oracle(tmp_path):
    from conftest import make_audio
    from masr_b200 import synth
    vocab = synth.vocabulary()
    pred = make_predictor(tmp_path)
    eng = pred.predictor
    x1, x2 = make_audio("speech", 81, 16000 * 2), make_audio("speech", 82, 16000 * 3)
    plain = pred.predict(audio_data=x1.copy())
    assert pred.predict(audio_data=x1.copy(), hotwords=[]) == plain              # [] is the path without hotwords
    hws = hotwords_from(eng, vocab)
    g = pred._graph(hws)
    H = oh.HotwordMatcher(g.tokens, 1.5)
    one = pred.predict(audio_data=x1.copy(), hotwords=hws)
    toks, score = restate(eng, 0, H)
    assert one["text"] == ids_to_text(toks, vocab) and F(one["score"]) == score
    batch = pred.predict_batch([x1.copy(), x2.copy()], hotwords=hws)
    for b in range(2):
        toks, score = restate(eng, b, H)
        assert batch[b]["text"] == ids_to_text(toks, vocab) and F(batch[b]["score"]) == score
    assert batch[0] == one
    assert pred.predict_batch([x1.copy(), x2.copy()], hotwords=[]) == pred.predict_batch([x1.copy(), x2.copy()])
    rec = np.concatenate([x1, np.zeros(8000, np.float32), x2])
    stamps = [{"start": 0, "end": len(x1)}, {"start": len(x1) + 8000, "end": len(rec)}]
    long = pred.predict_long(rec.copy(), vad_predictor=_Stamps(stamps), hotwords=hws)
    texts, scores = [], []
    for b in range(2):
        toks, score = restate(eng, b, H)
        texts.append(ids_to_text(toks, vocab))
        scores.append(float(score))
    assert long["text"] == "，".join(t for t in texts if t) and long["score"] == round(sum(scores) / 2, 2)
    assert pred.predict_long(rec.copy(), vad_predictor=_Stamps(stamps), hotwords=[]) == \
        pred.predict_long(rec.copy(), vad_predictor=_Stamps(stamps))
    with pytest.raises(ValueError, match="not in the vocabulary"):
        pred.predict(audio_data=x1.copy(), hotwords=["a"])


def stream(pred_or_pool, pcm, slot=None):
    """predict_stream (or one pool slot) over pcm in 0.5 s pushes -> every non-None result."""
    out = []
    for s in range(0, len(pcm), 8000):
        chunk, end = pcm[s:s + 8000].tobytes(), s + 8000 >= len(pcm)
        r = pred_or_pool.predict_stream(audio_data=chunk, is_end=end) if slot is None else \
            pred_or_pool.push({slot: chunk}, is_end=end)[slot]
        if r is not None:
            out.append(r)
    return out


def test_stream_pool_slots_with_their_own_lists(tmp_path):
    """Each slot against the oracle bit for bit on the pool's own candidates, and against predict_stream of a predictor
    built with the slot's list (same text, score within 1e-3: the pool's batched encoder rounds differently, as without
    hotwords)."""
    from conftest import make_audio
    from masr_b200 import synth
    from test_gpu_stream_pool_beam import _Recorder
    vocab = synth.vocabulary()
    plain = make_predictor(tmp_path)
    x = make_audio("speech", 83, 16000 * 3)
    plain.predict(audio_data=x.copy())
    hws = hotwords_from(plain.predictor, vocab)
    hA, hB = hws[:3], hws[3:]
    predA, predB = make_predictor(tmp_path, hA), make_predictor(tmp_path, hB)
    H = {"A": oh.HotwordMatcher(predA._hotwords.tokens, 1.5), "B": oh.HotwordMatcher(predB._hotwords.tokens, 1.5),
         "none": None}
    pcm = (np.clip(x, -1, 1) * 32767).astype("<i2")
    want = {}
    for key, p in (("A", predA), ("B", predB), ("none", plain)):
        p.reset_stream()
        want[key] = stream(p, pcm)
    assert want["A"] != want["none"] or want["B"] != want["none"], "the hotwords changed no result"
    pool = predA.create_stream_pool(3, max_frames=400, max_hotword_nodes=64)
    rec = _Recorder(pool)
    pool.set_hotwords(1, [])
    pool.set_hotwords(2, hB)

    def check(s, key):
        got = []
        for i in range(0, len(pcm), 8000):                   # after every push: the oracle on the candidates so far
            r = pool.push({s: pcm[i:i + 8000].tobytes()}, is_end=i + 8000 >= len(pcm))[s]
            if r is None:
                continue
            (score, _, toks), = oh.prefix_beam_search_hot(None, None, None, beam_size=BEAM, cands_per_frame=rec.cands[s],
                                                          hotwords=H[key])
            assert r["text"] == ids_to_text(toks, vocab) and F(r["score"]) == F(score), (s, key, i)
            got.append(r)
        assert len(got) == len(want[key]), (s, key)
        for r, w in zip(got, want[key]):
            assert r["text"] == w["text"] and abs(r["score"] - w["score"]) < 1e-3, (s, key, r, w)

    for s, key in ((0, "A"), (1, "none"), (2, "B")):
        check(s, key)
    with pytest.raises(ValueError, match="since its reset"):
        pool.set_hotwords(2, hA)
    for s in range(3):                                       # the lists stay with the slots across resets
        pool.reset_stream(s)
    for s, key in ((0, "A"), (1, "none"), (2, "B")):
        check(s, key)
    pool.reset_stream(2)
    pool.set_hotwords(2, None)                               # back to the pool default
    check(2, "A")
    pool.reset_stream(0)
    with pytest.raises(ValueError, match="max_hotword_nodes"):
        pool.set_hotwords(0, ["".join(vocab[2 + 30 * i:32 + 30 * i]) for i in range(3)])    # 91 nodes > 64
    with pytest.raises(ValueError, match="without hotwords"):
        plain.create_stream_pool(2, max_frames=400).set_hotwords(0, hA)


def test_hotwords_with_greedy_decoding_are_refused(tmp_path):
    with pytest.raises(ValueError, match="ctc_greedy"):
        make_predictor(tmp_path, ["一丁"], decoder="ctc_greedy")
    greedy = make_predictor(tmp_path, decoder="ctc_greedy")
    from conftest import make_audio
    x = make_audio("speech", 84, 16000)
    assert greedy.predict(audio_data=x.copy(), hotwords=[]) == greedy.predict(audio_data=x.copy())
    with pytest.raises(ValueError, match="ctc_greedy"):
        greedy.predict(audio_data=x.copy(), hotwords=["一丁"])
