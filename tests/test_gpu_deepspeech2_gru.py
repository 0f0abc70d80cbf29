"""GPU (-m gpu): DeepSpeech2 with GRU recurrences (``encoder_conf.use_gru: True``) end to end: the engine against the reference's
frozen outputs and the oracle (whole utterance, uni and bi; chunk walks under both recurrence forms), the stream pool against
the single stream bit for bit, and ``MASRPredictor`` / ``StreamPool`` against ``predict_stream`` and the frozen reference
pushes (tests/golden/make_deepspeech2_gru_golden.py)."""
import json
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN, load_npz, make_audio
from masr_b200 import synth
from masr_b200.engine import subsampled_len
from masr_b200.text import ids_to_text
from oracle import beam as obeam, ctc as octc, deepspeech2 as od, deepspeech2_gru as og, fbank as ob, lm as olm
from test_gpu_deepspeech2_stream_pool import ALPHA, BETA, _compare, _reference, _streams
from test_gpu_stream_pool_beam import _Recorder, _drive

pytestmark = pytest.mark.gpu
V = synth.DEFAULT_VOCAB_SIZE
_W = {}


def weights(seed, streaming):
    if (seed, streaming) not in _W:
        _W[seed, streaming] = synth.deepspeech2_state_dict(seed, streaming=streaming, use_gru=True)
    return _W[seed, streaming]


@pytest.fixture(scope="module")
def engines():
    from masr_b200.deepspeech2 import DeepSpeech2Engine
    cache = {}

    def get(streaming):
        if streaming not in cache:
            cache[streaming] = DeepSpeech2Engine(weights(1 - int(streaming), streaming), streaming=streaming)
        return cache[streaming]
    return get


@pytest.mark.parametrize("streaming", [True, False])
def test_engine_matches_golden_and_oracle(engines, streaming):
    eng = engines(streaming)
    assert eng.w.cell == "gru" and eng.G == 3
    z, meta = load_npz("deepspeech2_gru_golden.npz")
    vocab = synth.vocabulary()
    m, = [m for m in meta if not m.get("chunks") and m["streaming"] == streaming]
    assert m["wseed"] == 1 - int(streaming)
    feat = z[m["name"] + "/feat"]
    res = eng.transcribe_features(torch.from_numpy(feat)[None].to(eng.device), [feat.shape[0]], None, return_frames=True)
    assert np.array_equal(res.frame_ids[0, :res.frame_lens[0]], z[m["name"] + "/ids"])
    assert ids_to_text(res.tokens[0], vocab) == m["text"]
    assert abs(res.scores[0] - m["score"]) < 1e-3
    probs = eng.posteriors(feat[None], [feat.shape[0]])[0]
    got = np.take_along_axis(probs, z[m["name"] + "/top_i"].astype(np.int64), axis=1)
    assert np.abs(got - z[m["name"] + "/top_p"]).max() < 5e-5
    # a ragged batch against the oracle
    sd = synth.to_torch(weights(m["wseed"], streaming))
    cfg = od.DS2Config(bidirectional=not streaming)
    lens = [16000 * 2 + 17, 9000, 16000 + 320, 400 + 160 * 30]
    waves = [make_audio("speech" if i % 2 == 0 else "noise", 190 + i, n) for i, n in enumerate(lens)]
    res = eng.transcribe(waves, return_frames=True)
    for i, w in enumerate(waves):
        with torch.no_grad():
            probs, _ = og.get_encoder_out(sd, cfg, torch.from_numpy(ob.featurize(w.copy()))[None])
        probs = probs.numpy()
        n = res.frame_lens[i]
        assert n == probs.shape[0]
        assert np.array_equal(probs.argmax(1), res.frame_ids[i, :n]), i
        score, _, toks = octc.greedy_decode(probs, vocab)
        assert toks == res.tokens[i] and abs(score - res.scores[i]) < 1e-3


@pytest.mark.parametrize("persistent", [True, False])
def test_encode_chunk_walk_matches_golden(engines, persistent):
    """``encode_chunk`` over the frozen 67-frame window walk (ending in a short window) against the reference's per-window
    top-8 posteriors, frame ids and h state; a GRU stream carries no c."""
    eng = engines(True)
    z, meta = load_npz("deepspeech2_gru_golden.npz")
    m, = [m for m in meta if m.get("chunks")]
    assert m["wseed"] == 0
    fd = torch.from_numpy(z[m["name"] + "/feat"]).to(eng.device)
    top_p, top_i, want_ids, want_h = (z[m["name"] + k] for k in ("/top_p", "/top_i", "/ids", "/h"))
    saved = eng.persistent_lstm
    eng.persistent_lstm = persistent
    try:
        st, row = eng.new_stream(), 0
        assert st.c is None
        for k, (cur, n) in enumerate(z[m["name"] + "/windows"]):
            ids, maxp, probs = eng.encode_chunk(fd[cur:cur + n], st, want_probs=True)
            t = probs.shape[0]
            rows = slice(row, row + t)
            row += t
            assert t == subsampled_len(int(n))
            got = np.take_along_axis(probs.cpu().numpy(), top_i[rows].astype(np.int64), axis=1)
            assert np.abs(got - top_p[rows]).max() < 5e-5, k
            assert np.array_equal(ids.cpu().numpy(), want_ids[rows]), k
            h = torch.stack([st.hT[l, st.cur[l], 0, :, 0] for l in range(5)]).cpu().numpy()
            assert np.abs(h - want_h[k]).max() < 2e-4, k
        assert row == want_ids.shape[0]
    finally:
        eng.persistent_lstm = saved


# ---------------------------------------------------------------------------------------------------------------------
S = 40                                                     # two lane groups: slots 32..39 live in the second
ROUNDS = [{0: 67, 32: 67, 39: 67}, {0: 67, 31: 67, 32: 40}, {0: 67, 31: 67, 32: 67, 39: 67}, {0: 67, 31: 50, 32: 67, 39: 67}]


def _bits(t):
    return t.contiguous().view(torch.int32)


@pytest.mark.parametrize("persistent", [True, False])
def test_pool_step_equals_single_stream_and_oracle(engines, persistent):
    """Every slot of a ``DeepSpeech2StreamPool`` over a GRU model equals ``encode_chunk`` on its own stream bit for bit, with
    the step replayed from a CUDA graph; idle slots keep their h lanes byte for byte; ``reset`` starts a slot afresh."""
    from masr_b200.stream_pool import DeepSpeech2StreamPool
    eng = engines(True)
    sd = synth.to_torch(weights(0, True))
    dev, cfg = eng.device, od.DS2Config()
    saved = eng.persistent_lstm
    eng.persistent_lstm = persistent
    try:
        pool = DeepSpeech2StreamPool(eng, S, keep_probs=True)
        assert pool.state.c is None
        slots = sorted({s for r in ROUNDS for s in r})
        feats = {s: torch.from_numpy(ob.featurize(make_audio("speech" if s % 2 == 0 else "noise", 800 + s, 16000 * 4)))
                 for s in slots + [5]}
        pos = {s: 0 for s in feats}
        single = {s: eng.new_stream() for s in feats}
        ost = {s: None for s in feats}

        def lane(s):
            st = pool.state
            return [_bits(st.hT[l, st.cur[l], s // 32, :, s % 32]).clone() for l in range(5)]

        def run(rnd):
            batch = torch.zeros(S, 67, 80, device=dev)
            nfr = [0] * S
            chunks = {}
            for s, n in rnd.items():
                chunks[s] = feats[s][pos[s]:pos[s] + n]
                pos[s] += 64
                batch[s, :n] = chunks[s].to(dev)
                nfr[s] = n
            idle = {s: lane(s) for s in feats if s not in rnd}
            ids, maxp, tout = pool.step(batch, nfr)
            torch.cuda.synchronize()
            assert pool.state.cur == [0] * 5
            for s, before in idle.items():
                assert all(torch.equal(a, b) for a, b in zip(before, lane(s))), s
            logits, probs = pool.b["logits"], pool.probs
            for s, ch in chunks.items():
                t = tout[s]
                assert t == subsampled_len(ch.shape[0]) and t > 0
                rows = slice(s * 16, s * 16 + t)
                sid, smp, _ = eng.encode_chunk(ch.to(dev), single[s])
                assert torch.equal(ids[s, :t], sid) and torch.equal(_bits(maxp[s, :t]), _bits(smp)), s
                assert torch.equal(_bits(logits[rows, :V]), _bits(single[s].last_logits[:, :V])), s
                assert all(torch.equal(a, b) for a, b in zip(lane(s), [_bits(single[s].hT[l, single[s].cur[l], 0, :, 0])
                                                                       for l in range(5)])), s
                with torch.no_grad():
                    pm, ost[s] = og.get_encoder_out(sd, cfg, ch[None], ost[s])
                pm = pm.numpy()
                assert np.array_equal(ids[s, :t].cpu().numpy(), pm.argmax(1)), s
                assert np.abs(probs[rows].cpu().numpy() - pm).max() < 5e-5

        for rnd in ROUNDS:
            run(rnd)
        assert pool._graph is not None and pool._graph_launches == (20 if persistent else 95)
        pool.reset(0)
        single[0], ost[0], pos[0] = eng.new_stream(), None, 128
        run({0: 67, 31: 67})
    finally:
        eng.persistent_lstm = saved


# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def char_lm3(tmp_path_factory):
    from masr_b200.lm import CharLM
    p = str(tmp_path_factory.mktemp("lm") / "o3.arpa")
    synth.character_lm_arpa(p, seed=3, order=3, n_chars=4200, n_sentences=600)
    return olm.read_arpa(p), CharLM(p, synth.vocabulary(V)), p


@pytest.fixture(scope="module")
def predictors(tmp_path_factory):
    """MASRPredictor over a GRU checkpoint (a plain state dict: the cell type comes from the weights), one per (streaming,
    decoder, LM path)."""
    from masr_b200.predict import MASRPredictor
    tmp = tmp_path_factory.mktemp("ds2gru")
    vp = str(tmp / "vocabulary.txt")
    synth.write_vocabulary(vp)
    cache = {}

    def get(streaming=True, decoder="ctc_greedy", lm_path="lm/none.klm"):
        key = (streaming, decoder, lm_path)
        if key not in cache:
            mp = str(tmp / f"ds2gru_{int(streaming)}.pt")
            if not os.path.exists(mp):
                torch.save(synth.to_torch(weights(1 - int(streaming), streaming)), mp)
            cfg = {"use_model": "deepspeech2", "streaming": streaming, "decoder": decoder,
                   "encoder_conf": {"num_rnn_layers": 5, "rnn_size": 1024, "use_gru": False},   # not read at inference
                   "preprocess_conf": {"feature_method": "fbank", "n_mels": 80, "sample_rate": 16000, "use_dB_normalization": True,
                                       "target_dB": -20},
                   "dataset_conf": {"dataset_vocab": vp},
                   "ctc_beam_search_decoder_conf": {"alpha": ALPHA, "beta": BETA, "beam_size": 16, "cutoff_prob": 0.99,
                                                    "cutoff_top_n": 40, "language_model_path": lm_path}}
            cache[key] = MASRPredictor(configs=cfg, model_path=mp, use_gpu=True)
        return cache[key]
    return get


def test_predictor_matches_reference_golden_and_oracle(predictors):
    """``predict`` and ``predict_stream`` against the reference predictor's frozen outputs; ``predict_batch`` and
    ``predict_batches`` against ``predict`` and the oracle, for the streaming and the bidirectional checkpoint."""
    with open(os.path.join(GOLDEN, "predictor_golden_deepspeech2_gru.json"), encoding="utf-8") as f:
        g = json.load(f)
    assert g["wseed"] == 0
    pred = predictors(True)
    assert pred.predictor.w.cell == "gru"
    x = make_audio(g["kind"], g["aseed"], g["samples"])
    whole = pred.predict(audio_data=x.copy())
    assert whole["text"] == g["whole"]["text"] and abs(whole["score"] - g["whole"]["score"]) < 1e-3
    pcm = (np.clip(x, -1, 1) * 32767).astype("<i2")
    push = g["push"]
    pred.reset_stream()
    got = [pred.predict_stream(audio_data=pcm[s:s + push].tobytes(), is_end=s + push >= len(pcm)) for s in range(0, len(pcm), push)]
    pred.reset_stream()
    assert len(got) == len(g["pushes_pcm"])
    for r, w in zip(got, g["pushes_pcm"]):
        assert (r is None) == (w is None), (r, w)
        if r is not None:
            assert r["text"] == w["text"] and abs(r["score"] - w["score"]) < 1e-3, (r, w)
    vocab = synth.vocabulary()
    waves = [make_audio("speech", 290 + i, n) for i, n in enumerate((16000 * 2 + 500, 12000, 16000 * 3))]
    for streaming in (True, False):
        p = predictors(streaming)
        cfg = od.DS2Config(bidirectional=not streaming)
        sd = synth.to_torch(weights(1 - int(streaming), streaming))
        batch = p.predict_batch([w.copy() for w in waves])
        piped = list(p.predict_batches([[w.copy() for w in waves[:2]], [waves[2].copy()]]))
        for w, b, q in zip(waves, batch, piped[0] + piped[1]):
            with torch.no_grad():
                probs = og.get_encoder_out(sd, cfg, torch.from_numpy(ob.featurize(w.copy()))[None])[0].numpy()
            score, text, _ = octc.greedy_decode(probs, vocab)
            one = p.predict(audio_data=w.copy())
            for r in (b, q, one):
                assert r["text"] == text and abs(r["score"] - score) < 1e-3, (streaming, r, text, score)


def test_greedy_pool_equals_predict_stream_and_reference(predictors):
    from masr_b200.stream_pool import DeepSpeech2StreamPool, StreamPool
    pred = predictors(True)
    streams, schedule = _streams()
    want = _reference(pred, streams)
    with open(os.path.join(GOLDEN, "predictor_golden_deepspeech2_gru.json"), encoding="utf-8") as f:
        g = json.load(f)
    pcm = (np.clip(make_audio(g["kind"], g["aseed"], g["samples"]), -1, 1) * 32767).astype("<i2")
    sp = pred.create_stream_pool(4, max_frames=20)
    assert sp.beam is None and isinstance(sp.pool, DeepSpeech2StreamPool) and sp.pool.use_graph
    assert _drive(sp, streams, schedule) == want
    gold = [sp.push({3: pcm[s:s + g["push"]].tobytes()}, is_end=s + g["push"] >= len(pcm))[3] for s in range(0, len(pcm), g["push"])]
    assert len(gold) == len(g["pushes_pcm"])
    for r, w in zip(gold, g["pushes_pcm"]):
        assert (r is None) == (w is None) and (r is None or (r["text"] == w["text"] and abs(r["score"] - w["score"]) < 1e-3))
    eager = StreamPool(pred.predictor, synth.vocabulary(), n_slots=4, use_graph=False, max_frames=20)
    assert _drive(eager, streams, schedule) == want


@pytest.mark.parametrize("with_lm", [False, True])
def test_beam_pool_equals_predict_stream(predictors, char_lm3, with_lm):
    olm3, _, path = char_lm3
    pred = predictors(True, "ctc_beam_search", path if with_lm else "lm/none.klm")
    assert (pred.lm is not None) == with_lm
    streams, schedule = _streams()
    want = _reference(pred, streams)
    sp = pred.create_stream_pool(4, max_frames=400)
    rec = _Recorder(sp)
    vocab = synth.vocabulary()

    def check(s, r):                                         # bit for bit against the restatement on the pool's own candidates
        c = rec.cands[s]
        if with_lm:
            (score, approx, toks), = olm.prefix_beam_search_lm(np.zeros((len(c), 1)), olm3, vocab, ALPHA, BETA, beam_size=16,
                                                              cands_per_frame=c, blank_logp_per_frame=rec.blp[s])
            score = approx
        else:
            (score, toks), = obeam.prefix_beam_search(np.zeros((len(c), 1)), beam_size=16, cands_per_frame=c)
        assert r["text"] == ids_to_text(toks, vocab) and np.float32(r["score"]) == np.float32(score), (s, r, score)
    _compare(_drive(sp, streams, schedule, check), want, nonempty=False)
