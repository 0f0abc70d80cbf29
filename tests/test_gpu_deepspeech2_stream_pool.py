"""GPU (-m gpu): many live DeepSpeech2 streams in one pool (``DeepSpeech2StreamPool`` behind ``StreamPool``).

Every stage of the pool's chunk step computes a row or lane independently of the batch, so each slot must equal the
single-stream path (``encode_chunk`` on a ``DeepSpeech2Stream``, what ``predict_stream`` runs) bit for bit, under both LSTM
forms and with the step replayed as a CUDA graph; the oracle pins the ids and posteriors.  Greedy and beam-search
``StreamPool``s equal ``predict_stream`` push by push, the beam also the CPU restatement on the pool's own candidates."""
import json
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN, make_audio
from masr_b200 import synth
from masr_b200.engine import subsampled_len
from masr_b200.text import ids_to_text
from oracle import beam as obeam, deepspeech2 as od, fbank as ob, lm as olm
from test_gpu_stream_pool_beam import _Recorder, _drive

pytestmark = pytest.mark.gpu
V = synth.DEFAULT_VOCAB_SIZE
PUSH = 8000
ALPHA, BETA = 0.5, 2.0


@pytest.fixture(scope="module")
def ds2():
    from masr_b200.deepspeech2 import DeepSpeech2Engine
    sdn = synth.deepspeech2_state_dict(0, streaming=True)
    return DeepSpeech2Engine(sdn, streaming=True), synth.to_torch(sdn)


@pytest.fixture(scope="module")
def char_lm3(tmp_path_factory):
    """A 3-gram character LM over nearly the whole synthetic vocabulary (the synthetic model emits arbitrary characters)."""
    from masr_b200.lm import CharLM
    p = str(tmp_path_factory.mktemp("lm") / "o3.arpa")
    synth.character_lm_arpa(p, seed=3, order=3, n_chars=4200, n_sentences=600)
    return olm.read_arpa(p), CharLM(p, synth.vocabulary(V)), p


@pytest.fixture(scope="module")
def predictors(tmp_path_factory):
    """MASRPredictor over a streaming deepspeech2 YAML, one per (decoder, LM path), built on first use."""
    from masr_b200.predict import MASRPredictor
    tmp = tmp_path_factory.mktemp("ds2")
    mp, vp = str(tmp / "deepspeech2.pt"), str(tmp / "vocabulary.txt")
    torch.save(synth.to_torch(synth.deepspeech2_state_dict(0, streaming=True)), mp)
    synth.write_vocabulary(vp)
    cache = {}

    def get(decoder="ctc_greedy", lm_path="lm/none.klm"):
        if (decoder, lm_path) not in cache:
            cfg = {"use_model": "deepspeech2", "streaming": True, "decoder": decoder,
                   "preprocess_conf": {"feature_method": "fbank", "n_mels": 80, "sample_rate": 16000, "use_dB_normalization": True,
                                       "target_dB": -20},
                   "dataset_conf": {"dataset_vocab": vp},
                   "ctc_beam_search_decoder_conf": {"alpha": ALPHA, "beta": BETA, "beam_size": 16, "cutoff_prob": 0.99,
                                                    "cutoff_top_n": 40, "language_model_path": lm_path}}
            cache[decoder, lm_path] = MASRPredictor(configs=cfg, model_path=mp, use_gpu=True)
        return cache[decoder, lm_path]
    return get


# ---------------------------------------------------------------------------------------------------------------------
# the pool step against the oracle and the single stream
S = 40                                                     # two lane groups: slots 32..39 live in the second
# slot -> feature frames of its chunk this round.  Slot 31 joins in round 1; slot 32 ends round 1 with a short chunk and
# takes another in round 2 (no reset); slot 39 idles in round 1; slot 5 is never used.
ROUNDS = [{0: 67, 32: 67, 39: 67}, {0: 67, 31: 67, 32: 40}, {0: 67, 31: 67, 32: 67, 39: 67}, {0: 67, 31: 50, 32: 67, 39: 67}]


def _bits(t):
    return t.contiguous().view(torch.int32)


@pytest.mark.parametrize("persistent", [True, False])
def test_pool_step_equals_single_stream_and_oracle(ds2, persistent):
    from masr_b200.stream_pool import DeepSpeech2StreamPool
    eng, sd = ds2
    dev, cfg = eng.device, od.DS2Config()
    saved = eng.persistent_lstm
    eng.persistent_lstm = persistent
    try:
        pool = DeepSpeech2StreamPool(eng, S, keep_probs=True)
        slots = sorted({s for r in ROUNDS for s in r})
        feats = {s: torch.from_numpy(ob.featurize(make_audio("speech" if s % 2 == 0 else "noise", 700 + s, 16000 * 4)))
                 for s in slots + [5]}
        pos = {s: 0 for s in feats}
        single = {s: eng.new_stream() for s in feats}
        ost = {s: None for s in feats}

        def lane(s):
            st = pool.state
            return [_bits(st.hT[l, st.cur[l], s // 32, :, s % 32]).clone() for l in range(5)] + [_bits(st.c[:, s]).clone()]

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
            assert pool.state.cur == [0] * 5                 # the state is back in the buffer the graph reads next round
            for s, before in idle.items():                   # idle (and never used) slots: h lane and c row byte for byte
                assert all(torch.equal(a, b) for a, b in zip(before, lane(s))), s
            logits, probs = pool.b["logits"], pool.probs
            for s, ch in chunks.items():
                t = tout[s]
                assert t == subsampled_len(ch.shape[0]) and t > 0
                rows = slice(s * 16, s * 16 + t)
                sid, smp, _ = eng.encode_chunk(ch.to(dev), single[s])
                assert torch.equal(ids[s, :t], sid) and torch.equal(_bits(maxp[s, :t]), _bits(smp)), s
                assert torch.equal(_bits(logits[rows, :V]), _bits(single[s].last_logits[:, :V])), s
                with torch.no_grad():
                    pm, ost[s] = od.get_encoder_out(sd, cfg, ch[None], ost[s])
                pm = pm.numpy()
                assert np.array_equal(ids[s, :t].cpu().numpy(), pm.argmax(1)), s
                assert np.abs(maxp[s, :t].cpu().numpy() - pm.max(1)).max() < 5e-5
                assert np.abs(probs[rows].cpu().numpy() - pm).max() < 5e-5

        for rnd in ROUNDS:
            run(rnd)
        assert pool._graph is not None and pool._graph_launches == (20 if persistent else 95)
        # reset: slot 0 starts again from a zero state, like a fresh stream
        pool.reset(0)
        single[0], ost[0], pos[0] = eng.new_stream(), None, 128
        run({0: 67, 31: 67})
    finally:
        eng.persistent_lstm = saved


def test_make_pool_rejects_a_bidirectional_model():
    from masr_b200.deepspeech2 import DeepSpeech2Engine
    from masr_b200.stream_pool import make_pool
    eng = DeepSpeech2Engine(synth.deepspeech2_state_dict(1, streaming=False), streaming=False)
    with pytest.raises(Exception, match="chunk decoding needs a streaming"):
        make_pool(eng, 2)


# ---------------------------------------------------------------------------------------------------------------------
# StreamPool against predict_stream
def _streams():
    """Four streams as lists of (PCM bytes, is_end) pushes, and a schedule of rounds (slot -> stream): stream 1 is silent in
    round 2, slot 2 is reset after stream 2 ends and reused for stream 3, slot 3 stays idle throughout."""
    lens = [6 * PUSH - 1234, 5 * PUSH - 3000, 3 * PUSH - 500, 3 * PUSH]
    kinds = ["speech", "speech", "noise", "speech"]
    out = []
    for i, (n, k) in enumerate(zip(lens, kinds)):
        pcm = (np.clip(make_audio(k, 300 + i, n), -1, 1) * 32767).astype("<i2")
        starts = list(range(0, n, PUSH))
        out.append([(pcm[s:s + PUSH].tobytes(), j == len(starts) - 1) for j, s in enumerate(starts)])
    schedule = [{0: 0, 1: 1, 2: 2}, {0: 0, 1: 1, 2: 2}, {0: 0, 2: 2}, {0: 0, 1: 1, 2: 3}, {0: 0, 1: 1, 2: 3}, {0: 0, 1: 1, 2: 3}]
    return out, schedule


def _reference(pred, streams):
    want = []
    for pieces in streams:
        pred.reset_stream()
        want.append([pred.predict_stream(audio_data=b, is_end=e) for b, e in pieces])
    pred.reset_stream()
    return want


def _compare(got, want, nonempty=True):
    """Beam results push by push: same text, score within 1e-3 (as the other pools' beam tests compare)."""
    for i, (g, w) in enumerate(zip(got, want)):
        assert len(g) == len(w)
        for r, x in zip(g, w):
            assert (r is None) == (x is None), (i, r, x)
            if r is not None:
                assert r["text"] == x["text"] and abs(r["score"] - x["score"]) < 1e-3, (i, r, x)
    assert not nonempty or any(r is not None and r["text"] for g in got for r in g)


def test_greedy_pool_equals_predict_stream_past_max_frames(predictors):
    from masr_b200.stream_pool import StreamPool
    pred = predictors()
    streams, schedule = _streams()
    want = _reference(pred, streams)
    with open(os.path.join(GOLDEN, "predictor_golden_deepspeech2.json"), encoding="utf-8") as f:
        g = json.load(f)
    pcm = (np.clip(make_audio(g["kind"], g["aseed"], g["samples"]), -1, 1) * 32767).astype("<i2")
    results = {}
    for use_graph in (True, False):
        # max_frames = 20 encoder frames (0.8 s): it bounds nothing without a beam search
        sp = StreamPool(pred.predictor, synth.vocabulary(), n_slots=4, use_graph=use_graph, max_frames=20)
        got = _drive(sp, streams, schedule)
        assert got == want                                    # text and score identical, push by push
        # the reference's frozen pushes, in the slot that idled so far
        gold = [sp.push({3: pcm[s:s + g["push"]].tobytes()}, is_end=s + g["push"] >= len(pcm))[3] for s in range(0, len(pcm), g["push"])]
        assert sp.pool.lens_host[3] > 20
        assert len(gold) == len(g["pushes_pcm"])
        for r, w in zip(gold, g["pushes_pcm"]):
            assert (r is None) == (w is None) and (r is None or (r["text"] == w["text"] and abs(r["score"] - w["score"]) < 1e-3))
        results[use_graph] = (got, gold)
    assert results[True] == results[False]                    # CUDA graph replay == eager launches


@pytest.mark.parametrize("with_lm", [False, True])
def test_beam_pool_equals_predict_stream_and_restatement(predictors, char_lm3, with_lm):
    from masr_b200.stream_pool import StreamPool
    olm3, _, path = char_lm3
    pred = predictors("ctc_beam_search", path if with_lm else "lm/none.klm")
    assert (pred.lm is not None) == with_lm and pred._beam_conf["beam_size"] == 16
    streams, schedule = _streams()
    want = _reference(pred, streams)
    sp = StreamPool(pred.predictor, synth.vocabulary(), n_slots=4, beam=pred._beam_conf, max_frames=400)
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
    _compare(_drive(sp, streams, schedule, check), want)


def test_beam_pool_bounds_a_slot_by_max_frames(predictors):
    """With a beam search, max_frames sizes each slot's prefix trie: a slot that would exceed it fails alone (its state kept),
    the other slot keeps decoding as predict_stream does."""
    from masr_b200.stream_pool import StreamPool, StreamSlotError
    pred = predictors("ctc_beam_search")
    pcm = [(np.clip(make_audio("speech", 400 + i, n), -1, 1) * 32767).astype("<i2") for i, n in enumerate((7 * PUSH, 20000))]
    pieces = [[(p[s:s + PUSH].tobytes(), s + PUSH >= len(p)) for s in range(0, len(p), PUSH)] for p in pcm]
    pieces[0] = [(b, False) for b, _ in pieces[0]]           # stream 0 never ends: it outgrows 40 frames (1.6 s)
    want = _reference(pred, pieces)
    sp = StreamPool(pred.predictor, synth.vocabulary(), n_slots=2, beam=pred._beam_conf, max_frames=40)
    failed = []
    for k in range(len(pieces[0])):
        msgs = {i: pieces[i][k] for i in range(2) if k < len(pieces[i])}
        for is_end in (False, True):
            grp = {i: b for i, (b, e) in msgs.items() if e == is_end}
            if not grp:
                continue
            try:
                out, errors = sp.push(grp, is_end=is_end), {}
            except StreamSlotError as e:
                out, errors = e.results, e.errors
            assert set(errors) <= {0}
            if 0 in errors:
                assert isinstance(errors[0], AssertionError) and "max_len: 40" in str(errors[0])
                failed.append(k)
            for i in grp:
                if i not in errors:
                    _compare([[out[i]]], [[want[i][k]]], nonempty=False)
    assert failed and failed == list(range(failed[0], len(pieces[0])))
    assert sp.pool.lens_host[0] <= 40
    sp.reset_stream(0)                                         # a reset slot decodes again
    _compare([[sp.push({0: b}, is_end=e)[0] for b, e in pieces[1]]], [want[1]], nonempty=False)


def test_create_stream_pool_and_sessions_follow_the_yaml(predictors, char_lm3):
    from masr_b200.serve import StreamSessions
    from masr_b200.stream_pool import DeepSpeech2StreamPool
    greedy = predictors().create_stream_pool(2, max_frames=400)
    assert greedy.beam is None and isinstance(greedy.pool, DeepSpeech2StreamPool)
    pred = predictors("ctc_beam_search", char_lm3[2])
    sp = pred.create_stream_pool(3, max_frames=400)
    assert isinstance(sp.pool, DeepSpeech2StreamPool) and sp.beam is not None and sp.beam.lm is pred.lm and sp.beam.beam == 16
    streams, _ = _streams()
    want = _reference(pred, streams[:2])
    sess = StreamSessions(sp)
    ids = [sess.open(), sess.open()]
    text = [None, None]
    for k in range(max(len(s) for s in streams[:2])):
        msgs = {}
        for i in range(2):
            if k < len(streams[i]):
                b, e = streams[i][k]
                msgs[ids[i]] = b + (b"end" if e else b"")
        replies = sess.feed(msgs)
        for i in range(2):
            if k < len(streams[i]):
                if want[i][k] is not None:
                    text[i] = want[i][k]["text"]
                assert replies[ids[i]] == {"code": 0, "result": text[i] or ""}, (i, k)
    assert any(text)
