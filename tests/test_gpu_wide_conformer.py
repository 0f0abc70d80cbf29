"""GPU (-m gpu): the wide Conformer (``output_size: 512``, ``attention_heads: 8``) end to end — the batched engine, the
drop-in predictor, streaming (greedy and beam), the stream pool and CUDA-graph replay — against the reference's frozen
outputs (tests/golden/conformer_wide_golden.npz, predictor_golden_wide.json) and the CPU oracle.  Tolerances are those of
tests/test_gpu_parity.py for the 256-wide model."""
import json
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN, load_npz, make_audio
from masr_b200 import synth
from masr_b200.text import ids_to_text
from oracle import beam as obeam, conformer as oc, ctc as octc, fbank as ob
from test_gpu_parity import ENC_TOL, PROB_TOL, SCORE_TOL
from test_wide_conformer import wide_config, wide_weights

pytestmark = pytest.mark.gpu
PUSH = 8000


@pytest.fixture(scope="module")
def engines():
    cache = {}

    def get(seed=0, streaming=True, **kw):
        from masr_b200.engine import ConformerEngine
        key = (seed, streaming, tuple(sorted(kw.items())))
        if key not in cache:
            cache[key] = ConformerEngine(wide_weights(seed), streaming=streaming, **kw)
            assert (cache[key].d, cache[key].h, cache[key].dk) == (512, 8, 64)
        return cache[key]

    return get


@pytest.fixture(scope="module")
def golden():
    with open(os.path.join(GOLDEN, "predictor_golden_wide.json"), encoding="utf-8") as f:
        return json.load(f)


def _predictor(tmp, decoder="ctc_greedy", sd=None, use_model="conformer"):
    from masr_b200.predict import MASRPredictor
    mp, vp = str(tmp / f"{use_model}_{decoder}.pt"), str(tmp / "vocabulary.txt")
    torch.save(synth.to_torch(wide_weights(0) if sd is None else sd), mp)
    synth.write_vocabulary(vp)
    cfg = {"use_model": use_model, "streaming": True, "decoder": decoder,
           "preprocess_conf": {"feature_method": "fbank", "n_mels": 80, "sample_rate": 16000, "use_dB_normalization": True,
                               "target_dB": -20},
           "dataset_conf": {"dataset_vocab": vp},
           "ctc_beam_search_decoder_conf": {"alpha": 0.5, "beta": 2.0, "beam_size": 16, "cutoff_prob": 0.99, "cutoff_top_n": 40,
                                            "language_model_path": "lm/none.klm"}}
    return MASRPredictor(configs=cfg, model_path=mp, use_gpu=True)


@pytest.fixture(scope="module")
def predictor(tmp_path_factory):
    return _predictor(tmp_path_factory.mktemp("wide"))


def _same(result, want):
    if want is None:
        return result is None
    return result is not None and result["text"] == want["text"] and abs(result["score"] - want["score"]) < SCORE_TOL


def _pushes(pcm):
    starts = list(range(0, len(pcm), PUSH))
    return [(pcm[s:s + PUSH].tobytes(), j == len(starts) - 1) for j, s in enumerate(starts)]


def test_encoder_golden(engines):
    z, meta = load_npz("conformer_wide_golden.npz")
    vocab = synth.vocabulary()
    assert {m["streaming"] for m in meta} == {True, False}
    for m in meta:
        eng = engines(m["wseed"], m["streaming"])
        assert not eng._ffn_fused()                       # the fused FFN kernel is built for d = 256
        feat = z[m["name"] + "/feat"]
        fd = torch.from_numpy(feat)[None].to(eng.device)
        enc, tl, T, ws = eng.encode(fd, [feat.shape[0]])
        assert enc.shape[1] == 512
        assert np.abs(enc.cpu().numpy() - z[m["name"] + "/enc"]).max() < ENC_TOL
        res = eng.transcribe_features(fd, [feat.shape[0]], None, return_frames=True)
        assert np.array_equal(res.frame_ids[0, :tl[0]], z[m["name"] + "/ids"])            # bit-exact ids
        assert ids_to_text(res.tokens[0], vocab) == m["text"]
        assert abs(res.scores[0] - m["score"]) < SCORE_TOL
        probs = eng.posteriors(feat[None], [feat.shape[0]])[0]
        got = np.take_along_axis(probs, z[m["name"] + "/top_i"].astype(np.int64), axis=1)
        assert np.abs(got - z[m["name"] + "/top_p"]).max() < PROB_TOL


def _oracle_rows(waves, seed, streaming):
    sd, cfg, vocab = synth.to_torch(wide_weights(seed)), wide_config(streaming), synth.vocabulary()
    out = []
    for w in waves:
        f = torch.from_numpy(ob.featurize(w.copy()))
        with torch.no_grad():
            probs = oc.get_encoder_out(sd, cfg, f[None])[0].numpy()
        out.append((octc.best_path(probs)[0],) + octc.greedy_decode(probs, vocab))
    return out


@pytest.mark.parametrize("streaming,wseed", [(True, 0), (False, 1)])
def test_ragged_batch_equals_single_utterance_oracle(engines, streaming, wseed):
    """Every row of a padded batch is computed as if it were alone; one row is shorter than one 16-frame chunk."""
    eng = engines(wseed, streaming)
    lens = [16000 * 3 + 17, 9000, 16000 * 2, 400 + 160 * 6, 16000 * 4]
    waves = [make_audio("speech" if i % 2 == 0 else "noise", 40 + i, n) for i, n in enumerate(lens)]
    res = eng.transcribe(waves, return_frames=True)
    for i, (ids, score, _, toks) in enumerate(_oracle_rows(waves, wseed, streaming)):
        n = res.frame_lens[i]
        assert n == len(ids) and np.array_equal(ids, res.frame_ids[i, :n]), i
        assert toks == res.tokens[i] and abs(score - res.scores[i]) < SCORE_TOL


def test_long_utterance_uses_both_attention_kernels(engines):
    """11 s (T = 274 > 256 frames) runs the mma.sync flash attention, 3 s the wgmma kernel, both with 8 heads."""
    eng = engines(0, True)
    waves = [make_audio("speech", 70, 16000 * 11), make_audio("speech", 71, 16000 * 3)]
    rows = _oracle_rows(waves, 0, True)
    for w, (ids, score, _, toks) in zip(waves, rows):
        res = eng.transcribe([w], return_frames=True)
        assert (res.frame_lens[0] > 256) == (len(w) > 16000 * 10)
        assert np.array_equal(ids, res.frame_ids[0, :res.frame_lens[0]])
        assert toks == res.tokens[0] and abs(score - res.scores[0]) < SCORE_TOL


def test_cuda_graph_replay_equals_eager(engines):
    waves = [synth.noise_audio(210 + i, 48000 + 1000 * i) for i in range(4)]
    graph, eager = engines(0, True), engines(0, True, use_graphs=False)
    want = eager.transcribe(waves, return_frames=True)
    for _ in range(3):                                    # capture, then replays
        got = graph.transcribe(waves, return_frames=True)
        assert got.tokens == want.tokens and got.scores == want.scores
        assert np.array_equal(got.frame_lens, want.frame_lens)
        for i, n in enumerate(want.frame_lens):           # (the replayed step pads the batch to its captured shape)
            assert np.array_equal(got.frame_ids[i, :n], want.frame_ids[i, :n])


def test_predictor_dropin(predictor, golden):
    g = golden
    x = make_audio(g["kind"], g["aseed"], g["samples"])
    assert _same(predictor.predict(audio_data=x.copy()), g["whole"])
    out = predictor.predict_batch([x.copy(), x[:20000].copy()])
    assert _same(out[0], g["whole"])
    outs = list(predictor.predict_batches([[x.copy()], [x[:20000].copy(), x.copy()]]))
    assert _same(outs[0][0], g["whole"]) and _same(outs[1][1], g["whole"]) and outs[1][0] == out[1]
    pcm = (np.clip(x, -1, 1) * 32767).astype("<i2")
    for rep in range(2):                                  # twice: reset_stream must restore a clean state
        predictor.reset_stream()
        got = [predictor.predict_stream(audio_data=b, is_end=e) for b, e in _pushes(pcm)]
        assert len(got) == len(g["pushes_pcm"])
        for r, w in zip(got, g["pushes_pcm"]):
            assert _same(r, w), (rep, r, w)
    predictor.reset_stream()


def test_streaming_beam_equals_one_shot_and_restatement(tmp_path):
    """``decoder: ctc_beam_search``: the whole-utterance search equals the CPU restatement on the engine's own candidates bit
    for bit; the streaming search returns a transcript after the last push and repeats itself after ``reset_stream`` (the
    pool test below compares it push by push with the pool's search)."""
    pred = _predictor(tmp_path, "ctc_beam_search")
    eng, vocab = pred.predictor, synth.vocabulary()
    x = make_audio("speech", 77, 16000 * 3 + 2000)
    whole = pred.predict(audio_data=x.copy())
    from masr_b200.engine import num_frames, subsampled_len
    cands = eng.last_beam_candidates()[0][:subsampled_len(num_frames(len(x)))]
    (score, toks), = obeam.prefix_beam_search(np.zeros((len(cands), 1)), beam_size=16, cands_per_frame=cands)
    assert whole["text"] == ids_to_text(toks, vocab) and np.float32(whole["score"]) == np.float32(score)
    pcm = (np.clip(x, -1, 1) * 32767).astype("<i2")
    pred.reset_stream()
    got = [pred.predict_stream(audio_data=b, is_end=e) for b, e in _pushes(pcm)]
    pred.reset_stream()
    again = [pred.predict_stream(audio_data=b, is_end=e) for b, e in _pushes(pcm)]
    pred.reset_stream()
    assert got == again and got[-1] is not None and got[-1]["text"]


@pytest.mark.parametrize("decoder", ["ctc_greedy", "ctc_beam_search"])
def test_stream_pool_equals_single_streams(tmp_path, decoder):
    """8 slots, 7 streams of different lengths (slot 7 never runs): every push of every slot equals ``predict_stream`` on
    that stream alone, and a slot that is idle in a round keeps its caches (the conv module's left context and its
    attention K|V rows) byte for byte."""
    from masr_b200.stream_pool import StreamPool
    pred = _predictor(tmp_path, decoder)
    lens = [6 * PUSH - 1234, 5 * PUSH - 3000, 3 * PUSH - 500, 3 * PUSH, 2 * PUSH + 77, 4 * PUSH + 4000, PUSH + 2000]
    streams = [_pushes((np.clip(make_audio("noise" if i % 3 == 2 else "speech", 300 + i, n), -1, 1) * 32767).astype("<i2"))
               for i, n in enumerate(lens)]
    want = []
    for pieces in streams:
        pred.reset_stream()
        want.append([pred.predict_stream(audio_data=b, is_end=e) for b, e in pieces])
    pred.reset_stream()
    sp = StreamPool(pred.predictor, synth.vocabulary(), n_slots=8, max_frames=400,
                    **({"beam": pred._beam_conf} if decoder == "ctc_beam_search" else {}))
    pool = sp.pool

    def state(s):
        return [pool.xcat[:, s, :pool.lorder].clone()] + [t[s * pool.cap:(s + 1) * pool.cap].clone() for kv in pool.kv for t in kv]

    got = [[] for _ in streams]
    for k in range(max(len(p) for p in streams)):
        live = [i for i, p in enumerate(streams) if k < len(p)]
        idle = {s: state(s) for s in range(8) if s not in live}
        for is_end in (False, True):
            msgs = {i: streams[i][k][0] for i in live if streams[i][k][1] == is_end}
            if msgs:
                out = sp.push(msgs, is_end=is_end)
                for i in msgs:
                    got[i].append(out[i])
        for s, before in idle.items():
            assert all(torch.equal(a, b) for a, b in zip(before, state(s))), (k, s)
    for i, (g, w) in enumerate(zip(got, want)):
        assert len(g) == len(w)
        for r, x in zip(g, w):
            assert _same(r, x), (i, r, x)
    assert any(r is not None and r["text"] for g in got for r in g)


def test_wide_squeezeformer_is_rejected_before_any_launch(tmp_path):
    from masr_b200.weights import UnsupportedConfig
    sd = synth.squeezeformer_state_dict(0, d=512, heads=8, ffn=64, num_blocks=12, streaming=True)
    with pytest.raises(UnsupportedConfig, match="512"):
        _predictor(tmp_path, sd=sd, use_model="squeezeformer")
