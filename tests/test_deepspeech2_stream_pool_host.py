"""CPU: ``StreamPool.push`` over the DeepSpeech2 pool's host-side rules, driven by stand-ins built from the ORACLE (fbank +
DeepSpeech2 chunk forward with each slot's carried (h, c) on torch-CPU).  DeepSpeech2 has no position table
(``DS2Weights.max_len == 0``) and a constant-size LSTM state, so a greedy slot has no length limit: three interleaved
streams, each longer than the pool's ``max_frames``, are never rejected and return, push by push, what one oracle
``predict_stream`` per stream returns; stream 0 is the utterance frozen from the reference's ``MASRPredictor.predict_stream``
(tests/golden/predictor_golden_deepspeech2.json).  The stand-in pool takes its length bound and chunk rule from
``DeepSpeech2StreamPool`` itself."""
import json
import os

import numpy as np
import torch

import test_stream_pool_host as host
from conftest import GOLDEN, make_audio
from masr_b200 import stream_pool as sp, synth
from masr_b200.deepspeech2 import DS2Weights
from masr_b200.engine import subsampled_len
from masr_b200.predict import CACHED_FEATURE_NUM, DECODING_WINDOW, chunk_starts
from oracle import ctc as octc, deepspeech2 as od, fbank as ob

MAX_FRAMES = 40                     # encoder frames (1.6 s): every stream below is longer


class OracleEngine(host.OracleEngine):
    """The host test's CPU fbank, with DeepSpeech2's weight record: ``max_len == 0``, no position table."""

    def __init__(self):
        super().__init__()
        self.w = DS2Weights(d_model=1024, heads=1, ffn=0, kernel=0, idim=80, vocab=synth.DEFAULT_VOCAB_SIZE, max_len=0)


class OracleDS2Pool:
    """``pool.step`` of the CUDA pool (ids / max-prob per slot, valid counts, per-slot frame counts) from the oracle's chunk
    forward with every slot's carried (h, c)."""

    SHORT_ONCE = sp.DeepSpeech2StreamPool.SHORT_ONCE
    OUT_ROWS = sp.DeepSpeech2StreamPool.OUT_ROWS
    frame_bounds = sp.DeepSpeech2StreamPool.frame_bounds

    def __init__(self, sd, n_slots, max_frames):
        self.sd, self.cfg, self.S = sd, od.DS2Config(), n_slots
        self.cap, self.beam = max_frames, None
        self.lens_host = [0] * n_slots
        self.st = [None] * n_slots

    def reset(self, slot):
        self.st[slot], self.lens_host[slot] = None, 0

    def step(self, feats, nframes):
        ids = torch.zeros(self.S, 16, dtype=torch.int32)
        maxp = torch.zeros(self.S, 16)
        tout = [subsampled_len(int(n)) for n in nframes]
        for s, n in enumerate(nframes):
            if tout[s]:
                with torch.no_grad():
                    probs, self.st[s] = od.get_encoder_out(self.sd, self.cfg, feats[s:s + 1, :n], self.st[s])
                ids[s, :tout[s]] = probs.argmax(1).to(torch.int32)
                maxp[s, :tout[s]] = probs.max(1).values
            self.lens_host[s] += tout[s]
        return ids, maxp, tout


def oracle_predict_stream(sd, pcm, push, vocab):
    state, gs, cfg = None, octc.GreedyStream(), od.DS2Config()
    remained, cached, out = None, None, []
    for s in range(0, len(pcm), push):
        is_end = s + push >= len(pcm)
        new = ob.pcm_bytes_to_float32(pcm[s:s + push].tobytes())
        remained = new if remained is None else np.concatenate([remained, new])
        x, _ = ob.normalize_gain(remained.copy())
        feat = ob.kaldi_fbank(ob.to_int16(x))
        cached = feat if cached is None else np.concatenate([cached, feat], axis=0)
        remained = x[160 * feat.shape[0]:]
        starts = chunk_starts(cached.shape[0], is_end)
        if not starts:
            out.append(None)
            continue
        res, end = None, None
        for cur in starts:
            end = min(cur + DECODING_WINDOW, cached.shape[0])
            with torch.no_grad():
                probs, state = od.get_encoder_out(sd, cfg, torch.from_numpy(cached[cur:end])[None], state)
            res = gs.push(probs.numpy(), vocab)
        cached = cached[end - CACHED_FEATURE_NUM:]
        out.append({"text": res[1], "score": res[0]})
    return out


def test_deepspeech2_pool_pushes_are_not_length_limited_and_match_predict_stream(monkeypatch):
    with open(os.path.join(GOLDEN, "predictor_golden_deepspeech2.json"), encoding="utf-8") as f:
        g = json.load(f)
    sd = synth.to_torch(synth.deepspeech2_state_dict(g["wseed"], streaming=True))
    vocab = synth.vocabulary()
    monkeypatch.setattr(sp, "make_pool", lambda eng, n, max_frames=3000: OracleDS2Pool(sd, n, max_frames))
    pool = sp.StreamPool(OracleEngine(), vocab, n_slots=4, max_frames=MAX_FRAMES)
    audios = [make_audio(g["kind"], g["aseed"], g["samples"]), make_audio("noise", 95, 16000 * 2 + 3000),
              make_audio("speech", 96, 16000 * 3)]
    pcms = [(np.clip(a, -1, 1) * 32767).astype("<i2") for a in audios]
    push = g["push"]
    want = [oracle_predict_stream(sd, p, push, vocab) for p in pcms]
    for r, w in zip(want[0], g["pushes_pcm"]):                # the stand-in reproduces the reference's frozen pushes
        assert (r is None) == (w is None) and (r is None or (r["text"] == w["text"] and abs(r["score"] - w["score"]) < 1e-3))
    got = [[] for _ in pcms]
    npush = [len(range(0, len(p), push)) for p in pcms]
    for k in range(max(npush)):
        mid = {i: pcms[i][k * push:(k + 1) * push].tobytes() for i in range(len(pcms)) if k < npush[i] - 1}
        last = {i: pcms[i][k * push:(k + 1) * push].tobytes() for i in range(len(pcms)) if k == npush[i] - 1}
        for grp, is_end in ((mid, False), (last, True)):
            if grp:
                out = pool.push(grp, is_end=is_end)            # (raises StreamSlotError if any slot were rejected)
                assert pool.last_errors == {}
                for i in grp:
                    got[i].append(out[i])
    assert all(pool.pool.lens_host[i] > MAX_FRAMES for i in range(len(pcms)))
    for i in range(len(pcms)):
        assert len(got[i]) == len(want[i])
        for r, w in zip(got[i], want[i]):
            assert (r is None) == (w is None), (i, r, w)
            if r is not None:
                assert r["text"] == w["text"], (i, r, w)
                assert abs(r["score"] - w["score"]) < 1e-4
    for r, w in zip(got[0], g["pushes_pcm"]):
        assert (r is None) == (w is None) and (r is None or (r["text"] == w["text"] and abs(r["score"] - w["score"]) < 1e-3))
    # a slot can be reset and reused: its state starts from zero again
    pool.reset_stream(1)
    out = pool.push({1: pcms[1][:push * 3].tobytes()}, is_end=True)
    ref = oracle_predict_stream(sd, pcms[1][:push * 3], push * 3, vocab)
    assert out[1]["text"] == ref[-1]["text"] and abs(out[1]["score"] - ref[-1]["score"]) < 1e-4
