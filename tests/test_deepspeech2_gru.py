"""DeepSpeech2 with GRU recurrences (``encoder_conf.use_gru: True``) on the CPU: the oracle's explicit GRU cell pinned to the
reference's frozen outputs (tests/golden/make_deepspeech2_gru_golden.py), and the weight loader on the reference's GRU key
layout."""
import json
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN, load_npz, make_audio
from masr_b200 import synth
from oracle import ctc as octc, deepspeech2 as od, deepspeech2_gru as og, fbank as ob

_W = {}


def weights(seed, streaming):
    if (seed, streaming) not in _W:
        _W[seed, streaming] = synth.deepspeech2_state_dict(seed, streaming=streaming, use_gru=True)
    return _W[seed, streaming]


def test_oracle_matches_reference_golden_whole_utterance():
    z, meta = load_npz("deepspeech2_gru_golden.npz")
    vocab = synth.vocabulary()
    cases = [m for m in meta if not m.get("chunks")]
    assert {m["streaming"] for m in cases} == {True, False}
    for m in cases:
        sd = synth.to_torch(weights(m["wseed"], m["streaming"]))
        cfg = od.DS2Config(bidirectional=not m["streaming"])
        feat = torch.from_numpy(z[m["name"] + "/feat"])[None]
        with torch.no_grad():
            probs, _ = og.get_encoder_out(sd, cfg, feat)
        probs = probs.numpy()
        assert np.array_equal(probs.argmax(1), z[m["name"] + "/ids"])
        got = np.take_along_axis(probs, z[m["name"] + "/top_i"].astype(np.int64), axis=1)
        assert np.abs(got - z[m["name"] + "/top_p"]).max() < 1e-5
        score, text, _ = octc.greedy_decode(probs, vocab)
        assert text == m["text"] and abs(score - m["score"]) < 1e-3


def test_oracle_matches_reference_golden_chunk_walk():
    """``get_encoder_out_chunk`` window by window with the h state carried (the GRU ignores c and returns c = h), ending in a
    short window: per-window top-8 posteriors and frame ids, and the h state after every window."""
    z, meta = load_npz("deepspeech2_gru_golden.npz")
    m, = [m for m in meta if m.get("chunks")]
    sd = synth.to_torch(weights(m["wseed"], True))
    cfg = od.DS2Config()
    feat = torch.from_numpy(z[m["name"] + "/feat"])[None]
    top_p, top_i, ids, want_h = (z[m["name"] + k] for k in ("/top_p", "/top_i", "/ids", "/h"))
    wins = z[m["name"] + "/windows"]
    assert wins[-1, 1] < 67
    st, row = None, 0
    for k, (cur, n) in enumerate(wins):
        with torch.no_grad():
            p, st = og.get_encoder_out(sd, cfg, feat[:, cur:cur + n], st)
        p = p.numpy()
        rows = slice(row, row + p.shape[0])
        row += p.shape[0]
        got = np.take_along_axis(p, top_i[rows].astype(np.int64), axis=1)
        assert np.abs(got - top_p[rows]).max() < 5e-6, k
        assert np.array_equal(p.argmax(1), ids[rows]), k
        assert torch.equal(st[0], st[1])                      # c is h again
        assert np.abs(st[0][:, 0].numpy() - want_h[k]).max() < 2e-5, k
    assert row == ids.shape[0]


def test_oracle_chunked_equals_whole_for_forward_gru():
    """Carrying h across chunks reproduces the whole-utterance GRU stack on the same subsampled frames."""
    sd = synth.to_torch(weights(0, True))
    cfg = od.DS2Config()
    feat = torch.from_numpy(ob.featurize(make_audio("speech", 5, 16000 * 2)))[None]
    st = None
    outs = []
    with torch.no_grad():
        for cur in range(0, feat.shape[1] - 67 + 1, 64):
            p, st = og.get_encoder_out(sd, cfg, feat[:, cur:cur + 67], st)
            outs.append(p)
        whole, _ = og.get_encoder_out(sd, cfg, feat[:, :64 * len(outs) + 3])
    assert torch.cat(outs).shape == whole.shape
    assert (torch.cat(outs) - whole).abs().max().item() < 1e-5


def test_oracle_chunk_path_reproduces_reference_predict_stream():
    """The oracle's chunked forward + greedy history reproduces the reference ``MASRPredictor.predict_stream`` on a GRU
    model push by push (tests/golden/predictor_golden_deepspeech2_gru.json)."""
    from masr_b200.predict import CACHED_FEATURE_NUM, DECODING_WINDOW, chunk_starts
    with open(os.path.join(GOLDEN, "predictor_golden_deepspeech2_gru.json"), encoding="utf-8") as f:
        g = json.load(f)
    sd = synth.to_torch(weights(g["wseed"], True))
    cfg = od.DS2Config()
    vocab = synth.vocabulary()
    x = make_audio(g["kind"], g["aseed"], g["samples"])
    with torch.no_grad():
        probs, _ = og.get_encoder_out(sd, cfg, torch.from_numpy(ob.featurize(x.copy()))[None])
    score, text, _ = octc.greedy_decode(probs.numpy(), vocab)
    assert text == g["whole"]["text"] and abs(score - g["whole"]["score"]) < 1e-3
    pcm = (np.clip(x, -1, 1) * 32767).astype("<i2")
    push = g["push"]
    state, gs = None, octc.GreedyStream()
    remained, cached, got = None, None, []
    for s in range(0, len(pcm), push):
        is_end = s + push >= len(pcm)
        new = ob.pcm_bytes_to_float32(pcm[s:s + push].tobytes())
        remained = new if remained is None else np.concatenate([remained, new])
        xn, _ = ob.normalize_gain(remained.copy())
        feat = ob.kaldi_fbank(ob.to_int16(xn))
        cached = feat if cached is None else np.concatenate([cached, feat], axis=0)
        remained = xn[160 * feat.shape[0]:]
        starts = chunk_starts(cached.shape[0], is_end)
        if not starts:
            got.append(None)
            continue
        res, end = None, None
        for cur in starts:
            end = min(cur + DECODING_WINDOW, cached.shape[0])
            with torch.no_grad():
                pr, state = og.get_encoder_out(sd, cfg, torch.from_numpy(cached[cur:end])[None], state)
            res = gs.push(pr.numpy(), vocab)
        cached = cached[end - CACHED_FEATURE_NUM:]
        got.append({"text": res[1], "score": res[0]})
    assert len(got) == len(g["pushes_pcm"])
    assert any(r is not None and r["text"] for r in got)
    for r, w in zip(got, g["pushes_pcm"]):
        assert (r is None) == (w is None)
        if r is not None:
            assert r["text"] == w["text"]
            assert abs(r["score"] - w["score"]) < 1e-3


def _small(streaming, seed=3):
    return synth.to_torch(synth.deepspeech2_state_dict(seed, streaming=streaming, layers=2, hidden=64, use_gru=True))


def test_check_supported_accepts_the_reference_gru_layout():
    """The reference's ``GRU`` wrapper nests ``nn.GRU`` one level deeper (``encoder.rnns.{l}.rnn.rnn.*``, gru.py:6-15) with
    3H gate rows; that layout loads, while 3H rows under the LSTM names and 4H rows under the GRU names are refused."""
    from masr_b200.weights import UnsupportedConfig, check_supported
    for streaming in (True, False):
        sd = _small(streaming)
        assert "encoder.rnns.1.rnn.rnn.weight_hh_l0" in sd and ("encoder.rnns.1.rnn.rnn.weight_hh_l0_reverse" in sd) != streaming
        assert not any(k.startswith("encoder.rnns.0.rnn.weight") for k in sd)
        check_supported(sd, "deepspeech2")
    with pytest.raises(UnsupportedConfig, match="use_gru"):
        check_supported({"encoder.rnns.0.rnn.weight_hh_l0": torch.zeros(3 * 16, 16)}, "deepspeech2")
    with pytest.raises(UnsupportedConfig, match="use_gru"):
        check_supported({"encoder.rnns.0.rnn.rnn.weight_hh_l0": torch.zeros(4 * 16, 16)}, "deepspeech2")


@pytest.mark.parametrize("streaming", [True, False])
def test_pack_folds_b_hr_b_hz_and_keeps_b_hn(streaming):
    """gates_x bias = b_ih + [b_hr, b_hz, 0]; b_hn [H] separately; layer 0's input columns permuted to the channels-last
    conv output with 3H rows; the cell type recorded."""
    from masr_b200.deepspeech2 import pack_deepspeech2
    sd = _small(streaming)
    w = pack_deepspeech2(sd, "cpu")
    H, dirs = 64, 1 if streaming else 2
    assert (w.cell, w.gates, w.hidden, w.dirs, w.d_model, len(w.rnn)) == ("gru", 3, H, dirs, H * dirs, 2)
    for l, ent in enumerate(w.rnn):
        for di, suf in enumerate(("", "_reverse")[:dirs]):
            p = f"encoder.rnns.{l}.rnn.rnn."
            bih, bhh = sd[p + "bias_ih_l0" + suf], sd[p + "bias_hh_l0" + suf]
            assert torch.equal(ent["bias"][di][:2 * H], bih[:2 * H] + bhh[:2 * H])
            assert torch.equal(ent["bias"][di][2 * H:], bih[2 * H:])
            assert torch.equal(ent["bhn"][di], bhh[2 * H:])
            assert torch.equal(ent["whh"][di], sd[p + "weight_hh_l0" + suf])
            wih = sd[p + "weight_ih_l0" + suf]
            if l == 0:      # column c*19 + f of the reference -> f*32 + c
                assert ent["wih"][di].shape == (3 * H, 19 * 32)
                assert torch.equal(ent["wih"][di].reshape(3 * H, 19, 32).permute(0, 2, 1).reshape(3 * H, -1), wih)
            else:
                assert torch.equal(ent["wih"][di], wih)


def test_lstm_weights_draw_the_same_numbers():
    """``use_gru`` is an appended option: the default LSTM weights are the ones every existing fixture was made from."""
    a = synth.deepspeech2_state_dict(2, layers=2, hidden=64)
    b = synth.deepspeech2_state_dict(2, layers=2, hidden=64, use_gru=False)
    assert a.keys() == b.keys() and all(np.array_equal(a[k], b[k]) for k in a)
    assert a["encoder.rnns.0.rnn.weight_hh_l0"].shape == (256, 64)
