"""DeepSpeech2 at ``encoder_conf.rnn_size: 2048`` on the CPU: the oracle (oracle/deepspeech2.py, oracle/deepspeech2_gru.py)
pinned to the reference's outputs frozen at that width for both cells (tests/golden/make_wide_deepspeech2_golden.py), and
the weight loader's reading of the width from the checkpoint."""
import json
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN, load_npz, make_audio
from masr_b200 import synth
from oracle import ctc as octc, deepspeech2 as od, deepspeech2_gru as og, fbank as ob

H = 2048
WSEED = {("lstm", True): 0, ("gru", True): 2, ("lstm", False): 1, ("gru", False): 1}     # the fixtures' weight seeds
_W = {}


def weights(cell, streaming):
    key = (cell, streaming)
    if key not in _W:
        _W[key] = synth.to_torch(synth.deepspeech2_state_dict(WSEED[key], streaming=streaming, hidden=H, use_gru=cell == "gru"))
    return _W[key]


def _oracle(cell, streaming, feat, state=None):
    cfg = od.DS2Config(hidden=H, bidirectional=not streaming)
    with torch.no_grad():
        return (od if cell == "lstm" else og).get_encoder_out(weights(cell, streaming), cfg, feat, state)


@pytest.mark.parametrize("cell", ["lstm", "gru"])
def test_oracle_matches_reference_golden_whole_utterance(cell):
    z, meta = load_npz("deepspeech2_wide_golden.npz")
    vocab = synth.vocabulary()
    cases = [m for m in meta if m["cell"] == cell and not m.get("chunks")]
    assert {m["streaming"] for m in cases} == {True, False}
    for m in cases:
        assert m["wseed"] == WSEED[cell, m["streaming"]] and m["text"]
        feat = torch.from_numpy(z[m["name"] + "/feat"])[None]
        probs = _oracle(cell, m["streaming"], feat)[0].numpy()
        assert probs.shape[0] == z[m["name"] + "/ids"].shape[0]
        assert np.array_equal(probs.argmax(1), z[m["name"] + "/ids"]), m["name"]
        got = np.take_along_axis(probs, z[m["name"] + "/top_i"].astype(np.int64), axis=1)
        assert np.abs(got - z[m["name"] + "/top_p"]).max() < 1e-5, m["name"]
        score, text, _ = octc.greedy_decode(probs, vocab)
        assert text == m["text"] and abs(score - m["score"]) < 1e-3


@pytest.mark.parametrize("cell", ["lstm", "gru"])
def test_oracle_matches_reference_golden_chunk_walk(cell):
    """``get_encoder_out_chunk`` window by window with the state carried, ending in a short window: per-window top-8
    posteriors and frame ids, the h state after every window and the LSTM's c state."""
    z, meta = load_npz("deepspeech2_wide_golden.npz")
    m, = [m for m in meta if m["cell"] == cell and m.get("chunks")]
    feat = torch.from_numpy(z[m["name"] + "/feat"])[None]
    top_p, top_i, ids, want_h = (z[m["name"] + k] for k in ("/top_p", "/top_i", "/ids", "/h"))
    want_c = z[m["name"] + "/c"] if cell == "lstm" else None
    wins = z[m["name"] + "/windows"]
    assert wins[-1, 1] < 67 and want_h.shape == (len(wins), 5, H)
    st, row = None, 0
    for k, (cur, n) in enumerate(wins):
        p, st = _oracle(cell, True, feat[:, cur:cur + n], st)
        p = p.numpy()
        rows = slice(row, row + p.shape[0])
        row += p.shape[0]
        assert np.array_equal(p.argmax(1), ids[rows]), k
        assert np.abs(np.take_along_axis(p, top_i[rows].astype(np.int64), axis=1) - top_p[rows]).max() < 1e-5, k
        assert np.abs(st[0].reshape(5, H).numpy() - want_h[k]).max() < 1e-5, k
        if want_c is not None:
            assert np.abs(st[1].reshape(5, H).numpy() - want_c[k]).max() < 1e-5, k
    assert row == ids.shape[0]


@pytest.mark.parametrize("cell", ["lstm", "gru"])
def test_oracle_matches_reference_predictor_whole_utterance(cell):
    """The reference ``MASRPredictor``'s frozen whole-utterance result (greedy) is the oracle's greedy decode of the same
    audio's features."""
    with open(os.path.join(GOLDEN, "predictor_golden_deepspeech2_wide.json"), encoding="utf-8") as f:
        g = json.load(f)
    assert g["hidden"] == H and g[cell]["wseed"] == WSEED[cell, True]
    x = make_audio(g["kind"], g["aseed"], g["samples"])
    probs = _oracle(cell, True, torch.from_numpy(ob.featurize(x.copy()))[None])[0].numpy()
    score, text, _ = octc.greedy_decode(probs, synth.vocabulary())
    assert text == g[cell]["whole"]["text"] and text and abs(score - g[cell]["whole"]["score"]) < 1e-3


@pytest.mark.parametrize("cell", ["lstm", "gru"])
def test_loader_reads_the_width_from_the_checkpoint(cell):
    from masr_b200.deepspeech2 import pack_deepspeech2
    sd = weights(cell, False)
    w = pack_deepspeech2(sd, "cpu")
    assert w.hidden == H and w.dirs == 2 and w.d_model == 2 * H and w.cell == cell and w.gates == (4 if cell == "lstm" else 3)
    assert all(tuple(x.shape) == (w.gates * H, H) for ent in w.rnn for x in ent["whh"])
    assert all(ent["ln"][0].shape == (2 * H,) for ent in w.rnn)
