"""CPU: the predictor's ``n_best=`` argument checks and the assembly of its ``'n_best'`` entries, with the engine stubbed
(no GPU): greedy decoding, non-integers and values outside 1..beam_size are refused before any work; entry 0 is always
the result's own text and score, including results without frames; without ``n_best`` nothing changes."""
import numpy as np
import pytest

from masr_b200.beam import check_n_best
from masr_b200.engine import nbest_lists
from masr_b200.predict import MASRPredictor
from masr_b200.text import nbest_dicts

VOCAB = ["<blank>", "<unk>", "a", "b", "<space>", "c"]


class _Featurizer:
    vocab_list = VOCAB
    vocab_size = len(VOCAB)


class _Engine:
    """``transcribe_beam`` as the GPU engine answers it: (tokens, scores[, onsets][, n-best lists])."""

    def __init__(self, toks, scores, hyps):
        self.toks, self.scores, self.hyps, self.calls = toks, scores, hyps, []

    def transcribe_beam(self, waves, **kw):
        self.calls.append(kw)
        out = (self.toks[:len(waves)], self.scores[:len(waves)])
        if kw.get("onsets"):
            out += ([list(range(len(t))) for t in self.toks[:len(waves)]],)
        n = kw.get("n_best")
        if n is not None:
            out += (nbest_lists(None, self, len(waves), n, out[0], out[1]) if n == 1 else
                    [h[:n] for h in self.hyps[:len(waves)]],)
        return out


def _predictor(engine, beam_size=8, decoder="ctc_beam_search"):
    p = object.__new__(MASRPredictor)
    p._text_featurizer = _Featurizer()
    p._beam_conf = {"beam_size": beam_size, "cutoff_prob": 0.99, "cutoff_top_n": 40} if decoder == "ctc_beam_search" else None
    p._hotwords, p._hotword_graphs, p._hotword_score = None, {}, 1.5
    p._sample_rate, p._resample, p._use_db, p._target_db = 16000, False, True, -20.0
    p.predictor = engine
    p.lm = None
    return p


def _engine():
    toks = [[2, 3], [], [5, 4, 2]]
    scores = [-1.5, 0.0, -3.25]
    hyps = [[([2, 3], -1.5), ([2], -2.0), ([3, 2], -2.5)], [([], 0.0)], [([5, 4, 2], -3.25), ([5, 2], -3.5)]]
    return _Engine(toks, scores, hyps)


def test_check_n_best():
    assert check_n_best(1, 8) == 1 and check_n_best(np.int64(8), 8) == 8
    for bad in (0, 9, -1):
        with pytest.raises(ValueError, match="out of range"):
            check_n_best(bad, 8)
    for bad in (2.0, 2.5, "3", True, None):
        with pytest.raises(ValueError, match="integer"):
            check_n_best(bad, 8)


def test_predictor_refuses_bad_n_best_before_any_work():
    eng = _engine()
    p = _predictor(eng)
    x = np.zeros(1600, np.float32)
    for bad in (0, 9, 2.5, "2", True):
        with pytest.raises(ValueError):
            p.predict(x, n_best=bad)
        with pytest.raises(ValueError):
            p.predict_batch([x], n_best=bad)
    assert eng.calls == []
    g = _predictor(eng, decoder="ctc_greedy")
    with pytest.raises(ValueError, match="ctc_greedy"):
        g.predict(x, n_best=2)
    with pytest.raises(ValueError, match="ctc_greedy"):
        g.predict_batch([x], n_best=1)
    with pytest.raises(ValueError, match="ctc_greedy"):
        g._n_best(3)
    assert eng.calls == []


def test_n_best_entries_are_assembled_with_the_result_first():
    eng = _engine()
    p = _predictor(eng)
    x = np.zeros(1600, np.float32)
    plain = p.predict_batch([x, x, x])
    assert all("n_best" not in r for r in plain) and eng.calls[-1]["n_best"] is None
    got = p.predict_batch([x, x, x], n_best=2)
    assert eng.calls[-1]["n_best"] == 2
    for r, q, hyps in zip(got, plain, eng.hyps):
        assert {k: r[k] for k in ("text", "score")} == q
        assert r["n_best"][0] == {"text": r["text"], "score": r["score"]}
        assert r["n_best"] == nbest_dicts(hyps[:2], VOCAB) and len(r["n_best"]) <= 2
    assert got[2]["n_best"][0]["text"] == "c a" and got[1]["n_best"] == [{"text": "", "score": 0.0}]
    one = p.predict(x, n_best=1, timestamps=True)
    assert one["n_best"] == [{"text": one["text"], "score": one["score"]}] and "tokens" in one


def test_nbest_lists_without_a_read_out():
    """n_best = 1, or no search (no frames): the result itself is the only entry, and nothing is launched."""
    toks, scores = [[2], []], [-0.5, 0.0]
    assert nbest_lists(None, None, 2, 5, toks, scores) == [[([2], -0.5)], [([], 0.0)]]
    assert nbest_lists(object(), None, 2, 1, toks, scores) == [[([2], -0.5)], [([], 0.0)]]


def test_stream_pool_refuses_n_best_without_beam_search():
    from masr_b200.stream_pool import StreamPool
    with pytest.raises(ValueError, match="ctc_beam_search"):
        StreamPool(None, VOCAB, 2, n_best=2)
    with pytest.raises(ValueError, match="out of range"):
        StreamPool(None, VOCAB, 2, beam={"beam_size": 4}, n_best=5)
