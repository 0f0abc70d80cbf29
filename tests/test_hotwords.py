"""CPU: hotword tokenization and validation, the automaton arrays of masr_b200.hotwords against the string restatement of
oracle/hotwords.py (the credit after every token of random token strings), the worked longest-match cases, and the
restated search: with no hotwords it is oracle.lm's search bit for bit, and a hotword flips the best prefix while the
reported score stays that prefix's score without hotwords."""
import math

import numpy as np
import pytest

from masr_b200.hotwords import MAX_TOKENS, HotwordGraph, graph_or_none, tokenize
from oracle import hotwords as oh
from oracle import lm as olm
from test_beam import rand_posteriors

F = np.float32
VOCAB = ["<blank>", "<unk>", "北", "京", "大", "学", "天", "安", "门", "A", "B", "C", "X", "<space>", "<eos>"]


def test_tokenize_and_merge():
    assert tokenize(["北京", "A B", "北京"], VOCAB) == [(2, 3), (9, 13, 10)]
    g = HotwordGraph(["北京", "北京", "北京大学"], VOCAB, 2.0)
    assert g.hotwords == ["北京", "北京大学"] and g.nodes == 5 and g.score == F(2.0)
    assert graph_or_none([], VOCAB) is None and graph_or_none(None, VOCAB) is None
    assert graph_or_none(g, VOCAB) is g


@pytest.mark.parametrize("hw,match", [("北Q", "'北Q'.*'Q'"), ("", "empty"), ("A" * (MAX_TOKENS + 1), "more than 32"),
                                      ("é", "'é'")])
def test_tokenize_rejects(hw, match):
    with pytest.raises(ValueError, match=match):
        tokenize([hw], VOCAB)


def test_rejects_blank_and_space_without_token():
    with pytest.raises(ValueError, match="blank"):
        tokenize(["北x"], ["x", "北"], blank=0)
    with pytest.raises(ValueError, match="' '"):
        tokenize(["A B"], ["<blank>", "A", "B"])
    assert len(tokenize(["A" * MAX_TOKENS], VOCAB)[0]) == MAX_TOKENS


@pytest.mark.parametrize("w", [-1.0, float("inf"), float("nan")])
def test_rejects_bad_score(w):
    with pytest.raises(ValueError, match="hotword_score"):
        HotwordGraph(["北京"], VOCAB, w)


def array_step(g, s, c):
    """The kernel's step over the graph arrays (root 0)."""
    def child(n):
        for a in range(g.arc_off[n], g.arc_off[n + 1]):
            if g.arc_tok[a] == c:
                return int(g.arc_next[a])
        return -1
    bank, cur, nxt = F(0), s, 0
    for _ in range(MAX_TOKENS + 1):
        ch = child(cur)
        if ch >= 0:
            nxt = ch
            break
        if cur == 0:
            break
        if g.tail[cur] >= 0:
            bank = F(bank + g.ta_acc[cur])
            cur = int(g.tail[cur])
        else:
            cur = int(g.fail[cur])
    delta = F(F(bank + g.acc[nxt]) - g.acc[s])
    return delta, (0 if g.leaf[nxt] else nxt)


def node_strings(g):
    out = {0: ()}
    for n in range(g.nodes):
        for a in range(g.arc_off[n], g.arc_off[n + 1]):
            out[int(g.arc_next[a])] = out[n] + (int(g.arc_tok[a]),)
    return out


@pytest.mark.parametrize("seed", range(12))
def test_graph_arrays_equal_string_restatement(seed):
    rng = np.random.default_rng(seed)
    alpha = "ABCX"[:2 + seed % 3]
    vocab = ["<blank>"] + list(alpha)
    words = set()
    for _ in range(int(rng.integers(1, 7))):
        L = int(rng.integers(1, 6))
        words.add("".join(rng.choice(list(alpha), L)))
        if rng.random() < 0.5:                                      # nested: a prefix or suffix of one already there
            w0 = sorted(words)[0]
            words.add(w0[:max(1, len(w0) - 1)] if rng.random() < 0.5 else w0[1:] or w0)
    w = float(rng.choice([0.5, 1.5, 0.3, 2.7]))
    g = HotwordGraph(sorted(words), vocab, w)
    H = oh.HotwordMatcher(g.tokens, w)
    strs = node_strings(g)
    for n, s in strs.items():
        assert g.acc[n] == H.acc(s) and bool(g.leaf[n]) == (n != 0 and H.leaf(s))
        assert g.fin[n] - g.acc[n] == H.readout(s) or g.acc[n] == 0
    for _ in range(40):
        toks = [int(t) for t in rng.integers(1, len(vocab), int(rng.integers(0, 25)))]
        s_arr, s_str, c_arr = 0, (), F(0)
        for t in toks:
            d_arr, s_arr = array_step(g, s_arr, t)
            d_str, s_str = H.step(s_str, t)
            assert d_arr == d_str and strs[s_arr] == s_str, (sorted(words), toks)
            c_arr = F(c_arr + d_arr)
        assert F(c_arr + F(g.fin[s_arr] - g.acc[s_arr])) == H.credit(toks)[0]


def credit(words, text, w=1.0):
    toks = tokenize(words, VOCAB)
    return float(oh.HotwordMatcher(toks, w).credit(tokenize([text], VOCAB)[0])[0])


def test_worked_cases():
    nested = ["北京", "北京大学"]
    assert credit(nested, "北京大学") == 4.0
    assert credit(nested, "北京天安门") == 2.0
    assert credit(nested, "北京大") == 2.0                       # the unfinished longer hotword earns nothing
    assert credit(nested, "北京北京大学") == 6.0
    assert credit(["北京大学"], "北京大") == 0.0
    assert credit(["AA", "AAA"], "AAA") == 3.0
    assert credit(["AA", "AAA"], "AA") == 2.0
    assert credit(["AA", "AAA"], "AAAA") == 3.0
    assert credit(["AA", "AAA"], "AAAAA") == 5.0
    assert credit(["ABX", "BC"], "ABC") == 2.0
    assert credit(["ABX", "BC"], "ABX") == 3.0
    assert credit(["ABX", "BC"], "AB") == 0.0
    assert credit(["ABX", "BC"], "ABXBC") == 5.0


@pytest.mark.parametrize("seed,beam", [(1, 16), (2, 300), (3, 4)])
def test_restated_search_without_hotwords_is_the_lm_search(seed, beam):
    V = len(VOCAB)
    probs, _ = rand_posteriors(seed, 40, V, peaky=3.0)
    ref = olm.prefix_beam_search_lm(probs, None, VOCAB, beam_size=beam, nbest=3)
    assert oh.prefix_beam_search_hot(probs, None, VOCAB, beam_size=beam, nbest=3) == ref
    empty = oh.HotwordMatcher([], 1.5)
    got = oh.prefix_beam_search_hot(probs, None, VOCAB, beam_size=beam, nbest=3, hotwords=empty)
    assert [(np.float32(a).tobytes(), np.float32(b).tobytes(), t) for a, b, t in got] == \
        [(np.float32(a).tobytes(), np.float32(b).tobytes(), t) for a, b, t in ref]


def crafted():
    """Three frames: 北 or 门 (门 more likely), then 京, then blank."""
    V = len(VOCAB)
    p = np.full((3, V), 1e-4, np.float32)
    p[0, VOCAB.index("门")], p[0, VOCAB.index("北")] = 0.6, 0.4
    p[1, VOCAB.index("京")] = 0.9
    p[2, 0] = 0.9
    return p / p.sum(1, keepdims=True)


def test_hotword_flips_best_and_reports_the_plain_score():
    probs = crafted()
    plain = olm.prefix_beam_search_lm(probs, None, VOCAB, beam_size=8, nbest=8)
    assert plain[0][2] == [VOCAB.index("门"), VOCAB.index("京")]
    H = oh.HotwordMatcher(tokenize(["北京"], VOCAB), 1.5)
    (score, approx, toks), = oh.prefix_beam_search_hot(probs, None, VOCAB, beam_size=8, hotwords=H)
    assert toks == [VOCAB.index("北"), VOCAB.index("京")]
    want = next(s for s, _, t in plain if t == toks)
    assert math.isclose(score, want, rel_tol=0, abs_tol=1e-5) and score == approx
    H0 = oh.HotwordMatcher(tokenize(["北京"], VOCAB), 0.0)                # zero credit: today's result
    assert oh.prefix_beam_search_hot(probs, None, VOCAB, beam_size=8, hotwords=H0)[0][2] == plain[0][2]


HOT_ENTRY_POINTS = {
    "masr_ctc_prefix_beam": "masr_ctc_prefix_beam_hot", "masr_ctc_prefix_beam_stream": "masr_ctc_prefix_beam_hot_stream",
    "masr_ctc_prefix_beam_pool": "masr_ctc_prefix_beam_hot_pool", "masr_ctc_prefix_beam_lm": "masr_ctc_prefix_beam_lm_hot",
    "masr_ctc_prefix_beam_lm_stream": "masr_ctc_prefix_beam_lm_hot_stream",
    "masr_ctc_prefix_beam_lm_pool": "masr_ctc_prefix_beam_lm_hot_pool",
    "masr_ctc_prefix_beam_wordlm": "masr_ctc_prefix_beam_wordlm_hot",
    "masr_ctc_prefix_beam_wordlm_stream": "masr_ctc_prefix_beam_wordlm_hot_stream",
    "masr_ctc_prefix_beam_wordlm_pool": "masr_ctc_prefix_beam_wordlm_hot_pool"}


def test_hot_entry_points_extend_the_plain_ones():
    """Each hotword entry point takes its plain counterpart's arguments, then the graph and the slot roots (the names
    masr_b200.beam.BeamSearch composes: the LM's BEAM + "_hot" + the form's suffix)."""
    from masr_b200 import _lib
    for plain, hot in HOT_ENTRY_POINTS.items():
        p, h = _lib.SIGNATURES[plain], _lib.SIGNATURES[hot]
        assert h[:len(p) - 1] == p[:-1] and h[len(p) - 1:] == [_lib._hgp, _lib._vp, _lib._vp], hot
        assert hasattr(_lib.load(), hot)


@pytest.mark.parametrize("plain,hot", [("masr_ctc_prefix_beam_state_size", "masr_ctc_prefix_beam_hot_state_size"),
                                       ("masr_ctc_prefix_beam_lm_state_size", "masr_ctc_prefix_beam_lm_hot_state_size"),
                                       ("masr_ctc_prefix_beam_wordlm_state_size", "masr_ctc_prefix_beam_wordlm_hot_state_size")])
def test_hot_state_carries_one_more_int_per_beam_entry(plain, hot):
    import ctypes as C
    from masr_b200 import _lib
    sizes = {}
    for name in (plain, hot):
        si, sf = C.c_int64(0), C.c_int64(0)
        _lib.call(name, C.byref(si), C.byref(sf))
        sizes[name] = (si.value, sf.value)
    (pi, pf), (hi, hf) = sizes.values()
    assert hi == pi + 512 and hf == pf


@pytest.fixture(scope="module")
def arpas(tmp_path_factory):
    from masr_b200 import synth
    from oracle import word_lm as owl
    cv = synth.vocabulary(300)
    pc = str(tmp_path_factory.mktemp("lm") / "c.arpa")
    chars = synth.character_lm_arpa(pc, seed=3, order=3, n_chars=80, n_sentences=600, vocab_size=300)
    ev = synth.english_vocabulary()
    pw = str(tmp_path_factory.mktemp("wlm") / "w.arpa")
    synth.word_lm_arpa(pw, seed=3, order=3, n_words=120)
    return cv, olm.read_arpa(pc), [cv.index(c) for c in chars], ev, owl.WordLM(pw, ev)


def bits(res):
    return [(np.float32(a).tobytes(), np.float32(b).tobytes(), t) for a, b, t in res]


@pytest.mark.parametrize("seed,beam", [(4, 16), (5, 300)])
def test_restated_char_lm_search_without_hotwords_is_the_lm_search(arpas, seed, beam):
    cv, lm, ids, _, _ = arpas
    _, lg = rand_posteriors(seed, 40, len(cv), peaky=3.0)
    lg[:, ids] += 3.0
    e = np.exp(lg - lg.max(1, keepdims=True))
    probs = (e / e.sum(1, keepdims=True)).astype(np.float32)
    ref = olm.prefix_beam_search_lm(probs, lm, cv, 0.8, 1.0, beam_size=beam, nbest=3)
    for H in (None, oh.HotwordMatcher([], 1.5)):
        assert bits(oh.prefix_beam_search_hot(probs, lm, cv, 0.8, 1.0, beam_size=beam, nbest=3, hotwords=H)) == bits(ref)


@pytest.mark.parametrize("seed,beam", [(6, 16), (7, 300)])
def test_restated_word_lm_search_without_hotwords_is_the_word_lm_search(arpas, seed, beam):
    from oracle import word_lm as owl
    _, _, _, ev, o = arpas
    _, lg = rand_posteriors(seed, 50, len(ev), peaky=3.0)
    lg[:, sorted({t for ch in o.lex.child for t in ch})] += 1.0
    lg[:, o.space] += 2.0
    e = np.exp(lg - lg.max(1, keepdims=True))
    cands, blp = owl.prune_candidates((e / e.sum(1, keepdims=True)).astype(np.float32))
    ref = owl.WordLmSearch(o, 1.0, 1.5, beam).push(cands, blp)
    assert any(o.space in t for _, _, t in ref.result(3)), "no word was completed: the test exercises no LM term"
    for H in (None, oh.HotwordMatcher([], 1.5)):
        got = oh.WordLmSearchHot(o, 1.0, 1.5, beam, hotwords=H).push(cands, blp)
        assert bits(got.result(3)) == bits(ref.result(3)) and got.attempts == ref.attempts
