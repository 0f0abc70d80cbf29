"""Word n-gram LM fusion with the lexicon constraint (CPU): the C++ loader (masr_word_lm_load_arpa) against the oracle
(oracle/word_lm.py) — tables, lexicon, dict_size and rejected files — and hand-checked searches showing the restatement
applies each rule: the reset on the first attempt after <space>, beta only on <space>, the read-out term and approx."""
import math

import numpy as np
import pytest

from oracle import lm as olm, word_lm as owl

F = np.float32
LN10 = math.log(10.0)
VOCAB = ["<blank>", "a", "b", "<space>"]
A, B_, SP = 1, 2, 3

TINY_ARPA = """\\data\\
ngram 1=7
ngram 2=3

\\1-grams:
-99\t<s>\t-0.2
-0.8\t</s>
-1.5\t<unk>
-0.5\ta\t-0.3
-0.7\tab\t-0.1
-0.9\tb
-1.1\tc1

\\2-grams:
-0.2\t<s> a
-0.4\ta b
-0.6\tab </s>

\\end\\
"""


def write(tmp_path, text, name="w.arpa"):
    p = tmp_path / name
    p.write_text(text, encoding="utf-8")
    return str(p)


def c_word_lm(path, vocab):
    from masr_b200 import build
    from masr_b200.lm import WordLM
    build.build()
    return WordLM(path, vocab)


def decode_tables(c):
    """The C++ hash tables -> {order: {(ids...): (ln p, ln bo)}} (24-bit ids packed from bit 0 of the 4-word key)."""
    keys = c.keys.reshape(-1, 4).astype(np.uint64)
    vals = c.vals.reshape(-1, 2)
    out = {}
    for n in range(1, c.order + 1):
        lo, cnt = c._layout.off[n], c._layout.mask[n] + 1
        tab = {}
        for s in range(lo, lo + cnt):
            k = keys[s]
            if int(k[0]) == 0xFFFFFFFF:
                continue
            big = int(k[0]) | int(k[1]) << 32 | int(k[2]) << 64 | int(k[3]) << 96
            tab[tuple((big >> (24 * j)) & 0xFFFFFF for j in range(n))] = (vals[s, 0], vals[s, 1])
        out[n] = tab
    return out


def oracle_tables(o):
    ids = dict(o.lex.word_id)
    ids["<s>"], ids["</s>"] = o.lex.bos, o.lex.eos
    out = {}
    for n in range(1, o.order + 1):
        out[n] = {tuple(ids[w] for w in g): v for g, v in o.lm.ngrams[n].items() if all(w in ids for w in g)}
    return out


def test_tiny_word_lm_loader_and_oracle_agree(tmp_path):
    p = write(tmp_path, TINY_ARPA)
    o = owl.WordLM(p, VOCAB)
    c = c_word_lm(p, VOCAB)
    assert o.lex.words == ["a", "ab", "b"] and o.dict_size == 3 == c.dict_size          # c1 cannot be spelled; <unk> is no word
    assert (c.order, c.space, c.is_character_based, c.read_counts) == (2, SP, False, [7, 3])
    off, tok, nxt, word = o.lex.csr()
    assert (off, tok, nxt, word) == ([0, 2, 3, 3, 3], [A, B_, B_], [1, 3, 2], [-1, 0, 1, 2])
    assert c.lex_off.tolist() == off and c.lex_tok.tolist() == tok and c.lex_next.tolist() == nxt and c.lex_word.tolist() == word
    # root -a-> 1 (word a) -b-> 2 (word ab); root -b-> 3 (word b)
    assert o.lex.child[0] == {A: 1, B_: 3} and o.lex.child[1] == {B_: 2} and o.lex.word == [-1, 0, 1, 2]
    assert decode_tables(c) == oracle_tables(o)
    assert c.kept_counts == [5, 3]
    assert o.lnp(["a"], "b") == F(-0.4 * LN10)
    assert o.lnp(["b"], "a") == F(F(0.0 * LN10) + F(-0.5 * LN10))                        # b has no backoff weight
    assert o.lnp(["a"], "c1") == olm.OOV_SCORE and o.lnp(["c1"], "a") == olm.OOV_SCORE
    from masr_b200.lm import CharLM
    assert not CharLM(p, VOCAB).is_character_based                                      # masr_lm_load_arpa: as before


@pytest.mark.parametrize("order", [3, 5])
def test_synthetic_word_lm_loader_and_oracle_agree(tmp_path, order):
    from masr_b200 import synth
    vocab = synth.english_vocabulary()
    p = str(tmp_path / "w.arpa")
    words = synth.word_lm_arpa(p, seed=order, order=order, n_words=150)
    o = owl.WordLM(p, vocab)
    c = c_word_lm(p, vocab)
    assert o.dict_size == c.dict_size == len(words) - 4                               # the four unspellable words are left out
    assert not {"abc1", "Hello", "café", "x-ray"} & set(o.lex.words)
    assert any(w[:-1] in o.lex.word_id for w in o.lex.words if len(w) > 1)            # words that prefix other words
    assert [c.lex_off.tolist(), c.lex_tok.tolist(), c.lex_next.tolist(), c.lex_word.tolist()] == list(map(list, o.lex.csr()))
    assert decode_tables(c) == oracle_tables(o)
    assert c.read_counts == o.lm.counts
    assert c.describe() == f"is_character_based = False, max_order = {order}, dict_size = {o.dict_size}"


def test_more_than_65536_words(tmp_path):
    from masr_b200 import synth
    vocab = synth.english_vocabulary()
    p = str(tmp_path / "big.arpa")
    synth.word_lm_arpa(p, seed=9, order=2, n_words=100, extra_unigrams=70_000)
    o = owl.WordLM(p, vocab)
    c = c_word_lm(p, vocab)
    assert o.dict_size == c.dict_size > 70_000
    assert c.lex_word.tolist() == o.lex.word
    assert decode_tables(c) == oracle_tables(o)


def _huge_count(s):
    return s.replace("ngram 1=7", f"ngram 1={(1 << 24)}")


def _order6(s):
    return (s.replace("ngram 2=3", "ngram 2=3\nngram 3=0\nngram 4=0\nngram 5=0\nngram 6=0")
             .replace("\\end\\", "\\3-grams:\n\n\\4-grams:\n\n\\5-grams:\n\n\\6-grams:\n\n\\end\\"))


@pytest.mark.parametrize("bad,vocab,match", [
    (_huge_count, VOCAB, "24-bit"),                                     # word ids beyond the supported width
    (_order6, VOCAB, "order 6"),                                        # 6 ids of 24 bits do not fit the key
    (lambda s: s, ["<blank>", "a", "b", " "], "<space>"),              # a vocabulary without <space>
    (lambda s: s.replace("ab\t", "x\t").replace("c1", "y").replace("ab </s>", "x </s>"), VOCAB, "character-based"),
    (lambda s: s.replace("ngram 2=3", "ngram 2=4"), VOCAB, "count mismatch"),
    (lambda s: s.replace("\\end\\", ""), VOCAB, "section mismatch"),
    (lambda s: s.replace("-0.4\ta b", "-0.4x\ta b"), VOCAB, "malformed"),
])
def test_rejected_word_lm_files(tmp_path, bad, vocab, match):
    from masr_b200 import _lib
    p = write(tmp_path, bad(TINY_ARPA))
    with pytest.raises(olm.ArpaError):
        owl.WordLM(p, vocab)
    with pytest.raises(_lib.MasrB200Error, match=match):
        c_word_lm(p, vocab)


# ---- hand-checked searches ----------------------------------------------------------------------------------------
@pytest.fixture
def tiny(tmp_path):
    return owl.WordLM(write(tmp_path, TINY_ARPA), VOCAB)


def search(w, frames, alpha=1.0, beta=0.5, beam=16):
    s = owl.WordLmSearch(w, alpha, beta, beam, min_cutoff=False)
    s.push(frames, [F(-1.0)] * len(frames))
    return s


def beam_of(s):
    """{token tuple: carried score} of the beam (before the read-out)."""
    return {s.toks_of[n]: logaddexp(pb, pnb) for n, pb, pnb in s.beam}


def logaddexp(a, b):
    from oracle.beam import logaddexp32
    return logaddexp32(a, b)


def test_beta_only_on_space(tiny):
    l1, l2 = F(-0.25), F(-0.75)
    s = search(tiny, [[(A, l1)], [(SP, l2)]], alpha=1.5, beta=0.5)
    got = beam_of(s)
    assert got == {(A, SP): F(F(F(l1 + l2) + F(F(1.5) * tiny.lnp(["<s>"], "a"))) + F(0.5))}
    s = search(tiny, [[(A, l1)], [(B_, l2)]], alpha=1.5, beta=0.5)
    assert beam_of(s) == {(A, B_): F(l1 + l2)}                         # letters: no LM term, no beta


def test_lexicon_rejects_and_space_needs_a_word_end(tiny):
    l = F(-0.5)
    s = search(tiny, [[(B_, l)], [(A, l), (0, l)]])                    # "ba" is no prefix of a lexicon word
    assert beam_of(s) == {(B_,): F(l + l)}
    s = search(tiny, [[(SP, l)]])                                      # <space> at the root: rejected
    assert beam_of(s) == {}


def test_reset_on_first_attempt_after_space(tiny):
    l = F(-0.5)
    # after "a ", the first attempt (b) is rejected and resets the prefix; nothing else is tried in that frame
    s = search(tiny, [[(A, l)], [(SP, l)], [(B_, l)]])
    assert beam_of(s) == {}
    assert s.attempts == 1
    # a repeated <space> with p_b("a ") = -inf adds nothing but is the first attempt: b is then accepted from the root
    s = search(tiny, [[(A, l)], [(SP, l)], [(SP, l), (B_, l)]])
    got = beam_of(s)
    assert set(got) == {(A, SP), (A, SP, B_)} and s.attempts == 1
    assert got[(A, SP)] == F(beam_of(search(tiny, [[(A, l)], [(SP, l)]]))[(A, SP)] + l)
    # the reset is kept with the prefix: later frames do not reject again
    s = search(tiny, [[(A, l)], [(SP, l)], [(SP, l)], [(B_, l)]])
    assert set(beam_of(s)) == {(A, SP, B_)} and s.attempts == 1
    # the cut-off prefix makes no attempt (min_cutoff): the reset waits for the next frame that tries it
    s = owl.WordLmSearch(tiny, 1.0, 0.5, beam_size=1)
    s.push([[(A, l)], [(SP, l)], [(B_, F(-30.0))]], [F(-1.0), F(-1.0), F(-0.01)])
    assert s.attempts == 0


def test_readout_and_approx(tiny):
    alpha, beta = F(1.5), F(0.5)
    l = F(-0.5)
    # trailing complete word "ab": + alpha lnP(ab | <s>) + beta on the side
    s = search(tiny, [[(A, l)], [(B_, l)]], alpha, beta)
    carried = beam_of(s)[(A, B_)]
    (score, approx, toks), = s.result()
    lnp = tiny.lnp(["<s>"], "ab")
    assert toks == [A, B_] and F(score) == F(carried + F(F(alpha * lnp) + beta))
    S = F(lnp + tiny.lnp(["ab"], "</s>"))
    assert F(approx) == F(F(F(score) - F(F(2.0) * beta)) - F(alpha * S))
    assert beam_of(s)[(A, B_)] == carried                              # the read-out never enters the carried state
    # a trailing partial word that is no word end: lnP = -1000 (and its </s> term is out of vocabulary too)
    w2 = owl.WordLM.__new__(owl.WordLM)
    w2.__dict__.update(tiny.__dict__)
    w2.lex = owl.Lexicon(tiny.lm, VOCAB, ["ab"])
    s = search(w2, [[(A, l)]], alpha, beta)
    (score, approx, toks), = s.result()
    assert toks == [A] and F(score) == F(l + F(F(alpha * olm.OOV_SCORE) + beta))
    assert F(approx) == F(F(F(score) - beta) - F(alpha * F(olm.OOV_SCORE + olm.OOV_SCORE)))
    # a prefix ending in <space> gets no read-out term; the best is chosen after the term, ties by beam rank
    s = search(tiny, [[(A, l)], [(SP, l)]], alpha, beta)
    (score, _, toks), = s.result()
    assert toks == [A, SP] and F(score) == beam_of(s)[(A, SP)]


def test_two_frame_path_sum(tiny):
    """Every surviving prefix's carried score is the float32 path sum of its alignments plus its LM terms."""
    la, lb, lbl = F(math.log(0.5)), F(math.log(0.3)), F(math.log(0.2))
    fr = [(A, la), (B_, lb), (0, lbl)]
    s = search(tiny, [fr, fr], alpha=0.0, beta=0.0)
    got = beam_of(s)
    # "a": a a | a - | - a ; "b": b b | b - | - b ; "ab": a b ; "ba" rejected ; "" : - -
    assert got[(A,)] == logaddexp(logaddexp(F(la + la), F(la + lbl)), F(lbl + la))
    assert got[(A, B_)] == F(la + lb)
    assert got[()] == F(lbl + lbl)
    assert (B_, A) not in got


def test_oracle_hypotheses_split_into_lexicon_words(tmp_path):
    from masr_b200 import synth
    from oracle.beam import prune_frame
    vocab = synth.english_vocabulary()
    p = str(tmp_path / "w.arpa")
    synth.word_lm_arpa(p, seed=3, order=3, n_words=60)
    w = owl.WordLM(p, vocab)
    rng = np.random.default_rng(0)
    lex_tok = sorted({t for d in w.lex.child for t in d})
    for seed in range(3):
        logits = rng.normal(0, 1.5, (60, len(vocab))).astype(np.float32)
        logits[:, lex_tok + [w.space]] += 2.0
        logits[:, 0] += 2.5
        pr = np.exp(logits - logits.max(1, keepdims=True))
        pr = (pr / pr.sum(1, keepdims=True)).astype(np.float32)
        cands = [[(c, F(math.log(float(pc)))) for c, pc in prune_frame(q, 0.99, 40)] for q in pr]
        blp = [F(math.log(float(q[0]))) for q in pr]
        out = owl.prefix_beam_search_wordlm(w, cands, blp, alpha=1.0, beta=1.0, beam_size=32, nbest=8)
        assert out
        for _, _, toks in out:
            text = "".join(vocab[t] if t != w.space else " " for t in toks)
            assert "  " not in text and not text.startswith(" ")
            pieces = text.split(" ")
            for word in pieces[:-1]:
                assert word in w.lex.word_id, (word, text)
            n = 0
            for ch in pieces[-1]:
                n = w.lex.child[n][vocab.index(ch)]                    # a trailing piece is a lexicon prefix


def test_word_lm_entry_points_by_name(tmp_path):
    """masr_word_lm_load_arpa / _info / _export called directly agree with the WordLM built on them."""
    import ctypes as C
    from masr_b200 import _lib
    p = write(tmp_path, TINY_ARPA)
    w = c_word_lm(p, VOCAB)
    lib = _lib.load()
    h = C.c_void_p()
    vocab = "\n".join(VOCAB).encode()
    _lib.call("masr_word_lm_load_arpa", C.c_char_p(p.encode()), C.c_char_p(vocab), len(VOCAB), C.byref(h))
    try:
        info = (C.c_int64 * 32)()
        _lib.call("masr_word_lm_info", h, info)
        assert (info[_lib.LM_INFO_DICT_SIZE], info[_lib.WORD_LM_INFO_NODES], info[_lib.WORD_LM_INFO_ARCS],
                info[_lib.WORD_LM_INFO_SPACE], info[_lib.LM_INFO_CHAR_BASED]) == (3, 4, 3, SP, 0)
        keys = np.empty(info[_lib.LM_INFO_KEY_WORDS], np.uint32)
        vals = np.empty(info[_lib.LM_INFO_VAL_FLOATS], np.float32)
        off, tok, nxt, wd = (np.empty(n, np.int32) for n in (5, 3, 3, 4))
        lay = _lib.WordLmTables()
        _lib.call("masr_word_lm_export", h, keys.ctypes.data, vals.ctypes.data, off.ctypes.data, tok.ctypes.data, nxt.ctypes.data,
                  wd.ctypes.data, C.byref(lay))
        assert np.array_equal(keys, w.keys) and np.array_equal(vals, w.vals) and wd.tolist() == [-1, 0, 1, 2]
        assert (lay.order, lay.bos, lay.eos, lay.space, lay.root, lay.nodes, lay.dict_size) == (2, 3, 4, SP, 0, 4, 3)
    finally:
        lib.masr_lm_free(h)
