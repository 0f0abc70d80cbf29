"""Character n-gram LM fusion (CPU): the ARPA reader of the oracle and of the library's C++ loader, the generated LM's
normalisation, and the defining properties of the fused prefix beam search restatement (oracle/lm.py)."""
import itertools
import math

import numpy as np
import pytest

from oracle import beam as obeam, ctc as octc, lm as olm

SMALL_ARPA = """some header text

\\data\\
ngram 1=6
ngram 2=4

\\1-grams:
-99\t<s>\t-0.30103
-0.69897\t</s>
-1.0\t<unk>
-0.52288\t甲\t-0.2
-0.60206\t乙\t-0.1
-0.9\t丙

\\2-grams:
-0.1\t<s> 甲
-0.3\t甲 乙
-0.4\t乙 甲
-0.2\t甲 </s>

\\end\\
"""


def write(tmp_path, text, name="lm.arpa"):
    p = tmp_path / name
    p.write_text(text, encoding="utf-8")
    return str(p)


def c_loader(path, vocab):
    from masr_b200 import build
    from masr_b200.lm import CharLM
    build.build()
    return CharLM(path, vocab)


def test_small_arpa_oracle_and_loader_agree(tmp_path):
    p = write(tmp_path, SMALL_ARPA)
    o = olm.read_arpa(p)
    vocab = ["<blank>", "<unk>", "甲", "乙", "丁", "<eos>"]          # 丙 is not a model token; 丁 is not an LM word
    c = c_loader(p, vocab)
    assert (o.order, o.counts, o.is_character_based, o.dict_size) == (2, [6, 4], True, 6)
    assert (c.order, c.read_counts, c.is_character_based, c.dict_size) == (o.order, o.counts, o.is_character_based, o.dict_size)
    assert c.kept_counts == [4, 4]                                  # <s>, </s>, 甲, 乙 (<unk> and 丙 are no query's target)
    assert c.tok2lm.tolist() == [-1, -1, 2, 3, -1, -1]
    assert o.lnp(["甲"], "乙") == np.float32(-0.3 * math.log(10))
    assert o.lnp(["乙"], "乙") == np.float32(np.float32(-0.1 * math.log(10)) + np.float32(-0.60206 * math.log(10)))
    assert o.lnp(["丁"], "甲") == olm.OOV_SCORE and o.lnp(["甲"], "<unk>") == olm.OOV_SCORE
    word = write(tmp_path, SMALL_ARPA.replace("-0.9\t丙", "-0.9\t丙丁"), "word.arpa")
    assert not olm.read_arpa(word).is_character_based
    assert not c_loader(word, vocab).is_character_based


@pytest.mark.parametrize("bad,match", [
    (lambda s: s.replace("\\data\\", "\\dada\\"), "data"),
    (lambda s: s.replace("ngram 2=4", "ngram 2=5"), "count mismatch"),
    (lambda s: s.replace("ngram 2=4", "ngram 3=4"), "count mismatch"),
    (lambda s: s.replace("\\2-grams:", "\\3-grams:"), "section mismatch"),
    (lambda s: s.replace("\\end\\", ""), "section mismatch"),
    (lambda s: s.replace("-99\t<s>\t-0.30103\n", "-99\t<x>\t-0.30103\n"), "<s>"),
    (lambda s: s.replace("-0.69897\t</s>", "-0.69897\t<y>"), "</s>"),
    (lambda s: s.replace("ngram 2=4", "ngram 2=4\nngram 3=0\nngram 4=0\nngram 5=0\nngram 6=0\nngram 7=0")
     .replace("\\end\\", "\\3-grams:\n\n\\4-grams:\n\n\\5-grams:\n\n\\6-grams:\n\n\\7-grams:\n\n\\end\\"), "order 7"),
    (lambda s: s.replace("-0.3\t甲 乙", "-0.3x\t甲 乙"), "malformed"),
    (lambda s: s.replace("-0.3\t甲 乙", "-0.3\t甲 乙 丙 丁"), "malformed"),
    (lambda s: s.replace("ngram 1=6", "ngram 1=six"), "malformed"),
])
def test_malformed_arpa_is_rejected(tmp_path, bad, match):
    from masr_b200 import _lib
    p = write(tmp_path, bad(SMALL_ARPA))
    with pytest.raises(olm.ArpaError, match=match):
        olm.read_arpa(p)
    with pytest.raises(_lib.MasrB200Error, match=match):
        c_loader(p, ["<blank>", "甲", "乙"])


def test_kenlm_binary_is_identified(tmp_path):
    from masr_b200 import _lib
    from masr_b200.lm import sniff
    p = tmp_path / "lm.klm"
    p.write_bytes(b"mmap lm http://kheafield.com/code format version 5\n\x00\x01\x02")
    assert sniff(str(p)) == "kenlm_binary"
    assert sniff(write(tmp_path, SMALL_ARPA)) == "arpa"
    assert sniff(str(tmp_path / "none.klm")) == "missing"
    with pytest.raises(olm.ArpaError, match="KenLM binary"):
        olm.read_arpa(str(p))
    with pytest.raises(_lib.MasrB200Error, match="KenLM binary"):
        c_loader(str(p), ["<blank>", "甲"])


def lnp64(lm, ctx, w):
    """The backoff definition in float64 without the OOV rule (so <unk> gets its real mass)."""
    acc = 0.0
    for L in range(lm.order - 1, -1, -1):
        h = tuple(ctx[len(ctx) - L:]) if L else ()
        e = lm.ngrams[L + 1].get(h + (w,))
        if e is not None:
            return acc + float(e[0])
        if L >= 1 and h in lm.ngrams[L]:
            acc += float(lm.ngrams[L][h][1])
    raise AssertionError((ctx, w))


@pytest.mark.parametrize("order", [3, 5])
def test_generated_lm_is_normalised(tmp_path, order):
    from masr_b200 import synth
    p = str(tmp_path / "g.arpa")
    chars = synth.character_lm_arpa(p, seed=order, order=order, n_sentences=300)
    lm = olm.read_arpa(p)
    assert lm.order == order and lm.is_character_based and lm.unigrams == set(chars) | {"<s>", "</s>", "<unk>"}
    for n in range(1, order):        # lmplz convention: backoffs only on n-grams that prefix a longer one
        prefixes = {g[:-1] for g in lm.ngrams[n + 1]}
        assert all(bo == 0 or g in prefixes for g, (_, bo) in lm.ngrams[n].items())
    rng = np.random.default_rng(0)
    seen = list(lm.ngrams[order - 1]) if order > 1 else [()]
    words = chars + ["</s>", "<unk>"]
    for i in range(40):
        if i % 2:
            ctx = list(seen[int(rng.integers(len(seen)))])                 # a context the corpus has
        else:
            ctx = [chars[int(j)] for j in rng.integers(0, len(chars), int(rng.integers(0, order)))]   # <s>-padded below
        ctx = lm.window(ctx)
        total = sum(math.exp(lnp64(lm, ctx, w)) for w in words)
        assert abs(total - 1.0) < 1e-5, (ctx, total)
        for w in words[:-1]:
            if all(lm.in_vocab(x) for x in ctx):
                assert abs(float(lm.lnp(ctx, w)) - lnp64(lm, ctx, w)) < 1e-5 * max(1.0, abs(lnp64(lm, ctx, w)))


def tiny_lm(tmp_path):
    """甲 乙 丙 in the LM (乙 strongly after 甲), 丁 a model token outside it."""
    text = """\\data\\
ngram 1=6
ngram 2=4

\\1-grams:
-99\t<s>\t-0.2
-0.8\t</s>
-2.0\t<unk>
-0.7\t甲\t-0.15
-0.6\t乙\t-0.25
-0.65\t丙\t-0.1

\\2-grams:
-0.3\t<s> 甲
-0.05\t甲 乙
-1.5\t甲 丙
-0.4\t乙 </s>

\\end\\
"""
    return olm.read_arpa(write(tmp_path, text)), ["<blank>", "甲", "乙", "丙", "丁"]


def brute_force(p):
    mass = {}
    T, V = p.shape
    for path in itertools.product(range(V), repeat=T):
        key = tuple(octc.collapse(path))
        mass[key] = mass.get(key, 0.0) + float(np.prod([p[t, c] for t, c in enumerate(path)]))
    return mass


def test_exhaustive_fused_score_is_ctc_mass_plus_lm(tmp_path):
    lm, vocab = tiny_lm(tmp_path)
    from test_beam import rand_posteriors
    p, _ = rand_posteriors(11, 4, len(vocab), peaky=1.0, blank_boost=0.0)
    mass = brute_force(p)
    alpha, beta = 0.7, 0.4
    res = olm.prefix_beam_search_lm(p, lm, vocab, alpha, beta, beam_size=500, cutoff_prob=1.0, cutoff_top_n=len(vocab), nbest=500)
    assert len(res) == len(mass)
    for score, approx, toks in res:
        words = [vocab[c] for c in toks]
        lmsum = sum(float(lm.lnp(lm.window(words[:j]), words[j])) for j in range(len(words)))
        want = math.log(mass[tuple(toks)]) + alpha * lmsum + beta * len(toks)
        assert abs(score - want) < 1e-4 * max(1.0, abs(want)), (toks, score, want)
        S = float(lm.sentence_lnp(words))
        assert abs(approx - (score - len(toks) * beta - alpha * S)) < 1e-4 * max(1.0, abs(approx))


@pytest.mark.parametrize("seed,beam", [(1, 1), (2, 8), (3, 64)])
def test_zero_weights_without_cut_equal_the_no_lm_search(tmp_path, seed, beam):
    from masr_b200 import synth
    from test_beam import rand_posteriors
    lm = olm.read_arpa(_gen(tmp_path))
    vocab = synth.vocabulary(60)
    p, _ = rand_posteriors(seed, 40, 60)
    want = obeam.prefix_beam_search(p, beam_size=beam, cutoff_prob=0.99, cutoff_top_n=20, nbest=beam)
    got = olm.prefix_beam_search_lm(p, lm, vocab, 0.0, 0.0, beam_size=beam, cutoff_prob=0.99, cutoff_top_n=20, nbest=beam,
                                    min_cutoff=False)
    assert [(s, t) for s, _, t in got] == want
    plain = olm.prefix_beam_search_lm(p, None, vocab, beam_size=beam, cutoff_prob=0.99, cutoff_top_n=20, nbest=beam)
    assert [(s, t) for s, _, t in plain] == want and all(a == s for s, a, _ in plain)


def _gen(tmp_path):
    from masr_b200 import synth
    p = str(tmp_path / "g60.arpa")
    synth.character_lm_arpa(p, seed=4, order=3, n_chars=20, vocab_size=60)
    return p


def test_strong_alpha_flips_to_the_lm_bigram(tmp_path):
    lm, vocab = tiny_lm(tmp_path)
    # 甲, blank, then an acoustically ambiguous frame: 丙 (0.5) slightly ahead of 乙 (0.45); the LM has 甲 乙 >> 甲 丙
    p = np.full((3, len(vocab)), 1e-4, np.float32)
    p[0, 1], p[1, 0], p[2, 3], p[2, 2] = 0.9996, 0.9996, 0.5, 0.45
    p /= p.sum(1, keepdims=True)
    kw = dict(beam_size=16, cutoff_prob=1.0, cutoff_top_n=len(vocab))
    assert olm.prefix_beam_search_lm(p, None, vocab, **kw)[0][2] == [1, 3]
    assert olm.prefix_beam_search_lm(p, lm, vocab, 0.02, 0.0, **kw)[0][2] == [1, 3]
    assert olm.prefix_beam_search_lm(p, lm, vocab, 2.0, 0.0, **kw)[0][2] == [1, 2]


def test_oov_context_scores_minus_1000(tmp_path):
    lm, vocab = tiny_lm(tmp_path)
    assert lm.lnp(["丁"], "甲") == olm.OOV_SCORE == lm.lnp(["甲"], "丁")
    assert lm.lnp(["<s>"], "甲") == np.float32(-0.3 * math.log(10))
    # 丁 甲: both extensions score -1000 (the OOV word itself, then the OOV context of 甲)
    p = np.full((2, len(vocab)), 1e-3, np.float32)
    p[0, 4], p[1, 1] = 0.99, 0.99
    p /= p.sum(1, keepdims=True)
    mass = brute_force(p)
    alpha, beta = 0.01, 0.0
    res = olm.prefix_beam_search_lm(p, lm, vocab, alpha, beta, beam_size=100, cutoff_prob=1.0, cutoff_top_n=len(vocab), nbest=100)
    score = {tuple(t): s for s, _, t in res}
    assert abs(score[(4, 1)] - (math.log(mass[(4, 1)]) + alpha * -2000.0)) < 1e-4 * 20
    assert abs(score[(1,)] - (math.log(mass[(1,)]) + alpha * float(lm.lnp(["<s>"], "甲")))) < 1e-4
