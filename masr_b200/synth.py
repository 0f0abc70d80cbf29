"""Deterministic synthetic fixtures: weights, vocabulary, CMVN statistics and audio.

The reference ships no trained weights, vocabulary or golden vectors (SURVEY.md §4, §8c), so
every parity test, the smoke test and ``bench.py`` run on synthetic data that can be
regenerated bit-identically on any machine from a seed (``numpy.random.Generator`` streams
are stable across platforms).  The tensors follow the *reference's* ``state_dict`` layout
(key names and shapes probed from ``ConformerModel(...).state_dict()``, see
masr/model_utils/conformer/{model,encoder,attention,convolution,subsampling}.py), so the
very same dict can be fed to ``reference_model.load_state_dict`` (to make golden vectors in the
build container) and to :class:`masr_b200.engine.Engine` (on the GPU box).

Nothing in here depends on the reference tree or on the oracle.
"""
from __future__ import annotations

import json
import math
import os
from typing import Dict, List

import numpy as np

DEFAULT_VOCAB_SIZE = 4233  # SURVEY.md §8: WeNet AISHELL-1 unit count; a free parameter, reported with every number


def _uniform(rng, shape, bound):
    return rng.uniform(-bound, bound, size=shape).astype(np.float32)


def _linear(rng, sd, name, out_f, in_f, bias=True, gain=1.0):
    b = gain / math.sqrt(in_f)
    sd[name + ".weight"] = _uniform(rng, (out_f, in_f), b)
    if bias:
        sd[name + ".bias"] = _uniform(rng, (out_f,), b)


def _layer_norm(rng, sd, name, dim):
    # non-trivial affine parameters so a kernel that drops gamma/beta cannot pass
    sd[name + ".weight"] = (1.0 + 0.1 * rng.standard_normal(dim)).astype(np.float32)
    sd[name + ".bias"] = (0.1 * rng.standard_normal(dim)).astype(np.float32)


def cmvn_stats(seed: int = 0, dim: int = 80):
    """Synthetic global CMVN constants in the value range of real log-mel features
    (fbank of sigma=0.1 noise has mean ~20.6, std ~3.1 — SURVEY.md §8d)."""
    rng = np.random.default_rng(1000 + seed)
    mean = (20.6 + 1.5 * rng.standard_normal(dim)).astype(np.float32)
    istd = (1.0 / (3.1 * (1.0 + 0.1 * rng.uniform(-1, 1, dim)))).astype(np.float32)
    return mean, istd


def conformer_state_dict(seed: int = 0,
                         vocab_size: int = DEFAULT_VOCAB_SIZE,
                         input_dim: int = 80,
                         output_size: int = 256,
                         attention_heads: int = 4,
                         linear_units: int = 2048,
                         num_blocks: int = 12,
                         cnn_module_kernel: int = 15,
                         ctc_gain: float = 6.0,
                         blank_bias: float = 12.3) -> Dict[str, np.ndarray]:
    """Encoder + CTC-head tensors of a Conformer in the reference layout.

    ``ctc_gain`` sharpens the CTC posterior and ``blank_bias`` lifts the blank logit so the
    greedy path contains blanks and repeats (default-init posteriors are flat and never
    blank — SURVEY.md §7 "hard parts").  The attention *decoder* of the reference model
    (166 tensors) is not on the inference path and is not generated.
    """
    rng = np.random.default_rng(seed)
    d, h = output_size, attention_heads
    dk = d // h
    sd: Dict[str, np.ndarray] = {}
    mean, istd = cmvn_stats(seed, input_dim)
    sd["encoder.global_cmvn.mean"] = mean
    sd["encoder.global_cmvn.istd"] = istd
    # Conv2dSubsampling4 (conformer/subsampling.py:65-91)
    sd["encoder.embed.conv.0.weight"] = _uniform(rng, (d, 1, 3, 3), 1.0 / 3.0)
    sd["encoder.embed.conv.0.bias"] = _uniform(rng, (d,), 1.0 / 3.0)
    b2 = 1.0 / math.sqrt(d * 9)
    sd["encoder.embed.conv.2.weight"] = _uniform(rng, (d, d, 3, 3), b2)
    sd["encoder.embed.conv.2.bias"] = _uniform(rng, (d,), b2)
    f2 = ((input_dim - 1) // 2 - 1) // 2
    _linear(rng, sd, "encoder.embed.out.0", d, d * f2)
    for i in range(num_blocks):
        p = f"encoder.encoders.{i}."
        xav = math.sqrt(6.0 / (h + dk))
        sd[p + "self_attn.pos_bias_u"] = _uniform(rng, (h, dk), xav)
        sd[p + "self_attn.pos_bias_v"] = _uniform(rng, (h, dk), xav)
        for nm in ("linear_q", "linear_k", "linear_v", "linear_out"):
            _linear(rng, sd, p + "self_attn." + nm, d, d)
        _linear(rng, sd, p + "self_attn.linear_pos", d, d, bias=False)
        for ff in ("feed_forward", "feed_forward_macaron"):
            _linear(rng, sd, p + ff + ".w_1", linear_units, d)
            _linear(rng, sd, p + ff + ".w_2", d, linear_units)
        bpw = 1.0 / math.sqrt(d)
        sd[p + "conv_module.pointwise_conv1.weight"] = _uniform(rng, (2 * d, d, 1), bpw)
        sd[p + "conv_module.pointwise_conv1.bias"] = _uniform(rng, (2 * d,), bpw)
        bdw = 1.0 / math.sqrt(cnn_module_kernel)
        sd[p + "conv_module.depthwise_conv.weight"] = _uniform(rng, (d, 1, cnn_module_kernel), bdw)
        sd[p + "conv_module.depthwise_conv.bias"] = _uniform(rng, (d,), bdw)
        _layer_norm(rng, sd, p + "conv_module.norm", d)
        sd[p + "conv_module.pointwise_conv2.weight"] = _uniform(rng, (d, d, 1), bpw)
        sd[p + "conv_module.pointwise_conv2.bias"] = _uniform(rng, (d,), bpw)
        for nm in ("norm_ff", "norm_mha", "norm_ff_macaron", "norm_conv", "norm_final"):
            _layer_norm(rng, sd, p + nm, d)
    _layer_norm(rng, sd, "encoder.after_norm", d)
    _linear(rng, sd, "ctc.ctc_lo", vocab_size, d, gain=ctc_gain)
    sd["ctc.ctc_lo.bias"][0] += np.float32(blank_bias)
    return sd


def efficient_conformer_state_dict(seed: int = 0, vocab_size: int = DEFAULT_VOCAB_SIZE, blank_bias: float = 8.5,
                                   **kw) -> Dict[str, np.ndarray]:
    """EfficientConformer (configs/efficient_conformer.yml + constructor defaults): the Conformer tensors with
    pos_bias_u/v of blocks 0-3 widened to [4, 192] (grouped attention), depthwise kernel 7 in blocks 4-11, and the
    (unused at inference, concat_after=False) ``concat_linear`` of the strided block 3
    (efficient_conformer/encoder.py:124-175, attention.py:27-33)."""
    sd = conformer_state_dict(seed, vocab_size, blank_bias=blank_bias, **kw)
    rng = np.random.default_rng(500 + seed)
    d = sd["encoder.after_norm.weight"].shape[0]
    h = sd["encoder.encoders.0.self_attn.pos_bias_u"].shape[0]
    dk = d // h
    k0 = sd["encoder.encoders.0.conv_module.depthwise_conv.weight"].shape[2]
    nblocks = 1 + max(int(k.split(".")[2]) for k in sd if k.startswith("encoder.encoders."))
    for i in range(nblocks):
        p = f"encoder.encoders.{i}."
        if i <= 3:
            xav = math.sqrt(6.0 / (h + 3 * dk))
            sd[p + "self_attn.pos_bias_u"] = _uniform(rng, (h, 3 * dk), xav)
            sd[p + "self_attn.pos_bias_v"] = _uniform(rng, (h, 3 * dk), xav)
        else:
            ks = k0 // 2
            sd[p + "conv_module.depthwise_conv.weight"] = _uniform(rng, (d, 1, ks), 1.0 / math.sqrt(ks))
    _linear(rng, sd, "encoder.encoders.3.concat_linear", d, 2 * d)
    return sd


def squeezeformer_state_dict(seed: int = 0, vocab_size: int = DEFAULT_VOCAB_SIZE, streaming: bool = True, input_dim: int = 80,
                             d: int = 256, heads: int = 4, ffn: int = 2048, num_blocks: int = 12, kernel: int = 31,
                             ctc_gain: float = 6.0, blank_bias: float = None) -> Dict[str, np.ndarray]:
    """Squeezeformer tensors in the reference layout (configs/squeezeformer.yml; squeezeformer/encoder.py:20-166):
    adaptive scale/bias per sub-module, BatchNorm running statistics in the conv module, the time-reduction
    depthwise conv (kernel 1 when streaming, 5 otherwise) and the recover linear."""
    rng = np.random.default_rng(900 + seed)
    if blank_bias is None:
        blank_bias = 10.6 if streaming else 8.6
    dk = d // heads
    sd: Dict[str, np.ndarray] = {}
    mean, istd = cmvn_stats(seed, input_dim)
    sd["encoder.global_cmvn.mean"] = mean
    sd["encoder.global_cmvn.istd"] = istd
    sd["encoder.embed.pw_conv.weight"] = _uniform(rng, (d, 1, 3, 3), 1.0 / 3.0)
    sd["encoder.embed.pw_conv.bias"] = _uniform(rng, (d,), 1.0 / 3.0)
    b2 = 1.0 / math.sqrt(d * 9)
    sd["encoder.embed.dw_conv.weight"] = _uniform(rng, (d, d, 3, 3), b2)
    sd["encoder.embed.dw_conv.bias"] = _uniform(rng, (d,), b2)
    f2 = ((input_dim - 1) // 2 - 1) // 2
    _linear(rng, sd, "encoder.embed.input_proj.0", d, d * f2, gain=1.0 / math.sqrt(d) * 2)   # input is pre-scaled by sqrt(d)
    _layer_norm(rng, sd, "encoder.preln", d)

    def ada(p):
        sd[p + "ada_scale"] = (1.0 + 0.1 * rng.standard_normal((1, 1, d))).astype(np.float32)
        sd[p + "ada_bias"] = (0.1 * rng.standard_normal((1, 1, d))).astype(np.float32)

    for i in range(num_blocks):
        p = f"encoder.encoders.{i}."
        xav = math.sqrt(6.0 / (heads + dk))
        sd[p + "self_attn.pos_bias_u"] = _uniform(rng, (heads, dk), xav)
        sd[p + "self_attn.pos_bias_v"] = _uniform(rng, (heads, dk), xav)
        ada(p + "self_attn.")
        for nm in ("linear_q", "linear_k", "linear_v", "linear_out"):
            _linear(rng, sd, p + "self_attn." + nm, d, d)
        _linear(rng, sd, p + "self_attn.linear_pos", d, d, bias=False)
        for ff in ("ffn1", "ffn2"):
            ada(p + ff + ".")
            _linear(rng, sd, p + ff + ".w_1", ffn, d)
            _linear(rng, sd, p + ff + ".w_2", d, ffn)
        c = p + "conv_module."
        ada(c)
        bpw = 1.0 / math.sqrt(d)
        sd[c + "pointwise_conv1.weight"] = _uniform(rng, (2 * d, d, 1), bpw)
        sd[c + "pointwise_conv1.bias"] = _uniform(rng, (2 * d,), bpw)
        sd[c + "depthwise_conv.weight"] = _uniform(rng, (d, 1, kernel), 1.0 / math.sqrt(kernel))
        sd[c + "depthwise_conv.bias"] = _uniform(rng, (d,), 1.0 / math.sqrt(kernel))
        _layer_norm(rng, sd, c + "norm", d)                                     # BatchNorm affine
        sd[c + "norm.running_mean"] = (0.05 * rng.standard_normal(d)).astype(np.float32)
        sd[c + "norm.running_var"] = (0.1 + 0.05 * rng.uniform(0, 1, d)).astype(np.float32)
        sd[c + "norm.num_batches_tracked"] = np.array(1000, np.int64)
        sd[c + "pointwise_conv2.weight"] = _uniform(rng, (d, d, 1), bpw)
        sd[c + "pointwise_conv2.bias"] = _uniform(rng, (d,), bpw)
        for nm in ("layer_norm1", "layer_norm2", "layer_norm3", "layer_norm4"):
            _layer_norm(rng, sd, p + nm, d)
    kt = 1 if streaming else 5
    sd["encoder.time_reduction_layer.dw_conv.weight"] = _uniform(rng, (d, 1, kt), 1.0 / math.sqrt(kt))
    sd["encoder.time_reduction_layer.dw_conv.bias"] = _uniform(rng, (d,), 1.0 / math.sqrt(kt))
    sd["encoder.time_reduction_layer.pw_conv.weight"] = _uniform(rng, (d, d, 1), 1.0 / math.sqrt(d))
    sd["encoder.time_reduction_layer.pw_conv.bias"] = _uniform(rng, (d,), 1.0 / math.sqrt(d))
    _linear(rng, sd, "encoder.time_recover_layer", d, d)
    _linear(rng, sd, "ctc.ctc_lo", vocab_size, d, gain=ctc_gain)
    sd["ctc.ctc_lo.bias"][0] += np.float32(blank_bias)
    return sd


def deepspeech2_state_dict(seed: int = 0, vocab_size: int = DEFAULT_VOCAB_SIZE, streaming: bool = True, input_dim: int = 80,
                           layers: int = 5, hidden: int = 1024, ctc_gain: float = 4.0, blank_bias: float = 9.0,
                           use_gru: bool = False) -> Dict[str, np.ndarray]:
    """DeepSpeech2 tensors in the reference layout (deepspeech2/{conv,encoder,model}.py): Conv2d(1,32,3,2), Conv2d(32,32,3,2),
    5 x LSTM(1024) (+ ``_reverse`` weights when not streaming) with LayerNorm, ``decoder.ctc_lo``.  ``use_gru``: GRU(1024)
    layers instead, under the keys the reference's ``GRU`` wrapper gives them (``encoder.rnns.{l}.rnn.rnn.*``, gru.py:6-15)."""
    rng = np.random.default_rng(1300 + seed)
    sd: Dict[str, np.ndarray] = {}
    mean, istd = cmvn_stats(seed, input_dim)
    sd["encoder.global_cmvn.mean"] = mean
    sd["encoder.global_cmvn.istd"] = istd
    sd["encoder.conv.conv.0.weight"] = _uniform(rng, (32, 1, 3, 3), 1.0 / 3.0)
    sd["encoder.conv.conv.0.bias"] = _uniform(rng, (32,), 1.0 / 3.0)
    b2 = 1.0 / math.sqrt(32 * 9)
    sd["encoder.conv.conv.2.weight"] = _uniform(rng, (32, 32, 3, 3), b2)
    sd["encoder.conv.conv.2.bias"] = _uniform(rng, (32,), b2)
    f2 = ((input_dim - 1) // 2 - 1) // 2
    dirs = 1 if streaming else 2
    insz = 32 * f2
    k = 1.0 / math.sqrt(hidden)
    gates = 3 if use_gru else 4
    for l in range(layers):
        p = f"encoder.rnns.{l}.rnn." + ("rnn." if use_gru else "")
        for suf in ("", "_reverse")[:dirs]:
            sd[p + "weight_ih_l0" + suf] = _uniform(rng, (gates * hidden, insz), k)
            sd[p + "weight_hh_l0" + suf] = _uniform(rng, (gates * hidden, hidden), k)
            sd[p + "bias_ih_l0" + suf] = _uniform(rng, (gates * hidden,), k)
            sd[p + "bias_hh_l0" + suf] = _uniform(rng, (gates * hidden,), k)
        _layer_norm(rng, sd, f"encoder.rnns.{l}.layer_norm", hidden * dirs)
        insz = hidden * dirs
    _linear(rng, sd, "decoder.ctc_lo", vocab_size, hidden * dirs, gain=ctc_gain)
    sd["decoder.ctc_lo.bias"][0] += np.float32(blank_bias)
    return sd


def vocabulary(vocab_size: int = DEFAULT_VOCAB_SIZE) -> List[str]:
    """``<blank>``, ``<unk>``, CJK code points…, one ``<space>``, ``<eos>`` last — the order
    the reference's ``create_data`` writes (masr/trainer.py:480-488)."""
    toks = ["<blank>", "<unk>"]
    n_mid = vocab_size - 3
    toks += [chr(0x4E00 + i) for i in range(n_mid - 1)]
    toks += ["<space>"]
    toks += ["<eos>"]
    assert len(toks) == vocab_size
    return toks


def write_vocabulary(path: str, vocab_size: int = DEFAULT_VOCAB_SIZE):
    """One ``token\\tcount`` per line, line index == id (text_featurizer.py:52-59)."""
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    with open(path, "w", encoding="utf-8") as f:
        for i, t in enumerate(vocabulary(vocab_size)):
            f.write(f"{t}\t{max(1, vocab_size - i)}\n")


def write_mean_istd(path: str, seed: int = 0, dim: int = 80):
    """``{"mean": [...], "istd": [...], "feature_method": ...}`` (normalizer.py:88-92)."""
    mean, istd = cmvn_stats(seed, dim)
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    with open(path, "w", encoding="utf-8") as f:
        json.dump({"mean": [float(v) for v in mean], "istd": [float(v) for v in istd],
                   "feature_method": "fbank"}, f)


def character_lm_arpa(path: str, seed: int = 0, order: int = 3, n_chars: int = 60, n_sentences: int = 400,
                      max_len: int = 20, vocab_size: int = DEFAULT_VOCAB_SIZE, discount: float = 0.5, branch: int = 4):
    """Write a character n-gram LM as ARPA with lmplz conventions and return its character list.

    A corpus of ``n_sentences`` sentences is sampled from a random first-order Markov chain over ``n_chars`` characters
    of the synthetic CJK vocabulary (each character has ``branch`` likely successors); the rest of the vocabulary is left
    out of the LM, so decoding with it exercises the out-of-vocabulary rule.  The model is a backoff model with absolute discounting D:
      unigrams  P(w) = (c(w) + 1) / (N + |W|) over W = characters + </s> + <unk>  (<s> is written with log10 p = -99)
      n >= 2    P(w | h) = (c(h w) - D) / c(h) for seen (h, w); otherwise bo(h) P(w | h[1:]) with
                bo(h) = (D N1+(h .) / c(h)) / (1 - sum over seen w of P(w | h[1:]))
    so every P(. | h) sums to 1.  Backoffs are written only on n-grams that prefix a longer one, as lmplz does.
    Sentences are ``<s> c1 .. cm </s>``."""
    rng = np.random.default_rng(seed)
    cjk = vocabulary(vocab_size)[2:-2]
    assert n_chars < len(cjk)
    pick = rng.permutation(len(cjk))[:n_chars]
    chars = [cjk[i] for i in sorted(pick)]
    succ = rng.integers(0, n_chars, (n_chars, branch))
    weights = rng.dirichlet(np.ones(branch))
    sents = []
    for _ in range(n_sentences):
        m = int(rng.integers(1, max_len + 1))
        s = [int(rng.integers(0, n_chars))]
        for _ in range(m - 1):
            s.append(int(succ[s[-1], rng.choice(branch, p=weights)]) if rng.random() < 0.85 else int(rng.integers(0, n_chars)))
        sents.append(["<s>"] + [chars[i] for i in s] + ["</s>"])
    _write_backoff_arpa(path, sents, chars + ["</s>", "<unk>"], order, discount)
    return chars


def _write_backoff_arpa(path: str, sents, words, order: int, discount: float, extra_unigrams=()):
    """An absolute-discounting backoff LM of ``sents`` (lists ``<s> .. </s>``) over the unigram set ``words``, written as
    ARPA with lmplz conventions (see character_lm_arpa).  ``extra_unigrams``: words appended to the unigram section, each
    with the probability of an unseen word (the unigram distribution then no longer sums to 1)."""
    counts: List[Dict[tuple, int]] = [dict() for _ in range(order + 1)]
    for s in sents:
        for n in range(1, order + 1):
            for i in range(len(s) - n + 1):
                g = tuple(s[i:i + n])
                if g[-1] == "<s>":
                    continue
                counts[n][g] = counts[n].get(g, 0) + 1
    N = sum(counts[1].values())
    prob: List[Dict[tuple, float]] = [dict() for _ in range(order + 1)]
    for w in words:
        prob[1][(w,)] = (counts[1].get((w,), 0) + 1) / (N + len(words))
    ctx_total: List[Dict[tuple, list]] = [dict() for _ in range(order + 1)]   # h -> [c(h), N1+(h .), seen lower mass]
    for n in range(2, order + 1):
        for g, c in counts[n].items():
            e = ctx_total[n - 1].setdefault(g[:-1], [0, 0, 0.0])
            e[0] += c
            e[1] += 1
        for g, c in counts[n].items():
            h = g[:-1]
            prob[n][g] = (c - discount) / ctx_total[n - 1][h][0]
            ctx_total[n - 1][h][2] += prob[n - 1][g[1:]]          # (h[1:], w) is a sub-n-gram, so it is stored
    backoff: Dict[tuple, float] = {}
    for n in range(1, order):
        for h, (ch, n1p, lower) in ctx_total[n].items():
            backoff[h] = (discount * n1p / ch) / (1.0 - lower)
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    grams = [None] + [sorted(prob[n]) for n in range(1, order + 1)]
    grams[1] = [("<s>",)] + grams[1] + [(w,) for w in extra_unigrams]
    with open(path, "w", encoding="utf-8") as f:
        f.write("\\data\\\n")
        for n in range(1, order + 1):
            f.write(f"ngram {n}={len(grams[n])}\n")
        for n in range(1, order + 1):
            f.write(f"\n\\{n}-grams:\n")
            for g in grams[n]:
                p = -99.0 if g == ("<s>",) else math.log10(prob[n][g] if g in prob[n] else 1.0 / (N + len(words)))
                line = f"{p:.8g}\t{' '.join(g)}"
                if n < order and g in backoff:
                    line += f"\t{math.log10(backoff[g]):.8g}"
                f.write(line + "\n")
        f.write("\n\\end\\\n")


ENGLISH_LETTERS = "abcdefghijklmnopqrstuvwxyz'"


def english_vocabulary() -> List[str]:
    """``<blank>``, ``<unk>``, a-z, ``'``, ``<space>``: the vocabulary of an English character model (30 tokens; ' ' is
    written as ``<space>``, as TextFeaturizer does)."""
    return ["<blank>", "<unk>"] + list(ENGLISH_LETTERS) + ["<space>"]


def _letters(i: int) -> str:
    s = ""
    while True:
        s = ENGLISH_LETTERS[i % 26] + s
        i = i // 26 - 1
        if i < 0:
            return s


def word_lm_arpa(path: str, seed: int = 0, order: int = 3, n_words: int = 200, n_sentences: int = 600, max_len: int = 12,
                 discount: float = 0.5, branch: int = 4, extra_unigrams: int = 0) -> List[str]:
    """Write a word n-gram LM as ARPA with lmplz conventions (the model of character_lm_arpa over words) and return its
    corpus words.  The words are random a-z / ' strings; a fifth of them also occur without their last letter, so some
    words are prefixes of others; four are not spellable with ``english_vocabulary()`` (a digit, an upper-case letter,
    an accented letter, a '-') and stay in the corpus, so their n-grams exist but no hypothesis can reach them.
    ``extra_unigrams``: that many more spellable unigrams (unseen in the corpus; e.g. > 65536 for the 24-bit word ids)."""
    rng = np.random.default_rng(seed)
    words: List[str] = []
    seen = set()
    while len(words) < n_words:
        w = "".join(ENGLISH_LETTERS[i] for i in rng.integers(0, 26, int(rng.integers(1, 8))))
        if rng.random() < 0.05 and len(w) > 2:
            w = w[:2] + "'" + w[2:]
        if w not in seen:
            seen.add(w)
            words.append(w)
    for w in list(words[:n_words // 5]):
        if len(w) >= 2 and w[:-1] not in seen:
            seen.add(w[:-1])
            words.append(w[:-1])
    words += ["abc1", "Hello", "café", "x-ray"]
    n = len(words)
    succ = rng.integers(0, n, (n, branch))
    weights = rng.dirichlet(np.ones(branch))
    sents = []
    for _ in range(n_sentences):
        m = int(rng.integers(1, max_len + 1))
        s = [int(rng.integers(0, n))]
        for _ in range(m - 1):
            s.append(int(succ[s[-1], rng.choice(branch, p=weights)]) if rng.random() < 0.85 else int(rng.integers(0, n)))
        sents.append(["<s>"] + [words[i] for i in s] + ["</s>"])
    extra = [f"qq'{_letters(i)}" for i in range(extra_unigrams)]
    _write_backoff_arpa(path, sents, words + ["</s>", "<unk>"], order, discount, extra)
    return words


def noise_audio(seed: int, num_samples: int, sigma: float = 0.1) -> np.ndarray:
    """BASELINE.md §5 synthetic input: ``0.1 * standard_normal`` float32 (RMS ~ -20 dB)."""
    rng = np.random.default_rng(seed)
    return (sigma * rng.standard_normal(num_samples)).astype(np.float32)


def speechlike_audio(seed: int, num_samples: int, sample_rate: int = 16000) -> np.ndarray:
    """A non-stationary test signal: gliding harmonics under a syllable-rate envelope plus a
    noise floor, so successive encoder frames differ and the greedy path varies."""
    rng = np.random.default_rng(7000 + seed)
    t = np.arange(num_samples, dtype=np.float64) / sample_rate
    f0 = 110.0 + 60.0 * np.sin(2 * np.pi * 0.7 * t + rng.uniform(0, 6.28))
    phase = 2 * np.pi * np.cumsum(f0) / sample_rate
    sig = np.zeros(num_samples)
    for k in range(1, 12):
        fk = rng.uniform(0.3, 1.0) / k
        sig += fk * np.sin(k * phase + rng.uniform(0, 6.28)) * (0.6 + 0.4 * np.sin(2 * np.pi * rng.uniform(0.5, 3.0) * t))
    env = 0.5 * (1 + np.sin(2 * np.pi * rng.uniform(2.5, 4.5) * t + rng.uniform(0, 6.28)))
    env = env ** 2
    sig = sig * env * 0.08 + 0.004 * rng.standard_normal(num_samples)
    return sig.astype(np.float32)


def to_torch(sd: Dict[str, np.ndarray]):
    import torch
    return {k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in sd.items()}
