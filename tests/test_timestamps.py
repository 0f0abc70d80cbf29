"""CPU: token and word times — greedy frame spans, the beam restatements' token onsets and masr_b200/timestamps.py,
including predict_long's sentence assembly over a scripted VAD."""
import glob
import math
import os

import numpy as np
import pytest

from conftest import GOLDEN
from masr_b200 import synth, timestamps as ts
from oracle import beam as obeam, lm as olm, word_lm as owl
import beam_onsets as bo

F = np.float32


def spans_loop(ids, blank=0):
    """The greedy spans stated frame by frame: a non-blank id that differs from the previous frame's starts a token, the
    same id continues the last token's run."""
    out, prev = [], None
    for t, i in enumerate(int(x) for x in ids):
        if i != blank and i == prev:
            out[-1][2] = t + 1
        elif i != blank:
            out.append([i, t, t + 1])
        prev = i
    return [o[0] for o in out], [o[1] for o in out], [o[2] for o in out]


def golden_ids():
    out = []
    for path in sorted(glob.glob(os.path.join(GOLDEN, "*_golden.npz"))):
        z = np.load(path)
        out += [(os.path.basename(path), k, z[k]) for k in z.files if k.endswith("/ids")]
    return out


def test_greedy_spans_of_every_golden_family():
    cases = golden_ids()
    fams = {name for name, _, _ in cases}
    assert {"conformer_golden.npz", "efficient_golden.npz", "squeezeformer_golden.npz", "deepspeech2_golden.npz"} <= fams
    for name, key, ids in cases:
        toks, s, e = ts.greedy_spans(ids)
        assert (toks, s, e) == spans_loop(ids), (name, key)
        collapsed = [int(i) for j, i in enumerate(ids) if i != 0 and (j == 0 or ids[j - 1] != i)]
        assert toks == collapsed, (name, key)
        assert all(a < b for a, b in zip(s, e)) and all(b <= a for a, b in zip(s[1:], e[:-1]))


@pytest.mark.parametrize("ids,want", [
    ([5, 5, 0, 3], ([5, 3], [0, 3], [2, 4])),                 # runs at the first and the last frame
    ([0, 4, 4, 0, 4, 0], ([4, 4], [1, 4], [3, 5])),           # a repeat split by a blank is two tokens
    ([7, 8, 8, 7], ([7, 8, 7], [0, 1, 3], [1, 3, 4])),        # adjacent runs of different tokens
    ([0, 0, 0], ([], [], [])),                                # all blank
    ([], ([], [], [])),
    ([9], ([9], [0], [1])),
])
def test_greedy_span_edges(ids, want):
    assert ts.greedy_spans(np.asarray(ids, np.int32)) == want == spans_loop(ids)


# ---- the restatements' onsets -----------------------------------------------------------------------------------------
def peaky_frames(seed, T, ids, k=3, conc=0.5):
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(T):
        pick = [int(c) for c in rng.choice(ids, k, replace=False)]
        out.append([(c, F(math.log(p))) for c, p in zip(pick, rng.dirichlet(np.ones(k) * conc))])
    return out


@pytest.fixture(scope="module")
def lms(tmp_path_factory):
    d = tmp_path_factory.mktemp("ts_lm")
    vocab = synth.vocabulary()
    cp = str(d / "c3.arpa")
    chars = synth.character_lm_arpa(cp, seed=5, order=3, n_chars=12, n_sentences=300)
    cids = [vocab.index(c) for c in chars][:4]
    wvocab = synth.english_vocabulary()
    wp = str(d / "w2.arpa")
    synth.word_lm_arpa(wp, seed=2, order=2, n_words=40)
    return vocab, olm.read_arpa(cp), [0, 1] + cids, wvocab, owl.WordLM(wp, wvocab)


def word_frames(seed, wvocab, wlm, T):
    """Frames that spell lexicon words separated by <space>: the spelled token, blank and a random letter per frame."""
    rng = np.random.default_rng(seed)
    words = [w for w in wlm.lex.words if w.isalpha()]
    spell = []
    while len(spell) < T:
        spell += [wvocab.index(c) for c in words[rng.integers(len(words))]] + [wlm.space]
    out, i = [], 0
    for _ in range(T):
        other = int(rng.integers(2, 28))
        p = rng.dirichlet([3.0, 1.5, 1.0])
        out.append([(spell[i], F(math.log(p[0]))), (0, F(math.log(p[1])))] + ([(other, F(math.log(p[2])))] if other != spell[i] else []))
        i += int(rng.random() < 0.6)
    return out


def mode_frames(mode, lms, seed, T):
    _, _, cids, wvocab, wlm = lms
    if mode == "word":
        return word_frames(seed, wvocab, wlm, T)
    return peaky_frames(seed, T, cids if mode == "char" else [0, 1, 2, 3, 4])


def search_kw(mode, lms):
    vocab, clm, _, _, wlm = lms
    return {"plain": {}, "char": dict(lm=clm, vocab=vocab, alpha=0.6, beta=0.4), "word": dict(lm=wlm, alpha=0.6, beta=0.4)}[mode]


@pytest.mark.parametrize("mode", ["plain", "char", "word"])
def test_onsets_increase_along_every_prefix(lms, mode):
    """Every prefix of every frame's beam: its tokens' onsets strictly increase and the last is the frame it entered the
    beam; the reported prefix is the restatement's one-shot result."""
    checked = 0
    for seed in range(3):
        frames = mode_frames(mode, lms, seed, 24)
        blps = [F(-1.0)] * len(frames)
        for beam in (2, 8):
            per_frame, best = bo.beams(mode, frames, blps, beam, **search_kw(mode, lms))
            first = bo.first_frames(per_frame)
            for t, bm in enumerate(per_frame):
                for p in bm:
                    fr = bo.onsets(per_frame, p)
                    assert all(a < b for a, b in zip(fr, fr[1:])), (p, fr)
                    assert not p or fr[-1] == first[p] <= t
                    checked += len(fr)
            kw = search_kw(mode, lms)
            if mode == "plain":
                want = obeam.prefix_beam_search(np.zeros((len(frames), 1)), beam_size=beam, cands_per_frame=frames)[0][1]
            elif mode == "char":
                want = olm.prefix_beam_search_lm(np.zeros((len(frames), 1)), kw["lm"], kw["vocab"], 0.6, 0.4, beam_size=beam,
                                                 cands_per_frame=frames, blank_logp_per_frame=blps)[0][2]
            else:
                want = (owl.prefix_beam_search_wordlm(kw["lm"], frames, blps, 0.6, 0.4, beam_size=beam) or [(0, 0, [])])[0][2]
            assert best == list(want)
    assert checked > 300


def test_word_search_beams_do_not_depend_on_the_chunking(lms):
    """The word-LM search pushed one frame at a time holds, after every frame, the beam of one push of all frames so far —
    and pushed in chunks of 7 and 64 the same beam at every chunk end: the per-frame beams, hence the onsets, are those of
    the one-shot search."""
    _, _, _, _, wlm = lms
    frames = mode_frames("word", lms, 0, 130)
    blps = [F(-1.0)] * len(frames)
    per_frame, best = bo.beams("word", frames, blps, 16, lm=wlm, alpha=0.6, beta=0.4)
    for t in (0, 1, 6, 40, 129):
        s = owl.WordLmSearch(wlm, 0.6, 0.4, 16).push(frames[:t + 1], blps[:t + 1])
        assert [tuple(s.toks_of[n]) for n, _, _ in s.beam] == per_frame[t], t
    for chunk in (7, 64):
        s = owl.WordLmSearch(wlm, 0.6, 0.4, 16)
        for t0 in range(0, len(frames), chunk):
            s.push(frames[t0:t0 + chunk], blps[t0:t0 + chunk])
            t = min(t0 + chunk, len(frames)) - 1
            assert [tuple(s.toks_of[n]) for n, _, _ in s.beam] == per_frame[t], (chunk, t)
    assert len(best) > 2 and bo.onsets(per_frame, best) == sorted(set(bo.onsets(per_frame, best)))


def test_a_prefix_that_leaves_the_beam_and_returns_keeps_its_first_onset():
    per_frame = [[(), (4,)], [(), (1,)], [(), (2,)], [(1,), (1, 3)], [(1, 3), (4,)]]
    assert bo.onsets(per_frame, (1, 3)) == [1, 3]
    assert bo.onsets(per_frame, (4,)) == [0]
    # and such returns happen in the restated search over peaky frames at beam 3
    returns = 0
    for seed in range(3):
        per_frame, _ = bo.beams("plain", peaky_frames(seed, 30, [0, 1, 2, 3], conc=0.5), beam=3)
        last = {}
        for t, bm in enumerate(per_frame):
            for p in bm:
                returns += p in last and last[p] < t - 1
                last[p] = t
    assert returns > 0


def test_frames_readout_rejects_bad_arguments():
    """masr_ctc_prefix_beam_frames refuses null pointers and a trie too small for one node before launching anything;
    B = 0 is a no-op (the library cross-compiles for sm_90a without a GPU)."""
    from masr_b200 import _lib, build
    build.build()
    buf = np.zeros(64, np.int32)
    p = buf.ctypes.data
    _lib.call("masr_ctc_prefix_beam_frames", p, p, 100, p, 8, p, 0, p, 8, None)
    with pytest.raises(_lib.MasrB200Error, match="null pointer"):
        _lib.call("masr_ctc_prefix_beam_frames", p, p, 100, None, 8, p, 1, p, 8, None)
    with pytest.raises(_lib.MasrB200Error, match="trie_cap=4 out of range"):
        _lib.call("masr_ctc_prefix_beam_frames", p, p, 4, p, 8, p, 1, p, 8, None)
    assert buf.tolist() == [0] * 64


# ---- timestamps.py ----------------------------------------------------------------------------------------------------
def test_frame_clock_per_family():
    from masr_b200.deepspeech2 import DeepSpeech2Engine
    from masr_b200.engine import ConformerEngine, EfficientConformerEngine
    from masr_b200.squeezeformer import SqueezeformerEngine
    for cls, dt in ((ConformerEngine, 0.04), (SqueezeformerEngine, 0.04), (DeepSpeech2Engine, 0.04),
                    (EfficientConformerEngine, 0.08)):
        assert ts.frame_seconds(object.__new__(cls)) == pytest.approx(dt, abs=1e-12), cls.__name__
    toks = ts.token_times([2, 3], [1, 250], [2, 252], ["<blank>", "<unk>", "a", "b"], 0.04, offset=1.25)
    assert toks == [{'token': 'a', 'start': 1.29, 'end': 1.33}, {'token': 'b', 'start': 11.25, 'end': 11.33}]


def test_word_grouping():
    vocab = ["<blank>", "<unk>", "<space>", "h", "i", "y", "o"]
    r = ts.attach({}, [3, 4, 2, 5, 6, 2], [0, 2, 4, 6, 9, 12], [1, 3, 5, 7, 10, 13], vocab, 0.04)
    assert [t['token'] for t in r['tokens']] == ["h", "i", "<space>", "y", "o", "<space>"]
    assert r['words'] == [{'word': 'hi', 'start': 0.0, 'end': 0.12}, {'word': 'yo', 'start': 0.24, 'end': 0.4}]
    r = ts.attach({}, [2, 2, 3, 2], [0, 1, 2, 3], [1, 2, 3, 4], vocab, 0.04)         # leading / repeated <space>, last word
    assert r['words'] == [{'word': 'h', 'start': 0.08, 'end': 0.12}]
    r = ts.beam_result({}, [3, 4], [5, 9], vocab[:2] + ["x", "h", "i"], 0.08)          # no <space>: tokens only
    assert r == {'tokens': [{'token': 'h', 'start': 0.4, 'end': 0.48}, {'token': 'i', 'start': 0.72, 'end': 0.8}]}


class _ScriptedVAD:
    def __init__(self, stamps):
        self.stamps = stamps

    def get_speech_timestamps(self, samples, sr):
        return [dict(s) for s in self.stamps]


class _FakeEngine:
    """Greedy ``transcribe`` with frame ids derived from each waveform's length (as the real engine: one id per 640
    samples), so a segment's spans are known in advance."""
    device = "cpu"

    @staticmethod
    def ids(n):
        T = n // 640
        return np.asarray([(0, 5, 5, 0, 6, 7, 7, 7)[(t + n // 3200) % 8] for t in range(T)], np.int32)

    def transcribe(self, waves, use_db, target_db, return_frames=False, rates=None):
        from masr_b200.engine import GreedyResult
        ids = [self.ids(len(w)) for w in waves]
        T = max(len(i) for i in ids)
        fid = np.zeros((len(waves), T), np.int32)
        for b, i in enumerate(ids):
            fid[b, :len(i)] = i
        toks = [ts.greedy_spans(i)[0] for i in ids]
        return GreedyResult(toks, [float(len(t)) for t in toks], fid if return_frames else None,
                            np.asarray([len(i) for i in ids], np.int32), np.zeros(len(waves), np.int32))


def test_predict_long_sentences_with_a_scripted_vad():
    from masr_b200.predict import MASRPredictor
    from masr_b200.text import TextFeaturizer
    p = object.__new__(MASRPredictor)
    vocab = ["<blank>", "<unk>", "<space>", "d", "e", "a", "b", "c"]
    p._text_featurizer = object.__new__(TextFeaturizer)
    p._text_featurizer._vocab_list = vocab
    p._beam_conf, p._sample_rate, p._resample, p._use_db, p._target_db = None, 16000, False, True, -20.0
    p.predictor = _FakeEngine()
    stamps = [{'start': 1000, 'end': 20000}, {'start': 30001, 'end': 30500}, {'start': 41234, 'end': 90000}]
    vad = _ScriptedVAD(stamps)
    audio = np.zeros(100000, np.float32)
    plain = p.predict_long(audio, vad_predictor=vad)
    timed = p.predict_long(audio, vad_predictor=vad, timestamps=True)
    assert {k: timed[k] for k in ('text', 'score')} == plain and set(timed) == {'text', 'score', 'sentences'}
    sents = timed['sentences']
    assert len(sents) == 2                                   # the 499-sample segment has no frame: no text, no sentence
    for sent, st in zip(sents, (stamps[0], stamps[2])):
        assert (sent['start'], sent['end']) == (round(st['start'] / 16000, 3), round(st['end'] / 16000, 3))
        toks, s, e = spans_loop(_FakeEngine.ids(st['end'] - st['start']))
        assert sent['text'] == ''.join(vocab[t] for t in toks).replace('<space>', ' ')
        assert sent['tokens'] == [{'token': vocab[t], 'start': round(st['start'] / 16000 + a * 0.04, 3),
                                   'end': round(st['start'] / 16000 + b * 0.04, 3)} for t, a, b in zip(toks, s, e)]
        assert sent['start'] <= sent['tokens'][0]['start'] and sent['tokens'][-1]['end'] <= sent['end'] + 0.04
        assert sent['words'] == ts.word_times(sent['tokens'])
    assert plain['text'] == '，'.join(s['text'] for s in sents)
