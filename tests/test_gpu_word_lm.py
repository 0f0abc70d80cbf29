"""GPU (-m gpu): word n-gram LM fusion with the lexicon constraint — the query kernel against oracle/word_lm.py, the fused
search (one-shot, streaming, stream-pool slots) against the restatement bit for bit, and MASRPredictor with an English
vocabulary and a word ARPA file."""
import ctypes as C

import numpy as np
import pytest
import torch

from masr_b200.text import ids_to_text
from oracle import word_lm as owl
from test_beam import rand_posteriors

pytestmark = pytest.mark.gpu
F = np.float32


@pytest.fixture(scope="module")
def wlms(tmp_path_factory):
    from masr_b200 import synth
    from masr_b200.lm import WordLM
    vocab = synth.english_vocabulary()
    out = {}
    for key, order, extra in ((3, 3, 0), (5, 5, 0), ("big", 3, 70_000)):
        p = str(tmp_path_factory.mktemp("wlm") / f"{key}.arpa")
        synth.word_lm_arpa(p, seed=order, order=order, n_words=120, extra_unigrams=extra)
        out[key] = (owl.WordLM(p, vocab), WordLM(p, vocab), p)
    return vocab, out


def dev_stream():
    return torch.device("cuda", torch.cuda.current_device()), torch.cuda.current_stream().cuda_stream


@pytest.mark.parametrize("key", [3, 5, "big"])
def test_word_query_kernel_equals_oracle(wlms, key):
    vocab, d = wlms
    o, w, _ = d[key]
    order = o.order
    rng = np.random.default_rng(7)
    Q = 100_000
    n = o.dict_size
    if key == "big":
        assert n > 65_536
    names = o.lex.words + ["<s>", "</s>"]
    corpus = [i for i, x in enumerate(o.lex.words) if not x.startswith("qq'")]     # words with n-grams beyond unigrams
    pool = np.array(corpus + [n, n + 1, -1, n - 1], np.int64)
    prob = np.r_[np.full(len(corpus), 0.9 / len(corpus)), np.full(4, 0.1 / 4)]
    ctx = rng.choice(pool, (Q, order - 1), p=prob)
    pad = rng.integers(0, order, Q)
    for j in range(order - 1):
        ctx[pad > j, j] = n
    word = rng.choice(pool, Q, p=prob)
    got = w.score(ctx, word)
    from masr_b200 import _lib                                         # the entry point WordLM.score wraps, called by name
    dev, st = dev_stream()
    c_d = torch.as_tensor(ctx[:1000].astype(np.int32)).to(dev).contiguous()
    w_d = torch.as_tensor(word[:1000].astype(np.int32)).to(dev)
    out = torch.full((1000,), float("nan"), device=dev)
    _lib.call("masr_word_lm_score_f32", C.byref(w.tables(dev)), c_d.data_ptr(), w_d.data_ptr(), 1000, out.data_ptr(), st)
    assert np.array_equal(out.cpu().numpy().view(np.int32), got[:1000].view(np.int32))
    name =lambda i: names[i] if i >= 0 else "<oov>"
    want = np.array([o.lnp([name(t) for t in ctx[q]], name(word[q])) for q in range(Q)], np.float32)
    assert np.array_equal(got.view(np.int32), want.view(np.int32)), np.flatnonzero(got != want)[:10]
    assert (want == -1000).any() and (want > -1000).mean() > 0.3


def topk(logits, V, top_n=40, cut=0.99):
    from masr_b200 import _lib
    dev = logits.device
    M = logits.shape[0]
    cid = torch.zeros(M, 40, dtype=torch.int32, device=dev); clp = torch.zeros(M, 40, device=dev)
    cn = torch.zeros(M, dtype=torch.int32, device=dev); blp = torch.zeros(M, device=dev)
    if M:
        _lib.call("masr_ctc_topk_blank_f32", logits.data_ptr(), logits.stride(0), M, V, top_n, cut, 0, cid.data_ptr(),
                  clp.data_ptr(), cn.data_ptr(), blp.data_ptr(), torch.cuda.current_stream().cuda_stream)
    return cid, clp, cn, blp


def host_cands(cid, clp, cn, blp, rows):
    cid_h, clp_h, cn_h, blp_h = cid.cpu().numpy(), clp.cpu().numpy(), cn.cpu().numpy(), blp.cpu().numpy()
    return [[(int(cid_h[r, k]), clp_h[r, k]) for k in range(cn_h[r])] for r in rows], [blp_h[r] for r in rows]


def wl_logits(seed, T, o, dev):
    """rand_posteriors logits with the lexicon's letters and <space> lifted, so the search extends with words."""
    V = len(o.vocab)
    _, logits = rand_posteriors(seed, T, V, peaky=3.0)
    letters = sorted({t for ch in o.lex.child for t in ch})
    logits[:, letters] += 1.0
    logits[:, o.space] += 2.0
    L = torch.zeros(T, 32, device=dev)
    L[:, :V] = torch.from_numpy(logits).to(dev)
    return L


def workspace(B, T):
    from masr_b200 import _lib
    dev, _ = dev_stream()
    pool_n, trie_n = C.c_int64(0), C.c_int64(0)
    _lib.call("masr_ctc_prefix_beam_workspace", B, T, C.byref(pool_n), C.byref(trie_n))
    return (torch.empty(pool_n.value, device=dev), torch.empty(B * trie_n.value, dtype=torch.int32, device=dev),
            torch.empty(B * trie_n.value, dtype=torch.int32, device=dev), trie_n.value)


def one_shot(w, cid, clp, cn, blp, bstride, lens, beam, alpha, beta):
    from masr_b200 import _lib
    dev, st = dev_stream()
    B, T = len(lens), max(lens)
    pool, tp, tt, cap = workspace(B, T)
    ld = torch.tensor(lens, dtype=torch.int32, device=dev)
    otok = torch.zeros(B, T, dtype=torch.int32, device=dev); on = torch.zeros(B, dtype=torch.int32, device=dev)
    osc, oap = torch.zeros(B, device=dev), torch.zeros(B, device=dev)
    _lib.call("masr_ctc_prefix_beam_wordlm", cid.data_ptr(), clp.data_ptr(), cn.data_ptr(), blp.data_ptr(), bstride, ld.data_ptr(),
              B, beam, 0, C.byref(w.tables(dev)), alpha, beta, pool.data_ptr(), tp.data_ptr(), tt.data_ptr(), cap, otok.data_ptr(), T,
              on.data_ptr(), osc.data_ptr(), oap.data_ptr(), st)
    torch.cuda.synchronize()
    return [(otok[b, :on[b].item()].cpu().tolist(), F(osc[b].item()), F(oap[b].item())) for b in range(B)]


@pytest.mark.parametrize("key,seed,T,beam,cut,alpha,beta", [
    (3, 1, 60, 300, 0.99, 1.0, 2.0), (3, 2, 45, 16, 1.0, 0.8, -0.5), (5, 3, 60, 500, 1.0, 1.0, 1.5), (5, 4, 40, 1, 0.99, 2.2, 4.3),
    (3, 5, 50, 16, 0.99, 0.5, 0.0), (3, 6, 70, 300, 0.99, 0.0, 0.0), (5, 7, 80, 500, 0.99, 0.6, -1.0),
    ("big", 8, 60, 300, 0.99, 1.2, 0.7)])
def test_gpu_wordlm_beam_equals_restatement(wlms, key, seed, T, beam, cut, alpha, beta):
    vocab, d = wlms
    o, w, _ = d[key]
    dev, _ = dev_stream()
    lens = [T, T // 2]
    L = torch.cat([wl_logits(seed, T, o, dev), wl_logits(seed + 100, T, o, dev)])
    cid, clp, cn, blp = topk(L, len(vocab), 40, cut)
    got = one_shot(w, cid, clp, cn, blp, T, lens, beam, alpha, beta)
    spaces = 0
    for b in range(2):
        cands, blps = host_cands(cid, clp, cn, blp, range(b * T, b * T + lens[b]))
        (score, approx, toks), = owl.prefix_beam_search_wordlm(o, cands, blps, alpha, beta, beam_size=beam)
        assert got[b][0] == toks, (b, got[b][0], toks)
        assert got[b][1] == F(score), (b, got[b][1], score)
        assert got[b][2] == F(approx), (b, got[b][2], approx)
        for word in ids_to_text(toks, vocab).split(" ")[:-1]:
            assert word in o.lex.word_id
        spaces += toks.count(o.space)
    assert spaces > 0


@pytest.mark.parametrize("key,seed,T,beam,chunks", [(3, 11, 75, 300, (16, 7)), (5, 12, 50, 32, (5, 13))])
def test_gpu_wordlm_streaming_equals_one_shot(wlms, key, seed, T, beam, chunks):
    from masr_b200 import _lib
    vocab, d = wlms
    o, w, _ = d[key]
    dev, st = dev_stream()
    cid, clp, cn, blp = topk(wl_logits(seed, T, o, dev), len(vocab))
    alpha, beta = 1.0, 1.5
    si, sf = C.c_int64(0), C.c_int64(0)
    _lib.call("masr_ctc_prefix_beam_wordlm_state_size", C.byref(si), C.byref(sf))
    for chunk in chunks:
        pool, tp, tt, cap = workspace(1, T)
        otok = torch.zeros(1, T, dtype=torch.int32, device=dev); on = torch.zeros(1, dtype=torch.int32, device=dev)
        osc, oap = torch.zeros(1, device=dev), torch.zeros(1, device=dev)
        sti = torch.zeros(si.value, dtype=torch.int32, device=dev); stf = torch.zeros(sf.value, device=dev)
        done = 0
        while done < T:
            n = min(chunk, T - done)
            ld = torch.tensor([n], dtype=torch.int32, device=dev)
            _lib.call("masr_ctc_prefix_beam_wordlm_stream", cid[done:].data_ptr(), clp[done:].data_ptr(), cn[done:].data_ptr(),
                      blp[done:].data_ptr(), T, ld.data_ptr(), 1, beam, 0, C.byref(w.tables(dev)), alpha, beta, pool.data_ptr(),
                      tp.data_ptr(), tt.data_ptr(), cap, sti.data_ptr(), stf.data_ptr(), 1 if done else 0, otok.data_ptr(), T,
                      on.data_ptr(), osc.data_ptr(), oap.data_ptr(), st)
            done += n
            got = (otok[0, :on.item()].cpu().tolist(), F(osc.item()), F(oap.item()))
            assert got == one_shot(w, cid, clp, cn, blp, T, [done], beam, alpha, beta)[0], (chunk, done)


def test_gpu_wordlm_pool_slots_equal_restatement(wlms):
    """Three slots pushed unevenly (a slot idle in some pushes, one reset mid-way): after every push each active slot
    equals the restatement over its frames since its reset; an idle slot's state, trie and outputs stay byte for byte."""
    from masr_b200 import _lib
    vocab, d = wlms
    o, w, _ = d[5]
    dev, st = dev_stream()
    S, R, beam, alpha, beta = 3, 12, 64, 1.0, 1.5
    frames_cap = 200
    si, sf = C.c_int64(0), C.c_int64(0)
    _lib.call("masr_ctc_prefix_beam_wordlm_state_size", C.byref(si), C.byref(sf))
    pool, _, _, _ = workspace(S, 1)
    cap = 5 * (frames_cap * beam + 1)
    tp = torch.full((S * cap,), -1, dtype=torch.int32, device=dev)
    tt = torch.zeros(S * cap, dtype=torch.int32, device=dev)
    sti = torch.zeros(S, si.value, dtype=torch.int32, device=dev); stf = torch.zeros(S, sf.value, device=dev)
    fresh = torch.ones(S, dtype=torch.int32, device=dev)
    otok = torch.zeros(S, frames_cap, dtype=torch.int32, device=dev)
    on = torch.zeros(S, dtype=torch.int32, device=dev)
    osc, oap = torch.zeros(S, device=dev), torch.zeros(S, device=dev)
    utt = {s: wl_logits(40 + s, 150, o, dev) for s in range(S)}
    pos = [0] * S
    search = [owl.WordLmSearch(o, alpha, beta, beam) for _ in range(S)]
    plan = [(12, 5, 12), (12, 0, 7), (3, 12, 0), ("reset", 12, 12), (12, 12, 4), (0, 9, 12)]
    for step, p in enumerate(plan):
        if p[0] == "reset":                       # slot 0 starts a new utterance
            fresh[0] = 1
            tp[cap // 5:cap].fill_(-1)
            utt[0] = wl_logits(90, 150, o, dev)
            pos[0] = 0
            search[0] = owl.WordLmSearch(o, alpha, beta, beam)
            p = (12,) + p[1:]
        L = torch.zeros(S * R, 32, device=dev)
        for s in range(S):
            L[s * R:s * R + p[s]] = utt[s][pos[s]:pos[s] + p[s]]
        cid, clp, cn, blp = topk(L, len(vocab))
        ld = torch.tensor(p, dtype=torch.int32, device=dev)
        before = [(sti[s].clone(), stf[s].clone(), tp[s * cap:(s + 1) * cap].clone(), tt[s * cap:(s + 1) * cap].clone(),
                   otok[s].clone(), on[s].clone(), osc[s].clone(), oap[s].clone()) for s in range(S)]
        _lib.call("masr_ctc_prefix_beam_wordlm_pool", cid.data_ptr(), clp.data_ptr(), cn.data_ptr(), blp.data_ptr(), R, ld.data_ptr(),
                  S, beam, 0, C.byref(w.tables(dev)), alpha, beta, pool.data_ptr(), tp.data_ptr(), tt.data_ptr(), cap, sti.data_ptr(),
                  stf.data_ptr(), fresh.data_ptr(), otok.data_ptr(), frames_cap, on.data_ptr(), osc.data_ptr(), oap.data_ptr(), st)
        torch.cuda.synchronize()
        for s in range(S):
            if p[s] == 0:
                after = (sti[s], stf[s], tp[s * cap:(s + 1) * cap], tt[s * cap:(s + 1) * cap], otok[s], on[s], osc[s], oap[s])
                assert all(torch.equal(x, y) for x, y in zip(before[s], after)), (step, s)
                continue
            cands, blps = host_cands(cid, clp, cn, blp, range(s * R, s * R + p[s]))
            (score, approx, toks), = search[s].push(cands, blps).result()
            pos[s] += p[s]
            got = (otok[s, :on[s].item()].cpu().tolist(), F(osc[s].item()), F(oap[s].item()))
            assert got == (toks, F(score), F(approx)), (step, s)
    assert fresh.sum().item() == 0


# ---- MASRPredictor with an English vocabulary and a word ARPA ------------------------------------------------------
def make_predictor(tmp, lm_path, vocab):
    from masr_b200 import synth
    from masr_b200.predict import MASRPredictor
    mp, vp = str(tmp / "m.pt"), str(tmp / "vocabulary.txt")
    torch.save(synth.to_torch(synth.conformer_state_dict(0, vocab_size=len(vocab), ctc_gain=2.0)), mp)
    with open(vp, "w", encoding="utf-8") as f:
        for i, t in enumerate(vocab):
            f.write(f"{t}\t{len(vocab) - i}\n")
    cfg = {"use_model": "conformer", "streaming": True, "decoder": "ctc_beam_search",
           "preprocess_conf": {"feature_method": "fbank", "n_mels": 80, "sample_rate": 16000, "use_dB_normalization": True, "target_dB": -20},
           "dataset_conf": {"dataset_vocab": vp},
           "ctc_beam_search_decoder_conf": {"alpha": 1.2, "beta": 0.8, "beam_size": 64, "cutoff_prob": 0.99, "cutoff_top_n": 40,
                                            "language_model_path": lm_path}}
    return MASRPredictor(configs=cfg, model_path=mp, use_gpu=True)


def restate(eng, o, b, T_b):
    ws, T, B = eng._last_beam
    cands = eng.last_beam_candidates()[b][:T_b]
    blp = ws["blank_lp"][b * T:b * T + T_b].cpu().numpy()
    (score, approx, toks), = owl.prefix_beam_search_wordlm(o, cands, blp, 1.2, 0.8, beam_size=64)
    return toks, F(approx)


def test_predictor_with_word_arpa_lm(tmp_path, wlms):
    from conftest import make_audio
    from masr_b200.engine import StreamBeam
    from masr_b200.evaluate import evaluate
    from masr_b200.lm import WordLM
    vocab, d = wlms
    o, _, path = d[3]
    pred = make_predictor(tmp_path, path, vocab)
    assert isinstance(pred.lm, WordLM) and pred.lm.order == 3 and not pred.lm.is_character_based
    assert pred.lm.dict_size == o.dict_size
    eng = pred.predictor

    def check_words(text):
        for word in text.split(" ")[:-1]:
            assert word in o.lex.word_id, (word, text)

    x1, x2 = make_audio("speech", 81, 16000 * 2), make_audio("speech", 82, 16000 * 3)
    one = pred.predict(audio_data=x1.copy())
    T0 = int(eng._last_beam[0]["tlens"][0].item())
    toks, approx = restate(eng, o, 0, T0)
    assert one["text"] == ids_to_text(toks, vocab) and F(one["score"]) == approx
    check_words(one["text"])
    batch = pred.predict_batch([x1.copy(), x2.copy()])
    tl = [int(t) for t in eng._last_beam[0]["tlens"][:2].cpu()]
    for b in range(2):
        toks, approx = restate(eng, o, b, tl[b])
        assert batch[b]["text"] == ids_to_text(toks, vocab) and F(batch[b]["score"]) == approx
        check_words(batch[b]["text"])
    assert batch[0] == one
    assert list(pred.predict_batches([[x1.copy(), x2.copy()], [x2.copy()]])) == [batch, [batch[1]]]
    # streaming: the StreamBeam's own candidates, restated after every push
    pred.reset_stream()
    sb = StreamBeam(eng, **pred._beam_conf)
    seen = {"cands": [], "blp": []}
    orig = sb.push

    def push(logits, rows):
        out = orig(logits, rows)
        n, ids, lp = sb.cand_n[:rows].cpu().numpy(), sb.cand_id[:rows].cpu().numpy(), sb.cand_lp[:rows].cpu().numpy()
        seen["cands"] += [[(int(ids[t, k]), lp[t, k]) for k in range(n[t])] for t in range(rows)]
        seen["blp"] += list(sb.blank_lp[:rows].cpu().numpy())
        return out
    sb.push = push
    pred._sbeam = sb
    pcm = (np.clip(x2, -1, 1) * 32767).astype("<i2")
    pieces = [(pcm[s:s + 8000].tobytes(), s + 8000 >= len(pcm)) for s in range(0, len(pcm), 8000)]
    streamed = []
    for b, e in pieces:
        r = pred.predict_stream(audio_data=b, is_end=e)
        streamed.append(r)
        if r is None:
            continue
        (score, approx, toks), = owl.prefix_beam_search_wordlm(o, seen["cands"], seen["blp"], 1.2, 0.8, beam_size=64)
        assert r["text"] == ids_to_text(toks, vocab) and F(r["score"]) == F(approx)
        check_words(r["text"])
    assert sum(r is not None for r in streamed) >= 2
    # the stream pool decodes a slot as predict_stream does
    sp = pred.create_stream_pool(2, max_frames=400)
    assert sp.beam is not None and sp.beam.lm is pred.lm
    for (b, e), want in zip(pieces, streamed):
        assert sp.push({1: b}, is_end=e)[1] == want
    err, n = evaluate(pred, [(x1.copy(), "ab cd"), (x2.copy(), "ef")], batch_size=2, metrics_type="wer")
    assert n == 2 and np.isfinite(err)


def test_word_lm_without_space_token_runs_without_lm(tmp_path, wlms):
    from conftest import make_audio
    vocab, d = wlms
    _, _, path = d[3]
    novocab = [t if t != "<space>" else "_" for t in vocab]
    pred = make_predictor(tmp_path, path, novocab)
    assert pred.lm is None
    assert isinstance(pred.predict(audio_data=make_audio("speech", 83, 16000)), dict)
