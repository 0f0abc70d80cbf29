"""GPU (-m gpu): character n-gram LM fusion — the device tables and query kernel against oracle/lm.py, the fused prefix
beam search (one-shot and streaming) against the restatement bit for bit, and MASRPredictor with an ARPA file."""
import ctypes as C

import numpy as np
import pytest
import torch

from masr_b200.text import ids_to_text
from oracle import beam as obeam, lm as olm
from test_beam import rand_posteriors

pytestmark = pytest.mark.gpu
V = 4233


@pytest.fixture(scope="module")
def lms(tmp_path_factory):
    from masr_b200 import synth
    from masr_b200.lm import CharLM
    vocab = synth.vocabulary(V)
    out = {}
    for order in (3, 5):
        p = str(tmp_path_factory.mktemp("lm") / f"o{order}.arpa")
        chars = synth.character_lm_arpa(p, seed=order, order=order, n_chars=80, n_sentences=600)
        out[order] = (olm.read_arpa(p), CharLM(p, vocab), [vocab.index(c) for c in chars], p)
    return vocab, out


@pytest.mark.parametrize("order", [3, 5])
def test_query_kernel_equals_oracle(lms, order):
    vocab, d = lms
    olm_, clm, ids, _ = d[order]
    rng = np.random.default_rng(order)
    Q = 100_000
    pool = np.array(ids + [-1, -2, 1, 5, 17, 4000], np.int64)          # LM characters, <s>, </s>, <unk>, OOV tokens
    prob = np.r_[np.full(len(ids), 0.9 / len(ids)), np.full(6, 0.1 / 6)]
    ctx = rng.choice(pool, (Q, order - 1), p=prob)
    pad = rng.integers(0, order, Q)                                    # <s> left padding of various lengths
    for j in range(order - 1):
        ctx[pad > j, j] = -1
    word = rng.choice(pool, Q, p=prob)
    got = clm.score(ctx, word)
    name = lambda t: "<s>" if t == -1 else "</s>" if t == -2 else vocab[t]
    want = np.array([olm_.lnp([name(t) for t in ctx[q]], name(word[q])) for q in range(Q)], np.float32)
    assert np.array_equal(got.view(np.int32), want.view(np.int32)), np.flatnonzero(got != want)[:10]
    assert (want == -1000).any() and (want > -1000).mean() > 0.3


def topk(logits, dev, top_n, cut):
    from masr_b200 import _lib
    M = logits.shape[0]
    cid = torch.empty(M, 40, dtype=torch.int32, device=dev); clp = torch.empty(M, 40, device=dev)
    cn = torch.empty(M, dtype=torch.int32, device=dev); blp = torch.empty(M, device=dev)
    _lib.call("masr_ctc_topk_blank_f32", logits.data_ptr(), logits.stride(0), M, V, top_n, cut, 0, cid.data_ptr(), clp.data_ptr(),
              cn.data_ptr(), blp.data_ptr(), torch.cuda.current_stream().cuda_stream)
    return cid, clp, cn, blp


def lm_logits(seed, T, ids, dev):
    """rand_posteriors logits with the LM's characters lifted, so the search extends with LM words and OOV tokens alike."""
    _, logits = rand_posteriors(seed, T, V)
    logits[:, ids] += 3.0
    ldl = (V + 15) // 16 * 16
    L = torch.zeros(T, ldl, device=dev)
    L[:, :V] = torch.from_numpy(logits).to(dev)
    return L


@pytest.mark.parametrize("order,seed,T,beam,cut,alpha,beta", [
    (3, 1, 60, 300, 0.99, 2.2, 4.3), (3, 2, 45, 16, 1.0, 0.8, -0.5), (5, 3, 60, 300, 1.0, 1.0, 1.5), (5, 4, 40, 1, 0.99, 2.2, 4.3),
    (5, 5, 50, 16, 0.99, 0.5, 0.0), (3, 6, 70, 300, 0.99, 0.0, 0.0)])
def test_gpu_lm_beam_equals_restatement(lms, order, seed, T, beam, cut, alpha, beta):
    from masr_b200 import _lib
    vocab, d = lms
    olm_, clm, ids, _ = d[order]
    dev = torch.device("cuda", torch.cuda.current_device())
    st = torch.cuda.current_stream().cuda_stream
    lens = [T, T // 2]
    B = len(lens)
    L = torch.cat([lm_logits(seed, T, ids, dev), lm_logits(seed + 100, T, ids, dev)])
    cid, clp, cn, blp = topk(L, dev, 40, cut)
    pool_n, trie_n = C.c_int64(0), C.c_int64(0)
    _lib.call("masr_ctc_prefix_beam_workspace", B, T, C.byref(pool_n), C.byref(trie_n))
    pool = torch.empty(pool_n.value, device=dev); tp = torch.empty(B * trie_n.value, dtype=torch.int32, device=dev)
    tt = torch.empty_like(tp)
    ld = torch.tensor(lens, dtype=torch.int32, device=dev)
    otok = torch.zeros(B, T, dtype=torch.int32, device=dev); on = torch.zeros(B, dtype=torch.int32, device=dev)
    osc, oap = torch.zeros(B, device=dev), torch.zeros(B, device=dev)
    _lib.call("masr_ctc_prefix_beam_lm", cid.data_ptr(), clp.data_ptr(), cn.data_ptr(), blp.data_ptr(), T, ld.data_ptr(), B, beam, 0,
              C.byref(clm.tables(dev)), alpha, beta, pool.data_ptr(), tp.data_ptr(), tt.data_ptr(), trie_n.value, otok.data_ptr(), T,
              on.data_ptr(), osc.data_ptr(), oap.data_ptr(), st)
    torch.cuda.synchronize()
    cid_h, clp_h, cn_h, blp_h = cid.cpu().numpy(), clp.cpu().numpy(), cn.cpu().numpy(), blp.cpu().numpy()
    ph = torch.softmax(L[:, :V], 1).cpu().numpy()
    assert np.allclose(blp_h, np.log(ph[:, 0]), atol=2e-5)
    for r in range(B * T):                            # == the candidate's own log-probability when blank is a candidate
        for k in range(cn_h[r]):
            if cid_h[r, k] == 0:
                assert blp_h[r] == clp_h[r, k]
    any_lm = False
    for b in range(B):
        rows = range(b * T, b * T + lens[b])
        cands = [[(int(cid_h[r, k]), clp_h[r, k]) for k in range(cn_h[r])] for r in rows]
        (score, approx, toks), = olm.prefix_beam_search_lm(ph[b * T: b * T + lens[b]], olm_, vocab, alpha, beta, beam_size=beam,
                                                          cutoff_prob=cut, cands_per_frame=cands,
                                                          blank_logp_per_frame=[blp_h[r] for r in rows])
        got = otok[b, :on[b].item()].cpu().tolist()
        assert got == toks, (b, got, toks)
        assert np.float32(osc[b].item()) == np.float32(score), (b, osc[b].item(), score)
        assert np.float32(oap[b].item()) == np.float32(approx), (b, oap[b].item(), approx)
        any_lm |= any(olm_.in_vocab(vocab[c]) for c in toks)
    assert any_lm


@pytest.mark.parametrize("order,seed,T,beam,chunk", [(3, 7, 75, 300, 16), (5, 8, 50, 32, 7)])
def test_gpu_lm_streaming_equals_one_shot(lms, order, seed, T, beam, chunk):
    from masr_b200 import _lib
    vocab, d = lms
    _, clm, ids, _ = d[order]
    dev = torch.device("cuda", torch.cuda.current_device())
    st = torch.cuda.current_stream().cuda_stream
    cid, clp, cn, blp = topk(lm_logits(seed, T, ids, dev), dev, 40, 0.99)
    tab = C.byref(clm.tables(dev))
    alpha, beta = 2.2, 4.3
    pool_n, trie_n, si, sf = C.c_int64(0), C.c_int64(0), C.c_int64(0), C.c_int64(0)
    _lib.call("masr_ctc_prefix_beam_workspace", 1, T, C.byref(pool_n), C.byref(trie_n))
    _lib.call("masr_ctc_prefix_beam_lm_state_size", C.byref(si), C.byref(sf))

    def bufs():
        return (torch.empty(pool_n.value, device=dev), torch.empty(trie_n.value, dtype=torch.int32, device=dev),
                torch.empty(trie_n.value, dtype=torch.int32, device=dev), torch.zeros(1, T, dtype=torch.int32, device=dev),
                torch.zeros(1, dtype=torch.int32, device=dev), torch.zeros(1, device=dev), torch.zeros(1, device=dev))

    def one_shot(n):
        pool, tp, tt, otok, on, osc, oap = bufs()
        ld = torch.tensor([n], dtype=torch.int32, device=dev)
        _lib.call("masr_ctc_prefix_beam_lm", cid.data_ptr(), clp.data_ptr(), cn.data_ptr(), blp.data_ptr(), T, ld.data_ptr(), 1, beam,
                  0, tab, alpha, beta, pool.data_ptr(), tp.data_ptr(), tt.data_ptr(), trie_n.value, otok.data_ptr(), T, on.data_ptr(),
                  osc.data_ptr(), oap.data_ptr(), st)
        return otok[0, :on.item()].cpu().tolist(), osc.item(), oap.item()

    pool, tp, tt, otok, on, osc, oap = bufs()
    sti = torch.zeros(si.value, dtype=torch.int32, device=dev); stf = torch.zeros(sf.value, device=dev)
    done = 0
    while done < T:
        n = min(chunk, T - done)
        ld = torch.tensor([n], dtype=torch.int32, device=dev)
        _lib.call("masr_ctc_prefix_beam_lm_stream", cid[done:].data_ptr(), clp[done:].data_ptr(), cn[done:].data_ptr(),
                  blp[done:].data_ptr(), T, ld.data_ptr(), 1, beam, 0, tab, alpha, beta, pool.data_ptr(), tp.data_ptr(), tt.data_ptr(),
                  trie_n.value, sti.data_ptr(), stf.data_ptr(), 1 if done else 0, otok.data_ptr(), T, on.data_ptr(), osc.data_ptr(),
                  oap.data_ptr(), st)
        done += n
        assert (otok[0, :on.item()].cpu().tolist(), osc.item(), oap.item()) == one_shot(done), done


def make_predictor(tmp, lm_path, streaming=True):
    from conftest import synth_weights
    from masr_b200 import synth
    from masr_b200.predict import MASRPredictor
    mp, vp = str(tmp / "m.pt"), str(tmp / "vocabulary.txt")
    torch.save(synth.to_torch(synth_weights(0)), mp)
    synth.write_vocabulary(vp)
    cfg = {"use_model": "conformer", "streaming": streaming, "decoder": "ctc_beam_search",
           "preprocess_conf": {"feature_method": "fbank", "n_mels": 80, "sample_rate": 16000, "use_dB_normalization": True, "target_dB": -20},
           "dataset_conf": {"dataset_vocab": vp},
           "ctc_beam_search_decoder_conf": {"alpha": 2.2, "beta": 4.3, "beam_size": 64, "cutoff_prob": 0.99, "cutoff_top_n": 40,
                                            "language_model_path": lm_path}}
    return MASRPredictor(configs=cfg, model_path=mp, use_gpu=True)


def test_predictor_with_arpa_lm(tmp_path, lms):
    from conftest import make_audio
    from masr_b200.engine import StreamBeam
    vocab, d = lms
    olm_, _, _, path = d[3]
    pred = make_predictor(tmp_path, path)
    assert pred.lm is not None and pred.lm.order == 3 and pred.lm.is_character_based
    eng = pred.predictor
    x1, x2 = make_audio("speech", 81, 16000 * 2), make_audio("speech", 82, 16000 * 3)
    one = pred.predict(audio_data=x1.copy())
    lens = [int(t) for t in eng._last_beam[0]["tlens"][:1].cpu()]
    toks, approx = restate_len(eng, olm_, vocab, 0, lens[0])
    assert one["text"] == ids_to_text(toks, vocab) and np.float32(one["score"]) == approx
    batch = pred.predict_batch([x1.copy(), x2.copy()])
    tl = [int(t) for t in eng._last_beam[0]["tlens"][:2].cpu()]
    for b in range(2):
        toks, approx = restate_len(eng, olm_, vocab, b, tl[b])
        assert batch[b]["text"] == ids_to_text(toks, vocab) and np.float32(batch[b]["score"]) == approx
    assert batch[0] == one
    piped = list(pred.predict_batches([[x1.copy(), x2.copy()], [x2.copy()], [x1.copy()]]))
    assert piped == [batch, [batch[1]], [one]]
    # streaming: the StreamBeam's own candidates of every chunk, restated one-shot after every push
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
    pushes = 0
    for s in range(0, len(pcm), 8000):
        r = pred.predict_stream(audio_data=pcm[s:s + 8000].tobytes(), is_end=s + 8000 >= len(pcm))
        if r is None:
            continue
        (score, approx, toks), = olm.prefix_beam_search_lm(np.zeros((len(seen["cands"]), 1)), olm_, vocab, 2.2, 4.3, beam_size=64,
                                                          cands_per_frame=seen["cands"], blank_logp_per_frame=seen["blp"])
        assert r["text"] == ids_to_text(toks, vocab) and np.float32(r["score"]) == approx
        pushes += 1
    assert pushes >= 2


def restate_len(eng, olm_, vocab, b, T_b):
    ws, T, B = eng._last_beam
    cands = eng.last_beam_candidates()[b][:T_b]
    blp = ws["blank_lp"][b * T:b * T + T_b].cpu().numpy()
    (score, approx, toks), = olm.prefix_beam_search_lm(np.zeros((T_b, 1)), olm_, vocab, 2.2, 4.3, beam_size=64,
                                                      cands_per_frame=cands, blank_logp_per_frame=blp)
    return toks, np.float32(approx)


def test_predictor_with_kenlm_binary_runs_without_lm(tmp_path):
    from conftest import make_audio
    klm = tmp_path / "zh.klm"
    klm.write_bytes(b"mmap lm http://kheafield.com/code format version 5\n" + bytes(64))
    pred = make_predictor(tmp_path, str(klm), streaming=False)
    assert pred.lm is None
    x = make_audio("speech", 83, 16000 * 2)
    out = pred.predict(audio_data=x.copy())
    eng = pred.predictor
    T_b = int(eng._last_beam[0]["tlens"][0].item())
    (score, toks), = obeam.prefix_beam_search(np.zeros((T_b, 1)), beam_size=64, cands_per_frame=eng.last_beam_candidates()[0][:T_b])
    from masr_b200 import synth
    assert out["text"] == ids_to_text(toks, synth.vocabulary()) and np.float32(out["score"]) == np.float32(score)
