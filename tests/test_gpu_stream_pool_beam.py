"""GPU (-m gpu): the CTC prefix beam search of every slot of a stream pool (``StreamPool(beam=...)``, the pool entry points
masr_ctc_prefix_beam_pool / masr_ctc_prefix_beam_lm_pool) — per slot equal to the single-stream search, to the CPU
restatement bit for bit on the pool's own candidates, and to ``MASRPredictor.predict_stream`` push by push."""
import ctypes as C

import numpy as np
import pytest
import torch

from conftest import make_audio, synth_weights
from masr_b200 import synth
from masr_b200.text import ids_to_text
from oracle import beam as obeam, lm as olm
from test_beam import rand_posteriors

pytestmark = pytest.mark.gpu
V = synth.DEFAULT_VOCAB_SIZE
PUSH = 8000


# ---------------------------------------------------------------------------------------------------------------------
# C ABI: one launch with a fresh, a resumed and an idle slot
def _topk(logits, dev, lm):
    from masr_b200 import _lib
    M = logits.shape[0]
    cid = torch.zeros(M, 40, dtype=torch.int32, device=dev); clp = torch.zeros(M, 40, device=dev)
    cn = torch.zeros(M, dtype=torch.int32, device=dev); blp = torch.zeros(M, device=dev)
    st = torch.cuda.current_stream().cuda_stream
    if lm:
        _lib.call("masr_ctc_topk_blank_f32", logits.data_ptr(), logits.stride(0), M, V, 40, 0.99, 0, cid.data_ptr(), clp.data_ptr(),
                  cn.data_ptr(), blp.data_ptr(), st)
    else:
        _lib.call("masr_ctc_topk_f32", logits.data_ptr(), logits.stride(0), M, V, 40, 0.99, cid.data_ptr(), clp.data_ptr(),
                  cn.data_ptr(), st)
    return cid, clp, cn, blp


def _logits(seed, T, dev, lift=None):
    _, lg = rand_posteriors(seed, T, V)
    if lift is not None:
        lg[:, lift] += 3.0
    L = torch.zeros(T, (V + 15) // 16 * 16, device=dev)
    L[:, :V] = torch.from_numpy(lg).to(dev)
    return L


@pytest.fixture(scope="module")
def char_lm(tmp_path_factory):
    """Character LMs over nearly the whole synthetic vocabulary: the synthetic models emit arbitrary characters, and an
    out-of-vocabulary extension costs alpha * -1000, which would leave every transcript empty."""
    from masr_b200.lm import CharLM
    vocab = synth.vocabulary(V)
    out = {}
    for order in (3, 5):
        p = str(tmp_path_factory.mktemp("lm") / f"o{order}.arpa")
        chars = synth.character_lm_arpa(p, seed=order, order=order, n_chars=4200, n_sentences=600)
        out[order] = (olm.read_arpa(p), CharLM(p, vocab), [vocab.index(c) for c in chars], p)
    return out


@pytest.mark.parametrize("lm_order", [None, 3])
def test_pool_abi_fresh_resumed_idle(char_lm, lm_order):
    from masr_b200 import _lib
    dev = torch.device("cuda", torch.cuda.current_device())
    st = torch.cuda.current_stream().cuda_stream
    lm = lm_order is not None
    clm, lift = (char_lm[lm_order][1], char_lm[lm_order][2]) if lm else (None, None)
    tab = C.byref(clm.tables(dev)) if lm else None
    alpha, beta, beam = 0.5, 2.0, 24
    S, R = 3, 40                                           # slots, candidate rows per slot and launch (bstride)
    # whole sequences: slot 0 a fresh utterance of 33 frames; slot 1 = 27 frames, then 35 more; slot 2 = 30 frames, then idle
    seqs = {0: _topk(_logits(11, 33, dev, lift), dev, lm), 1: _topk(_logits(12, 62, dev, lift), dev, lm),
            2: _topk(_logits(13, 30, dev, lift), dev, lm)}
    frames = 62
    pool_n, trie_n, si, sf = C.c_int64(0), C.c_int64(0), C.c_int64(0), C.c_int64(0)
    _lib.call("masr_ctc_prefix_beam_workspace", S, 1, C.byref(pool_n), C.byref(trie_n))
    _lib.call("masr_ctc_prefix_beam_lm_state_size" if lm else "masr_ctc_prefix_beam_state_size", C.byref(si), C.byref(sf))
    cap = 5 * (frames * beam + 1)                          # sized by beam_size, not by the 512 cap
    scratch = torch.empty(pool_n.value, device=dev)
    tp = torch.full((S * cap,), -1, dtype=torch.int32, device=dev); tt = torch.zeros_like(tp)
    sti = torch.zeros(S, si.value, dtype=torch.int32, device=dev); stf = torch.zeros(S, sf.value, device=dev)
    fresh = torch.ones(S, dtype=torch.int32, device=dev)
    otok = torch.zeros(S, frames, dtype=torch.int32, device=dev); on = torch.zeros(S, dtype=torch.int32, device=dev)
    osc, oap = torch.zeros(S, device=dev), torch.zeros(S, device=dev)

    def launch(rows):                                      # rows: slot -> (first frame, count)
        cid = torch.zeros(S * R, 40, dtype=torch.int32, device=dev); clp = torch.zeros(S * R, 40, device=dev)
        cn = torch.zeros(S * R, dtype=torch.int32, device=dev); blp = torch.zeros(S * R, device=dev)
        lens = torch.zeros(S, dtype=torch.int32, device=dev)
        for s, (a, n) in rows.items():
            c = seqs[s]
            cid[s * R:s * R + n], clp[s * R:s * R + n], cn[s * R:s * R + n], blp[s * R:s * R + n] = (
                c[0][a:a + n], c[1][a:a + n], c[2][a:a + n], c[3][a:a + n])
            lens[s] = n
        if lm:
            _lib.call("masr_ctc_prefix_beam_lm_pool", cid.data_ptr(), clp.data_ptr(), cn.data_ptr(), blp.data_ptr(), R, lens.data_ptr(),
                      S, beam, 0, tab, alpha, beta, scratch.data_ptr(), tp.data_ptr(), tt.data_ptr(), cap, sti.data_ptr(), stf.data_ptr(),
                      fresh.data_ptr(), otok.data_ptr(), frames, on.data_ptr(), osc.data_ptr(), oap.data_ptr(), st)
        else:
            _lib.call("masr_ctc_prefix_beam_pool", cid.data_ptr(), clp.data_ptr(), cn.data_ptr(), R, lens.data_ptr(), S, beam, 0,
                      scratch.data_ptr(), tp.data_ptr(), tt.data_ptr(), cap, sti.data_ptr(), stf.data_ptr(), fresh.data_ptr(),
                      otok.data_ptr(), frames, on.data_ptr(), osc.data_ptr(), st)
        torch.cuda.synchronize()

    def one_shot(s, n):
        c = seqs[s]
        tcap = C.c_int64(0)
        _lib.call("masr_ctc_prefix_beam_workspace", 1, n, C.byref(pool_n), C.byref(tcap))
        sc = torch.empty(pool_n.value, device=dev)
        p1 = torch.empty(tcap.value, dtype=torch.int32, device=dev); t1 = torch.empty_like(p1)
        ld = torch.tensor([n], dtype=torch.int32, device=dev)
        ot = torch.zeros(1, frames, dtype=torch.int32, device=dev); o_n = torch.zeros(1, dtype=torch.int32, device=dev)
        o_s, o_a = torch.zeros(1, device=dev), torch.zeros(1, device=dev)
        if lm:
            _lib.call("masr_ctc_prefix_beam_lm", c[0].data_ptr(), c[1].data_ptr(), c[2].data_ptr(), c[3].data_ptr(), n, ld.data_ptr(), 1,
                      beam, 0, tab, alpha, beta, sc.data_ptr(), p1.data_ptr(), t1.data_ptr(), tcap.value, ot.data_ptr(), frames,
                      o_n.data_ptr(), o_s.data_ptr(), o_a.data_ptr(), st)
        else:
            _lib.call("masr_ctc_prefix_beam", c[0].data_ptr(), c[1].data_ptr(), c[2].data_ptr(), n, ld.data_ptr(), 1, beam, 0,
                      sc.data_ptr(), p1.data_ptr(), t1.data_ptr(), tcap.value, ot.data_ptr(), frames, o_n.data_ptr(), o_s.data_ptr(), st)
        torch.cuda.synchronize()
        k = int(o_n.item())
        return ot[0, :k].cpu().tolist(), o_s.cpu().numpy().view(np.int32)[0], o_a.cpu().numpy().view(np.int32)[0]

    def got(s):
        k = int(on[s].item())
        return otok[s, :k].cpu().tolist(), osc[s:s + 1].cpu().numpy().view(np.int32)[0], oap[s:s + 1].cpu().numpy().view(np.int32)[0]

    # launch 1: slot 1 and slot 2 start (fresh), slot 0 has no frames yet
    launch({1: (0, 27), 2: (0, 30)})
    assert fresh.cpu().tolist() == [1, 0, 0]                # the kernel cleared the flags of the slots it initialised
    for s, n in ((1, 27), (2, 30)):
        want = one_shot(s, n)
        assert got(s)[:2] == want[:2] and (not lm or got(s)[2] == want[2]), s
    # launch 2: slot 0 fresh, slot 1 resumed, slot 2 idle (lens = 0) -> byte for byte untouched
    idle_before = [x.clone() for x in (sti[2], stf[2], otok[2], on[2:3], osc[2:3], oap[2:3], tp[2 * cap:3 * cap], tt[2 * cap:3 * cap])]
    launch({0: (0, 33), 1: (27, 35)})
    idle_after = (sti[2], stf[2], otok[2], on[2:3], osc[2:3], oap[2:3], tp[2 * cap:3 * cap], tt[2 * cap:3 * cap])
    for a, b in zip(idle_before, idle_after):
        assert torch.equal(a.view(torch.int32) if a.dtype == torch.float32 else a, b.view(torch.int32) if b.dtype == torch.float32 else b)
    for s, n in ((0, 33), (1, 62)):
        g, w = got(s), one_shot(s, n)
        assert g[0] == w[0] and g[1] == w[1], (s, g, w)     # tokens and score bit for bit (resumed == concatenated)
        if lm:
            assert g[2] == w[2], (s, g, w)                 # approx_ctc too
    assert len(got(1)[0]) > 0


# ---------------------------------------------------------------------------------------------------------------------
# StreamPool(beam=...) over the models
ALPHA, BETA = 0.5, 2.0


def _predictor(tmp, use_model="conformer", lm_path="lm/none.klm", beam_size=16, decoder="ctc_beam_search"):
    from masr_b200.predict import MASRPredictor
    if use_model == "conformer":
        sd = synth_weights(0)
    elif use_model == "squeezeformer":
        sd = synth.squeezeformer_state_dict(0, streaming=True)
    else:
        sd = synth.efficient_conformer_state_dict(0)
    mp, vp = str(tmp / f"{use_model}.pt"), str(tmp / "vocabulary.txt")
    torch.save(synth.to_torch(sd), mp)
    synth.write_vocabulary(vp)
    cfg = {"use_model": use_model, "streaming": True, "decoder": decoder,
           "preprocess_conf": {"feature_method": "fbank", "n_mels": 80, "sample_rate": 16000, "use_dB_normalization": True, "target_dB": -20},
           "dataset_conf": {"dataset_vocab": vp},
           "ctc_beam_search_decoder_conf": {"alpha": ALPHA, "beta": BETA, "beam_size": beam_size, "cutoff_prob": 0.99, "cutoff_top_n": 40,
                                            "language_model_path": lm_path}}
    return MASRPredictor(configs=cfg, model_path=mp, use_gpu=True)


def _streams():
    """Four streams as lists of (PCM bytes, is_end) pushes, and a schedule of rounds (slot -> stream): stream 1 is silent in
    round 2, slot 2 is reset after stream 2 ends and reused for stream 3, slot 3 stays idle throughout."""
    lens = [6 * PUSH - 1234, 5 * PUSH - 3000, 3 * PUSH - 500, 3 * PUSH]
    kinds = ["speech", "speech", "noise", "speech"]
    out = []
    for i, (n, k) in enumerate(zip(lens, kinds)):
        pcm = (np.clip(make_audio(k, 300 + i, n), -1, 1) * 32767).astype("<i2")
        starts = list(range(0, n, PUSH))
        out.append([(pcm[s:s + PUSH].tobytes(), j == len(starts) - 1) for j, s in enumerate(starts)])
    schedule = [{0: 0, 1: 1, 2: 2}, {0: 0, 1: 1, 2: 2}, {0: 0, 2: 2}, {0: 0, 1: 1, 2: 3}, {0: 0, 1: 1, 2: 3}, {0: 0, 1: 1, 2: 3}]
    return out, schedule


def _reference(pred, streams):
    want = []
    for pieces in streams:
        pred.reset_stream()
        want.append([pred.predict_stream(audio_data=b, is_end=e) for b, e in pieces])
    pred.reset_stream()
    return want


class _Recorder:
    """Keeps every slot's candidates (and blank log-probabilities) since its last reset, read back after each pool step."""

    def __init__(self, sp):
        self.sp, self.cands, self.blp = sp, [[] for _ in range(sp.S)], [[] for _ in range(sp.S)]
        orig_step, orig_reset = sp.pool.step, sp.reset_stream
        bm = sp.beam
        R = sp.pool.OUT_ROWS

        def step(feats, nframes):
            r = orig_step(feats, nframes)
            tout = r[2]
            ids, lp, n = bm.cand_id.cpu().numpy(), bm.cand_lp.cpu().numpy(), bm.cand_n.cpu().numpy()
            bl = bm.blank_lp.cpu().numpy() if bm.lm is not None else None
            for s in range(sp.S):
                for t in range(tout[s]):
                    row = s * R + t
                    self.cands[s].append([(int(ids[row, k]), lp[row, k]) for k in range(n[row])])
                    if bl is not None:
                        self.blp[s].append(bl[row])
            return r

        def reset(slot):
            orig_reset(slot)
            self.cands[slot], self.blp[slot] = [], []

        sp.pool.step, sp.reset_stream = step, reset


def _drive(sp, streams, schedule, check=None):
    got = [[] for _ in streams]
    pos = [0] * len(streams)
    for rnd in schedule:
        ends = {s: streams[i][pos[i]][1] for s, i in rnd.items()}          # one push per stream and round
        for is_end in (False, True):
            msgs = {s: i for s, i in rnd.items() if ends[s] == is_end}
            if not msgs:
                continue
            out = sp.push({s: streams[i][pos[i]][0] for s, i in msgs.items()}, is_end=is_end)
            assert set(out) == set(msgs)
            for s, i in msgs.items():
                got[i].append(out[s])
                pos[i] += 1
                if out[s] is not None and check is not None:
                    check(s, out[s])
                if is_end:
                    sp.reset_stream(s)
    assert pos == [len(p) for p in streams]
    return got


def _compare(got, want):
    for i, (g, w) in enumerate(zip(got, want)):
        assert len(g) == len(w)
        for r, x in zip(g, w):
            assert (r is None) == (x is None), (i, r, x)
            if r is not None:
                assert r["text"] == x["text"], (i, r, x)
                assert abs(r["score"] - x["score"]) < 1e-3, (i, r, x)
    assert any(r is not None and r["text"] for g in got for r in g)


def test_conformer_pool_beam_equals_predict_stream_and_restatement(tmp_path):
    from masr_b200.stream_pool import StreamPool
    pred = _predictor(tmp_path)
    assert pred.lm is None and pred._beam_conf["beam_size"] == 16
    streams, schedule = _streams()
    want = _reference(pred, streams)
    results = {}
    for use_graph in (True, False):
        sp = StreamPool(pred.predictor, synth.vocabulary(), n_slots=4, beam=pred._beam_conf, use_graph=use_graph, max_frames=400)
        rec = _Recorder(sp)

        def check(s, r):                                   # bit for bit against the restatement on the pool's own candidates
            c = rec.cands[s]
            (score, toks), = obeam.prefix_beam_search(np.zeros((len(c), 1)), beam_size=16, cands_per_frame=c)
            assert r["text"] == ids_to_text(toks, synth.vocabulary()) and np.float32(r["score"]) == np.float32(score), (s, r, score)
        results[use_graph] = _drive(sp, streams, schedule, check)
        _compare(results[use_graph], want)
        assert sp.beam.fresh.cpu().tolist() == [1, 1, 1, 1]   # every used slot was reset after its last push; slot 3 never ran
    assert results[True] == results[False]                   # CUDA graph replay == eager launches


@pytest.mark.parametrize("order", [3, 5])
def test_conformer_pool_beam_with_lm(tmp_path, char_lm, order):
    from masr_b200.stream_pool import StreamPool
    olm_, _, _, path = char_lm[order]
    pred = _predictor(tmp_path, lm_path=path)
    assert pred.lm is not None and pred.lm.order == order
    streams, schedule = _streams()
    want = _reference(pred, streams)
    sp = StreamPool(pred.predictor, synth.vocabulary(), n_slots=4, beam=pred._beam_conf, max_frames=400)
    rec = _Recorder(sp)
    vocab = synth.vocabulary()

    def check(s, r):
        c = rec.cands[s]
        (score, approx, toks), = olm.prefix_beam_search_lm(np.zeros((len(c), 1)), olm_, vocab, ALPHA, BETA, beam_size=16,
                                                          cands_per_frame=c, blank_logp_per_frame=rec.blp[s])
        assert r["text"] == ids_to_text(toks, vocab) and np.float32(r["score"]) == np.float32(approx), (s, r, approx)
    got = _drive(sp, streams, schedule, check)
    _compare(got, want)


@pytest.mark.parametrize("use_model", ["squeezeformer", "efficient_conformer"])
def test_family_pools_beam_equal_predict_stream(tmp_path, use_model):
    from masr_b200.stream_pool import StreamPool
    pred = _predictor(tmp_path, use_model)
    streams, schedule = _streams()
    want = _reference(pred, streams)
    sp = StreamPool(pred.predictor, synth.vocabulary(), n_slots=4, beam=pred._beam_conf, max_frames=400)
    assert sp.pool.OUT_ROWS == (8 if use_model == "efficient_conformer" else 16)
    _compare(_drive(sp, streams, schedule), want)


def test_create_stream_pool_and_sessions_follow_the_yaml(tmp_path, char_lm):
    from masr_b200.serve import StreamSessions
    greedy = _predictor(tmp_path, decoder="ctc_greedy")
    assert greedy.create_stream_pool(2, max_frames=400).beam is None
    pred = _predictor(tmp_path, lm_path=char_lm[3][3])
    sp = pred.create_stream_pool(3, max_frames=400)
    assert sp.beam is not None and sp.beam.lm is pred.lm and sp.beam.beam == 16
    with pytest.raises(ValueError, match="beam_size"):
        from masr_b200.stream_pool import StreamPool
        StreamPool(pred.predictor, synth.vocabulary(), 1, beam=dict(pred._beam_conf, beam_size=513))
    streams, _ = _streams()
    want = _reference(pred, streams[:2])
    sess = StreamSessions(sp)
    ids = [sess.open(), sess.open()]
    text = [None, None]
    for k in range(max(len(s) for s in streams[:2])):
        msgs = {}
        for i in range(2):
            if k < len(streams[i]):
                b, e = streams[i][k]
                msgs[ids[i]] = b + (b"end" if e else b"")
        replies = sess.feed(msgs)
        for i in range(2):
            if k < len(streams[i]):
                if want[i][k] is not None:
                    text[i] = want[i][k]["text"]
                assert replies[ids[i]] == {"code": 0, "result": text[i] or ""}, (i, k)
    assert any(text)
