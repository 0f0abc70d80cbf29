"""GPU (-m gpu): token onsets of the prefix beam search (masr_ctc_prefix_beam_frames) against the restatements, in every
form, and token times end to end through MASRPredictor, StreamPool and SegmentingStreamPool for all four families."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from conftest import make_audio, synth_weights
from masr_b200 import synth, timestamps as ts
from oracle import silero_vad as sv
import beam_onsets as bo
from test_gpu_beam_contract import BEAM_CAP, SENT, V, Rows, Search, bits, char_lms, grid_logits, topk_rows, word_lms  # noqa: F401

pytestmark = pytest.mark.gpu
F = np.float32


@pytest.fixture(scope="module")
def rt():
    from kernel_contract import runtime
    return runtime()


def readout(rt, s, B):
    """masr_ctc_prefix_beam_frames over Search ``s`` -> per slot the onsets of its reported tokens (past them: untouched)."""
    fr = torch.full((B, s.tok_stride), SENT, dtype=torch.int32, device=rt.dev)
    rt.call("masr_ctc_prefix_beam_frames", s.tp.data_ptr(), s.tt.data_ptr(), s.cap, s.otok.data_ptr(), s.tok_stride,
            s.on.data_ptr(), B, fr.data_ptr(), s.tok_stride, rt.st())
    torch.cuda.synchronize()
    n, h = s.on.cpu().numpy(), fr.cpu().numpy()
    assert all((h[b, n[b]:] == SENT).all() for b in range(B))
    return [h[b, :n[b]].tolist() for b in range(B)]


def case(rt, mode, char_lms, word_lms, B, T, seed):
    """Candidate frames of B utterances of T frames, and the search settings of ``mode``."""
    if mode == "word":
        vocab, d = word_lms
        o, lm = d[2]
        rng = np.random.default_rng(seed)
        logits = rng.standard_normal((B * T, len(vocab))).astype(np.float32) * 2.0
        logits[:, lm.space] += 1.5
        fr, bl = topk_rows(rt, logits, 40, 0.99, 0)
        kw, Vv = dict(lm=lm, alpha=0.8, beta=-1.0), len(vocab)
    else:
        vocab, d = char_lms
        o, lm, ids, _ = d[3]
        fr, bl = topk_rows(rt, grid_logits(seed, B * T, V, ids + [1, 9], 0, -8.0), 40, 0.99, 0)
        kw, Vv = (dict(lm=lm, alpha=0.6, beta=0.5) if mode == "char" else {}), V
    frames = [fr[b * T:(b + 1) * T] for b in range(B)]
    blps = [bl[b * T:(b + 1) * T] for b in range(B)]
    return frames, blps, kw, Vv, (o, vocab)


@pytest.mark.parametrize("mode", ["plain", "char", "word"])
def test_onsets_equal_the_restatement_in_every_form(rt, char_lms, word_lms, mode):
    """One-shot onsets == the restatement's on the kernel's own candidates; streaming in chunks of 1, 7 and 64 and the pool
    form in two launches == one-shot; the read-out writes nothing but its output, and a search followed by it reports
    what the same search reports without it."""
    B, T, beam = 2, 40, 16                     # (the onsets' definition reruns the restatement per frame: O(T^2))
    frames, blps, kw, Vv, (o, vocab) = case(rt, mode, char_lms, word_lms, B, T, 7)
    rows = Rows(rt, frames, blps, bstride=T, Vv=Vv)
    one = Search(rt, mode, beam, B, T, **kw)
    one.run("one", rows, [T] * B)
    plain = Search(rt, mode, beam, B, T, **kw)
    plain.run("one", rows, [T] * B)
    snap = [bits(x).clone() for x in (one.tp, one.tt, one.otok, one.on, one.osc, one.oap)]
    got = readout(rt, one, B)
    assert all(torch.equal(x, bits(y)) for x, y in zip(snap, (one.tp, one.tt, one.otok, one.on, one.osc, one.oap)))
    assert torch.equal(one.otok, plain.otok) and torch.equal(one.on, plain.on) and torch.equal(bits(one.osc), bits(plain.osc))
    lo = {"plain": None, "char": o, "word": o}[mode]
    total = 0
    for b in range(B):
        toks, want = bo.best_onsets(mode, frames[b], blps[b], beam, lo, vocab, kw.get("alpha", 0.0), kw.get("beta", 0.0))
        assert one.best(b)[0] == toks and got[b] == want, b
        assert all(x < y for x, y in zip(want, want[1:]))
        total += len(want)
    assert total > 10
    for chunk in (1, 7, 64):
        s = Search(rt, mode, beam, B, T, **kw)
        for t0 in range(0, T, chunk):
            s.run("stream", rows, [min(chunk, T - t0)] * B, t0, resume=t0 > 0)
        assert readout(rt, s, B) == got and torch.equal(s.otok, one.otok), chunk
    p = Search(rt, mode, beam, B, T, **kw)
    p.run("pool", rows, [15] * B)
    p.run("pool", rows, [T - 15] * B, 15)
    assert readout(rt, p, B) == got


def test_onsets_with_the_trie_at_capacity_over_200_frames(rt):
    """The capacity case of the beam contract (every frame's beam is all new children, the trie fills to 1 + 40 + 512 * 199
    nodes): the best prefix is one token per frame, so its onsets are 0 .. 199, in chunks of 1, 7 and 64 and one-shot."""
    T, beam = 200, BEAM_CAP
    rng = np.random.default_rng(11)
    sets = [list(range(1, 41)), list(range(41, 81))]
    frames = [[(c, F(np.log(p))) for c, p in zip(sets[t % 2], rng.dirichlet(np.ones(40)))] for t in range(T)]
    rows = Rows(rt, [frames], bstride=T)
    one = Search(rt, "plain", beam, 1, T)
    one.run("one", rows, [T])
    assert readout(rt, one, 1) == [list(range(T))]
    for chunk in (1, 7, 64):
        s = Search(rt, "plain", beam, 1, T)
        for t0 in range(0, T, chunk):
            s.run("stream", rows, [min(chunk, T - t0)], t0, resume=t0 > 0)
        assert readout(rt, s, 1) == [list(range(T))], chunk


def test_prefixes_that_leave_the_beam_and_return_keep_their_first_onset(rt):
    """Beam 3 over peaky frames, one frame per call: prefixes drop out and are re-created later.  After every frame the
    onsets of the reported prefix are those of the definition (the first frame each of its prefixes was in the beam)."""
    returns = 0
    for seed in range(4):
        rng = np.random.default_rng(seed)
        T = 30
        frames = []
        for _ in range(T):
            ids = list(rng.choice([0, 1, 2, 3], 3, replace=False))
            frames.append([(int(c), F(np.log(p))) for c, p in zip(ids, rng.dirichlet(np.ones(3) * 0.5))])
        per_frame, _ = bo.beams("plain", frames, beam=3)
        last = {}
        for t, bm in enumerate(per_frame):
            for p in bm:
                returns += p in last and last[p] < t - 1
                last[p] = t
        rows = Rows(rt, [frames], bstride=T)
        s = Search(rt, "plain", 3, 1, T)
        for t in range(T):
            s.run("stream", rows, [1], t, resume=t > 0)
            toks = s.best(0)[0]
            assert list(per_frame[t][0]) == toks and readout(rt, s, 1) == [bo.onsets(per_frame[:t + 1], toks)], (seed, t)
    assert returns > 0


def _pool_launch(rt, s, rows, ld):
    """Search.run's pool launch without the synchronisation (so it can be captured)."""
    cid, clp, cn, blp = rows.ptrs(0)
    lm = [blp] if s.mode != "plain" else []
    lmw = [C.byref(s.lm.tables(rt.dev)), s.alpha, s.beta] if s.mode != "plain" else []
    rt.call(s.name + "_pool", cid, clp, cn, *lm, rows.bstride, ld.data_ptr(), s.B, s.beam, s.blank, *lmw, s.pool.data_ptr(),
            s.tp.data_ptr(), s.tt.data_ptr(), s.cap, s.sti.data_ptr(), s.stf.data_ptr(), s.fresh.data_ptr(), s.otok.data_ptr(),
            s.tok_stride, s.on.data_ptr(), s.osc.data_ptr(), *([s.oap.data_ptr()] if s.mode != "plain" else []), rt.st())


@pytest.mark.parametrize("mode", ["plain", "char"])
def test_pool_onsets_with_resets_idle_slots_and_graph_replay(rt, char_lms, word_lms, mode):
    """Six pool slots over three steps replayed from one CUDA graph: ragged lengths with idle slots, slot 2 reset (fresh,
    hash range cleared) before the third step.  Each slot's onsets count from its reset and equal a one-shot search over
    its frames since then; an idle slot's clock stands still."""
    B, T, beam = 6, 12, 32
    frames, blps, kw, Vv, _ = case(rt, mode, char_lms, word_lms, B, 3 * T, 3)
    sched = [[T, 5, 0, T, 1, 0], [0, T, T, 3, 0, 7], [T, 0, 9, T, 2, 0]]
    s = Search(rt, mode, beam, B, 3 * T, **kw)
    stage = Rows(rt, [f[:T] for f in frames], [b[:T] for b in blps], bstride=T, Vv=Vv)
    ld = torch.zeros(B, dtype=torch.int32, device=rt.dev)
    pos, since = [0] * B, [0] * B                                 # frames consumed; first frame since the last reset
    graph = None
    for k, lens in enumerate(sched):
        step = Rows(rt, [frames[b][pos[b]:pos[b] + lens[b]] for b in range(B)],
                    [blps[b][pos[b]:pos[b] + lens[b]] for b in range(B)], bstride=T, Vv=Vv, seed=k)
        for x, y in ((stage.cid, step.cid), (stage.clp, step.clp), (stage.cn, step.cn), (stage.blp, step.blp)):
            x.copy_(y)
        ld.copy_(torch.tensor(lens, dtype=torch.int32))
        if k == 2:
            s.fresh[2] = 1
            s.tp[2 * s.cap + s.cap // 5:3 * s.cap] = -1
            since[2] = pos[2]
        if graph is None:
            _pool_launch(rt, s, stage, ld)                        # (eager once: the kernel's shared-memory attribute)
            torch.cuda.synchronize()
            s.fresh.fill_(1)
            s.tp.fill_(-1)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                _pool_launch(rt, s, stage, ld)
        graph.replay()
        torch.cuda.synchronize()
        pos = [p + n for p, n in zip(pos, lens)]
        got = readout(rt, s, B)
        for b in range(B):
            if pos[b] == since[b]:
                continue
            ref = Search(rt, mode, beam, 1, 3 * T, **kw)
            ref.run("one", Rows(rt, [frames[b][since[b]:pos[b]]], [blps[b][since[b]:pos[b]]], bstride=3 * T, Vv=Vv), [pos[b] - since[b]])
            assert s.best(b)[:2] == ref.best(0)[:2] and got[b] == readout(rt, ref, 1)[0], (k, b)
        clock = s.tt.view(B, s.cap)[:, 4 * (s.cap // 5)].cpu().tolist()
        assert all(clock[b] == pos[b] - since[b] for b in range(B) if pos[b] > since[b]), (k, clock)


# ---- end to end ---------------------------------------------------------------------------------------------------------
FAMILIES = ["conformer", "efficient_conformer", "squeezeformer", "deepspeech2"]


def _predictor(tmp, use_model, decoder="ctc_greedy"):
    import yaml
    from masr_b200.predict import MASRPredictor
    sd = {"conformer": lambda: synth_weights(0), "deepspeech2": lambda: synth.deepspeech2_state_dict(0, streaming=True),
          "squeezeformer": lambda: synth.squeezeformer_state_dict(0, streaming=True),
          "efficient_conformer": lambda: synth.efficient_conformer_state_dict(0)}[use_model]()
    mp, vp = str(tmp / f"{use_model}.pt"), str(tmp / "vocabulary.txt")
    torch.save(synth.to_torch(sd), mp)
    synth.write_vocabulary(vp)
    cfg = {"use_model": use_model, "streaming": True, "decoder": decoder,
           "preprocess_conf": {"feature_method": "fbank", "n_mels": 80, "sample_rate": 16000, "use_dB_normalization": True,
                               "target_dB": -20},
           "dataset_conf": {"dataset_vocab": vp},
           "ctc_beam_search_decoder_conf": {"beam_size": 16, "cutoff_prob": 0.99, "cutoff_top_n": 40,
                                            "language_model_path": "lm/none.klm"}}
    p = str(tmp / f"{use_model}.yml")
    with open(p, "w", encoding="utf-8") as f:
        yaml.safe_dump(cfg, f)
    return MASRPredictor(configs=p, model_path=mp, use_gpu=True)


def _pieces(x, n=8000):
    return [x[i:i + n] for i in range(0, len(x), n)]


def _stream(pred, x, timestamps=True):
    pred.reset_stream()
    out = None
    ps = _pieces(x)
    for i, p in enumerate(ps):
        r = pred.predict_stream(p, is_end=i == len(ps) - 1, timestamps=timestamps)
        out = r if r is not None else out
    return out


@pytest.mark.parametrize("use_model", FAMILIES)
def test_end_to_end_token_times(tmp_path, use_model):
    """Greedy and beam, whole utterance and stream, per family: the times are the frame spans of what the decoder saw
    (greedy: the frame ids; beam: the restatement's onsets on the kernel's own candidates), text and score are unchanged by
    asking for times, and an 8-slot StreamPool per slot equals predict_stream."""
    vocab = synth.vocabulary()
    x = make_audio("speech", 91, 16000 * 3 + 1234)
    xs = [make_audio("speech", 100 + i, 16000 * (1 + i % 3) + 3000 * i) for i in range(8)]
    for decoder in ("ctc_greedy", "ctc_beam_search"):
        pred = _predictor(tmp_path, use_model, decoder)
        dt = ts.frame_seconds(pred.predictor)
        assert dt == (0.08 if use_model == "efficient_conformer" else 0.04)
        r = pred.predict(x.copy(), timestamps=True)
        assert {k: r[k] for k in ("text", "score")} == pred.predict(x.copy())
        if decoder == "ctc_greedy":
            g = pred.predictor.transcribe([x.copy()], return_frames=True)
            toks, s, e = ts.greedy_spans(g.frame_ids[0, :g.frame_lens[0]])
            assert toks == g.tokens[0]
        else:
            cands = pred.predictor.last_beam_candidates()[0]
            toks, s = bo.best_onsets("plain", cands, beam=16)
            e = [f + 1 for f in s]
        assert len(toks) > 3
        assert r["tokens"] == ts.token_times(toks, s, e, vocab, dt)
        assert [b["text"] for b in pred.predict_batch([x.copy(), xs[0].copy()], timestamps=True)][:1] == [r["text"]]
        # predict_stream: greedy spans of the concatenated chunk ids; beam onsets of the one-shot search over the chunks'
        # candidates (recorded from the streaming search itself)
        seen = []
        if decoder == "ctc_beam_search":
            from masr_b200.engine import StreamBeam
            push0 = StreamBeam.push

            def spy(self, logits, rows):
                out = push0(self, logits, rows)
                n = self.cand_n[:rows].cpu().numpy()
                ci, cl = self.cand_id[:rows].cpu().numpy(), self.cand_lp[:rows].cpu().numpy()
                seen.extend([[(int(ci[t, k]), F(cl[t, k])) for k in range(n[t])] for t in range(rows)])
                return out
            StreamBeam.push = spy
        try:
            st = _stream(pred, x)
        finally:
            if decoder == "ctc_beam_search":
                StreamBeam.push = push0
        if decoder == "ctc_greedy":
            toks, s, e = ts.greedy_spans(pred._hist_ids)
        else:
            toks, s = bo.best_onsets("plain", seen, beam=16)
            e = [f + 1 for f in s]
        assert st["tokens"] == ts.token_times(toks, s, e, vocab, dt) and len(toks) > 3
        assert {k: st[k] for k in ("text", "score")} == _stream(pred, x, timestamps=False)
        want = [_stream(pred, a) for a in xs]
        sp = pred.create_stream_pool(8, timestamps=True)
        got = [None] * 8
        pieces = [_pieces(a) for a in xs]
        for k in range(max(len(p) for p in pieces)):
            for end in (False, True):                             # (StreamPool.push takes one is_end for the push)
                msg = {i: p[k] for i, p in enumerate(pieces) if k < len(p) and (k == len(p) - 1) == end}
                for i, res in (sp.push(msg, is_end=end) if msg else {}).items():
                    got[i] = res if res is not None else got[i]
        for i in range(8):
            assert got[i]["text"] == want[i]["text"] and got[i]["tokens"] == want[i]["tokens"], (decoder, i)
            assert abs(got[i]["score"] - want[i]["score"]) < 1e-3


class _Stamps:
    def __init__(self, stamps):
        self.stamps = stamps

    def get_speech_timestamps(self, samples, sr):
        return [dict(s) for s in self.stamps]


def _inside(tokens, start, end, dt):
    return all(start <= t["start"] < t["end"] <= end + dt + 1e-9 for t in tokens)


@pytest.mark.parametrize("use_model", FAMILIES)
def test_long_form_token_times_lie_inside_their_segments(tmp_path, use_model):
    """predict_long (scripted VAD) and SegmentingStreamPool (the silero VAD on the GPU): every sentence / segment's tokens
    lie inside it (a beam token's end is its onset + one frame), times absolute; text and score as without times."""
    z = lambda n: np.zeros(n, np.float32)
    rec = np.concatenate([z(5000), make_audio("speech", 7, 16000 * 2), z(20000), make_audio("speech", 8, 25000), z(4000)])
    stamps = [{"start": 4000, "end": 38000}, {"start": 56000, "end": 83000}]
    for decoder in ("ctc_greedy", "ctc_beam_search"):
        pred = _predictor(tmp_path, use_model, decoder)
        dt = ts.frame_seconds(pred.predictor)
        timed = pred.predict_long(rec.copy(), vad_predictor=_Stamps(stamps), timestamps=True)
        assert {k: timed[k] for k in ("text", "score")} == pred.predict_long(rec.copy(), vad_predictor=_Stamps(stamps))
        assert timed["sentences"]
        for sent in timed["sentences"]:
            st = next(s for s in stamps if round(s["start"] / 16000, 3) == sent["start"])
            assert sent["end"] == round(st["end"] / 16000, 3) and _inside(sent["tokens"], sent["start"], sent["end"], dt)
            one = pred.predict(rec[st["start"]:st["end"]].copy(), timestamps=True)
            assert sent["text"] == one["text"] and [t["token"] for t in sent["tokens"]] == [t["token"] for t in one["tokens"]]
        if not os.path.exists(sv.MODEL_PATH):
            continue
        sp = pred.create_stream_pool(2, vad_model_path=sv.MODEL_PATH, timestamps=True)
        segs = []
        streams = [rec, rec[3000:]]
        pieces = [_pieces(a) for a in streams]
        for k in range(max(len(p) for p in pieces)):
            msg = {i: p[k] for i, p in enumerate(pieces) if k < len(p)}
            for i, res in sp.push(msg, is_end={i: k == len(pieces[i]) - 1 for i in msg}).items():
                segs += res["segments"]
                if res["partial"] is not None:
                    assert _inside(res["partial"]["tokens"], res["partial"]["start"] / 16000, len(streams[i]) / 16000, dt)
        assert segs and any(g["tokens"] for g in segs)
        for g in segs:
            assert _inside(g["tokens"], g["start"] / 16000, g["end"] / 16000, dt), g
