"""GPU (-m gpu): the N-best read-out of the prefix beam search (the six ``*_nbest`` entry points through
masr_b200.beam.BeamSearch.nbest) against the oracles' ``nbest=`` / ``result(nbest)`` on the GPU's own top-k candidates, bit
for bit (token ids, fused and reported float32 scores): no LM, character LM (orders 3 and 5) and word LM, each with and
without hotwords, at beam 1, 16, 300 and 512 and n = 1, 2, 7, the beam size and past the live entries; tied scores from
coarse-grid logits; a stream fed in chunks equal to the whole utterance; pool slots with ragged lengths, a reset and their
own hotword lists, with the buffers the read-out must not write checked byte for byte; refused arguments.  Hypothesis 0
is always the search's own result (one-shot, streaming and pool forms)."""
import ctypes as C

import numpy as np
import pytest
import torch

from masr_b200 import _lib
from masr_b200.beam import ONE_SHOT, POOL, STREAM, BeamSearch
from masr_b200.hotwords import HotwordBuffer, HotwordGraph
from oracle import hotwords as oh
from oracle import lm as olm
from oracle import word_lm as owl
from test_beam import rand_posteriors

pytestmark = pytest.mark.gpu
F = np.float32
AB = {"none": (0.0, 0.0), "char3": (0.8, 1.0), "char5": (0.6, 0.5), "word": (1.0, 1.5)}
# (LM kind, hotwords) -> the read-out entry point BeamSearch.nbest launches
NAMES = {("none", False): "masr_ctc_prefix_beam_nbest", ("char", False): "masr_ctc_prefix_beam_lm_nbest",
         ("word", False): "masr_ctc_prefix_beam_wordlm_nbest", ("none", True): "masr_ctc_prefix_beam_hot_nbest",
         ("char", True): "masr_ctc_prefix_beam_lm_hot_nbest", ("word", True): "masr_ctc_prefix_beam_wordlm_hot_nbest"}


class Eng:
    """The launch surface BeamSearch needs from an engine."""

    def __init__(self, V):
        self.V = V

    def _k(self, tag, name, *args, n=1):
        _lib.call(name, *args, torch.cuda.current_stream().cuda_stream)


@pytest.fixture(scope="module")
def kinds(tmp_path_factory):
    from masr_b200 import synth
    from masr_b200.lm import CharLM, WordLM
    cv = synth.vocabulary(300)
    out = {"none": None}
    ids = None
    for order in (3, 5):
        p = str(tmp_path_factory.mktemp(f"lm{order}") / "c.arpa")
        chars = synth.character_lm_arpa(p, seed=3, order=order, n_chars=80, n_sentences=600, vocab_size=300)
        ids = ids or [cv.index(c) for c in chars]
        out[f"char{order}"] = (cv, CharLM(p, cv), olm.read_arpa(p), ids)
    out["none"] = (cv, None, None, ids)
    ev = synth.english_vocabulary()
    pw = str(tmp_path_factory.mktemp("wlm") / "w.arpa")
    synth.word_lm_arpa(pw, seed=3, order=3, n_words=120)
    o = owl.WordLM(pw, ev)
    letters = sorted({t for ch in o.lex.child for t in ch})
    out["word"] = (ev, WordLM(pw, ev), o, letters + [o.space])
    hws = {"char": ["".join(cv[i] for i in ids[j:j + L]) for j, L in ((0, 2), (0, 4), (5, 3), (9, 2))],
           "word": [w for w in o.lex.words if 2 <= len(w) <= 6][:5]}
    return out, hws


def logits_for(seed, T, V, lift, dev, grid=None):
    _, lg = rand_posteriors(seed, T, V, peaky=3.0)
    lg[:, lift] += 2.5
    if grid is not None:                                     # coarse grid: many exactly equal candidate log-probabilities
        lg = np.round(lg / grid) * grid
    L = torch.zeros(T, (V + 15) // 16 * 16, device=dev)
    L[:, :V] = torch.from_numpy(lg.astype(np.float32)).to(dev)
    return L


def cands(bs, rows):
    cid, clp, cn = bs.cand_id.cpu().numpy(), bs.cand_lp.cpu().numpy(), bs.cand_n.cpu().numpy()
    blp = bs.blank_lp.cpu().numpy() if bs.blank_lp is not None else np.zeros(len(cn), np.float32)
    return [[(int(cid[r, k]), clp[r, k]) for k in range(cn[r])] for r in rows], [blp[r] for r in rows]


def oracle(kind, olm_, vocab, cl, blp, beam, H, n):
    """-> [(tokens, fused score, reported score)] best first, at most n."""
    alpha, beta = AB[kind]
    if kind == "word":
        res = oh.WordLmSearchHot(olm_, alpha, beta, beam, hotwords=H).push(cl, blp).result(n)
    else:
        res = oh.prefix_beam_search_hot(None, olm_, vocab, alpha, beta, beam, cands_per_frame=cl, blank_logp_per_frame=blp,
                                        hotwords=H, nbest=n)
    return [(toks, F(s), F(a)) for s, a, toks in res]


def got_nbest(res, b):
    tok, cnt, sc, fu, nh = (x.cpu().numpy() for x in res)
    return [(tok[b, h, :cnt[b, h]].tolist(), F(fu[b, h]), F(sc[b, h])) for h in range(int(nh[b]))]


def got_search(bs, b):
    n = int(bs.count[b].item())
    return bs.out_tok[b, :n].cpu().tolist(), F(bs.fused[b].item()), F(bs.score[b].item())


def setup(kinds, kind, hot):
    table, hws = kinds
    vocab, lm, olm_, lift = table[kind]
    g = H = None
    if hot:
        g = HotwordGraph(hws["word" if kind == "word" else "char"], vocab, 2.0)
        H = oh.HotwordMatcher(g.tokens, 2.0)
    return vocab, lm, olm_, lift, g, H


def base_kind(kind):
    return "char" if kind.startswith("char") else kind


@pytest.mark.parametrize("beam", [1, 16, 300, 512])
@pytest.mark.parametrize("hot", [False, True])
@pytest.mark.parametrize("kind", ["none", "char3", "char5", "word"])
def test_nbest_equals_oracle(kinds, kind, hot, beam):
    """Three utterances (one of 1 frame: fewer live entries than n) searched by the streaming form from the root; every
    n's list equals the oracle's first n, and hypothesis 0 equals the streaming and the one-shot searches' results."""
    vocab, lm, olm_, lift, g, H = setup(kinds, kind, hot)
    dev, V, T = torch.device("cuda"), len(vocab), 40
    alpha, beta = AB[kind]
    eng = Eng(V)
    L = torch.cat([logits_for(s, T, V, lift, dev) for s in (1, 2, 3)])
    lens = [T, 1, T - 9]
    ld = torch.tensor(lens, dtype=torch.int32, device=dev)
    bs = BeamSearch(dev, STREAM, 3, 3 * T, T, beam, 0.99, 40, lm, alpha, beta, g)
    one = BeamSearch(dev, ONE_SHOT, 3, 3 * T, T, beam, 0.99, 40, lm, alpha, beta, g)
    assert bs.name[:-len(STREAM)] + "_nbest" == NAMES[(base_kind(kind), hot)]
    for s in (bs, one):
        s.topk(eng, L, L.stride(0), 3 * T)
        s.search(eng, ld.data_ptr(), 3, T)
    torch.cuda.synchronize()
    wants = []
    for b in range(3):
        cl, blp = cands(bs, range(b * T, b * T + lens[b]))
        wants.append(oracle(kind, olm_, vocab, cl, blp, beam, H, beam))
        assert got_search(bs, b) == got_search(one, b), b
        # (an empty beam — the word LM's lexicon can reject every extension at beam 1 — reports no tokens at -inf)
        assert got_search(bs, b) == (wants[b][0] if wants[b] else ([], F(-np.inf), F(-np.inf))), b
    assert beam < 300 or len(wants[1]) < beam             # the 1-frame slot: fewer live entries than the beam
    for n in sorted({1, 2, 7, beam} & set(range(1, beam + 1))):
        res = bs.nbest(eng, 3, n)
        for b in range(3):
            got = got_nbest(res, b)
            assert got == wants[b][:n], (n, b)
            assert not got or got[0] == got_search(bs, b)
    # past the live entries (n up to 512, which the host caps at the beam size): count = the live entries
    res = bs.nbest(eng, 3, beam) if beam == 512 else None
    if res is None:
        n = 512
        tok = torch.full((3, n, T), -7, dtype=torch.int32, device=dev)
        cnt, nh = torch.full((3, n), -7, dtype=torch.int32, device=dev), torch.full((3,), -7, dtype=torch.int32, device=dev)
        sc, fu = torch.zeros(3, n, device=dev), torch.zeros(3, n, device=dev)
        args = [bs.trie_par.data_ptr(), bs.trie_tok.data_ptr(), bs.trie_cap, bs.state_i.data_ptr(), bs.state_f.data_ptr(),
                None, 3, n]
        if lm is not None:
            args += [C.byref(lm.tables(dev)), alpha, beta]
        args += [tok.data_ptr(), T, cnt.data_ptr()] + ([fu.data_ptr(), sc.data_ptr()] if lm is not None else [sc.data_ptr()])
        args += [nh.data_ptr()] + ([C.byref(g.tables(dev)), bs.slot_root.data_ptr()] if hot else [])
        _lib.call(NAMES[(base_kind(kind), hot)], *args, torch.cuda.current_stream().cuda_stream)
        res = (tok, cnt, sc, fu if lm is not None else sc, nh)
    for b in range(3):
        assert got_nbest(res, b) == wants[b], b


@pytest.mark.parametrize("kind,hot", [("none", False), ("char3", True), ("word", False), ("word", True)])
def test_tied_scores(kinds, kind, hot):
    """Logits on a grid of 1.0: many beam entries with exactly equal scores, ordered by beam rank as the oracle does."""
    vocab, lm, olm_, lift, g, H = setup(kinds, kind, hot)
    dev, V, T, beam = torch.device("cuda"), len(vocab), 30, 64
    alpha, beta = AB[kind]
    eng = Eng(V)
    L = torch.cat([logits_for(s, T, V, lift, dev, grid=1.0) for s in (4, 5)])
    ld = torch.tensor([T, T], dtype=torch.int32, device=dev)
    bs = BeamSearch(dev, STREAM, 2, 2 * T, T, beam, 0.99, 40, lm, alpha, beta, g)
    bs.topk(eng, L, L.stride(0), 2 * T)
    bs.search(eng, ld.data_ptr(), 2, T)
    res = bs.nbest(eng, 2, beam)
    ties = 0
    for b in range(2):
        cl, blp = cands(bs, range(b * T, (b + 1) * T))
        want = oracle(kind, olm_, vocab, cl, blp, beam, H, beam)
        got = got_nbest(res, b)
        assert got == want, b
        sel = [x[1] for x in got]
        ties += sum(x == y for x, y in zip(sel, sel[1:]))
    assert ties > 0 or kind != "none", "no tied scores: the test does not exercise the tie order"


@pytest.mark.parametrize("kind", ["none", "char5", "word"])
def test_chunked_stream_equals_whole(kinds, kind):
    """A stream fed in chunks of 7 and of 64 frames reads out the same N-best as one launch over all its frames."""
    vocab, lm, olm_, lift, g, H = setup(kinds, kind, True)
    dev, V, T, beam, n = torch.device("cuda"), len(vocab), 150, 300, 10
    alpha, beta = AB[kind]
    eng = Eng(V)
    L = logits_for(7, T, V, lift, dev)
    whole = BeamSearch(dev, STREAM, 1, T, T, beam, 0.99, 40, lm, alpha, beta, g)
    whole.topk(eng, L, L.stride(0), T)
    ld = torch.tensor([T], dtype=torch.int32, device=dev)
    whole.search(eng, ld.data_ptr(), 1, T)
    want = got_nbest(whole.nbest(eng, 1, n), 0)
    cl, blp = cands(whole, range(T))
    assert want == oracle(kind, olm_, vocab, cl, blp, beam, H, n)
    for chunk in (7, 64):
        sb = BeamSearch(dev, STREAM, 1, chunk, T, beam, 0.99, 40, lm, alpha, beta, g)
        done = 0
        while done < T:
            m = min(chunk, T - done)
            sb.topk(eng, L[done:done + m], L.stride(0), m)
            ld.fill_(m)
            sb.search(eng, ld.data_ptr(), 1, chunk, resume=1 if done else 0)
            done += m
        assert got_nbest(sb.nbest(eng, 1, n), 0) == want, chunk


@pytest.mark.parametrize("kind", ["none", "char3", "word"])
def test_pool_slots(kinds, kind):
    """Five slots (lists A, B, none, A, and slot 4 never requested): ragged steps with 0-frame slots, slot 0 reset with
    list B mid-run.  After each step the read-out of slots 0..3 equals the oracle for every slot with frames, a reset
    slot reports 0 hypotheses and leaves its rows alone, the unrequested slot's rows are never written, and the search's
    state, trie and outputs are byte for byte what they were before the read-out."""
    vocab, lm, olm_, lift, _, _ = setup(kinds, kind, False)
    table, hws = kinds
    hw = hws["word" if kind == "word" else "char"]
    dev, V, S, R, beam, frames_cap, n = torch.device("cuda"), len(vocab), 5, 12, 48, 120, 9
    alpha, beta = AB[kind]
    eng = Eng(V)
    gA, gB = HotwordGraph(hw[:2], vocab, 2.0), HotwordGraph(hw[2:], vocab, 2.0)
    buf = HotwordBuffer(dev, S + 1, max(gA.nodes, gB.nodes))
    buf.put(0, gA)
    buf.put(1, gB)
    buf.put(3, gA)
    roots = torch.tensor([buf.root(0), buf.root(1), -1, buf.root(3), -1], dtype=torch.int32, device=dev)
    bs = BeamSearch(dev, POOL, S, S * R, frames_cap, beam, 0.99, 40, lm, alpha, beta, buf, slot_root=roots)
    assert bs.name[:-len(POOL)] + "_nbest" == NAMES[(base_kind(kind), True)]
    Hs = [oh.HotwordMatcher(x.tokens, 2.0) for x in (gA, gB)] + [None, oh.HotwordMatcher(gA.tokens, 2.0), None]
    utt = {s: logits_for(60 + s, 100, V, lift, dev) for s in range(S)}
    pos, hist, fresh = [0] * S, [([], []) for _ in range(S)], [True] * S
    plan = [(12, 5, 0, 3, 12), (12, 0, 7, 12, 4), ("reset", 12, 12, 0, 0), (0, 12, 4, 9, 2), (7, 0, 0, 12, 0)]
    for step, p in enumerate(plan):
        if p[0] == "reset":
            bs.fresh[0] = 1
            bs.trie_par[bs.trie_cap // 5:bs.trie_cap].fill_(-1)
            buf.put(0, gB)
            Hs[0] = Hs[1]
            utt[0], pos[0], hist[0], fresh[0] = logits_for(95, 100, V, lift, dev), 0, ([], []), True
            p = (0,) + p[1:]
        Lg = torch.zeros(S * R, utt[0].shape[1], device=dev)
        for s in range(S):
            Lg[s * R:s * R + p[s]] = utt[s][pos[s]:pos[s] + p[s]]
        bs.topk(eng, Lg, Lg.stride(0), S * R)
        ld = torch.tensor(p, dtype=torch.int32, device=dev)
        bs.search(eng, ld.data_ptr(), S, R)
        torch.cuda.synchronize()
        for s in range(S):
            if p[s]:
                cl, blp = cands(bs, range(s * R, s * R + p[s]))
                hist[s][0].extend(cl)
                hist[s][1].extend(blp)
                pos[s] += p[s]
                fresh[s] = False
        # the read-out's outputs pre-filled with a sentinel, the search's buffers snapshotted
        res = bs.nbest(eng, S - 1, n)                        # (allocates; the sentinel pass is the one checked)
        for x in (bs.nb_tok, bs.nb_out, bs.nb_n):
            x.view(torch.int32).fill_(-7)
        before = [x.clone() for x in (bs.state_i, bs.state_f, bs.trie_par, bs.trie_tok, bs.out, bs.out_tok, bs.fresh)]
        res = bs.nbest(eng, S - 1, n)
        torch.cuda.synchronize()
        after = (bs.state_i, bs.state_f, bs.trie_par, bs.trie_tok, bs.out, bs.out_tok, bs.fresh)
        assert all(torch.equal(x, y) for x, y in zip(before, after)), step
        nh = res[4].cpu().numpy()
        raw_tok, raw_out = bs.nb_tok.view(torch.int32).cpu().numpy(), bs.nb_out.view(torch.int32).cpu().numpy()
        assert nh[S - 1] == -7 and (raw_tok[S - 1] == -7).all() and (raw_out[:, S - 1] == -7).all(), step
        for s in range(S - 1):
            if fresh[s]:
                assert nh[s] == 0, (step, s)
                assert (raw_tok[s] == -7).all() and (raw_out[:, s] == -7).all(), (step, s)
                continue
            want = oracle(kind, olm_, vocab, hist[s][0], hist[s][1], beam, Hs[s], n)
            got = got_nbest(res, s)
            assert got == want, (step, s)
            assert got[0] == got_search(bs, s), (step, s)


def test_refused_arguments_write_nothing(kinds):
    """n outside 1..512, null pointers and unset tables are refused by every read-out entry point, before any write."""
    vocab, lm, olm_, lift, g, H = setup(kinds, "word", True)
    table, _ = kinds
    clm = table["char3"][1]
    dev, V, T = torch.device("cuda"), len(vocab), 10
    eng = Eng(V)
    bs = BeamSearch(dev, STREAM, 2, 2 * T, T, 8, 0.99, 40, None, 0.0, 0.0, g)
    L = torch.cat([logits_for(s, T, V, lift, dev) for s in (1, 2)])
    bs.topk(eng, L, L.stride(0), 2 * T)
    ld = torch.tensor([T, T], dtype=torch.int32, device=dev)
    bs.search(eng, ld.data_ptr(), 2, T)
    n = 4
    tok = torch.full((2, n, T), -7, dtype=torch.int32, device=dev)
    cnt, nh = torch.full((2, n), -7, dtype=torch.int32, device=dev), torch.full((2,), -7, dtype=torch.int32, device=dev)
    sc, ap = torch.full((2, n), -7.0, device=dev), torch.full((2, n), -7.0, device=dev)
    empty_w, empty_c = _lib.WordLmTables(), _lib.LmTables()
    stream = torch.cuda.current_stream().cuda_stream

    def args(name, nn=n, state_i=bs.state_i.data_ptr(), out_count=nh.data_ptr(), tables=None):
        a = [bs.trie_par.data_ptr(), bs.trie_tok.data_ptr(), bs.trie_cap, state_i, bs.state_f.data_ptr(), None, 2, nn]
        if "_lm_" in name or "_wordlm_" in name:
            t = tables if tables is not None else (lm.tables(dev) if "_wordlm_" in name else clm.tables(dev))
            a += [C.byref(t), 1.0, 0.5]
        a += [tok.data_ptr(), T, cnt.data_ptr(), sc.data_ptr()] + ([ap.data_ptr()] if ("_lm_" in name or "_wordlm_" in name) else [])
        a += [out_count]
        if "_hot_" in name:
            a += [C.byref(g.tables(dev)), bs.slot_root.data_ptr()]
        return a + [stream]

    for name in NAMES.values():
        for bad in (dict(nn=0), dict(nn=513), dict(state_i=None), dict(out_count=None)):
            with pytest.raises(_lib.MasrB200Error, match="out of range|null pointer"):
                _lib.call(name, *args(name, **bad))
        if "_wordlm_" in name:
            with pytest.raises(_lib.MasrB200Error, match="tables not set"):
                _lib.call(name, *args(name, tables=empty_w))
        if "_lm_" in name:
            with pytest.raises(_lib.MasrB200Error, match="tables not set"):
                _lib.call(name, *args(name, tables=empty_c))
        if "_hot_" in name:
            a = args(name)
            a[-3] = None                                     # no graph
            with pytest.raises(_lib.MasrB200Error, match="hotword"):
                _lib.call(name, *a)
    torch.cuda.synchronize()
    for x in (tok, cnt, nh):
        assert (x == -7).all()
    assert (sc == -7.0).all() and (ap == -7.0).all()
    with pytest.raises(ValueError):
        bs.nbest(eng, 2, 9)                                  # past the beam size
    with pytest.raises(ValueError):
        BeamSearch(dev, ONE_SHOT, 1, T, T, 8).nbest(eng, 1, 2)
