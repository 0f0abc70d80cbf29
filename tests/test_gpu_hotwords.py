"""GPU (-m gpu): hotword biasing in the prefix beam search (the ``*_hot`` entry points through masr_b200.beam.BeamSearch)
against oracle/hotwords.py on the GPU's own top-k candidates, bit for bit (prefix, reported score, fused or approx score):
no LM, character LM and word LM, in the one-shot, streaming and pool forms, at beam 300 and 512; pool slots with
different lists, no list, a reset and a full region; token onsets unchanged by the feature."""
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
    p = str(tmp_path_factory.mktemp("lm") / "c.arpa")
    chars = synth.character_lm_arpa(p, seed=3, order=3, n_chars=80, n_sentences=600, vocab_size=300)
    ids = [cv.index(c) for c in chars]
    ev = synth.english_vocabulary()
    pw = str(tmp_path_factory.mktemp("wlm") / "w.arpa")
    synth.word_lm_arpa(pw, seed=3, order=3, n_words=120)
    o = owl.WordLM(pw, ev)
    letters = sorted({t for ch in o.lex.child for t in ch})
    # hotwords: runs of the lifted tokens (character vocab), lexicon words and word pairs (English vocab)
    c_hw = ["".join(cv[i] for i in ids[j:j + L]) for j, L in ((0, 2), (0, 4), (5, 3), (9, 2), (12, 5))]
    words = [w for w in o.lex.words if 2 <= len(w) <= 6][:6]
    w_hw = words + [words[0] + " " + words[1], "zz"[:1] + words[2][:2]]
    return {"none": (cv, None, None, ids, c_hw), "char": (cv, CharLM(p, cv), olm.read_arpa(p), ids, c_hw),
            "word": (ev, WordLM(pw, ev), o, letters + [o.space], w_hw)}


def logits_for(seed, T, V, lift, dev):
    _, lg = rand_posteriors(seed, T, V, peaky=3.0)
    lg[:, lift] += 2.5
    L = torch.zeros(T, (V + 15) // 16 * 16, device=dev)
    L[:, :V] = torch.from_numpy(lg).to(dev)
    return L


def cands(bs, rows):
    cid, clp, cn = bs.cand_id.cpu().numpy(), bs.cand_lp.cpu().numpy(), bs.cand_n.cpu().numpy()
    blp = bs.blank_lp.cpu().numpy() if bs.blank_lp is not None else np.zeros(len(cn), np.float32)
    return [[(int(cid[r, k]), clp[r, k]) for k in range(cn[r])] for r in rows], [blp[r] for r in rows]


def oracle(kind, olm_, vocab, cl, blp, beam, alpha, beta, H):
    if kind == "word":
        s = oh.WordLmSearchHot(olm_, alpha, beta, beam, hotwords=H)
        (score, approx, toks), = s.push(cl, blp).result()
        return toks, F(score), F(approx)
    (score, approx, toks), = oh.prefix_beam_search_hot(None, olm_, vocab, alpha, beta, beam, cands_per_frame=cl,
                                                      blank_logp_per_frame=blp, hotwords=H)
    return toks, F(score), F(approx)


def got(bs, b, kind):
    """(tokens, fused score, reported score (approx_ctc with an LM)), as the oracle returns them."""
    n = int(bs.count[b].item())
    return bs.out_tok[b, :n].cpu().tolist(), F(bs.fused[b].item()), F(bs.score[b].item())


AB = {"none": (0.0, 0.0), "char": (0.8, 1.0), "word": (1.0, 1.5)}


@pytest.mark.parametrize("beam", [300, 512])
@pytest.mark.parametrize("kind", ["none", "char", "word"])
def test_one_shot_equals_oracle(kinds, kind, beam):
    vocab, lm, olm_, lift, hws = kinds[kind]
    dev, V, T = torch.device("cuda"), len(vocab), 60
    g = HotwordGraph(hws, vocab, 2.0)
    H = oh.HotwordMatcher(g.tokens, 2.0)
    alpha, beta = AB[kind]
    eng = Eng(V)
    L = torch.cat([logits_for(s, T, V, lift, dev) for s in (1, 2, 3)])
    lens = [T, T // 2, T]
    bs = BeamSearch(dev, ONE_SHOT, 3, 3 * T, T, beam, 0.99, 40, lm, alpha, beta, g,
                    slot_root=torch.tensor([0, 0, -1], dtype=torch.int32, device=dev))
    plain = BeamSearch(dev, ONE_SHOT, 3, 3 * T, T, beam, 0.99, 40, lm, alpha, beta)
    ld = torch.tensor(lens, dtype=torch.int32, device=dev)
    for s in (bs, plain):
        s.topk(eng, L, L.stride(0), 3 * T)
        s.search(eng, ld.data_ptr(), 3, T)
    torch.cuda.synchronize()
    flipped = 0
    for b in range(3):
        cl, blp = cands(bs, range(b * T, b * T + lens[b]))
        want = oracle(kind, olm_, vocab, cl, blp, beam, alpha, beta, H if b < 2 else None)
        assert got(bs, b, kind) == want, (kind, b)
        flipped += got(plain, b, kind)[0] != want[0]
    assert got(bs, 2, kind) == got(plain, 2, kind)            # root -1: the search without hotwords, bit for bit
    assert flipped > 0, "the hotwords changed no result: the test does not exercise them"
    # token onsets: the hot search's read-out equals a host walk of its own trie and node clock, for the slots with
    # hotwords too, onsets strictly increase, and the slot without hotwords reads out the plain search's onsets
    fr_h, fr_p = bs.frames(eng, 3).cpu().numpy(), plain.frames(eng, 3).cpu().numpy()
    tp, tt, cap = bs.trie_par.cpu().numpy(), bs.trie_tok.cpu().numpy(), bs.trie_cap
    nc = cap // 5
    for b in range(3):
        par, tok, onset = tp[b * cap:b * cap + nc], tt[b * cap:b * cap + nc], tt[b * cap + 2 * nc:b * cap + 3 * nc]
        n, node, walk = int(bs.count[b]), 0, []
        for t in bs.out_tok[b, :n].cpu().tolist():
            node = int(np.nonzero((par[1:] == node) & (tok[1:] == t))[0][0]) + 1
            walk.append(int(onset[node]))
        assert fr_h[b, :n].tolist() == walk and all(x < y for x, y in zip(walk, walk[1:])), b
    assert np.array_equal(fr_h[2, :int(bs.count[2])], fr_p[2, :int(plain.count[2])])


@pytest.mark.parametrize("kind", ["none", "char", "word"])
def test_streaming_equals_one_shot(kinds, kind):
    vocab, lm, olm_, lift, hws = kinds[kind]
    dev, V, T, beam = torch.device("cuda"), len(vocab), 75, 300
    g = HotwordGraph(hws, vocab, 1.5)
    H = oh.HotwordMatcher(g.tokens, 1.5)
    alpha, beta = AB[kind]
    eng = Eng(V)
    L = logits_for(7, T, V, lift, dev)
    for chunk in (16, 7):                                    # the stream pool's chunk sizes (16 frames, and an odd one)
        sb = BeamSearch(dev, STREAM, 1, chunk, T, beam, 0.99, 40, lm, alpha, beta, g)
        ld = torch.zeros(1, dtype=torch.int32, device=dev)
        done, cl_all, blp_all = 0, [], []
        while done < T:
            n = min(chunk, T - done)
            sb.topk(eng, L[done:done + n], L.stride(0), n)
            ld.fill_(n)
            sb.search(eng, ld.data_ptr(), 1, chunk, resume=1 if done else 0)
            torch.cuda.synchronize()
            cl, blp = cands(sb, range(n))
            cl_all += cl
            blp_all += blp
            done += n
        assert got(sb, 0, kind) == oracle(kind, olm_, vocab, cl_all, blp_all, beam, alpha, beta, H), chunk


@pytest.mark.parametrize("kind", ["none", "char", "word"])
def test_pool_slots_with_their_own_lists(kinds, kind):
    """Four slots: list A, list B, the default list and none; pushed unevenly, slot 0 reset and given list B mid-run;
    slot 1's region filled to max_hotword_nodes."""
    vocab, lm, olm_, lift, hws = kinds[kind]
    dev, V, S, R, beam, frames_cap = torch.device("cuda"), len(vocab), 4, 12, 64, 200
    alpha, beta = AB[kind]
    eng = Eng(V)
    gA, gB, gD = (HotwordGraph(h, vocab, 2.0) for h in (hws[:2], hws[2:], hws[1:3]))
    buf = HotwordBuffer(dev, S + 1, gB.nodes)                # slot 1's region exactly full
    buf.put(0, gA)
    buf.put(1, gB)
    buf.put(S, gD)                                           # the pool default
    roots = torch.tensor([buf.root(0), buf.root(1), buf.root(S), -1], dtype=torch.int32, device=dev)
    bs = BeamSearch(dev, POOL, S, S * R, frames_cap, beam, 0.99, 40, lm, alpha, beta, buf, slot_root=roots)
    Hs = [oh.HotwordMatcher(x.tokens, 2.0) for x in (gA, gB, gD)] + [None]
    utt = {s: logits_for(40 + s, 150, V, lift, dev) for s in range(S)}
    pos, hist = [0] * S, [([], []) for _ in range(S)]
    plan = [(12, 5, 12, 3), (12, 0, 7, 12), ("reset", 12, 12, 0), (12, 12, 4, 9)]
    for step, p in enumerate(plan):
        if p[0] == "reset":
            bs.fresh[0] = 1
            bs.trie_par[bs.trie_cap // 5:bs.trie_cap].fill_(-1)
            buf.put(0, gB)
            Hs[0] = Hs[1]
            utt[0], pos[0], hist[0] = logits_for(90, 150, V, lift, dev), 0, ([], [])
            p = (12,) + p[1:]
        L = torch.zeros(S * R, utt[0].shape[1], device=dev)
        for s in range(S):
            L[s * R:s * R + p[s]] = utt[s][pos[s]:pos[s] + p[s]]
        bs.topk(eng, L, L.stride(0), S * R)
        ld = torch.tensor(p, dtype=torch.int32, device=dev)
        bs.search(eng, ld.data_ptr(), S, R)
        torch.cuda.synchronize()
        for s in range(S):
            if p[s] == 0:
                continue
            cl, blp = cands(bs, range(s * R, s * R + p[s]))
            hist[s][0].extend(cl)
            hist[s][1].extend(blp)
            pos[s] += p[s]
            assert got(bs, s, kind) == oracle(kind, olm_, vocab, hist[s][0], hist[s][1], beam, alpha, beta, Hs[s]), (step, s)
