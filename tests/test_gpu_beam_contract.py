"""The CTC prefix beam search kernels (csrc/beam.cu: no LM, character LM, word LM; one-shot, streaming and pool forms)
against a float64 CTC forward and, entry by entry, against the float32 restatements (oracle/beam.py, lm.py, word_lm.py),
at their selection, tie, capacity and LM-order edges.

The streaming form's saved state is the whole ranked beam: per entry its node, p_b, p_nb and score, and the trie spells its
prefix.  So every rank is compared, not only the best one: a wrong survivor or a wrong p_b / p_nb split deep in the beam
fails here even when it would not change the best prefix yet.  Where no live prefix is ever pruned (nbeam < beam at every
frame) the search is exact, and then every entry's p_b and p_nb equal the float64 CTC forward of its prefix.

Conventions of tests/kernel_contract.py: candidate rows past a valid length (and slots past a row's count) hold garbage
(random ids, count 40, log-probability 0), outputs start as NaN or sentinels, and what a form must not write is checked
untouched.  CPU part: the float64 references themselves, the restatement's log-sum-exp and the launcher rejections."""
import ctypes as C
import itertools
import math

import numpy as np
import pytest
import torch

from oracle import beam as obeam, lm as olm, word_lm as owl

F = np.float32
NEG = -math.inf
BEAM_CAP, BK_MAX = 512, 40
SENT = -7777                     # sentinel of the int outputs
V = 4233

# Largest errors against float64, measured on an H100 (the kernel equals the restatement bit for bit, so the CPU measures
# the same numbers): see the commit message.  Error scale: |x - x64| / (1 + |x64|) on log-probabilities.
TOL_CTC = 8e-7                   # p_b, p_nb, score of a lossless search vs ctc_forward64 (measured 2.0e-7)
TOL_LM = 1.2e-6                  # fused score vs forward64 + alpha lnP64 + beta |l|, approx vs its definition (2.9e-7)


# ---- float64 references --------------------------------------------------------------------------------------------------
def lae(a, b):
    if a == NEG:
        return b
    if b == NEG:
        return a
    m = max(a, b)
    return m + math.log(math.exp(a - m) + math.exp(b - m))


def ctc_forward64(cands, labels, blank):
    """(ln p_b, ln p_nb) of ``labels`` after the frames ``cands`` ([(id, ln p)] per frame; a token outside a frame's list
    has probability 0): the CTC alpha recursion over the extended label (blank, l1, blank, l2, .., blank) in float64;
    p_b = the final blank state, p_nb = the final label state."""
    ext = [blank]
    for c in labels:
        ext += [c, blank]
    S = len(ext)
    alpha = [NEG] * S
    alpha[0] = 0.0                                   # before the first frame: the empty alignment
    start = True
    for fr in cands:
        p = {}
        for c, lp in fr:
            p[int(c)] = lae(p.get(int(c), NEG), float(lp))
        new = [NEG] * S
        for s in range(S):
            if start:                                    # the first frame enters at the first blank or first label
                prev = 0.0 if s in (0, 1) else NEG
            else:
                prev = alpha[s]
                if s >= 1:
                    prev = lae(prev, alpha[s - 1])
                if s >= 2 and ext[s] != blank and ext[s] != ext[s - 2]:
                    prev = lae(prev, alpha[s - 2])
            e = p.get(ext[s], NEG)
            new[s] = NEG if prev == NEG or e == NEG else prev + e
        alpha, start = new, False
    if start:
        return (0.0, NEG) if not labels else (NEG, NEG)
    return alpha[S - 1], (alpha[S - 2] if labels else NEG)


def collapse(path, blank):
    out, prev = [], None
    for c in path:
        if c != blank and c != prev:
            out.append(c)
        prev = c
    return tuple(out)


def enumerate64(cands, blank):
    """{labels: (ln p_b, ln p_nb)} by summing every alignment of the candidate lists (tiny cases only)."""
    mass = {}
    for path in itertools.product(*[[(int(c), float(lp)) for c, lp in fr] for fr in cands]):
        ids = [c for c, _ in path]
        lp = sum(l for _, l in path)
        key = collapse(ids, blank)
        pb, pnb = mass.get(key, (NEG, NEG))
        mass[key] = (lae(pb, lp), pnb) if ids[-1] == blank else (pb, lae(pnb, lp))
    return mass


class Arpa64:
    """lnP(w | window) by the standard backoff rule in float64, straight from the ARPA text (OOV or <unk> -> -1000)."""

    def __init__(self, path):
        self.ng, n = {}, 0
        for ln in open(path, encoding="utf-8"):
            s = ln.strip()
            if s.startswith("\\") and s.endswith("-grams:"):
                n = int(s[1:s.index("-")])
                continue
            if n and s and not s.startswith("\\"):
                f = s.split()
                self.ng[tuple(f[1:n + 1])] = (float(f[0]) * math.log(10), float(f[n + 1]) * math.log(10) if len(f) == n + 2 else 0.0)
        self.order = max(len(k) for k in self.ng)
        self.uni = {k[0] for k in self.ng if len(k) == 1}

    def lnp(self, ctx, w, top=None):
        """``top``: the longest history length looked up (default N - 1)."""
        ok = lambda x: x in self.uni and x != "<unk>"
        if not ok(w) or not all(ok(x) for x in ctx):
            return -1000.0
        acc = 0.0
        for L in range(self.order - 1 if top is None else top, -1, -1):
            h = tuple(ctx[len(ctx) - L:]) if L else ()
            if h + (w,) in self.ng:
                return acc + self.ng[h + (w,)][0]
            if L and h in self.ng:
                acc += self.ng[h][1]
        return -1000.0

    def window(self, words):
        n1 = self.order - 1
        w = list(words[max(0, len(words) - n1):]) if n1 else []
        return ["<s>"] * (n1 - len(w)) + w

    def prefix_lnp(self, words):
        return sum(self.lnp(self.window(words[:j]), words[j]) for j in range(len(words)))

    def sentence_lnp(self, words):
        N = self.order
        sent = ["<s>"] * N if not words else ["<s>"] * (N - 1) + list(words)
        sent.append("</s>")
        return sum(self.lnp(sent[i:i + N - 1], sent[i + N - 1]) for i in range(len(sent) - N + 1))


def rel(x, x64, scale=None):
    """|x - x64| / (1 + scale), scale = |x64| or, for a sum that cancels, the sum of its terms' magnitudes."""
    if x64 == NEG or x == NEG:
        assert x == x64, (x, x64)
        return 0.0
    return abs(float(x) - x64) / (1.0 + (abs(x64) if scale is None else scale))


# ---- candidate lists -----------------------------------------------------------------------------------------------------
def lossless_cands(seed, T, letters, blank, K=(3,)):
    """Small hand-built candidate lists: blank and K - 1 of ``letters`` per frame, Dirichlet probabilities.  With three
    letters, K = 3 and T = 7 the search holds 112 .. 344 live prefixes: below beam 512, so nothing is pruned."""
    rng = np.random.default_rng(seed)
    letters = [c for c in letters if c != blank]
    out = []
    for _ in range(T):
        k = int(rng.choice(K))
        ids = [blank] + [int(c) for c in rng.choice(letters, k - 1, replace=False)]
        p = rng.dirichlet(np.ones(k))
        out.append([(int(c), F(math.log(q))) for c, q in zip(ids, p)])
    return out


def grid_logits(seed, T, Vv, ids, blank, low, n_hi=12):
    """Logits on a coarse grid (few distinct values per frame, so ctc_topk emits tied candidates), lifted tokens drawn from
    a small id set (repeats and merges); ``low`` sets the tail: -8 keeps >= 40 candidates below cutoff_prob 1.0."""
    rng = np.random.default_rng(seed)
    L = np.full((T, Vv), low, np.float32)
    for t in range(T):
        pick = rng.choice(ids, min(n_hi, len(ids)), replace=False)
        L[t, pick] = rng.choice([0.0, 1.0, 2.0, 3.0], len(pick))
        if rng.random() < 0.6:
            L[t, blank] = rng.choice([1.0, 2.0, 4.0])
    return L


def topk_rows(rt, logits, top_n, cut, blank):
    """ctc_topk (with ln p_blank) on the device -> host (cid [R,40], clp, cn, blp)."""
    R, Vv = logits.shape
    ldl = (Vv + 15) // 16 * 16
    L = torch.zeros(R, ldl, device=rt.dev)
    L[:, :Vv] = torch.from_numpy(logits).to(rt.dev)
    cid = torch.zeros(R, BK_MAX, dtype=torch.int32, device=rt.dev); clp = torch.zeros(R, BK_MAX, device=rt.dev)
    cn = torch.zeros(R, dtype=torch.int32, device=rt.dev); blp = torch.zeros(R, device=rt.dev)
    rt.call("masr_ctc_topk_blank_f32", L.data_ptr(), ldl, R, Vv, top_n, cut, blank, cid.data_ptr(), clp.data_ptr(),
            cn.data_ptr(), blp.data_ptr(), rt.st())
    torch.cuda.synchronize()
    cn_h = cn.cpu().numpy()
    return [[(int(i), F(l)) for i, l in zip(cid[r, :cn_h[r]].cpu().numpy(), clp[r, :cn_h[r]].cpu().numpy())] for r in range(R)], \
        [F(x) for x in blp.cpu().numpy()]


class Rows:
    """Candidate rows of B utterances, bstride rows apart, on the device; garbage wherever no valid candidate is."""

    def __init__(self, rt, frames, blps=None, bstride=None, Vv=V, seed=0):
        B = len(frames)
        self.bstride = bstride or max(1, max(len(f) for f in frames))
        R = B * self.bstride
        rng = np.random.default_rng(1000 + seed)
        cid = rng.integers(0, Vv, (R, BK_MAX)).astype(np.int32)
        clp = np.zeros((R, BK_MAX), np.float32)
        cn = np.full(R, BK_MAX, np.int32)
        blp = np.zeros(R, np.float32)
        for b, fr in enumerate(frames):
            for t, row in enumerate(fr):
                r = b * self.bstride + t
                cn[r] = len(row)
                for k, (c, lp) in enumerate(row):
                    cid[r, k], clp[r, k] = c, lp
                blp[r] = blps[b][t] if blps is not None else F(-1.0)
        self.frames, self.blps = frames, blps
        self.cid, self.clp = torch.from_numpy(cid).to(rt.dev), torch.from_numpy(clp).to(rt.dev)
        self.cn, self.blp = torch.from_numpy(cn).to(rt.dev), torch.from_numpy(blp).to(rt.dev)

    def ptrs(self, t0):
        return (self.cid.data_ptr() + 4 * BK_MAX * t0, self.clp.data_ptr() + 4 * BK_MAX * t0, self.cn.data_ptr() + 4 * t0,
                self.blp.data_ptr() + 4 * t0)


class Search:
    """Buffers of one search configuration for B utterances of up to ``frames`` frames, trie sized by the contract
    trie_cap = 5 (frames beam + 1); ``run`` launches one form, ``entries`` reads the saved beam back through the trie."""

    def __init__(self, rt, mode, beam, B, frames, blank=0, lm=None, alpha=0.0, beta=0.0, tok_stride=None):
        self.rt, self.mode, self.beam, self.B, self.blank = rt, mode, beam, B, blank
        self.lm, self.alpha, self.beta = lm, alpha, beta
        self.cap = 5 * (frames * beam + 1)
        self.name = {"plain": "masr_ctc_prefix_beam", "char": "masr_ctc_prefix_beam_lm", "word": "masr_ctc_prefix_beam_wordlm"}[mode]
        si, sf = C.c_int64(0), C.c_int64(0)
        rt.call(self.name + "_state_size", C.byref(si), C.byref(sf))
        dev = rt.dev
        self.pool = torch.full((B * (BEAM_CAP + BEAM_CAP * BK_MAX),), float("nan"), device=dev)
        self.tp = torch.full((B * self.cap,), -1, dtype=torch.int32, device=dev)
        self.tt = torch.full((B * self.cap,), SENT, dtype=torch.int32, device=dev)
        self.sti = torch.full((B, si.value), SENT, dtype=torch.int32, device=dev)
        self.stf = torch.full((B, sf.value), float("nan"), device=dev)
        self.tok_stride = tok_stride or max(1, frames)
        self.otok = torch.full((B, self.tok_stride), SENT, dtype=torch.int32, device=dev)
        self.on = torch.full((B,), SENT, dtype=torch.int32, device=dev)
        self.osc = torch.full((B,), float("nan"), device=dev)
        self.oap = torch.full((B,), float("nan"), device=dev)
        self.fresh = torch.ones(B, dtype=torch.int32, device=dev)

    def run(self, form, rows, lens, t0=0, resume=0):
        rt = self.rt
        cid, clp, cn, blp = rows.ptrs(t0)
        ld = torch.tensor(lens, dtype=torch.int32, device=rt.dev)
        lm = [blp] if self.mode != "plain" else []
        lmw = [C.byref(self.lm.tables(rt.dev)), self.alpha, self.beta] if self.mode != "plain" else []
        head = [cid, clp, cn] + lm + [rows.bstride, ld.data_ptr(), self.B, self.beam, self.blank] + lmw + \
               [self.pool.data_ptr(), self.tp.data_ptr(), self.tt.data_ptr(), self.cap]
        tail = [self.otok.data_ptr(), self.tok_stride, self.on.data_ptr(), self.osc.data_ptr()] + \
               ([self.oap.data_ptr()] if self.mode != "plain" else []) + [rt.st()]
        st = [self.sti.data_ptr(), self.stf.data_ptr()]
        if form == "one":
            rt.call(self.name, *head, *tail)
        elif form == "stream":
            rt.call(self.name + "_stream", *head, *st, resume, *tail)
        else:
            rt.call(self.name + "_pool", *head, *st, self.fresh.data_ptr(), *tail)
        torch.cuda.synchronize()

    def entries(self, b):
        """The saved beam of utterance b, rank order: [(prefix, p_b, p_nb, score, node)] (+ nbeam, nnodes checks)."""
        sti, stf = self.sti[b].cpu().numpy(), self.stf[b].cpu().numpy()
        node_cap = self.cap // 5
        tp = self.tp[b * self.cap: b * self.cap + node_cap].cpu().numpy()
        tt = self.tt[b * self.cap: b * self.cap + node_cap].cpu().numpy()
        nbeam, nnodes = int(sti[3 * BEAM_CAP]), int(sti[3 * BEAM_CAP + 1])
        assert 1 <= nnodes <= node_cap and 0 <= nbeam <= self.beam
        out = []
        for r in range(nbeam):
            node, par, last = int(sti[r]), int(sti[BEAM_CAP + r]), int(sti[2 * BEAM_CAP + r])
            assert 0 <= node < nnodes
            toks, x = [], node
            while x > 0:
                toks.append(int(tt[x]))
                x = int(tp[x])
            toks = tuple(toks[::-1])
            assert (par, last) == ((-1, -1) if node == 0 else (int(tp[node]), int(tt[node])))
            pb, pnb, sc = F(stf[r]), F(stf[BEAM_CAP + r]), F(stf[2 * BEAM_CAP + r])
            assert obeam.logaddexp32(pb, pnb).view(np.int32) == sc.view(np.int32), (r, pb, pnb, sc)
            out.append((toks, pb, pnb, sc, node))
        assert len({e[0] for e in out}) == nbeam, "two beam entries spell the same prefix"
        assert all(out[i][3] >= out[i + 1][3] for i in range(nbeam - 1))
        return out

    def best(self, b):
        n = int(self.on[b])
        return list(self.otok[b, :n].cpu().numpy()), F(self.osc[b].item()), F(self.oap[b].item())


def bits(t):
    return t.reshape(-1).view(torch.int32) if t.is_floating_point() else t.reshape(-1)


def same_beam(got, want):
    """got: Search.entries; want: [(prefix, float32 score)] in rank order — prefix and score bit for bit at every rank."""
    assert len(got) == len(want), (len(got), len(want))
    for r, (g, (toks, sc)) in enumerate(zip(got, want)):
        assert g[0] == tuple(toks), (r, g[0], toks)
        assert g[3].view(np.int32) == F(sc).view(np.int32), (r, g[3], sc)


def restate(mode, frames, blps, beam, blank, lm=None, vocab=None, alpha=0.0, beta=0.0):
    """The restatement's whole beam [(prefix, score)] and its reported best (prefix, score, approx)."""
    T = len(frames)
    if mode == "plain":
        out = obeam.prefix_beam_search(np.zeros((T, 1)), beam_size=beam, blank=blank, nbest=beam, cands_per_frame=frames)
        return [(tuple(t), F(s)) for s, t in out], (out[0][1], F(out[0][0]), F(out[0][0]))
    if mode == "char":
        out = olm.prefix_beam_search_lm(np.zeros((T, 1)), lm, vocab, alpha, beta, beam_size=beam, blank=blank, nbest=beam,
                                        cands_per_frame=frames, blank_logp_per_frame=blps)
        return [(tuple(t), F(s)) for s, _, t in out], (out[0][2], F(out[0][0]), F(out[0][1]))
    s = owl.WordLmSearch(lm, alpha, beta, beam, blank).push(frames, blps)
    (sc, ap, toks), = s.result(1)
    return [(s.toks_of[n], obeam.logaddexp32(pb, pnb)) for n, pb, pnb in s.beam], (toks, F(sc), F(ap))


# ---- CPU part ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed,T,blank", [(0, 4, 0), (1, 5, 2), (2, 3, 1), (3, 5, 0)])
def test_ctc_forward64_equals_enumeration(seed, T, blank):
    cands = lossless_cands(seed, T, [0, 1, 2, 3], blank, K=(2, 3))
    cands[0] = cands[0][1:]                                   # a frame without blank
    cands[1] = cands[1] + [(9, F(NEG))]                       # a -inf candidate: probability 0
    mass = enumerate64(cands, blank)
    assert len(mass) > 3
    for labels, (pb, pnb) in mass.items():
        fb, fnb = ctc_forward64(cands, list(labels), blank)
        for a, b in ((fb, pb), (fnb, pnb)):
            assert (a == NEG and b == NEG) or abs(a - b) < 1e-12, (labels, a, b)
    assert ctc_forward64(cands, [7], blank) == (NEG, NEG)     # a token no frame lists
    assert ctc_forward64([], [], blank) == (0.0, NEG)


@pytest.mark.parametrize("mode", ["plain", "char"])
def test_restatement_lossless_equals_float64(tmp_path, mode):
    """The float64 tolerances, derived on the CPU from the restatement (which the kernel equals bit for bit): in lossless
    searches every entry's score == ctc_forward64 (character LM: + alpha lnP64 + beta |l|, lnP64 from the ARPA text)."""
    from masr_b200 import synth
    vocab = synth.vocabulary(V)
    letters, lm, a64, alpha, beta = [1, 2, 3], None, None, 0.0, 0.0
    if mode == "char":
        p = str(tmp_path / "o3.arpa")
        letters = [vocab.index(c) for c in synth.character_lm_arpa(p, seed=3, order=3, n_chars=24, n_sentences=600)[:2]] + [1]
        lm, a64, alpha, beta = olm.read_arpa(p), Arpa64(p), 0.7, 1.3
    worst, most = 0.0, 0
    for seed in range(20):
        frames = lossless_cands(seed, 7, letters, 0)
        for t in range(1, 8):
            out = olm.prefix_beam_search_lm(np.zeros((t, 1)), lm, vocab, alpha, beta, beam_size=BEAM_CAP, nbest=BEAM_CAP,
                                            cands_per_frame=frames[:t], blank_logp_per_frame=[F(-1.0)] * t)
            most = max(most, len(out))
        for s, approx, toks in out:
            pb, pnb = ctc_forward64(frames, toks, 0)
            want = lae(pb, pnb)
            scale = abs(want)
            if mode == "char":
                words = [vocab[c] for c in toks]
                lm_t, len_t, sent_t = alpha * a64.prefix_lnp(words), beta * len(toks), alpha * a64.sentence_lnp(words)
                scale += abs(lm_t) + abs(len_t)
                want += lm_t + len_t
                worst = max(worst, rel(F(approx), s - len_t - sent_t, abs(s) + abs(len_t) + abs(sent_t)))
            worst = max(worst, rel(F(s), want, scale))
    print(f"[max error] restatement ({mode}) vs float64: {worst:.3g}, most live prefixes {most}")
    assert 100 < most < BEAM_CAP
    assert worst < (TOL_CTC if mode == "plain" else TOL_LM)


def test_logaddexp32_against_float64():
    """exp32_det, log1p32_det, logaddexp32 over a sweep with their edges: d = 0, d around -87, u in {0, 2^-126, 1}."""
    ds = np.r_[0.0, -1e-30, -1e-7, np.linspace(-86.99, 0, 4001), -86.999, -87.0, np.nextafter(F(-87.0), F(0))]
    worst_e = 0.0
    for d in ds.astype(np.float32):
        got, want = float(obeam.exp32_det(d)), math.exp(float(d))
        worst_e = max(worst_e, abs(got - want) / want)
    # below -87 the result is flushed to 0 (exp(-87) = 1.6e-38, next to the smallest normal float32)
    for d in (np.nextafter(F(-87.0), F(-100)), F(-87.01), F(-100.0), F(-3e38)):
        assert float(obeam.exp32_det(d)) == 0.0
    assert float(obeam.exp32_det(F(0.0))) == 1.0
    us = np.r_[0.0, 2.0 ** -126, 1e-30, np.linspace(0, 1, 4001), 1.0].astype(np.float32)
    worst_l = 0.0
    for u in us:
        got, want = float(obeam.log1p32_det(u)), math.log1p(float(u))
        worst_l = max(worst_l, abs(got - want) / max(want, 2.0 ** -149))
    assert float(obeam.log1p32_det(F(0.0))) == 0.0
    rng = np.random.default_rng(0)
    worst_a = 0.0
    for a, b in rng.uniform(-120, 5, (4000, 2)).astype(np.float32):
        got, want = float(obeam.logaddexp32(a, b)), lae(float(a), float(b))
        worst_a = max(worst_a, abs(got - want) / (1.0 + abs(want)))
    assert obeam.logaddexp32(F(NEG), F(-3.0)) == F(-3.0) and obeam.logaddexp32(F(-3.0), F(NEG)) == F(-3.0)
    print(f"[max error] exp32_det {worst_e:.3g} rel, log1p32_det {worst_l:.3g} rel, logaddexp32 {worst_a:.3g}")
    # "a few ulp" of oracle/beam.py, as numbers: exp32_det and log1p32_det within 8 ulp (2^-24) relative, logaddexp32 within
    # 2 ulp of 1 + |result| (measured: 4, 3.2 and 1)
    assert worst_e < 4 * 2.0 ** -24 * 2 and worst_l < 4 * 2.0 ** -24 * 2 and worst_a < 2 * 2.0 ** -23


ENTRY_POINTS = [m + f for m in ("masr_ctc_prefix_beam", "masr_ctc_prefix_beam_lm", "masr_ctc_prefix_beam_wordlm")
                for f in ("", "_stream", "_pool")]


@pytest.fixture(scope="module")
def lib():
    from masr_b200 import build, _lib
    build.build()                      # nvcc cross-compiles sm_90a without a GPU
    return _lib.load()


@pytest.mark.parametrize("name", ENTRY_POINTS)
def test_launcher_rejects_beam_size_out_of_range(lib, name):
    """beam_size 0 and 513 (BEAM_CAP + 1) are refused before anything is launched, by each of the nine entry points."""
    from masr_b200 import _lib
    buf = np.zeros(64, np.int32)
    p = buf.ctypes.data
    tables = []
    if "_wordlm" in name:
        t = _lib.WordLmTables(keys=p, vals=p, lex_off=p, lex_tok=p, lex_next=p, lex_word=p, order=2, nodes=1, space=3)
        tables = [C.byref(t), 1.0, 0.5]
    elif "_lm" in name:
        t = _lib.LmTables(keys=p, vals=p, tok2lm=p, order=3)
        tables = [C.byref(t), 1.0, 0.5]
    lm = [p] if tables else []
    for beam in (0, BEAM_CAP + 1, -1):
        head = [p, p, p] + lm + [1, p, 1, beam, 0] + tables + [p, p, p, 100]
        tail = [p, 1, p, p] + ([p] if tables else []) + [None]
        if name.endswith("_stream"):
            args = head + [p, p, 0] + tail
        elif name.endswith("_pool"):
            args = head + [p, p, p] + tail
        else:
            args = head + tail
        with pytest.raises(_lib.MasrB200Error, match=f"beam_size={beam} out of range"):
            _lib.call(name, *args)
    assert buf.tolist() == [0] * 64                          # nothing written


# ---- GPU part ------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def rt():
    from kernel_contract import runtime
    return runtime()


BEAMS = [1, 2, 31, 32, 33, 255, 256, 257, 511, 512]


@pytest.mark.gpu
@pytest.mark.parametrize("cut", [1.0, 0.99])
@pytest.mark.parametrize("beam", BEAMS)
def test_whole_beam_equals_restatement(rt, beam, cut):
    """Tied candidates from coarse-grid logits; cutoff 1.0 / top 40 gives K = 40 every frame (a pool of 512 + 40 beam
    entries); the streaming form fed in two chunks, the whole beam compared after each; one-shot and pool == streaming."""
    T, blank = 6, 0
    ids = list(range(2, 32))
    frames, blps = topk_rows(rt, grid_logits(beam, T, V, ids, blank, -8.0 if cut == 1.0 else -20.0), 40, cut, blank)
    if cut == 1.0:
        assert all(len(f) == BK_MAX for f in frames)
    assert any(len({lp for _, lp in f}) < len(f) for f in frames)             # tied candidates
    rows = Rows(rt, [frames], [blps], bstride=T + 3)
    s = Search(rt, "plain", beam, 1, T)
    for t0, n in ((0, 2), (2, T - 2)):
        s.run("stream", rows, [n], t0, resume=t0 > 0)
        want, (btoks, bsc, _) = restate("plain", frames[:t0 + n], None, beam, blank)
        same_beam(s.entries(0), want)
        assert s.best(0)[:2] == (btoks, bsc)
    stream = s.best(0)
    one = Search(rt, "plain", beam, 1, T)
    one.run("one", rows, [T])
    pool = Search(rt, "plain", beam, 1, T)
    pool.run("pool", rows, [2])
    pool.run("pool", rows, [T - 2], 2)
    for o in (one, pool):
        assert o.best(0)[:2] == stream[:2]
    assert torch.equal(pool.sti, s.sti) and torch.equal(bits(pool.stf), bits(s.stf))


def tie_frames(n_tok, blank):
    """Two frames of blank + n_tok tied tokens: frame 2 makes n_tok (n_tok - 1) children of one score, spread over pool
    chunks, below the existing prefixes — the threshold of a beam of 40 .. 512 falls inside that tie group."""
    toks = [t for t in range(1, n_tok + 2) if t != blank][:n_tok]
    row = [(blank, F(math.log(0.5)))] + [(t, F(math.log(0.5 / n_tok))) for t in toks]
    return [row, list(row), [(blank, F(math.log(0.7)))] + [(t, F(math.log(0.3 / n_tok))) for t in toks[::-1]]]


@pytest.mark.gpu
@pytest.mark.parametrize("beam", [33, 257, 511, 512])
def test_threshold_inside_a_tie_group_spanning_chunks(rt, beam):
    """The tie rule where it decides the survivors: existing prefixes by rank, then children by (parent rank, candidate
    order).  1482 tied children span three 512-entry compaction chunks; at beam 512 the parked tied entries meet the
    entries above the threshold exactly.  A third frame reverses the candidate order under tied parents."""
    frames = tie_frames(39, 0)
    rows = Rows(rt, [frames], bstride=4)
    s = Search(rt, "plain", beam, 1, 3)
    for t in range(3):
        s.run("stream", rows, [1], t, resume=t > 0)
        want, _ = restate("plain", frames[:t + 1], None, beam, 0)
        got = s.entries(0)
        same_beam(got, want)
        if t == 1:
            sc = [e[3] for e in got]
            assert sc[-1] == sc[-2] and sum(x == sc[-1] for x in sc) < 39 * 38      # cut inside the tie group
    # an existing prefix tied with a new child: both score ln(0.25); the existing one ranks first
    f2 = [[(0, F(math.log(0.5))), (5, F(math.log(0.5)))], [(0, F(math.log(0.5))), (6, F(math.log(0.5)))]]
    rows = Rows(rt, [f2], bstride=2)
    s = Search(rt, "plain", 4, 1, 2)
    s.run("stream", rows, [2])
    want, _ = restate("plain", f2, None, 4, 0)
    got = s.entries(0)
    same_beam(got, want)
    assert [e[0] for e in got] == [(), (5,), (6,), (5, 6)] and len({e[3] for e in got}) == 1


@pytest.fixture(scope="module")
def char_lms(tmp_path_factory):
    from masr_b200 import synth
    from masr_b200.lm import CharLM
    vocab = synth.vocabulary(V)
    out = {}
    for order in (1, 2, 3, 6):
        p = str(tmp_path_factory.mktemp("lm") / f"o{order}.arpa")
        chars = synth.character_lm_arpa(p, seed=order, order=order, n_chars=24, n_sentences=600)
        out[order] = (olm.read_arpa(p), CharLM(p, vocab), [vocab.index(c) for c in chars], Arpa64(p))
    return vocab, out


def lossless_check(s, frames, blank, lm64=None, vocab=None, alpha=0.0, beta=0.0):
    worst = 0.0
    for toks, pb, pnb, sc, _ in s.entries(0):
        fb, fnb = ctc_forward64(frames, toks, blank)
        if lm64 is None:
            worst = max(worst, rel(pb, fb), rel(pnb, fnb), rel(sc, lae(fb, fnb)))
        else:
            lm_t, len_t = alpha * lm64.prefix_lnp([vocab[c] for c in toks]), beta * len(toks)
            worst = max(worst, rel(sc, lae(fb, fnb) + lm_t + len_t, abs(lae(fb, fnb)) + abs(lm_t) + abs(len_t)))
    return worst


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["plain", "char"])
def test_lossless_beam_equals_float64(rt, char_lms, mode):
    """Small T and K with up to a few hundred live prefixes at beam 512, so nothing is ever pruned: every entry's p_b, p_nb
    and score == ctc_forward64 of its prefix (character LM: + alpha lnP64 + beta |l|; approx == its float64 definition)."""
    vocab, d = char_lms
    o, clm, ids, a64 = d[3]
    alpha, beta = (0.0, 0.0) if mode == "plain" else (0.7, 1.3)
    letters = ids[:2] + [1] if mode == "char" else [1, 2, 3]          # char: two LM characters and <unk> (OOV)
    worst, apx, most = 0.0, 0.0, 0
    for seed in range(12):
        frames = lossless_cands(seed, 7, letters, 0)
        rows = Rows(rt, [frames], [[F(-1.0)] * 7], bstride=7)
        s = Search(rt, mode, BEAM_CAP, 1, 7, lm=clm if mode == "char" else None, alpha=alpha, beta=beta)
        for t in range(7):                                              # one frame per call: nbeam < beam at every frame
            s.run("stream", rows, [1], t, resume=t > 0)
            most = max(most, len(s.entries(0)))
        assert most < BEAM_CAP
        want, (btoks, bsc, bap) = restate(mode, frames, [F(-1.0)] * 7, BEAM_CAP, 0, o, vocab, alpha, beta)
        same_beam(s.entries(0), want)
        worst = max(worst, lossless_check(s, frames, 0, a64 if mode == "char" else None, vocab, alpha, beta))
        if mode == "char":
            toks, sc, ap = s.best(0)
            len_t, sent_t = len(toks) * beta, alpha * a64.sentence_lnp([vocab[c] for c in toks])
            apx = max(apx, rel(ap, float(sc) - len_t - sent_t, abs(float(sc)) + abs(len_t) + abs(sent_t)))
    print(f"[max error] lossless {mode}: entries {worst:.3g}, approx {apx:.3g}, most live prefixes {most}")
    assert most > 100
    assert worst < (TOL_CTC if mode == "plain" else TOL_LM) and apx < TOL_LM


@pytest.mark.gpu
@pytest.mark.parametrize("blank", [0, 2116, V - 1])
def test_candidate_row_edges(rt, char_lms, blank):
    """A -inf candidate log-probability, frames with blank only and with one non-blank token only, a repeated token across
    them — at blank 0, a middle id and V - 1, plain and character LM; lossless, so float64 applies too."""
    vocab, d = char_lms
    o, clm, ids, a64 = d[2]
    a, b, c = ids[0], ids[1], 1
    assert blank not in (a, b, c)
    lg = lambda p: F(math.log(p))
    frames = [[(a, lg(0.6)), (blank, lg(0.3)), (b, F(NEG))], [(blank, F(0.0))], [(a, F(0.0))], [(a, lg(0.5)), (c, lg(0.5))],
              [(blank, lg(0.9)), (b, lg(0.1))], [(b, F(0.0))], [(b, F(NEG)), (blank, F(NEG)), (a, F(0.0))]]
    T = len(frames)
    blps = [F(-2.0)] * T
    for mode, alpha, beta in (("plain", 0.0, 0.0), ("char", 0.9, -0.4)):
        rows = Rows(rt, [frames], [blps], bstride=T)
        s = Search(rt, mode, 16, 1, T, blank=blank, lm=clm if mode == "char" else None, alpha=alpha, beta=beta)
        for t in range(T):
            s.run("stream", rows, [1], t, resume=t > 0)
            want, best = restate(mode, frames[:t + 1], blps[:t + 1], 16, blank, o, vocab, alpha, beta)
            same_beam(s.entries(0), want)
            got = s.best(0)
            assert got[:2] == (list(best[0]), best[1]) and (mode == "plain" or got[2] == best[2])
        e = lossless_check(s, frames, blank, a64 if mode == "char" else None, vocab, alpha, beta)
        assert e < TOL_LM, e


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["plain", "char"])
def test_batch_of_150_ragged_utterances(rt, char_lms, mode):
    """150 utterances in one launch (more CTAs than SMs) with lengths 0 .. 64, bstride 80 > T, tok_stride T + 7 and garbage
    rows past each length: one-shot best == the restatement; out_tok past out_n untouched; length 0 = the empty prefix."""
    vocab, d = char_lms
    o, clm, ids, _ = d[3]
    B, T = 150, 64
    lens = [b % 65 for b in range(B)]
    frames = [lossless_cands(b, lens[b], ids[:6] + [1, 7, 9], 0, K=(1, 2, 4, 6)) for b in range(B)]
    blps = [[F(-1.5)] * lens[b] for b in range(B)]
    rows = Rows(rt, frames, blps, bstride=80, seed=3)
    s = Search(rt, mode, 16, B, T, lm=clm if mode == "char" else None, alpha=1.1, beta=0.6, tok_stride=T + 7)
    s.run("one", rows, lens)
    otok = s.otok.cpu().numpy()
    for b in range(B):
        toks, sc, ap = s.best(b)
        if lens[b] == 0:
            assert toks == [] and sc == 0.0
        else:
            _, (wt, ws, wa) = restate(mode, frames[b], blps[b], 16, 0, o, vocab, 1.1, 0.6)
            assert (toks, sc) == (list(wt), ws), b
            if mode == "char":
                assert ap == wa, b
        assert (otok[b, len(toks):] == SENT).all()


@pytest.mark.gpu
def test_trie_at_capacity_over_200_frames(rt):
    """K = 40 with two disjoint token sets on alternate frames and no blank: every frame's beam is all new children, so the
    trie fills to 1 + 40 + 512 * 199 of its 5 (200 * 512 + 1) contract.  One frame per call == chunks of 7 and 64 ==
    one-shot, state and trie bit for bit; the first frames == the restatement."""
    T, beam = 200, BEAM_CAP
    rng = np.random.default_rng(11)
    sets = [list(range(1, 41)), list(range(41, 81))]
    frames = [[(c, F(math.log(p))) for c, p in zip(sets[t % 2], rng.dirichlet(np.ones(40)))] for t in range(T)]
    rows = Rows(rt, [frames], bstride=T)
    runs = {}
    for chunk in (1, 7, 64):
        s = Search(rt, "plain", beam, 1, T)
        for t0 in range(0, T, chunk):
            s.run("stream", rows, [min(chunk, T - t0)], t0, resume=t0 > 0)
            if chunk == 1 and t0 == 4:
                want, _ = restate("plain", frames[:5], None, beam, 0)
                same_beam(s.entries(0), want)
        runs[chunk] = s
    one = Search(rt, "plain", beam, 1, T)
    one.run("one", rows, [T])
    ref = runs[1]
    got = ref.entries(0)
    assert int(ref.sti[0, 3 * BEAM_CAP + 1]) == 1 + 40 + beam * (T - 1) and len(got) == beam
    assert all(len(e[0]) == T for e in got)
    nodes = ref.cap // 5                  # (the hash part of the trie depends on the order of concurrent inserts)
    for s in (runs[7], runs[64], one):
        assert torch.equal(s.tp[:nodes], ref.tp[:nodes]) and torch.equal(s.tt[:nodes], ref.tt[:nodes])
        assert s.best(0)[:2] == ref.best(0)[:2]
    for s in (runs[7], runs[64]):
        assert torch.equal(s.sti, ref.sti) and torch.equal(bits(s.stf), bits(ref.stf))


@pytest.mark.gpu
def test_prefix_that_leaves_the_beam_and_comes_back(rt):
    """Small beams over peaky frames: prefixes drop out of the beam and are re-created later.  Such a prefix keeps its node
    id (the persistent (parent, token) hash) and the beam equals the restatement at every frame, which merges the mass of
    a child of a returning prefix into that child's existing entry."""
    returns = 0
    for seed in range(6):
        rng = np.random.default_rng(seed)
        T = 30
        frames = []
        for _ in range(T):
            ids = list(rng.choice([0, 1, 2, 3], 3, replace=False))
            frames.append([(int(c), F(math.log(p))) for c, p in zip(ids, rng.dirichlet(np.ones(3) * 0.5))])
        rows = Rows(rt, [frames], bstride=T)
        s = Search(rt, "plain", 3, 1, T)
        node_of, seen_at = {}, {}
        for t in range(T):
            s.run("stream", rows, [1], t, resume=t > 0)
            want, _ = restate("plain", frames[:t + 1], None, 3, 0)
            got = s.entries(0)
            same_beam(got, want)
            for toks, _, _, _, node in got:
                assert node_of.setdefault(toks, node) == node, (toks, node_of[toks], node)
                if toks in seen_at and seen_at[toks] < t - 1:
                    returns += 1
                seen_at[toks] = t
    assert returns > 0


@pytest.mark.gpu
@pytest.mark.parametrize("order,alpha,beta", [(1, 1.0, 2.0), (2, 0.8, -1.5), (6, 1.2, -1.5), (6, 0.9, 0.0), (6, 0.0, 2.0),
                                              (2, 1.5, 0.0)])
def test_char_lm_orders_at_beam_512(rt, char_lms, order, alpha, beta):
    """Character LM of orders 1, 2 and 6 (the only order whose 6-grams use the high half of the key and the third int of
    the saved window), beta < 0 (min_cutoff subtracts max(0, beta)), alpha = 0; beam 512 with K = 40, so the beam is full
    and min_cutoff is on.  Streaming in chunks 3 + 2 + 3 (the windows saved and restored) == restatement at every rank;
    one-shot and pool == streaming, approx included."""
    vocab, d = char_lms
    o, clm, ids, _ = d[order]
    T = 8
    frames, blps = topk_rows(rt, grid_logits(order, T, V, ids + [1, 4000], 0, -8.0), 40, 1.0, 0)
    rows = Rows(rt, [frames], [blps], bstride=T)
    s = Search(rt, "char", BEAM_CAP, 1, T, lm=clm, alpha=alpha, beta=beta)
    for t0, n in ((0, 3), (3, 2), (5, 3)):
        s.run("stream", rows, [n], t0, resume=t0 > 0)
    want, (bt, bs, ba) = restate("char", frames, blps, BEAM_CAP, 0, o, vocab, alpha, beta)
    same_beam(s.entries(0), want)
    assert s.best(0) == (list(bt), bs, ba)
    assert len(s.entries(0)) == BEAM_CAP
    for form in ("one", "pool"):
        x = Search(rt, "char", BEAM_CAP, 1, T, lm=clm, alpha=alpha, beta=beta)
        x.run(form, rows, [T])
        assert x.best(0) == s.best(0)


@pytest.mark.gpu
def test_char_lm_order_6_windows(rt, char_lms):
    """Frames that spell a 6-gram of the order-6 LM, one frame per call: the 6-gram query packs its sixth id into the high
    half of the key, and the saved five-id window fills the third int of the state — each restored every frame.  Lossless,
    so the fused scores equal forward64 + alpha lnP64 + beta |l| as well as the restatement."""
    vocab, d = char_lms
    o, clm, ids, a64 = d[6]
    def distinct(k):                       # a 6-gram whose lnP differs from the backoff a lost 6-gram would give
        return abs(a64.ng[k][0] - (a64.ng.get(k[:5], (0.0, 0.0))[1] + a64.lnp(list(k[:5]), k[5], top=4))) > 0.1
    gram = next(k for k in sorted(a64.ng) if len(k) == 6 and "<s>" not in k and "</s>" not in k
                and all(k[j] != k[j + 1] for j in range(5)) and distinct(k))
    spell = [vocab.index(w) for w in gram]
    frames = []
    for t in range(7):
        x = spell[t] if t < 6 else ids[0]
        other = next(c for c in ids[t * 5 % len(ids):] + ids if c != x)
        frames.append([(x, F(math.log(0.6))), (0, F(math.log(0.15)))] + ([(other, F(math.log(0.25)))] if t % 2 else []))
    blps = [F(math.log(0.15))] * 7
    rows = Rows(rt, [frames], [blps], bstride=7)
    s = Search(rt, "char", BEAM_CAP, 1, 7, lm=clm, alpha=1.0, beta=0.5)
    for t in range(7):
        s.run("stream", rows, [1], t, resume=t > 0)
        want, (bt, bs, ba) = restate("char", frames[:t + 1], blps[:t + 1], BEAM_CAP, 0, o, vocab, 1.0, 0.5)
        same_beam(s.entries(0), want)
        assert s.best(0) == (list(bt), bs, ba)
    got = s.entries(0)
    assert any(e[0][:6] == tuple(spell) for e in got) and len(got) < BEAM_CAP
    assert lossless_check(s, frames, 0, a64, vocab, 1.0, 0.5) < TOL_LM


@pytest.fixture(scope="module")
def word_lms(tmp_path_factory):
    from masr_b200 import synth
    from masr_b200.lm import WordLM
    vocab = synth.english_vocabulary()
    out = {}
    for order in (1, 2, 5):
        p = str(tmp_path_factory.mktemp("wlm") / f"w{order}.arpa")
        synth.word_lm_arpa(p, seed=order, order=order, n_words=60)
        out[order] = (owl.WordLM(p, vocab), WordLM(p, vocab))
    return vocab, out


@pytest.mark.gpu
@pytest.mark.parametrize("order", [1, 2, 5])
def test_word_lm_batch_at_beam_512(rt, word_lms, order):
    """Word LM of orders 1, 2 and 5 at beam 512, beta < 0, 140 utterances in one launch (two CTA waves): every saved beam
    == the restatement at every rank; best and approx of streaming, one-shot and pool agree."""
    vocab, d = word_lms
    o, w = d[order]
    B, T, Vw = 140, 7, len(vocab)
    alpha, beta = 0.8, -1.0
    rng = np.random.default_rng(order)
    logits = rng.standard_normal((B * T, Vw)).astype(np.float32) * 2.0
    logits[:, w.space] += 1.5
    fr_all, blp_all = topk_rows(rt, logits, 40, 0.99, 0)
    lens = [T - (b % 3) for b in range(B)]
    frames = [fr_all[b * T: b * T + lens[b]] for b in range(B)]
    blps = [blp_all[b * T: b * T + lens[b]] for b in range(B)]
    rows = Rows(rt, frames, blps, bstride=T, Vv=Vw)
    s = Search(rt, "word", BEAM_CAP, B, T, lm=w, alpha=alpha, beta=beta)
    s.run("stream", rows, lens)
    full = 0
    for b in list(range(0, B, 10)) + [133, 137, 139]:              # (the other utterances: through the forms below)
        want, (bt, bs, ba) = restate("word", frames[b], blps[b], BEAM_CAP, 0, o, vocab, alpha, beta)
        got = s.entries(b)
        same_beam(got, want)
        full += len(got) == BEAM_CAP
        assert s.best(b) == (list(bt), bs, ba), b
    assert full > 0
    for form in ("one", "pool"):
        x = Search(rt, "word", BEAM_CAP, B, T, lm=w, alpha=alpha, beta=beta)
        x.run(form, rows, lens)
        assert torch.equal(x.on, s.on) and torch.equal(x.osc, s.osc) and torch.equal(x.oap, s.oap)
        assert torch.equal(x.otok, s.otok)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["plain", "char", "word"])
def test_pool_slots_at_beam_512(rt, char_lms, word_lms, mode):
    """40 pool slots at beam 512 and K = 40 (word: K = V = 30) over two launches with ragged lengths that include 0: a slot
    with frames == the streaming form over the same frames (whole beam, best, approx); a slot with no frames stays byte for
    byte as it was (state, trie, outputs); a slot marked fresh again restarts at the root."""
    if mode == "word":
        vocab, d = word_lms
        o, lmo = d[2]
        Vv, ids = len(vocab), list(range(2, 30))
    else:
        vocab, d = char_lms
        o, lmo, ids, _ = d[3]
        Vv, ids = V, ids + [1, 9]
    kw = dict(lm=lmo if mode != "plain" else None, alpha=0.6, beta=-0.5)
    B, T = 40, 6
    fr_all, blp_all = topk_rows(rt, grid_logits(17, B * T, Vv, ids, 0, -8.0), 40, 1.0, 0)
    fr = [fr_all[b * T:(b + 1) * T] for b in range(B)]
    bl = [blp_all[b * T:(b + 1) * T] for b in range(B)]
    lens1 = [(0, 1, 2, 3)[b % 4] for b in range(B)]
    lens2 = [(2, 0, 3, 1, 0)[b % 5] for b in range(B)]
    rows1 = Rows(rt, [fr[b][:lens1[b]] for b in range(B)], [bl[b][:lens1[b]] for b in range(B)], bstride=T, Vv=Vv, seed=1)
    rows2 = Rows(rt, [fr[b][lens1[b]:lens1[b] + lens2[b]] for b in range(B)], [bl[b][lens1[b]:lens1[b] + lens2[b]] for b in range(B)],
                 bstride=T, Vv=Vv, seed=2)
    pool = Search(rt, mode, BEAM_CAP, B, T, **kw)
    pool.run("pool", rows1, lens1)
    assert pool.fresh.cpu().tolist() == [int(n == 0) for n in lens1]

    def snap(b):
        c = pool.cap
        return [bits(x).clone() for x in (pool.sti[b], pool.stf[b], pool.tp[b * c:(b + 1) * c], pool.tt[b * c:(b + 1) * c],
                                          pool.otok[b], pool.on[b], pool.osc[b], pool.oap[b])]
    before = [snap(b) for b in range(B)]
    pool.fresh[7] = 1                                   # slot 7 ends its utterance: marked fresh, its hash range reset
    pool.tp[7 * pool.cap + pool.cap // 5: 8 * pool.cap] = -1
    pool.run("pool", rows2, lens2)
    for b in range(B):
        if lens2[b] == 0:
            assert all(torch.equal(x, y) for x, y in zip(snap(b), before[b])), b
            continue
        restart = b == 7 or lens1[b] == 0
        sb = Search(rt, mode, BEAM_CAP, 1, T, **kw)
        if not restart:
            sb.run("stream", Rows(rt, [fr[b][:lens1[b]]], [bl[b][:lens1[b]]], bstride=T, Vv=Vv), [lens1[b]])
        sb.run("stream", Rows(rt, [fr[b][lens1[b]:lens1[b] + lens2[b]]], [bl[b][lens1[b]:lens1[b] + lens2[b]]], bstride=T, Vv=Vv),
               [lens2[b]], resume=not restart)
        assert [e[:4] for e in pool.entries(b)] == [e[:4] for e in sb.entries(0)], b
        got, want = pool.best(b), sb.best(0)
        assert got[:2] == want[:2] and (mode == "plain" or got[2] == want[2]), b
