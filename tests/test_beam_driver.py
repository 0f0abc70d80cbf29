"""CPU: the host side of the GPU prefix beam search (masr_b200.beam.BeamSearch and its StreamBeam / PoolBeam forms).  For
every form and LM kind each launch names an entry point of include/masr_b200.h with its exact arity and argument types,
and every buffer sits at the parameter the header names for it.  No kernel runs: the engine is a fake that records its
calls."""
import ctypes
import gc
import os
import re
import weakref

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "masr_b200.h")


def header_params():
    """function name -> its parameter names, in order, as include/masr_b200.h declares them."""
    src = re.sub(r"/\*.*?\*/", "", open(HEADER, encoding="utf-8").read(), flags=re.S)
    decl = re.findall(r"\b(?:int|const char\*)\s+(masr_[a-z0-9_]+)\s*\(([^;]*?)\)\s*;", src, flags=re.S)
    return {name: [re.search(r"(\w+)\s*$", p).group(1) for p in params.split(",") if p.strip() not in ("", "void")]
            for name, params in decl}


@pytest.fixture(scope="module")
def lib():
    from masr_b200 import build, _lib
    build.build()                      # nvcc cross-compiles sm_90a without a GPU; only host-side sizes are queried here
    return _lib.load()


class FakeEngine:
    """The engine surface the search uses; `_k` records (tag, entry point, arguments) instead of launching."""
    device = torch.device("cpu")
    V, Vpad = 29, 32

    def __init__(self):
        self.calls = []
        self.d2h_bytes = 0

    def _k(self, tag, name, *args, n=1):
        self.calls.append((tag, name, args))


def stub_lm(kind):
    """An LM with the surface the search uses (its entry-point base name and its device tables) and no file behind it."""
    from masr_b200 import _lib, lm
    if kind is None:
        return None
    real, tables = (lm.CharLM, _lib.LmTables) if kind == "char" else (lm.WordLM, _lib.WordLmTables)

    class Stub:
        BEAM = real.BEAM

        def __init__(self):
            self.t = tables()

        def tables(self, device):
            return self.t
    return Stub()


def check_call(decl, call, expect):
    """The recorded call matches its ctypes signature (plus the stream `_k` appends) and has `expect` {parameter: value}."""
    from masr_b200 import _lib
    tag, name, args = call
    argtypes = _lib.SIGNATURES[name]
    assert len(args) + 1 == len(argtypes) == len(decl[name]), name
    for a, t in zip(args + (0,), argtypes):
        t.from_param(a)
    got = dict(zip(decl[name], args))
    for p, v in expect.items():
        assert got[p] == v, (name, p, got[p], v)
    return got


@pytest.mark.parametrize("kind", [None, "char", "word"])
@pytest.mark.parametrize("form", ["one_shot", "stream", "pool"])
def test_search_launches_match_the_header(lib, form, kind):
    from masr_b200 import _lib, beam
    decl = header_params()
    S, R, F, K = 3, 12, 10, 7
    eng, lm = FakeEngine(), stub_lm(kind)
    bs = beam.BeamSearch(eng.device, getattr(beam, form.upper()), S, S * R, F, beam_size=K, cutoff_prob=0.9, cutoff_top_n=5,
                         lm=lm, alpha=0.5, beta=1.5)
    base = {None: "masr_ctc_prefix_beam", "char": "masr_ctc_prefix_beam_lm", "word": "masr_ctc_prefix_beam_wordlm"}[kind]
    # buffers: candidate rows 40 wide, the state the library sizes, the trie each form is sized by
    assert bs.cand_id.shape == bs.cand_lp.shape == (S * R, beam.BK_MAX) and bs.cand_n.shape == (S * R,)
    assert (bs.blank_lp is None) == (lm is None) and (lm is None or bs.blank_lp.shape == (S * R,))
    assert bs.out_tok.shape == (S, F) and bs.out.shape == (3, S)
    pool_n, trie_n, si, sf = (ctypes.c_int64() for _ in range(4))
    _lib.call("masr_ctc_prefix_beam_workspace", S, F, ctypes.byref(pool_n), ctypes.byref(trie_n))
    assert bs.scratch.numel() == pool_n.value
    assert bs.trie_cap == (5 * (F * K + 1) if form == "pool" else trie_n.value)
    assert bs.trie_par.numel() == bs.trie_tok.numel() == S * bs.trie_cap
    if form == "one_shot":
        assert bs.state_i is None and bs.state_f is None
    else:
        _lib.call(base + "_state_size", ctypes.byref(si), ctypes.byref(sf))
        assert bs.state_i.shape == (S, si.value) and bs.state_f.shape == (S, sf.value)
    if form == "pool":
        assert (bs.trie_par == -1).all() and (bs.fresh == 1).all()
    else:
        assert bs.fresh is None

    logits = torch.zeros(S * R, eng.Vpad)
    lens = torch.zeros(S, dtype=torch.int32)
    bs.topk(eng, logits, eng.Vpad, S * R)
    bs.search(eng, lens.data_ptr(), S, R, resume=1)
    topk, search = eng.calls
    assert (topk[0], topk[1], search[0], search[1]) == (
        "ctc_topk", "masr_ctc_topk_f32" if lm is None else "masr_ctc_topk_blank_f32", "prefix_beam",
        base + {"one_shot": "", "stream": "_stream", "pool": "_pool"}[form])
    cands = {"cand_id": bs.cand_id.data_ptr(), "cand_logp": bs.cand_lp.data_ptr(), "cand_cnt": bs.cand_n.data_ptr()}
    blank = {} if lm is None else {"blank_logp": bs.blank_lp.data_ptr()}
    check_call(decl, topk, {"logits": logits.data_ptr(), "ldl": eng.Vpad, "M": S * R, "V": eng.V, "top_n": 5, "cutoff_prob": 0.9,
                            **cands, **blank, **({} if lm is None else {"blank": 0})})
    expect = {**cands, **blank, "bstride": R, "lens": lens.data_ptr(), "B": S, "beam_size": K, "blank": 0,
              "pool": bs.scratch.data_ptr(), "trie_parent": bs.trie_par.data_ptr(), "trie_tok": bs.trie_tok.data_ptr(),
              "trie_cap": bs.trie_cap, "out_tok": bs.out_tok.data_ptr(), "tok_stride": F, "out_n": bs.out[1].data_ptr()}
    if form != "one_shot":
        expect.update(state_i=bs.state_i.data_ptr(), state_f=bs.state_f.data_ptr())
    if form == "stream":
        expect["resume"] = 1
    if form == "pool":
        expect["fresh"] = bs.fresh.data_ptr()
    # the reported score (approx_ctc with an LM) is out[0] in every mode, the fused score out[2] with an LM
    if lm is None:
        expect.update(out_score=bs.out[0].data_ptr())
        assert bs.score.data_ptr() == bs.fused.data_ptr() == bs.out[0].data_ptr()
    else:
        expect.update(out_score=bs.out[2].data_ptr(), out_approx=bs.out[0].data_ptr(), alpha=0.5, beta=1.5)
        assert bs.score.data_ptr() == bs.out[0].data_ptr() and bs.fused.data_ptr() == bs.out[2].data_ptr()
    got = check_call(decl, search, expect)
    assert set(decl[search[1]]) - set(expect) - {"stream"} <= {"lm_host"}
    if lm is not None:
        assert ctypes.addressof(got["lm_host"]._obj) == ctypes.addressof(lm.t)


@pytest.mark.parametrize("kind", [None, "char"])
def test_stream_and_pool_forms_drive_the_search(lib, kind):
    """StreamBeam resumes from the second push on and skips the top-k of an empty chunk; PoolBeam searches every slot over
    the pool's device length row and rejects a beam its trie is not sized for."""
    from masr_b200.engine import StreamBeam
    from masr_b200.stream_pool import CHUNK_OUT, PoolBeam
    eng = FakeEngine()
    sb = StreamBeam(eng, beam_size=8, max_frames=40, max_chunk=16, lm=stub_lm(kind))
    logits = torch.zeros(16, eng.Vpad)
    assert sb.push(logits, 16) == ([], 0.0) and sb.push(logits, 0) == ([], 0.0)
    assert [c[0] for c in eng.calls] == ["ctc_topk", "prefix_beam", "prefix_beam"]
    resume = header_params()[eng.calls[1][1]].index("resume")
    assert [eng.calls[1][2][resume], eng.calls[2][2][resume]] == [0, 1]
    assert eng.d2h_bytes == 16

    class Pool:
        QLEN, QLEN2, S, OUT_ROWS, cap = 0, 3, 4, CHUNK_OUT, 64

        def __init__(self):
            self.eng, self.b, self.meta = eng, {"logits": torch.zeros(4 * CHUNK_OUT, eng.Vpad)}, torch.zeros(6, 4, dtype=torch.int32)

        def _m(self, row):
            return self.meta[row].data_ptr()
    pool = Pool()
    with pytest.raises(ValueError, match="out of range"):
        PoolBeam(pool, beam_size=513)
    pb = PoolBeam(pool, beam_size=8, lm=stub_lm(kind))
    eng.calls.clear()
    pb.launch()
    (_, _, targs), (_, name, sargs) = eng.calls
    p = dict(zip(header_params()[name], sargs))
    assert (targs[0], targs[2]) == (pool.b["logits"].data_ptr(), 4 * CHUNK_OUT)
    assert (p["lens"], p["B"], p["bstride"], p["tok_stride"]) == (pool.meta[Pool.QLEN].data_ptr(), 4, CHUNK_OUT, 65)
    pb.fresh.zero_()
    pb.trie_par.zero_()
    pb.reset(2)
    cap = pb.trie_cap
    assert pb.fresh.tolist() == [0, 0, 1, 0]
    assert (pb.trie_par[2 * cap + cap // 5:3 * cap] == -1).all() and (pb.trie_par[:2 * cap + cap // 5] == 0).all()


@pytest.mark.parametrize("kind", [None, "char", "word"])
def test_kept_search_frees_its_engine_and_lm(lib, kind):
    """A one-shot search the engine keeps for reuse (in a workspace) holds neither the engine nor the caller's LM: both are
    freed by reference counting as soon as they are dropped, with the cyclic collector off, and the kept search no longer
    fits a call once its LM is gone."""
    from masr_b200 import beam
    eng, lm = FakeEngine(), stub_lm(kind)
    settings = (8, 0.9, 5, lm, 0.5, 1.5)
    eng.ws = {"beam": beam.BeamSearch(eng.device, beam.ONE_SHOT, 2, 2 * 6, 6, *settings)}
    bs = eng.ws["beam"]
    assert bs.fits(2, 6, *settings) and bs.lm is lm
    assert not bs.fits(3, 6, *settings) and not bs.fits(2, 7, *settings) and not bs.fits(2, 6, 8, 0.95, 5, lm, 0.5, 1.5)
    bs.topk(eng, torch.zeros(12, eng.Vpad), eng.Vpad, 12)
    bs.search(eng, torch.zeros(2, dtype=torch.int32).data_ptr(), 2, 6)
    gc_on = gc.isenabled()
    gc.disable()
    try:
        e_ref = weakref.ref(eng)
        del eng
        assert e_ref() is None
        if kind is not None:
            l_ref = weakref.ref(lm)
            settings = lm = None
            assert l_ref() is None and bs.lm is None
            assert not bs.fits(2, 6, 8, 0.9, 5, None, 0.5, 1.5)     # built for an LM: never reused without one
    finally:
        if gc_on:
            gc.enable()
