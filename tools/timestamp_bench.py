"""Dev tool: what token onsets cost the prefix beam search.  The one-shot searches without an LM
(masr_ctc_prefix_beam), with a character LM (masr_ctc_prefix_beam_lm) and with a word LM (masr_ctc_prefix_beam_wordlm)
record every node's onset frame as they allocate it; masr_ctc_prefix_beam_frames then reads the reported prefixes' onsets
out.  Same inputs as tools/word_lm_bench.py: B = 32 utterances x 248 frames (10 s of 40 ms frames) of synthetic top-k
candidates over the 30-token English vocabulary, beam 300 and 500, synthetic 5-gram word and character LMs.  Kernel time
from CUDA events around each launch; one read-out launch per batch after each search.

``--ab LIB``: also load another build of the library (e.g. one made from an earlier commit, without the onset store) and
run its searches on the same inputs, alternating the two libraries round by round; its tokens and scores must equal this
build's bit for bit.  One JSON line per (library, search, beam) with the median and range, plus the card's name and power
limit.  Usage: python tools/timestamp_bench.py [--rounds N] [--ab path/to/libmasr_b200.so]"""
import argparse
import ctypes as C
import json
import os
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from masr_b200 import _lib, synth
from word_lm_bench import B, T, ALPHA, BETA, card, lms

ENTRY = {"no_lm": "masr_ctc_prefix_beam", "char_lm": "masr_ctc_prefix_beam_lm", "word_lm": "masr_ctc_prefix_beam_wordlm"}


def other_library(path):
    """``path`` with the prototypes of the search entry points declared."""
    lib = C.CDLL(os.path.abspath(path))
    for name in list(ENTRY.values()) + ["masr_ctc_prefix_beam_workspace"]:
        fn = getattr(lib, name)
        fn.argtypes, fn.restype = _lib.SIGNATURES[name], C.c_int
    lib.masr_last_error.restype = C.c_char_p
    return lib


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=9)
    ap.add_argument("--ab", metavar="LIB", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda", torch.cuda.current_device())
    st = torch.cuda.current_stream().cuda_stream
    vocab = synth.english_vocabulary()
    V = len(vocab)
    with tempfile.TemporaryDirectory() as tmp:
        wlm, clm = lms(tmp, vocab)
    rng = np.random.default_rng(0)
    logits = rng.standard_normal((B * T, V)).astype(np.float32) * 3.0
    for t in range(1, B * T):
        logits[t] = 0.5 * logits[t] + 0.5 * logits[t - 1]
    logits[:, 0] += 2.0
    logits[:, 2:2 + 27] += 1.0
    logits[:, wlm.space] += 2.0
    L = torch.zeros(B * T, 32, device=dev)
    L[:, :V] = torch.from_numpy(logits).to(dev)
    M = B * T
    cid = torch.empty(M, 40, dtype=torch.int32, device=dev); clp = torch.empty(M, 40, device=dev)
    cn = torch.empty(M, dtype=torch.int32, device=dev); blp = torch.empty(M, device=dev)
    _lib.call("masr_ctc_topk_blank_f32", L.data_ptr(), 32, M, V, 40, 0.99, 0, cid.data_ptr(), clp.data_ptr(), cn.data_ptr(),
              blp.data_ptr(), st)
    pool_n, trie_n = C.c_int64(0), C.c_int64(0)
    _lib.call("masr_ctc_prefix_beam_workspace", B, T, C.byref(pool_n), C.byref(trie_n))
    pool = torch.empty(pool_n.value, device=dev)
    tp = torch.empty(B * trie_n.value, dtype=torch.int32, device=dev); tt = torch.empty_like(tp)
    lens = torch.full((B,), T, dtype=torch.int32, device=dev)
    otok = torch.zeros(B, T, dtype=torch.int32, device=dev); on = torch.zeros(B, dtype=torch.int32, device=dev)
    osc, oap = torch.zeros(B, device=dev), torch.zeros(B, device=dev)
    ofr = torch.zeros(B, T, dtype=torch.int32, device=dev)
    wt, ct = wlm.tables(dev), clm.tables(dev)
    common = (pool.data_ptr(), tp.data_ptr(), tt.data_ptr(), trie_n.value, otok.data_ptr(), T, on.data_ptr(), osc.data_ptr())
    libs = {"this": None}
    if args.ab:
        libs["ab"] = other_library(args.ab)

    def call(lib, name, *a):
        if lib is None:
            _lib.call(name, *a)
        elif getattr(lib, name)(*a) != 0:
            raise RuntimeError(f"{name}: {lib.masr_last_error().decode()}")

    def launch(lib, kind, beam):
        head = (cid.data_ptr(), clp.data_ptr(), cn.data_ptr())
        if kind == "no_lm":
            call(lib, ENTRY[kind], *head, T, lens.data_ptr(), B, beam, 0, *common, st)
        else:
            tables = C.byref(ct) if kind == "char_lm" else C.byref(wt)
            call(lib, ENTRY[kind], *head, blp.data_ptr(), T, lens.data_ptr(), B, beam, 0, tables, ALPHA, BETA, *common,
                 oap.data_ptr(), st)

    def readout():
        _lib.call("masr_ctc_prefix_beam_frames", tp.data_ptr(), tt.data_ptr(), trie_n.value, otok.data_ptr(), T, on.data_ptr(),
                  B, ofr.data_ptr(), T, st)

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        return e0.elapsed_time(e1)

    def result():
        n = on.cpu().numpy()
        return [otok[b, :n[b]].cpu().tolist() for b in range(B)], osc.cpu().view(torch.int32).tolist(), \
            oap.cpu().view(torch.int32).tolist()

    name, power = card()
    kinds = tuple(ENTRY)
    for beam in (300, 500):
        times = {(l, k): [] for l in libs for k in kinds}
        rtimes = {k: [] for k in kinds}
        for l in libs:
            for k in kinds:
                launch(libs[l], k, beam)                       # warm-up
        readout()
        same = True
        for _ in range(args.rounds):
            for k in kinds:
                outs = {}
                for l in libs:
                    times[(l, k)].append(timed(lambda: launch(libs[l], k, beam)))
                    outs[l] = result()
                    if l == "this":
                        rtimes[k].append(timed(readout))
                same &= all(o == outs["this"] for o in outs.values())
        torch.cuda.synchronize()
        for (l, k), t in times.items():
            t = sorted(t)
            line = {"library": l, "search": k, "beam": beam, "B": B, "frames": T, "kernel_ms_median": round(t[len(t) // 2], 4),
                    "kernel_ms_min": round(t[0], 4), "kernel_ms_max": round(t[-1], 4), "rounds": args.rounds,
                    "card": name, "power_limit": power}
            if l == "this":
                r = sorted(rtimes[k])
                line.update(frames_readout_ms_median=round(r[len(r) // 2], 4), frames_readout_ms_max=round(r[-1], 4))
            if args.ab:
                line["outputs_equal_across_libraries"] = bool(same)
            print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
