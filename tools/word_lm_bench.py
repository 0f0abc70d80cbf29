"""Dev tool: the fused prefix beam search with a word LM (masr_ctc_prefix_beam_wordlm: lexicon constraint, LM term per
word) against the character-LM (masr_ctc_prefix_beam_lm) and no-LM (masr_ctc_prefix_beam) searches on the SAME top-k
candidates: B = 32 utterances x 248 frames (10 s of 40 ms frames) over the 30-token English vocabulary, beam 300 and 500,
alpha 1.0 / beta 1.5.  Synthetic posteriors with the lexicon's letters and <space> lifted; synthetic 5-gram LMs (a word
LM of ~5000 words, a character LM over the same corpus' letters) generated into a temporary directory.  Kernel time from
CUDA events around each launch, the three searches alternated round by round; one JSON line per (search, beam) with the
median and range, plus the card's name and power limit.  Usage: python tools/word_lm_bench.py [--rounds N]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from masr_b200 import _lib, synth
from masr_b200.lm import CharLM, WordLM

B, T, ALPHA, BETA = 32, 248, 1.0, 1.5


def card():
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                             str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    return torch.cuda.get_device_name(), pl


def lms(tmp, vocab):
    wp, cp = os.path.join(tmp, "word5.arpa"), os.path.join(tmp, "char5.arpa")
    words = synth.word_lm_arpa(wp, seed=1, order=5, n_words=5000, n_sentences=20000)
    rng = np.random.default_rng(2)
    letters = [w for w in words if all(ch in synth.ENGLISH_LETTERS for ch in w)]
    sents = [["<s>"] + [ch for w in rng.choice(letters, int(rng.integers(2, 12))) for ch in w] + ["</s>"] for _ in range(20000)]
    synth._write_backoff_arpa(cp, sents, list(synth.ENGLISH_LETTERS) + ["</s>", "<unk>"], 5, 0.5)
    return WordLM(wp, vocab), CharLM(cp, vocab)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
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
    wt, ct = wlm.tables(dev), clm.tables(dev)
    common = (pool.data_ptr(), tp.data_ptr(), tt.data_ptr(), trie_n.value, otok.data_ptr(), T, on.data_ptr(), osc.data_ptr())

    def launch(kind, beam):
        if kind == "no_lm":
            _lib.call("masr_ctc_prefix_beam", cid.data_ptr(), clp.data_ptr(), cn.data_ptr(), T, lens.data_ptr(), B, beam, 0, *common, st)
        elif kind == "char_lm":
            _lib.call("masr_ctc_prefix_beam_lm", cid.data_ptr(), clp.data_ptr(), cn.data_ptr(), blp.data_ptr(), T, lens.data_ptr(), B,
                      beam, 0, C.byref(ct), ALPHA, BETA, *common, oap.data_ptr(), st)
        else:
            _lib.call("masr_ctc_prefix_beam_wordlm", cid.data_ptr(), clp.data_ptr(), cn.data_ptr(), blp.data_ptr(), T, lens.data_ptr(),
                      B, beam, 0, C.byref(wt), ALPHA, BETA, *common, oap.data_ptr(), st)

    name, power = card()
    kinds = ("no_lm", "char_lm", "word_lm")
    cands = float(cn.float().mean().item())
    for beam in (300, 500):
        times = {k: [] for k in kinds}
        words = None
        for k in kinds:
            launch(k, beam)                                   # warm-up
        for _ in range(args.rounds):
            for k in kinds:
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                launch(k, beam)
                e1.record()
                e1.synchronize()
                times[k].append(e0.elapsed_time(e1))
                if k == "word_lm":
                    n = on.cpu().numpy()
                    tok = otok.cpu().numpy()
                    words = float(np.mean([(tok[b, :n[b]] == wlm.space).sum() for b in range(B)]))
        for k in kinds:
            t = sorted(times[k])
            print(json.dumps({"search": k, "beam": beam, "B": B, "frames": T, "mean_candidates_per_frame": round(cands, 2),
                              "kernel_ms_median": round(t[len(t) // 2], 3), "kernel_ms_min": round(t[0], 3),
                              "kernel_ms_max": round(t[-1], 3), "rounds": args.rounds,
                              "word_lm": {"order": wlm.order, "dict_size": wlm.dict_size} if k == "word_lm" else None,
                              "char_lm_order": clm.order if k == "char_lm" else None,
                              "spaces_per_best_hypothesis": words if k == "word_lm" else None,
                              "card": name, "power_limit": power}), flush=True)


if __name__ == "__main__":
    main()
