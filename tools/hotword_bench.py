"""Dev tool: the cost of hotword biasing in the GPU prefix beam search.  For each LM kind (none, character LM, word LM) and
beam (300, 512), the one-shot search kernel of a batch of synthetic utterances without hotwords (the plain entry point)
and with 100 and 2000 hotwords (the ``*_hot`` entry points) on the SAME top-k candidates, event-timed, the searches
alternated round by round.  Prints one JSON line per (kind, beam, hotwords) with the card's name and power limit.

    python tools/hotword_bench.py [--batch 32] [--frames 300] [--rounds 5]
"""
from __future__ import annotations

import argparse
import json
import os
import random
import subprocess
import sys
import tempfile

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from masr_b200 import _lib, synth                                    # noqa: E402
from masr_b200.beam import ONE_SHOT, BeamSearch                       # noqa: E402
from masr_b200.hotwords import HotwordGraph                           # noqa: E402
from masr_b200.lm import CharLM, WordLM                               # noqa: E402


class Eng:
    def __init__(self, V):
        self.V = V

    def _k(self, tag, name, *args, n=1):
        _lib.call(name, *args, torch.cuda.current_stream().cuda_stream)


def WordLM_words(wlm, vocab):
    """Every word of a WordLM's lexicon, spelled from its trie."""
    out, stack = [], [(0, "")]
    while stack:
        n, s = stack.pop()
        if n and wlm.lex_word[n] >= 0:
            out.append(s)
        for a in range(int(wlm.lex_off[n]), int(wlm.lex_off[n + 1])):
            stack.append((int(wlm.lex_next[a]), s + vocab[int(wlm.lex_tok[a])]))
    return sorted(out)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True).stdout.strip()
    return q or torch.cuda.get_device_name()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--frames", type=int, default=300)
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    dev, B, T = torch.device("cuda"), a.batch, a.frames
    tmp = tempfile.mkdtemp()
    cv, ev = synth.vocabulary(), synth.english_vocabulary()
    pc, pw = os.path.join(tmp, "c.arpa"), os.path.join(tmp, "w.arpa")
    chars = synth.character_lm_arpa(pc, seed=3, order=3, n_chars=80, n_sentences=600)
    synth.word_lm_arpa(pw, seed=3, order=3, n_words=200, extra_unigrams=3000)
    kinds = {"none": (cv, None, [cv.index(c) for c in chars]), "char": (cv, CharLM(pc, cv), [cv.index(c) for c in chars]),
             "word": (ev, WordLM(pw, ev), list(range(2, len(ev))))}
    info = card()
    for kind, (vocab, lm, lift) in kinds.items():
        V = len(vocab)
        rng = np.random.default_rng(0)
        lg = rng.standard_normal((B * T, V)).astype(np.float32) * 3.0
        lg[:, 0] += 2.0
        lg[:, lift] += 2.0
        L = torch.zeros(B * T, (V + 15) // 16 * 16, device=dev)
        L[:, :V] = torch.from_numpy(lg).to(dev)
        r = random.Random(1)
        toks = [vocab[i] for i in lift if vocab[i] != "<space>"]
        graphs = {0: None}
        for n in (100, 2000):
            if kind == "word":                       # lexicon words (the lexicon rejects any other word)
                words = [w for w in WordLM_words(lm, vocab) if len(w) >= 2]
                hw = r.sample(words, min(n, len(words)))
            else:
                hw = {"".join(r.choice(toks) for _ in range(r.randint(2, 6))) for _ in range(n)}
            graphs[n] = HotwordGraph(hw, vocab, 1.5)
        lens = torch.full((B,), T, dtype=torch.int32, device=dev)
        eng = Eng(V)
        alpha, beta = (0.0, 0.0) if lm is None else (0.8, 1.0)
        for beam in (300, 512):
            searches = {n: BeamSearch(dev, ONE_SHOT, B, B * T, T, beam, 0.99, 40, lm, alpha, beta, g) for n, g in graphs.items()}
            for s in searches.values():
                s.topk(eng, L, L.stride(0), B * T)
                s.search(eng, lens.data_ptr(), B, T)                   # warm-up
            times = {n: [] for n in searches}
            for _ in range(a.rounds):
                for n, s in searches.items():
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    s.search(eng, lens.data_ptr(), B, T)
                    e1.record()
                    e1.synchronize()
                    times[n].append(e0.elapsed_time(e1))
            for n, t in times.items():
                print(json.dumps({"card": info, "lm": kind, "beam": beam, "hotwords": n,
                                  "nodes": 0 if graphs[n] is None else graphs[n].nodes, "batch": B, "frames": T,
                                  "search_ms_median": round(float(np.median(t)), 3), "search_ms_min": round(min(t), 3)}),
                      flush=True)


if __name__ == "__main__":
    main()
