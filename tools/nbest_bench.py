"""Dev tool: the cost of the N-best read-out of the GPU prefix beam search.

1. The read-out kernel alone (``BeamSearch.nbest``) after a streaming-form search of a batch of synthetic utterances, for
   each LM kind (none, character LM, word LM), beam (300, 500) and n (2, 10, 300), event-timed over ``--reps`` launches.
2. ``StreamPool.push`` of a synthetic streaming Conformer with the beam search at 64 slots (one 0.5 s message per slot
   and push), with ``n_best`` unset and ``n_best`` = 10, the two pools alternated push by push; host clock around each
   push, which ends in device-to-host copies.
Prints one JSON line per measurement with the card's name and power limit.

    python tools/nbest_bench.py [--batch 32] [--frames 300] [--reps 50] [--slots 64] [--pushes 12]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from masr_b200 import _lib, synth                                    # noqa: E402
from masr_b200.beam import STREAM, BeamSearch                         # noqa: E402
from masr_b200.lm import CharLM, WordLM                               # noqa: E402


class Eng:
    def __init__(self, V):
        self.V = V

    def _k(self, tag, name, *args, n=1):
        _lib.call(name, *args, torch.cuda.current_stream().cuda_stream)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True).stdout.strip()
    return q or torch.cuda.get_device_name()


def readout(a, info, tmp):
    dev, B, T = torch.device("cuda"), a.batch, a.frames
    cv, ev = synth.vocabulary(), synth.english_vocabulary()
    pc, pw = os.path.join(tmp, "c.arpa"), os.path.join(tmp, "w.arpa")
    chars = synth.character_lm_arpa(pc, seed=3, order=5, n_chars=80, n_sentences=600)
    synth.word_lm_arpa(pw, seed=3, order=3, n_words=200, extra_unigrams=3000)
    kinds = {"none": (cv, None, [cv.index(c) for c in chars]), "char": (cv, CharLM(pc, cv), [cv.index(c) for c in chars]),
             "word": (ev, WordLM(pw, ev), list(range(2, len(ev))))}
    for kind, (vocab, lm, lift) in kinds.items():
        V = len(vocab)
        rng = np.random.default_rng(0)
        lg = rng.standard_normal((B * T, V)).astype(np.float32) * 3.0
        lg[:, 0] += 2.0
        lg[:, lift] += 2.0
        L = torch.zeros(B * T, (V + 15) // 16 * 16, device=dev)
        L[:, :V] = torch.from_numpy(lg).to(dev)
        lens = torch.full((B,), T, dtype=torch.int32, device=dev)
        eng = Eng(V)
        alpha, beta = (0.0, 0.0) if lm is None else (0.8, 1.0)
        for beam in (300, 500):
            s = BeamSearch(dev, STREAM, B, B * T, T, beam, 0.99, 40, lm, alpha, beta)
            s.topk(eng, L, L.stride(0), B * T)
            s.search(eng, lens.data_ptr(), B, T)
            live = float(s.nbest(eng, B, beam)[4].float().mean())
            for n in (2, 10, 300):
                s.nbest(eng, B, n)                                        # warm-up
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(a.reps):
                    s.nbest(eng, B, n)
                e1.record()
                e1.synchronize()
                print(json.dumps({"card": info, "what": "nbest_readout", "lm": kind, "beam": beam, "n": n, "batch": B,
                                  "frames": T, "live_entries_mean": round(live, 1),
                                  "readout_ms": round(e0.elapsed_time(e1) / a.reps, 4)}), flush=True)


def pool_push(a, info, tmp):
    from masr_b200.predict import MASRPredictor
    mp, vp = os.path.join(tmp, "m.pt"), os.path.join(tmp, "vocabulary.txt")
    torch.save(synth.to_torch(synth.conformer_state_dict(0)), mp)
    synth.write_vocabulary(vp)
    cfg = {"use_model": "conformer", "streaming": True, "decoder": "ctc_beam_search",
           "preprocess_conf": {"feature_method": "fbank", "n_mels": 80, "sample_rate": 16000, "use_dB_normalization": True,
                               "target_dB": -20},
           "dataset_conf": {"dataset_vocab": vp},
           "ctc_beam_search_decoder_conf": {"beam_size": 300, "cutoff_prob": 0.99, "cutoff_top_n": 40,
                                            "language_model_path": ""}}
    pred = MASRPredictor(configs=cfg, model_path=mp, use_gpu=True)
    S, P = a.slots, a.pushes
    pools = {None: pred.create_stream_pool(S, max_frames=1000), 10: pred.create_stream_pool(S, max_frames=1000, n_best=10)}
    audio = [(np.clip(synth.speechlike_audio(100 + s, 8000 * (P + 1)), -1, 1) * 32767).astype("<i2") for s in range(S)]
    times = {k: [] for k in pools}
    for k in range(P + 1):                                    # push 0 warms up (and captures the step graphs)
        msg = {s: audio[s][k * 8000:(k + 1) * 8000].tobytes() for s in range(S)}
        for nb, pool in pools.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            pool.push(msg)
            t1 = time.perf_counter()
            if k:
                times[nb].append((t1 - t0) * 1e3)
    for nb, t in times.items():
        print(json.dumps({"card": info, "what": "stream_pool_push", "slots": S, "beam": 300, "n_best": nb,
                          "pushes": len(t), "push_ms_median": round(float(np.median(t)), 3),
                          "push_ms_min": round(min(t), 3)}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--frames", type=int, default=300)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--slots", type=int, default=64)
    ap.add_argument("--pushes", type=int, default=12)
    a = ap.parse_args()
    info = card()
    tmp = tempfile.mkdtemp()
    readout(a, info, tmp)
    pool_push(a, info, tmp)


if __name__ == "__main__":
    main()
