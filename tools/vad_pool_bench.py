"""What the streaming VAD adds to a stream-pool push, and what it saves (H100).  For S slots and 0.5 s pushes (synthetic
Conformer, greedy): ``vad_ms`` = one ``VadSlots.advance`` of every slot (host gather, encoder + slot recurrence, the
probabilities back), ``pool_ms`` = one ``StreamPool.push`` of every slot, and on silence-heavy audio (1-4 s of speech
between 3-12 s of near-silence) the share of (slot, push) pairs of a ``SegmentingStreamPool`` that feed nothing to the
recogniser, with its push time.  Host clock around each push ended by a device synchronise; medians after a warm-up.

    python tools/vad_pool_bench.py --slots 64 256
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

from conftest import synth_weights  # noqa: E402
from masr_b200 import synth  # noqa: E402
from masr_b200.predict import MASRPredictor  # noqa: E402
from oracle import silero_vad as sv  # noqa: E402

PUSH = 8000


def median_ms(fn, steps, warmup):
    out = []
    for k in range(steps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn(k)
        torch.cuda.synchronize()
        out.append((time.perf_counter() - t0) * 1e3)
    return round(float(np.median(out[warmup:])), 3)


def silence_heavy(seed, n):
    rng, parts = np.random.default_rng(seed), []
    while sum(len(p) for p in parts) < n:
        parts.append((rng.standard_normal(int(rng.integers(3, 13)) * 16000) * 1e-4).astype(np.float32))
        parts.append(synth.speechlike_audio(int(rng.integers(1 << 30)), int(rng.integers(1, 5)) * 16000))
    return np.concatenate(parts)[:n]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--slots", type=int, nargs="+", default=[64, 256])
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--seconds", type=int, default=60, help="silence-heavy audio per slot")
    args = ap.parse_args()
    tmp = tempfile.mkdtemp()
    mp, vp = os.path.join(tmp, "m.pt"), os.path.join(tmp, "vocabulary.txt")
    torch.save(synth.to_torch(synth_weights(0)), mp)
    synth.write_vocabulary(vp)
    pred = MASRPredictor(configs={"use_model": "conformer", "streaming": True, "decoder": "ctc_greedy",
                                  "preprocess_conf": {"sample_rate": 16000}, "dataset_conf": {"dataset_vocab": vp}},
                         model_path=mp, use_gpu=True)
    print("card:", subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                  capture_output=True, text=True).stdout.strip())
    steps = args.warmup + args.reps
    for S in args.slots:
        audio = [synth.speechlike_audio(1000 + i, PUSH * steps) for i in range(S)]
        piece = lambda src, k: {s: src[s][k * PUSH:(k + 1) * PUSH] for s in range(S)}
        seg, pool = pred.create_stream_pool(S, vad_model_path=sv.MODEL_PATH), pred.create_stream_pool(S)
        slots = seg.vad.slots(S)                                   # (state of its own: the pool's slots stay fresh)
        row = {"slots": S, "vad_ms": median_ms(lambda k: slots.advance(piece(audio, k)), steps, args.warmup),
               "pool_ms": median_ms(lambda k: pool.push(piece(audio, k)), steps, args.warmup)}
        quiet = [silence_heavy(2000 + i, args.seconds * 16000) for i in range(S)]
        fed, asr_push, now = set(), seg.pool.push, [0]            # (push, slot) pairs that reached the recogniser
        seg.pool.push = lambda a, *x, **kw: (fed.update((now[0], s) for s in a), asr_push(a, *x, **kw))[1]

        def seg_push(k):
            now[0] = k
            seg.push(piece(quiet, k))
        n_push = args.seconds * 16000 // PUSH
        row["segmenting_push_ms"] = median_ms(seg_push, n_push, args.warmup)
        row["skipped"] = round(1 - len(fed) / (S * n_push), 3)
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
