"""The silero VAD on the H100 (``GpuSileroVAD``, csrc/vad.cu): time of the window-parallel encoder and of the
single-CTA recurrence for 1, 10 and 60 minute recordings at 512-sample windows, each from CUDA events over ``--iters``
launches after a warm-up, with the recurrence's time per recurrent step (steps = windows * window / 512).  The host
baseline is the reference's loop, one onnxruntime session call per window, timed on the 1-minute recording when
onnxruntime is installed and reported as "not measured" otherwise.  Prints the card name and power limit first and one
JSON line at the end.

    python tools/vad_bench.py [--model oracle/_ref/silero_vad.onnx] [--iters 5] [--window 512]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from masr_b200 import build as _build, synth  # noqa: E402
from masr_b200.vad import GpuSileroVAD  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True).stdout.strip()
    except OSError:
        return torch.cuda.get_device_name()


def recording(minutes: int) -> np.ndarray:
    """Speech-like stretches and noise, deterministic from the length."""
    n = 16000 * 60 * minutes
    rng = np.random.default_rng(minutes)
    parts, total = [], 0
    while total < n:
        k = int(rng.integers(16000, 16000 * 8))
        parts.append(synth.speechlike_audio(int(rng.integers(1 << 30)), k) if rng.random() < 0.6
                     else synth.noise_audio(int(rng.integers(1 << 30)), k) * np.float32(0.1))
        total += k
    return np.concatenate(parts)[:n].astype(np.float32)


def event_ms(fn, iters):
    fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    times = []
    for _ in range(iters):
        s.record()
        fn()
        e.record()
        e.synchronize()
        times.append(s.elapsed_time(e))
    return float(np.median(times)), float(np.min(times))


def host_baseline(path, audio, W):
    try:
        import onnxruntime
    except ImportError:
        return "not measured (onnxruntime is not installed)"
    sess = onnxruntime.InferenceSession(path)
    h = np.zeros((2, 1, 64), np.float32)
    c = np.zeros((2, 1, 64), np.float32)
    t0 = time.perf_counter()
    for s in range(0, len(audio), W):
        chunk = np.pad(audio[s:s + W], (0, max(0, W - len(audio[s:s + W]))))
        _, h, c = sess.run(None, {"input": chunk[None], "h": h, "c": c, "sr": np.array(16000, np.int64)})
    return (time.perf_counter() - t0) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default=os.path.join(ROOT, "oracle", "_ref", "silero_vad.onnx"))
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--window", type=int, default=512)
    ap.add_argument("--minutes", default="1,10,60")
    args = ap.parse_args()
    _build.build()
    print("card:", card(), flush=True)
    v = GpuSileroVAD(args.model, device="cuda:0", window_size_samples=args.window)
    W, T = args.window, args.window // 512
    rows = []
    for minutes in (int(m) for m in args.minutes.split(",")):
        a = recording(minutes)
        x = torch.from_numpy(a).cuda()
        gx = v.encode(x)
        enc_med, enc_min = event_ms(lambda: v.encode(x), args.iters)
        rec_med, rec_min = event_ms(lambda: v.recur(gx), args.iters)
        tot_med, _ = event_ms(lambda: v.recur(v.encode(x)), args.iters)
        windows = (len(a) + W - 1) // W
        row = {"minutes": minutes, "windows": windows, "steps": windows * T, "encoder_ms": enc_med,
               "recurrence_ms": rec_med, "total_ms": tot_med, "encoder_ms_min": enc_min, "recurrence_ms_min": rec_min,
               "recurrence_us_per_step": rec_med * 1e3 / (windows * T),
               "encoder_us_per_window": enc_med * 1e3 / windows,
               "realtime_factor": minutes * 60e3 / tot_med}
        print(json.dumps(row), flush=True)
        rows.append(row)
    host = host_baseline(args.model, recording(1), W)
    print(json.dumps({"card": card(), "window": W, "iters": args.iters, "gpu": rows, "host_onnxruntime_1min_ms": host}))


if __name__ == "__main__":
    main()
