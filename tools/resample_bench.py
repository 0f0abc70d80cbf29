"""Resampling to 16 kHz on the H100: kernel time of ``masr_resample_f32`` for 32 x 10 s batches at 48 / 44.1 / 8 kHz
(CUDA events over >= 50 launches after a warm-up), with outputs/s and the tap / float64 operation counts derived from the
shapes; then end-to-end ``MASRPredictor.predict_batches`` audio-s/s on the same audio at 48 kHz against 16 kHz, the two
alternated.  One process; prints the card name and power limit first and one JSON line at the end.

    python tools/resample_bench.py [--iters 50] [--batches 6] [--reps 3]
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
sys.path.insert(0, ROOT)

from masr_b200 import _lib, build as _build, synth  # noqa: E402
from masr_b200.resample import MODEL_RATE, device_table, kaiser_best_table, offsets, output_length  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True).stdout.strip()
    except OSError:
        return torch.cuda.get_device_name()


def tap_count(n, sr):
    """Taps resampy's loop takes for n input samples at sr (both wings of every output), from the shapes."""
    n_out = output_length(n, sr)
    ratio = MODEL_RATE / sr
    scale = min(1.0, ratio)
    step = int(scale * 512)
    nwin = len(kaiser_best_table())
    t = np.arange(n_out) * (1.0 / ratio)
    m = t.astype(np.int64)
    frac = scale * (t - m)
    off_l = (frac * 512).astype(np.int64)
    off_r = ((scale - frac) * 512).astype(np.int64)
    return n_out, int(np.minimum(m + 1, (nwin - off_l) // step).sum() + np.minimum(n - m - 1, (nwin - off_r) // step).sum())


def kernel_leg(sr, B, seconds, iters):
    dev = torch.device("cuda", torch.cuda.current_device())
    n = int(sr * seconds)
    waves = [synth.speechlike_audio(100 + i, n) for i in range(B)]
    out = [output_length(n, sr)] * B
    xo, yo = offsets([n] * B), offsets(out)
    x = torch.from_numpy(np.concatenate(waves)).to(dev)
    y = torch.empty(int(yo[-1]), device=dev)
    xo_d, yo_d = torch.from_numpy(xo).to(dev), torch.from_numpy(yo).to(dev)
    r_d = torch.full((B,), sr, dtype=torch.int32, device=dev)
    tab = device_table(dev)
    st = torch.cuda.current_stream().cuda_stream

    def launch():
        _lib.call("masr_resample_f32", x.data_ptr(), xo_d.data_ptr(), r_d.data_ptr(), MODEL_RATE, B, tab.data_ptr(),
                  tab.numel(), y.data_ptr(), yo_d.data_ptr(), out[0], sr, st)
    for _ in range(5):
        launch()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        launch()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / iters
    n_out, taps = tap_count(n, sr)
    outputs, taps = B * n_out, B * taps
    # per tap: 2 table loads, scale*WIN twice + difference + eta*delta + add (5 fp64 ops for the weight), the product and
    # the accumulate (2), and the float32 <-> float64 round trip of the accumulator (2 conversions)
    return {"rate": sr, "batch": f"{B} x {seconds:g} s", "kernel_ms": round(ms, 4), "outputs_per_s": round(outputs / ms * 1e3, 1),
            "taps": taps, "fp64_ops": 7 * taps, "f32_f64_conversions": 2 * taps,
            "fp64_gflops": round(7 * taps / ms * 1e-6, 1), "launches_timed": iters}


def e2e_leg(nbatches, reps, B=32, seconds=10.0):
    import yaml
    from masr_b200.predict import MASRPredictor
    tmp = tempfile.mkdtemp(prefix="resample_bench_")
    mp, vp = os.path.join(tmp, "m.pt"), os.path.join(tmp, "vocabulary.txt")
    torch.save(synth.to_torch(synth.conformer_state_dict(0)), mp)
    synth.write_vocabulary(vp)
    cfg = {"use_model": "conformer", "streaming": True, "decoder": "ctc_greedy",
           "preprocess_conf": {"feature_method": "fbank", "n_mels": 80, "sample_rate": 16000, "use_dB_normalization": True,
                               "target_dB": -20},
           "dataset_conf": {"dataset_vocab": vp}}
    cp = os.path.join(tmp, "c.yml")
    with open(cp, "w") as f:
        yaml.safe_dump(cfg, f)
    pred = MASRPredictor(configs=cp, model_path=mp, use_gpu=True, resample=True)
    a48 = [[synth.speechlike_audio(1000 + 37 * k + i, int(48000 * seconds)) for i in range(B)] for k in range(nbatches)]
    a16 = [[synth.speechlike_audio(1000 + 37 * k + i, int(16000 * seconds)) for i in range(B)] for k in range(nbatches)]

    def run(batches, sr):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in pred.predict_batches(batches, sample_rate=sr):
            pass
        torch.cuda.synchronize()
        return nbatches * B * seconds / (time.perf_counter() - t0)
    run(a48[:2], 48000)
    run(a16[:2], 16000)
    r48, r16 = [], []
    for _ in range(reps):
        r48.append(run(a48, 48000))
        r16.append(run(a16, 16000))
    return {"batches": f"{nbatches} x {B} x {seconds:g} s", "audio_s_per_s_48k": [round(v) for v in r48],
            "audio_s_per_s_16k": [round(v) for v in r16]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--batches", type=int, default=6)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("resample_bench needs a CUDA device")
    _build.build()
    print("card:", card(), flush=True)
    res = {"card": card(), "kernel": [kernel_leg(sr, 32, 10.0, max(50, args.iters)) for sr in (48000, 44100, 8000)]}
    for k in res["kernel"]:
        print(k, flush=True)
    res["end_to_end"] = e2e_leg(args.batches, args.reps)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
