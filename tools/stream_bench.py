"""Dev tool / BASELINE.json config 3: `configs/squeezeformer.yml` streaming, N live streams (default 64), every stream pushes
0.5 s (8000-sample) int16 PCM chunks; `StreamPool.push` = the `predict_stream` semantics of the reference for every stream
(67-frame windows, stride 64, greedy) with one batched chunk step per round.  Prints one JSON line: audio-s/s, per-push
latency (ms), launches per push.  Also runs the Conformer, the EfficientConformer and the DeepSpeech2 with --model.
Synthetic audio + weights.

--decoder ctc_beam_search decodes every slot with the GPU prefix beam search (``StreamPool(beam=...)``; --beam-size, and
--lm-order N fuses a synthetic N-gram character ARPA LM from ``synth.character_lm_arpa``).  The beam kernels' time per
round (top-k + prefix beam, CUDA events) is taken over --prof-pushes extra pushes launched eagerly after the timed ones."""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from masr_b200 import synth
from masr_b200.stream_pool import StreamPool

ap = argparse.ArgumentParser()
ap.add_argument("--model", default="squeezeformer", choices=["squeezeformer", "conformer", "efficient_conformer", "deepspeech2"])
ap.add_argument("--streams", type=int, default=64)
ap.add_argument("--pushes", type=int, default=40)
ap.add_argument("--warm", type=int, default=6)
ap.add_argument("--decoder", default="ctc_greedy", choices=["ctc_greedy", "ctc_beam_search"])
ap.add_argument("--beam-size", type=int, default=300)
ap.add_argument("--lm-order", type=int, default=0, help="0: no LM")
# the synthetic LM covers nearly the whole vocabulary and gets mild weights: the synthetic models emit arbitrary characters,
# and with the shipped config's alpha 2.2 / beta 4.3 the LM would leave every transcript empty (nothing to check)
ap.add_argument("--alpha", type=float, default=0.5)
ap.add_argument("--beta", type=float, default=2.0)
ap.add_argument("--prof-pushes", type=int, default=3)
args = ap.parse_args()

if args.model == "squeezeformer":
    from masr_b200.squeezeformer import SqueezeformerEngine
    eng = SqueezeformerEngine(synth.squeezeformer_state_dict(0, streaming=True), streaming=True)
elif args.model == "efficient_conformer":
    from masr_b200.engine import EfficientConformerEngine
    eng = EfficientConformerEngine(synth.efficient_conformer_state_dict(0), streaming=True)
elif args.model == "deepspeech2":
    from masr_b200.deepspeech2 import DeepSpeech2Engine
    eng = DeepSpeech2Engine(synth.deepspeech2_state_dict(0, streaming=True), streaming=True)
else:
    from masr_b200.engine import ConformerEngine
    eng = ConformerEngine(synth.conformer_state_dict(0), streaming=True)
S, PUSH = args.streams, 8000
beam = None
if args.decoder == "ctc_beam_search":
    beam = {"beam_size": args.beam_size, "cutoff_prob": 0.99, "cutoff_top_n": 40}
    if args.lm_order:
        import tempfile
        from masr_b200.lm import CharLM
        with tempfile.TemporaryDirectory() as td:
            arpa = os.path.join(td, f"char{args.lm_order}.arpa")
            synth.character_lm_arpa(arpa, seed=args.lm_order, order=args.lm_order, n_chars=4200, n_sentences=600)
            beam.update(lm=CharLM(arpa, synth.vocabulary()), alpha=args.alpha, beta=args.beta)
prof_pushes = args.prof_pushes if beam is not None else 0
n_push = args.warm + args.pushes + prof_pushes
total = n_push * PUSH
# every fourth stream carries speech-like audio (non-empty transcripts for the correctness check), the rest noise
pcm = [(np.clip(synth.speechlike_audio(500 + s, total) if s % 4 == 0 else synth.noise_audio(500 + s, total), -1, 1) * 32767).astype("<i2")
       for s in range(S)]
max_frames = (total // 160) // 4 + 64
pool = StreamPool(eng, synth.vocabulary(), n_slots=S, max_frames=max_frames, beam=beam)
lat = []
last_result = {}
l0 = None
beam_ms = None
for k in range(n_push):
    if k == args.warm + args.pushes:
        # eager launches with per-kernel CUDA events (graph replay == eager, tests/test_gpu_stream_pool_beam.py)
        wall = time.perf_counter() - t_start
        launches = eng.launches - l0
        pool.pool.use_graph = False
        eng.prof = {}
    if k == args.warm:
        torch.cuda.synchronize()
        t_start = time.perf_counter()
        l0 = eng.launches
    t0 = time.perf_counter()
    out = pool.push({s: pcm[s][k * PUSH:(k + 1) * PUSH].tobytes() for s in range(S)}, is_end=False)
    for s_, v_ in out.items():
        if v_ is not None:
            last_result[s_] = v_
    torch.cuda.synchronize()
    if args.warm <= k < args.warm + args.pushes:
        lat.append((time.perf_counter() - t0) * 1e3)
if prof_pushes:
    prof, eng.prof = eng.prof, None
    rounds = len(prof.get("prefix_beam", []))
    beam_ms = {tag: sum(a.elapsed_time(b) for a, b in prof[tag]) / max(rounds, 1) for tag in ("ctc_topk", "prefix_beam")}
    beam_ms["rounds"] = rounds
else:
    wall = time.perf_counter() - t_start
    launches = eng.launches - l0
# correctness on a sample (VERDICT r1: the stream lines carried no check): the same PCM of a few streams through a fresh
# ONE-slot pool (= the single-stream predict_stream path the parity tests pin to the reference goldens) must give the same text
verified = {}
texts = {s: last_result.get(s, {}).get("text", "") for s in range(S)}
for s in sorted({0, S // 2, S - 1}):
    solo = StreamPool(eng, synth.vocabulary(), n_slots=1, max_frames=max_frames, beam=beam)
    r = None
    for k in range(n_push):
        r = solo.push({0: pcm[s][k * PUSH:(k + 1) * PUSH].tobytes()}, is_end=False)[0] or r
    verified[s] = bool(r is not None and r["text"] == texts[s] and (s % 4 != 0 or len(r["text"]) > 0))
assert all(verified.values()), verified
audio = S * args.pushes * PUSH / 16000.0
lat = np.asarray(lat)
dec = args.decoder if beam is None else f"ctc_beam_search beam {args.beam_size}" + (f", {args.lm_order}-gram char LM, alpha {args.alpha}, beta {args.beta}" if args.lm_order else "")
print(json.dumps({"config": f"{args.model} streaming, {S} live streams x {args.pushes} pushes of 0.5 s, predict_stream semantics, {dec}",
                  "gpu": torch.cuda.get_device_name(),
                  "audio_seconds_per_second": audio / wall, "push_latency_ms": {"mean": float(lat.mean()), "p50": float(np.median(lat)),
                                                                                "p95": float(np.percentile(lat, 95)), "max": float(lat.max())},
                  "real_time_factor_per_stream": (wall / args.pushes) / 0.5, "kernel_launches_per_push": launches / args.pushes,
                  "beam_kernel_ms_per_round": beam_ms,
                  "sample_text_len": len(texts[0]),
                  "streams_equal_single_stream_path": {str(k): v for k, v in verified.items()}}))
