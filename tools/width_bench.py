"""Dev tool: the 32 x 10 s causal Conformer step at both supported model widths, d = 256 (4 heads) and d = 512 (8 heads), in
one process: synthetic weights, 12 blocks, ffn 2048, ctc_greedy.  After warm-up the two engines run alternately; one JSON line
per width with
  * audio-seconds per second (host clock around blocking `transcribe` calls, which end in a device synchronise),
  * the per-tag kernel times of one step from the engine's event profiler (`eng.prof`; event pairs around single eager
    launches, so each includes launch latency), and
  * for conv-2, the two FFN GEMMs and the depthwise kernel the FLOPs / bytes the algorithm needs, computed from shapes,
    beside the time, with the achieved rate,
and the card's name and power limit.  The 512 step's token ids are checked against the CPU oracle on one utterance first.
Exits non-zero without a GPU.  Dev measurements, not bench.py values."""
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

if not torch.cuda.is_available():
    sys.exit("width_bench needs a CUDA device (sm_90a); nothing is measured without one")

from masr_b200 import synth  # noqa: E402
from masr_b200.engine import ConformerEngine, num_frames, subsampled_len  # noqa: E402
from oracle import conformer as oc, ctc as octc, fbank as ob  # noqa: E402

WIDTHS = {256: 4, 512: 8}
FFN, KERNEL, B, SAMPLES = 2048, 15, 32, 160000
REPS, ROUNDS = 5, 3


def card():
    """Name and power limit of the current device (query only)."""
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
        name, limit = [s.strip() for s in q.split(",")[:2]]
        return {"gpu": name, "power_limit": limit}
    except Exception:
        return {"gpu": torch.cuda.get_device_name(), "power_limit": "unknown"}


def work(d):
    """Useful work of one launch of the reported kernels at the batch shape, from shapes alone."""
    T = subsampled_len(num_frames(SAMPLES))
    M = B * T
    return {
        "conv2": {"flop": 2.0 * M * 19 * d * 9 * d},
        "ffn_w1": {"flop": 2.0 * M * d * FFN},
        "ffn_w2": {"flop": 2.0 * M * d * FFN},
        # depthwise conv + LayerNorm + SiLU: fp32 rows in, one fp16 (h, l) pair out; 2 k FMA-flops per element
        "dwconv_ln_silu": {"flop": 2.0 * KERNEL * M * d, "bytes": M * d * (4 + 2 * 2)},
    }


def main():
    waves = [synth.noise_audio(1000 + i, SAMPLES) for i in range(B)]
    audio = B * SAMPLES / 16000.0
    engines, sds = {}, {}
    for d, h in WIDTHS.items():
        sds[d] = synth.conformer_state_dict(0, output_size=d, attention_heads=h, linear_units=FFN, cnn_module_kernel=KERNEL)
        engines[d] = ConformerEngine(sds[d], streaming=True)
    for d, eng in engines.items():                          # warm-up: module load, workspaces, graph capture
        for _ in range(2):
            out = eng.transcribe(waves)
        if d == 512:
            feat = torch.from_numpy(ob.featurize(waves[0].copy()))
            with torch.no_grad():
                probs = oc.get_encoder_out(synth.to_torch(sds[d]), oc.ConformerConfig(d_model=d, heads=WIDTHS[d]), feat[None])[0].numpy()
            assert list(out.tokens[0]) == list(octc.collapse(octc.best_path(probs)[0])), "d = 512: token ids differ from the CPU oracle"
    secs = {d: [] for d in WIDTHS}
    for _ in range(ROUNDS):                                 # alternate the widths: drift of the shared card hits both
        for d, eng in engines.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(REPS):
                eng.transcribe(waves)
            torch.cuda.synchronize()
            secs[d].append((time.perf_counter() - t0) / REPS)
    info = card()
    for d, eng in engines.items():
        eng.profile(True)                                   # (profiled steps launch eagerly, not from the CUDA graph)
        eng.transcribe(waves)
        torch.cuda.synchronize()
        summ = eng.profile_summary()
        eng.profile(False)
        kernels = {tag: {"launches": n, "ms": round(ms, 4)} for tag, (n, ms) in sorted(summ.items())}
        for tag, wk in work(d).items():
            if tag in kernels:
                per = kernels[tag]["ms"] / kernels[tag]["launches"] * 1e-3
                kernels[tag]["per_launch"] = {k: v for k, v in wk.items()}
                kernels[tag]["per_launch"]["ms"] = round(per * 1e3, 4)
                kernels[tag]["per_launch"]["tflop_per_s"] = round(wk["flop"] / per / 1e12, 2)
                if "bytes" in wk:
                    kernels[tag]["per_launch"]["gb_per_s"] = round(wk["bytes"] / per / 1e9, 1)
        best = min(secs[d])
        print(json.dumps({"tool": "width_bench", "d_model": d, "heads": WIDTHS[d], "blocks": 12, "ffn": FFN, "batch": f"{B} x 10 s causal",
                          "ffn_fused": eng._ffn_fused(), "ms_per_batch": [round(s * 1e3, 3) for s in secs[d]],
                          "audio_seconds_per_second": round(audio / best, 1), "ids_match_cpu_oracle": True if d == 512 else None,
                          "kernel_ms_per_step": kernels, **info}), flush=True)


if __name__ == "__main__":
    main()
