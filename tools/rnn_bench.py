"""Dev tool: the DeepSpeech2 recurrences, LSTM against GRU (``encoder_conf.use_gru``), in one session.

  kernel  ``masr_lstm_seq_f32`` / ``masr_gru_seq_f32`` at B = 32, T = 250, H = 1024 (10 s utterances, one layer and
          direction): CUDA events around --reps launches after --warmup launches, the two kernels alternated in --rounds
          blocks; median and spread of the blocks.  Also the achieved FP32 rate from the recurrent MACs (B T G H^2).
  pool    one round of the DeepSpeech2 stream pool (``StreamPool`` over synthetic audio) at 64 and 256 streams for either
          cell: the chunk step's CUDA graph replayed 20 times between CUDA events, then 8 pushes launched eagerly with the
          engine's per-tag event timing (recurrence, input projections, the rest), as the LSTM rows of DESIGN.md §9 were taken.

  wide    H = 2048: ``masr_{lstm,gru}_seq_tc_f16x2`` against the per-step form at B = 1 and B = 32, T = 250, alternated;
          the pool rounds again with 2048-wide weights.

Prints one JSON line per measurement and the card's name, power limit and SM clock read in the same run."""
import ctypes
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from masr_b200 import _lib, synth
from masr_b200.deepspeech2 import DeepSpeech2Engine
from masr_b200.stream_pool import StreamPool


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[torch.cuda.current_device()]
    except Exception as e:                      # (the timing does not depend on it; say why it is missing)
        return f"nvidia-smi unavailable: {e}"


def kernel_times(B=32, T=250, H=1024, warmup=20, reps=50, rounds=5):
    dev = torch.device("cuda")
    g = torch.Generator(device="cpu").manual_seed(0)
    lens = torch.full((B,), T, dtype=torch.int32, device=dev)
    nbytes = ctypes.c_int64()
    _lib.call("masr_lstm_seq_workspace_bytes", B, H, ctypes.byref(nbytes))
    ws = torch.empty(nbytes.value, dtype=torch.uint8, device=dev)
    hT = torch.zeros((B + 31) // 32, H, 32, device=dev)
    out = torch.empty(B * T, H, device=dev)
    st = torch.cuda.current_stream().cuda_stream
    args = {}
    for cell, G in (("lstm", 4), ("gru", 3)):
        gx = (torch.randn(B * T, G * H, generator=g) * 0.5).to(dev)
        whh = (torch.randn(G * H, H, generator=g) / H ** 0.5).to(dev)
        aux = torch.zeros(B, H, device=dev) if cell == "lstm" else (torch.randn(H, generator=g) * 0.1).to(dev)
        args[cell] = (f"masr_{cell}_seq_f32", gx, G * H, whh, aux)
    p = lambda t: t.data_ptr()

    def launch(cell):
        fn, gx, ldg, whh, aux = args[cell]
        _lib.call(fn, p(gx), ldg, T, p(whh), p(hT), p(hT), p(aux), p(out), None, None, H, 0, p(lens), B, H, T, 0, p(ws),
                  nbytes.value, st)

    for cell in args:
        for _ in range(warmup):
            launch(cell)
    torch.cuda.synchronize()
    ms = {c: [] for c in args}
    for _ in range(rounds):
        for cell in args:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(reps):
                launch(cell)
            e1.record()
            e1.synchronize()
            ms[cell].append(e0.elapsed_time(e1) / reps)
    res = {}
    for cell, G in (("lstm", 4), ("gru", 3)):
        v = np.asarray(ms[cell])
        flop = 2.0 * B * T * G * H * H
        res[cell] = {"ms_median": float(np.median(v)), "ms_min": float(v.min()), "ms_max": float(v.max()),
                     "recurrent_tflops": flop / (np.median(v) * 1e-3) / 1e12}
    return {"measure": f"seq kernel, B={B} T={T} H={H}, {rounds} alternating blocks of {reps} launches", **res,
            "gru_over_lstm": res["gru"]["ms_median"] / res["lstm"]["ms_median"]}


def wide_kernel_times(B=32, T=250, warmup=3, rounds=5):
    """H = 2048: the tensor-core persistent kernel (masr_{lstm,gru}_seq_tc_f16x2) against the per-step form (T launches of
    masr_{lstm,gru}_step_f32), alternated in `rounds` blocks, one call (one layer and direction) per block and form.  Rates
    from the recurrent MACs (B T G H^2) and from the W_hh bytes one step needs (G H^2 x 4 B: the fp32 matrix, or the pair)."""
    H = 2048
    dev = torch.device("cuda")
    g = torch.Generator(device="cpu").manual_seed(1)
    lens = torch.full((B,), T, dtype=torch.int32, device=dev)
    nbytes = ctypes.c_int64()
    _lib.call("masr_rnn_seq_tc_workspace_bytes", B, H, ctypes.byref(nbytes))
    ws = torch.empty(nbytes.value, dtype=torch.uint8, device=dev)
    nb = (B + 31) // 32
    hT, hA, hB = (torch.zeros(nb, H, 32, device=dev) for _ in range(3))
    out = torch.empty(B * T, H, device=dev)
    st = torch.cuda.current_stream().cuda_stream
    p = lambda t: t.data_ptr()
    res = {}
    for cell, G in (("lstm", 4), ("gru", 3)):
        gx = (torch.randn(B * T, G * H, generator=g) * 0.5).to(dev)
        whh = (torch.randn(G * H, H, generator=g) / H ** 0.5).to(dev)
        packed = torch.empty(G * H * H * 4, dtype=torch.uint8, device=dev)
        _lib.call("masr_rnn_tc_pack_f16x2", p(whh), p(packed), G, H, st)
        aux = torch.zeros(B, H, device=dev) if cell == "lstm" else (torch.randn(H, generator=g) * 0.1).to(dev)

        def tc():
            _lib.call(f"masr_{cell}_seq_tc_f16x2", p(gx), G * H, T, p(packed), p(hT), p(hT), p(aux), p(out), None, None, H, 0,
                      p(lens), B, H, T, 0, p(ws), nbytes.value, st)

        def step():
            for s in range(T):
                _lib.call(f"masr_{cell}_step_f32", p(gx), G * H, T, p(whh), p(hA if s % 2 == 0 else hB), p(hB if s % 2 == 0 else hA),
                          p(aux), p(out), None, None, H, 0, p(lens), B, H, s, 0, st)

        forms = {"seq_tc": tc, "step": step}
        for f in forms.values():
            for _ in range(warmup):
                f()
        torch.cuda.synchronize()
        ms = {k: [] for k in forms}
        for _ in range(rounds):
            for k, f in forms.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                f()
                e1.record()
                e1.synchronize()
                ms[k].append(e0.elapsed_time(e1))
        flop = 2.0 * B * T * G * H * H
        wbytes = 4.0 * G * H * H * T
        cres = {}
        for k in forms:
            v = np.asarray(ms[k])
            m = float(np.median(v))
            cres[k] = {"ms_median": m, "ms_min": float(v.min()), "ms_max": float(v.max()), "us_per_step": m * 1e3 / T,
                       "recurrent_tflops": flop / (m * 1e-3) / 1e12, "whh_bytes_per_s_TB": wbytes / (m * 1e-3) / 1e12}
        cres["step_over_seq_tc"] = cres["step"]["ms_median"] / cres["seq_tc"]["ms_median"]
        res[cell] = cres
    return {"measure": f"H=2048 seq_tc vs per-step, B={B} T={T}, {rounds} alternating blocks of one call", **res}


def pool_round(eng, S, warm=6, prof_pushes=8, replays=20):
    PUSH = 8000
    n_push = warm + prof_pushes
    pcm = [(np.clip(synth.speechlike_audio(500 + s, n_push * PUSH) if s % 4 == 0 else synth.noise_audio(500 + s, n_push * PUSH),
                    -1, 1) * 32767).astype("<i2") for s in range(S)]
    pool = StreamPool(eng, synth.vocabulary(), n_slots=S)
    for k in range(warm):
        pool.push({s: pcm[s][k * PUSH:(k + 1) * PUSH].tobytes() for s in range(S)})
    torch.cuda.synchronize()
    g = pool.pool._graph
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(replays):
        g.replay()
    e1.record()
    e1.synchronize()
    graph_ms = e0.elapsed_time(e1) / replays
    pool.pool.use_graph = False
    eng.prof = {}
    for k in range(warm, n_push):
        pool.push({s: pcm[s][k * PUSH:(k + 1) * PUSH].tobytes() for s in range(S)})
    torch.cuda.synchronize()
    prof, eng.prof = eng.prof, None
    rec_tag = f"{eng.w.cell}_seq" if eng.persistent_lstm else f"{eng.w.cell}_step"
    rounds = len(prof[rec_tag]) // (len(eng.w.rnn) * (1 if eng.persistent_lstm else 16))
    tot = {tag: sum(a.elapsed_time(b) for a, b in evs) / rounds for tag, evs in prof.items()}
    rec, proj = tot.pop(rec_tag), tot.pop("lstm_xproj")
    rest = sum(tot.values())
    # the recurrence computes every lane of every group of 32 slots, active or not
    flop = 2.0 * 16 * len(eng.w.rnn) * eng.G * eng.H * eng.H * 32 * ((S + 31) // 32)
    return {"measure": f"deepspeech2 {eng.w.cell} stream pool round", "streams": S, "round_graph_ms": graph_ms,
            "recurrence_ms": rec, "input_projections_ms": proj, "rest_ms": rest, "recurrence_share": rec / (rec + proj + rest),
            "recurrence_tflops": flop / (rec * 1e-3) / 1e12, "eager_rounds": rounds, "graph_launches": pool.pool._graph_launches}


def main():
    """``rnn_bench.py [1024] [2048]``: the H = 1024 kernels and pools, the H = 2048 ones, or both (the default)."""
    widths = [int(a) for a in sys.argv[1:]] or [1024, 2048]
    torch.cuda.init()
    print(json.dumps({"gpu": card()}), flush=True)
    if 1024 in widths:
        print(json.dumps(kernel_times()), flush=True)
    if 2048 in widths:
        for B in (1, 32):
            print(json.dumps(wide_kernel_times(B=B)), flush=True)
    for H in widths:
        for use_gru in (False, True):
            eng = DeepSpeech2Engine(synth.deepspeech2_state_dict(0, streaming=True, hidden=H, use_gru=use_gru), streaming=True)
            for S in (64, 256):
                print(json.dumps({"hidden": H, **pool_round(eng, S)}), flush=True)
            del eng
            torch.cuda.empty_cache()
    print(json.dumps({"gpu": card()}), flush=True)


if __name__ == "__main__":
    main()
