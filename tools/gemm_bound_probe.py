"""Dev tool: what bounds the tc_gemm mainloop?  Times the FFN / embed GEMM shapes with the profiling switches of
MASR_TC_FLAGS — 32: no TMA loads (the MMAs run on stale shared memory: tensor pipe + operand reads only),
64: no MMAs (TMA streaming only) — for the single-CTA and the cta_group::2 kernels.  Outputs are garbage under the switches;
only the timings mean something.  20 launches in a CUDA graph, best of 5 replays."""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from masr_b200 import _lib

_lib.load()
_lib.call("masr_check_device")
dev = torch.device("cuda", torch.cuda.current_device())
REP = 20


def P(t):
    return None if t is None else t.data_ptr()


def split(x):
    h = torch.empty(x.shape, dtype=torch.float16, device=dev)
    l = torch.empty_like(h)
    _lib.call("masr_split_f16", P(x), P(h), P(l), x.numel(), torch.cuda.current_stream().cuda_stream)
    return h, l


def time_graph(run):
    for _ in range(2):
        run(torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(side):
        with torch.cuda.graph(g, stream=side, capture_error_mode="thread_local"):
            for _ in range(REP):
                run(side.cuda_stream)
    g.replay()
    torch.cuda.synchronize()
    best = 1e9
    for _ in range(5):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        g.replay()
        e1.record()
        e1.synchronize()
        best = min(best, e0.elapsed_time(e1))
    return best / REP * 1e3


M = 7936
skip = set(filter(None, os.environ.get("PROBE_SKIP", "").split(",")))
shapes = set(sys.argv[1:])
for name, N, K, epi, want_c, want_p, want_r in (("ffn_w2", 256, 2048, 5, True, False, True), ("embed", 256, 4864, 4, True, False, False),
                                                  ("ffn_w1", 2048, 256, 1, False, True, False), ("qkv", 768, 256, 0, True, True, False)):
    if shapes and name not in shapes:
        continue
    Ah, Al = split(torch.randn(M, K, device=dev))
    Wh, Wl = split(torch.randn(N, K, device=dev) * 0.05)
    b = torch.randn(N, device=dev)
    ldc = N
    C = torch.empty(M, ldc, device=dev) if want_c else None
    Ch = torch.empty(M, ldc, dtype=torch.float16, device=dev) if want_p else None
    Cl = torch.empty_like(Ch) if want_p else None
    R = torch.randn(M, ldc, device=dev) if want_r else None

    def run(s):
        _lib.call("masr_gemm_tc_f16x2", P(Ah), P(Al), K, P(Wh), P(Wl), P(b), P(R), ldc, P(C), P(Ch), P(Cl), ldc, M, N, K, epi, 0.5, s)

    row = {"op": name, "N": N, "K": K}
    for label, flags in (("full", 1), ("no_tma", 33), ("no_mma", 65), ("neither", 97)):
        if label in skip:
            continue
        os.environ["MASR_TC_FLAGS"] = str(flags)
        print(f"# {name} {label} ...", flush=True)
        row[f"{label}_us"] = round(time_graph(run), 2)
        print(f"#   {row[f'{label}_us']} us", flush=True)
    os.environ["MASR_TC_FLAGS"] = "1"
    print(json.dumps(row), flush=True)
