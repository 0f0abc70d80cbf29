"""Dev tool: what bounds the fused FFN kernel (masr_ffn_tc_f16x2, M = 7936, d = 256, F = 2048)?  Times the launch under
the profiling switches of MASR_FFN_FLAGS — 1: no TMA loads (the MMAs run on stale stages), 2: no MMAs, 4: no hidden
epilogue (no bias / SiLU / split / store of H) — and their combinations.  Outputs are garbage under the switches; only the
timings mean something.  20 launches in a CUDA graph, best of 5 replays.  Prints us per launch, the bytes each launch
streams from L2 (X pairs once per hidden chunk of every row block, W1 and W2 pairs once per hidden chunk of every 2-CTA
cluster's row-block pair, which the TMA multicast delivers to both CTAs; from the shapes) and the implied rate.
AB_LIB=path loads another build of the library; PROBE_WSETS=20 gives every launch its own weights, cold in HBM."""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from masr_b200 import _lib

if os.environ.get("AB_LIB"):
    _lib.LIB_PATH = os.path.abspath(os.environ["AB_LIB"])
_lib.load()
_lib.call("masr_check_device")
dev = torch.device("cuda", torch.cuda.current_device())
REP = 20
M, D, F = 7936, 256, 2048
FM, FHC = 64, 128                                   # rows per row block, hidden columns per chunk (csrc/ffn_tc.cu)


def P(t):
    return t.data_ptr()


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


Ah, Al = split(torch.randn(M, D, device=dev))
# PROBE_WSETS=n: the launches cycle through n weight sets (4 MB each), so with n = 20 every launch finds its weights cold
# in HBM, as the 24 FFN modules of a model step do; the default, one set, keeps them in L2
WSETS = int(os.environ.get("PROBE_WSETS", "1"))
wsets = [split(torch.randn(F, D, device=dev) / 16) + split(torch.randn(D, F, device=dev) / 45) for _ in range(WSETS)]
b1, b2 = torch.randn(F, device=dev) * 0.1, torch.randn(D, device=dev) * 0.1
x = torch.randn(M, D, device=dev)
launch = [0]


def run(s):
    W1h, W1l, W2h, W2l = wsets[launch[0] % WSETS]
    launch[0] += 1
    _lib.call("masr_ffn_tc_f16x2", P(Ah), P(Al), D, P(W1h), P(W1l), P(b1), P(W2h), P(W2l), P(b2), P(x), D, M, D, F, 0.5, s)


nrb, nch = (M + FM - 1) // FM, F // FHC
npairs = (nrb + 1) // 2
l2_bytes = nch * (nrb * FM * D + npairs * (FHC * D + D * FHC)) * 4   # h and l halves of X, W1 and W2 K-blocks per chunk
mma_flop = 3 * 2 * M * 2 * D * F
row = {"lib": os.environ.get("AB_LIB", "in-tree"), "gpu": torch.cuda.get_device_name(), "M": M, "F": F, "weight_sets": WSETS,
       "l2_bytes_per_launch": l2_bytes}
for label, flags in (("full", 0), ("no_loads", 1), ("no_mma", 2), ("no_epilogue", 4), ("loads_only", 6),
                     ("mma_only", 5), ("neither", 3)):
    os.environ["MASR_FFN_FLAGS"] = str(flags)
    us = time_graph(run)
    row[f"{label}_us"] = round(us, 2)
    print(f"# {label:12s} {us:8.2f} us  {l2_bytes / us * 1e-6:5.2f} TB/s of L2 reads if loading"
          f"  {mma_flop / us * 1e-6:6.1f} TFLOP/s of MMA work if multiplying", flush=True)
os.environ.pop("MASR_FFN_FLAGS")
row["full_l2_TBps"] = round(l2_bytes / row["full_us"] * 1e-6, 2)
row["loads_only_l2_TBps"] = round(l2_bytes / row["loads_only_us"] * 1e-6, 2)
row["epilogue_bubble_us"] = round(row["full_us"] - row["no_epilogue_us"], 2)
print(json.dumps(row), flush=True)
