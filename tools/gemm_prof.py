"""Dev tool (run under ncu): a handful of masr_gemm_tc_f16x2 launches on the FFN shapes of the headline step
(M = 7936): w_1 once per MASR_TC_FLAGS value in GP_FLAGS (default 1), then w_2.  `ncu --set full -k regex:tc_gemm -c 4 ...`."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from masr_b200 import _lib

_lib.load()
_lib.call("masr_check_device")
dev = torch.device("cuda", torch.cuda.current_device())
M = 7936
st = torch.cuda.current_stream().cuda_stream


def P(t):
    return None if t is None else t.data_ptr()


def pair(r, c):
    x = torch.randn(r, c, device=dev)
    h = torch.empty(r, c, dtype=torch.float16, device=dev)
    l = torch.empty_like(h)
    _lib.call("masr_split_f16", P(x), P(h), P(l), x.numel(), st)
    return h, l


def run(N, K, epi, want_c, want_p, want_r, flags, reps=2):
    os.environ["MASR_TC_FLAGS"] = str(flags)
    Ah, Al = pair(M, K)
    Wh, Wl = pair(N, K)
    b = torch.randn(N, device=dev)
    C = torch.empty(M, N, device=dev) if want_c else None
    Ch = torch.empty(M, N, dtype=torch.float16, device=dev) if want_p else None
    Cl = torch.empty_like(Ch) if want_p else None
    R = torch.randn(M, N, device=dev) if want_r else None
    for _ in range(reps):
        _lib.call("masr_gemm_tc_f16x2", P(Ah), P(Al), K, P(Wh), P(Wl), P(b), P(R), N, P(C), P(Ch), P(Cl), N, M, N, K, epi, 0.5, st)
    torch.cuda.synchronize()


for fl in os.environ.get("GP_FLAGS", "1").split(","):
    run(2048, 256, 1, False, True, False, int(fl))
run(256, 2048, 5, True, False, True, 5)
