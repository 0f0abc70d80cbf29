"""Dev tool: A/B of the headline device step (32 x 10 s, conformer streaming, greedy; inputs resident; one CUDA graph per
variant) under different kernel-selection environments, INTERLEAVED in one process so that box-to-box and thermal drift
cancel: every round replays each variant's graph `REPS` times (L2 flushed before every replay, CUDA events), `ROUNDS` rounds.
Also checks that every variant produces the same token ids.  Variants: name=ENV1:VAL1,ENV2:VAL2 ... on the command line
(switches the library reads per launch), e.g.
    python tools/step_ab.py default= unstaged=MASR_TC_FLAGS:0
Without arguments the default variant alone runs (with AB_LIB: the step time of another build of the library).
Not a bench value."""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from masr_b200 import _lib

if os.environ.get("AB_LIB"):                      # A/B of two builds of the library: load this one instead of the in-tree .so
    _lib.LIB_PATH = os.path.abspath(os.environ["AB_LIB"])
from masr_b200 import synth
from masr_b200.engine import ConformerEngine

ROUNDS = int(os.environ.get("AB_ROUNDS", "4"))
REPS = int(os.environ.get("AB_REPS", "8"))
variants = []
for a in sys.argv[1:]:
    name, _, envs = a.partition("=")
    variants.append((name, dict(kv.split(":") for kv in envs.split(",") if kv)))
if not variants:
    variants = [("default", {})]
touched = sorted({k for _, e in variants for k in e})

eng = ConformerEngine(synth.conformer_state_dict(0, 4233), streaming=True)
waves = [synth.speechlike_audio(100 + i, 160000) if i % 2 else synth.noise_audio(100 + i, 160000) for i in range(32)]
flush = torch.empty(256 << 20, dtype=torch.uint8, device=eng.device)
steps, toks = {}, {}
for name, env in variants:
    for k in touched:
        os.environ.pop(k, None)
    os.environ.update(env)
    eng._graphs.clear()
    st = eng.prepare_resident(waves)
    for _ in range(3):
        ws = st()
    torch.cuda.synchronize()
    steps[name] = st
    toks[name] = ws["out_pack"].clone()
for k in touched:
    os.environ.pop(k, None)
same = all(bool(torch.equal(toks[variants[0][0]], t)) for t in toks.values())
ms = {n: [] for n, _ in variants}
for r in range(ROUNDS):
    order = variants if r % 2 == 0 else variants[::-1]
    for name, _ in order:
        tot = 0.0
        for _ in range(REPS):
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            steps[name]()
            e1.record()
            e1.synchronize()
            tot += e0.elapsed_time(e1)
        ms[name].append(tot / REPS)
out = {"lib": os.environ.get("AB_LIB", "in-tree"), "identical_outputs": same, "rounds": ROUNDS, "reps": REPS,
       "ms_per_step": {n: {"median": round(float(np.median(v)), 4), "min": round(min(v), 4), "all": [round(x, 4) for x in v]} for n, v in ms.items()}}
print(json.dumps(out))
sys.exit(0 if same else 1)
