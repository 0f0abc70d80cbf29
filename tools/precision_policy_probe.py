"""Dev experiment (CPU): per-layer / per-GEMM mixed-precision policies for the tensor-core path (VERDICT r1 item 3).

For every dense contraction of the Conformer the operands are rounded the way a tensor-core scheme would round them, now
chosen PER CALL SITE (block index x GEMM kind) instead of uniformly (tests/precision_probe.py):

    split   activations and weights kept to 22 bits (h + l)   3 MMAs per product   (the shipped scheme)
    a16     activations fp16, weights 22 bits                  2 MMAs  (drops Al.Wh)
    w16     activations 22 bits, weights fp16                  2 MMAs  (drops Ah.Wl)
    fp16    both fp16                                          1 MMA
    bf16    both bf16                                          1 MMA

and the per-frame CTC argmaxes are compared with the float32 oracle on the bench batch (32 x 10 s) — the acceptance bar
is 0 flips (BASELINE.json: bit-exact greedy ids).  Prints a markdown table: policy, MMA cost relative to all-split
(weighted by the FLOPs of each call site), flipped argmaxes, max |d posterior|.

    python tools/precision_policy_probe.py [n_utterances] > precision_policy.md
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
import torch.nn.functional as F

from masr_b200 import synth
from oracle import conformer as oc, fbank as ob

_linear, _conv1d, _conv2d = F.linear, F.conv1d, F.conv2d
COST = {"split": 3, "a16": 2, "w16": 2, "fp16": 1, "bf16": 1, "fp32": 3}
STATE = {"policy": None, "w1_calls": 0, "flops": {}, }


def r11(t):
    return t.half().float()


def r22(t):
    h = t.half().float()
    return h + ((t - h) * 2048.0).half().float() / 2048.0


def rb(t):
    return t.bfloat16().float()


ROUND = {"split": (r22, r22), "a16": (r11, r22), "w16": (r22, r11), "fp16": (r11, r11), "bf16": (rb, rb), "fp32": (lambda t: t, lambda t: t)}


def site_mode(kind):
    layer = min(11, STATE["w1_calls"] // 2) if kind not in ("conv2", "embed", "ctc") else -1
    pol = STATE["policy"]
    mode = pol(layer, kind)
    return mode


def account(kind, mode, flops):
    d = STATE["flops"]
    d["total"] = d.get("total", 0) + 3 * flops
    d["used"] = d.get("used", 0) + COST[mode] * flops


def linear(x, w, b=None):
    n, k = w.shape
    if n == 2048:
        kind = "ffn_w1"
    elif k == 2048:
        kind = "ffn_w2"
    elif k > 2048:
        kind = "embed"
    elif n > 2048:
        kind = "ctc"
    else:
        kind = "attn_proj"                       # q, k, v, out (and linear_pos, which the engine precomputes in fp32)
    mode = site_mode(kind)
    if kind == "ffn_w2":
        STATE["w1_calls"] += 0
    ra, rw = ROUND[mode]
    account(kind, mode, 2.0 * x.numel() / k * n * k)
    y = _linear(ra(x), rw(w), b)
    if kind == "ffn_w1":
        STATE["w1_calls"] += 1
    return y


def conv1d(x, w, b=None, *a, **k):
    if w.shape[-1] == 1 and k.get("groups", 1) == 1:
        mode = site_mode("conv_pw")
        ra, rw = ROUND[mode]
        account("conv_pw", mode, 2.0 * x.shape[0] * x.shape[2] * w.shape[0] * w.shape[1])
        return _conv1d(ra(x), rw(w), b, *a, **k)
    return _conv1d(x, w, b, *a, **k)


def conv2d(x, w, b=None, *a, **k):
    if w.shape[1] > 1:
        mode = site_mode("conv2")
        ra, rw = ROUND[mode]
        y = _conv2d(ra(x), rw(w), b, *a, **k)
        account("conv2", mode, 2.0 * y.numel() * w.shape[1] * 9)
        return y
    return _conv2d(x, w, b, *a, **k)


def run(feats, sd, cfg, policy):
    STATE["policy"] = policy
    STATE["flops"] = {}
    ids, probs = [], []
    with torch.no_grad():
        for f in feats:
            STATE["w1_calls"] = 0
            p = oc.get_encoder_out(sd, cfg, f)[0]
            ids.append(p.argmax(1).numpy())
            probs.append(p.numpy())
    return np.concatenate(ids), np.concatenate(probs), STATE["flops"]["used"] / STATE["flops"]["total"]


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 32
    torch.set_num_threads(max(1, (os.cpu_count() or 2) - 2))
    sd = synth.to_torch(synth.conformer_state_dict(0))
    cfg = oc.ConformerConfig()
    feats = [torch.from_numpy(ob.featurize(synth.noise_audio(i, 160000)))[None] for i in range(n)]    # bench.make_waves(rank 0)
    policies = [("fp32 (reference arithmetic)", lambda l, k: "fp32"), ("all split (shipped)", lambda l, k: "split")]
    for m in ("fp16", "bf16", "a16", "w16"):
        policies.append((f"all {m}", (lambda mm: lambda l, k: mm)(m)))
    for kk in (1, 2, 4, 6, 8, 10, 12):
        policies.append((f"fp16 in blocks 0..{kk - 1}, split after + conv2/embed/ctc",
                         (lambda c: lambda l, k: "fp16" if 0 <= l < c else "split")(kk)))
    for kk in (2, 6, 12):
        policies.append((f"a16 in blocks 0..{kk - 1}, split elsewhere", (lambda c: lambda l, k: "a16" if 0 <= l < c else "split")(kk)))
        policies.append((f"w16 in blocks 0..{kk - 1}, split elsewhere", (lambda c: lambda l, k: "w16" if 0 <= l < c else "split")(kk)))
    for kind in ("ffn_w1", "ffn_w2", "attn_proj", "conv_pw", "conv2", "embed", "ctc"):
        for m in ("fp16", "a16", "w16"):
            policies.append((f"{m} for {kind} only (all blocks), split elsewhere", (lambda kd, mm: lambda l, k: mm if k == kd else "split")(kind, m)))
    for m in ("fp16", "w16", "a16"):
        policies.append((f"{m} for ffn_w1+ffn_w2 in blocks 0..5 only", (lambda mm: lambda l, k: mm if (k in ("ffn_w1", "ffn_w2") and 0 <= l < 6) else "split")(m)))
    F.linear, F.conv1d, F.conv2d = linear, conv1d, conv2d
    try:
        base_ids, base_p, _ = run(feats, sd, cfg, policies[0][1])
        print(f"# Mixed-precision policy probe — {n} x 10 s (bench batch, weight seed 0), {base_ids.size} frames; bar: 0 flipped argmaxes\n")
        print("| policy | MMA cost vs all-split | flipped argmaxes | max abs d(posterior) |")
        print("|---|---:|---:|---:|")
        for name, pol in policies[1:]:
            ids, p, cost = run(feats, sd, cfg, pol)
            print(f"| {name} | {cost:.3f} | {int((ids != base_ids).sum())} | {np.abs(p - base_p).max():.2e} |", flush=True)
    finally:
        F.linear, F.conv1d, F.conv2d = _linear, _conv1d, _conv2d


if __name__ == "__main__":
    main()
