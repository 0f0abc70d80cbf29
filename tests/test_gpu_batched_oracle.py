"""The batched whole-utterance encoders (``ConformerEngine`` at d = 256 and at d = 512 / 8 heads, ``SqueezeformerEngine``,
``EfficientConformerEngine``, causal and non-causal) against the float64 oracle forward (``encode`` / ``get_encoder_out``
of oracle/conformer.py, squeezeformer.py, efficient_conformer.py with the state dict and the features cast to double),
every utterance run alone through the oracle (the B = 1 semantics every row of a ragged batch must keep).

Each batch is given as subsampled lengths T (feature frames F = 4T + 3 + r, r in 0..3 so conv-1's parity varies) and
reaches one edge of the batched program: every residue mod 2, 3 and 6 (half-rate blocks, attention groups of 3, conv-2
row tiles) plus a row without output frames; the largest batch on the wgmma attention kernel (T <= 256) and the same
utterances beside a 257-frame row on the mma.sync kernel; the half-rate blocks' switch at T = 512 / 513; a 30 s batch;
M = B*T at and across the GEMMs' 128-row tiles.  Per row, over its valid frames: the encoder output of ``engine.encode``,
the posteriors of ``engine.posteriors``, and the fused CTC head's ``maxp`` (``transcribe_features``) within a float64
bound; the frame ids bit for bit wherever the float64 top-2 margin exceeds twice that bound; the frame counts exactly.

Bit-identity properties, on every batch:
  * zero feature rows past each length and log-mel-sized garbage there give bit-identical valid outputs (no kernel reads
    past a row's length);
  * a pass whose cached workspace (every floating buffer, fp16 pairs, the conv-1 parity planes and the CTC head's
    partials included) was filled with NaN first gives finite, bit-identical valid outputs (no kernel reads a buffer
    element an earlier stage of the same pass did not write);
  * each row equals the same utterance run alone whenever both calls make the same attention dispatch (wgmma at
    T <= 256, and at T <= 512 for the half-rate blocks): no stage's result for a row depends on the batch.

The CUDA-graph step (``transcribe`` with Fmax padded to a multiple of 32) gives the eager step's frame ids and ``maxp``
bit for bit, and its ``maxp`` keeps the float64 bound; engines with ``max_len = 300`` match the oracle at T = 299 (the
last row of the position table, and of its ``[::2]`` half-rate form) and reject T = 300 before launching anything.

The synthetic weights have no blank bias (CTC gain 6), so at least 90% of the compared frames are non-blank and the ids
check skips (for a margin below twice the bound) at most 2% of them.

Largest errors measured on an NVIDIA H100 80GB HBM3 at a 700 W power limit over every case of this file (causal and
non-causal together), and the bounds (`TOL`, about 4x); max |engine - float64|:

    model                 encoder output       posteriors, maxp
    conformer (d = 256)   1.3e-5 / 5e-5        6.9e-6 / 2.5e-5     (the fp32 GEMM build: 7.6e-6, 3.6e-6)
    wide (d = 512)        1.8e-5 / 7e-5        4.7e-6 / 2e-5
    squeezeformer         1.4e-5 / 6e-5        5.9e-6 / 2.4e-5
    efficient             8.7e-6 / 3.5e-5      2.6e-6 / 1e-5

Every maximum comes from the 30 s batch (749 queries, each over 749 keys at the full rate and 375 in the half-rate
blocks); the batches of up to 257 frames stay within about half of it (posteriors at most 3.5e-6).  The Squeezeformer's
posterior bound is twice its stream pool's (1.2e-5): the pool's maximum came from 16-frame chunks, while here the
non-causal model's 749-frame row (5.9e-6; the streaming model's reaches 4.9e-6) is compared in one piece.

Every bit-identity property holds for every family and batch, with the conv-1 parity planes poisoned as well: the conv-2
implicit GEMM reads only plane elements conv-1 wrote for the rows it keeps, so no kernel relies on the planes' zero fill.
"""
from collections import defaultdict

import numpy as np
import pytest
import torch

from conftest import make_audio
from kernel_contract import garbage, report
from masr_b200 import synth
from masr_b200.engine import num_frames, subsampled_len
from oracle import conformer as oc, efficient_conformer as oec, fbank as ob, squeezeformer as osq

gpu = pytest.mark.gpu
CTC_GAIN = 6.0

# variant -> (weights, streaming, gemm)
VARIANTS = {
    "conformer": ("conformer", True, "tc"),
    "conformer_nc": ("conformer", False, "tc"),
    "conformer_simt": ("conformer", True, "simt"),
    "wide": ("wide", True, "tc"),
    "wide_nc": ("wide", False, "tc"),
    "squeezeformer": ("squeezeformer", True, "tc"),
    "squeezeformer_nc": ("squeezeformer_nc", False, "tc"),
    "efficient": ("efficient", True, "tc"),
    "efficient_nc": ("efficient", False, "tc"),
}
FAMILY = {"conformer": "conformer", "wide": "wide", "squeezeformer": "squeezeformer", "squeezeformer_nc": "squeezeformer",
          "efficient": "efficient"}

# max |engine - float64| bounds per family: encoder output, posteriors and maxp
TOL = {
    "conformer": {"enc": 5e-5, "probs": 2.5e-5},
    "wide": {"enc": 7e-5, "probs": 2e-5},
    "squeezeformer": {"enc": 6e-5, "probs": 2.4e-5},
    "efficient": {"enc": 3.5e-5, "probs": 1e-5},
}
MEASURED = defaultdict(float)     # (variant, quantity) -> largest error seen in this session


# ---- batches: (T, k) per row; k picks one of several utterances of the same length --------------------------------
def _rows(ts):
    return [(t, 0) for t in ts]


BATCHES = {
    "short": _rows([1, 2, 3, 4, 5, 6, 0, 43]),
    "tc5_ceiling": _rows([256, 255, 129, 128, 1]),
    "mma_first": _rows([257, 255, 129, 128, 1]),
    "half_switch_tc5": _rows([512, 511, 3]),
    "half_switch_mma": _rows([513, 2]),
    "long": _rows([749, 250, 377, 1]),
    "m128": _rows([128]),
    "m129": _rows([129]),
    "m129_b3": [(43, k) for k in range(3)],
    "m128_b64": [(2, k % 8) for k in range(64)],
    "b33_mixed": [(k % 6 + 1, k // 6) for k in range(33)],
}
HALF_RATE_ONLY = ("half_switch_tc5", "half_switch_mma")
CASES = [(v, b) for v in VARIANTS for b in BATCHES
         if not (b in HALF_RATE_ONLY and FAMILY[VARIANTS[v][0]] not in ("squeezeformer", "efficient"))
         and not (v == "conformer_simt" and b not in ("short", "long"))]


def frames_of(t, k):
    return 4 * t + 3 + (t + k) % 4


_FEATS = {}


def utterance(t, k):
    """Log-mel features [F, 80] of utterance (T, k): F = frames_of(t, k) frames, speech or noise."""
    key = (t, k)
    if key not in _FEATS:
        F = frames_of(t, k)
        n = 400 + 160 * (F - 1) + (37 * t + 11 * k) % 160
        kind = "speech" if (t + k) % 3 else "noise"
        f = ob.featurize(make_audio(kind, 5000 + 7 * t + 1000 * k, n))
        assert f.shape[0] == F and subsampled_len(F) == t, (t, k, f.shape)
        _FEATS[key] = f
    return _FEATS[key]


# ---- weights, engines, oracle ------------------------------------------------------------------------------------
_SD = {}


def weights(name):
    if name not in _SD:
        kw = dict(blank_bias=0.0, ctc_gain=CTC_GAIN)
        if name == "conformer":
            _SD[name] = synth.conformer_state_dict(0, **kw)
        elif name == "wide":
            _SD[name] = synth.conformer_state_dict(0, output_size=512, attention_heads=8, **kw)
        elif name == "squeezeformer":
            _SD[name] = synth.squeezeformer_state_dict(0, streaming=True, **kw)
        elif name == "squeezeformer_nc":
            _SD[name] = synth.squeezeformer_state_dict(0, streaming=False, **kw)
        else:
            _SD[name] = synth.efficient_conformer_state_dict(0, **kw)
    return _SD[name]


def state_dict(name, dtype):
    return {k: (v.to(dtype) if v.is_floating_point() else v) for k, v in synth.to_torch(weights(name)).items()}


def oracle(name, causal, max_len=5000):
    """(oracle module, its config) of a weight set."""
    if name == "conformer":
        return oc, oc.ConformerConfig(causal=causal, max_len=max_len)
    if name == "wide":
        return oc, oc.ConformerConfig(d_model=512, heads=8, causal=causal, max_len=max_len)
    if name.startswith("squeezeformer"):
        return osq, osq.SqueezeformerConfig(causal=causal, max_len=max_len)
    return oec, oec.EfficientConfig(causal=causal, max_len=max_len)


def make_engine(variant, max_len=5000):
    from masr_b200.engine import ConformerEngine, EfficientConformerEngine
    from masr_b200.squeezeformer import SqueezeformerEngine
    name, streaming, gemm = VARIANTS[variant]
    cls = {"conformer": ConformerEngine, "wide": ConformerEngine, "squeezeformer": SqueezeformerEngine,
           "squeezeformer_nc": SqueezeformerEngine, "efficient": EfficientConformerEngine}[name]
    return cls(weights(name), streaming=streaming, max_len=max_len, gemm=gemm)


class Oracle:
    """float64 (encoder output, posteriors) of single utterances, cached per (weights, causal, max_len, utterance)."""

    def __init__(self):
        self.sd, self.cache = {}, {}

    def __call__(self, name, causal, f, key=None, max_len=5000):
        ck = None if key is None else (name, causal, max_len, key)
        if ck is not None and ck in self.cache:
            return self.cache[ck]
        if name not in self.sd:
            self.sd[name] = state_dict(name, torch.float64)
        sd = self.sd[name]
        mod, cfg = oracle(name, causal, max_len)
        with torch.no_grad():
            enc = mod.encode(sd, cfg, torch.from_numpy(f).double()[None])
            out = enc[0], oc.ctc_probs(sd, enc)[0]
        if ck is not None:
            self.cache[ck] = out
        return out


@pytest.fixture(scope="module")
def ref():
    return Oracle()


@pytest.fixture(scope="module")
def engines():
    cache = {}

    def get(variant):
        if variant not in cache:
            cache[variant] = make_engine(variant)
        return cache[variant]

    yield get
    if MEASURED:
        print("\n[max error] " + ", ".join(f"{m}.{q}={v:.3g}" for (m, q), v in sorted(MEASURED.items())))


# ---- one batched pass ----------------------------------------------------------------------------------------------
def batch_features(feats, pad):
    """[B, Fmax, 80] float32 with zeros (pad="zero") or ±30 garbage (pad="garbage") past each row's frames."""
    B, Fmax = len(feats), max(f.shape[0] for f in feats)
    x = np.zeros((B, Fmax, 80), np.float32)
    if pad == "garbage":
        x[:] = (garbage((B, Fmax, 80), 300 + B) * 0.03).numpy()
    for b, f in enumerate(feats):
        x[b, :f.shape[0]] = f
    return x


def poison_workspace(eng, B, Fmax):
    """NaN in every floating buffer of the cached (B, Fmax) workspace: fp32 tensors, fp16 pairs, the conv-1 parity planes,
    and the CTC head's softmax partials (a byte buffer of float32 / int32 words)."""
    ws = eng._ws[(B, Fmax)]
    n = 0
    for k, v in ws.items():
        for t in (v if isinstance(v, tuple) else (v,)):
            if not isinstance(t, torch.Tensor):
                continue
            if k == "ctc_part":
                t = t.view(torch.float32)
            if t.is_floating_point():
                t.fill_(float("nan"))
                n += 1
    assert n > 0
    return ws


def run_batch(eng, x, frames, poison=False):
    """encode, posteriors and the fused-head greedy pass of one batch -> per-row dicts of the valid outputs."""
    B, Fmax = x.shape[:2]
    xd = torch.from_numpy(x).to(eng.device)
    if poison:
        poison_workspace(eng, B, Fmax)
    enc, tl, T, _ = eng.encode(xd, frames)
    assert T > 0
    enc = enc.view(B, T, -1).cpu()
    if poison:
        poison_workspace(eng, B, Fmax)
    probs = torch.from_numpy(eng.posteriors(x, frames))
    if poison:
        poison_workspace(eng, B, Fmax)
    res = eng.transcribe_features(xd, frames, return_frames=True)
    maxp = eng._ws[(B, Fmax)]["maxp"][:B * T].view(B, T).cpu()
    assert probs.shape[:2] == (B, T) and res.frame_ids.shape == (B, T)
    assert list(res.frame_lens) == list(tl)
    rows = []
    for b in range(B):
        n = tl[b]
        rows.append({"enc": enc[b, :n], "probs": probs[b, :n], "maxp": maxp[b, :n],
                     "ids": torch.from_numpy(res.frame_ids[b, :n].astype(np.int64)), "n": n})
    return rows


def same_rows(a, b, what):
    for i, (ra, rb) in enumerate(zip(a, b)):
        assert ra["n"] == rb["n"], (what, i)
        for q in ("enc", "probs", "maxp", "ids"):
            assert torch.equal(ra[q], rb[q]), f"{what}: row {i} {q} differs"


def dispatch(eng, T):
    """The attention kernels a batch of encoder length T runs on: wgmma at T <= 256 (full-rate blocks) and, for the
    half-rate blocks of the Squeezeformer / EfficientConformer, at (T + 1) // 2 <= 256."""
    if eng.gemm_path != "tc":
        return ()
    half = any(eng._half_rate(i) for i in range(len(eng.w.layers)))
    return (T <= 256,) + (((T + 1) // 2 <= 256,) if half else ())


class Check:
    """Per-row float64 comparisons of one test, with the informative-frame counts of the ids check."""

    def __init__(self, variant):
        self.variant = variant
        self.tol = TOL[FAMILY[VARIANTS[variant][0]]]
        self.err = defaultdict(float)
        self.frames = self.nonblank = self.skipped = 0

    def record(self, q, got, want):
        assert torch.isfinite(got).all(), f"{self.variant}: non-finite {q}"
        e = (got.double() - want).abs().max().item() if got.numel() else 0.0
        self.err[q] = max(self.err[q], e)
        MEASURED[self.variant, q] = max(MEASURED[self.variant, q], e)

    def row(self, r, enc, probs, with_enc=True):
        n = probs.shape[0]
        assert r["n"] == n, (self.variant, r["n"], n)
        if with_enc:
            self.record("enc", r["enc"], enc)
            self.record("probs", r["probs"], probs)
        top = probs.topk(2, dim=1).values
        self.record("maxp", r["maxp"], top[:, 0])
        sure = (top[:, 0] - top[:, 1]) > 2 * self.tol["probs"]
        am = probs.argmax(1)
        assert torch.equal(r["ids"][sure], am[sure]), f"{self.variant}: frame ids differ from the float64 argmax"
        self.frames += n
        self.nonblank += int((am != 0).sum())
        self.skipped += int((~sure).sum())

    def finish(self, case):
        report(f"{self.variant} {case}", frames=self.frames, nonblank=self.nonblank / max(self.frames, 1),
               skipped=self.skipped, **self.err)
        for q, e in self.err.items():
            bound = self.tol["probs" if q == "maxp" else q]
            assert e <= bound, f"{self.variant} {case}: {q} error {e:.3g} > {bound:.3g}"
        assert self.frames > 0
        assert self.nonblank >= 0.9 * self.frames, (self.nonblank, self.frames)
        assert self.skipped <= 0.02 * self.frames, (self.skipped, self.frames)


# ---- CPU: the float64 oracle whole-utterance forward ----------------------------------------------------------------
@pytest.mark.parametrize("name,causal", [("conformer", True), ("conformer", False), ("wide", True), ("wide", False),
                                         ("squeezeformer", True), ("squeezeformer_nc", False), ("efficient", True),
                                         ("efficient", False)])
def test_float64_oracle_forward_matches_float32(name, causal):
    """The whole-utterance oracle in float64 (the float32 position table widened, as the chunk oracle does) at T = 1, 32
    and 749: it runs, stays float64, and its posteriors agree with the float32 forward to 1e-5, so the GPU tests' bound
    measures the engine alone."""
    mod, cfg = oracle(name, causal)
    sd32, sd64 = state_dict(name, torch.float32), state_dict(name, torch.float64)
    f = ob.featurize(make_audio("speech", 70, 16000 * 31))
    for t in (1, 32, 749):
        x = torch.from_numpy(f[:4 * t + 3])[None]
        with torch.no_grad():
            p32 = mod.get_encoder_out(sd32, cfg, x)
            p64 = mod.get_encoder_out(sd64, cfg, x.double())
        assert p32.dtype == torch.float32 and p64.dtype == torch.float64
        assert p64.shape == p32.shape
        assert (p64 - p32.double()).abs().max().item() < 1e-5


# ---- GPU ------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("variant,batch", CASES)
def test_ragged_batch_against_float64(variant, batch, engines, ref):
    """One batch of `BATCHES` through one engine: every row against its float64 forward alone, then the bit-identity
    properties (zero vs garbage padding, NaN-poisoned workspace, each row alone under the same attention dispatch)."""
    eng = engines(variant)
    name, causal, _ = VARIANTS[variant]
    rows = BATCHES[batch]
    feats = [utterance(t, k) for t, k in rows]
    frames = [f.shape[0] for f in feats]
    zero = run_batch(eng, batch_features(feats, "zero"), frames)
    T = subsampled_len(max(frames))                  # the batch's encoder length at the full frame rate
    chk = Check(variant)
    for (t, k), f, r in zip(rows, feats, zero):
        if t == 0:
            assert r["n"] == 0
            continue
        enc, probs = ref(name, causal, f, (t, k))
        chk.row(r, enc, probs)
    xg = batch_features(feats, "garbage")
    garb = run_batch(eng, xg, frames)
    same_rows(zero, garb, "garbage padding")
    poisoned = run_batch(eng, xg, frames, poison=True)
    same_rows(garb, poisoned, "poisoned workspace")
    alone = {}
    compared = 0
    for (t, k), f, r in zip(rows, feats, zero):
        if t == 0 or dispatch(eng, t) != dispatch(eng, T):
            continue
        if (t, k) not in alone:
            alone[t, k] = run_batch(eng, f[None], [f.shape[0]])[0]
        same_rows([r], [alone[t, k]], f"row T={t} alone")
        compared += 1
    assert compared > 0
    chk.finish(batch)


@gpu
@pytest.mark.parametrize("variant", ("conformer", "wide", "squeezeformer", "efficient"))
def test_graph_step_equals_eager(variant, engines, ref):
    """``transcribe`` through the CUDA graph (Fmax padded to a multiple of 32) against the eager step on the same
    waveforms: frame ids and maxp bit-identical, and the graph's maxp within the float64 bound of the oracle run on the
    GPU's own features."""
    eng = engines(variant)
    name, causal, _ = VARIANTS[variant]
    lens = [16000 * 3 + 17, 9000, 16000 * 5 + 333, 400 + 160 * 6, 16000 * 2 + 1601]
    waves = [make_audio("speech" if i % 2 == 0 else "noise", 80 + i, n) for i, n in enumerate(lens)]
    B = len(waves)
    frames = [num_frames(n) for n in lens]
    Fmax = max(frames)
    q = eng.GRAPH_FRAME_QUANTUM
    Fpad = (Fmax + q - 1) // q * q
    assert Fpad > Fmax and dispatch(eng, subsampled_len(Fpad)) == dispatch(eng, subsampled_len(Fmax))
    assert eng.use_graphs
    try:
        eng.use_graphs = False
        eager = eng.transcribe(waves, return_frames=True)
        Te = eager.frame_ids.shape[1]
        emaxp = eng._ws[(B, Fmax)]["maxp"][:B * Te].view(B, Te).cpu()
    finally:
        eng.use_graphs = True
    graph = eng.transcribe(waves, return_frames=True)
    g = eng._graphs[(B, Fpad, True, -20.0, 0)]
    Tg = g["T"]
    gmaxp = g["ws"]["maxp"][:B * Tg].view(B, Tg).cpu()
    assert list(graph.frame_lens) == list(eager.frame_lens)
    assert graph.tokens == eager.tokens and graph.scores == eager.scores
    feats, fb_frames, _ = eng.fbank(waves)
    feats = feats.cpu().numpy()
    assert fb_frames == frames
    chk = Check(variant)
    for b in range(B):
        n = int(eager.frame_lens[b])
        assert np.array_equal(graph.frame_ids[b, :n], eager.frame_ids[b, :n]), b
        assert torch.equal(gmaxp[b, :n], emaxp[b, :n]), b
        if n == 0:
            continue
        _, probs = ref(name, causal, feats[b, :frames[b]])
        chk.row({"n": n, "maxp": gmaxp[b, :n], "ids": torch.from_numpy(graph.frame_ids[b, :n].astype(np.int64))}, None,
                probs, with_enc=False)
    chk.finish("graph")


@gpu
@pytest.mark.parametrize("variant", ("conformer", "wide", "squeezeformer", "efficient"))
def test_max_len_edge(variant, ref):
    """Engines with a 300-row position table: T = 299 (the table's last row; rows of pe[::2] in the half-rate blocks)
    beside a short row matches the float64 forward with the same table; T = 300 raises the reference's assertion from
    every batched entry point and launches nothing."""
    eng = make_engine(variant, max_len=300)
    name, causal, _ = VARIANTS[variant]
    rows = [(299, 0), (43, 1)]
    feats = [utterance(t, k) for t, k in rows]
    frames = [f.shape[0] for f in feats]
    out = run_batch(eng, batch_features(feats, "garbage"), frames)
    chk = Check(variant)
    for (t, k), f, r in zip(rows, feats, out):
        enc, probs = ref(name, causal, f, (t, k), max_len=300)
        chk.row(r, enc, probs)
    f300 = utterance(300, 0)
    x = batch_features([f300, feats[1]], "zero")
    fr = [f300.shape[0], frames[1]]
    n0 = eng.launches
    msg = "offset: 0 \\+ x.shape\\[1\\]: 300 is larger than the max_len: 300"
    with pytest.raises(AssertionError, match=msg):
        eng.encode(torch.from_numpy(x).to(eng.device), fr)
    with pytest.raises(AssertionError, match=msg):
        eng.posteriors(x, fr)
    with pytest.raises(AssertionError, match=msg):
        eng.transcribe_features(torch.from_numpy(x).to(eng.device), fr)
    assert eng.launches == n0
    chk.finish("max_len")
