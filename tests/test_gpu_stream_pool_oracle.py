"""The Conformer-family stream pools (``ConformerStreamPool`` at d = 256 and at d = 512 / 8 heads, ``SqueezeformerStreamPool``,
``EfficientConformerStreamPool``) chunk by chunk against the float64 oracle chunk forward (``get_encoder_out_chunk`` of
oracle/conformer.py, squeezeformer.py, efficient_conformer.py with the state dict and the features cast to double).

After every ``pool.step`` each slot that decoded a chunk is compared with its own ``ChunkState``: the CTC posteriors of
every output frame (``keep_probs``) and ``maxp`` within a float64 bound, the frame ids bit for bit wherever the float64
top-2 margin exceeds twice that bound.  Then EVERY slot's state is compared: the K|V cache rows ``[s*cap, s*cap + n)`` of
every layer (fp16 pairs as h + l/2048, the EfficientConformer's grouped layers in float32; half-rate layers against the
oracle's ``[::2]``, which undoes its ``repeat_interleave``) and the conv left context ``xcat[i][s, :lorder]`` against
``cnn_cache``; a slot without frames must keep zeros there.  Before every step each K|V row past a slot's fill holds
±1e3 garbage and each feature row past a slot's frames log-mel-sized garbage, so a misplaced append or shift, a key
count off by one or a read past ``k_lens`` shows up as an error, not as plausible text.

The synthetic weights have no blank bias (the default CTC gain of 6), so the argmax of every frame measured is non-blank
and the maximum posteriors spread over 0.03-0.9: every case asserts that at least 90% of the compared frames are non-blank,
and that the ids check skips (for a margin below twice the bound) at most 2% of them.

Largest errors measured on an NVIDIA H100 80GB HBM3 at a 700 W power limit over every case of this file, and the bounds
(`TOL`, about 4x); max |pool - float64|:

    model                 posteriors, maxp     K|V cache values     conv left context
    conformer (d = 256)   7.2e-6 / 3e-5        9.4e-6 / 4e-5        2.0e-5 / 8e-5
    wide (d = 512)        4.5e-6 / 2e-5        1.3e-5 / 5e-5        2.0e-5 / 8e-5
    squeezeformer         3.2e-6 / 1.2e-5      8.4e-6 / 3e-5        1.8e-5 / 7e-5
    efficient             3.9e-6 / 1.5e-5      5.1e-6 / 2e-5        9.2e-6 / 3.5e-5

The same stream in a one-slot pool and in the last slot of a 33-slot pool, and the eager and the graph-replayed steps,
are bit-identical: no kernel of the chunk step changes its schedule with the number of slots.
"""
from collections import defaultdict

import numpy as np
import pytest
import torch

from conftest import make_audio
from kernel_contract import garbage, report, same
from masr_b200 import synth
from oracle import conformer as oc, efficient_conformer as oec, fbank as ob, squeezeformer as osq

gpu = pytest.mark.gpu
WIN, HOP = 67, 64                 # predict_stream's decoding window and its advance (3 frames overlap)
CTC_GAIN = 6.0
MODELS = ("conformer", "wide", "squeezeformer", "efficient")

# max |pool - float64| bounds per model: posteriors and maxp, K|V cache values, conv left context values
TOL = {
    "conformer": {"probs": 3e-5, "kv": 4e-5, "conv": 8e-5},
    "wide": {"probs": 2e-5, "kv": 5e-5, "conv": 8e-5},
    "squeezeformer": {"probs": 1.2e-5, "kv": 3e-5, "conv": 7e-5},
    "efficient": {"probs": 1.5e-5, "kv": 2e-5, "conv": 3.5e-5},
}
MEASURED = defaultdict(float)     # (model, quantity) -> largest error seen in this session

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
        else:
            _SD[name] = synth.efficient_conformer_state_dict(0, **kw)
    return _SD[name]


def state_dict(name, dtype):
    return {k: (v.to(dtype) if v.is_floating_point() else v) for k, v in synth.to_torch(weights(name)).items()}


def oracle(name, max_len=5000):
    """(oracle module, its config) of a model."""
    if name == "conformer":
        return oc, oc.ConformerConfig(max_len=max_len)
    if name == "wide":
        return oc, oc.ConformerConfig(d_model=512, heads=8, max_len=max_len)
    if name == "squeezeformer":
        return osq, osq.SqueezeformerConfig(causal=True, max_len=max_len)
    return oec, oec.EfficientConfig(max_len=max_len)


def make_engine(name, max_len=5000):
    from masr_b200.engine import ConformerEngine, EfficientConformerEngine
    from masr_b200.squeezeformer import SqueezeformerEngine
    cls = {"conformer": ConformerEngine, "wide": ConformerEngine, "squeezeformer": SqueezeformerEngine,
           "efficient": EfficientConformerEngine}[name]
    return cls(weights(name), streaming=True, max_len=max_len)


def pool_class(name):
    from masr_b200 import stream_pool as sp
    return {"conformer": sp.ConformerStreamPool, "wide": sp.ConformerStreamPool, "squeezeformer": sp.SqueezeformerStreamPool,
            "efficient": sp.EfficientConformerStreamPool}[name]


@pytest.fixture(scope="module")
def feats():
    """Log-mel streams: A 42 s of speech (64 windows), B 20 s of noise, C 15 s and D 8 s of speech."""
    spec = {"A": ("speech", 50, 42), "B": ("noise", 51, 20), "C": ("speech", 52, 15), "D": ("speech", 53, 8)}
    return {k: ob.featurize(make_audio(kind, seed, 16000 * sec)) for k, (kind, seed, sec) in spec.items()}


@pytest.fixture(scope="module")
def engines():
    cache = {}

    def get(name):
        if name not in cache:
            cache[name] = make_engine(name)
        return cache[name]

    yield get
    if MEASURED:
        print("\n[max error] " + ", ".join(f"{m}.{q}={v:.3g}" for (m, q), v in sorted(MEASURED.items())))


def pair_or_f32(bufs, rows):
    if len(bufs) == 1:
        return bufs[0][rows].double()
    return bufs[0][rows].double() + bufs[1][rows].double() / 2048.0


def oracle_kv(att, i, half):
    """Layer i of the oracle's ``att_cache`` [blocks, h, t, 2*dk] as the pool's K|V rows [t', 2d] (heads side by side,
    K then V); a half-rate layer keeps every other row."""
    a = att[i][:, ::2] if half else att[i]
    h, t, two_dk = a.shape
    dk = two_dk // 2
    return torch.cat([a[..., :dk].transpose(0, 1).reshape(t, h * dk), a[..., dk:].transpose(0, 1).reshape(t, h * dk)], 1)


class PoolRun:
    """One pool of `S` slots with keep_probs, a float64 oracle ChunkState per slot (check=True), garbage past every fill."""

    def __init__(self, name, S, max_frames, eng, use_graph=True, check=True, max_len=5000, seed=0):
        self.name, self.S, self.eng = name, S, eng
        self.pool = pool_class(name)(eng, S, max_frames=max_frames, use_graph=use_graph, keep_probs=True)
        self.mod, self.cfg = oracle(name, max_len)
        self.sd = state_dict(name, torch.float64) if check else None
        self.states = [self.mod.ChunkState() for _ in range(S)]
        self.tol = TOL[name]
        dev = eng.device
        p = self.pool
        nl = len(eng.w.layers)
        # (buffers, rows per slot, half rate) of every layer's K|V cache; (buffers, lorder) of every conv left context
        self.kv, self.conv = [], []
        for i in range(nl):
            bufs = (p.kv32[i],) if getattr(p, "kv32", {}).get(i) is not None else tuple(p.kv[i])
            rows = bufs[0].shape[0] // S
            self.kv.append((bufs, rows, rows != p.cap))
            x = p.xcat[i]
            self.conv.append(((x,) if isinstance(x, torch.Tensor) else tuple(x), eng.w.layers[i].kernel - 1))
        big = max(b[0].shape[0] for b, _, _ in self.kv)
        g = garbage((big, self.kv[0][0][0].shape[1]), 100 + seed).to(dev)
        self.kv_garbage = {torch.float32: g, torch.float16: g.half()}
        self.feat_garbage = (garbage((S, WIN, 80), 200 + seed) * 0.03).to(dev)      # ±30: log-mel sized
        self.batch = torch.empty(S, WIN, 80, device=dev)
        self.err = defaultdict(float)
        self.frames = self.nonblank = self.skipped = 0
        self.garble()

    # ---- state --------------------------------------------------------------------------------------------------
    def fill(self, s, half):
        n = self.pool.lens_host[s]
        return (n + 1) // 2 if half else n

    def garble(self):
        """±1e3 in every K|V row past each slot's fill."""
        dev = self.eng.device
        for bufs, rows, half in self.kv:
            r = torch.arange(self.S * rows, device=dev)
            fills = torch.tensor([self.fill(s, half) for s in range(self.S)], device=dev)
            keep = (r % rows < fills[r // rows])[:, None]
            for b in bufs:
                b.copy_(torch.where(keep, b, self.kv_garbage[b.dtype][:b.shape[0]]))

    def reset(self, s):
        self.pool.reset(s)
        self.states[s] = self.mod.ChunkState()
        self.garble()

    def snapshot(self):
        return [b.clone() for bufs, _, _ in self.kv for b in bufs] + [b.clone() for bufs, _ in self.conv for b in bufs]

    # ---- one step -----------------------------------------------------------------------------------------------
    def step(self, chunks):
        """chunks: slot -> float32 log-mel rows [n, 80] (n <= 67).  -> (ids [S, R], maxp [S, R], probs [S, R, V], tout)."""
        S, p = self.S, self.pool
        nfr = [0] * S
        self.batch.copy_(self.feat_garbage)
        for s, c in chunks.items():
            self.batch[s, :len(c)] = torch.from_numpy(c).to(self.batch.device)
            nfr[s] = len(c)
        self.garble()
        ids, maxp, tout = p.step(self.batch, nfr)
        R = p.OUT_ROWS
        out = ids.clone(), maxp.clone(), p.probs.view(S, R, -1).clone(), list(tout)
        for s in range(S):
            if nfr[s] == 0:
                assert tout[s] == 0, s
        if self.sd is not None:
            self.check(chunks, *out)
        return out

    def _record(self, q, got, ref):
        assert torch.isfinite(got).all(), f"{self.name}: non-finite {q}"
        e = (got.cpu().double() - ref.cpu().double()).abs().max().item() if got.numel() else 0.0
        key = "probs" if q == "maxp" else q
        self.err[q] = max(self.err[q], e)
        MEASURED[self.name, q] = max(MEASURED[self.name, q], e)
        assert e <= self.tol[key], f"{self.name}: {q} error {e:.3g} > {self.tol[key]:.3g}"

    def check(self, chunks, ids, maxp, probs, tout):
        tol = self.tol["probs"]
        for s, c in chunks.items():
            with torch.no_grad():
                ref = self.mod.get_encoder_out_chunk(self.sd, self.cfg, torch.from_numpy(c).double()[None], self.states[s], -1)[0]
            t = tout[s]
            assert t == ref.shape[0], (s, t, ref.shape)
            self._record("probs", probs[s, :t], ref)
            top = ref.topk(2, dim=1).values
            self._record("maxp", maxp[s, :t], top[:, 0])
            sure = (top[:, 0] - top[:, 1]) > 2 * tol
            am = ref.argmax(1)
            got = ids[s, :t].cpu().long()
            assert torch.equal(got[sure], am[sure]), (s, got, am)
            self.frames += t
            self.nonblank += int((am != 0).sum())
            self.skipped += int((~sure).sum())
        self.check_state()

    def check_state(self):
        for s in range(self.S):
            st = self.states[s]
            for i, (bufs, rows, half) in enumerate(self.kv):
                n = self.fill(s, half)
                if st.att_cache is None:
                    assert n == 0, (s, i)
                    continue
                ref = oracle_kv(st.att_cache, i, half)
                assert ref.shape[0] == n, (self.name, s, i, ref.shape[0], n)
                self._record("kv", pair_or_f32(bufs, slice(s * rows, s * rows + n)), ref)
            for i, (bufs, lorder) in enumerate(self.conv):
                got = pair_or_f32(tuple(b[s] for b in bufs), slice(0, lorder))
                if st.cnn_cache is None:
                    assert torch.count_nonzero(got) == 0, (self.name, s, i)
                    continue
                self._record("conv", got, st.cnn_cache[i][0][:, -lorder:].t())

    def assert_informative(self):
        assert self.frames > 0
        assert self.nonblank >= 0.9 * self.frames, (self.nonblank, self.frames)
        assert self.skipped <= 0.02 * self.frames, (self.skipped, self.frames)

    def report(self, case):
        report(f"{self.name} {case}", frames=self.frames, nonblank=self.nonblank / max(self.frames, 1),
               skipped=self.skipped, **self.err)


def windows(f, start, n_windows, last=WIN):
    """n consecutive predict_stream windows of f from frame `start`; the last one `last` frames long."""
    return [f[start + k * HOP:start + k * HOP + (WIN if k < n_windows - 1 else last)] for k in range(n_windows)]


def ragged_rounds(feats):
    """S = 5 over 64 rounds.  Slot 0 is the long stream: 64 windows, 1024 cached frames (the key count crosses 64, 128, 256
    and 512 at the full and at the half rate).  Slot 1 joins at round 3 and ends after 10 windows with a 45-frame chunk;
    slot 2 idles through rounds 4-11; slot 3 ends at round 8 with a 30-frame chunk; slot 4 stays empty throughout."""
    rounds = [{} for _ in range(64)]
    for r, c in enumerate(windows(feats["A"], 0, 64)):
        rounds[r][0] = c
    for k, c in enumerate(windows(feats["B"], 0, 10, last=45)):
        rounds[3 + k][1] = c
    for r, c in zip(list(range(4)) + list(range(12, 22)), windows(feats["C"], 0, 14)):
        rounds[r][2] = c
    for k, c in enumerate(windows(feats["D"], 0, 9, last=30)):
        rounds[k][3] = c
    return rounds


# ---- CPU: the float64 oracle chunk forward --------------------------------------------------------------------------
@pytest.mark.parametrize("name", ("conformer", "squeezeformer", "efficient"))
def test_float64_oracle_chunk_forward_matches_float32(name):
    """Four chunks (the last one short) through the float32 and the float64 oracle: posteriors and both caches agree to
    1e-4, so the float64 run computes the same function and the pool tests' bound measures the pool alone."""
    f = ob.featurize(make_audio("speech", 60, 16000 * 3))
    mod, cfg = oracle(name)
    sd32, sd64 = state_dict(name, torch.float32), state_dict(name, torch.float64)
    s32, s64 = mod.ChunkState(), mod.ChunkState()
    for c in windows(f, 0, 4, last=40):
        x = torch.from_numpy(c)[None]
        with torch.no_grad():
            p32 = mod.get_encoder_out_chunk(sd32, cfg, x, s32, -1)
            p64 = mod.get_encoder_out_chunk(sd64, cfg, x.double(), s64, -1)
        assert p32.dtype == torch.float32 and p64.dtype == torch.float64
        assert (p64 - p32.double()).abs().max().item() < 1e-4
        assert (s64.att_cache - s32.att_cache.double()).abs().max().item() < 1e-4
        assert (s64.cnn_cache - s32.cnn_cache.double()).abs().max().item() < 1e-4
        assert s64.offset == s32.offset


# ---- GPU ------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("name", MODELS)
def test_ragged_long_streams_and_slot_reuse(name, feats, engines):
    """Ragged concurrency (`ragged_rounds`), one slot to 1024 cached frames, then slot reuse: the 1024-frame slot is reset,
    its stale rows garbled, and a short stream in it matches a fresh oracle state.  For the pools that take one short
    chunk per stream, the slot that ended with one must be reset before it decodes again."""
    run = PoolRun(name, 5, 1100, engines(name))
    for chunks in ragged_rounds(feats):
        run.step(chunks)
    assert run.pool.lens_host[0] == 1024 and run.pool.lens_host[4] == 0
    if run.pool.SHORT_ONCE:
        before = list(run.pool.lens_host)
        with pytest.raises(AssertionError):
            run.pool.step(run.batch, [0, 0, 0, WIN, 0])
        assert run.pool.lens_host == before
    run.reset(0)
    run.reset(3)
    for k, c in enumerate(windows(feats["D"], 200, 3, last=50)):
        run.step({0: c, 3: windows(feats["C"], 100, 3)[k]})
    run.assert_informative()
    run.report("ragged")


@gpu
@pytest.mark.parametrize("name", ("conformer", "wide"))
def test_conformer_every_key_count_residue(name, feats, engines):
    """Chunks of random lengths (7..67 feature frames: 1..16 encoder frames) mid-stream, which the Conformer pool allows:
    slot 0's key count takes every residue mod 16 and passes 256; slot 1 idles at random; slot 2 decodes full windows."""
    rng = np.random.default_rng(7)
    run = PoolRun(name, 3, 600, engines(name))
    pos = {0: 0, 1: 0, 2: 0}
    src = {0: feats["A"], 1: feats["B"], 2: feats["C"]}
    residues = set()
    for r in range(48):
        chunks = {}
        for s in range(3):
            if s == 1 and rng.random() < 0.3 or s == 2 and r >= 20:
                continue
            n = WIN if s == 2 else int(rng.integers(7, WIN + 1))
            chunks[s] = src[s][pos[s]:pos[s] + n]
            pos[s] += n
        run.step(chunks)
        residues.add(run.pool.lens_host[0] % 16)
    assert residues == set(range(16)) and run.pool.lens_host[0] > 256
    run.assert_informative()
    run.report("residues")


@gpu
@pytest.mark.parametrize("name", MODELS)
def test_capacity_edge(name, feats, engines):
    """max_frames = 401 (the Conformer pool keeps it, the family pools round it to 416): the last slot is filled to
    exactly `cap`, one more frame raises the capacity error and changes no slot's state, and a later step still matches."""
    run = PoolRun(name, 3, 401, engines(name))
    cap = run.pool.cap
    assert cap == (401 if name in ("conformer", "wide") else 416)
    last = windows(feats["A"], 0, cap // 16 + (cap % 16 > 0), last=WIN if cap % 16 == 0 else 7)
    for k, c in enumerate(last):
        chunks = {2: c}
        if k < 10:
            chunks[0] = windows(feats["B"], 0, 10)[k]
        if k % 3 == 0:
            chunks[1] = windows(feats["C"], 0, 9)[k // 3]
        run.step(chunks)
    assert run.pool.lens_host[2] == cap
    before, lens = run.snapshot(), list(run.pool.lens_host)
    run.batch.copy_(run.feat_garbage)
    with pytest.raises(AssertionError, match="capacity"):
        run.pool.step(run.batch, [WIN, 0, 7])
    assert run.pool.lens_host == lens
    assert all(torch.equal(a, b) for a, b in zip(before, run.snapshot()))
    run.step({0: windows(feats["B"], 10 * HOP, 1)[0], 1: feats["D"][:WIN]})
    run.assert_informative()
    run.report("cap")


@gpu
def test_max_len_edge(feats):
    """An engine with a 90-row position table: a key count of max_len - 1 = 89 is accepted and matches the oracle with the
    same table, 90 is rejected and changes nothing."""
    eng = make_engine("conformer", max_len=90)
    run = PoolRun("conformer", 2, 200, eng, max_len=90)
    assert run.pool.frame_bounds() == (200, 90)
    for k, c in enumerate(windows(feats["A"], 0, 6, last=41)):
        run.step({1: c, 0: feats["B"][k * HOP:k * HOP + WIN]} if k < 3 else {1: c})
    assert run.pool.lens_host == [48, 89]
    before, lens = run.snapshot(), list(run.pool.lens_host)
    with pytest.raises(AssertionError, match="capacity"):
        run.pool.step(run.batch, [0, 7])
    assert run.pool.lens_host == lens
    assert all(torch.equal(a, b) for a, b in zip(before, run.snapshot()))
    run.step({0: feats["B"][3 * HOP:3 * HOP + WIN]})
    run.assert_informative()
    run.report("max_len")


@gpu
@pytest.mark.parametrize("name", MODELS)
def test_slot_position_and_pool_size_invariance(name, feats, engines):
    """The same stream in slot 0 of a one-slot pool and in the last slot of a 33-slot pool whose other slots are busy:
    posteriors, ids, maxp and every cache row bit-identical (no stage's result for a row depends on the batch)."""
    eng = engines(name)
    one = PoolRun(name, 1, 200, eng, seed=1)
    many = PoolRun(name, 33, 200, eng, check=False, seed=2)
    mine = windows(feats["D"], 0, 8, last=35)
    for k, c in enumerate(mine):
        a = one.step({0: c})
        others = {s: feats["A"][(s * 97 + k * HOP) % 3000:(s * 97 + k * HOP) % 3000 + WIN] for s in range(32) if (s + k) % 4}
        b = many.step({**others, 32: c})
        t = a[3][0]
        assert b[3][32] == t
        assert torch.equal(a[0][0, :t], b[0][32, :t]) and torch.equal(a[1][0, :t], b[1][32, :t])
        assert torch.equal(a[2][0, :t], b[2][32, :t])
    for (ba, ra, half), (bb, rb, _) in zip(one.kv, many.kv):
        n = one.fill(0, half)
        for x, y in zip(ba, bb):
            assert torch.equal(x[:n], y[32 * rb:32 * rb + n])
    for (ba, lorder), (bb, _) in zip(one.conv, many.conv):
        for x, y in zip(ba, bb):
            assert torch.equal(x[0, :lorder], y[32, :lorder])
    one.report("invariance")


@gpu
@pytest.mark.parametrize("name", MODELS)
def test_graph_replay_equals_eager(name, feats, engines):
    """use_graph=False against the default CUDA-graph replay over a ragged schedule (late join, idling, short final
    chunks, a reset and reuse): outputs and every state buffer bit-identical after every step."""
    eng = engines(name)
    runs = [PoolRun(name, 4, 300, eng, use_graph=g, check=False) for g in (True, False)]
    rounds = [{} for _ in range(12)]
    for k, c in enumerate(windows(feats["A"], 0, 12)):
        rounds[k][0] = c
    for k, c in enumerate(windows(feats["B"], 0, 6, last=50)):
        rounds[2 + k][1] = c
    for r, c in zip((0, 1, 6, 7, 8), windows(feats["C"], 0, 5, last=20)):
        rounds[r][2] = c
    for r, chunks in enumerate(rounds):
        if r == 9:
            for run in runs:
                run.reset(1)
            chunks = {**chunks, 1: feats["D"][:WIN]}
        a, b = (run.step(chunks) for run in runs)
        for x, y in zip(a[:3], b[:3]):
            assert same(x, y), r
        assert a[3] == b[3]
        for x, y in zip(runs[0].snapshot(), runs[1].snapshot()):
            assert same(x, y), r
    assert runs[0].pool._graph is not None and runs[1].pool._graph is None
