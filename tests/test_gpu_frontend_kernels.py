"""The audio front-end kernels of csrc/fbank.cu, one C-ABI entry point at a time (``masr_wave_gain_f32``,
``masr_fbank_workspace_bytes``, ``masr_fbank_f32``), against float64 references of the operation the reference runs
(masr/data_utils/audio.py:256-304,519-574 and torchaudio kaldi.py:514-645, restated step by step in oracle/fbank.py):

  quantize   fl32(x * g), * 2^15, clip to [-32768, 32767], truncate toward zero: the exact int16 samples
  fbank64    frames (snip_edges), DC removal, replicate-left pre-emphasis, povey window, 512-point rFFT, power, mel,
             log(max(e, FLT_EPSILON)), all in float64 from the float32 constants that define the operation (window, mel
             banks, pre-emphasis coefficient)
  gain64     10^((target_db - 10 log10(mean(x^2))) / 20), mean square 0 -> 1

Features are held, element by element, to the normwise error bound of a float32 FFT carried into a mel bin:

    |log max(e^, eps) - log max(e, eps)|  <=  1e-6 + C * 2^-24 * E_f * S_m / max(e, eps)

with e the float64 mel energy, E_f the frame's total power (bins 0..256) and S_m the bin's filter weight sum: quiet bins
beside loud ones get the slack float32 needs, loud bins are held near 1e-5.  On natural signals the mean |delta| must also
stay at or below 5e-6, which catches a small systematic error (a slightly wrong table) that no single element shows.
The CPU tests pin the references and the bar: torchaudio's own float32 output (tests/golden/fbank_golden.npz) meets it with
C = 2 (it reaches 1.28, mean |delta| 1.5e-6).  The kernel is held to C = 8; on an H100 80GB HBM3 (700 W power limit) it
reached C = 5.1 (16 x 30 s batch) with a mean |delta| of at most 1.5e-6 on natural signals.  Crafted inputs reach the
kernels' edges: impulses at every sample position of a frame (each lands in a different lane / register / even-odd slot of
the load, pre-emphasis and window), samples on and one float32 ulp either side of an int16 step with both signs, full-scale
clipping, lengths at frame and 8192-sample-chunk edges, 30 s utterances.

Conventions of tests/kernel_contract.py: garbage before and after the packed samples, outputs pre-filled with NaN (or an int
sentinel) with a guard region behind every output and workspace buffer that must stay untouched.
"""
import ctypes

import numpy as np
import pytest
import torch

from conftest import load_npz, make_audio
from kernel_contract import P, garbage, nan, report, runtime
from masr_b200 import _lib
from oracle import fbank as ob

NUM_MEL = ob.NUM_MEL
EPS = float(ob.EPS)                     # FLT_EPSILON, the log floor (kaldi.py:18,633)
LOG_EPS = np.float32(np.log(EPS))
ABS = 1e-6
C_REF = 2.0                             # torchaudio's golden output reaches 1.28
C_KERNEL = 8.0                          # the kernel reached 5.1 (H100, see the module docstring)
MEAN_TOL = 5e-6
GUARD = 64                              # sentinel elements behind every output and workspace buffer
SENT = -7                               # int sentinel
KSUM = 8192                             # samples per partial sum of the mean square (kSumChunk)
STATUS_GAIN_EXCEEDED = 1

WIN64 = ob.povey_window().astype(np.float64)
MEL64 = ob.mel_banks().astype(np.float64)               # [80, 257]
S_M = MEL64.sum(1)
PREEMPH64 = float(np.float32(ob.PREEMPH))               # the float32 tensor is scaled by the float32 coefficient


# ---- float64 references --------------------------------------------------------------------------------------------------

def quantize(x, g=None):
    """audio.py:264,566-574 on float32 samples: y = fl32(x * g) (no gain: y = x), y * 2^15, clip, truncate toward zero."""
    y = np.asarray(x, np.float32)
    if g is not None:
        y = y * np.float32(g)
    y = y * np.float32(32768.0)
    return np.trunc(np.clip(y, np.float32(-32768.0), np.float32(32767.0))).astype(np.int32)


def fbank64(q):
    """int16 samples -> (log-mel [F, 80], mel energy e [F, 80], frame power total E_f [F]), every step in float64."""
    x = np.asarray(q, np.float64)
    F = ob.num_frames(x.shape[0])
    if F == 0:
        return np.zeros((0, NUM_MEL)), np.zeros((0, NUM_MEL)), np.zeros(0)
    idx = np.arange(ob.FRAME_LEN)[None, :] + ob.FRAME_SHIFT * np.arange(F)[:, None]
    fr = x[idx]                                                            # kaldi.py:82 (snip_edges)
    fr = fr - fr.mean(axis=1, keepdims=True)                               # :183-186
    prev = np.concatenate([fr[:, :1], fr[:, :-1]], axis=1)                 # :195-197 replicate-left
    fr = (fr - PREEMPH64 * prev) * WIN64                                   # :198-204
    spec = np.fft.rfft(fr, n=ob.NFFT, axis=1)                              # :207-211,616
    p = spec.real ** 2 + spec.imag ** 2                                    # :618
    e = p @ MEL64.T                                                        # :630
    return np.log(np.maximum(e, EPS)), e, p.sum(1)                         # :633


def gain64(x, target_db=-20.0):
    """audio.py:287-304,519-529 in float64 (mean square 0 -> 1, audio.py:526-527)."""
    x = np.asarray(x, np.float64)
    ms = float(np.mean(x * x)) if x.size else 0.0
    if ms == 0:
        ms = 1.0
    return 10.0 ** ((target_db - 10.0 * np.log10(ms)) / 20.0)


class Bar:
    """The energy-relative bound over many utterances; keeps the worst ratio C observed and the mean / max |delta|."""

    def __init__(self, C=C_KERNEL):
        self.C, self.ratio, self.sum, self.count, self.max = C, 0.0, 0.0, 0, 0.0

    def add(self, got, q, rows=None, what=""):
        ref, e, E = fbank64(q)
        n = ref.shape[0] if rows is None else min(rows, ref.shape[0])
        ref, e, E = ref[:n], e[:n], E[:n]
        d = np.abs(np.asarray(got[:n], np.float64) - ref)
        slack = 2.0 ** -24 * E[:, None] * S_M[None, :] / np.maximum(e, EPS)
        with np.errstate(divide="ignore", invalid="ignore"):
            r = np.where(d > ABS, (d - ABS) / slack, 0.0)
        bad = np.argwhere(d > ABS + self.C * slack)
        if bad.size:
            f, m = bad[0]
            raise AssertionError(f"{what}: {len(bad)} elements over the bar, first frame {f} bin {m}: kernel "
                                 f"{got[f, m]!r}, float64 {ref[f, m]!r}, ratio {r[f, m]:.3g} > C = {self.C}")
        if d.size:
            self.ratio, self.max = max(self.ratio, float(r.max())), max(self.max, float(d.max()))
            self.sum += float(d.sum())
            self.count += d.size
        return self

    @property
    def mean(self):
        return self.sum / max(1, self.count)

    def report(self, name, natural=False):
        report(name, C=self.ratio, mean_abs=self.mean, max_abs=self.max)
        if natural:
            assert self.mean <= MEAN_TOL, (name, self.mean)


# ---- crafted inputs ------------------------------------------------------------------------------------------------------

def impulse_sweep(A=1000):
    """400 one-frame utterances (int16 values): utterance p is a DC level plus an impulse of +-A LSB at sample p."""
    out = []
    for p in range(ob.FRAME_LEN):
        q = np.full(ob.FRAME_LEN, (p * 7919) % 4001 - 2000, np.int32)
        q[p] += A if (p // 2) % 2 == 0 else -A
        out.append(q)
    return out


def on_step(k, where, g):
    """float32 inputs x whose fl32(x * g) is k/2^15 (where == 0), one float32 ulp below it (-1) or above it (+1).
    -> (x, hit): hit marks the samples that reach their target exactly (a gain above 1 skips some products)."""
    t = (np.asarray(k, np.float64) / 32768).astype(np.float32)
    t = np.where(where < 0, np.nextafter(t, np.float32(-np.inf)), np.where(where > 0, np.nextafter(t, np.float32(np.inf)), t))
    if g is None:
        return t, np.ones(t.shape, bool)
    g32 = np.float32(g)
    x0 = (t.astype(np.float64) / float(g32)).astype(np.float32)
    x, hit = x0.copy(), x0 * g32 == t
    for to in (np.float32(np.inf), np.float32(-np.inf)):
        c = x0
        for _ in range(4):
            c = np.nextafter(c, to)
            ok = ~hit & (c * g32 == t)
            x[ok], hit = c[ok], hit | ok
    return x, hit


QUANT_GAINS = [None, 0.1, 0.70710677, 3.3, 1000.0]


def quant_utterances(g, seed):
    """Signals a few LSB in amplitude over a DC offset, every sample on or one ulp beside an int16 step: one sample quantised
    one LSB off changes its frame's spectrum by O(1).  Then samples at and beyond full scale (the clip is asymmetric:
    32767 / -32768) and, with a gain of 10, a full-scale square wave driven into saturation.
    -> (float32 waves, per-wave coverage (k, where, hit) of the stepped ones)."""
    rng = np.random.default_rng(seed)
    waves, cover = [], []
    for D in (0, 1000, -1000, 20000, -20000):
        n = int(rng.integers(800, 2000))
        k = D + rng.integers(-3, 4, n)
        where = rng.integers(-1, 2, n)
        x, hit = on_step(k, where, g)
        waves.append(x)
        cover.append((k, where, hit))
    f32 = np.float32
    pos = np.array([1.0, 1.5, 2.0, np.nextafter(f32(1), f32(2)), np.nextafter(f32(1), f32(0)), 32767 / 32768,
                    32766 / 32768, 32765 / 32768], f32)
    for v in (pos, -pos, np.array([-1.0, np.nextafter(f32(-1), f32(-2))], f32)):
        x = rng.choice(v, 1200)
        waves.append(x if g is None else (x.astype(np.float64) / np.float32(g)).astype(f32))
    return waves, cover


def square_wave(n=2000):
    t = np.arange(n)
    return (0.9 * np.sign(np.sin(2 * np.pi * t / 50 + 0.3))).astype(np.float32)


# ---- kernel calls --------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def rt():
    return runtime()


def pack(rt, waves, lead, seed):
    """float32 rows packed behind `lead` garbage samples, GUARD garbage samples after the last row -> device samples and
    int64 offsets (the first row starts at `lead`)."""
    lengths = [len(w) for w in waves]
    offs = np.full(len(waves) + 1, lead, np.int64)
    offs[1:] += np.cumsum(lengths, dtype=np.int64)
    buf = garbage((int(offs[-1]) + GUARD,), seed).numpy()
    for w, a in zip(waves, offs):
        buf[a:a + len(w)] = w
    return torch.from_numpy(buf).to(rt.dev), torch.from_numpy(offs).to(rt.dev)


def run_fbank(rt, waves, gain=None, Fmax=None, lead=3, seed=0):
    """One masr_fbank_f32 launch -> features [B, Fmax, 80] on the host.  Checks the output contract on every call: the
    guards behind feats and num_frames untouched, num_frames the kaldi frame count (also past Fmax), every row below
    min(F, Fmax) finite, every row at or past F exactly +0.0."""
    B = len(waves)
    F = [ob.num_frames(len(w)) for w in waves]
    Fmax = max(F, default=0) if Fmax is None else Fmax
    wave, offs = pack(rt, waves, lead, seed)
    g = None if gain is None else torch.tensor(np.asarray(gain, np.float32), device=rt.dev)
    feats = nan((B * Fmax * NUM_MEL + GUARD,), rt.dev)
    nf = torch.full((B + GUARD,), SENT, dtype=torch.int32, device=rt.dev)
    rt.call("masr_fbank_f32", P(wave), P(offs), P(g), B, Fmax, P(feats), P(nf), rt.st())
    fh, nfh = feats.cpu().numpy(), nf.cpu().numpy()
    assert np.isnan(fh[B * Fmax * NUM_MEL:]).all(), "written past feats[B, Fmax, 80]"
    assert (nfh[B:] == SENT).all(), "written past num_frames[B]"
    assert nfh[:B].tolist() == F
    fh = fh[:B * Fmax * NUM_MEL].reshape(B, Fmax, NUM_MEL)
    for b in range(B):
        n = min(F[b], Fmax)
        assert np.isfinite(fh[b, :n]).all(), b
        assert (fh[b, n:] == 0).all() and not np.signbit(fh[b, n:]).any(), b
    return fh


def run_gain(rt, waves, target_db=-20.0, max_gain_db=300.0, max_samples=None, lead=5, seed=1):
    """One masr_wave_gain_f32 launch on a workspace of exactly masr_fbank_workspace_bytes bytes -> (gain, status) on the
    host.  The guards behind gain, status and the workspace must stay untouched."""
    B = len(waves)
    if max_samples is None:
        max_samples = max((len(w) for w in waves), default=0)
    wave, offs = pack(rt, waves, lead, seed)
    nbytes = ctypes.c_int64(-1)
    rt.call("masr_fbank_workspace_bytes", B, max_samples, ctypes.byref(nbytes))
    assert nbytes.value == 8 * B * max(1, -(-max_samples // KSUM))
    ws = torch.full((nbytes.value + GUARD,), 0xA5, dtype=torch.uint8, device=rt.dev)
    gain = nan((B + GUARD,), rt.dev)
    status = torch.full((B + GUARD,), SENT, dtype=torch.int32, device=rt.dev)
    rt.call("masr_wave_gain_f32", P(wave), P(offs), B, max_samples, target_db, max_gain_db, P(gain), P(status), P(ws),
            rt.st())
    gh, sh, wh = gain.cpu().numpy(), status.cpu().numpy(), ws.cpu().numpy()
    assert np.isnan(gh[B:]).all() and (sh[B:] == SENT).all() and (wh[nbytes.value:] == 0xA5).all()
    assert np.isfinite(gh[:B]).all() and set(sh[:B].tolist()) <= {0, STATUS_GAIN_EXCEEDED}
    return gh[:B], sh[:B]


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.int32)


# ---- CPU: the references and the bar ---------------------------------------------------------------------------------------

def test_fbank64_meets_the_bar_against_torchaudio_golden():
    """torchaudio's float32 output (frozen from the reference) is within the bar of fbank64 at C = 2, with a mean |delta|
    under 5e-6: the bar is fair to a correct float32 implementation."""
    z, meta = load_npz("fbank_golden.npz")
    bar = Bar(C_REF)
    for m in meta:
        bar.add(z[m["name"] + "/feat"], z[m["name"] + "/int16"], what=m["name"])
    bar.report("torchaudio golden vs fbank64", natural=True)


def test_quantize_is_the_reference_chain_and_separates_roundings():
    """quantize() equals oracle.fbank.to_int16 after normalize_gain's in-place `y *= factor`, and the crafted samples tell
    truncation toward zero from floor and from round-to-nearest, and the int16 clip from a symmetric one."""
    seen = set()
    for i, g in enumerate(QUANT_GAINS):
        waves, cover = quant_utterances(g, i)
        for x in waves + [square_wave()]:
            y = x.copy()
            if g is not None:
                y *= np.float32(g)
            q = quantize(x, g)
            assert np.array_equal(q, ob.to_int16(y).astype(np.int32))
            s = np.clip(y.astype(np.float64) * 32768, -32768, 32767)
            if (q != np.floor(s)).any():
                seen.add("floor")
            if (q != np.rint(s)).any():
                seen.add("rint")
            if (q == -32768).any():
                seen.add("-32768")
            if (q == 32767).any():
                seen.add("32767")
        for k, where, hit in cover:
            for sgn in (-1, 1):
                for w in (-1, 0, 1):
                    if (hit & (np.sign(k) == sgn) & (where == w)).sum() >= 10:
                        seen.add((g, sgn, w))
        assert all((g, s, w) in seen for s in (-1, 1) for w in (-1, 0, 1)), g
    assert {"floor", "rint", "-32768", "32767"} <= seen
    sq = quantize(square_wave(), 10.0)
    assert sq.max() == 32767 and sq.min() == -32768


def test_gain64_against_the_numpy_float32_chain():
    """gain64 agrees with oracle.fbank.normalize_gain (the reference's float32 chain) to 2e-6."""
    for i, (kind, n, sc) in enumerate([("speech", 9000, 1.0), ("speech", 8193, 0.01), ("noise", 16000, 3.0), ("noise", 1, 1e-3)]):
        x = make_audio(kind, i, n, sc)
        assert abs(gain64(x) / float(ob.normalize_gain(x)[1]) - 1) < 2e-6
    assert gain64(np.zeros(100, np.float32), -20.0) == 0.1


# ---- GPU: masr_fbank_f32 -------------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_fbank_golden_int16_samples(rt):
    """Each golden utterance's int16 samples, passed as int16 / 2^15 with no gain (which quantises back to the same
    integers), against fbank64 and against torchaudio's frozen output."""
    z, meta = load_npz("fbank_golden.npz")
    qs = [z[m["name"] + "/int16"].astype(np.int32) for m in meta]
    waves = [(q.astype(np.float32) / np.float32(32768)) for q in qs]
    assert all(np.array_equal(quantize(w), q) for w, q in zip(waves, qs))
    got = run_fbank(rt, waves)
    bar, gold = Bar(), 0.0
    for b, (m, q) in enumerate(zip(meta, qs)):
        F = ob.num_frames(len(q))
        bar.add(got[b], q, what=m["name"])
        ref, e, E = fbank64(q)
        d = np.abs(got[b, :F].astype(np.float64) - z[m["name"] + "/feat"])
        assert (d <= 2 * ABS + (C_KERNEL + C_REF) * 2.0 ** -24 * E[:, None] * S_M / np.maximum(e, EPS)).all(), m["name"]
        gold = max(gold, float(d.max()))
    bar.report("fbank golden int16", natural=True)
    report("fbank golden int16 vs torchaudio", max_abs=gold)


LENGTHS = [0, 1, 399, 400, 401, 559, 560, 561, 16000, 160123, 480000]


@pytest.mark.gpu
def test_fbank_lengths_fmax_and_num_frames(rt):
    """Lengths at the frame edges up to 30 s in one packed batch, each row with its own gain.  Fmax = max F (not a multiple
    of the 16 frames per CTA) against fbank64; Fmax = max F + 37 and Fmax < max F give the same first rows bit for bit
    (rows past F exactly 0.0, num_frames the full count); Fmax = 0 still writes num_frames; B = 0 writes nothing."""
    waves = [make_audio("speech" if i % 2 else "noise", 40 + i, n, 0.5 + 0.3 * i) for i, n in enumerate(LENGTHS)]
    gains = np.float32(0.37) + np.float32(0.11) * np.arange(len(waves), dtype=np.float32)
    F = [ob.num_frames(n) for n in LENGTHS]
    Fm = max(F)
    assert Fm % 16 and F[:5] == [0, 0, 0, 1, 1]
    full = run_fbank(rt, waves, gains)
    bar = Bar()
    for b, (w, g) in enumerate(zip(waves, gains)):
        bar.add(full[b], quantize(w, g), what=f"n={LENGTHS[b]}")
    bar.report("fbank lengths", natural=True)
    for Fmax in (Fm + 37, 500, 1):
        got = run_fbank(rt, waves, gains, Fmax=Fmax, lead=8, seed=3)
        for b in range(len(waves)):
            n = min(F[b], Fmax)
            assert np.array_equal(bits(got[b, :n]), bits(full[b, :n])), (Fmax, b)
    assert run_fbank(rt, waves, gains, Fmax=0).shape == (len(waves), 0, NUM_MEL)
    assert run_fbank(rt, [], None, Fmax=0).shape == (0, 0, NUM_MEL)
    assert run_fbank(rt, [], None, Fmax=5).shape == (0, 5, NUM_MEL)


@pytest.mark.gpu
def test_fbank_fmax_0_with_zero_byte_buffers(rt):
    """A batch of sub-frame chunks allocated the obvious way: feats [B, 0, 80] (and, when every row is empty, the samples)
    are zero-byte buffers with no address.  With Fmax = 0 those may be NULL and num_frames is still written; with
    Fmax > 0 a NULL feats or wave is still refused."""
    waves = [make_audio("speech", 50 + i, n) for i, n in enumerate([399, 1, 0, 250])]
    wave, offs = pack(rt, waves, 3, 0)
    empty = torch.empty(len(waves), 0, NUM_MEL, device=rt.dev)
    for feats in (None, P(empty)):
        nf = torch.full((len(waves) + GUARD,), SENT, dtype=torch.int32, device=rt.dev)
        rt.call("masr_fbank_f32", P(wave), P(offs), None, len(waves), 0, feats, P(nf), rt.st())
        assert nf.cpu().tolist() == [0] * len(waves) + [SENT] * GUARD
    nothing = torch.empty(0, device=rt.dev)
    offs0 = torch.zeros(4, dtype=torch.int64, device=rt.dev)
    for w in (None, P(nothing)):
        nf = torch.full((3 + GUARD,), SENT, dtype=torch.int32, device=rt.dev)
        rt.call("masr_fbank_f32", w, P(offs0), None, 3, 0, None, P(nf), rt.st())
        assert nf.cpu().tolist() == [0] * 3 + [SENT] * GUARD
    rt.call("masr_fbank_f32", None, P(offs0), None, 3, 0, None, None, rt.st())       # nothing to write
    nf = torch.full((len(waves),), SENT, dtype=torch.int32, device=rt.dev)
    for w, f in ((P(wave), None), (None, P(nan((len(waves) * NUM_MEL,), rt.dev)))):
        with pytest.raises(_lib.MasrB200Error, match="null pointer"):
            rt.call("masr_fbank_f32", w, P(offs), None, len(waves), 1, f, P(nf), rt.st())
    assert (nf.cpu() == SENT).all()


@pytest.mark.gpu
def test_fbank_impulse_sweep(rt):
    """An impulse at every sample position of a frame over a per-utterance DC level: covers each (lane, register, even /
    odd) slot of the load, the pre-emphasis neighbour across registers (p = 64 j - 1, 64 j), the replicate-left sample 0,
    and the tail p = 384..399."""
    qs = impulse_sweep()
    got = run_fbank(rt, [q.astype(np.float32) / np.float32(32768) for q in qs])
    bar = Bar()
    for p, q in enumerate(qs):
        bar.add(got[p], q, what=f"impulse at {p}")
    bar.report("fbank impulse sweep")


@pytest.mark.gpu
def test_fbank_constant_frames_are_exactly_the_log_floor(rt):
    """A constant frame (any integer level, digital silence included) has zero energy after DC removal: every bin is
    float32(log(FLT_EPSILON)) bit for bit, with or without a gain."""
    levels = [0, 1, -1, 7, -32768, 32767, 12345, -20000]
    got = run_fbank(rt, [np.full(1200, v / 32768, np.float32) for v in levels])
    assert got.shape == (len(levels), 6, NUM_MEL)
    assert (bits(got) == bits(LOG_EPS)).all()
    waves = [np.full(1000, 0.3, np.float32), np.full(900, -0.9, np.float32), np.zeros(401, np.float32)]
    gains = [0.70710677, 3.3, 1000.0]
    got = run_fbank(rt, waves, gains)
    for b, (w, g) in enumerate(zip(waves, gains)):
        F = ob.num_frames(len(w))
        assert len(set(quantize(w, g).tolist())) == 1 and (bits(got[b, :F]) == bits(LOG_EPS)).all(), b


@pytest.mark.gpu
def test_fbank_quantisation_bit_exact(rt):
    """Few-LSB signals whose samples sit on, one ulp below and one ulp above an int16 step (both signs), full-scale and
    clipped samples, and a square wave that a gain of 10 drives into saturation.  One sample quantised one LSB off breaks
    the bar, so passing it means the kernel used exactly quantize()'s int16 samples."""
    bar = Bar()
    for i, g in enumerate(QUANT_GAINS):
        waves, _ = quant_utterances(g, i)
        got = run_fbank(rt, waves, None if g is None else [g] * len(waves), lead=3 + i, seed=i)
        for b, x in enumerate(waves):
            bar.add(got[b], quantize(x, g), what=f"gain {g} row {b}")
    sq = square_wave()
    got = run_fbank(rt, [sq], [10.0])
    bar.add(got[0], quantize(sq, 10.0), what="square wave")
    bar.report("fbank quantisation")


@pytest.mark.gpu
def test_fbank_long_batch_with_kernel_gains(rt):
    """B = 16 utterances of 30 s, speech-like and noise, with the gains masr_wave_gain_f32 computes for them."""
    waves = [make_audio("speech" if b % 2 else "noise", 60 + b, 30 * 16000, [1.0, 0.02, 4.0, 0.3][b % 4]) for b in range(16)]
    gains, status = run_gain(rt, waves)
    assert (status == 0).all()
    assert all(abs(g / gain64(w) - 1) <= 1e-6 for g, w in zip(gains, waves))
    got = run_fbank(rt, waves, gains)
    bar = Bar()
    for b, (w, g) in enumerate(zip(waves, gains)):
        bar.add(got[b], quantize(w, g), what=f"row {b}")
    bar.report("fbank 16 x 30 s", natural=True)


@pytest.mark.gpu
def test_fbank_row_independent_of_position_neighbours_fmax_and_launch(rt):
    """An utterance's rows are bit-identical at another batch position and offset, beside other neighbours, with another
    Fmax and on a second launch (the stream pool's slot == single-stream promise rests on it)."""
    u, gu = make_audio("speech", 77, 7777, 0.6), 0.83
    Fu = ob.num_frames(len(u))
    a = dict(waves=[u, make_audio("noise", 1, 5000), make_audio("speech", 2, 300)], gain=[gu, 1.7, 0.2])
    first = run_fbank(rt, **a)
    Bar().add(first[0], quantize(u, gu), what="u").report("fbank independence row")
    again = run_fbank(rt, **a)
    assert np.array_equal(bits(first), bits(again))
    wider = run_fbank(rt, **a, Fmax=Fu + 5, lead=4)
    moved = run_fbank(rt, [make_audio("speech", 3, 20000, 2.0), np.zeros(0, np.float32), make_audio("noise", 4, 401), u],
                      [3.0, 1.0, 0.5, gu], lead=10, seed=5)
    for other in (wider[0], moved[3]):
        assert np.array_equal(bits(other[:Fu]), bits(first[0, :Fu]))


# ---- GPU: masr_wave_gain_f32 / masr_fbank_workspace_bytes -----------------------------------------------------------------

def _check_gains(name, waves, gains, status, target_db=-20.0):
    """Where |rms_db| and the required gain are under 64 dB, relative error <= 1e-6 against gain64 (one float32 ulp of
    rms_db moves the gain by 8.8e-7 there) and <= 2e-6 against the numpy float32 chain; further out, where a float32 ulp
    of the dB values is twice as large, <= 2e-6 against gain64.  An empty row gets a finite gain."""
    e64 = enp = 0.0
    for w, g, s in zip(waves, gains, status):
        assert s == 0 and np.isfinite(g)
        if len(w) == 0:
            continue
        rel = abs(g / gain64(w, target_db) - 1)
        rms_db = 10 * np.log10(max(float(np.mean(np.asarray(w, np.float64) ** 2)), 1e-300))
        if abs(rms_db) < 64 and abs(target_db - rms_db) < 64:
            assert rel <= 1e-6, (len(w), rms_db, rel)
            relnp = abs(g / float(ob.normalize_gain(w, target_db)[1]) - 1)
            assert relnp <= 2e-6, (len(w), relnp)
            e64, enp = max(e64, rel), max(enp, relnp)
        else:
            assert rel <= 2e-6, (len(w), rms_db, rel)
    report(name, rel_vs_float64=e64, rel_vs_numpy=enp)


@pytest.mark.gpu
def test_wave_gain_lengths_and_batches(rt):
    """Lengths at the 8192-sample chunk edges up to 30 s; a batch whose max_samples is far above most rows; B = 1 and
    B = 300; and the empty row."""
    lengths = [0, 1, 8191, 8192, 8193, 3 * KSUM, 480000]
    waves = [make_audio("speech" if i % 2 else "noise", 80 + i, n, 10.0 ** (i % 3 - 1.5)) for i, n in enumerate(lengths)]
    gains, status = run_gain(rt, waves)
    _check_gains("wave_gain chunk edges", waves, gains, status)
    far, fst = run_gain(rt, waves[1:6], max_samples=480000, lead=9, seed=7)
    assert np.array_equal(bits(far), bits(gains[1:6])) and (fst == 0).all()
    one, ost = run_gain(rt, [waves[4]])
    assert np.array_equal(bits(one), bits(gains[4:5]))
    rng = np.random.default_rng(300)
    many = [make_audio("speech" if i % 3 else "noise", 100 + i, int(rng.integers(0, 20000)), 10.0 ** rng.uniform(-2.5, 0.5))
            for i in range(300)]
    many[:3] = [np.zeros(0, np.float32), np.zeros(7, np.float32), make_audio("noise", 99, KSUM)]
    g300, s300 = run_gain(rt, many)
    _check_gains("wave_gain B = 300", many, g300, s300)
    assert g300[1] == np.float32(0.1)                     # all-zero row: mean square 0 -> 1, gain 10^(-20/20)


def _gain_chain32(x, target_db):
    """The kernel's required gain in dB, g = fl32(target_db - 10 * fl32(log10(ms))) with one rounding (a fused
    multiply-add), ms = fl32(sum of fl32(x^2) in double / n); exact for samples whose squares sum exactly in double."""
    x = np.asarray(x, np.float32)
    s = float(np.sum((x * x).astype(np.float64)))
    ms = np.float32(s / len(x)) if len(x) else np.float32(0)
    if ms == 0:
        ms = np.float32(1)
    L = float(np.float32(np.log10(np.float64(ms))))
    return np.float32(float(np.float32(target_db)) - 10.0 * L)       # exact in double: 10 L has at most 28 bits


def _pow_gain(g_db):
    return np.float32(10.0 ** float(np.float32(np.float32(g_db) / np.float32(20))))


@pytest.mark.gpu
def test_wave_gain_status_boundary(rt):
    """max_gain_db exactly at the kernel's float32 required gain passes (status 0, gain fl32(10^(g/20))); one float32 ulp
    below it sets MASR_STATUS_GAIN_EXCEEDED and clamps the gain, where the reference raises ValueError.  Samples on a
    1/1024 grid square and sum exactly, so the host restates the kernel's float32 chain bit for bit.  (numpy's own g can
    differ from it by a few float32 ulps: its float32 log10 is not always correctly rounded.)"""
    rng = np.random.default_rng(11)
    for i, target in enumerate((-20.0, 0.0, -45.0)):
        x = (rng.integers(-40, 41, 3000 + 777 * i) / 1024).astype(np.float32)
        g = _gain_chain32(x, target)
        gain, status = run_gain(rt, [x], target, float(g))
        assert status.tolist() == [0] and bits(gain[0]) == bits(_pow_gain(g)), (target, g)
        below = np.nextafter(g, np.float32(-np.inf))
        gain, status = run_gain(rt, [x], target, float(below))
        assert status.tolist() == [STATUS_GAIN_EXCEEDED] and bits(gain[0]) == bits(_pow_gain(below)), (target, g)


@pytest.mark.gpu
def test_wave_gain_mixed_status_batch(rt):
    """Rows that need more than max_gain_db and rows that do not, in one batch, at target_db -20, 0 and -45."""
    base = make_audio("speech", 5, 12000)
    rms = 10 * np.log10(np.mean(base.astype(np.float64) ** 2))
    waves = [(base * np.float32(10 ** ((lvl - rms) / 20))).astype(np.float32) for lvl in (-5, -25, -45, -65)]
    max_gain_db = 10.0
    for target in (-20.0, 0.0, -45.0):
        need = [20 * np.log10(gain64(w, target)) for w in waves]
        assert all(abs(n - max_gain_db) > 0.01 for n in need)
        want_status = [int(n > max_gain_db) for n in need]
        assert 0 < sum(want_status) < len(waves)
        gain, status = run_gain(rt, waves, target, max_gain_db)
        assert status.tolist() == want_status, target
        for g, n, s in zip(gain, need, want_status):
            if s:
                assert bits(g) == bits(_pow_gain(max_gain_db))
            else:
                assert abs(g / 10 ** (n / 20) - 1) <= 1e-6


@pytest.mark.gpu
def test_wave_gain_workspace_and_empty_rows(rt):
    """The workspace is exactly masr_fbank_workspace_bytes bytes (the guard behind it is checked on every call); with
    max_samples = 0 it is one chunk per row, and empty rows get the gain of mean square 1."""
    for B, ms, want in [(0, 0, 0), (3, 0, 24), (1, KSUM, 8), (1, KSUM + 1, 16), (300, 480000, 300 * 59 * 8)]:
        nbytes = ctypes.c_int64(-1)
        rt.call("masr_fbank_workspace_bytes", B, ms, ctypes.byref(nbytes))
        assert nbytes.value == want, (B, ms)
    for target in (-20.0, 0.0, -45.0):
        gain, status = run_gain(rt, [np.zeros(0, np.float32)] * 3, target, max_samples=0)
        assert (status == 0).all() and (bits(gain) == bits(_pow_gain(target))).all()
    gain, status = run_gain(rt, [])
    assert gain.shape == (0,) and status.shape == (0,)


@pytest.mark.gpu
def test_wave_gain_independent_of_position_neighbours_and_launch(rt):
    """An utterance's gain is bit-identical at another batch position, beside other neighbours, with another max_samples
    and on a second launch."""
    u = make_audio("speech", 12, 30000, 0.3)
    a = [u, make_audio("noise", 13, 9000), make_audio("speech", 14, 100)]
    first, _ = run_gain(rt, a)
    again, _ = run_gain(rt, a)
    assert np.array_equal(bits(first), bits(again))
    moved, _ = run_gain(rt, [make_audio("noise", 15, 70000, 5.0), np.zeros(0, np.float32), u], max_samples=480000, lead=2)
    assert bits(moved[2]) == bits(first[0])


# ---- GPU: the engine without dB normalisation ------------------------------------------------------------------------------

@pytest.mark.gpu
def test_engine_fbank_without_db_normalization(gpu_engines):
    """ConformerEngine.fbank(use_db_normalization=False), the preprocess_conf.use_dB_normalization: False path: no gain
    launch (last_gain None) and the features of the unscaled samples, loud (clipping) and quiet."""
    eng = gpu_engines()
    waves = [make_audio("speech", 31, 16333, 30.0), make_audio("speech", 32, 8000), make_audio("speech", 33, 24001, 0.001),
             make_audio("noise", 34, 401, 0.05), make_audio("speech", 35, 11111, 0.2)]
    eng.fbank(waves[:2])
    assert eng.last_gain is not None
    feats, frames, status = eng.fbank(waves, use_db_normalization=False)
    assert eng.last_gain is None
    assert frames == [ob.num_frames(len(w)) for w in waves] and status.cpu().tolist() == [0] * len(waves)
    f = feats.cpu().numpy()
    bar = Bar()
    for b, w in enumerate(waves):
        bar.add(f[b], quantize(w), what=f"row {b}")
        assert (f[b, frames[b]:] == 0).all()
    bar.report("engine fbank, no dB normalisation", natural=True)
