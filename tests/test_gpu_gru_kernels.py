"""GPU (-m gpu): the GRU recurrence kernels of DeepSpeech2 with ``use_gru: True`` (``masr_gru_seq_f32``, ``masr_gru_step_f32``)
against float64 ``torch.nn.GRU`` over ``pack_padded_sequence`` (masr/model_utils/deepspeech2/encoder.py:41-43, gru.py:6-22).

As in test_gpu_family_kernels.py, every input row past a valid length holds large finite garbage and every output buffer
starts as NaN.  Observed maximum errors are given per test (H100 80GB HBM3); the tolerances are about 4x those."""
import ctypes
import math

import pytest
import torch
import torch.nn.functional as F

from kernel_contract import P, assert_pair_reconstructs, err, garbage, nan, report, runtime, same
from test_gpu_family_kernels import from_T, to_T

pytestmark = pytest.mark.gpu

GRU_IN = 16


@pytest.fixture(scope="module")
def rt():
    return runtime()


def _gru_problem(H, B, T, seed):
    """Seeded inputs of one bidirectional GRU layer with non-zero b_hh.  x, W_ih, b_ih and b_hh live on coarse dyadic grids,
    so the float64 W_ih x + b_ih + [b_hr, b_hz, 0] is exactly the float32 gates_x the kernels read."""
    g = torch.Generator().manual_seed(seed)
    if B == 1:
        lens = [T]
    else:
        lens = torch.randint(0, T + 1, (B,), generator=g).tolist()
        lens[:4] = [T, 0, 1, T - 1]
    x = torch.randint(-16, 17, (B, T, GRU_IN), generator=g).double() / 8
    w_ih = torch.randint(-32, 33, (2, 3 * H, GRU_IN), generator=g).double() / 64
    b_ih = torch.randint(-256, 257, (2, 3 * H), generator=g).double() / 512
    b_hh = torch.randint(-256, 257, (2, 3 * H), generator=g).double() / 512
    w_hh = torch.randn(2, 3 * H, H, generator=g) / math.sqrt(H)
    h0 = torch.randn(2, B, H, generator=g) * 0.5
    fold = torch.cat([b_hh[:, :2 * H], torch.zeros(2, H, dtype=torch.float64)], 1)
    gx = torch.stack([F.linear(x, w_ih[d], b_ih[d] + fold[d]) for d in range(2)])      # [2, B, T, 3H] float64
    assert torch.equal(gx.float().double(), gx)
    return dict(H=H, B=B, T=T, lens=lens, x=x, w_ih=w_ih, b_ih=b_ih, b_hh=b_hh, w_hh=w_hh, h0=h0, gx=gx.float(),
                bhn=b_hh[:, 2 * H:].float())


def _gru_reference(pb):
    """torch.nn.GRU(bidirectional, float64) over pack_padded_sequence -> out [B, T, 2H], h_n [2, B, H] (the state after each
    utterance's last valid step; utterances of length 0 keep h0)."""
    H, B, T, lens = pb["H"], pb["B"], pb["T"], pb["lens"]
    gru = torch.nn.GRU(GRU_IN, H, batch_first=True, bidirectional=True, dtype=torch.float64)
    with torch.no_grad():
        for d, sfx in enumerate(("", "_reverse")):
            getattr(gru, "weight_ih_l0" + sfx).copy_(pb["w_ih"][d])
            getattr(gru, "weight_hh_l0" + sfx).copy_(pb["w_hh"][d].double())
            getattr(gru, "bias_ih_l0" + sfx).copy_(pb["b_ih"][d])
            getattr(gru, "bias_hh_l0" + sfx).copy_(pb["b_hh"][d])
    out = torch.zeros(B, T, 2 * H, dtype=torch.float64)
    hn = pb["h0"].double().clone()
    idx = [i for i in range(B) if lens[i] > 0]
    if idx:
        it = torch.tensor(idx)
        packed = torch.nn.utils.rnn.pack_padded_sequence(pb["x"][it], torch.tensor([lens[i] for i in idx]), batch_first=True,
                                                         enforce_sorted=False)
        with torch.no_grad():
            o, h = gru(packed, pb["h0"][:, it].double())
        out[it] = torch.nn.utils.rnn.pad_packed_sequence(o, batch_first=True, total_length=T)[0]
        hn[:, it] = h
    return out, hn


class _GruRun:
    """Device buffers of one bidirectional layer: gates_x per direction [B*bstride, 3H] (garbage past every length), one
    [B*bstride, 2H] output with the forward direction at col_off 0 and the reverse one at col_off H, as fp32 and as pair."""

    def __init__(self, rt, pb):
        H, B, T = pb["H"], pb["B"], pb["T"]
        self.rt, self.pb, self.bstride = rt, pb, T + 2
        bs = self.bstride
        self.gx = []
        for d in range(2):
            buf = garbage((B, bs, 3 * H), 20 + d)
            for i, n in enumerate(pb["lens"]):
                buf[i, :n] = pb["gx"][d, i, :n]
            self.gx.append(buf.view(B * bs, 3 * H).to(rt.dev))
        self.whh = [pb["w_hh"][d].to(rt.dev) for d in range(2)]
        self.bhn = [pb["bhn"][d].to(rt.dev) for d in range(2)]
        self.lens = torch.tensor(pb["lens"], dtype=torch.int32, device=rt.dev)
        self.out = nan((B * bs, 2 * H), rt.dev)
        self.oh, self.ol = nan((B * bs, 2 * H), rt.dev, torch.float16), nan((B * bs, 2 * H), rt.dev, torch.float16)

    def seq(self, d, h0T, hNT, fp32_out=True):
        pb, rt = self.pb, self.rt
        nbytes = ctypes.c_int64()
        rt.call("masr_lstm_seq_workspace_bytes", pb["B"], pb["H"], ctypes.byref(nbytes))
        ws = torch.empty(nbytes.value, dtype=torch.uint8, device=rt.dev)
        rt.call("masr_gru_seq_f32", P(self.gx[d]), 3 * pb["H"], self.bstride, P(self.whh[d]), P(h0T), P(hNT), P(self.bhn[d]),
                P(self.out) if fp32_out else None, P(self.oh), P(self.ol), 2 * pb["H"], d * pb["H"], P(self.lens), pb["B"],
                pb["H"], max(pb["lens"]), d, P(ws), nbytes.value, rt.st())

    def step(self, d, h0T):
        """T launches of the per-step kernel with ping-pong state buffers; returns the final state buffer."""
        pb, rt = self.pb, self.rt
        bufs = [h0T.clone(), torch.full_like(h0T, float("nan"))]
        T = max(pb["lens"])
        for s in range(T):
            rt.call("masr_gru_step_f32", P(self.gx[d]), 3 * pb["H"], self.bstride, P(self.whh[d]), P(bufs[s % 2]),
                    P(bufs[1 - s % 2]), P(self.bhn[d]), P(self.out), P(self.oh), P(self.ol), 2 * pb["H"], d * pb["H"],
                    P(self.lens), pb["B"], pb["H"], s, d, rt.st())
        return bufs[T % 2]

    def check_rows(self, ref_out):
        """Valid rows against the reference (fp32 and pair); every row past a length is left untouched."""
        pb, bs = self.pb, self.bstride
        H = pb["H"]
        torch.cuda.synchronize()
        out, oh, ol = (t.cpu().view(pb["B"], bs, 2 * H) for t in (self.out, self.oh, self.ol))
        e = 0.0
        for i, n in enumerate(pb["lens"]):
            e = max(e, err(out[i, :n], ref_out[i, :n]))
            assert_pair_reconstructs(oh[i, :n], ol[i, :n], out[i, :n])
            assert torch.isnan(out[i, n:]).all() and torch.isnan(oh[i, n:].float()).all() and torch.isnan(ol[i, n:].float()).all()
        return e


@pytest.mark.parametrize("H,B,T", [(128, 1, 37), (128, 64, 48), (512, 33, 40), (1024, 1, 30), (1024, 33, 100), (1024, 64, 50)])
def test_gru_seq_and_step(rt, H, B, T):
    """masr_gru_seq_f32 and masr_gru_step_f32, both directions into one [M, 2H] output, non-zero h0 and b_hh (b_hn inside
    the product with r), ragged lengths (0, 1, T-1, T), 33 utterances = two 32-lane chunks with padding lanes.  Final h per
    utterance = the state after its last valid step.  Observed max error (H100 80GB HBM3, 400 W): seq out 1.6e-6, h 1.3e-6;
    step out 2.2e-6, h 1.8e-6; seq vs step 3.1e-6 (H = 1024, B = 64); tolerance 8e-6 / 1e-5."""
    pb = _gru_problem(H, B, T, seed=H + B + 1)
    ref_out, ref_h = _gru_reference(pb)
    results = {}
    for impl in ("seq", "step"):
        run = _GruRun(rt, pb)
        eh = 0.0
        finals = []
        for d in range(2):
            h0T = to_T(pb["h0"][d], 30 + d).to(rt.dev)
            if impl == "seq":
                hNT = nan(h0T.shape, rt.dev)
                run.seq(d, h0T, hNT)
            else:
                hNT = run.step(d, h0T)
            torch.cuda.synchronize()
            hN = from_T(hNT, B)
            for i, n in enumerate(pb["lens"]):
                if n == 0:      # never active: state untouched
                    assert torch.equal(hN[i], pb["h0"][d, i])
            eh = max(eh, err(hN, ref_h[d]))
            finals.append(hN)
        eo = run.check_rows(ref_out)
        results[impl] = (run.out.cpu(), finals, (eo, eh))
        report(f"gru {impl} H={H} B={B} T={T}", out=eo, h=eh)
    (so, sf, _), (to, tf, _) = results["seq"], results["step"]
    valid = ~torch.isnan(so)
    assert torch.equal(valid, ~torch.isnan(to))
    diff = max((so[valid] - to[valid]).abs().max().item(), max((a - b).abs().max().item() for a, b in zip(sf, tf)))
    report(f"gru seq vs step H={H} B={B}", diff=diff)
    for impl, (_, _, (eo, eh)) in results.items():
        assert eo < 8e-6 and eh < 8e-6, (impl, eo, eh)
    assert diff < 1e-5


def test_gru_seq_zero_steps_and_aliasing(rt):
    """T = 0 copies h0 to hN and leaves the output untouched; hN_T == h0_T gives bit for bit the non-aliased result;
    pair-only output (out = NULL) reconstructs the fp32 one."""
    H, B, T = 256, 5, 30
    pb = _gru_problem(H, B, T, seed=8)
    run = _GruRun(rt, pb)
    h0T = to_T(pb["h0"][0], 40).to(rt.dev)
    run0 = _GruRun(rt, dict(pb, lens=[0] * B))
    hNT = nan(h0T.shape, rt.dev)
    run0.seq(0, h0T, hNT)
    torch.cuda.synchronize()
    assert torch.equal(hNT, h0T)
    assert torch.isnan(run0.out).all() and torch.isnan(run0.oh.float()).all()
    hNT = nan(h0T.shape, rt.dev)
    run.seq(0, h0T, hNT)
    run_a = _GruRun(rt, pb)
    hA = h0T.clone()
    run_a.seq(0, hA, hA, fp32_out=False)
    torch.cuda.synchronize()
    assert torch.equal(hA, hNT)
    assert same(run_a.oh, run.oh) and same(run_a.ol, run.ol) and torch.isnan(run_a.out).all()
    v = ~torch.isnan(run.out)
    assert_pair_reconstructs(run.oh[v], run.ol[v], run.out[v])


def test_gru_rejects_bad_arguments(rt):
    """Host-side MASR_REQUIRE before any launch: H % 128 != 0, H > 1024, a short workspace and null pointers (b_hn, the
    workspace) for the persistent kernel; the same in/out state buffer, H % 4 != 0 and a null b_hn for the per-step one."""
    from masr_b200._lib import MasrB200Error
    B, Hmax, T = 3, 1152, 4
    gx = torch.zeros(B * T, 3 * Hmax, device=rt.dev); whh = torch.zeros(3 * Hmax, Hmax, device=rt.dev)
    hA = torch.zeros(1, Hmax, 32, device=rt.dev); hB = torch.zeros_like(hA); bhn = torch.zeros(Hmax, device=rt.dev)
    out = torch.zeros(B * T, 2 * Hmax, device=rt.dev); lens = torch.full((B,), T, dtype=torch.int32, device=rt.dev)
    need = ctypes.c_int64()
    rt.call("masr_lstm_seq_workspace_bytes", B, Hmax, ctypes.byref(need))
    ws = torch.zeros(need.value, dtype=torch.uint8, device=rt.dev)

    def seq(H, nbytes, b=bhn, w=ws):
        rt.call("masr_gru_seq_f32", P(gx), 3 * H, T, P(whh), P(hA), P(hB), P(b), P(out), None, None, 2 * H, 0, P(lens), B, H, T,
                0, P(w), nbytes, rt.st())

    def step(H, h_out, b=bhn):
        rt.call("masr_gru_step_f32", P(gx), 3 * H, T, P(whh), P(hA), P(h_out), P(b), P(out), None, None, 2 * H, 0, P(lens), B,
                H, 0, 0, rt.st())

    for H in (192, 1152):
        with pytest.raises(MasrB200Error, match="masr_gru_seq_f32: H="):
            seq(H, need.value)
    n256 = ctypes.c_int64()
    rt.call("masr_lstm_seq_workspace_bytes", B, 256, ctypes.byref(n256))
    with pytest.raises(MasrB200Error, match="workspace"):
        seq(256, n256.value - 1)
    for kw in ({"b": None}, {"w": None}):
        with pytest.raises(MasrB200Error, match="null pointer"):
            seq(256, n256.value, **kw)
    with pytest.raises(MasrB200Error, match="distinct"):
        step(256, hA)
    with pytest.raises(MasrB200Error, match="distinct"):
        step(130, hB)
    with pytest.raises(MasrB200Error, match="null pointer"):
        step(256, hB, b=None)
    torch.cuda.synchronize()
    assert torch.all(hB == 0) and torch.all(out == 0)       # nothing ran
