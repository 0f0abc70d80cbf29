"""GPU (-m gpu): the kernels of the DeepSpeech2, EfficientConformer and Squeezeformer families, one C-ABI entry point at a
time, against float64 CPU references written from the reference modules:

  LSTM                 masr/model_utils/deepspeech2/encoder.py:36-45  (torch.nn.LSTM over pack_padded_sequence)
  grouped attention    masr/model_utils/efficient_conformer/attention.py:35-69,120-182  (pad4group view + softmax)
  strided dwconv/pool  masr/model_utils/efficient_conformer/convolution.py:40-48, encoder.py:173-175,520-523
  relpos attention     masr/model_utils/conformer/attention.py:107-118,230-251  (the stream pools' K|V cache layout)
  dwconv + BN + SiLU   masr/model_utils/squeezeformer/convolution.py:136-142
  time reduce/recover  masr/model_utils/squeezeformer/time_reduction.py:53-76,174-197, encoder.py:198-204
  post-norm + ada      masr/model_utils/squeezeformer/encoder.py:412-463, positionwise.py:57-58

Every input row past a valid length holds large finite garbage (not zeros: a kernel that reads past a length must not see the
same zeros the reference pads with) and every output buffer starts as NaN, so both out-of-range reads and writes outside a
kernel's stated contract fail.  Each test's docstring gives the maximum error observed on an H100 80GB HBM3 (400 W power
limit); the tolerances are at most about 4x that.
"""
import ctypes
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from kernel_contract import P, assert_pair_reconstructs, err, garbage, nan, pair_value, relpos_reference, report, runtime, same

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def rt():
    return runtime()


def ceil2(n):
    return (n + 1) // 2


# ---- DeepSpeech2: LSTM ---------------------------------------------------------------------------------------------------

LSTM_IN = 16


def _lstm_problem(H, B, T, seed):
    """Seeded inputs of one bidirectional layer.  x and W_ih live on coarse dyadic grids, so the float64 input projection
    W_ih x + b is exactly the float32 gates_x the kernels read: the reference sees bit-for-bit the kernels' inputs."""
    g = torch.Generator().manual_seed(seed)
    if B == 1:
        lens = [T]
    else:
        lens = torch.randint(0, T + 1, (B,), generator=g).tolist()
        lens[:4] = [T, 0, 1, T - 1]
    x = torch.randint(-16, 17, (B, T, LSTM_IN), generator=g).double() / 8
    w_ih = torch.randint(-32, 33, (2, 4 * H, LSTM_IN), generator=g).double() / 64
    b = torch.randint(-256, 257, (2, 4 * H), generator=g).double() / 512
    w_hh = torch.randn(2, 4 * H, H, generator=g) / math.sqrt(H)
    h0 = torch.randn(2, B, H, generator=g) * 0.5
    c0 = torch.randn(2, B, H, generator=g) * 0.5
    gx = torch.stack([F.linear(x, w_ih[d], b[d]) for d in range(2)])          # [2, B, T, 4H] float64
    assert torch.equal(gx.float().double(), gx)
    return dict(H=H, B=B, T=T, lens=lens, x=x, w_ih=w_ih, b=b, w_hh=w_hh, h0=h0, c0=c0, gx=gx.float())


def _lstm_reference(pb):
    """torch.nn.LSTM(bidirectional, float64) over pack_padded_sequence: the reference DeepSpeech2 layer
    (deepspeech2/encoder.py:36-45).  Returns out [B, T, 2H], h_n / c_n [2, B, H] (the state after each utterance's last
    valid step; utterances of length 0 keep h0 / c0)."""
    H, B, T, lens = pb["H"], pb["B"], pb["T"], pb["lens"]
    lstm = torch.nn.LSTM(LSTM_IN, H, batch_first=True, bidirectional=True, dtype=torch.float64)
    with torch.no_grad():
        for d, sfx in enumerate(("", "_reverse")):
            getattr(lstm, "weight_ih_l0" + sfx).copy_(pb["w_ih"][d])
            getattr(lstm, "weight_hh_l0" + sfx).copy_(pb["w_hh"][d].double())
            getattr(lstm, "bias_ih_l0" + sfx).copy_(pb["b"][d])
            getattr(lstm, "bias_hh_l0" + sfx).zero_()
    out = torch.zeros(B, T, 2 * H, dtype=torch.float64)
    hn, cn = pb["h0"].double().clone(), pb["c0"].double().clone()
    idx = [i for i in range(B) if lens[i] > 0]
    if idx:
        it = torch.tensor(idx)
        packed = torch.nn.utils.rnn.pack_padded_sequence(pb["x"][it], torch.tensor([lens[i] for i in idx]), batch_first=True,
                                                         enforce_sorted=False)
        with torch.no_grad():
            o, (h, c) = lstm(packed, (pb["h0"][:, it].double(), pb["c0"][:, it].double()))
        out[it] = torch.nn.utils.rnn.pad_packed_sequence(o, batch_first=True, total_length=T)[0]
        hn[:, it], cn[:, it] = h, c
    return out, hn, cn


def to_T(h, seed):
    """[B, H] -> the kernels' transposed, 32-lane batch-chunked state [ceil(B/32)][H][32]; padding lanes hold garbage."""
    B, H = h.shape
    nb = (B + 31) // 32
    full = garbage((nb * 32, H), seed)
    full[:B] = h
    return full.view(nb, 32, H).transpose(1, 2).contiguous()


def from_T(hT, B):
    H = hT.shape[1]
    return hT.cpu().transpose(1, 2).reshape(-1, H)[:B]


class _LstmRun:
    """Device buffers of one bidirectional layer: gates_x per direction [B*bstride, 4H] (garbage past every length), one
    [B*bstride, 2H] output with the forward direction at col_off 0 and the reverse one at col_off H, as fp32 and as pair."""

    def __init__(self, rt, pb):
        H, B, T = pb["H"], pb["B"], pb["T"]
        self.rt, self.pb, self.bstride = rt, pb, T + 2
        bs = self.bstride
        self.gx = []
        for d in range(2):
            buf = garbage((B, bs, 4 * H), 20 + d)
            for i, n in enumerate(pb["lens"]):
                buf[i, :n] = pb["gx"][d, i, :n]
            self.gx.append(buf.view(B * bs, 4 * H).to(rt.dev))
        self.whh = [pb["w_hh"][d].to(rt.dev) for d in range(2)]
        self.lens = torch.tensor(pb["lens"], dtype=torch.int32, device=rt.dev)
        self.out = nan((B * bs, 2 * H), rt.dev)
        self.oh, self.ol = nan((B * bs, 2 * H), rt.dev, torch.float16), nan((B * bs, 2 * H), rt.dev, torch.float16)

    def seq(self, d, h0T, hNT, c, fp32_out=True):
        pb, rt = self.pb, self.rt
        nbytes = ctypes.c_int64()
        rt.call("masr_lstm_seq_workspace_bytes", pb["B"], pb["H"], ctypes.byref(nbytes))
        ws = torch.empty(nbytes.value, dtype=torch.uint8, device=rt.dev)
        rt.call("masr_lstm_seq_f32", P(self.gx[d]), 4 * pb["H"], self.bstride, P(self.whh[d]), P(h0T), P(hNT), P(c),
                P(self.out) if fp32_out else None, P(self.oh), P(self.ol), 2 * pb["H"], d * pb["H"], P(self.lens), pb["B"],
                pb["H"], max(pb["lens"]), d, P(ws), nbytes.value, rt.st())

    def step(self, d, h0T, c):
        """T launches of the per-step kernel with ping-pong state buffers; returns the final state buffer."""
        pb, rt = self.pb, self.rt
        bufs = [h0T.clone(), torch.full_like(h0T, float("nan"))]
        T = max(pb["lens"])
        for s in range(T):
            rt.call("masr_lstm_step_f32", P(self.gx[d]), 4 * pb["H"], self.bstride, P(self.whh[d]), P(bufs[s % 2]),
                    P(bufs[1 - s % 2]), P(c), P(self.out), P(self.oh), P(self.ol), 2 * pb["H"], d * pb["H"], P(self.lens),
                    pb["B"], pb["H"], s, d, rt.st())
        return bufs[T % 2]

    def check_rows(self, ref_out):
        """Valid rows against the reference (fp32 and pair); every row past a length is left untouched."""
        pb, bs = self.pb, self.bstride
        H = pb["H"]
        torch.cuda.synchronize()
        out, oh, ol = self.out.cpu().view(pb["B"], bs, 2 * H), self.oh.cpu().view(pb["B"], bs, 2 * H), self.ol.cpu().view(pb["B"], bs, 2 * H)
        e = 0.0
        for i, n in enumerate(pb["lens"]):
            e = max(e, err(out[i, :n], ref_out[i, :n]))
            assert_pair_reconstructs(oh[i, :n], ol[i, :n], out[i, :n])
            assert torch.isnan(out[i, n:]).all() and torch.isnan(oh[i, n:].float()).all() and torch.isnan(ol[i, n:].float()).all()
        return e


@pytest.mark.parametrize("H,B,T", [(128, 1, 37), (128, 64, 48), (512, 5, 64), (512, 33, 40), (1024, 33, 100)])
def test_lstm_seq_and_step(rt, H, B, T):
    """masr_lstm_seq_f32 and masr_lstm_step_f32, both directions into one [M, 2H] output, non-zero h0/c0, ragged lengths
    (0, 1, T-1, T), 33 utterances = two 32-lane chunks with padding lanes.  Final h / c per utterance = the state after its
    last valid step.  Observed max error (H100): out 1.1e-6, h 5.6e-7, c 8.8e-7, seq vs step 1.2e-6; tolerance 4e-6."""
    pb = _lstm_problem(H, B, T, seed=H + B)
    ref_out, ref_h, ref_c = _lstm_reference(pb)
    results = {}
    for impl in ("seq", "step"):
        run = _LstmRun(rt, pb)
        eh = ec = 0.0
        finals = []
        for d in range(2):
            h0T = to_T(pb["h0"][d], 30 + d).to(rt.dev)
            c = pb["c0"][d].clone().to(rt.dev)
            if impl == "seq":
                hNT = nan(h0T.shape, rt.dev)
                run.seq(d, h0T, hNT, c)
            else:
                hNT = run.step(d, h0T, c)
            torch.cuda.synchronize()
            hN, cN = from_T(hNT, B), c.cpu()
            for i, n in enumerate(pb["lens"]):
                if n == 0:      # never active: state and output untouched
                    assert torch.equal(hN[i], pb["h0"][d, i]) and torch.equal(cN[i], pb["c0"][d, i])
            eh, ec = max(eh, err(hN, ref_h[d])), max(ec, err(cN, ref_c[d]))
            finals.append((hN, cN))
        eo = run.check_rows(ref_out)
        results[impl] = (run.out.cpu(), finals, (eo, eh, ec))
        report(f"lstm {impl} H={H} B={B} T={T}", out=eo, h=eh, c=ec)
    (so, sf, _), (to, tf, _) = results["seq"], results["step"]
    valid = ~torch.isnan(so)
    assert torch.equal(valid, ~torch.isnan(to))
    diff = max((so[valid] - to[valid]).abs().max().item(),
               max((a - b).abs().max().item() for (ha, ca), (hb, cb) in zip(sf, tf) for a, b in ((ha, hb), (ca, cb))))
    report(f"lstm seq vs step H={H} B={B}", diff=diff)
    for impl, (_, _, (eo, eh, ec)) in results.items():
        assert eo < 4e-6 and eh < 4e-6 and ec < 4e-6, (impl, eo, eh, ec)
    assert diff < 4e-6


def test_lstm_seq_zero_steps_and_aliasing(rt):
    """T = 0 copies h0 to hN and leaves c and the output untouched; hN_T == h0_T (allowed by the header) gives bit for bit
    the non-aliased result; pair-only output (out = NULL) reconstructs the fp32 one."""
    H, B, T = 256, 5, 30
    pb = _lstm_problem(H, B, T, seed=7)
    run = _LstmRun(rt, pb)
    h0T = to_T(pb["h0"][0], 40).to(rt.dev)
    # T = 0: every utterance empty
    empty = dict(pb, lens=[0] * B)
    run0 = _LstmRun(rt, empty)
    hNT, c = nan(h0T.shape, rt.dev), pb["c0"][0].clone().to(rt.dev)
    run0.seq(0, h0T, hNT, c)
    torch.cuda.synchronize()
    assert torch.equal(hNT, h0T) and torch.equal(c.cpu(), pb["c0"][0])
    assert torch.isnan(run0.out).all() and torch.isnan(run0.oh.float()).all()
    # separate and aliased state buffers
    hNT, c1 = nan(h0T.shape, rt.dev), pb["c0"][0].clone().to(rt.dev)
    run.seq(0, h0T, hNT, c1)
    run_a = _LstmRun(rt, pb)
    hA, c2 = h0T.clone(), pb["c0"][0].clone().to(rt.dev)
    run_a.seq(0, hA, hA, c2, fp32_out=False)
    torch.cuda.synchronize()
    assert torch.equal(hA, hNT) and torch.equal(c1, c2)
    assert same(run_a.oh, run.oh) and same(run_a.ol, run.ol) and torch.isnan(run_a.out).all()
    assert_pair_reconstructs(run.oh[~torch.isnan(run.out)], run.ol[~torch.isnan(run.out)], run.out[~torch.isnan(run.out)])


def test_lstm_rejects_bad_arguments(rt):
    """Host-side MASR_REQUIRE before any launch: H % 128 != 0, H > 1024 and a short workspace for the persistent kernel,
    the same in/out state buffer for the per-step kernel."""
    from masr_b200._lib import MasrB200Error
    B, Hmax, T = 3, 1152, 4
    gx = torch.zeros(B * T, 4 * Hmax, device=rt.dev); whh = torch.zeros(4 * Hmax, Hmax, device=rt.dev)
    hA = torch.zeros(1, Hmax, 32, device=rt.dev); hB = torch.zeros_like(hA); c = torch.zeros(B, Hmax, device=rt.dev)
    out = torch.zeros(B * T, 2 * Hmax, device=rt.dev); lens = torch.full((B,), T, dtype=torch.int32, device=rt.dev)
    need = ctypes.c_int64()
    rt.call("masr_lstm_seq_workspace_bytes", B, Hmax, ctypes.byref(need))
    ws = torch.zeros(need.value, dtype=torch.uint8, device=rt.dev)

    def seq(H, nbytes):
        rt.call("masr_lstm_seq_f32", P(gx), 4 * H, T, P(whh), P(hA), P(hB), P(c), P(out), None, None, 2 * H, 0, P(lens), B, H, T,
                0, P(ws), nbytes, rt.st())

    for H in (192, 1152):
        with pytest.raises(MasrB200Error):
            seq(H, need.value)
    n256 = ctypes.c_int64()
    rt.call("masr_lstm_seq_workspace_bytes", B, 256, ctypes.byref(n256))
    with pytest.raises(MasrB200Error):
        seq(256, n256.value - 1)
    with pytest.raises(MasrB200Error):
        rt.call("masr_lstm_step_f32", P(gx), 1024, T, P(whh), P(hA), P(hA), P(c), P(out), None, None, 512, 0, P(lens), B, 256,
                0, 0, rt.st())
    torch.cuda.synchronize()
    assert torch.all(hB == 0) and torch.all(out == 0)       # nothing ran


# ---- EfficientConformer: grouped attention -------------------------------------------------------------------------------

def grouped_reference(q, k, v, p, pos_u, pos_v, heads=4, group=3):
    """GroupedRelPositionMultiHeadedAttention core in float64 (efficient_conformer/attention.py:35-69,120-182): queries
    [Tq, d] and keys / values / pos rows [Tk, d] are each zero-padded to a multiple of `group` from their own first frame
    (pad4group) and the memory of `group` consecutive frames is viewed as `heads` heads of width group*d_k; scores scaled by
    1/sqrt(group*d_k), no rel_shift; the padded query frames are dropped."""
    d = q.shape[1]
    dg = d // heads * group

    def regroup(t):
        t = F.pad(t.double(), (0, 0, 0, (-t.shape[0]) % group))
        return t.reshape(-1, heads, dg).transpose(0, 1)                 # [heads, frames/group, dg]
    qg, kg, vg, pg = regroup(q), regroup(k), regroup(v), regroup(p)
    s = ((qg + pos_u.double()[:, None]) @ kg.transpose(1, 2) + (qg + pos_v.double()[:, None]) @ pg.transpose(1, 2)) / math.sqrt(dg)
    ctx = (torch.softmax(s, -1) @ vg).transpose(0, 1).reshape(-1, d)
    return ctx[:q.shape[0]]


@pytest.mark.parametrize("lens", [[1], [2], [5, 0, 3, 4, 1, 2], [241, 0, 48, 49, 50, 1], [300, 200, 97]])
def test_grouped_attention(rt, lens):
    """masr_grouped_attention_f32, d_model 256, 4 heads, group 3: T % 3 in {0, 1, 2}, T = 1 / 2, an empty utterance, and
    T >= 200 (several 16-group query CTAs and 8-group key tiles).  Q|K|V share one [B*bstride, 3d] buffer (pitch 3d); the P
    table is shared by the batch, so rows past a short utterance's length are real data it must read as zero padding.
    Outputs of frames >= lens[b] are not stored.  Observed max error (H100): 9.3e-7; tolerance 3e-6."""
    g = torch.Generator().manual_seed(sum(lens) + len(lens))
    B, H, dk, G, d = len(lens), 4, 64, 3, 256
    Tm = max(lens)
    bs = Tm + 4
    qkv = garbage((B, bs, 3 * d), 1)
    for i, n in enumerate(lens):
        qkv[i, :n] = torch.randn(n, 3 * d, generator=g)
    ptab = garbage((Tm + 5, d), 2)
    ptab[:Tm] = torch.randn(Tm, d, generator=g)
    pu, pv = torch.randn(H, G * dk, generator=g) * 0.3, torch.randn(H, G * dk, generator=g) * 0.3
    qd, pd, ud, vd = qkv.view(B * bs, 3 * d).to(rt.dev), ptab.to(rt.dev), pu.to(rt.dev), pv.to(rt.dev)
    ld = torch.tensor(lens, dtype=torch.int32, device=rt.dev)
    O = nan((B * bs, 3 * d), rt.dev)
    Oh, Ol = nan((B * bs, 3 * d), rt.dev, torch.float16), nan((B * bs, 3 * d), rt.dev, torch.float16)
    rt.call("masr_grouped_attention_f32", P(qd), qd.data_ptr() + 4 * d, qd.data_ptr() + 8 * d, P(pd), 3 * d, bs, P(ud), P(vd),
            P(O), P(Oh), P(Ol), P(ld), B, H, dk, G, Tm, rt.st())
    torch.cuda.synchronize()
    O, Oh, Ol = O.cpu().view(B, bs, 3 * d), Oh.cpu().view(B, bs, 3 * d), Ol.cpu().view(B, bs, 3 * d)
    e = 0.0
    written = torch.zeros(B, bs, 3 * d, dtype=torch.bool)
    for i, n in enumerate(lens):
        if n == 0:
            continue
        ref = grouped_reference(qkv[i, :n, :d], qkv[i, :n, d:2 * d], qkv[i, :n, 2 * d:], ptab[:n], pu, pv)
        e = max(e, err(O[i, :n, :d], ref))
        assert_pair_reconstructs(Oh[i, :n, :d], Ol[i, :n, :d], O[i, :n, :d])
        written[i, :n, :d] = True
    assert torch.isnan(O[~written]).all() and torch.isnan(Oh[~written].float()).all()
    report(f"grouped attention lens={lens}", out=e)
    assert e < 3e-6


def test_grouped_attention_cache(rt):
    """masr_grouped_attention_cache_f32 in the stream pool's layout: queries [S*C, d] with C = 16 (16 % 3 = 1), K|V
    interleaved with pitch 2d and slot pitch cap, k_lens = cache + chunk with cache % 3 in {0, 1, 2}; P row j = key j.
    Keys are grouped from key 0, queries from the first chunk frame.  A short final chunk and an idle slot (q_len 0) leave
    their other rows untouched.  Observed max error (H100): 5.6e-7; tolerance 2e-6."""
    g = torch.Generator().manual_seed(3)
    S, C, cap, H, dk, G, d = 6, 16, 256, 4, 64, 3, 256
    q_lens = [16, 16, 16, 16, 5, 0]
    cache = [0, 3, 7, 32, 209, 20]
    k_lens = [c + q for c, q in zip(cache, q_lens)]
    Q = garbage((S, C, d), 3)
    KV = garbage((S, cap, 2 * d), 4)
    for s in range(S):
        Q[s, :q_lens[s]] = torch.randn(q_lens[s], d, generator=g)
        KV[s, :k_lens[s]] = torch.randn(k_lens[s], 2 * d, generator=g)
    ptab = garbage((cap + 3, d), 5)
    ptab[:max(k_lens)] = torch.randn(max(k_lens), d, generator=g)
    pu, pv = torch.randn(H, G * dk, generator=g) * 0.3, torch.randn(H, G * dk, generator=g) * 0.3
    qd, kvd, pd = Q.view(S * C, d).to(rt.dev), KV.view(S * cap, 2 * d).to(rt.dev), ptab.to(rt.dev)
    qld, kld = torch.tensor(q_lens, dtype=torch.int32, device=rt.dev), torch.tensor(k_lens, dtype=torch.int32, device=rt.dev)
    O = nan((S * C, d), rt.dev)
    Oh, Ol = nan((S * C, d), rt.dev, torch.float16), nan((S * C, d), rt.dev, torch.float16)
    ud, vd = pu.to(rt.dev), pv.to(rt.dev)
    rt.call("masr_grouped_attention_cache_f32", P(qd), d, C, P(kvd), kvd.data_ptr() + 4 * d, 2 * d, cap, P(pd), P(ud), P(vd), P(O),
            P(Oh), P(Ol), P(qld), P(kld), S, H, dk, G, C, rt.st())
    torch.cuda.synchronize()
    O, Oh, Ol = O.cpu().view(S, C, d), Oh.cpu().view(S, C, d), Ol.cpu().view(S, C, d)
    e = 0.0
    for s in range(S):
        n, kl = q_lens[s], k_lens[s]
        if n:
            ref = grouped_reference(Q[s, :n], KV[s, :kl, :d], KV[s, :kl, d:], ptab[:kl], pu, pv)
            e = max(e, err(O[s, :n], ref))
            assert_pair_reconstructs(Oh[s, :n], Ol[s, :n], O[s, :n])
        assert torch.isnan(O[s, n:]).all() and torch.isnan(Oh[s, n:].float()).all() and torch.isnan(Ol[s, n:].float()).all()
    report("grouped attention cache", out=e)
    assert e < 2e-6


# ---- relative-position attention at the stream pools' shapes -------------------------------------------------------------

@pytest.mark.parametrize("skew", [False, True])
@pytest.mark.parametrize("fn", ["masr_relpos_attention_f32", "masr_relpos_attention_tc", "masr_relpos_attention_tc5"])
def test_relpos_attention_stream_shapes(rt, fn, skew):
    """The stream pools' call (stream_pool.py:207,339,475): q_lens <= 16 < k_lens (16 .. 300, many 32-key tiles); Q in its
    own [S*C, 3d] buffer; K/V as the pool's cache (pitch 2d, slot pitch cap; fp32 for _f32, fp16 pairs for _tc / _tc5).
    skew: scores with a standard deviation near 10 and, for the first queries of each slot, a dominant key in the LAST key
    tile (the online-softmax rescale).  Query rows in [q_len, max_q) are written as zeros.  _tc5 (keys <= 256) runs the
    layout its header allows beyond the engine's q_lens == k_lens == max_q: every key set is longer than max_q, and the
    LAST slot holds the longest one (256 keys), so its K/V rows reach far past (S-1)*cap + max_q.
    Observed max error (H100): f32 1.7e-6 / skewed 9.1e-6, tc 1.1e-6 / skewed 7.7e-6, tc5 9.2e-7 / skewed 4.2e-6;
    tolerance 4e-6 / 2e-5 (the
    skewed scores are ~10x larger, and so is their fp32 rounding)."""
    g = torch.Generator().manual_seed(11 + skew)
    S, C, cap, H, dk, d = 6, 16, 320, 4, 64, 256
    q_lens = [16, 16, 16, 1, 9, 0]
    k_lens = [16, 33, 96, 300, 41, 20]
    if fn == "masr_relpos_attention_tc5":
        q_lens = [16, 16, 1, 9, 0, 16]
        k_lens = [17, 33, 96, 41, 20, 256]
    qs = 7.0 if skew else 1.0
    Q = garbage((S, C, 3 * d), 6)
    KV = garbage((S, cap, 2 * d), 7)
    for s in range(S):
        Q[s, :q_lens[s], :d] = torch.randn(q_lens[s], d, generator=g) * qs
        KV[s, :k_lens[s]] = torch.randn(k_lens[s], 2 * d, generator=g)
        if skew:
            for i in range(min(4, q_lens[s])):
                KV[s, k_lens[s] - 1 - i, :d] = 0.1 * Q[s, i, :d]
    ptab = garbage((cap + 5, d), 8)
    ptab[:max(k_lens)] = torch.randn(max(k_lens), d, generator=g)
    pu, pv = torch.randn(H, dk, generator=g) * 0.3, torch.randn(H, dk, generator=g) * 0.3
    qd, kvd, pd = Q.view(S * C, 3 * d).to(rt.dev), KV.view(S * cap, 2 * d).to(rt.dev), ptab.to(rt.dev)
    ud, vd = pu.to(rt.dev), pv.to(rt.dev)
    qld, kld = torch.tensor(q_lens, dtype=torch.int32, device=rt.dev), torch.tensor(k_lens, dtype=torch.int32, device=rt.dev)
    O = nan((S * C, d), rt.dev)
    Oh, Ol = nan((S * C, d), rt.dev, torch.float16), nan((S * C, d), rt.dev, torch.float16)
    if fn == "masr_relpos_attention_f32":
        rt.call(fn, P(qd), 3 * d, C, P(kvd), kvd.data_ptr() + 4 * d, 2 * d, cap, P(pd), d, P(ud), P(vd), P(O), P(Oh), P(Ol), d, C,
                P(qld), P(kld), S, H, dk, C, rt.st())
    else:
        def split(x):
            h = torch.empty(x.shape, dtype=torch.float16, device=rt.dev); l = torch.empty_like(h)
            rt.call("masr_split_f16", P(x), P(h), P(l), x.numel(), rt.st())
            return h, l
        (kh, kl), (ph, pl) = split(kvd), split(pd)
        if fn == "masr_relpos_attention_tc5":
            rt.call(fn, P(qd), 3 * d, C, P(kh), P(kl), kh.data_ptr() + 2 * d, kl.data_ptr() + 2 * d, 2 * d, cap, P(ph),
                    P(pl), d, ptab.shape[0], P(ud), P(vd), P(O), P(Oh), P(Ol), d, C, P(qld), P(kld), S, H, dk, C, rt.st())
        else:
            rt.call(fn, P(qd), 3 * d, C, P(kh), P(kl), kh.data_ptr() + 2 * d, kl.data_ptr() + 2 * d, 2 * d, cap, P(ph), P(pl), d,
                    P(ud), P(vd), P(O), P(Oh), P(Ol), d, C, P(qld), P(kld), S, H, dk, C, rt.st())
    torch.cuda.synchronize()
    O, Oh, Ol = O.cpu().view(S, C, d), Oh.cpu().view(S, C, d), Ol.cpu().view(S, C, d)
    e = 0.0
    for s in range(S):
        n, kl_ = q_lens[s], k_lens[s]
        if n:
            ref = relpos_reference(Q[s, :n, :d], KV[s, :kl_, :d], KV[s, :kl_, d:], ptab[:kl_], pu, pv, H)
            e = max(e, err(O[s, :n], ref))
            assert_pair_reconstructs(Oh[s, :n], Ol[s, :n], O[s, :n])
        assert torch.all(O[s, n:] == 0) and torch.all(Oh[s, n:] == 0) and torch.all(Ol[s, n:] == 0)
    report(f"{fn} stream skew={skew}", out=e)
    assert e < (2e-5 if skew else 4e-6)


# ---- depthwise convolutions ----------------------------------------------------------------------------------------------

DW_C = 256


def _dw_problem(seed, lens, ks, ldg, extra_rows):
    g = torch.Generator().manual_seed(seed)
    B, Tm = len(lens), max(lens)
    gb = Tm + extra_rows
    x = garbage((B, gb, ldg), seed)
    for i, n in enumerate(lens):
        x[i, :n, :DW_C] = torch.randn(n, DW_C, generator=g)
    w = torch.randn(DW_C, ks, generator=g) / math.sqrt(ks)
    bias = torch.randn(DW_C, generator=g) * 0.1
    pad = torch.randn(DW_C, generator=g)
    return g, x, w, bias, pad, gb


def _dw_conv_reference(xb, n, w, bias, pad, lpad, stride, out_rows, causal):
    """Depthwise Conv1d of one utterance's first n rows (rows >= n are the zeros the contract reads), left context `pad`
    (causal: GLU of the pointwise bias, convolution.py:103) or symmetric zero padding -> [out_rows, C] float64."""
    ks = w.shape[1]
    L = max(stride * out_rows + ks, n)
    xe = torch.zeros(L, DW_C, dtype=torch.float64)
    xe[:n] = xb[:n, :DW_C].double()
    if causal:
        xe = torch.cat([pad.double()[None].expand(lpad, DW_C), xe])
        r = F.conv1d(xe.t()[None], w.double()[:, None], bias.double(), stride=stride, groups=DW_C)
    else:
        r = F.conv1d(xe.t()[None], w.double()[:, None], bias.double(), stride=stride, padding=lpad, groups=DW_C)
    return r[0].t()[:out_rows]


def _call_bn(rt, xd, ldg, gb, w, bias, sc, sh, pad, y, yh, yl, ldy, yb, ld, B, ks, lpad, out_rows):
    rt.call("masr_dwconv_bn_silu_f32", P(xd), ldg, gb, P(w), P(bias), P(sc), P(sh), P(pad), P(y), P(yh), P(yl), ldy, yb, P(ld), B,
            DW_C, ks, lpad, out_rows, rt.st())


def _call_ln(rt, xd, ldg, gb, w, bias, ga, be, pad, y, yh, yl, ldy, yb, ld, B, ks, lpad, stride, out_rows):
    rt.call("masr_dwconv_ln_silu_strided_f32", P(xd), ldg, gb, P(w), P(bias), P(ga), P(be), P(pad), P(y), P(yh), P(yl), ldy, yb,
            P(ld), B, DW_C, ks, lpad, stride, out_rows, 1e-5, rt.st())


DW_LENS = [0, 1, 4, 5, 16, 17, 64, 65]


@pytest.mark.parametrize("ks,causal", [(15, True), (15, False), (31, True), (31, False)])
def test_dwconv_bn_silu(rt, ks, causal):
    """masr_dwconv_bn_silu_f32 (Squeezeformer conv module): depthwise conv -> BatchNorm1d(eval) -> SiLU, BN folded into
    scale / shift the way squeezeformer.py does; reference with the unfolded running statistics.  Lengths end on and one
    past the 4-frame warp and 16-frame CTA tiles; every row < out_rows follows the contract (rows >= in_len read 0), rows
    >= out_rows are untouched.  Observed max error (H100): 1.3e-6; tolerance 5e-6."""
    lens, ldg, ldy = DW_LENS, DW_C + 4, DW_C + 8
    g, x, w, bias, pad, gb = _dw_problem(ks, lens, ks, ldg, 6)
    B, out_rows = len(lens), max(lens)
    yb = out_rows + 3
    mean, var = torch.randn(DW_C, generator=g) * 0.5, torch.rand(DW_C, generator=g) + 0.5
    bw, bb = 1 + 0.1 * torch.randn(DW_C, generator=g), 0.1 * torch.randn(DW_C, generator=g)
    bn_eps = 1e-3
    scale = bw / torch.sqrt(var + bn_eps)
    shift = bb - mean * scale
    lpad = ks - 1 if causal else (ks - 1) // 2
    d = lambda t: t.contiguous().to(rt.dev)
    y = nan((B * yb, ldy), rt.dev)
    yh, yl = nan((B * yb, ldy), rt.dev, torch.float16), nan((B * yb, ldy), rt.dev, torch.float16)
    ld = torch.tensor(lens, dtype=torch.int32, device=rt.dev)
    _call_bn(rt, d(x.view(B * gb, ldg)), ldg, gb, d(w), d(bias), d(scale), d(shift), d(pad) if causal else None, y, yh, yl, ldy,
             yb, ld, B, ks, lpad, out_rows)
    torch.cuda.synchronize()
    y, yh, yl = y.cpu().view(B, yb, ldy), yh.cpu().view(B, yb, ldy), yl.cpu().view(B, yb, ldy)
    e = 0.0
    for i, n in enumerate(lens):
        r = _dw_conv_reference(x[i], n, w, bias, pad, lpad, 1, out_rows, causal)
        ref = F.silu(F.batch_norm(r.t()[None], mean.double(), var.double(), bw.double(), bb.double(), training=False,
                                  eps=bn_eps)[0].t())
        e = max(e, err(y[i, :out_rows, :DW_C], ref))
        assert_pair_reconstructs(yh[i, :out_rows, :DW_C], yl[i, :out_rows, :DW_C], y[i, :out_rows, :DW_C])
    assert torch.isnan(y[:, out_rows:]).all() and torch.isnan(y[:, :, DW_C:]).all() and torch.isnan(yh[:, out_rows:].float()).all()
    report(f"dwconv_bn_silu k={ks} causal={causal}", out=e)
    assert e < 5e-6


def _ln_silu_reference(r, ga, be):
    return F.silu(F.layer_norm(r, (DW_C,), ga.double(), be.double(), 1e-5))


@pytest.mark.parametrize("causal", [True, False])
def test_dwconv_ln_silu_stride2(rt, causal):
    """masr_dwconv_ln_silu_strided_f32, stride 2, k = 15 (EfficientConformer block 3): odd and even lengths, out_rows =
    ceil(max len / 2); rows < ceil(len/2) are the module's output, the rest of out_rows read zeros past in_len.
    Observed max error (H100): 1.4e-6; tolerance 5e-6."""
    lens = [0, 1, 2, 15, 16, 31, 32, 33, 64, 65]
    ks, ldg, ldy = 15, DW_C + 4, DW_C + 8
    g, x, w, bias, pad, gb = _dw_problem(100 + causal, lens, ks, ldg, 5)
    ga, be = 1 + 0.1 * torch.randn(DW_C, generator=g), 0.1 * torch.randn(DW_C, generator=g)
    B, out_rows = len(lens), ceil2(max(lens))
    yb = out_rows + 2
    lpad = ks - 1 if causal else (ks - 1) // 2
    d = lambda t: t.contiguous().to(rt.dev)
    y = nan((B * yb, ldy), rt.dev)
    yh, yl = nan((B * yb, ldy), rt.dev, torch.float16), nan((B * yb, ldy), rt.dev, torch.float16)
    ld = torch.tensor(lens, dtype=torch.int32, device=rt.dev)
    _call_ln(rt, d(x.view(B * gb, ldg)), ldg, gb, d(w), d(bias), d(ga), d(be), d(pad) if causal else None, y, yh, yl, ldy, yb, ld,
             B, ks, lpad, 2, out_rows)
    torch.cuda.synchronize()
    y, yh, yl = y.cpu().view(B, yb, ldy), yh.cpu().view(B, yb, ldy), yl.cpu().view(B, yb, ldy)
    e = 0.0
    for i, n in enumerate(lens):
        ref = _ln_silu_reference(_dw_conv_reference(x[i], n, w, bias, pad, lpad, 2, out_rows, causal), ga, be)
        e = max(e, err(y[i, :out_rows, :DW_C], ref))
        assert_pair_reconstructs(yh[i, :out_rows, :DW_C], yl[i, :out_rows, :DW_C], y[i, :out_rows, :DW_C])
    assert torch.isnan(y[:, out_rows:]).all() and torch.isnan(y[:, :, DW_C:]).all()
    report(f"dwconv_ln_silu stride 2 causal={causal}", out=e)
    assert e < 5e-6


def test_dwconv_ln_silu_stride2_chunk(rt):
    """The stream pool's strided call (stream_pool.py:486): lpad = 0, [cache ++ chunk] rows per slot with per-slot in_lens,
    8 output rows, pair output only.  Observed max error (H100): 1.1e-6; tolerance 4e-6."""
    lens = [30, 29, 17, 14, 0]
    ks, LC, out_rows = 15, 30, 8
    g, x, w, bias, pad, gb = _dw_problem(200, lens, ks, DW_C, LC - max(lens))
    ga, be = 1 + 0.1 * torch.randn(DW_C, generator=g), 0.1 * torch.randn(DW_C, generator=g)
    B = len(lens)
    d = lambda t: t.contiguous().to(rt.dev)
    yh, yl = nan((B * out_rows, DW_C), rt.dev, torch.float16), nan((B * out_rows, DW_C), rt.dev, torch.float16)
    ld = torch.tensor(lens, dtype=torch.int32, device=rt.dev)
    _call_ln(rt, d(x.view(B * gb, DW_C)), DW_C, gb, d(w), d(bias), d(ga), d(be), None, None, yh, yl, DW_C, out_rows, ld, B, ks, 0,
             2, out_rows)
    torch.cuda.synchronize()
    r = pair_value(yh, yl).view(B, out_rows, DW_C)
    e = 0.0
    for i, n in enumerate(lens):
        ref = _ln_silu_reference(_dw_conv_reference(x[i], n, w, bias, pad, 0, 2, out_rows, False), ga, be)
        e = max(e, err(r[i], ref))
    report("dwconv_ln_silu stride 2 chunk", out=e)
    assert e < 4e-6


def _dwconv_outputs(path):
    """Outputs of the depthwise-conv kernels on fixed seeded inputs, saved to `path` (.npz).  Run in a child process, where
    MASR_DW_TW (read once per process) selects the frames-per-warp variant."""
    from masr_b200 import _lib
    _lib.load()
    dev = torch.device("cuda", 0)

    class R:
        call = staticmethod(_lib.call)

        @staticmethod
        def st():
            return torch.cuda.current_stream().cuda_stream

    lens = DW_LENS
    B, out_rows = len(lens), max(lens)
    ld = torch.tensor(lens, dtype=torch.int32, device=dev)
    res = {}
    for ks, causal, stride in [(7, False, 1), (15, True, 1), (31, False, 1), (15, True, 2), (15, False, 2)]:
        g, x, w, bias, pad, gb = _dw_problem(300 + ks + stride, lens, ks, DW_C, 3)
        ga, be = 1 + 0.1 * torch.randn(DW_C, generator=g), 0.1 * torch.randn(DW_C, generator=g)
        rows = out_rows if stride == 1 else ceil2(out_rows)
        lpad = ks - 1 if causal else (ks - 1) // 2
        y = nan((B * rows, DW_C), dev)
        yh, yl = nan((B * rows, DW_C), dev, torch.float16), nan((B * rows, DW_C), dev, torch.float16)
        dd = lambda t: t.contiguous().to(dev)
        _call_ln(R, dd(x.view(B * gb, DW_C)), DW_C, gb, dd(w), dd(bias), dd(ga), dd(be), dd(pad) if causal else None, y, yh, yl,
                 DW_C, rows, ld, B, ks, lpad, stride, rows)
        res[f"ln_k{ks}_c{int(causal)}_s{stride}"] = y
        res[f"ln_k{ks}_c{int(causal)}_s{stride}_h"] = yh
        if stride == 1 and ks in (15, 31):
            yb = nan((B * rows, DW_C), dev)
            _call_bn(R, dd(x.view(B * gb, DW_C)), DW_C, gb, dd(w), dd(bias), dd(ga), dd(be), dd(pad) if causal else None, yb, None,
                     None, DW_C, rows, ld, B, ks, lpad, rows)
            res[f"bn_k{ks}_c{int(causal)}"] = yb
    torch.cuda.synchronize()
    np.savez(path, **{k: v.cpu().float().numpy() for k, v in res.items()})


def test_dwconv_tw8_variant_bit_identical(rt, tmp_path):
    """MASR_DW_TW=8 (8 output frames per warp, selected once per process) against the default 4-frame kernel, each in a
    child process that has exited before the comparison: the per-output FMA order is the same, so the outputs must be
    bit-identical."""
    outs = {}
    for tw in ("4", "8"):
        path = str(tmp_path / f"dw_tw{tw}.npz")
        code = (f"import sys; sys.path[:0] = [{ROOT!r}, {os.path.join(ROOT, 'tests')!r}]; "
                f"import test_gpu_family_kernels as t; t._dwconv_outputs({path!r})")
        args = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", code]
        r = subprocess.run(args, env={**os.environ, "MASR_DW_TW": tw}, cwd=ROOT, capture_output=True, text=True, timeout=900)
        assert r.returncode == 0, r.stderr[-3000:]
        outs[tw] = dict(np.load(path))
    assert outs["4"].keys() == outs["8"].keys() and len(outs["4"]) == 12
    for k, a in outs["4"].items():
        assert np.isfinite(a).all(), k
        assert np.array_equal(a, outs["8"][k]), k


# ---- Squeezeformer / EfficientConformer time-axis helpers --------------------------------------------------------------------

TIME_LENS = [0, 1, 2, 3, 16, 17, 64, 65]


def _time_problem(seed, lens, D=256, extra=3):
    g = torch.Generator().manual_seed(seed)
    B, Tm = len(lens), max(lens)
    bs = Tm + extra
    x = garbage((B, bs, D), seed)
    for i, n in enumerate(lens):
        x[i, :n] = torch.randn(n, D, generator=g)
    return g, x, bs


@pytest.mark.parametrize("k,pad", [(1, 0), (5, 3)])
def test_time_reduce_dw_split(rt, k, pad):
    """masr_time_reduce_dw_split_f16: TimeReductionLayerStream (k 1, pad 0) and TimeReductionLayer1D (k 5, pad 3) depthwise
    convs against F.conv1d(stride=2, groups=d) on each utterance alone, rows < ceil(len/2); the pair output only; rows >=
    out_rows untouched.  Observed max error (H100): k1 7.0e-7, k5 7.9e-7 (outputs up to ~10); tolerance 2.5e-6."""
    lens, D = TIME_LENS, 256
    g, x, bs = _time_problem(50 + k, lens, D)
    w, bias = torch.randn(D, k, generator=g) / math.sqrt(k), torch.randn(D, generator=g) * 0.1
    B, out_rows = len(lens), ceil2(max(lens))
    ob = out_rows + 2
    yh, yl = nan((B * ob, D), rt.dev, torch.float16), nan((B * ob, D), rt.dev, torch.float16)
    ld = torch.tensor(lens, dtype=torch.int32, device=rt.dev)
    xd, wd, bd = x.view(B * bs, D).to(rt.dev), w.to(rt.dev), bias.to(rt.dev)
    rt.call("masr_time_reduce_dw_split_f16", P(xd), bs, P(wd), P(bd), P(yh), P(yl), ob, P(ld), B, out_rows, k, pad, D, rt.st())
    torch.cuda.synchronize()
    r = pair_value(yh, yl).view(B, ob, D)
    e = 0.0
    for i, n in enumerate(lens):
        if n:
            ref = F.conv1d(x[i, :n].double().t()[None], w.double()[:, None], bias.double(), stride=2, padding=pad, groups=D)[0].t()
            e = max(e, err(r[i, :ceil2(n)], ref[:ceil2(n)]))
    assert torch.isnan(r[:, out_rows:]).all()
    report(f"time_reduce k={k}", out=e)
    assert e < 2.5e-6


def test_upsample2_add(rt):
    """masr_upsample2_add_f32: bit-exact against saved + z.repeat_interleave(2)[:T] in fp32 (odd T); rows past T untouched."""
    g = torch.Generator().manual_seed(9)
    B, T, D = 3, 37, 256
    fb, hb = T + 3, ceil2(T) + 2
    saved, z = torch.randn(B, fb, D, generator=g), torch.randn(B, hb, D, generator=g)
    saved[:, T:] = garbage((B, fb - T, D), 9)
    z[:, ceil2(T):] = garbage((B, hb - ceil2(T), D), 10)
    out = nan((B * fb, D), rt.dev)
    sd, zd = saved.view(B * fb, D).to(rt.dev), z.view(B * hb, D).to(rt.dev)
    rt.call("masr_upsample2_add_f32", P(sd), P(zd), P(out), fb, hb, B, T, D, rt.st())
    out = out.cpu().view(B, fb, D)
    for b in range(B):
        assert torch.equal(out[b, :T], saved[b, :T] + z[b].repeat_interleave(2, dim=0)[:T])
    assert torch.isnan(out[:, T:]).all()


def test_avgpool2_time(rt):
    """masr_avgpool2_time_f32: bit-exact against F.avg_pool1d(2, 2, ceil_mode=True, count_include_pad=False) in fp32 per
    utterance (the odd tail is a single element); rows in [ceil(len/2), out_rows) are 0, rows past out_rows untouched."""
    lens, D = TIME_LENS, 256
    g, x, bs = _time_problem(60, lens, D)
    B, out_rows = len(lens), ceil2(max(lens))
    ob = out_rows + 2
    y = nan((B * ob, D), rt.dev)
    ld = torch.tensor(lens, dtype=torch.int32, device=rt.dev)
    xd = x.view(B * bs, D).to(rt.dev)
    rt.call("masr_avgpool2_time_f32", P(xd), bs, P(y), ob, P(ld), B, out_rows, D, rt.st())
    y = y.cpu().view(B, ob, D)
    for i, n in enumerate(lens):
        if n:
            ref = F.avg_pool1d(x[i, :n].t()[None], 2, 2, ceil_mode=True, count_include_pad=False)[0].t()
            assert torch.equal(y[i, :ceil2(n)], ref), i
        assert torch.all(y[i, ceil2(n):out_rows] == 0)
    assert torch.isnan(y[:, out_rows:]).all()


# ---- LayerNorms: Squeezeformer post-norm + adaptive scale, DeepSpeech2 widths ------------------------------------------------

def _ln_inputs(M, D, ldx, seed):
    """Rows of 100 + N(0, 1): a large mean next to the spread (the two-pass variance); garbage in the row pitch past D."""
    g = torch.Generator().manual_seed(seed)
    x = garbage((M, ldx), seed)
    x[:, :D] = 100 + torch.randn(M, D, generator=g)
    ga, be = 1 + 0.1 * torch.randn(D, generator=g), 0.1 * torch.randn(D, generator=g)
    return g, x, ga, be


def _ln_reference(x, D, ga, be):
    return F.layer_norm(x[:, :D].double(), (D,), ga.double(), be.double(), 1e-5)


@pytest.mark.parametrize("with_y", [False, True])
@pytest.mark.parametrize("ada", [False, True])
def test_layernorm_ada_split(rt, ada, with_y):
    """masr_layernorm_ada_split_f16 with / without the ada (scale, bias) pair and the fp32 y; ldx, ldy > D; M = 1003 (not a
    multiple of the 8 rows per CTA).  Observed max error (H100): 1.4e-5 without ada, 1.8e-5 with it; tolerance 4e-5.  The
    float32 mean of rows around 100 is off by about one ulp of 100 (7.6e-6), and that error reaches every output."""
    M, D, ldx, ldy = 1003, 256, 264, 260
    g, x, ga, be = _ln_inputs(M, D, ldx, 70 + 2 * ada + with_y)
    asc, abi = 1 + 0.2 * torch.randn(D, generator=g), 0.2 * torch.randn(D, generator=g)
    d = lambda t: t.contiguous().to(rt.dev)
    y = nan((M, ldy), rt.dev)
    yh, yl = nan((M, ldy), rt.dev, torch.float16), nan((M, ldy), rt.dev, torch.float16)
    xd, gd, bd, ad, abd = d(x), d(ga), d(be), d(asc), d(abi)
    rt.call("masr_layernorm_ada_split_f16", P(xd), ldx, P(gd), P(bd), P(y) if with_y else None, P(ad) if ada else None,
            P(abd) if ada else None, P(yh), P(yl), ldy, M, D, 1e-5, rt.st())
    torch.cuda.synchronize()
    ref = _ln_reference(x, D, ga, be)
    pref = asc.double() * ref + abi.double() if ada else ref
    errs = {"pair": err(pair_value(yh[:, :D], yl[:, :D]), pref)}
    if with_y:
        errs["y"] = err(y[:, :D], ref)
        if not ada:
            assert_pair_reconstructs(yh[:, :D], yl[:, :D], y[:, :D])
        assert torch.isnan(y[:, D:]).all()
    else:
        assert torch.isnan(y).all()
    assert torch.isnan(yh[:, D:].float()).all() and torch.isnan(yl[:, D:].float()).all()
    report(f"layernorm_ada ada={ada} y={with_y}", **errs)
    assert max(errs.values()) < 4e-5


@pytest.mark.parametrize("scaled", [False, True])
@pytest.mark.parametrize("M,D", [(37, 256), (3, 1000)])
def test_affine_split(rt, M, D, scaled):
    """masr_affine_split_f16 with and without scale / bias; M*D/4 is not a multiple of the 256-thread block and nothing past
    M*D is written.  Observed max error (H100): 1.4e-6 on outputs up to ~20 (about one float32 ulp); tolerance 5e-6."""
    g = torch.Generator().manual_seed(M + D + scaled)
    x = torch.randn(M * D, generator=g) * 3
    s, b = 1 + 0.3 * torch.randn(D, generator=g), 0.5 * torch.randn(D, generator=g)
    yh, yl = nan((M * D + 64,), rt.dev, torch.float16), nan((M * D + 64,), rt.dev, torch.float16)
    xd, sd, bd = x.to(rt.dev), s.to(rt.dev), b.to(rt.dev)
    rt.call("masr_affine_split_f16", P(xd), P(sd) if scaled else None, P(bd) if scaled else None, P(yh), P(yl), M, D, rt.st())
    torch.cuda.synchronize()
    r = pair_value(yh[:M * D], yl[:M * D])
    if scaled:
        e = err(r, (x.double().view(M, D) * s.double() + b.double()).view(-1))
        report(f"affine_split M={M} D={D}", out=e)
        assert e < 5e-6
    else:
        assert_pair_reconstructs(yh[:M * D], yl[:M * D], x)
    assert torch.isnan(yh[M * D:].float()).all() and torch.isnan(yl[M * D:].float()).all()


@pytest.mark.parametrize("D", [512, 1024, 2048])
def test_layernorm_wide(rt, D):
    """masr_layernorm_f32 at D = 512 / 1024 / 2048 (DeepSpeech2) and masr_layernorm_split_f16 at 1024 / 2048: out of place
    with ldx > D, in place (bit-identical, the row pitch past D untouched), large-mean rows, M = 77.
    Observed max error (H100): 1.4e-5 (the large mean, as in test_layernorm_ada_split); tolerance 3e-5."""
    M, ldx = 77, D + 4
    g, x, ga, be = _ln_inputs(M, D, ldx, D)
    xd, gd, bd = x.to(rt.dev), ga.to(rt.dev), be.to(rt.dev)
    y = nan((M, ldx), rt.dev)
    rt.call("masr_layernorm_f32", P(xd), ldx, P(gd), P(bd), P(y), ldx, M, D, 1e-5, rt.st())
    ref = _ln_reference(x, D, ga, be)
    errs = {"y": err(y[:, :D], ref)}
    assert torch.isnan(y[:, D:]).all()
    if D in (1024, 2048):
        yh, yl = nan((M, ldx), rt.dev, torch.float16), nan((M, ldx), rt.dev, torch.float16)
        rt.call("masr_layernorm_split_f16", P(xd), ldx, P(gd), P(bd), P(yh), P(yl), ldx, M, D, 1e-5, rt.st())
        assert_pair_reconstructs(yh[:, :D], yl[:, :D], y[:, :D])
        errs["pair"] = err(pair_value(yh[:, :D], yl[:, :D]), ref)
    xi = xd.clone()
    rt.call("masr_layernorm_f32", P(xi), ldx, P(gd), P(bd), P(xi), ldx, M, D, 1e-5, rt.st())
    torch.cuda.synchronize()
    assert torch.equal(xi[:, :D], y[:, :D]) and torch.equal(xi[:, D:], xd[:, D:])
    report(f"layernorm D={D}", **errs)
    assert max(errs.values()) < 3e-5


def test_layernorm_rejects_unsupported_width(rt):
    from masr_b200._lib import MasrB200Error
    x = torch.zeros(8, 1024, device=rt.dev); ga = torch.ones(1024, device=rt.dev); be = torch.zeros(1024, device=rt.dev)
    h = torch.zeros(8, 1024, dtype=torch.float16, device=rt.dev); l = torch.zeros_like(h)
    with pytest.raises(MasrB200Error):
        rt.call("masr_layernorm_f32", P(x), 1024, P(ga), P(be), P(x), 1024, 8, 768, 1e-5, rt.st())
    with pytest.raises(MasrB200Error):
        rt.call("masr_layernorm_split_f16", P(x), 1024, P(ga), P(be), P(h), P(l), 1024, 8, 512, 1e-5, rt.st())
    with pytest.raises(MasrB200Error):
        rt.call("masr_layernorm_ada_split_f16", P(x), 1024, P(ga), P(be), None, None, None, P(h), P(l), 1024, 8, 512, 1e-5, rt.st())
    torch.cuda.synchronize()
    assert torch.all(h == 0)
