"""GPU (-m gpu): DeepSpeech2 at ``encoder_conf.rnn_size: 2048`` (the large-data size of configs/deepspeech2.yml).

* ``masr_{lstm,gru}_seq_tc_f16x2`` (the tensor-core persistent recurrence) and the per-step kernels at H = 2048 against
  float64 ``torch.nn.LSTM`` / ``torch.nn.GRU`` over ``pack_padded_sequence``, with the conventions of
  test_gpu_family_kernels.py (garbage past every length, NaN-filled outputs);
* their host-side rejections (nothing launched, nothing written);
* both LayerNorm entry points at D = 4096 (the bidirectional model's 2 x 2048) against float64;
* the engine, uni and bi, LSTM and GRU, whole utterances and the chunk walk against the reference's outputs frozen at
  rnn_size 2048 (tests/golden/make_wide_deepspeech2_golden.py) and a ragged batch against the oracle, under both
  recurrence forms;
* the stream pool (8 and 33 slots, a CUDA graph replay) against the single stream bit for bit, and ``StreamPool`` (greedy
  and beam) against ``predict_stream``, under both forms;
* ``MASRPredictor.predict`` / ``predict_stream`` of both cells against the reference predictor's frozen results.

Error budget of the tensor-core product: W_hh and h_{t-1} enter as fp16 (h, l) pairs, each within 2^-22 relative of its
fp32 value, and the dropped l.l product is 2^-22 smaller than the main one, so every product term carries about 2^-21
relative error against 2^-24 for the fp32 kernels.  Over K = 2048 terms of size |w||h| <= 0.05 (W ~ N(0, 1/H)) that is
~1e-7 per gate per step; the LSTM / GRU cells are contractive, so the error after 250 steps stays at a few times the one-
step error.  Observed maxima (H100 80GB HBM3, 700 W): after up to 250 steps out 3.3e-6, h 2.4e-6, c 1.8e-6 (GRU outputs
are the larger); the per-step fp32 kernels 2.0e-6; tensor-core vs per-step 3.2e-6; the engine's posteriors 1.6e-6 from the
oracle.  Tolerances: 2e-5 for the kernels (6x), 5e-5 for posteriors (as the other DeepSpeech2 tests)."""
import ctypes
import json
import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import GOLDEN, load_npz, make_audio
from kernel_contract import P, assert_pair_reconstructs, err, garbage, nan, report, runtime, same
from masr_b200 import synth
from masr_b200.engine import subsampled_len
from oracle import ctc as octc, deepspeech2 as od, deepspeech2_gru as og, fbank as ob
from masr_b200.text import ids_to_text
from test_gpu_deepspeech2_stream_pool import ALPHA, BETA, _compare, _streams
from test_gpu_deepspeech2_stream_pool import _reference as _stream_reference
from test_gpu_family_kernels import from_T, to_T
from test_gpu_stream_pool_beam import _drive

pytestmark = pytest.mark.gpu

H = 2048
RNN_IN = 16
V = synth.DEFAULT_VOCAB_SIZE


@pytest.fixture(scope="module")
def rt():
    return runtime()


def _problem(cell, B, T, seed):
    """Seeded inputs of one bidirectional layer (x, W_ih and the biases on dyadic grids, so the float64 input projection is
    exactly the float32 gates_x the kernels read).  Lengths include 0 (a lane finished from the start), 1, T-1 and T."""
    G = 4 if cell == "lstm" else 3
    g = torch.Generator().manual_seed(seed)
    if B == 1:
        lens = [T]
    else:
        lens = torch.randint(0, T + 1, (B,), generator=g).tolist()
        lens[:4] = [T, 0, 1, max(T - 1, 0)][:B]
    x = torch.randint(-16, 17, (B, T, RNN_IN), generator=g).double() / 8
    w_ih = torch.randint(-32, 33, (2, G * H, RNN_IN), generator=g).double() / 64
    b_ih = torch.randint(-256, 257, (2, G * H), generator=g).double() / 512
    b_hh = torch.randint(-256, 257, (2, G * H), generator=g).double() / 512
    w_hh = torch.randn(2, G * H, H, generator=g) / math.sqrt(H)
    h0 = torch.randn(2, B, H, generator=g) * 0.5
    c0 = torch.randn(2, B, H, generator=g) * 0.5
    if cell == "lstm":
        fold = b_hh
    else:      # b_hr, b_hz fold into gates_x; b_hn stays inside the product with r
        fold = torch.cat([b_hh[:, :2 * H], torch.zeros(2, H, dtype=torch.float64)], 1)
    gx = torch.stack([F.linear(x, w_ih[d], b_ih[d] + fold[d]) for d in range(2)])
    assert torch.equal(gx.float().double(), gx)
    return dict(cell=cell, G=G, B=B, T=T, lens=lens, x=x, w_ih=w_ih, b_ih=b_ih, b_hh=b_hh, w_hh=w_hh, h0=h0, c0=c0,
                gx=gx.float(), bhn=b_hh[:, 2 * H:].float())


def _reference(pb):
    """float64 torch.nn.LSTM / GRU (bidirectional) over pack_padded_sequence -> out [B, T, 2H], h_n, c_n [2, B, H]."""
    B, T, lens = pb["B"], pb["T"], pb["lens"]
    lstm = pb["cell"] == "lstm"
    dev = torch.device("cuda")
    mod = (torch.nn.LSTM if lstm else torch.nn.GRU)(RNN_IN, H, batch_first=True, bidirectional=True, dtype=torch.float64).to(dev)
    with torch.no_grad():
        for d, sfx in enumerate(("", "_reverse")):
            getattr(mod, "weight_ih_l0" + sfx).copy_(pb["w_ih"][d])
            getattr(mod, "weight_hh_l0" + sfx).copy_(pb["w_hh"][d].double())
            getattr(mod, "bias_ih_l0" + sfx).copy_(pb["b_ih"][d])
            getattr(mod, "bias_hh_l0" + sfx).copy_(pb["b_hh"][d])
    out = torch.zeros(B, T, 2 * H, dtype=torch.float64)
    hn, cn = pb["h0"].double().clone(), pb["c0"].double().clone()
    idx = [i for i in range(B) if lens[i] > 0]
    if idx:
        it = torch.tensor(idx)
        packed = torch.nn.utils.rnn.pack_padded_sequence(pb["x"][it].to(dev), torch.tensor([lens[i] for i in idx]),
                                                         batch_first=True, enforce_sorted=False)
        h0 = pb["h0"][:, it].double().to(dev)
        with torch.no_grad():
            if lstm:
                o, (h, c) = mod(packed, (h0, pb["c0"][:, it].double().to(dev)))
                cn[:, it] = c.cpu()
            else:
                o, h = mod(packed, h0)
        out[it] = torch.nn.utils.rnn.pad_packed_sequence(o, batch_first=True, total_length=T)[0].cpu()
        hn[:, it] = h.cpu()
    return out, hn, cn


class _Run:
    """Device buffers of one bidirectional layer: gates_x per direction (garbage past every length), one [B*bstride, 2H]
    output (forward at col_off 0, reverse at H) as fp32 and as pair, W_hh packed for the tensor-core kernel."""

    def __init__(self, rt, pb):
        B, T, G = pb["B"], pb["T"], pb["G"]
        self.rt, self.pb, self.bstride = rt, pb, T + 2
        bs = self.bstride
        self.gx = []
        for d in range(2):
            buf = garbage((B, bs, G * H), 20 + d)
            for i, n in enumerate(pb["lens"]):
                buf[i, :n] = pb["gx"][d, i, :n]
            self.gx.append(buf.view(B * bs, G * H).to(rt.dev))
        self.whh = [pb["w_hh"][d].to(rt.dev) for d in range(2)]
        self.packed = []
        for d in range(2):
            buf = torch.empty(G * H * H * 4, dtype=torch.uint8, device=rt.dev)
            rt.call("masr_rnn_tc_pack_f16x2", P(self.whh[d]), P(buf), G, H, rt.st())
            self.packed.append(buf)
        self.bhn = [pb["bhn"][d].to(rt.dev) for d in range(2)]
        self.lens = torch.tensor(pb["lens"], dtype=torch.int32, device=rt.dev)
        self.out = nan((B * bs, 2 * H), rt.dev)
        self.oh, self.ol = nan((B * bs, 2 * H), rt.dev, torch.float16), nan((B * bs, 2 * H), rt.dev, torch.float16)

    def aux(self, d, c):
        return c if self.pb["cell"] == "lstm" else self.bhn[d]

    def seq_tc(self, d, h0T, hNT, c, fp32_out=True):
        pb, rt = self.pb, self.rt
        nbytes = ctypes.c_int64()
        rt.call("masr_rnn_seq_tc_workspace_bytes", pb["B"], H, ctypes.byref(nbytes))
        ws = torch.empty(nbytes.value, dtype=torch.uint8, device=rt.dev)
        fn = "masr_lstm_seq_tc_f16x2" if pb["cell"] == "lstm" else "masr_gru_seq_tc_f16x2"
        rt.call(fn, P(self.gx[d]), pb["G"] * H, self.bstride, P(self.packed[d]), P(h0T), P(hNT), P(self.aux(d, c)),
                P(self.out) if fp32_out else None, P(self.oh), P(self.ol), 2 * H, d * H, P(self.lens), pb["B"], H,
                max(pb["lens"]), d, P(ws), nbytes.value, rt.st())

    def step(self, d, h0T, c):
        pb, rt = self.pb, self.rt
        bufs = [h0T.clone(), torch.full_like(h0T, float("nan"))]
        T = max(pb["lens"])
        fn = "masr_lstm_step_f32" if pb["cell"] == "lstm" else "masr_gru_step_f32"
        for s in range(T):
            rt.call(fn, P(self.gx[d]), pb["G"] * H, self.bstride, P(self.whh[d]), P(bufs[s % 2]), P(bufs[1 - s % 2]),
                    P(self.aux(d, c)), P(self.out), P(self.oh), P(self.ol), 2 * H, d * H, P(self.lens), pb["B"], H, s, d, rt.st())
        return bufs[T % 2]

    def check_rows(self, ref_out):
        pb, bs = self.pb, self.bstride
        torch.cuda.synchronize()
        out, oh, ol = (t.cpu().view(pb["B"], bs, 2 * H) for t in (self.out, self.oh, self.ol))
        e = 0.0
        for i, n in enumerate(pb["lens"]):
            e = max(e, err(out[i, :n], ref_out[i, :n]))
            assert_pair_reconstructs(oh[i, :n], ol[i, :n], out[i, :n])
            assert torch.isnan(out[i, n:]).all() and torch.isnan(oh[i, n:].float()).all() and torch.isnan(ol[i, n:].float()).all()
        return e


def _run_impl(rt, pb, impl, alias=False, fp32_out=True):
    """Both directions of `impl` ("tc" or "step") -> (errors vs float64, fp32 output, final (h, c) per direction)."""
    ref_out, ref_h, ref_c = _reference(pb)
    run = _Run(rt, pb)
    B = pb["B"]
    eh = ec = 0.0
    finals = []
    for d in range(2):
        h0T = to_T(pb["h0"][d], 30 + d).to(rt.dev)
        c = pb["c0"][d].clone().to(rt.dev)
        if impl == "tc":
            hNT = h0T if alias else nan(h0T.shape, rt.dev)
            run.seq_tc(d, h0T, hNT, c, fp32_out=fp32_out)
        else:
            hNT = run.step(d, h0T, c)
        torch.cuda.synchronize()
        hN, cN = from_T(hNT, B), c.cpu()
        for i, n in enumerate(pb["lens"]):
            if n == 0:              # finished from the start: state untouched
                assert torch.equal(hN[i], pb["h0"][d, i]) and torch.equal(cN[i], pb["c0"][d, i])
        eh = max(eh, err(hN, ref_h[d]))
        if pb["cell"] == "lstm":
            ec = max(ec, err(cN, ref_c[d]))
        finals.append((hN, cN))
    eo = run.check_rows(ref_out) if fp32_out else None
    return (eo, eh, ec), run, finals


TOL = 2e-5


@pytest.mark.parametrize("cell", ["lstm", "gru"])
@pytest.mark.parametrize("B,T", [(1, 1), (1, 250), (7, 16), (32, 250), (33, 16), (33, 250)])
def test_seq_tc_against_float64(rt, cell, B, T):
    """masr_{lstm,gru}_seq_tc_f16x2, both directions into one [M, 2H] output, non-zero h0 / c0 / b_hh, ragged lengths with a
    lane finished from the start, 33 utterances = two lane groups."""
    pb = _problem(cell, B, T, seed=B * 1000 + T + (7 if cell == "gru" else 0))
    (eo, eh, ec), run, _ = _run_impl(rt, pb, "tc")
    report(f"{cell} seq_tc H={H} B={B} T={T}", out=eo, h=eh, c=ec)
    assert eo < TOL and eh < TOL and ec < TOL, (eo, eh, ec)


@pytest.mark.parametrize("cell", ["lstm", "gru"])
def test_seq_tc_aliasing_pair_output_and_step_kernel(rt, cell):
    """h0_T == hN_T gives bit for bit the non-aliased result, a pair-only output equals the pair of the fp32 run, and the
    per-step kernel at H = 2048 meets the same float64 reference and agrees with the tensor-core form."""
    pb = _problem(cell, 9, 40, seed=77 if cell == "lstm" else 78)
    _, run_a, fin_a = _run_impl(rt, pb, "tc")
    _, run_b, fin_b = _run_impl(rt, pb, "tc", alias=True, fp32_out=False)
    for (ha, ca), (hb, cb) in zip(fin_a, fin_b):
        assert torch.equal(ha, hb) and torch.equal(ca, cb)
    assert same(run_a.oh, run_b.oh) and same(run_a.ol, run_b.ol) and torch.isnan(run_b.out).all()
    (eo, eh, ec), run_s, fin_s = _run_impl(rt, pb, "step")
    report(f"{cell} step H={H} B=9 T=40", out=eo, h=eh, c=ec)
    assert eo < TOL and eh < TOL and ec < TOL, (eo, eh, ec)
    so, to = run_a.out.cpu(), run_s.out.cpu()
    valid = ~torch.isnan(so)
    assert torch.equal(valid, ~torch.isnan(to))
    diff = (so[valid] - to[valid]).abs().max().item()
    report(f"{cell} seq_tc vs step", diff=diff)
    assert diff < TOL


def test_seq_tc_zero_steps(rt):
    """Every utterance empty: hN = h0, c and every output untouched."""
    pb = _problem("lstm", 5, 8, seed=5)
    pb["lens"] = [0] * 5
    run = _Run(rt, pb)
    h0T = to_T(pb["h0"][0], 40).to(rt.dev)
    hNT, c = nan(h0T.shape, rt.dev), pb["c0"][0].clone().to(rt.dev)
    nbytes = ctypes.c_int64()
    rt.call("masr_rnn_seq_tc_workspace_bytes", 5, H, ctypes.byref(nbytes))
    ws = torch.empty(nbytes.value, dtype=torch.uint8, device=rt.dev)
    rt.call("masr_lstm_seq_tc_f16x2", P(run.gx[0]), 4 * H, run.bstride, P(run.packed[0]), P(h0T), P(hNT), P(c), P(run.out),
            P(run.oh), P(run.ol), 2 * H, 0, P(run.lens), 5, H, 0, 0, P(ws), nbytes.value, rt.st())
    torch.cuda.synchronize()
    assert torch.equal(hNT, h0T) and torch.equal(c.cpu(), pb["c0"][0])
    assert torch.isnan(run.out).all() and torch.isnan(run.oh.float()).all()


def test_seq_tc_rejects_bad_arguments(rt):
    """Host-side MASR_REQUIRE before any launch: H other than 2048, a short workspace and null pointers (packed weights,
    c_state / b_hn, the workspace); the packer rejects other widths and gate counts.  Nothing is written.

    The remaining refusal, a grid whose 128 CTAs cannot all be resident at once (occupancy per SM x SMs < H / 16, checked
    with cudaOccupancyMaxActiveBlocksPerMultiprocessor for the kernel's real registers and shared memory), is not provoked
    here: an H100 (132 SMs, one 216 KiB CTA each) always has room, and shrinking the device a process sees would need a
    device-level setting (MPS SM limits) that a test must not change."""
    from masr_b200._lib import MasrB200Error
    B, T = 3, 4
    gx = torch.zeros(B * T, 4 * 4096, device=rt.dev)
    wp = torch.zeros(4 * H * H * 4, dtype=torch.uint8, device=rt.dev)
    hA = torch.zeros(1, 4096, 32, device=rt.dev); hB = torch.zeros_like(hA); c = torch.zeros(B, 4096, device=rt.dev)
    out = torch.zeros(B * T, 2 * 4096, device=rt.dev); lens = torch.full((B,), T, dtype=torch.int32, device=rt.dev)
    need = ctypes.c_int64()
    rt.call("masr_rnn_seq_tc_workspace_bytes", B, 4096, ctypes.byref(need))
    ws = torch.zeros(need.value, dtype=torch.uint8, device=rt.dev)
    n2048 = ctypes.c_int64()
    rt.call("masr_rnn_seq_tc_workspace_bytes", B, H, ctypes.byref(n2048))

    def seq(fn, Hx, nbytes, w=wp, a=c, work=ws):
        G = 4 if "lstm" in fn else 3
        rt.call(fn, P(gx), G * Hx, T, P(w), P(hA), P(hB), P(a), P(out), None, None, 2 * Hx, 0, P(lens), B, Hx, T, 0, P(work),
                nbytes, rt.st())

    for fn in ("masr_lstm_seq_tc_f16x2", "masr_gru_seq_tc_f16x2"):
        for Hx in (1024, 2176, 4096):
            with pytest.raises(MasrB200Error, match=fn + ": H="):
                seq(fn, Hx, need.value)
        with pytest.raises(MasrB200Error, match="workspace"):
            seq(fn, H, n2048.value - 1)
        for kw in ({"w": None}, {"a": None}, {"work": None}):
            with pytest.raises(MasrB200Error, match="null pointer"):
                seq(fn, H, n2048.value, **kw)
    pk = torch.zeros(16, dtype=torch.uint8, device=rt.dev)
    for G, Hx in ((4, 1024), (2, H), (5, H)):
        with pytest.raises(MasrB200Error, match="masr_rnn_tc_pack_f16x2"):
            rt.call("masr_rnn_tc_pack_f16x2", P(gx), P(pk), G, Hx, rt.st())
    with pytest.raises(MasrB200Error, match="null pointer"):
        rt.call("masr_rnn_tc_pack_f16x2", None, P(pk), 4, H, rt.st())
    torch.cuda.synchronize()
    assert torch.all(hB == 0) and torch.all(out == 0) and torch.all(c == 0) and torch.all(pk == 0)


def test_layernorm_4096(rt):
    """masr_layernorm_f32 and masr_layernorm_split_f16 at D = 4096 (row pitches wider than D) against float64."""
    D, M, ld = 4096, 37, 4096 + 64
    g = torch.Generator().manual_seed(4096)
    x = torch.randn(M, ld, generator=g) * 3 + 0.5
    gamma, beta = torch.randn(D, generator=g), torch.randn(D, generator=g)
    xd = x[:, :D].double()
    ref = (xd - xd.mean(1, keepdim=True)) / torch.sqrt(xd.var(1, unbiased=False, keepdim=True) + 1e-5) * gamma.double() + beta.double()
    dx, dg, db = x.to(rt.dev), gamma.to(rt.dev), beta.to(rt.dev)
    y = nan((M, ld), rt.dev)
    yh, yl = nan((M, ld), rt.dev, torch.float16), nan((M, ld), rt.dev, torch.float16)
    rt.call("masr_layernorm_f32", P(dx), ld, P(dg), P(db), P(y), ld, M, D, 1e-5, rt.st())
    rt.call("masr_layernorm_split_f16", P(dx), ld, P(dg), P(db), P(yh), P(yl), ld, M, D, 1e-5, rt.st())
    torch.cuda.synchronize()
    e = err(y[:, :D], ref)
    report("layernorm D=4096", f32=e)
    assert e < 1e-5
    assert torch.isnan(y[:, D:]).all() and torch.isnan(yh[:, D:].float()).all()
    assert_pair_reconstructs(yh[:, :D], yl[:, :D], y[:, :D])


# ---- engine: the reference frozen at rnn_size 2048 (tests/golden/make_wide_deepspeech2_golden.py) ------------------------
_W = {}


WSEED = {("lstm", True): 0, ("gru", True): 2, ("lstm", False): 1, ("gru", False): 1}     # the frozen fixtures' weight seeds


def weights(cell, streaming):
    key = (cell, streaming)
    if key not in _W:
        _W[key] = synth.deepspeech2_state_dict(WSEED[key], streaming=streaming, hidden=H, use_gru=cell == "gru")
    return _W[key]


@pytest.fixture(scope="module")
def engines():
    from masr_b200.deepspeech2 import DeepSpeech2Engine
    cache = {}

    def get(cell, streaming):
        if (cell, streaming) not in cache:
            for k in list(cache):                   # one 2048-wide model at a time
                del cache[k]
            torch.cuda.empty_cache()
            cache[cell, streaming] = DeepSpeech2Engine(weights(cell, streaming), streaming=streaming)
        return cache[cell, streaming]
    return get


def _oracle(cell, streaming, feats, state=None):
    sd = synth.to_torch(weights(cell, streaming))
    cfg = od.DS2Config(hidden=H, bidirectional=not streaming)
    with torch.no_grad():
        return (od if cell == "lstm" else og).get_encoder_out(sd, cfg, feats[None], state)


@pytest.mark.parametrize("cell", ["lstm", "gru"])
@pytest.mark.parametrize("streaming", [True, False])
def test_engine_whole_utterances_against_golden_and_oracle(engines, cell, streaming):
    """The reference's frozen utterance: frame ids bit-exact, greedy text and score, top-8 posteriors within 5e-5, under
    both recurrence forms.  Then a ragged batch against the oracle (ids, text, posteriors within 5e-5), with the
    tensor-core and per-step recurrences agreeing within the same bound."""
    eng = engines(cell, streaming)
    assert eng.H == H and eng.w.cell == cell and eng.rnn_form == "seq_tc"
    vocab = synth.vocabulary()
    z, meta = load_npz("deepspeech2_wide_golden.npz")
    m, = [m for m in meta if m["cell"] == cell and not m.get("chunks") and m["streaming"] == streaming]
    assert m["wseed"] == WSEED[cell, streaming] and m["text"]
    feat = z[m["name"] + "/feat"]
    for persistent in (True, False):
        eng.persistent_lstm = persistent
        try:
            res = eng.transcribe_features(torch.from_numpy(feat)[None].to(eng.device), [feat.shape[0]], None,
                                          return_frames=True)
            probs = eng.posteriors(feat[None], [feat.shape[0]])[0]
        finally:
            eng.persistent_lstm = True
        assert np.array_equal(res.frame_ids[0, :res.frame_lens[0]], z[m["name"] + "/ids"]), persistent
        assert ids_to_text(res.tokens[0], vocab) == m["text"] and abs(res.scores[0] - m["score"]) < 1e-3, persistent
        got = np.take_along_axis(probs, z[m["name"] + "/top_i"].astype(np.int64), axis=1)
        e = np.abs(got - z[m["name"] + "/top_p"]).max()
        report(f"ds2 {cell} {'uni' if streaming else 'bi'} golden persistent={persistent}", top8=e)
        assert e < 5e-5
    lens = [16000 * 2 + 17, 9000, 16000 + 320, 400 + 160 * 30]
    waves = [make_audio("speech" if i % 2 == 0 else "noise", 390 + i, n) for i, n in enumerate(lens)]
    feats = [ob.featurize(w.copy()) for w in waves]
    Fmax = max(f.shape[0] for f in feats)
    batch = np.zeros((len(feats), Fmax, 80), np.float32)
    for i, f in enumerate(feats):
        batch[i, :f.shape[0]] = f
    res = eng.transcribe(waves, return_frames=True)
    post = {}
    for persistent in (True, False):
        eng.persistent_lstm = persistent
        try:
            post[persistent] = eng.posteriors(batch, [f.shape[0] for f in feats])
        finally:
            eng.persistent_lstm = True
    for i, f in enumerate(feats):
        probs = _oracle(cell, streaming, torch.from_numpy(f))[0].numpy()
        n = res.frame_lens[i]
        assert n == probs.shape[0]
        assert np.array_equal(probs.argmax(1), res.frame_ids[i, :n]), i
        score, _, toks = octc.greedy_decode(probs, vocab)
        assert toks == res.tokens[i] and abs(score - res.scores[i]) < 1e-3
        e = np.abs(post[True][i][:n] - probs).max()
        d = np.abs(post[True][i][:n] - post[False][i][:n]).max()
        report(f"ds2 {cell} {'uni' if streaming else 'bi'} utt {i}", oracle=e, tc_vs_step=d)
        assert e < 5e-5 and d < 5e-5


@pytest.mark.parametrize("cell", ["lstm", "gru"])
@pytest.mark.parametrize("persistent", [True, False])
def test_encode_chunk_walk_matches_golden(engines, cell, persistent):
    """``encode_chunk`` over the reference's frozen 67-frame window walk (ending in a short window): per-window frame ids
    bit-exact, top-8 posteriors within 5e-5, the carried h (and the LSTM's c) within 2e-4 of the reference's."""
    eng = engines(cell, True)
    z, meta = load_npz("deepspeech2_wide_golden.npz")
    m, = [m for m in meta if m["cell"] == cell and m.get("chunks")]
    assert m["wseed"] == WSEED[cell, True]
    fd = torch.from_numpy(z[m["name"] + "/feat"]).to(eng.device)
    top_p, top_i, want_ids, want_h = (z[m["name"] + k] for k in ("/top_p", "/top_i", "/ids", "/h"))
    want_c = z[m["name"] + "/c"] if cell == "lstm" else None
    eng.persistent_lstm = persistent
    try:
        st, row = eng.new_stream(), 0
        assert (st.c is None) == (cell == "gru")
        for k, (cur, n) in enumerate(z[m["name"] + "/windows"]):
            ids, maxp, probs = eng.encode_chunk(fd[cur:cur + n], st, want_probs=True)
            t = probs.shape[0]
            rows = slice(row, row + t)
            row += t
            assert t == subsampled_len(int(n))
            got = np.take_along_axis(probs.cpu().numpy(), top_i[rows].astype(np.int64), axis=1)
            assert np.abs(got - top_p[rows]).max() < 5e-5, k
            assert np.array_equal(ids.cpu().numpy(), want_ids[rows]), k
            h = torch.stack([st.hT[l, st.cur[l], 0, :, 0] for l in range(5)]).cpu().numpy()
            eh = np.abs(h - want_h[k]).max()
            ec = np.abs(st.c[:, 0].cpu().numpy() - want_c[k]).max() if want_c is not None else 0.0
            report(f"ds2 {cell} chunk {k} persistent={persistent}", h=eh, c=ec)
            assert eh < 2e-4 and ec < 2e-4, k
        assert row == want_ids.shape[0] and n < 67
    finally:
        eng.persistent_lstm = True


def _bits(t):
    return t.contiguous().view(torch.int32)


@pytest.mark.parametrize("cell", ["lstm", "gru"])
@pytest.mark.parametrize("slots", [8, 33])
@pytest.mark.parametrize("persistent", [True, False])
def test_pool_step_equals_single_stream(engines, cell, slots, persistent):
    """Every live slot of a ``DeepSpeech2StreamPool`` at H = 2048 equals ``encode_chunk`` on its own stream bit for bit
    (ids, max-prob, logits, every layer's h), with the step replayed from a CUDA graph; idle slots keep their state."""
    from masr_b200.stream_pool import DeepSpeech2StreamPool
    eng = engines(cell, True)
    dev = eng.device
    eng.persistent_lstm = persistent
    try:
        pool = DeepSpeech2StreamPool(eng, slots)
        live = sorted({0, 3, slots - 1} | ({31, 32} if slots > 32 else set()))
        feats = {s: torch.from_numpy(ob.featurize(make_audio("speech" if s % 2 == 0 else "noise", 900 + s, 16000 * 3)))
                 for s in live}
        single = {s: eng.new_stream() for s in live}
        for r in range(4):
            active = live if r != 1 else live[:2]
            batch = torch.zeros(slots, 67, 80, device=dev)
            nfr = [0] * slots
            for s in active:
                batch[s] = feats[s][r * 64:r * 64 + 67].to(dev)
                nfr[s] = 67
            st = pool.state
            idle = {s: [_bits(st.hT[l, st.cur[l], s // 32, :, s % 32]).clone() for l in range(5)] for s in live if s not in active}
            ids, maxp, tout = pool.step(batch, nfr)
            torch.cuda.synchronize()
            for s, before in idle.items():
                assert all(torch.equal(a, _bits(st.hT[l, st.cur[l], s // 32, :, s % 32])) for l, a in enumerate(before)), s
            for s in active:
                t = tout[s]
                sid, smp, _ = eng.encode_chunk(batch[s], single[s])
                assert torch.equal(ids[s, :t], sid) and torch.equal(_bits(maxp[s, :t]), _bits(smp)), (r, s)
                assert torch.equal(_bits(pool.b["logits"][s * 16:s * 16 + t, :V]), _bits(single[s].last_logits[:, :V])), (r, s)
                for l in range(5):
                    assert torch.equal(_bits(st.hT[l, st.cur[l], s // 32, :, s % 32]),
                                       _bits(single[s].hT[l, single[s].cur[l], 0, :, 0])), (r, s, l)
        assert pool._graph is not None
    finally:
        eng.persistent_lstm = True


# ---- MASRPredictor -------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def predictors(tmp_path_factory):
    """MASRPredictor over the streaming 2048-wide checkpoint of either cell (a plain state dict: the width and the cell type
    come from the weights), one per (cell, decoder); one cell's predictors are kept at a time."""
    from masr_b200.predict import MASRPredictor
    tmp = tmp_path_factory.mktemp("ds2wide")
    vp = str(tmp / "vocabulary.txt")
    synth.write_vocabulary(vp)
    cache = {}

    def get(cell, decoder="ctc_greedy"):
        if (cell, decoder) not in cache:
            for k in [k for k in cache if k[0] != cell]:
                del cache[k]
            torch.cuda.empty_cache()
            mp = str(tmp / f"ds2wide_{cell}.pt")
            if not os.path.exists(mp):
                torch.save(synth.to_torch(weights(cell, True)), mp)
            cfg = {"use_model": "deepspeech2", "streaming": True, "decoder": decoder,
                   "encoder_conf": {"num_rnn_layers": 5, "rnn_size": 2048, "use_gru": cell == "gru"},
                   "preprocess_conf": {"feature_method": "fbank", "n_mels": 80, "sample_rate": 16000, "use_dB_normalization": True,
                                       "target_dB": -20},
                   "dataset_conf": {"dataset_vocab": vp},
                   "ctc_beam_search_decoder_conf": {"alpha": ALPHA, "beta": BETA, "beam_size": 16, "cutoff_prob": 0.99,
                                                    "cutoff_top_n": 40, "language_model_path": "lm/none.klm"}}
            cache[cell, decoder] = MASRPredictor(configs=cfg, model_path=mp, use_gpu=True)
        return cache[cell, decoder]
    return get


@pytest.mark.parametrize("cell", ["lstm", "gru"])
def test_predictor_matches_reference_golden(predictors, cell):
    """``predict`` and ``predict_stream`` against the reference ``MASRPredictor``'s frozen whole-utterance result and PCM
    pushes, under both recurrence forms; a ``create_stream_pool`` slot reproduces the same pushes."""
    with open(os.path.join(GOLDEN, "predictor_golden_deepspeech2_wide.json"), encoding="utf-8") as f:
        g = json.load(f)
    assert g["hidden"] == H and g[cell]["wseed"] == WSEED[cell, True] and g[cell]["whole"]["text"]
    pred = predictors(cell)
    eng = pred.predictor
    assert eng.H == H and eng.w.cell == cell and eng.rnn_form == "seq_tc"
    x = make_audio(g["kind"], g["aseed"], g["samples"])
    pcm = (np.clip(x, -1, 1) * 32767).astype("<i2")
    push = g["push"]
    want = g[cell]

    def check(got):
        assert len(got) == len(want["pushes_pcm"])
        for r, w in zip(got, want["pushes_pcm"]):
            assert (r is None) == (w is None), (r, w)
            if r is not None:
                assert r["text"] == w["text"] and abs(r["score"] - w["score"]) < 1e-3, (r, w)

    for persistent in (True, False):
        eng.persistent_lstm = persistent
        try:
            whole = pred.predict(audio_data=x.copy())
            assert whole["text"] == want["whole"]["text"] and abs(whole["score"] - want["whole"]["score"]) < 1e-3
            pred.reset_stream()
            check([pred.predict_stream(audio_data=pcm[s:s + push].tobytes(), is_end=s + push >= len(pcm))
                   for s in range(0, len(pcm), push)])
            pred.reset_stream()
            sp = pred.create_stream_pool(2, max_frames=400)
            check([sp.push({1: pcm[s:s + push].tobytes()}, is_end=s + push >= len(pcm))[1] for s in range(0, len(pcm), push)])
            del sp
        finally:
            eng.persistent_lstm = True


@pytest.mark.parametrize("cell", ["lstm", "gru"])
@pytest.mark.parametrize("decoder", ["ctc_greedy", "ctc_beam_search"])
@pytest.mark.parametrize("slots", [8, 33])
@pytest.mark.parametrize("persistent", [True, False])
def test_stream_pool_equals_predict_stream(predictors, cell, decoder, slots, persistent):
    """A ``StreamPool`` of 8 or 33 slots over the 2048-wide model, greedy or prefix beam: four streams (one silent for a
    round, one slot reset and reused) in slots spread over both lane groups, push by push equal to ``predict_stream`` on
    each stream alone (greedy: identical results; beam: same text, score within 1e-3), under both recurrence forms."""
    from masr_b200.stream_pool import StreamPool
    pred = predictors(cell, decoder)
    eng = pred.predictor
    streams, schedule = _streams()
    where = {0: 0, 1: slots - 1, 2: 31 if slots > 32 else 3}         # the helper's slots 0, 1, 2 -> slots of this pool
    schedule = [{where[s]: i for s, i in rnd.items()} for rnd in schedule]
    eng.persistent_lstm = persistent
    try:
        want = _stream_reference(pred, streams)
        beam = pred._beam_conf if decoder == "ctc_beam_search" else None
        sp = StreamPool(eng, synth.vocabulary(), n_slots=slots, beam=beam, max_frames=400)
        got = _drive(sp, streams, schedule)
        assert sp.pool.use_graph and sp.pool._graph is not None
    finally:
        eng.persistent_lstm = True
    if beam is None:
        assert got == want
    else:
        _compare(got, want)
