"""The fp32 kernels of the chunk (``predict_stream``) path and the DeepSpeech2 front-end, and the CTC decode head of every
non-fused path, one C-ABI entry point at a time against float64 CPU references:

  masr_gemm_f32                 torch.nn.functional.linear + every epilogue, at the call sites of encode_chunk, the
                                DeepSpeech2 layer-0 input projection and the positional projection (bias NULL)
  masr_conv1_cmvn_relu_f32      GlobalCMVN + Conv2d(1, C, 3, 2) + ReLU (cmvn.py:29-31, subsampling.py:81-82)
  masr_conv2_s2_relu_f32        Conv2d(C, C, 3, 2) + ReLU as an implicit GEMM (subsampling.py:83-84)
  masr_ctc_frame_argmax_f32     CTCLoss.softmax + the first argmax of greedy_decoder (ctc.py:70, ctc_greedy_decoder.py:21)
  masr_ctc_greedy_collapse      greedy_decoder's collapse and score sum (ctc_greedy_decoder.py:23-30)
  masr_ctc_topk_f32 / _blank    the per-frame candidate pruning of the prefix beam search (cutoff_top_n, cutoff_prob)

Conventions of tests/kernel_contract.py: garbage past every valid length (+1e3 in the logit columns [V, ldl), so a read
past V wins every maximum), NaN-filled outputs with sentinel rows and columns, valid outputs finite.  Each docstring gives
the maximum error observed on an H100 80GB HBM3 (700 W power limit); the tolerances are at most about 4x that.  The
GEMM-like tolerances are multiples of the float32 dot-product error scale u * (sqrt(K) * sqrt(sum_k a_k^2 w_k^2) + |y|),
u = 2^-24, per output element.

The last section runs without a GPU: the launchers refuse bad arguments before anything is launched.
"""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from kernel_contract import GARBAGE, P, err, garbage, gemm_scale, nan, ratio, report, runtime, same

gpu = pytest.mark.gpu

U32 = 2.0 ** -24
EPI_BIAS, EPI_SILU, EPI_RELU, EPI_GLU, EPI_SCALE, EPI_RESIDUAL = range(6)


@pytest.fixture(scope="module")
def rt():
    return runtime()


def rup(n, m):
    return (n + m - 1) // m * m


def all_nan(t):
    return bool(torch.isnan(t.detach().float().cpu()).all())


def outside(shape, rows, cols):
    """Mask of everything outside [:rows, :cols] of a 2-D buffer."""
    m = torch.ones(shape, dtype=torch.bool)
    m[:rows, :cols] = False
    return m


def padded(x, tail, seed):
    """x flattened into a larger 1-D buffer whose `tail` extra elements hold garbage."""
    buf = garbage((x.numel() + tail,), seed)
    buf[:x.numel()] = x.reshape(-1)
    return buf


# ---- masr_gemm_f32 -----------------------------------------------------------------------------------------------------------

def _gemm_cases():
    """(tag, M, N, K, lda, ldc, alpha).  lda / ldc: "K" / "N" = production pitch, "+36" = a row pitch past K that is not a
    multiple of 16, "odd" = ldc % 4 == 1 (the scalar-store epilogue)."""
    cases = []
    for d in (256, 512):
        for M in (1, 5, 16):
            lda = "+36" if M == 5 else "K"
            cases += [("embed", M, d, 19 * d, lda, "N", math.sqrt(d)),     # Conv2dSubsampling4.out x sqrt(d), K = 19 d
                      ("ffn_w1", M, 2048, d, lda, "N", 0.5), ("ffn_w2", M, d, 2048, lda, "N", 0.5),
                      ("proj", M, d, d, lda, "N", 0.5), ("ctc_head", M, 4233, d, lda, "Vpad", 0.5)]
        cases += [("conv_glu", 30, 2 * d, d, "K", "N", 0.5),                 # lorder + chunk = 14 + 16 rows
                  ("pos_proj", 5000, d, d, "K", "N", 0.5)]                  # linear_pos over the 5000-row table
    cases += [("ds2_xproj", 150, 4096, 608, "+36", "N", 0.5), ("ds2_xproj", 2000, 4096, 608, "K", "N", 0.5),
              ("ds2_xproj_gru", 2000, 3072, 608, "K", "N", 0.5),
              ("tiles64", 1000, 2048, 256, "K", "N", 0.5), ("tiles128", 1056, 2048, 256, "K", "odd", 0.5)]
    cases += [("round1", 1, 256, 256, "K", "N", 0.25), ("round1", 130, 2048, 256, "+36", "odd", 0.25),
              ("round1", 77, 256, 2048, "K", "odd", 0.25), ("round1", 129, 4233, 256, "K", "Vpad", 0.25),
              ("round1", 300, 256, 4864, "K", "N", 0.25)]
    return cases


GEMM_CASES = _gemm_cases()
GEMM_RATIO_TOL = 8.0


def _gemm_reference(epi, y, s, R, alpha):
    """(reference, error bound) of one epilogue over float64 y = A.W^T + b and its error scale s."""
    if epi == EPI_BIAS:
        return y, s
    if epi == EPI_SILU:
        r = F.silu(y)
        return r, 1.1 * s + 8 * U32 * r.abs()
    if epi == EPI_RELU:
        return F.relu(y), s
    if epi == EPI_GLU:
        v, g = y[:, 0::2], y[:, 1::2]
        r = v * torch.sigmoid(g)
        return r, torch.sigmoid(g) * s[:, 0::2] + 0.25 * v.abs() * s[:, 1::2] + 8 * U32 * r.abs()
    if epi == EPI_SCALE:
        r = alpha * y
        return r, abs(alpha) * s + 2 * U32 * r.abs()
    r = R + alpha * y
    return r, abs(alpha) * s + 2 * U32 * r.abs()


@gpu
@pytest.mark.parametrize("tag,M,N,K,lda,ldc,alpha", GEMM_CASES,
                         ids=[f"{c[0]}-M{c[1]}-N{c[2]}-K{c[3]}" for c in GEMM_CASES])
def test_gemm_f32_float64(rt, tag, M, N, K, lda, ldc, alpha):
    """masr_gemm_f32, all six epilogues and bias NULL, against float64: the encode_chunk call sites at d = 256 and 512
    (M = 1, 5, 16; the embed at K = 19 d, 9728 for d = 512; the CTC head at N = V = 4233 with ldc = Vpad; the GLU at
    M = lorder + 16 = 30), the positional projection over 5000 rows, the DeepSpeech2 layer-0 input projection (K = 608),
    both sides of the 64 / 128 tile switch at 132 tiles (M = 1000 / 1056 at N = 2048), and the round-1 shapes.  A sits in a
    garbage-filled buffer (lda = K or K + 36), the residual in its own one (ldr = ldc + 12, garbage past N); C is NaN-filled
    with 3 sentinel rows and sentinel columns [N, ldc) (GLU: [N/2, ldc)) that must stay NaN.  RESIDUAL with C == residual
    equals the out-of-place result bit for bit.
    Observed max error (H100), in units of the float32 error scale: 3.7 (the DeepSpeech2 input projection, M = 150); 1.3 to
    2.8 at the chunk shapes; tolerance 8."""
    g = torch.Generator().manual_seed(M * 131 + N * 7 + K)
    lda = K + 36 if lda == "+36" else K
    ldc = {"N": rup(N, 4) + 8, "Vpad": rup(N, 16), "odd": N + 5}[ldc]
    ldr = ldc + 12
    A = torch.randn(M, K, generator=g)
    W = torch.randn(N, K, generator=g) / math.sqrt(K)
    b = torch.randn(N, generator=g)
    R = torch.randn(M, N, generator=g) * 2
    Abuf = garbage((M + 2, lda), 1)
    Abuf[:M, :K] = A
    Rbuf = garbage((M + 3, ldr), 2)
    Rbuf[:M, :N] = R
    Ad, Wd, bd, Rd = Abuf.to(rt.dev), W.to(rt.dev), padded(b, 8, 3).to(rt.dev), Rbuf.to(rt.dev)
    y0 = A.double() @ W.double().t()
    y = y0 + b.double()
    s, s0 = gemm_scale(A, W, y), gemm_scale(A, W, y0)

    def run(epi, bias=bd, residual=None, C=None, ldr_=ldr):
        C = nan((M + 3, ldc), rt.dev) if C is None else C
        rt.call("masr_gemm_f32", P(Ad), lda, P(Wd), P(bias), P(residual), ldr_, P(C), ldc, M, N, K, epi, alpha, rt.st())
        torch.cuda.synchronize()
        return C.cpu()

    res = {}
    outs = {}
    for epi in range(6):
        if epi == EPI_GLU and N % 4:
            continue
        C = run(epi, residual=Rd if epi == EPI_RESIDUAL else None)
        No = N // 2 if epi == EPI_GLU else N
        ref, bound = _gemm_reference(epi, y, s, R.double(), alpha)
        res[f"epi{epi}"] = ratio(C[:M, :No], ref, bound + 1e-30)
        assert all_nan(C[outside(C.shape, M, No)]), f"epilogue {epi} wrote outside [M, N)"
        outs[epi] = C
    C = run(EPI_BIAS, bias=None)
    res["nobias"] = ratio(C[:M, :N], y0, s0 + 1e-30)
    assert all_nan(C[outside(C.shape, M, N)])
    # in place: residual == C (the residual stream x of encode_chunk), ldr = ldc
    Cx = nan((M + 3, ldc), rt.dev)
    Cx[:M, :N] = R.to(rt.dev)
    Cx = run(EPI_RESIDUAL, residual=Cx, C=Cx, ldr_=ldc)
    assert same(Cx, outs[EPI_RESIDUAL]), "in-place RESIDUAL differs from the out-of-place result"
    assert torch.equal(Rd.cpu(), Rbuf) and torch.equal(Ad.cpu(), Abuf), "an input buffer was written"
    report(f"gemm_f32 {tag} M={M} N={N} K={K} lda={lda} ldc={ldc}", **res)
    assert max(res.values()) < GEMM_RATIO_TOL, res


@gpu
@pytest.mark.parametrize("d", [256, 512])
@pytest.mark.parametrize("M", [1, 5, 16])
def test_gemm_f32_kv_cache_append(rt, d, M):
    """The k|v projection of encode_chunk (engine.py:1141): W points d rows into the packed [3d, d] q|k|v weight, the bias d
    entries into the packed bias, and C at row cache_start + cache_len of the [cap, 2d] attention cache (ldc = 2d).  The
    rows around the target keep their NaN.  Observed max error (H100): 2.5 error scales (d = 512, M = 16); tolerance 8."""
    g = torch.Generator().manual_seed(d + M)
    cap, start, t1 = 64, 3, 11
    A = torch.randn(M, d, generator=g)
    wqkv = torch.randn(3 * d, d, generator=g) / math.sqrt(d)
    bqkv = torch.randn(3 * d, generator=g)
    Ad, wd, bd = A.to(rt.dev), wqkv.to(rt.dev), bqkv.to(rt.dev)
    kv = nan((cap, 2 * d), rt.dev)
    row = start + t1
    rt.call("masr_gemm_f32", P(Ad), d, wd.data_ptr() + 4 * d * d, bd.data_ptr() + 4 * d, None, 0, kv.data_ptr() + 4 * row * 2 * d,
            2 * d, M, 2 * d, d, EPI_BIAS, 1.0, rt.st())
    torch.cuda.synchronize()
    kv = kv.cpu()
    W = wqkv[d:]
    y = A.double() @ W.double().t() + bqkv[d:].double()
    r = ratio(kv[row:row + M], y, gemm_scale(A, W, y))
    assert all_nan(kv[:row]) and all_nan(kv[row + M:]), "k|v rows written outside the appended chunk"
    report(f"gemm_f32 k|v append d={d} M={M}", kv=r)
    assert r < GEMM_RATIO_TOL


# ---- convolution subsampling ----------------------------------------------------------------------------------------------

CONV_CASES = ([(C, Fm, B, 80, True) for C in (32, 256, 512) for Fm in (7, 9, 67) for B in (1, 3)]
              + [(32, 998, 3, 80, True), (256, 998, 1, 80, True), (512, 998, 1, 80, True)]
              + [(32, 67, 3, 83, True), (256, 130, 1, 83, True), (256, 67, 3, 80, False)])
CONV1_RATIO_TOL = 8.0
CONV2_RATIO_TOL = 8.0


def conv_ratio(out, x, w, b, K):
    """max |out - relu(conv(x))| in units of the float32 dot-product error scale of the convolution (stride 2)."""
    pre = F.conv2d(x, w, b, stride=2)
    s = U32 * (math.sqrt(K) * torch.sqrt(F.conv2d(x * x, w * w, stride=2)) + pre.abs())
    return ratio(out, F.relu(pre).permute(0, 2, 3, 1), s.permute(0, 2, 3, 1) + 1e-30)


def _check_subsampling(rt, C, Fm, B, idim, cmvn):
    """conv-1 then conv-2 on one seeded problem against float64; returns the two errors in error scales.  feats, mean /
    istd and both weights sit in buffers with garbage tails; conv-2 reads its input from a copy of conv-1's output with a
    garbage tail, so each kernel is measured against float64 of its own input.  Both outputs are NaN-filled past their
    extent and must stay so."""
    g = torch.Generator().manual_seed(C * 1000 + Fm * 10 + B + idim)
    feats = torch.randn(B, Fm, idim, generator=g) * 3 + 20
    mean = torch.randn(idim, generator=g) + 20
    istd = torch.rand(idim, generator=g) * 0.3 + 0.2
    w1, b1 = torch.randn(C, 1, 3, 3, generator=g) / 3, torch.randn(C, generator=g) / 3
    w2, b2 = torch.randn(C, C, 3, 3, generator=g) / math.sqrt(9 * C), torch.randn(C, generator=g) / math.sqrt(9 * C)
    F1, W1 = (Fm - 1) // 2, (idim - 1) // 2
    T2, W2 = (F1 - 1) // 2, (W1 - 1) // 2
    n1, n2 = B * F1 * W1 * C, B * T2 * W2 * C
    fd, md, sd = padded(feats, 3 * idim, 1).to(rt.dev), padded(mean, 16, 2).to(rt.dev), padded(istd, 16, 3).to(rt.dev)
    w1d, b1d = padded(w1, 64, 4).to(rt.dev), padded(b1, 16, 5).to(rt.dev)
    w2d, b2d = padded(w2.permute(0, 2, 3, 1), 64, 6).to(rt.dev), padded(b2, 16, 7).to(rt.dev)
    c1 = nan((n1 + 4 * C,), rt.dev)
    rt.call("masr_conv1_cmvn_relu_f32", P(fd), P(md) if cmvn else None, P(sd) if cmvn else None, P(w1d), P(b1d), P(c1),
            B, Fm, idim, F1, W1, C, rt.st())
    c1in = padded(c1[:n1].cpu(), 4 * C, 8).to(rt.dev)
    out = nan((n2 + 3 * C,), rt.dev)
    rt.call("masr_conv2_s2_relu_f32", P(c1in), P(w2d), P(b2d), P(out), B, F1, W1, T2, W2, C, rt.st())
    torch.cuda.synchronize()
    c1, out = c1.cpu(), out.cpu()
    assert all_nan(c1[n1:]) and all_nan(out[n2:]), "a convolution wrote past its output"
    x = feats.double()
    if cmvn:
        x = (x - mean.double()) * istd.double()
    e1 = conv_ratio(c1[:n1].view(B, F1, W1, C), x.unsqueeze(1), w1.double(), b1.double(), 9)
    c1v = c1[:n1].view(B, F1, W1, C).permute(0, 3, 1, 2).double()
    e2 = conv_ratio(out[:n2].view(B, T2, W2, C), c1v, w2.double(), b2.double(), 9 * C)
    report(f"conv subsampling C={C} Fm={Fm} B={B} idim={idim} cmvn={cmvn}", conv1=e1, conv2=e2)
    return e1, e2


@gpu
@pytest.mark.parametrize("C,Fm,B,idim,cmvn", CONV_CASES)
def test_subsampling_convs_float64(rt, C, Fm, B, idim, cmvn):
    """masr_conv1_cmvn_relu_f32 and masr_conv2_s2_relu_f32 against float64 conv2d (stride 2) + ReLU on the CMVN-ed input:
    C = 32 (DeepSpeech2), 256 and 512 (Conformer); Fm = 7 (the smallest chunk), 9, 67 (the decoding window) and 998, so F1 =
    3, 4, 33, 498 rows (not all multiples of the 4-row conv-1 tile); idim 80 and 83 (W1 = 39 / 41); CMVN NULL once.
    Observed max error (H100), in error scales: conv-1 2.8, conv-2 2.5 (C = 256 / 512, Fm = 998); tolerances 8 / 8."""
    e1, e2 = _check_subsampling(rt, C, Fm, B, idim, cmvn)
    assert e1 < CONV1_RATIO_TOL and e2 < CONV2_RATIO_TOL


@gpu
def test_subsampling_convs_round1(rt):
    """The round-1 shape, B = 2 utterances of 47 frames at C = 256 (F1 = 23 rows: not a multiple of the 4-row conv-1
    tile), under the same float64 and sentinel checks.  Observed max error (H100), in error scales: conv-1 2.3, conv-2 1.8;
    tolerances 8 / 7."""
    e1, e2 = _check_subsampling(rt, 256, 47, 2, 80, True)
    assert e1 < CONV1_RATIO_TOL and e2 < 7.0


def _front_reference(feats, mean, istd, w1, b1, w2, b2):
    """float64 GlobalCMVN -> Conv2d -> ReLU -> Conv2d -> ReLU -> x.transpose(1, 2).reshape(b, t, c * f), as the reference
    modules flatten (subsampling.py:110, deepspeech2/conv.py)."""
    x = ((feats.double() - mean.double()) * istd.double()).unsqueeze(1)
    x = F.relu(F.conv2d(x, w1.double(), b1.double(), stride=2))
    x = F.relu(F.conv2d(x, w2.double(), b2.double(), stride=2))
    b, c, t, f = x.shape
    return x.transpose(1, 2).reshape(b, t, c * f)


def _front_kernels(rt, w, feats, B, Fm, C):
    """conv-1 -> conv-2 through the packed weights -> the [B * T2, 19 C] conv-2 output on the device."""
    idim = feats.shape[2]
    F1, W1 = (Fm - 1) // 2, (idim - 1) // 2
    T2, W2 = (F1 - 1) // 2, (W1 - 1) // 2
    fd = feats.contiguous().to(rt.dev)
    c1 = nan((B * F1 * W1 * C,), rt.dev)
    rt.call("masr_conv1_cmvn_relu_f32", P(fd), P(w.cmvn_mean), P(w.cmvn_istd), P(w.conv1_w), P(w.conv1_b), P(c1), B, Fm, idim,
            F1, W1, C, rt.st())
    c2 = nan((B * T2, W2 * C), rt.dev)
    rt.call("masr_conv2_s2_relu_f32", P(c1), P(w.conv2_w), P(w.conv2_b), P(c2), B, F1, W1, T2, W2, C, rt.st())
    return c2, B * T2, W2 * C


@gpu
@pytest.mark.parametrize("gru", [False, True])
def test_deepspeech2_front_and_input_projection(rt, gru):
    """conv-1 -> conv-2 -> the layer-0 input projection (masr_gemm_f32, K = 19 * 32 = 608) with the weights
    pack_deepspeech2 builds from a synth state dict (weight_ih_l0 with its columns permuted to the channels-last conv
    output), against float64 Conv2d -> ReLU -> Conv2d -> ReLU -> flatten -> Linear(weight_ih_l0, bias_ih_l0 + bias_hh_l0)
    (GRU: + bias_hh_l0 of the r and z gates only; b_hn stays inside the cell).  Pins the permutation and the kernels'
    layouts together.  Observed max error (H100): 2.6e-7 (|gx| <= 0.41); tolerance 1e-6."""
    from masr_b200 import synth
    from masr_b200.deepspeech2 import pack_deepspeech2
    sd = synth.to_torch(synth.deepspeech2_state_dict(3, layers=1, use_gru=gru))
    w = pack_deepspeech2(sd, rt.dev)
    B, Fm = 2, 150
    g = torch.Generator().manual_seed(4)
    feats = torch.randn(B, Fm, 80, generator=g) * 3.1 + 20.6
    c2, M, K = _front_kernels(rt, w, feats, B, Fm, 32)
    GH = w.rnn[0]["wih"][0].shape[0]
    gx = nan((M + 2, GH + 8), rt.dev)
    rt.call("masr_gemm_f32", P(c2), K, P(w.rnn[0]["wih"][0]), P(w.rnn[0]["bias"][0]), None, 0, P(gx), GH + 8, M, GH, K, EPI_BIAS,
            1.0, rt.st())
    torch.cuda.synchronize()
    gx = gx.cpu()
    p = "encoder.rnns.0.rnn." + ("rnn." if gru else "")
    x = _front_reference(feats, sd["encoder.global_cmvn.mean"], sd["encoder.global_cmvn.istd"], sd["encoder.conv.conv.0.weight"],
                         sd["encoder.conv.conv.0.bias"], sd["encoder.conv.conv.2.weight"], sd["encoder.conv.conv.2.bias"])
    bias = sd[p + "bias_ih_l0"].double() + sd[p + "bias_hh_l0"].double()
    if gru:
        bias[2 * GH // 3:] -= sd[p + "bias_hh_l0"].double()[2 * GH // 3:]
    ref = x.reshape(M, K) @ sd[p + "weight_ih_l0"].double().t() + bias
    e = err(gx[:M, :GH], ref)
    assert all_nan(gx[outside(gx.shape, M, GH)])
    report(f"deepspeech2 front + input projection gru={gru}", gx=e, max_abs=ref.abs().max().item())
    assert e < 1e-6


@gpu
@pytest.mark.parametrize("d", [256, 512])
def test_conformer_front_and_embed(rt, d):
    """conv-1 -> conv-2 -> the embed GEMM (BIAS_SCALE, alpha = sqrt(d)) with the weights pack_conformer builds from a synth
    state dict (embed.out.0.weight with its columns permuted to the channels-last conv output), against float64
    Conv2dSubsampling4 (Conv2d -> ReLU -> Conv2d -> ReLU -> flatten -> Linear) x sqrt(d) (embedding.py:98).
    Observed max error (H100): 1.4e-5 at d = 256 (|x| <= 7.2), 2.8e-5 at d = 512 (|x| <= 10.3); tolerance 5e-5 * d / 256."""
    from masr_b200 import synth
    from masr_b200.weights import pack_conformer
    sd = synth.to_torch(synth.conformer_state_dict(5, output_size=d, attention_heads=d // 64, num_blocks=1))
    w = pack_conformer(sd, rt.dev, max_len=64)
    B, Fm = 2, 67
    g = torch.Generator().manual_seed(6)
    feats = torch.randn(B, Fm, 80, generator=g) * 3.1 + 20.6
    c2, M, K = _front_kernels(rt, w, feats, B, Fm, d)
    x_out = nan((M + 2, d + 8), rt.dev)
    rt.call("masr_gemm_f32", P(c2), K, P(w.embed_w), P(w.embed_b), None, 0, P(x_out), d + 8, M, d, K, EPI_SCALE, math.sqrt(d),
            rt.st())
    torch.cuda.synchronize()
    x_out = x_out.cpu()
    x = _front_reference(feats, sd["encoder.global_cmvn.mean"], sd["encoder.global_cmvn.istd"], sd["encoder.embed.conv.0.weight"],
                         sd["encoder.embed.conv.0.bias"], sd["encoder.embed.conv.2.weight"], sd["encoder.embed.conv.2.bias"])
    ref = (x.reshape(M, K) @ sd["encoder.embed.out.0.weight"].double().t() + sd["encoder.embed.out.0.bias"].double()) * math.sqrt(d)
    e = err(x_out[:M, :d], ref)
    assert all_nan(x_out[outside(x_out.shape, M, d)])
    report(f"conformer front + embed d={d}", x=e, max_abs=ref.abs().max().item())
    assert e < 5e-5 * d / 256


# ---- CTC frame argmax ------------------------------------------------------------------------------------------------------

def _argmax_logits(V, seed):
    """[M, V] float32 logits: random rows, then rows with exact ties (ids i and i + 256: one thread's stride; 250 and 260:
    the lower id in the higher warp; V // 2 and V - 1), a constant row, an all-negative row and a row near +200 (exp
    overflows float32 without the max subtraction)."""
    g = torch.Generator().manual_seed(seed)
    L = torch.randn(40, V, generator=g) * 3
    L[::3, 0] += 6.0                                            # blank-dominated frames, as the CTC head produces
    r = 30
    for i, j in ((3, 259), (250, 260), (V // 2, V - 1), (0, 1), (31, 32), (255, 256)):
        if j < V and i != j:
            L[r] = torch.randn(V, generator=g)
            L[r, i] = L[r, j] = 9.0
            r += 1
    L[36] = 0.5                                                 # constant: the first id
    L[37] = -torch.rand(V, generator=g) * 50 - 100             # every logit negative
    L[38] = torch.randn(V, generator=g) * 2 + 200
    return L


ARGMAX_V = [1, 2, 29, 255, 256, 257, 4233, 5120, 6000]
ARGMAX_CASES = sorted({(V, ldl) for V in ARGMAX_V for ldl in (V, rup(V, 16), V + 37)})
PROB_TOL = 4e-7


@gpu
@pytest.mark.parametrize("V,ldl", ARGMAX_CASES)
def test_ctc_frame_argmax_float64(rt, V, ldl):
    """masr_ctc_frame_argmax_f32 against float64: ids equal numpy's first argmax exactly (ties inside one thread's stride,
    across warps, at V - 1); maxp and probs against the float64 softmax.  V from 1 to 6000 (past the 5120 of the top-k
    kernel: this one has no vocabulary limit) at ldl = V, round-up-16(V) and V + 37, with +1e3 in [V, ldl).  probs is
    written once into a NaN-filled [M + 2, V + 5] buffer, once not at all (NULL): ids / maxp identical.  ids / maxp past M
    and probs past V keep their sentinels.  Observed max error (H100), probs and maxp: 2.5e-7 (V = 256, ldl = 293);
    tolerance 4e-7."""
    L = _argmax_logits(V, V * 7 + ldl)
    M = L.shape[0]
    buf = garbage((M + 2, max(ldl, V)), V)
    buf[:M, :V] = L
    buf[:M, V:] = GARBAGE
    Ld = buf.to(rt.dev)
    ldp = V + 5
    outs = []
    for with_probs in (True, False):
        ids = torch.full((M + 3,), -7, dtype=torch.int32, device=rt.dev)
        mp = nan((M + 3,), rt.dev)
        probs = nan((M + 2, ldp), rt.dev) if with_probs else None
        rt.call("masr_ctc_frame_argmax_f32", P(Ld), ldl, M, V, P(ids), P(mp), P(probs), ldp, rt.st())
        torch.cuda.synchronize()
        outs.append((ids.cpu(), mp.cpu(), None if probs is None else probs.cpu()))
    (ids, mp, probs), (ids2, mp2, _) = outs
    assert torch.equal(ids, ids2) and same(mp, mp2), "probs = NULL changed ids / maxp"
    assert torch.all(ids[M:] == -7) and all_nan(mp[M:]), "ids / maxp written past M"
    assert all_nan(probs[outside(probs.shape, M, V)]), "probs written past [M, V)"
    ref_ids = L.numpy().astype(np.float64).argmax(1)
    assert np.array_equal(ids[:M].numpy(), ref_ids), np.nonzero(ids[:M].numpy() != ref_ids)
    if V > 259:
        assert ref_ids[30] == 3 and ref_ids[31] == 250
    p = torch.softmax(L.double(), 1)
    e_p, e_mp = err(probs[:M, :V], p), err(mp[:M], p.max(1).values)
    report(f"ctc_frame_argmax V={V} ldl={ldl}", probs=e_p, maxp=e_mp)
    assert e_p < PROB_TOL and e_mp < PROB_TOL


@gpu
def test_ctc_argmax_then_collapse_round1(rt):
    """The round-1 case end to end: 3 x 40 frames of V = 4233 (blank-heavy logits, a tie 7 / 100 -> 7 and a repeated
    frame), argmax -> collapse (lens 40, 17, 1) against float64 and oracle/ctc.py, psum bit-exact to the float32
    left-to-right sum."""
    from oracle import ctc as octc
    g = torch.Generator().manual_seed(5)
    B, T, V = 3, 40, 4233
    lens = [40, 17, 1]
    logits = torch.randn(B * T, V, generator=g) * 3
    logits[:, 0] += 6.0
    logits[5, 100] = logits[5, 7] = 50.0
    logits[6] = logits[5]
    ldl = rup(V, 16)
    L = torch.full((B * T, ldl), GARBAGE)
    L[:, :V] = logits
    Ld = L.to(rt.dev)
    ids = torch.full((B * T,), -7, dtype=torch.int32, device=rt.dev)
    mp = nan((B * T,), rt.dev)
    rt.call("masr_ctc_frame_argmax_f32", P(Ld), ldl, B * T, V, P(ids), P(mp), None, V, rt.st())
    ld = torch.tensor(lens, dtype=torch.int32, device=rt.dev)
    tok = torch.full((B, T), -7, dtype=torch.int32, device=rt.dev)
    nt, pc = (torch.full((B,), -7, dtype=torch.int32, device=rt.dev) for _ in range(2))
    ps = nan((B,), rt.dev)
    rt.call("masr_ctc_greedy_collapse", P(ids), P(mp), T, P(ld), B, 0, P(tok), T, P(nt), P(ps), P(pc), rt.st())
    torch.cuda.synchronize()
    ref_ids = logits.double().numpy().argmax(1)
    assert np.array_equal(ids.cpu().numpy(), ref_ids) and ref_ids[5] == 7 == ref_ids[6]
    assert err(mp, torch.softmax(logits.double(), 1).max(1).values) < PROB_TOL
    mph, tok = mp.cpu().numpy(), tok.cpu()
    for b, n in enumerate(lens):
        fr = ref_ids[b * T: b * T + n]
        k = int(nt[b])
        assert tok[b, :k].tolist() == octc.collapse(fr) and torch.all(tok[b, k:] == -7)
        acc = np.float32(0)
        for t in range(n):
            if fr[t] != 0:
                acc = np.float32(acc + mph[b * T + t])
        assert int(pc[b]) == int((fr != 0).sum()) and ps[b].item() == float(acc)


# ---- CTC greedy collapse ---------------------------------------------------------------------------------------------------

def collapse_reference(fr, blank):
    out, prev = [], None
    for c in fr:
        if c != prev and c != blank:
            out.append(int(c))
        prev = c
    return out


def _check_collapse(rt, ids, mp, lens, blank, V):
    """masr_ctc_greedy_collapse over utterance b = frames ids[b, :lens[b]] / mp[b, :lens[b]] of [B, T] arrays, in a
    [B, T + 3] layout whose rows past lens[b] hold non-blank garbage ids (>= V) and NaN max-probs: a read there changes the
    tokens or makes psum NaN.  Tokens must equal the collapse of the frame ids with the sentinel untouched past ntok,
    pcount the non-blank count and psum the float32 left-to-right sum bit for bit; outputs past B keep their sentinels."""
    B, T = ids.shape
    bstride = T + 3
    rng = np.random.default_rng(V + blank)
    idb = rng.integers(V, 2 * V, (B, bstride)).astype(np.int32)
    mpb = np.full((B, bstride), np.nan, np.float32)
    for b, n in enumerate(lens):
        idb[b, :n], mpb[b, :n] = ids[b, :n], mp[b, :n]
    d = lambda a: torch.from_numpy(a).to(rt.dev)
    idd, mpd, ld = d(idb), d(mpb), d(np.asarray(lens, np.int32))
    tok_stride = T + 5
    tok = torch.full((B, tok_stride), -7, dtype=torch.int32, device=rt.dev)
    nt, pc = (torch.full((B + 2,), -7, dtype=torch.int32, device=rt.dev) for _ in range(2))
    ps = nan((B + 2,), rt.dev)
    rt.call("masr_ctc_greedy_collapse", P(idd), P(mpd), bstride, P(ld), B, blank, P(tok), tok_stride, P(nt), P(ps), P(pc), rt.st())
    torch.cuda.synchronize()
    tok, nt, ps, pc = tok.cpu().numpy(), nt.cpu().numpy(), ps.cpu().numpy(), pc.cpu().numpy()
    assert np.all(nt[B:] == -7) and np.all(pc[B:] == -7) and np.isnan(ps[B:]).all()
    for b, n in enumerate(lens):
        fr = ids[b, :n]
        want = collapse_reference(fr, blank)
        assert nt[b] == len(want) and tok[b, :nt[b]].tolist() == want, b
        assert np.all(tok[b, nt[b]:] == -7), f"tokens written past ntok in utterance {b}"
        acc = np.float32(0)
        for t in range(n):
            if fr[t] != blank:
                acc = np.float32(acc + mp[b, t])
        assert pc[b] == int((fr != blank).sum()), b
        assert ps[b].tobytes() == acc.tobytes(), (b, ps[b], acc)


@gpu
@pytest.mark.parametrize("blank_kind", ["zero", "five", "last"])
def test_ctc_greedy_collapse_ragged(rt, blank_kind):
    """masr_ctc_greedy_collapse over B = 300 utterances with blank = 0, 5 and V - 1 (V = 4233; with blank 5 or V - 1, id 0
    is an ordinary token): lengths 0, 1, the 256-frame tile borders (255 / 256 / 257, 511 / 512 / 513, 768), 700 and 1500
    with a run across the first tile border and a 30-frame blank run, the rest random; checks of _check_collapse."""
    V = 4233
    blank = {"zero": 0, "five": 5, "last": V - 1}[blank_kind]
    rng = np.random.default_rng(9 + blank)
    fixed = [0, 1, 255, 256, 257, 511, 512, 513, 768, 700, 1500, 0, 2]
    B = 300
    lens = fixed + rng.integers(0, 1600, B - len(fixed)).tolist()
    T = max(lens)
    symbols = np.array([blank] + [s for s in (0, 1, 2, 3, 4) if s != blank][:3], np.int32)   # few symbols -> many repeats
    ids = symbols[rng.integers(0, 4, (B, T))]
    mp = rng.random((B, T)).astype(np.float32)
    ids[9, 250:262] = symbols[3]                              # a run across the first tile border (length 700)
    ids[10, 500:530] = blank                                  # (length 1500)
    _check_collapse(rt, ids, mp, lens, blank, V)


@gpu
def test_ctc_greedy_collapse_round1(rt):
    """The round-1 case, blank 0: lengths 0, 1, 255, 256, 257, 700 and 1500 over ids 0..3 (many repeats and blanks), a
    run of one id across the first 256-frame tile border (utterance 5) and a 30-frame blank run (utterance 6), with the
    garbage, sentinel and bit-exact psum checks of _check_collapse."""
    rng = np.random.default_rng(9)
    lens = [0, 1, 255, 256, 257, 700, 1500]
    B, T = len(lens), max(lens)
    ids = rng.integers(0, 4, size=(B, T)).astype(np.int32)
    ids[5, 250:262] = 3
    ids[6, 500:530] = 0
    mp = rng.random((B, T)).astype(np.float32)
    _check_collapse(rt, ids, mp, lens, 0, 4233)


# ---- CTC top-k candidates --------------------------------------------------------------------------------------------------

TOPK_V = [1, 2, 29, 39, 40, 41, 256, 257, 4233, 5119, 5120]
TOPK_N = [1, 7, 40]
TOPK_CUT = [0.0, 0.5, 0.99, 1.0]
CUT_EPS = 1e-5
LN_MIN_NORMAL = math.log(2.0 ** -126)
LOGP_TOL = 1.2e-5


def _topk_logits(V, seed):
    """[M, V] float32 logits: random rows at three temperatures, a constant row, plateaus of equal logits that straddle
    every top-n boundary (3 distinct leaders, then up to 60 tied ids scattered over threads and warps), a tied plateau at
    the top, and peaky rows (a few logits near 0, the rest 100..200 below: posteriors under 2^-126)."""
    g = torch.Generator().manual_seed(seed)
    rows = [torch.randn(V, generator=g) * s for s in (1.0, 3.0, 3.0, 6.0, 10.0)]
    rows.append(torch.full((V,), 0.25))
    for lead in (3, 0):
        x = torch.randn(V, generator=g) - 5.0
        perm = torch.randperm(V, generator=g)
        plateau = perm[lead:lead + 60]
        x[plateau] = 3.0
        for k in range(min(lead, V)):
            x[perm[k]] = 5.0 - 0.5 * k
        rows.append(x)
    for k in range(6):
        x = -100.0 - torch.rand(V, generator=g) * 100
        top = torch.randperm(V, generator=g)[:min(V, 2 + k)]
        x[top] = -torch.rand(len(top), generator=g) * (1 + k)
        rows.append(x)
    return torch.stack(rows)


def _accepted_counts(cum, n_max, cut):
    """Counts the cumulative rule allows: the smallest k with cum[k] >= cut (else n_max), where a float64 cumulative sum
    within CUT_EPS of cut may fall on either side in float32."""
    ok = set()
    for k in range(1, n_max + 1):
        if (k == 1 or cum[k - 1] < cut + CUT_EPS) and (k == n_max or cum[k] >= cut - CUT_EPS):
            ok.add(k)
    return ok


@gpu
@pytest.mark.parametrize("V", TOPK_V)
def test_ctc_topk_float64(rt, V):
    """masr_ctc_topk_f32 and masr_ctc_topk_blank_f32 (blank 0 and V - 1) against float64 at top_n 1, 7, 40 and cutoff_prob
    0, 0.5, 0.99, 1: candidate ids in float64 rank order (probability descending, id ascending on ties: the plateaus make
    every top-n boundary a tie), cand_cnt by the cumulative rule (either side where the float64 sum is within 1e-5 of
    cutoff_prob), cand_logp and blank_logp against float64 log-softmax wherever p >= 2^-126, blank_logp == cand_logp bit
    for bit when blank is a candidate.  V up to the 5120 register limit, ldl = V + 37 with +1e3 in [V, ldl).  Slots past
    cand_cnt, rows past M keep their sentinels.
    Below 2^-126 (peaky rows at cutoff_prob 1) the float32 posterior is subnormal or zero: the kernel's logarithm there is
    pinned as it is, finite or -inf, never NaN and never above ln 2^-126 + 1.
    Observed max error (H100): cand_logp 3.4e-6 (V = 41), blank_logp 3.5e-6 (V = 257); tolerance 1.2e-5."""
    L = _topk_logits(V, V)
    M = L.shape[0]
    ldl = V + 37
    buf = garbage((M + 2, ldl), V)
    buf[:M, :V] = L
    buf[:M, V:] = GARBAGE
    Ld = buf.to(rt.dev)
    x = L.double()
    lp = torch.log_softmax(x, 1)
    p = lp.exp()
    order = [np.lexsort((np.arange(V), -x[m].numpy())) for m in range(M)]
    e_lp = e_blank = 0.0
    tiny = ambiguous = 0
    for top_n in TOPK_N:
        n_max = min(top_n, V)
        for cut in TOPK_CUT:
            for blank in (None, 0, V - 1):
                if blank == V - 1 and V == 1:
                    continue
                cid = torch.full((M + 2, 40), -7, dtype=torch.int32, device=rt.dev)
                clp = nan((M + 2, 40), rt.dev)
                cnt = torch.full((M + 2,), -7, dtype=torch.int32, device=rt.dev)
                blp = nan((M + 2,), rt.dev)
                if blank is None:
                    rt.call("masr_ctc_topk_f32", P(Ld), ldl, M, V, top_n, cut, P(cid), P(clp), P(cnt), rt.st())
                else:
                    rt.call("masr_ctc_topk_blank_f32", P(Ld), ldl, M, V, top_n, cut, blank, P(cid), P(clp), P(cnt), P(blp), rt.st())
                torch.cuda.synchronize()
                cid, clp, cnt, blp = cid.cpu(), clp.cpu(), cnt.cpu(), blp.cpu()
                assert torch.all(cid[M:] == -7) and all_nan(clp[M:]) and torch.all(cnt[M:] == -7) and all_nan(blp[M:])
                for m in range(M):
                    n = int(cnt[m])
                    want = order[m][:n_max]
                    cum = np.concatenate([[0.0], np.cumsum(p[m].numpy()[want])])       # cum[k]: the first k candidates
                    ok = _accepted_counts(cum, n_max, cut)
                    ambiguous += len(ok) > 1
                    assert n in ok, (top_n, cut, m, n, sorted(ok))
                    assert cid[m, :n].tolist() == want[:n].tolist(), (top_n, cut, m)
                    assert torch.all(cid[m, n:] == -7) and all_nan(clp[m, n:]), "slots past cand_cnt written"
                    got, ref = clp[m, :n].double(), lp[m, want[:n]]
                    assert not torch.isnan(got).any()
                    normal = ref >= LN_MIN_NORMAL
                    if normal.any():
                        e_lp = max(e_lp, err(got[normal], ref[normal]))
                    if (~normal).any():
                        sub = got[~normal]
                        tiny += int((~normal).sum())
                        assert torch.all(torch.isfinite(sub) | (sub == -math.inf)) and torch.all(sub <= LN_MIN_NORMAL + 1)
                    if blank is not None:
                        bl = blp[m].double()
                        assert not math.isnan(bl)
                        if lp[m, blank] >= LN_MIN_NORMAL:
                            e_blank = max(e_blank, abs(bl.item() - lp[m, blank].item()))
                        else:
                            assert bl <= LN_MIN_NORMAL + 1
                        hit = (cid[m, :n] == blank).nonzero()
                        if len(hit):
                            assert torch.equal(blp[m:m + 1], clp[m, hit[0]]), "blank_logp differs from its cand_logp"
    report(f"ctc_topk V={V}", cand_logp=e_lp, blank_logp=e_blank, subnormal_candidates=tiny, ambiguous_counts=ambiguous)
    assert e_lp < LOGP_TOL and e_blank < LOGP_TOL


# ---- argument checks (CPU: refused before any launch) ------------------------------------------------------------------------

@pytest.fixture(scope="module")
def lib():
    from masr_b200 import build, _lib
    build.build()                      # nvcc cross-compiles sm_90a without a GPU
    return _lib.load()


# fake device addresses: never dereferenced, every call below fails its argument checks first
A16, W16, C16 = 0x10000, 0x20000, 0x30000


def refused(name, *args, match):
    from masr_b200._lib import MasrB200Error, call
    with pytest.raises(MasrB200Error, match=match):
        call(name, *args)


def test_gemm_rejects_bad_arguments(lib):
    refused("masr_gemm_f32", A16, 24, W16, None, None, 0, C16, 4, 4, 4, 24, EPI_BIAS, 1.0, None,
            match="K=24 must be a positive multiple of 16")
    refused("masr_gemm_f32", A16, 24, W16, None, None, 0, C16, 4, 4, 4, 16, EPI_RESIDUAL, 1.0, None,
            match="residual epilogue needs a residual")
    refused("masr_gemm_f32", A16, 18, W16, None, None, 0, C16, 4, 4, 4, 16, EPI_BIAS, 1.0, None, match="lda=18 must be a multiple of 4")
    refused("masr_gemm_f32", A16 + 4, 16, W16, None, None, 0, C16, 4, 4, 4, 16, EPI_BIAS, 1.0, None,
            match="A and W must be 16-byte aligned")
    refused("masr_gemm_f32", A16, 16, W16, None, None, 0, C16, 4, 4, 6, 16, EPI_GLU, 1.0, None, match="GLU epilogue needs N % 4 == 0")


@pytest.mark.parametrize("off", [4, 8, 12])
def test_gemm_rejects_misaligned_output(lib, off):
    """C is written with 128-bit stores whenever ldc % 4 == 0: a C that is not 16-byte aligned is refused (for every ldc)."""
    for ldc in (4, 5):
        refused("masr_gemm_f32", A16, 16, W16, None, None, 0, C16 + off, ldc, 4, 4, 16, EPI_BIAS, 1.0, None,
                match="masr_gemm_f32: C must be 16-byte aligned")


@pytest.mark.parametrize("off", [4, 8, 12])
def test_conv2_rejects_misaligned_buffers(lib, off):
    """conv-2 loads c1 / w2p and stores out 128 bits at a time: each must be 16-byte aligned."""
    geo = (1, 3, 39, 1, 19, 32, None)
    refused("masr_conv2_s2_relu_f32", A16, W16, None, C16 + off, *geo, match="out must be 16-byte aligned")
    refused("masr_conv2_s2_relu_f32", A16 + off, W16, None, C16, *geo, match="c1 and w2p must be 16-byte aligned")
    refused("masr_conv2_s2_relu_f32", A16, W16 + off, None, C16, *geo, match="c1 and w2p must be 16-byte aligned")


def test_ctc_topk_rejects_bad_arguments(lib):
    """The register-resident top-k holds 20 x 256 logits (V <= 5120) and at most 40 candidates; blank must be a token."""
    args = (A16, 64, 4, 29)
    out = (C16, C16 + 0x1000, C16 + 0x2000)
    refused("masr_ctc_topk_f32", A16, 5184, 4, 5121, 40, 0.99, *out, None, match="vocabulary 5121 > 5120")
    refused("masr_ctc_topk_blank_f32", A16, 5184, 4, 5121, 40, 0.99, 0, *out, W16, None, match="vocabulary 5121 > 5120")
    for top_n in (0, 41):
        refused("masr_ctc_topk_f32", *args, top_n, 0.99, *out, None, match=f"cutoff_top_n={top_n} out of range")
        refused("masr_ctc_topk_blank_f32", *args, top_n, 0.99, 0, *out, W16, None, match=f"cutoff_top_n={top_n} out of range")
    for blank in (29, -1):
        refused("masr_ctc_topk_blank_f32", *args, 40, 0.99, blank, *out, W16, None, match=f"blank={blank} out of range")
