"""GPU (-m gpu): the wgmma FP16x2-split GEMM against a float64 reference, and against the fp32 SIMT
GEMM it replaces.  The bar is fp32-grade accuracy (DESIGN.md precision policy)."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def rt():
    from masr_b200 import _lib
    _lib.load()
    _lib.call("masr_check_device")

    class RT:
        dev = torch.device("cuda", torch.cuda.current_device())
        call = staticmethod(_lib.call)

        @staticmethod
        def st():
            return torch.cuda.current_stream().cuda_stream

    return RT


def P(t):
    return None if t is None else t.data_ptr()


def split(rt, x):
    x = x.contiguous()
    h = torch.empty(x.shape, dtype=torch.float16, device=rt.dev)
    l = torch.empty(x.shape, dtype=torch.float16, device=rt.dev)
    rt.call("masr_split_f16", P(x), P(h), P(l), x.numel(), rt.st())
    return h, l


def test_split_roundtrip(rt):
    g = torch.Generator().manual_seed(0)
    x = (torch.randn(100003, generator=g) * torch.logspace(-6, 2, 100003)).to(rt.dev)
    h, l = split(rt, x)
    back = h.float() + l.float() / 2048.0
    # 22 significand bits for normal-range values; tiny values bottom out at the fp16 subnormal spacing / 2^11
    assert ((back - x).abs() <= x.abs() * 2.0 ** -21 + 1e-10).all()


@pytest.mark.parametrize("M,N,K", [(128, 128, 64), (128, 128, 256), (200, 256, 256), (1000, 2048, 256), (777, 256, 2048),
                                   (129, 4233, 256), (300, 256, 4864), (5, 768, 256),
                                   # A-resident variant (K == 256, N >= 512): multi-tile groups, ragged last group,
                                   # several units per CTA (the resident A tile is reloaded)
                                   (7936, 2048, 256), (2500, 1100, 256), (12800, 1024, 256)])
def test_tc_gemm_fp32_grade(rt, M, N, K):
    g = torch.Generator().manual_seed(M + N + K)
    A = torch.randn(M, K, generator=g); W = torch.randn(N, K, generator=g) / math.sqrt(K)
    b = torch.randn(N, generator=g); R = torch.randn(M, N, generator=g)
    Ad, Wd, bd, Rd = (t.to(rt.dev) for t in (A, W, b, R))
    Ah, Al = split(rt, Ad)
    Wh, Wl = split(rt, Wd)
    ldc = (N + 7) // 8 * 8
    ref64 = (A.double() @ W.double().t() + b.double())
    ref32 = F.linear(A, W, b)
    fp32_err = (ref32.double() - ref64).abs().max().item()
    C = torch.full((M, ldc), float("nan"), device=rt.dev)
    rt.call("masr_gemm_tc_f16x2", P(Ah), P(Al), K, P(Wh), P(Wl), P(bd), None, 0, P(C), None, None, ldc, M, N, K, 0, 1.0, rt.st())
    torch.cuda.synchronize()
    err = (C[:, :N].cpu().double() - ref64).abs().max().item()
    assert not torch.isnan(C[:, :N]).any()
    assert err < max(4 * fp32_err, 2e-6 * math.sqrt(K / 256)), (err, fp32_err)
    # epilogues (fp32 out)
    for epi, ref in [(1, F.silu(ref32)), (2, F.relu(ref32)), (4, ref32 * 0.25), (5, R + 0.25 * ref32)]:
        C.fill_(float("nan"))
        rt.call("masr_gemm_tc_f16x2", P(Ah), P(Al), K, P(Wh), P(Wl), P(bd), P(Rd), N, P(C), None, None, ldc, M, N, K, epi, 0.25, rt.st())
        assert (C[:, :N].cpu() - ref).abs().max().item() < 2e-5 * max(1.0, math.sqrt(K / 256)), epi
    # pair output feeds the next GEMM: (Ch, Cl) must reconstruct the fp32 result to 2^-21
    Ch = torch.zeros(M, ldc, dtype=torch.float16, device=rt.dev); Cl = torch.zeros_like(Ch)
    C.fill_(float("nan"))
    rt.call("masr_gemm_tc_f16x2", P(Ah), P(Al), K, P(Wh), P(Wl), P(bd), None, 0, P(C), P(Ch), P(Cl), ldc, M, N, K, 1, 1.0, rt.st())
    back = Ch[:, :N].float() + Cl[:, :N].float() / 2048.0
    assert ((back - C[:, :N]).abs() / C[:, :N].abs().clamp_min(1e-3)).max().item() < 1e-6
    if N % 32 == 0:
        Wi = torch.stack([W[:N // 2], W[N // 2:]], 1).reshape(N, K).to(rt.dev)
        bi = torch.stack([b[:N // 2], b[N // 2:]], 1).reshape(N).to(rt.dev)
        Wih, Wil = split(rt, Wi)
        G = torch.full((M, N // 2), float("nan"), device=rt.dev)
        rt.call("masr_gemm_tc_f16x2", P(Ah), P(Al), K, P(Wih), P(Wil), P(bi), None, 0, P(G), None, None, N // 2, M, N, K, 3, 1.0, rt.st())
        assert (G.cpu() - F.glu(ref32, dim=1)).abs().max().item() < 2e-5


@pytest.mark.parametrize("B,Fm", [(2, 47), (1, 998), (3, 131)])
def test_conv_subsampling_tc(rt, B, Fm):
    """conv1 (parity planes, fp16 pairs) + conv2 (wgmma implicit GEMM) against F.conv2d."""
    g = torch.Generator().manual_seed(Fm)
    idim, C = 80, 256
    feats = torch.randn(B, Fm, idim, generator=g) * 3 + 20
    mean = torch.randn(idim, generator=g) + 20; istd = torch.rand(idim, generator=g) * 0.3 + 0.2
    w1 = torch.randn(C, 1, 3, 3, generator=g) / 3; b1 = torch.randn(C, generator=g) / 3
    w2 = torch.randn(C, C, 3, 3, generator=g) / 48; b2 = torch.randn(C, generator=g) / 48
    F1, W1 = (Fm - 1) // 2, (idim - 1) // 2
    T2, W2 = (F1 - 1) // 2, (W1 - 1) // 2
    TH = (F1 + 1) // 2
    d = lambda t: t.contiguous().to(rt.dev)
    fd, md, sd_, w1d, b1d, b2d = d(feats), d(mean), d(istd), d(w1.reshape(C, 9)), d(b1), d(b2)
    w2h, w2l = split(rt, d(w2.permute(0, 2, 3, 1).reshape(C, 9 * C)))
    ph = torch.zeros(4 * B * TH * 20 * C, dtype=torch.float16, device=rt.dev); pl = torch.zeros_like(ph)
    rt.call("masr_conv1_cmvn_relu_planes_f16", P(fd), P(md), P(sd_), P(w1d), P(b1d), P(ph), P(pl), B, Fm, idim, F1, W1, C, rt.st())
    out = torch.full((B, T2, W2, C), float("nan"), device=rt.dev)
    oh = torch.zeros(B * T2 * W2, C, dtype=torch.float16, device=rt.dev); ol = torch.zeros_like(oh)
    rt.call("masr_conv2_tc_f16x2", P(ph), P(pl), P(w2h), P(w2l), P(b2d), P(out), P(oh), P(ol), B, F1, T2, C, rt.st())
    x = ((feats - mean) * istd).unsqueeze(1)
    r1 = F.relu(F.conv2d(x, w1, b1, stride=2))
    r2 = F.relu(F.conv2d(r1, w2, b2, stride=2)).permute(0, 2, 3, 1)
    # planes reconstruct conv1
    planes = (ph.float() + pl.float() / 2048.0).view(4, B, TH, 20, C).cpu()
    rec = torch.zeros(B, F1, W1, C)
    for pt in range(2):
        for pf in range(2):
            sub = planes[pt * 2 + pf]
            nt, nf = len(range(pt, F1, 2)), len(range(pf, W1, 2))
            rec[:, pt::2, pf::2] = sub[:, :nt, :nf]
    assert (rec - r1.permute(0, 2, 3, 1)).abs().max().item() < 2e-5
    assert not torch.isnan(out).any()
    assert (out.cpu() - r2).abs().max().item() < 5e-5
    back = (oh.float() + ol.float() / 2048.0).view(B, T2, W2, C).cpu()
    assert (back - r2).abs().max().item() < 5e-5


@pytest.mark.parametrize("M,K,double", [(128, 256, False), (7936, 2048, False), (7936, 256, True), (1000, 2048, True),
                                        (21000, 256, False), (77, 256, True)])
def test_residual_layernorm_epilogue(rt, M, K, double):
    """masr_gemm_tc_residual_ln_f16x2 (cluster of 2 CTAs, row statistics over DSMEM) against torch: residual stream,
    LayerNorm-ed operand pair, optional second LayerNorm and fp32 copy.  M = 21000 runs several tiles per CTA (persistent
    loop through the exchange rounds), M = 77 a ragged last row block."""
    N = 256
    g = torch.Generator().manual_seed(M + K + int(double))
    A = torch.randn(M, K, generator=g); W = torch.randn(N, K, generator=g) / math.sqrt(K)
    b = torch.randn(N, generator=g); R = torch.randn(M, N, generator=g) * 3 + 0.5
    g1, b1 = torch.rand(N, generator=g) + 0.5, torch.randn(N, generator=g) * 0.1
    g2, b2 = torch.rand(N, generator=g) + 0.5, torch.randn(N, generator=g) * 0.1
    Ad, Wd, bd, g1d, b1d, g2d, b2d = (t.to(rt.dev) for t in (A, W, b, g1, b1, g2, b2))
    Ah, Al = split(rt, Ad)
    Wh, Wl = split(rt, Wd)
    X = R.clone().to(rt.dev)                                   # in place: X is the residual and receives the new stream
    Y2 = torch.full((M, N), float("nan"), device=rt.dev)
    Yh = torch.zeros(M, N, dtype=torch.float16, device=rt.dev); Yl = torch.zeros_like(Yh)
    rt.call("masr_gemm_tc_residual_ln_f16x2", P(Ah), P(Al), K, P(Wh), P(Wl), P(bd), P(X), N, 0.5, P(X), P(g1d), P(b1d),
            P(g2d) if double else None, P(b2d) if double else None, P(Y2), P(Yh), P(Yl), N, M, N, K, 1e-5, rt.st())
    torch.cuda.synchronize()
    x_new = R + 0.5 * F.linear(A, W, b)
    ln1 = F.layer_norm(x_new, (N,), g1, b1, 1e-5)
    want_x, want_y = (ln1, F.layer_norm(ln1, (N,), g2, b2, 1e-5)) if double else (x_new, ln1)
    tol = 2e-5 * max(1.0, math.sqrt(K / 256))
    assert (X.cpu() - want_x).abs().max().item() < tol
    assert (Y2.cpu() - want_y).abs().max().item() < 2 * tol
    back = (Yh.float() + Yl.float() / 2048.0).cpu()
    assert (back - Y2.cpu()).abs().max().item() < 2e-6
    # same result as the unfused pair of calls it replaces (summation order of the statistics aside)
    X2 = R.clone().to(rt.dev)
    rt.call("masr_gemm_tc_f16x2", P(Ah), P(Al), K, P(Wh), P(Wl), P(bd), P(X2), N, P(X2), None, None, N, M, N, K, 5, 0.5, rt.st())
    if not double:
        assert torch.equal(X2, X)                              # the residual stream itself is bit-identical
        Zh = torch.zeros_like(Yh); Zl = torch.zeros_like(Yl)
        rt.call("masr_layernorm_split_f16", P(X2), N, P(g1d), P(b1d), P(Zh), P(Zl), N, M, N, 1e-5, rt.st())
        assert ((Zh.float() + Zl.float() / 2048.0) - (Yh.float() + Yl.float() / 2048.0)).abs().max().item() < 2e-6


@pytest.mark.parametrize("M,V,K", [(7936, 4233, 256), (300, 4233, 256), (129, 1000, 1024), (64, 33, 256)])
def test_ctc_head_fused_argmax(rt, M, V, K):
    """masr_ctc_head_argmax_tc_f16x2 == the unfused GEMM + masr_ctc_frame_argmax_f32: ids bit-exact (incl. exact ties:
    duplicated weight rows must resolve to the lower index), max-probability within 1e-6."""
    g = torch.Generator().manual_seed(M + V + K)
    A = torch.randn(M, K, generator=g); W = torch.randn(V, K, generator=g) * (3.0 / math.sqrt(K))
    b = torch.randn(V, generator=g)
    W[V - 1] = W[5]; b[V - 1] = b[5]                            # an exact tie across column groups / tiles
    if V > 40:
        W[37] = W[36]; b[37] = b[36]                            # ... and inside one 32-column group
    Ad, Wd, bd = A.to(rt.dev), W.to(rt.dev), b.to(rt.dev)
    Ah, Al = split(rt, Ad)
    Wh, Wl = split(rt, Wd)
    Vp = (V + 15) // 16 * 16
    logits = torch.zeros(M, Vp, device=rt.dev)
    rt.call("masr_gemm_tc_f16x2", P(Ah), P(Al), K, P(Wh), P(Wl), P(bd), None, 0, P(logits), None, None, Vp, M, V, K, 0, 1.0, rt.st())
    ids0 = torch.zeros(M, dtype=torch.int32, device=rt.dev); mp0 = torch.zeros(M, device=rt.dev)
    rt.call("masr_ctc_frame_argmax_f32", P(logits), Vp, M, V, P(ids0), P(mp0), None, V, rt.st())
    wsb = torch.empty(3 * ((V + 31) // 32) * M * 4, dtype=torch.uint8, device=rt.dev)
    ids1 = torch.full((M,), -1, dtype=torch.int32, device=rt.dev); mp1 = torch.zeros(M, device=rt.dev)
    rt.call("masr_ctc_head_argmax_tc_f16x2", P(Ah), P(Al), K, P(Wh), P(Wl), P(bd), M, V, K, P(wsb), wsb.numel(), P(ids1), P(mp1), rt.st())
    torch.cuda.synchronize()
    assert torch.equal(ids0, ids1)
    ref = F.linear(A.double(), W.double(), b.double())
    assert (ids1.cpu() == V - 1).sum() == 0 and (ids1.cpu() == 37).sum() == 0      # ties resolve to the first index
    assert (mp0 - mp1).abs().max().item() < 1e-6
    assert (mp1.cpu().double() - torch.softmax(ref, 1).max(1).values).abs().max().item() < 2e-5


@pytest.mark.parametrize("M,K,ada", [(1024, 2048, True), (16, 256, True), (200, 256, False)])
def test_residual_postln_epilogue(rt, M, K, ada):
    """masr_gemm_tc_residual_postln_f16x2 (Squeezeformer post-norm blocks, used by the stream pools): the stream becomes
    LN(residual + A.W^T + bias), the operand pair carries the adaptive scale / bias of the next sub-module."""
    N = 256
    g = torch.Generator().manual_seed(M + K)
    A = torch.randn(M, K, generator=g); W = torch.randn(N, K, generator=g) / math.sqrt(K)
    b = torch.randn(N, generator=g); R = torch.randn(M, N, generator=g) * 2 - 0.3
    ga, be = torch.rand(N, generator=g) + 0.5, torch.randn(N, generator=g) * 0.1
    a_s, a_b = torch.rand(N, generator=g) + 0.5, torch.randn(N, generator=g) * 0.2
    Ad, Wd, bd, gd, bed, asd, abd = (t.to(rt.dev) for t in (A, W, b, ga, be, a_s, a_b))
    Ah, Al = split(rt, Ad)
    Wh, Wl = split(rt, Wd)
    X = R.clone().to(rt.dev)
    Yh = torch.zeros(M, N, dtype=torch.float16, device=rt.dev); Yl = torch.zeros_like(Yh)
    rt.call("masr_gemm_tc_residual_postln_f16x2", P(Ah), P(Al), K, P(Wh), P(Wl), P(bd), P(X), N, 1.0, P(X), P(gd), P(bed),
            P(asd) if ada else None, P(abd) if ada else None, P(Yh), P(Yl), N, M, N, K, 1e-5, rt.st())
    torch.cuda.synchronize()
    want_x = F.layer_norm(R + F.linear(A, W, b), (N,), ga, be, 1e-5)
    want_y = a_s * want_x + a_b if ada else want_x
    tol = 2e-5 * max(1.0, math.sqrt(K / 256))
    assert (X.cpu() - want_x).abs().max().item() < tol
    assert ((Yh.float() + Yl.float() / 2048.0).cpu() - want_y).abs().max().item() < 2 * tol


@pytest.mark.parametrize("M,N,K,epi", [(7936, 2048, 256, 1), (7936, 256, 2048, 5), (385, 264, 320, 0), (129, 4233, 256, 0),
                                       (2500, 512, 256, 3), (1000, 256, 4864, 4)])
def test_pair_kernel_bit_identical_to_single_cta(rt, M, N, K, epi, monkeypatch):
    """The pair form (a 256 x 128 tile per cluster of 2 CTAs, each CTA multicasting half of the W tile into both CTAs'
    shared memory) computes the same products in the same accumulation order as the single-CTA kernel: every output —
    fp32, the fp16 (h, l) pair — must be bit-identical, for full tiles, odd row-block counts and ragged column tiles."""
    g = torch.Generator().manual_seed(7 * M + N + K)
    Ah, Al = split(rt, torch.randn(M, K, generator=g).to(rt.dev))
    Wh, Wl = split(rt, (torch.randn(N, K, generator=g) / math.sqrt(K)).to(rt.dev))
    b = torch.randn(N, generator=g).to(rt.dev)
    No = N // 2 if epi == 3 else N
    ldc = (No + 7) // 8 * 8
    R = torch.randn(M, ldc, generator=g).to(rt.dev) if epi == 5 else None
    outs = {}
    for mode in ("0", "1"):
        monkeypatch.setenv("MASR_TC_PAIR", mode)
        C = torch.full((M, ldc), float("nan"), device=rt.dev)
        Ch = torch.full((M, ldc), float("nan"), dtype=torch.float16, device=rt.dev)
        Cl = torch.full((M, ldc), float("nan"), dtype=torch.float16, device=rt.dev)
        rt.call("masr_gemm_tc_f16x2", P(Ah), P(Al), K, P(Wh), P(Wl), P(b), P(R), ldc, P(C), P(Ch), P(Cl), ldc, M, N, K, epi, 0.5, rt.st())
        torch.cuda.synchronize()
        outs[mode] = (C, Ch, Cl)
    for a, c in zip(outs["0"], outs["1"]):
        assert torch.equal(a[:, :No].view(torch.int32 if a.dtype == torch.float32 else torch.int16),
                           c[:, :No].view(torch.int32 if c.dtype == torch.float32 else torch.int16))
    assert torch.isfinite(outs["1"][0][:, :No]).all()


@pytest.mark.parametrize("kernel,shape", [("conv2", (2, 998)), ("conv2", (3, 131)), ("ctc_head", (7936, 4233)),
                                          ("ctc_head", (300, 33))])
def test_pair_kernel_bit_identical_conv2_and_ctc_head(rt, kernel, shape, monkeypatch):
    """MASR_TC_PAIR=1 for the other two users of the pair form: masr_conv2_tc_f16x2 (several 6-row time tiles per
    utterance) and masr_ctc_head_argmax_tc_f16x2 (several row blocks; ids and maxp) give bit-identical outputs."""
    g = torch.Generator().manual_seed(sum(shape))
    C = 256
    if kernel == "conv2":
        B, Fm = shape
        F1 = (Fm - 1) // 2
        T2, TH = (F1 - 1) // 2, (F1 + 1) // 2
        ph, pl = split(rt, (torch.rand(4 * B * TH * 20 * C, generator=g) * 2).to(rt.dev))
        wh, wl = split(rt, (torch.randn(C, 9 * C, generator=g) / 48).to(rt.dev))
        b = torch.randn(C, generator=g).to(rt.dev)
    else:
        M, V = shape
        ah, al = split(rt, torch.randn(M, C, generator=g).to(rt.dev))
        wh, wl = split(rt, (torch.randn(V, C, generator=g) * (3.0 / math.sqrt(C))).to(rt.dev))
        b = torch.randn(V, generator=g).to(rt.dev)
        ws = torch.empty(3 * ((V + 31) // 32) * M * 4, dtype=torch.uint8, device=rt.dev)
    outs = {}
    for mode in ("0", "1"):
        monkeypatch.setenv("MASR_TC_PAIR", mode)
        if kernel == "conv2":
            rows = B * T2 * 19
            o = (torch.full((rows, C), float("nan"), device=rt.dev), torch.full((rows, C), float("nan"), dtype=torch.float16, device=rt.dev),
                 torch.full((rows, C), float("nan"), dtype=torch.float16, device=rt.dev))
            rt.call("masr_conv2_tc_f16x2", P(ph), P(pl), P(wh), P(wl), P(b), P(o[0]), P(o[1]), P(o[2]), B, F1, T2, C, rt.st())
        else:
            o = (torch.full((M,), -1, dtype=torch.int32, device=rt.dev), torch.full((M,), float("nan"), device=rt.dev))
            rt.call("masr_ctc_head_argmax_tc_f16x2", P(ah), P(al), C, P(wh), P(wl), P(b), M, V, C, P(ws), ws.numel(), P(o[0]), P(o[1]),
                    rt.st())
        torch.cuda.synchronize()
        outs[mode] = o
    for a, c in zip(outs["0"], outs["1"]):
        assert torch.isfinite(a.float()).all()
        assert torch.equal(a.view(torch.int32 if a.element_size() == 4 else torch.int16),
                           c.view(torch.int32 if c.element_size() == 4 else torch.int16))


@pytest.mark.parametrize("M,N,epi", [(7936, 768, 0), (7936, 2048, 1), (7936, 512, 3), (1000, 768, 0), (129, 2048, 1), (77, 512, 3),
                                     (385, 4233, 0)])
@pytest.mark.parametrize("pair", ["0", "1"])
def test_layernorm_prologue_gemm_bit_identical_to_separate_launches(rt, M, N, epi, pair, monkeypatch):
    """masr_gemm_tc_lnpre_f16x2 (every CTA normalises the rows of its own contiguous tile range, then multiplies) against
    masr_layernorm_split_f16 + masr_gemm_tc_f16x2: the operand pair it leaves behind and every output must be bit-identical —
    single-CTA and pair kernels, many tiles per CTA, fewer tiles than CTAs, ragged row blocks and column tiles."""
    monkeypatch.setenv("MASR_TC_PAIR", pair)
    K = 256
    g = torch.Generator().manual_seed(M * 3 + N + epi)
    x = (torch.randn(M, K, generator=g) * 3 + 0.5).to(rt.dev)
    gamma, beta = (1 + 0.1 * torch.randn(K, generator=g)).to(rt.dev), (0.1 * torch.randn(K, generator=g)).to(rt.dev)
    Wh, Wl = split(rt, (torch.randn(N, K, generator=g) / math.sqrt(K)).to(rt.dev))
    b = torch.randn(N, generator=g).to(rt.dev)
    No = N // 2 if epi == 3 else N
    ldc = (No + 7) // 8 * 8

    def outs():
        return (torch.full((M, ldc), float("nan"), device=rt.dev), torch.full((M, ldc), float("nan"), dtype=torch.float16, device=rt.dev),
                torch.full((M, ldc), float("nan"), dtype=torch.float16, device=rt.dev))

    def pairbuf():
        return (torch.full((M, K), float("nan"), dtype=torch.float16, device=rt.dev), torch.full((M, K), float("nan"), dtype=torch.float16, device=rt.dev))

    ah, al = pairbuf()
    C0, Ch0, Cl0 = outs()
    rt.call("masr_layernorm_split_f16", P(x), K, P(gamma), P(beta), P(ah), P(al), K, M, K, 1e-5, rt.st())
    rt.call("masr_gemm_tc_f16x2", P(ah), P(al), K, P(Wh), P(Wl), P(b), None, 0, P(C0), P(Ch0), P(Cl0), ldc, M, N, K, epi, 1.0, rt.st())
    bh, bl = pairbuf()
    C1, Ch1, Cl1 = outs()
    rt.call("masr_gemm_tc_lnpre_f16x2", P(x), K, P(gamma), P(beta), 1e-5, P(bh), P(bl), K, P(Wh), P(Wl), P(b), P(C1), P(Ch1), P(Cl1),
            ldc, M, N, K, epi, 1.0, rt.st())
    torch.cuda.synchronize()
    assert torch.equal(ah.view(torch.int16), bh.view(torch.int16)) and torch.equal(al.view(torch.int16), bl.view(torch.int16))
    assert torch.equal(C0[:, :No].view(torch.int32), C1[:, :No].view(torch.int32))
    assert torch.equal(Ch0[:, :No].view(torch.int16), Ch1[:, :No].view(torch.int16))
    assert torch.equal(Cl0[:, :No].view(torch.int16), Cl1[:, :No].view(torch.int16))
    assert torch.isfinite(C1[:, :No]).all()
