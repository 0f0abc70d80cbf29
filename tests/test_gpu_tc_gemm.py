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
                                   (7936, 2048, 256), (2500, 1100, 256), (12800, 1024, 256),
                                   # the Conformer's d = 256 projection shapes: ragged row blocks, several tiles per CTA
                                   (128, 256, 256), (77, 256, 256), (7936, 256, 256), (21000, 256, 256), (1000, 256, 2048),
                                   (1000, 256, 4864), (385, 264, 320), (2500, 512, 256), (77, 512, 256), (7936, 512, 256),
                                   (1000, 768, 256), (7936, 768, 256), (129, 2048, 256), (385, 4233, 256)])
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


@pytest.mark.parametrize("B,Fm", [(2, 47), (1, 998), (3, 131), (2, 998)])
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


@pytest.mark.parametrize("M,V,K", [(7936, 4233, 256), (300, 4233, 256), (129, 1000, 1024), (64, 33, 256), (300, 33, 256)])
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
