"""GPU (-m gpu): the fused Conformer feed-forward kernel masr_ffn_tc_f16x2 against the two launches it replaces
(masr_gemm_tc_f16x2 with MASR_EPI_BIAS_SILU into the hidden pair, then MASR_EPI_RESIDUAL), bit for bit, and against a
float64 reference at the fp32-grade tolerance of tests/test_gpu_tc_gemm.py."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

EPI_BIAS_SILU, EPI_RESIDUAL = 1, 5
D = 256


@pytest.fixture(scope="module")
def rt():
    from masr_b200 import _lib
    _lib.load()
    _lib.call("masr_check_device")

    class RT:
        lib = _lib
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


def make_inputs(rt, M, F, seed, extra_rows=3):
    """LayerNorm-like A, weights scaled like the model's, an fp32 residual stream with NaN rows past M."""
    g = torch.Generator().manual_seed(seed)
    A = torch.randn(M, D, generator=g)
    W1 = torch.randn(F, D, generator=g) / math.sqrt(D)
    b1 = torch.randn(F, generator=g) * 0.1
    W2 = torch.randn(D, F, generator=g) / math.sqrt(F)
    b2 = torch.randn(D, generator=g) * 0.1
    x = torch.full((M + extra_rows, D), float("nan"))
    x[:M] = torch.randn(M, D, generator=g)
    return A, W1, b1, W2, b2, x


def run_fused(rt, Ap, W1p, b1, W2p, b2, x, M, F, alpha=0.5, lda=D, ldx=D):
    rt.call("masr_ffn_tc_f16x2", P(Ap[0]), P(Ap[1]), lda, P(W1p[0]), P(W1p[1]), P(b1), P(W2p[0]), P(W2p[1]), P(b2), P(x), ldx,
            M, D, F, alpha, rt.st())


def run_two_launches(rt, Ap, W1p, b1, W2p, b2, x, M, F, alpha=0.5):
    hh = torch.empty(max(1, M), F, dtype=torch.float16, device=rt.dev)
    hl = torch.empty_like(hh)
    rt.call("masr_gemm_tc_f16x2", P(Ap[0]), P(Ap[1]), D, P(W1p[0]), P(W1p[1]), P(b1), None, 0, None, P(hh), P(hl), F, M, F, D,
            EPI_BIAS_SILU, 1.0, rt.st())
    rt.call("masr_gemm_tc_f16x2", P(hh), P(hl), F, P(W2p[0]), P(W2p[1]), P(b2), P(x), D, P(x), None, None, D, M, D, F,
            EPI_RESIDUAL, alpha, rt.st())


@pytest.mark.parametrize("M", [1, 63, 64, 65, 7936, 7937, 20000])
def test_fused_ffn_bit_identical_to_two_launches(rt, M):
    F = 2048
    A, W1, b1, W2, b2, x = make_inputs(rt, M, F, seed=M)
    Ad, W1d, b1d, W2d, b2d, xd = (t.to(rt.dev) for t in (A, W1, b1, W2, b2, x))
    Ap, W1p, W2p = split(rt, Ad), split(rt, W1d), split(rt, W2d)
    x_two = xd.clone()
    x_fused = xd.clone()
    run_two_launches(rt, Ap, W1p, b1d, W2p, b2d, x_two, M, F)
    run_fused(rt, Ap, W1p, b1d, W2p, b2d, x_fused, M, F)
    torch.cuda.synchronize()
    assert not torch.isnan(x_fused[:M]).any()
    assert torch.isnan(x_fused[M:]).all()                      # rows >= M untouched
    assert torch.equal(x_fused.view(torch.int32), x_two.view(torch.int32)), \
        (x_fused[:M] - x_two[:M]).abs().max().item()


@pytest.mark.parametrize("M,F", [(1000, 2048), (333, 256), (130, 512), (64, 1024)])
def test_fused_ffn_against_float64(rt, M, F):
    A, W1, b1, W2, b2, x = make_inputs(rt, M, F, seed=7 * M + F)
    Ad, W1d, b1d, W2d, b2d, xd = (t.to(rt.dev) for t in (A, W1, b1, W2, b2, x))
    Ap, W1p, W2p = split(rt, Ad), split(rt, W1d), split(rt, W2d)
    # the reference multiplies what the kernel is given: the (h, l) pairs, reconstructed in float64
    rec = lambda p: p[0].double().cpu() + p[1].double().cpu() / 2048.0
    A64, W164, W264 = rec(Ap), rec(W1p), rec(W2p)
    hid = torch.nn.functional.silu(A64 @ W164.t() + b1.double())
    want = x[:M].double() + 0.5 * (hid @ W264.t() + b2.double())
    run_fused(rt, Ap, W1p, b1d, W2p, b2d, xd, M, F)
    torch.cuda.synchronize()
    err = (xd[:M].cpu().double() - want).abs().max().item()
    assert err < 2e-5 * max(1.0, math.sqrt(F / 256)), err
    assert torch.isnan(xd[M:]).all()
    # F = 256 has a single accumulation chunk (no running sum); bit-identical to the two launches there as well
    x2 = x.to(rt.dev)
    run_two_launches(rt, Ap, W1p, b1d, W2p, b2d, x2, M, F)
    torch.cuda.synchronize()
    assert torch.equal(xd.view(torch.int32), x2.view(torch.int32))


def test_fused_ffn_rejections(rt):
    M, F = 64, 512
    A, W1, b1, W2, b2, x = make_inputs(rt, M, F, seed=1)
    Ad, W1d, b1d, W2d, b2d, xd = (t.to(rt.dev) for t in (A, W1, b1, W2, b2, x))
    Ap, W1p, W2p = split(rt, Ad), split(rt, W1d), split(rt, W2d)
    args = lambda lda=D, ldx=D, d=D, f=F, ap=Ap: (P(ap[0]), P(ap[1]), lda, P(W1p[0]), P(W1p[1]), P(b1d), P(W2p[0]), P(W2p[1]),
                                                  P(b2d), P(xd), ldx, M, d, f, 0.5, rt.st())
    lib = rt.lib.load()
    bad = {
        "d != 256": args(d=512),
        "d = 128": args(d=128),
        "F % 256 != 0": args(f=384),
        "F = 0": args(f=0),
        "lda not a multiple of 8": args(lda=260),
        "lda < d": args(lda=128),
        "odd ldx": args(ldx=257),
        "misaligned A": args(ap=(Ap[0][:, 1:], Ap[1][:, 1:])),
    }
    before = xd.clone()
    for what, a in bad.items():
        rc = lib.masr_ffn_tc_f16x2(*a)
        assert rc != 0, what
        assert "masr_ffn_tc_f16x2" in rt.lib.last_error(), what
    torch.cuda.synchronize()
    assert torch.equal(xd.view(torch.int32), before.view(torch.int32))
    # M = 0 is a no-op
    assert lib.masr_ffn_tc_f16x2(P(Ap[0]), P(Ap[1]), D, P(W1p[0]), P(W1p[1]), P(b1d), P(W2p[0]), P(W2p[1]), P(b2d), P(xd), D, 0, D,
                                 F, 0.5, rt.st()) == 0
