"""GPU (-m gpu): the fused feed-forward kernel masr_ffn_tc_f16x2, whose 2-CTA clusters share each weight K-block through a
TMA multicast, against the two launches it replaces (masr_gemm_tc_f16x2 with EPI_BIAS_SILU, then EPI_RESIDUAL), bit for
bit, at the edges of the cluster schedule: a single pair whose second CTA has no rows (M <= 64), a ragged second block,
one full pair, an odd number of row blocks (M = 64 x 125), the headline M = 7936, and clusters that walk several pairs
(M = 20000, 313 row blocks); rows >= M untouched."""
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
        dev = torch.device("cuda", torch.cuda.current_device())
        call = staticmethod(_lib.call)

        @staticmethod
        def st():
            return torch.cuda.current_stream().cuda_stream

    return RT


def P(t):
    return t.data_ptr()


def split(rt, x):
    x = x.contiguous()
    h = torch.empty(x.shape, dtype=torch.float16, device=rt.dev)
    l = torch.empty(x.shape, dtype=torch.float16, device=rt.dev)
    rt.call("masr_split_f16", P(x), P(h), P(l), x.numel(), rt.st())
    return h, l


@pytest.mark.parametrize("F", [256, 2048])
@pytest.mark.parametrize("M", [1, 63, 64, 65, 127, 128, 64 * 125, 7936, 20000])
def test_cluster_ffn_bit_identical_to_two_launches(rt, M, F):
    g = torch.Generator().manual_seed(5 * M + F)
    A = torch.randn(M, D, generator=g)
    W1 = torch.randn(F, D, generator=g) / math.sqrt(D)
    b1 = (torch.randn(F, generator=g) * 0.1).to(rt.dev)
    W2 = torch.randn(D, F, generator=g) / math.sqrt(F)
    b2 = (torch.randn(D, generator=g) * 0.1).to(rt.dev)
    x = torch.full((M + 3, D), float("nan"))
    x[:M] = torch.randn(M, D, generator=g)
    Ap, W1p, W2p = split(rt, A.to(rt.dev)), split(rt, W1.to(rt.dev)), split(rt, W2.to(rt.dev))
    x_two, x_fused = x.to(rt.dev), x.to(rt.dev)

    hh = torch.empty(M, F, dtype=torch.float16, device=rt.dev)
    hl = torch.empty_like(hh)
    rt.call("masr_gemm_tc_f16x2", P(Ap[0]), P(Ap[1]), D, P(W1p[0]), P(W1p[1]), P(b1), None, 0, None, P(hh), P(hl), F, M, F, D,
            EPI_BIAS_SILU, 1.0, rt.st())
    rt.call("masr_gemm_tc_f16x2", P(hh), P(hl), F, P(W2p[0]), P(W2p[1]), P(b2), P(x_two), D, P(x_two), None, None, D, M, D, F,
            EPI_RESIDUAL, 0.5, rt.st())
    rt.call("masr_ffn_tc_f16x2", P(Ap[0]), P(Ap[1]), D, P(W1p[0]), P(W1p[1]), P(b1), P(W2p[0]), P(W2p[1]), P(b2), P(x_fused), D,
            M, D, F, 0.5, rt.st())
    torch.cuda.synchronize()
    assert not torch.isnan(x_fused[:M]).any()
    assert torch.isnan(x_fused[M:]).all()                      # rows >= M untouched, by the CTA without rows as well
    assert torch.equal(x_fused.view(torch.int32), x_two.view(torch.int32)), (x_fused[:M] - x_two[:M]).abs().max().item()
