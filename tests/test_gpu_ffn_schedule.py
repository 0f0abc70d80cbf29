"""GPU (-m gpu): the fused feed-forward kernel masr_ffn_tc_f16x2 against the two launches it replaces, bit for bit, at the
edges of its chunk schedule: one or two hidden-chunk pairs per row block (F = 256, 512) and the full F = 2048; one row
block, one per CTA, several per CTA (the two H buffers alternate over the chunks of all of a CTA's row blocks), a ragged
last row block; rows >= M untouched; and launches repeated into the same residual stream."""
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


def weights(rt, F, seed):
    g = torch.Generator().manual_seed(seed)
    W1 = torch.randn(F, D, generator=g) / math.sqrt(D)
    b1 = torch.randn(F, generator=g) * 0.1
    W2 = torch.randn(D, F, generator=g) / math.sqrt(F)
    b2 = torch.randn(D, generator=g) * 0.1
    return split(rt, W1.to(rt.dev)), b1.to(rt.dev), split(rt, W2.to(rt.dev)), b2.to(rt.dev), F


def activations(rt, M, seed, extra_rows=3):
    """LayerNorm-like A and an fp32 residual stream with NaN rows past M."""
    g = torch.Generator().manual_seed(seed)
    A = torch.randn(M, D, generator=g)
    x = torch.full((M + extra_rows, D), float("nan"))
    x[:M] = torch.randn(M, D, generator=g)
    return split(rt, A.to(rt.dev)), x.to(rt.dev)


def fused(rt, Ap, w, x, M):
    W1p, b1, W2p, b2, F = w
    rt.call("masr_ffn_tc_f16x2", P(Ap[0]), P(Ap[1]), D, P(W1p[0]), P(W1p[1]), P(b1), P(W2p[0]), P(W2p[1]), P(b2), P(x), D,
            M, D, F, 0.5, rt.st())


def two_launches(rt, Ap, w, x, M):
    W1p, b1, W2p, b2, F = w
    hh = torch.empty(M, F, dtype=torch.float16, device=rt.dev)
    hl = torch.empty_like(hh)
    rt.call("masr_gemm_tc_f16x2", P(Ap[0]), P(Ap[1]), D, P(W1p[0]), P(W1p[1]), P(b1), None, 0, None, P(hh), P(hl), F, M, F, D,
            EPI_BIAS_SILU, 1.0, rt.st())
    rt.call("masr_gemm_tc_f16x2", P(hh), P(hl), F, P(W2p[0]), P(W2p[1]), P(b2), P(x), D, P(x), None, None, D, M, D, F,
            EPI_RESIDUAL, 0.5, rt.st())


def assert_same(x_fused, x_two, M):
    assert not torch.isnan(x_fused[:M]).any()
    assert torch.isnan(x_fused[M:]).all()                      # rows >= M untouched
    assert torch.equal(x_fused.view(torch.int32), x_two.view(torch.int32)), (x_fused[:M] - x_two[:M]).abs().max().item()


@pytest.mark.parametrize("F", [256, 512, 2048])
@pytest.mark.parametrize("M", [1, 63, 64, 65, 8448, 8449, 20000])
def test_fused_ffn_schedule_bit_identical(rt, M, F):
    w = weights(rt, F, seed=F)
    Ap, x = activations(rt, M, seed=M + F)
    x_two, x_fused = x.clone(), x.clone()
    two_launches(rt, Ap, w, x_two, M)
    fused(rt, Ap, w, x_fused, M)
    torch.cuda.synchronize()
    assert_same(x_fused, x_two, M)


@pytest.mark.parametrize("M", [65, 8449, 20000])
def test_fused_ffn_repeated_launches(rt, M):
    """Several launches, alternating between two FFN modules, update the same residual stream in place."""
    mods = [weights(rt, 2048, seed=11), weights(rt, 512, seed=12), weights(rt, 256, seed=13)]
    Ap, x = activations(rt, M, seed=3 * M)
    x_two, x_fused = x.clone(), x.clone()
    for w in mods + mods[::-1]:
        two_launches(rt, Ap, w, x_two, M)
        fused(rt, Ap, w, x_fused, M)
    torch.cuda.synchronize()
    assert_same(x_fused, x_two, M)
