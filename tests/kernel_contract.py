"""Shared conventions of the kernel-level GPU tests: each C-ABI entry point is called by name and compared with a float64
CPU reference.  Every input row past a valid length holds large finite garbage (not zeros: a kernel that reads past a
length must not see the same zeros the reference pads with) and every output buffer starts as NaN, so both out-of-range
reads and writes outside a kernel's stated contract fail."""
import math

import pytest
import torch

GARBAGE = 1e3


def runtime():
    """Body of the tests' module-scoped ``rt`` fixture: the loaded library on the current CUDA device."""
    if not torch.cuda.is_available():
        pytest.fail("gpu tests need a CUDA device (no CPU fallback exists)")
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
    # (device copies passed this way are bound to names first: a temporary freed inside one call's argument list can hand
    # its memory to the next argument's copy)
    return None if t is None else t.data_ptr()


def garbage(shape, seed):
    """Finite, large, seeded filler for every row past a valid length."""
    g = torch.Generator().manual_seed(10_000 + seed)
    return (torch.rand(shape, generator=g) * 2 - 1) * GARBAGE


def nan(shape, device, dtype=torch.float32):
    return torch.full(shape, float("nan"), dtype=dtype, device=device)


def pair_value(h, l):
    """The fp32-grade value an fp16 (h, l) operand pair stands for."""
    return h.double().cpu() + l.double().cpu() / 2048.0


def assert_pair_reconstructs(h, l, y):
    """h + l/2048 reproduces the kernel's fp32 result to 2^-21 relative (a tiny floor covers fp16 subnormals)."""
    y = y.double().cpu()
    r = pair_value(h, l)
    assert torch.isfinite(r).all()
    assert torch.all((r - y).abs() <= 2.0 ** -21 * y.abs() + 1e-10), (r - y).abs().max().item()


def same(a, b):
    """Bit-identical, NaN where the other is NaN (untouched rows of NaN-filled buffers)."""
    na, nb = torch.isnan(a), torch.isnan(b)
    return torch.equal(na, nb) and torch.equal(a[~na], b[~nb])


def err(out, ref):
    """max |out - ref|; the kernel output must be finite."""
    out = out.detach().double().cpu()
    assert torch.isfinite(out).all(), "non-finite kernel output in a valid row"
    return (out - ref.double()).abs().max().item() if out.numel() else 0.0


def gemm_scale(A, W, y):
    """Per-element float32 error scale of y = A.W^T (+ bias): u * (sqrt(K) * ||a_i o w_j||_2 + |y|), u = 2^-24."""
    K = A.shape[1]
    return 2.0 ** -24 * (math.sqrt(K) * torch.sqrt((A.double() ** 2) @ (W.double() ** 2).t()) + y.abs())


def ratio(out, ref, scale):
    """max |out - ref| / scale over the valid block; the kernel output must be finite."""
    out = out.detach().double().cpu()
    assert torch.isfinite(out).all(), "non-finite kernel output in a valid row"
    return ((out - ref) / scale).abs().max().item() if out.numel() else 0.0


def report(name, **errs):
    print(f"[max error] {name}: " + ", ".join(f"{k}={v:.3g}" for k, v in errs.items()))


def relpos_reference(q, k, v, p, pos_u, pos_v, heads):
    """RelPositionMultiHeadedAttention core in float64 (conformer/attention.py:230-251,107-118) of one utterance: queries
    [n, d], keys / values / linear_pos(pe) rows [klen, d] (P row j belongs to key j, no rel_shift) -> [n, d]."""
    n, d = q.shape
    kl, dk = k.shape[0], d // heads

    def hv(t, rows):
        return t.double().reshape(rows, heads, dk).transpose(0, 1)
    qh, kh, vh, ph = hv(q, n), hv(k, kl), hv(v, kl), hv(p, kl)
    s = ((qh + pos_u.double()[:, None]) @ kh.transpose(1, 2) + (qh + pos_v.double()[:, None]) @ ph.transpose(1, 2)) / math.sqrt(dk)
    return (torch.softmax(s, -1) @ vh).transpose(0, 1).reshape(n, d)
