"""GPU (-m gpu): the kernels of the Conformer batched path (what bench.py times), one C-ABI entry point at a time, against
float64 CPU references:

  relpos attention     masr/model_utils/conformer/attention.py:107-118,230-251  (_f32, the mma.sync _tc, the wgmma _tc5)
  tensor-core GEMMs    torch.nn.functional.linear + every epilogue
  CTC head             loss/ctc.py:70 softmax + ctc_greedy_decoder.py:21 first argmax, without the [M, V] logits
  conv subsampling     subsampling.py:81-84 (conv1 into parity planes, conv2 as an implicit GEMM)

Conventions of tests/kernel_contract.py: garbage past every valid length, NaN-filled outputs with sentinel rows past M and
sentinel columns past N, valid outputs finite.  Each docstring gives the maximum error observed on an H100 80GB HBM3
(400 W power limit); the tolerances are at most about 4x that.  The GEMM tolerances are multiples of a float32 dot-product
error scale, u * (sqrt(K) * sqrt(sum_k a_k^2 w_k^2) + |y|) with u = 2^-24, computed per output element.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from kernel_contract import (P, assert_pair_reconstructs, err, garbage, gemm_scale, nan, pair_value, ratio, relpos_reference,
                             report, runtime)

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24
H, DK, D = 4, 64, 256
TABLE_ROWS = 5000                           # the production linear_pos(pe) table (max_len 5000)


@pytest.fixture(scope="module")
def rt():
    return runtime()


def split(rt, x):
    x = x.contiguous()
    h = torch.empty(x.shape, dtype=torch.float16, device=rt.dev)
    l = torch.empty_like(h)
    rt.call("masr_split_f16", P(x), P(h), P(l), x.numel(), rt.st())
    return h, l


def outside(shape, rows, cols):
    """Mask of everything outside [:rows, :cols] of a 2-D buffer."""
    m = torch.ones(shape, dtype=torch.bool)
    m[:rows, :cols] = False
    return m


def all_nan(t, mask=None):
    t = t.cpu().float()
    return bool(torch.isnan(t if mask is None else t[mask]).all())


# ---- relative-position attention -------------------------------------------------------------------------------------------

ATTN_LENS = [[748, 1, 257, 0, 511, 64], [1500, 33], [257], [256, 0, 1, 129, 64], [255, 128, 17], [129]]
# (plain, skewed) tolerances per kernel; the skewed scores are ~10x larger, and so is their fp32 rounding
ATTN_TOL = {"masr_relpos_attention_f32": (1e-5, 8e-5), "masr_relpos_attention_tc": (1.5e-5, 5e-5),
            "masr_relpos_attention_tc5": (5e-6, 3e-5)}


class _AttnBatch:
    """The engine's batched call (engine._attention_tc): Q|K|V in one [B*T, 3d] buffer, T = max(lens), rows past each
    length hold garbage; the 5000-row P table holds garbage past T; O / Oh / Ol have a row pitch of d + 8 and 2 sentinel
    rows per utterance past max_q = T.  skew: queries ~7x larger (score standard deviation near 10) and, for the first 4
    queries of every utterance, a dominant key among its last 4 keys (the last key tile)."""

    def __init__(self, lens, skew):
        seed = sum(lens) + len(lens) + 7 * skew
        g = torch.Generator().manual_seed(seed)
        self.lens, self.skew = lens, skew
        self.B, self.T = len(lens), max(lens)
        qkv = garbage((self.B, self.T, 3 * D), seed)
        for i, n in enumerate(lens):
            qkv[i, :n, :D] = torch.randn(n, D, generator=g) * (7.0 if skew else 1.0)
            qkv[i, :n, D:] = torch.randn(n, 2 * D, generator=g)
            if skew:
                for j in range(min(4, n)):
                    qkv[i, n - 1 - j, D:2 * D] = 0.1 * qkv[i, j, :D]
        self.qkv = qkv
        self.ptab = garbage((TABLE_ROWS, D), seed + 1)
        self.ptab[:self.T] = torch.randn(self.T, D, generator=g)
        self.pu, self.pv = torch.randn(H, DK, generator=g) * 0.3, torch.randn(H, DK, generator=g) * 0.3

    def run(self, rt, fn, d_k=DK, max_q=None):
        B, T = self.B, self.T
        max_q = T if max_q is None else max_q
        self.ob, self.ldo = T + 2, D + 8
        qd = self.qkv.view(B * T, 3 * D).to(rt.dev)
        pd, ud, vd = self.ptab.to(rt.dev), self.pu.to(rt.dev), self.pv.to(rt.dev)
        ld = torch.tensor(self.lens, dtype=torch.int32, device=rt.dev)
        O = nan((B * self.ob, self.ldo), rt.dev)
        Oh, Ol = nan((B * self.ob, self.ldo), rt.dev, torch.float16), nan((B * self.ob, self.ldo), rt.dev, torch.float16)
        hh = D // d_k                                   # heads covering the d columns
        if fn == "masr_relpos_attention_f32":
            rt.call(fn, P(qd), 3 * D, T, qd.data_ptr() + 4 * D, qd.data_ptr() + 8 * D, 3 * D, T, P(pd), D, P(ud), P(vd), P(O), P(Oh),
                    P(Ol), self.ldo, self.ob, P(ld), P(ld), B, hh, d_k, max_q, rt.st())
        else:
            (qh, ql), (ph, pl) = split(rt, qd), split(rt, pd)
            kv = (qh.data_ptr() + 2 * D, ql.data_ptr() + 2 * D, qh.data_ptr() + 4 * D, ql.data_ptr() + 4 * D, 3 * D, T)
            if fn == "masr_relpos_attention_tc5":
                rt.call(fn, P(qd), 3 * D, T, *kv, P(ph), P(pl), D, TABLE_ROWS, P(ud), P(vd), P(O), P(Oh), P(Ol), self.ldo,
                        self.ob, P(ld), P(ld), B, hh, d_k, max_q, rt.st())
            else:
                rt.call(fn, P(qd), 3 * D, T, *kv, P(ph), P(pl), D, P(ud), P(vd), P(O), P(Oh), P(Ol), self.ldo, self.ob, P(ld),
                        P(ld), B, hh, d_k, max_q, rt.st())
        torch.cuda.synchronize()
        return tuple(t.cpu().view(B, self.ob, self.ldo) for t in (O, Oh, Ol))

    def check(self, outs):
        """Valid rows against float64, the pair against the fp32 output, padded query rows zero, sentinels NaN."""
        O, Oh, Ol = outs
        T = self.T
        e = 0.0
        for i, n in enumerate(self.lens):
            if n:
                q = self.qkv[i, :n]
                ref = relpos_reference(q[:, :D], q[:, D:2 * D], q[:, 2 * D:], self.ptab[:n], self.pu, self.pv, H)
                e = max(e, err(O[i, :n, :D], ref))
                assert_pair_reconstructs(Oh[i, :n, :D], Ol[i, :n, :D], O[i, :n, :D])
            for t in (O, Oh, Ol):
                assert torch.all(t[i, n:T, :D] == 0), "padded query rows must be zeros"
        for t in (O, Oh, Ol):
            assert all_nan(t[:, T:]) and all_nan(t[:, :, D:]), "write outside max_q rows / the heads' columns"
        return e


def _attn_cases(fn):
    return [(fn, lens, skew) for lens in ATTN_LENS for skew in (False, True)
            if fn != "masr_relpos_attention_tc5" or max(lens) <= 256]


@pytest.mark.parametrize("fn,lens,skew", [c for fn in ("masr_relpos_attention_f32", "masr_relpos_attention_tc",
                                                        "masr_relpos_attention_tc5") for c in _attn_cases(fn)])
def test_relpos_attention_batched(rt, fn, lens, skew):
    """The batched layout at ragged lengths: T up to 1500 (the mma.sync kernel's many 32-key tiles and online-softmax
    rescales), one-frame and empty utterances, 255 / 256 / 257 frames and 129 (one vs two 128-row query tiles of _tc5).
    Observed max error (H100), plain / skewed: f32 3.1e-6 / 2.9e-5 (T = 1500), tc 4.8e-6 (T = 1500) / 1.5e-5, tc5 1.6e-6 /
    9.6e-6; tolerances in ATTN_TOL, about 3x those."""
    batch = _AttnBatch(lens, skew)
    e = batch.check(batch.run(rt, fn))
    report(f"{fn} lens={lens} skew={skew}", out=e)
    assert e < ATTN_TOL[fn][skew]


@pytest.mark.parametrize("skew", [False, True])
@pytest.mark.parametrize("lens", [l for l in ATTN_LENS if max(l) <= 256])
def test_relpos_attention_tc5_agrees_with_tc(rt, lens, skew):
    """Where both apply (T <= 256), the wgmma kernel and the mma.sync kernel agree within the sum of their float64 bounds,
    and write zeros / leave NaN in exactly the same places.  (The fp16 halves of a pair may differ by one h ulp with l
    compensating, so pairs are compared by the value they stand for.)"""
    batch = _AttnBatch(lens, skew)
    (O5, h5, l5), (O, h, l) = batch.run(rt, "masr_relpos_attention_tc5"), batch.run(rt, "masr_relpos_attention_tc")
    diff = 0.0
    for x, y in ((O5.double(), O.double()), (pair_value(h5, l5), pair_value(h, l))):
        assert torch.equal(torch.isnan(x), torch.isnan(y))
        valid = ~torch.isnan(x)
        diff = max(diff, (x[valid] - y[valid]).abs().max().item())
    report(f"tc5 vs tc lens={lens} skew={skew}", diff=diff)
    assert diff < ATTN_TOL["masr_relpos_attention_tc5"][skew] + ATTN_TOL["masr_relpos_attention_tc"][skew]


def test_relpos_attention_rejects_unsupported(rt):
    """d_k != 64 is refused by all three kernels, max_q > 256 by _tc5, before anything is written."""
    from masr_b200._lib import MasrB200Error
    batch = _AttnBatch([40, 3], False)
    for fn in ("masr_relpos_attention_f32", "masr_relpos_attention_tc", "masr_relpos_attention_tc5"):
        with pytest.raises(MasrB200Error, match="d_k"):
            batch.run(rt, fn, d_k=32)
    batch = _AttnBatch([257, 3], False)
    with pytest.raises(MasrB200Error, match="max_q"):
        batch.run(rt, "masr_relpos_attention_tc5")


def test_relpos_attention_tc5_uses_at_most_256_keys(rt):
    """The header's precondition k_lens[b] <= 256 of _tc5 is not checked on the device: a longer key set is read as its
    first 256 keys.  This pins that documented behaviour (callers route such utterances to masr_relpos_attention_tc).
    Observed max error (H100): 1.0e-6; tolerance 4e-6."""
    g = torch.Generator().manual_seed(5)
    C, kl, cap = 16, 300, 320
    Q = torch.randn(C, 3 * D, generator=g)
    KV = torch.randn(cap, 2 * D, generator=g)
    ptab = torch.randn(cap, D, generator=g)
    pu, pv = torch.randn(H, DK, generator=g) * 0.3, torch.randn(H, DK, generator=g) * 0.3
    qd, kvd, pd, ud, vd = (t.to(rt.dev) for t in (Q, KV, ptab, pu, pv))
    (kh, klo), (ph, pl) = split(rt, kvd), split(rt, pd)
    qld = torch.tensor([C], dtype=torch.int32, device=rt.dev)
    kld = torch.tensor([kl], dtype=torch.int32, device=rt.dev)
    O = nan((C, D), rt.dev)
    rt.call("masr_relpos_attention_tc5", P(qd), 3 * D, C, P(kh), P(klo), kh.data_ptr() + 2 * D, klo.data_ptr() + 2 * D, 2 * D, cap,
            P(ph), P(pl), D, cap, P(ud), P(vd), P(O), None, None, D, C, P(qld), P(kld), 1, H, DK, C, rt.st())
    torch.cuda.synchronize()
    e = err(O, relpos_reference(Q[:, :D], KV[:256, :D], KV[:256, D:], ptab[:256], pu, pv, H))
    report("tc5 300 keys", out=e)
    assert e < 4e-6


# ---- tensor-core GEMM family -----------------------------------------------------------------------------------------------

def rup(n, m):
    return (n + m - 1) // m * m


def _pair_window(rt, A, col0, ld, seed):
    """A [M, K] as a column window (from column col0) of a wider fp16 pair buffer [M, ld] whose other columns hold garbage."""
    M, K = A.shape
    full = garbage((M, ld), seed)
    full[:, col0:col0 + K] = A
    h, l = split(rt, full.to(rt.dev))
    return (h, l), h.data_ptr() + 2 * col0, l.data_ptr() + 2 * col0


GEMM_SHAPES = [(1, 8, 64), (63, 120, 192), (64, 136, 320), (65, 264, 2304), (127, 4233, 64), (129, 4233, 2304), (257, 120, 4864),
               (129, 8, 4864), (7937, 136, 192), (7937, 264, 320)]
GEMM_RATIO_TOL = 8.0


@pytest.mark.parametrize("M,N,K", GEMM_SHAPES)
def test_tc_gemm_epilogues_float64(rt, M, N, K):
    """masr_gemm_tc_f16x2, every epilogue, fp32 and pair outputs in one call, against float64: A as a column window of a
    wider pair buffer (lda = K + 64), a residual in its own buffer (ldr = ldc + 16, garbage past N), 3 sentinel rows past M
    and sentinel columns past N (GLU: N/2) that must stay NaN.  K = 320 / 2304 end the 256-K chunked sum in a partial chunk.
    Observed max error (H100), in units of the float32 error scale: 2.3 (M = 7937, K = 192 / 320); tolerance 8."""
    g = torch.Generator().manual_seed(M * 31 + N * 7 + K)
    A = torch.randn(M, K, generator=g)
    a_pair, ah, al = _pair_window(rt, A, 32, K + 64, M + K)     # a_pair keeps the buffer alive
    Ng = rup(N, 32)                                    # the GLU form needs N % 32 == 0
    alpha = 0.25
    res = {}
    for epi in range(6):
        n_w = Ng if epi == 3 else N
        No = n_w // 2 if epi == 3 else n_w
        W = torch.randn(n_w, K, generator=g) / math.sqrt(K)
        b = torch.randn(n_w, generator=g)
        Wh, Wl = split(rt, W.to(rt.dev))
        bd = b.to(rt.dev)
        ldc = rup(No, 8) + 8
        ldr = ldc + 16
        R = garbage((M + 3, ldr), epi)
        R[:M, :No] = torch.randn(M, No, generator=g) * 2
        Rd = R.to(rt.dev)
        C = nan((M + 3, ldc), rt.dev)
        Ch, Cl = nan((M + 3, ldc), rt.dev, torch.float16), nan((M + 3, ldc), rt.dev, torch.float16)
        rt.call("masr_gemm_tc_f16x2", ah, al, K + 64, P(Wh), P(Wl), P(bd), P(Rd) if epi == 5 else None, ldr, P(C), P(Ch), P(Cl),
                ldc, M, n_w, K, epi, alpha, rt.st())
        torch.cuda.synchronize()
        y = A.double() @ W.double().t() + b.double()
        s = gemm_scale(A, W, y)
        if epi == 0:
            ref, bound = y, s
        elif epi == 1:
            ref, bound = F.silu(y), 1.1 * s + 8 * U32 * F.silu(y).abs()
        elif epi == 2:
            ref, bound = F.relu(y), s
        elif epi == 3:
            v, gt = y[:, 0::2], y[:, 1::2]
            ref = v * torch.sigmoid(gt)
            bound = torch.sigmoid(gt) * s[:, 0::2] + 0.25 * v.abs() * s[:, 1::2] + 8 * U32 * ref.abs()
        elif epi == 4:
            ref, bound = alpha * y, alpha * s
        else:
            ref = R[:M, :No].double() + alpha * y
            bound = alpha * s + 2 * U32 * ref.abs()
        C, Ch, Cl = C.cpu(), Ch.cpu(), Cl.cpu()
        res[epi] = ratio(C[:M, :No], ref, bound + 1e-30)
        assert_pair_reconstructs(Ch[:M, :No], Cl[:M, :No], C[:M, :No])
        mask = outside(C.shape, M, No)
        assert all_nan(C, mask) and all_nan(Ch, mask) and all_nan(Cl, mask), f"epilogue {epi} wrote outside [M, N]"
        assert torch.equal(Rd.cpu(), R)
    report(f"tc_gemm M={M} N={N} K={K}", **{f"epi{k}": v for k, v in res.items()})
    assert max(res.values()) < GEMM_RATIO_TOL, res


# ---- CTC head ----------------------------------------------------------------------------------------------------------------

CTC_MARGIN = 16.0        # ids are compared where the float64 top-two margin exceeds CTC_MARGIN x the row's GEMM error scale
CTC_MAXP_RATIO_TOL = 2.4  # maxp error in units of the row's largest GEMM error scale (d maxp / d logit <= 1 per logit)


def _ctc_problem(M, V, K, kind, seed):
    """Logits = A.W^T + b with: frames (m % 3 == 0) whose maximum is column V - 2, in the ragged last 32-column group;
    frames (m % 3 == 1) whose maximum is an exact tie between two identical weight rows inside one group (and, V > 40, a
    tie across groups exists for column 5 / V - 1).  kind "negative": every logit < 0, so a padding column read as 0 would
    win; "large": logits near 200, where exp overflows float32 without the max subtraction."""
    g = torch.Generator().manual_seed(seed)
    A = torch.randn(M, K, generator=g)
    W = torch.randn(V, K, generator=g) * (3.0 / math.sqrt(K))
    b = torch.randn(V, generator=g)
    t0 = 36 if V > 40 else 10
    W[t0 + 1], b[t0 + 1] = W[t0], b[t0]
    if V > 40:
        W[V - 1], b[V - 1] = W[5], b[5]
    for m0, col in ((0, V - 2), (1, t0)):
        u = W[col] / W[col].norm()
        A[m0::3] += 8.0 * u
    if kind == "negative":
        b -= 60.0
    elif kind == "large":
        b += 200.0
    return A, W, b


@pytest.mark.parametrize("M,V,K,kind", [(7937, 4233, 256, "plain"), (300, 4233, 256, "negative"), (129, 4233, 320, "large"),
                                        (65, 20, 256, "negative"), (1, 20, 64, "large"), (200, 33, 256, "plain")])
def test_ctc_head_float64(rt, M, V, K, kind):
    """masr_ctc_head_argmax_tc_f16x2 against float64 logits: ids equal the float64 argmax wherever the top-two margin
    exceeds the fp32-grade bound, and the FIRST of two exactly tied maxima; maxp against the float64 softmax maximum;
    ids / maxp past M untouched.  V = 20 and 33: a single or a one-column ragged group.  The maxp error grows with the
    logits' magnitude (1.0e-5 near 200), so it is bounded in units of the row's GEMM error scale.
    Observed max error (H100): 0.61 error scales (1.0e-5 absolute, logits near 200); tolerance 2.4."""
    A, W, b = _ctc_problem(M, V, K, kind, M + V + K)
    Ah, Al = split(rt, A.to(rt.dev))
    Wh, Wl = split(rt, W.to(rt.dev))
    bd = b.to(rt.dev)
    ws = torch.empty(3 * ((V + 31) // 32) * M * 4, dtype=torch.uint8, device=rt.dev)
    ids = torch.full((M + 5,), -7, dtype=torch.int32, device=rt.dev)
    mp = nan((M + 5,), rt.dev)
    rt.call("masr_ctc_head_argmax_tc_f16x2", P(Ah), P(Al), K, P(Wh), P(Wl), P(bd), M, V, K, P(ws), ws.numel(), P(ids), P(mp), rt.st())
    torch.cuda.synchronize()
    ids, mp = ids.cpu(), mp.cpu()
    y = A.double() @ W.double().t() + b.double()
    t0 = 36 if V > 40 else 10
    y[:, t0 + 1] = y[:, t0]                                      # identical weight rows: exact ties, whatever the BLAS order
    if V > 40:
        y[:, V - 1] = y[:, 5]
    if kind == "negative":
        assert y.max() < 0
    if kind == "large":
        assert y.max() > 89                                      # exp(89) > FLT_MAX
    top2 = y.topk(2, dim=1).values
    margin = top2[:, 0] - top2[:, 1]
    row_scale = gemm_scale(A, W, y).max(1).values
    tol = CTC_MARGIN * row_scale
    first = y.argmax(1)                                          # torch: the first maximal index
    sure = margin > tol
    tie = margin == 0
    assert sure.sum() + tie.sum() >= 0.9 * M
    assert torch.equal(ids[:M][sure].long(), first[sure]), "argmax differs from float64 where the margin is clear"
    assert torch.equal(ids[:M][tie].long(), first[tie]), "an exact tie must resolve to the first index"
    for m0, col in ((0, V - 2), (1, t0)):                      # the construction put the maxima where intended
        assert M <= m0 or (first[m0::3] == col).float().mean() > 0.9
    e = err(mp[:M], torch.softmax(y, 1).max(1).values)
    r = ratio(mp[:M], torch.softmax(y, 1).max(1).values, row_scale)
    assert torch.all(ids[M:] == -7) and torch.isnan(mp[M:]).all(), "ids / maxp written past M"
    report(f"ctc_head M={M} V={V} K={K} {kind}", maxp=e, maxp_ratio=r, checked=float(sure.sum() + tie.sum()) / M)
    assert r < CTC_MAXP_RATIO_TOL


# ---- convolution subsampling -----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("B,Fm", [(1, 7), (2, 9), (3, 131), (4, 998)])
def test_conv_subsampling_float64(rt, B, Fm):
    """masr_conv1_cmvn_relu_planes_f16 + masr_conv2_tc_f16x2 against float64 conv2d: Fm = 7 and 9 (T2 = 1, odd and even
    F1), 131 (odd F1, several 6-row time tiles), B = 4 at Fm = 998 (even F1, T2 = 248).  fp32 and pair outputs; rows past
    B*T2*19 untouched.  Observed max error (H100): conv1 planes 1.7e-6, conv2 2.0e-6; tolerance 6e-6 / 7e-6."""
    g = torch.Generator().manual_seed(B * 1000 + Fm)
    idim, C = 80, 256
    feats = torch.randn(B, Fm, idim, generator=g) * 3 + 20
    mean = torch.randn(idim, generator=g) + 20
    istd = torch.rand(idim, generator=g) * 0.3 + 0.2
    w1, b1 = torch.randn(C, 1, 3, 3, generator=g) / 3, torch.randn(C, generator=g) / 3
    w2, b2 = torch.randn(C, C, 3, 3, generator=g) / 48, torch.randn(C, generator=g) / 48
    F1, W1 = (Fm - 1) // 2, (idim - 1) // 2
    T2, W2 = (F1 - 1) // 2, (W1 - 1) // 2
    TH = (F1 + 1) // 2
    rows = B * T2 * W2
    d = lambda t: t.contiguous().to(rt.dev)
    fd, md, sd, w1d, b1d, b2d = d(feats), d(mean), d(istd), d(w1.reshape(C, 9)), d(b1), d(b2)
    w2h, w2l = split(rt, d(w2.permute(0, 2, 3, 1).reshape(C, 9 * C)))
    ph = torch.zeros(4 * B * TH * 20 * C, dtype=torch.float16, device=rt.dev)
    pl = torch.zeros_like(ph)
    rt.call("masr_conv1_cmvn_relu_planes_f16", P(fd), P(md), P(sd), P(w1d), P(b1d), P(ph), P(pl), B, Fm, idim, F1, W1, C, rt.st())
    out = nan((rows + 5, C), rt.dev)
    oh, ol = nan((rows + 5, C), rt.dev, torch.float16), nan((rows + 5, C), rt.dev, torch.float16)
    rt.call("masr_conv2_tc_f16x2", P(ph), P(pl), P(w2h), P(w2l), P(b2d), P(out), P(oh), P(ol), B, F1, T2, C, rt.st())
    torch.cuda.synchronize()
    x = ((feats.double() - mean.double()) * istd.double()).unsqueeze(1)
    r1 = F.relu(F.conv2d(x, w1.double(), b1.double(), stride=2))
    r2 = F.relu(F.conv2d(r1, w2.double(), b2.double(), stride=2)).permute(0, 2, 3, 1).reshape(rows, C)
    planes = pair_value(ph, pl).view(4, B, TH, 20, C)
    e1 = 0.0
    for pt in range(2):
        for pf in range(2):
            nt, nf = len(range(pt, F1, 2)), len(range(pf, W1, 2))
            e1 = max(e1, err(planes[pt * 2 + pf][:, :nt, :nf], r1.permute(0, 2, 3, 1)[:, pt::2, pf::2]))
    out, oh, ol = out.cpu(), oh.cpu(), ol.cpu()
    e2 = err(out[:rows], r2)
    assert_pair_reconstructs(oh[:rows], ol[:rows], out[:rows])
    assert all_nan(out[rows:]) and all_nan(oh[rows:]) and all_nan(ol[rows:]), "conv2 wrote past B*T2*19 rows"
    report(f"conv subsampling B={B} Fm={Fm}", conv1=e1, conv2=e2)
    assert e1 < 6e-6 and e2 < 7e-6
