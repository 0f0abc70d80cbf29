"""GPU (-m gpu): the FP16x2 operand split of the tensor-core kernels across operand magnitudes.

Every dense contraction on the GPU path takes its operands as fp16 pairs h = fp16(x), l = fp16((x - h) * 2^11) and
multiplies Ah.Wh + 2^-11 (Ah.Wl + Al.Wh) with fp32 accumulation.  The other float64 tests draw their operands at unit
scale; this file checks the split where its format ends (derived from the fp16 format):

  normal range   2^-14 <= |x| < 65520:  |h + l/2^11 - x| <= 2^-22 |x|
  small values   |x| < 2^-14:           l is an fp16 subnormal, an absolute floor of 2^-36 (half of 2^-24 / 2^11)
  overflow       |x| >= 65520:          h = +-inf, l = -+inf, and a product with the pair is NaN (inf - inf)

  1. every pair producer writes exactly the numpy restatement of the split of its own fp32 result, bit for bit, over
     magnitudes 2^-30 .. 2^16 and the format's edges;
  2. scaling operands by 2^k (k = +-4, +-8) scales the GEMM, conv-2 and attention outputs by exactly 2^k;
  3. the GEMM (every epilogue), the fused FFN and the CTC head against float64 over a grid of operand scales, bounded by
     the float32 error scale plus the split's absolute floor (derived in `floor_scale`);
  4. peaked attention (scores near +-100 and +-1000, a nearly one-hot softmax) whose maximum jumps in a late key block;
  5. an operand at >= 65520 poisons exactly the rows and columns it enters (the CTC head: maxp NaN, id 0), and leaves
     every other output bit-identical.

Conventions of tests/kernel_contract.py (garbage past valid lengths, NaN-filled outputs).  Each docstring gives the
maximum error ratio observed on an H100 80GB HBM3 (700 W power limit); DESIGN.md's precision policy lists them per cell.
"""
import ctypes
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from kernel_contract import P, garbage, gemm_scale, nan, pair_value, ratio, relpos_reference, report, runtime, same

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24
FLOOR = 2.0 ** -36                  # absolute representation floor of the pair (fp16 subnormal spacing 2^-24, / 2^11 / 2)
REL = 2.0 ** -22                    # relative representation bound in the normal range
F16_OVERFLOW = 65520.0              # fp16 round-to-nearest-even turns |x| >= 65520 into inf
RATIO_TOL = 8.0                     # the fp32-grade bound of the other float64 tests (units of the float32 error scale)
H, DK, D = 4, 64, 256


@pytest.fixture(scope="module")
def rt():
    return runtime()


def split(rt, x):
    x = x.contiguous()
    h = torch.empty(x.shape, dtype=torch.float16, device=rt.dev)
    l = torch.empty_like(h)
    rt.call("masr_split_f16", P(x), P(h), P(l), x.numel(), rt.st())
    return h, l


def rup(n, m):
    return (n + m - 1) // m * m


# ---- 1. the pair, bit for bit ---------------------------------------------------------------------------------------------

def restate(y32):
    """numpy restatement of split_f16 on float32 values: float16 round-to-nearest-even (overflow to inf), the residual
    (x - h) * 2^11 in float32, rounded again."""
    y = np.ascontiguousarray(np.asarray(y32, dtype=np.float32))
    with np.errstate(all="ignore"):
        h = y.astype(np.float16)
        l = ((y - h.astype(np.float32)) * np.float32(2048.0)).astype(np.float16)
    return h, l


def fma32(a, b, c):
    """float32 fma(a, b, c): the product of two float32 values is exact in float64, one rounding of the sum to float64 and
    one to float32 (double rounding differs from a single rounding only at a float32 midpoint: never for these inputs)."""
    return (np.asarray(a, np.float32).astype(np.float64) * np.asarray(b, np.float32).astype(np.float64)
            + np.asarray(c, np.float32).astype(np.float64)).astype(np.float32)


def edge_values():
    """The split's edges, both signs: +-0, fp16 subnormals, 2^-14 and its fp16 / fp32 neighbours, 65504, the largest
    float32 below 65520, 65520 and beyond."""
    f32 = np.float32
    pos = [2.0 ** -24, 3 * 2.0 ** -24, 2.0 ** -20, 1023 * 2.0 ** -24, 2.0 ** -14 - 2.0 ** -24, 2.0 ** -14, 2.0 ** -14 + 2.0 ** -24,
           float(np.nextafter(f32(2.0 ** -14), f32(0))), float(np.nextafter(f32(2.0 ** -14), f32(1))), 2.0 ** -30, 2.0 ** -25,
           1.0, 1.0 + 2.0 ** -23, 1.0 + 2.0 ** -11, 2048.0 + 1.0, 65504.0, 65504.0 + 8.0,
           float(np.nextafter(f32(F16_OVERFLOW), f32(0))), F16_OVERFLOW, 65536.0, 1e5]
    v = np.array([0.0] + pos, dtype=np.float32)
    return np.concatenate([v, -v])          # includes -0.0


def sweep_values(n, seed):
    """Log-spaced magnitudes 2^-30 .. 2^16 with random significands and signs, then the edges."""
    rng = np.random.default_rng(seed)
    mag = np.exp2(rng.uniform(-30, 16, n)) * rng.choice([-1.0, 1.0], n)
    return np.concatenate([edge_values(), mag.astype(np.float32)])


def check_pair(h, l, y32, what):
    """(h, l) == restate(y32) bit for bit, and the representation bound of the module docstring."""
    y = np.asarray(y32, dtype=np.float32)
    hw, lw = restate(y)
    hg = h.cpu().contiguous().numpy().reshape(y.shape)
    lg = l.cpu().contiguous().numpy().reshape(y.shape)
    bad = (hg.view(np.uint16) != hw.view(np.uint16)) | (lg.view(np.uint16) != lw.view(np.uint16))
    assert not bad.any(), f"{what}: {bad.sum()} pairs differ from the split of the fp32 result, e.g. " \
        f"x={y[bad][:3]} h={hg[bad][:3]} l={lg[bad][:3]} want h={hw[bad][:3]} l={lw[bad][:3]}"
    over = np.abs(y) >= F16_OVERFLOW
    assert np.all(np.isinf(hg[over])) and np.all(np.sign(hg[over]) == np.sign(y[over])), f"{what}: overflow must give h = +-inf"
    assert np.all(~np.isfinite(lg[over])), f"{what}: an overflowed pair must not carry a finite l"
    fin = ~over
    rec = hg[fin].astype(np.float64) + lg[fin].astype(np.float64) / 2048.0
    x = y[fin].astype(np.float64)
    assert np.all(np.abs(rec - x) <= REL * np.abs(x) + FLOOR), f"{what}: representation bound"
    return int(fin.sum()), int(over.sum())


def test_split_pair_bit_exact(rt):
    """masr_split_f16 against the numpy restatement over 2^-30 .. 2^16 and the edges (also the scalar tail: n % 4 != 0)."""
    for n in (40003, 7):
        x = sweep_values(n, n) if n > 7 else edge_values()[:n]
        xd = torch.from_numpy(x).to(rt.dev)
        h, l = split(rt, xd)
        fin, over = check_pair(h, l, x, f"masr_split_f16 n={x.size}")
        report(f"split n={x.size}", finite=fin, overflow=over)
    # the format's three ranges, measured: max |pair - x| / |x| in the normal range, max |pair - x| below 2^-14
    x = sweep_values(100000, 3)
    x = x[np.abs(x) < F16_OVERFLOW]
    h, l = split(rt, torch.from_numpy(x).to(rt.dev))
    e = np.abs(pair_value(h, l).numpy() - x.astype(np.float64))
    normal = np.abs(x) >= 2.0 ** -14
    rel = (e[normal] / np.abs(x[normal])).max()
    small = e[~normal].max()
    report("split representation", normal_rel=rel, normal_rel_in_2m22=rel / REL, small_abs_in_2m36=small / FLOOR)
    assert rel <= REL and small <= FLOOR


def column_sweep(n, seed):
    """Per-column magnitudes for the producers whose output is an affine function of a column parameter: log-spaced
    scales 2^-30 .. 2^16 and a set of columns with scale 0 whose output is exactly an edge value (the offset)."""
    rng = np.random.default_rng(seed)
    edges = edge_values()
    scale = (np.exp2(rng.uniform(-30, 16, n)) * rng.choice([-1.0, 1.0], n)).astype(np.float32)
    offset = np.zeros(n, np.float32)
    k = min(len(edges), n // 3)
    scale[:k] = 0.0
    offset[:k] = edges[:k]
    return torch.from_numpy(scale), torch.from_numpy(offset)


@pytest.mark.parametrize("Dn", [256, 1024])
def test_layernorm_pairs_bit_exact(rt, Dn):
    """masr_layernorm_split_f16 == the split of masr_layernorm_f32 (same kernel template); masr_layernorm2_split_f16 and
    masr_layernorm_ada_split_f16 (D = 256) == the split of their own fp32 outputs (ada: of fma(ada_scale, y, ada_bias))."""
    M = 67
    g = torch.Generator().manual_seed(Dn)
    x = torch.randn(M, Dn, generator=g) * 3 + 1
    gamma, beta = column_sweep(Dn, Dn)
    xd, gd, bd = x.to(rt.dev), gamma.to(rt.dev), beta.to(rt.dev)
    y = nan((M, Dn), rt.dev)
    rt.call("masr_layernorm_f32", P(xd), Dn, P(gd), P(bd), P(y), Dn, M, Dn, 1e-5, rt.st())
    yh, yl = nan((M, Dn), rt.dev, torch.float16), nan((M, Dn), rt.dev, torch.float16)
    rt.call("masr_layernorm_split_f16", P(xd), Dn, P(gd), P(bd), P(yh), P(yl), Dn, M, Dn, 1e-5, rt.st())
    torch.cuda.synchronize()
    fin, over = check_pair(yh, yl, y.cpu().numpy(), f"masr_layernorm_split_f16 D={Dn}")
    assert over > 0 and fin > 0
    if Dn != 256:
        return
    ones, zeros = torch.ones(Dn, device=rt.dev), torch.zeros(Dn, device=rt.dev)
    x1 = xd.clone()
    y2 = nan((M, Dn), rt.dev)
    yh.fill_(float("nan")); yl.fill_(float("nan"))
    rt.call("masr_layernorm2_split_f16", P(x1), Dn, P(ones), P(zeros), P(x1), P(gd), P(bd), P(y2), P(yh), P(yl), Dn, M, Dn, 1e-5,
            rt.st())
    torch.cuda.synchronize()
    check_pair(yh, yl, y2.cpu().numpy(), "masr_layernorm2_split_f16")
    # ada: LN at unit gamma, then the swept per-column scale / offset
    ya = nan((M, Dn), rt.dev)
    yh.fill_(float("nan")); yl.fill_(float("nan"))
    rt.call("masr_layernorm_ada_split_f16", P(xd), Dn, P(ones), P(zeros), P(ya), P(gd), P(bd), P(yh), P(yl), Dn, M, Dn, 1e-5,
            rt.st())
    torch.cuda.synchronize()
    check_pair(yh, yl, fma32(gamma.numpy()[None], ya.cpu().numpy(), beta.numpy()[None]), "masr_layernorm_ada_split_f16")


def test_affine_and_time_reduce_pairs_bit_exact(rt):
    """masr_affine_split_f16 (scale / bias per column; with none: the input itself, swept) and
    masr_time_reduce_dw_split_f16 (k = 5 and 1, stride 2, garbage past each length) against the split of their fp32 result
    restated as float32 fma."""
    Dn, M = 256, 160
    x = sweep_values(M * Dn - edge_values().size, 11).reshape(M, Dn)
    xd = torch.from_numpy(x).to(rt.dev)
    yh, yl = nan((M, Dn), rt.dev, torch.float16), nan((M, Dn), rt.dev, torch.float16)
    rt.call("masr_affine_split_f16", P(xd), None, None, P(yh), P(yl), M, Dn, rt.st())
    torch.cuda.synchronize()
    check_pair(yh, yl, x, "masr_affine_split_f16 (identity)")
    sc, off = column_sweep(Dn, 12)
    g = torch.Generator().manual_seed(13)
    xr = (torch.randn(M, Dn, generator=g) * 2).numpy()
    xrd, scd, offd = torch.from_numpy(xr).to(rt.dev), sc.to(rt.dev), off.to(rt.dev)
    yh.fill_(float("nan")); yl.fill_(float("nan"))
    rt.call("masr_affine_split_f16", P(xrd), P(scd), P(offd), P(yh), P(yl), M, Dn, rt.st())
    torch.cuda.synchronize()
    check_pair(yh, yl, fma32(sc.numpy()[None], xr, off.numpy()[None]), "masr_affine_split_f16")
    # time reduction: y[b, t] = bias + sum_j w[:, j] x[b, 2t - pad + j] (fma chain from the bias, taps ascending)
    lens = [37, 20, 1]
    B, Tin = len(lens), 40
    for k, pad in ((5, 2), (1, 0)):
        out_rows = (Tin + 2 * pad - k) // 2 + 1
        xin = garbage((B, Tin, Dn), k)
        for b, n in enumerate(lens):
            xin[b, :n] = torch.randn(n, Dn, generator=g)
        wsc, bias = column_sweep(Dn, 20 + k)
        w = (wsc[:, None] * (1 + torch.rand(Dn, k, generator=g))).contiguous()
        xdv, wd, bd = xin.to(rt.dev), w.to(rt.dev), bias.to(rt.dev)
        ld = torch.tensor(lens, dtype=torch.int32, device=rt.dev)
        oh = nan((B, out_rows + 1, Dn), rt.dev, torch.float16)
        ol = nan((B, out_rows + 1, Dn), rt.dev, torch.float16)
        rt.call("masr_time_reduce_dw_split_f16", P(xdv), Tin, P(wd), P(bd), P(oh), P(ol), out_rows + 1, P(ld), B, out_rows, k, pad, Dn,
                rt.st())
        torch.cuda.synchronize()
        want = np.empty((B, out_rows, Dn), np.float32)
        xn, wn = xin.numpy(), w.numpy()
        for b, n in enumerate(lens):
            for t in range(out_rows):
                acc = bias.numpy().copy()
                for j in range(k):
                    tau = 2 * t - pad + j
                    if 0 <= tau < n:
                        acc = fma32(wn[:, j], xn[b, tau], acc)
                want[b, t] = acc
        check_pair(oh[:, :out_rows], ol[:, :out_rows], want, f"masr_time_reduce_dw_split_f16 k={k}")
        assert torch.isnan(oh[:, out_rows:].float()).all() and torch.isnan(ol[:, out_rows:].float()).all()


def test_conv1_planes_bit_exact(rt):
    """masr_conv1_cmvn_relu_planes_f16 (no CMVN): every plane element == the split of relu(fma chain of the 9 taps from the
    bias), per-channel weights swept over 2^-30 .. 2^16 and channels whose output is an edge value (zero weights)."""
    B, Fm, idim, C = 2, 23, 80, 256
    F1, W1 = (Fm - 1) // 2, (idim - 1) // 2
    TH = (F1 + 1) // 2
    g = torch.Generator().manual_seed(5)
    feats = torch.randn(B, Fm, idim, generator=g)
    wsc, b1 = column_sweep(C, 31)
    b1 = b1.abs()                                           # relu: the edges are probed from the positive side
    w1 = (wsc[:, None] * torch.randn(C, 9, generator=g)).contiguous()
    fd, wd, bd = feats.to(rt.dev), w1.to(rt.dev), b1.to(rt.dev)
    ph = nan((4, B, TH, 20, C), rt.dev, torch.float16)
    pl = nan((4, B, TH, 20, C), rt.dev, torch.float16)
    rt.call("masr_conv1_cmvn_relu_planes_f16", P(fd), None, None, P(wd), P(bd), P(ph), P(pl), B, Fm, idim, F1, W1, C, rt.st())
    torch.cuda.synchronize()
    fn, wn = feats.numpy(), w1.numpy()
    y = np.empty((B, F1, W1, C), np.float32)
    for t in range(F1):
        for f in range(W1):
            acc = np.broadcast_to(b1.numpy(), (B, C)).copy()
            for kh in range(3):
                for kw in range(3):
                    acc = fma32(wn[:, kh * 3 + kw][None], fn[:, 2 * t + kh, 2 * f + kw][:, None], acc)
            y[:, t, f] = np.maximum(acc, np.float32(0))
    hp, lp = ph.cpu(), pl.cpu()
    for pt in range(2):
        for pf in range(2):
            nt, nf = len(range(pt, F1, 2)), len(range(pf, W1, 2))
            sub = y[:, pt::2, pf::2]
            check_pair(hp[pt * 2 + pf, :, :nt, :nf], lp[pt * 2 + pf, :, :nt, :nf], sub, f"conv1 plane ({pt},{pf})")


def test_gemm_pair_epilogue_bit_exact(rt):
    """masr_gemm_tc_f16x2 writing fp32 C and the (Ch, Cl) pair in one call: the pair is the split of C, over output columns
    scaled 2^-30 .. 2^16 (the top ones overflow fp16 and must carry inf) and columns that are exactly an edge value
    (zero weights, the edge as bias); every epilogue that writes N columns."""
    M, N, K = 130, 136, 64
    g = torch.Generator().manual_seed(17)
    A = torch.randn(M, K, generator=g)
    wsc, b = column_sweep(N, 18)
    # a weight element of magnitude >= 65520 would overflow the input pair itself: cap the weights below that
    wsc = wsc.clamp(-2.0 ** 13, 2.0 ** 13)
    W = (wsc[:, None] * torch.randn(N, K, generator=g) / math.sqrt(K)).contiguous()
    R = torch.randn(M, N, generator=g) * 1e3
    (Ah, Al), (Wh, Wl) = split(rt, A.to(rt.dev)), split(rt, W.to(rt.dev))
    bd, Rd = b.to(rt.dev), R.to(rt.dev)
    for epi in (0, 1, 2, 4, 5):
        C = nan((M, N), rt.dev)
        Ch, Cl = nan((M, N), rt.dev, torch.float16), nan((M, N), rt.dev, torch.float16)
        rt.call("masr_gemm_tc_f16x2", P(Ah), P(Al), K, P(Wh), P(Wl), P(bd), P(Rd) if epi == 5 else None, N, P(C), P(Ch), P(Cl), N, M,
                N, K, epi, 0.5, rt.st())
        torch.cuda.synchronize()
        c = C.cpu().numpy()
        assert np.isfinite(c).all()
        check_pair(Ch, Cl, c, f"gemm pair epilogue {epi}")
        if epi in (0, 2):
            assert (np.abs(c) >= F16_OVERFLOW).any(), "the sweep reaches the overflow edge"


# ---- 2. exact scale equivariance ---------------------------------------------------------------------------------------------

def robust_pair(h, l):
    """The pair with every half below 2^-6 or above 255 in magnitude set to 0: scaling it by 2^k, |k| <= 8, stays in
    fp16's normal range, so the scaled pair is exact."""
    h, l = h.clone(), l.clone()
    h[(h.abs() < 2.0 ** -6) | (h.abs() > 255)] = 0
    l[(l.abs() < 2.0 ** -6) | (l.abs() > 255)] = 0
    return h, l


def scale_pair(h, l, k):
    hs, ls = (h.double() * 2.0 ** k).half(), (l.double() * 2.0 ** k).half()
    assert torch.equal(hs.double(), h.double() * 2.0 ** k) and torch.equal(ls.double(), l.double() * 2.0 ** k)
    return hs, ls


KS = [4, -4, 8, -8]


def test_gemm_scale_equivariance(rt):
    """masr_gemm_tc_f16x2 with epilogues none, ReLU, scale, residual: scaling A's pair (then W's pair) and the bias and
    residual by 2^k scales C by exactly 2^k, bit for bit; also with the output pair (compared through C)."""
    M, N, K = 200, 264, 320
    g = torch.Generator().manual_seed(23)
    A = torch.randn(M, K, generator=g)
    W = torch.randn(N, K, generator=g) / math.sqrt(K) * 8
    b = torch.randn(N, generator=g)
    R = torch.randn(M, N, generator=g)
    (Ah, Al), (Wh, Wl) = robust_pair(*split(rt, A.to(rt.dev))), robust_pair(*split(rt, W.to(rt.dev)))

    def run(ah, al, wh, wl, bias, res, epi):
        C = nan((M + 2, N), rt.dev)
        bd, Rd = bias.to(rt.dev), res.to(rt.dev)
        rt.call("masr_gemm_tc_f16x2", P(ah), P(al), K, P(wh), P(wl), P(bd), P(Rd), N, P(C), None, None, N, M, N, K, epi, 0.75, rt.st())
        torch.cuda.synchronize()
        return C.cpu()

    for epi in (0, 2, 4, 5):
        base = run(Ah, Al, Wh, Wl, b, R, epi)
        assert torch.isfinite(base[:M]).all()
        for k in KS:
            s = 2.0 ** k
            Ahs, Als = scale_pair(Ah, Al, k)
            Whs, Wls = scale_pair(Wh, Wl, k)
            assert same(run(Ahs, Als, Wh, Wl, b * s, R * s, epi), base * s), f"epilogue {epi}: A * 2^{k}"
            assert same(run(Ah, Al, Whs, Wls, b * s, R * s, epi), base * s), f"epilogue {epi}: W * 2^{k}"


def test_conv2_scale_equivariance(rt):
    """masr_conv2_tc_f16x2 (ReLU): the conv-1 planes and the bias scaled by 2^k scale both outputs' fp32 by 2^k exactly."""
    B, Fm, idim, C = 2, 47, 80, 256
    F1, W1 = (Fm - 1) // 2, (idim - 1) // 2
    T2, TH = (F1 - 1) // 2, (F1 + 1) // 2
    g = torch.Generator().manual_seed(29)
    feats = torch.randn(B, Fm, idim, generator=g)
    w1, b1 = torch.randn(C, 9, generator=g) / 3, torch.randn(C, generator=g) / 3
    w2, b2 = torch.randn(C, 9 * C, generator=g) / 48, torch.randn(C, generator=g) / 48
    ph = torch.zeros(4 * B * TH * 20 * C, dtype=torch.float16, device=rt.dev)
    pl = torch.zeros_like(ph)
    fd, w1d, b1d = feats.to(rt.dev), w1.to(rt.dev), b1.to(rt.dev)
    rt.call("masr_conv1_cmvn_relu_planes_f16", P(fd), None, None, P(w1d), P(b1d), P(ph), P(pl), B, Fm, idim, F1, W1, C, rt.st())
    ph, pl = robust_pair(ph, pl)
    w2h, w2l = robust_pair(*split(rt, w2.to(rt.dev)))

    def run(h, l, bias):
        out = nan((B * T2 * 19 + 3, C), rt.dev)
        bd = bias.to(rt.dev)
        rt.call("masr_conv2_tc_f16x2", P(h), P(l), P(w2h), P(w2l), P(bd), P(out), None, None, B, F1, T2, C, rt.st())
        torch.cuda.synchronize()
        return out.cpu()

    base = run(ph, pl, b2)
    assert torch.isfinite(base[:B * T2 * 19]).all() and (base[:B * T2 * 19] > 0).float().mean() > 0.2
    for k in KS:
        assert same(run(*scale_pair(ph, pl, k), b2 * 2.0 ** k), base * 2.0 ** k), f"conv2: 2^{k}"


TABLE_ROWS = 5000
ATTN_FNS = ("masr_relpos_attention_f32", "masr_relpos_attention_tc", "masr_relpos_attention_tc5")


class Attn:
    """The batched attention call: Q|K|V in one [B*T, 3d] fp32 buffer with garbage past every length (the tensor-core
    kernels get its fp16 pair), a 5000-row P table with garbage past T, O with 2 sentinel rows per utterance and 8 sentinel
    columns.  `v_pair`: the pair buffer the tensor-core kernels read K / V from (default: the split of qkv)."""

    def __init__(self, qkv, ptab, pu, pv, lens):
        self.qkv, self.ptab, self.pu, self.pv, self.lens = qkv, ptab, pu, pv, lens
        self.B, self.T = qkv.shape[0], qkv.shape[1]

    def run(self, rt, fn, qkv=None, pair=None):
        B, T = self.B, self.T
        qkv = self.qkv if qkv is None else qkv
        ob, ldo = T + 2, D + 8
        qd = qkv.reshape(B * T, 3 * D).contiguous().to(rt.dev)
        pd, ud, vd = self.ptab.to(rt.dev), self.pu.to(rt.dev), self.pv.to(rt.dev)
        ld = torch.tensor(self.lens, dtype=torch.int32, device=rt.dev)
        O = nan((B * ob, ldo), rt.dev)
        if fn == "masr_relpos_attention_f32":
            rt.call(fn, P(qd), 3 * D, T, qd.data_ptr() + 4 * D, qd.data_ptr() + 8 * D, 3 * D, T, P(pd), D, P(ud), P(vd), P(O), None, None,
                    ldo, ob, P(ld), P(ld), B, H, DK, T, rt.st())
        else:
            qh, ql = split(rt, qd) if pair is None else pair
            ph, pl = split(rt, pd)
            kv = (qh.data_ptr() + 2 * D, ql.data_ptr() + 2 * D, qh.data_ptr() + 4 * D, ql.data_ptr() + 4 * D, 3 * D, T)
            if fn == "masr_relpos_attention_tc5":
                rt.call(fn, P(qd), 3 * D, T, *kv, P(ph), P(pl), D, TABLE_ROWS, P(ud), P(vd), P(O), None, None, ldo, ob, P(ld), P(ld),
                        B, H, DK, T, rt.st())
            else:
                rt.call(fn, P(qd), 3 * D, T, *kv, P(ph), P(pl), D, P(ud), P(vd), P(O), None, None, ldo, ob, P(ld), P(ld), B, H, DK, T,
                        rt.st())
        torch.cuda.synchronize()
        return O.cpu().view(B, ob, ldo)

    def error(self, O, want=None):
        """max |O - float64| over the valid rows; padded query rows zero, sentinels NaN."""
        e = 0.0
        for i, n in enumerate(self.lens):
            if n:
                q = self.qkv[i, :n]
                ref = relpos_reference(q[:, :D], q[:, D:2 * D], q[:, 2 * D:], self.ptab[:n], self.pu, self.pv, H)
                out = O[i, :n, :D].double()
                assert torch.isfinite(out).all()
                e = max(e, (out - ref).abs().max().item())
            assert torch.all(O[i, n:self.T, :D] == 0)
        assert torch.isnan(O[:, self.T:]).all() and torch.isnan(O[:, :, D:]).all()
        return e


def random_attn(lens, seed):
    g = torch.Generator().manual_seed(seed)
    B, T = len(lens), max(lens)
    qkv = garbage((B, T, 3 * D), seed)
    for i, n in enumerate(lens):
        qkv[i, :n] = torch.randn(n, 3 * D, generator=g)
    ptab = garbage((TABLE_ROWS, D), seed + 1)
    ptab[:T] = torch.randn(T, D, generator=g)
    return Attn(qkv, ptab, torch.randn(H, DK, generator=g) * 0.3, torch.randn(H, DK, generator=g) * 0.3, lens)


@pytest.mark.parametrize("fn", ATTN_FNS)
def test_attention_value_scale_equivariance(rt, fn):
    """All three relpos attention kernels: V (fp32, or its pair) scaled by 2^k scales O by exactly 2^k."""
    lens = [200, 1, 65, 0, 129] if fn == "masr_relpos_attention_tc5" else [300, 1, 65, 0, 129]
    a = random_attn(lens, 41)
    B, T = a.B, a.T
    if fn == "masr_relpos_attention_f32":
        base = a.run(rt, fn)
        for k in KS:
            q = a.qkv.clone()
            q[:, :, 2 * D:] *= 2.0 ** k
            assert same(a.run(rt, fn, qkv=q), base * 2.0 ** k), f"{fn}: V * 2^{k}"
        return
    qh, ql = split(rt, a.qkv.reshape(B * T, 3 * D).contiguous().to(rt.dev))
    vh, vl = robust_pair(qh[:, 2 * D:], ql[:, 2 * D:])
    qh[:, 2 * D:], ql[:, 2 * D:] = vh, vl
    base = a.run(rt, fn, pair=(qh, ql))
    for k in KS:
        sh, sl = qh.clone(), ql.clone()
        sh[:, 2 * D:], sl[:, 2 * D:] = scale_pair(vh, vl, k)
        assert same(a.run(rt, fn, pair=(sh, sl)), base * 2.0 ** k), f"{fn}: V * 2^{k}"


# ---- 3. float64 accuracy over operand scales -----------------------------------------------------------------------------

SCALES = [-16, -12, -8, 0, 8, 12]           # log2 of s_A and s_W
FP32_GRADE_MIN = -8                        # below 2^-8 (A) or 2^-8 / sqrt(K) (W rms) the split's floor is allowed to show


def floor_scale(A, W):
    """The split's absolute floor carried through y = A.W^T.  Each pair stands for its value within 2^-22 |x| + 2^-36
    (module docstring); the relative part is inside gemm_scale (2^-22 = 4u), the absolute part adds
        sum_k (2^-36 |w_jk| + 2^-36 |a_ik|) <= 2^-36 sqrt(K) (||a_i|| + ||w_j||)        (Cauchy-Schwarz)
    to element (i, j); the product of the two floors (2^-72 K) is below float64's own rounding here."""
    K = A.shape[1]
    return FLOOR * math.sqrt(K) * (A.double().norm(dim=1)[:, None] + W.double().norm(dim=1)[None, :])


def grid_cells(limit_y=None):
    cells = []
    for ea in SCALES:
        for ew in SCALES:
            if ea + ew > 24 or (limit_y is not None and ea + ew > limit_y):
                continue                                   # |y| would leave the range the epilogue is meant for
            cells.append((ea, ew))
    return cells


def test_gemm_float64_magnitude_grid(rt):
    """masr_gemm_tc_f16x2, every epilogue, A ~ 2^ea N(0, 1) and W ~ 2^ew N(0, 1/K) for ea, ew in SCALES (SiLU and GLU where
    |y| stays below about 1e3), against float64 of the fp32 operands.  Bound: the float32 error scale plus `floor_scale`;
    the plain float32 error scale alone (RATIO_TOL) where both scales are at least 2^-8.
    Observed (H100): with the floor <= 2.0 in every cell; the float32 scale alone <= 2.0 where both scales are >= 2^-8, but
    2.6 - 7.3 at s_W = 2^-12 (weight rms 1.4e-5) and 41 - 102 at s_W = 2^-16 (DESIGN.md lists every cell)."""
    M, N, K = 257, 288, 320                            # N % 32 == 0 (GLU), a ragged last 128-column tile
    worst, worst_plain = 0.0, 0.0
    for ea, ew in grid_cells():
        g = torch.Generator().manual_seed(1000 + 37 * ea + ew)
        sa, sw = 2.0 ** ea, 2.0 ** ew
        A = torch.randn(M, K, generator=g) * sa
        W = torch.randn(N, K, generator=g) / math.sqrt(K) * sw
        b = torch.randn(N, generator=g) * sa * sw
        R = torch.randn(M, N, generator=g) * sa * sw
        (Ah, Al), (Wh, Wl) = split(rt, A.to(rt.dev)), split(rt, W.to(rt.dev))
        bd, Rd = b.to(rt.dev), R.to(rt.dev)
        y = A.double() @ W.double().t() + b.double()
        s, fl = gemm_scale(A, W, y), floor_scale(A, W)
        out, plain = {}, {}
        for epi in range(6):
            if epi in (1, 3) and ea + ew > 8:
                continue
            No = N // 2 if epi == 3 else N
            C = nan((M + 1, No), rt.dev)
            if epi == 3:                                           # interleaved value / gate rows
                rt.call("masr_gemm_tc_f16x2", P(Ah), P(Al), K, P(Wh), P(Wl), P(bd), None, 0, P(C), None, None, No, M, N, K, 3, 1.0, rt.st())
            else:
                rt.call("masr_gemm_tc_f16x2", P(Ah), P(Al), K, P(Wh), P(Wl), P(bd), P(Rd), N, P(C), None, None, N, M, N, K, epi, 0.5, rt.st())
            torch.cuda.synchronize()
            C = C.cpu()
            assert torch.isnan(C[M:]).all()
            if epi == 0:
                ref, bnd, bnd0 = y, s + fl, s
            elif epi == 1:
                ref = F.silu(y)
                bnd0 = 1.1 * s + 8 * U32 * ref.abs()
                bnd = bnd0 + 1.1 * fl
            elif epi == 2:
                ref, bnd, bnd0 = F.relu(y), s + fl, s
            elif epi == 3:
                v, gt = y[:, 0::2], y[:, 1::2]
                ref = v * torch.sigmoid(gt)
                sg = torch.sigmoid(gt)
                bnd0 = sg * s[:, 0::2] + 0.25 * v.abs() * s[:, 1::2] + 8 * U32 * ref.abs()
                bnd = bnd0 + sg * fl[:, 0::2] + 0.25 * v.abs() * fl[:, 1::2]
            elif epi == 4:
                ref, bnd, bnd0 = 0.5 * y, 0.5 * (s + fl), 0.5 * s
            else:
                ref = R.double() + 0.5 * y
                bnd0 = 0.5 * s + 2 * U32 * ref.abs()
                bnd = bnd0 + 0.5 * fl
            out[epi] = ratio(C[:M], ref, bnd + 1e-300)
            plain[epi] = ratio(C[:M], ref, bnd0 + 1e-300)
        report(f"gemm grid s_A=2^{ea} s_W=2^{ew}", bound=max(out.values()), fp32_scale_only=max(plain.values()))
        worst = max(worst, max(out.values()))
        assert max(out.values()) < RATIO_TOL, (ea, ew, out)
        if min(ea, ew) >= FP32_GRADE_MIN:
            worst_plain = max(worst_plain, max(plain.values()))
            assert max(plain.values()) < RATIO_TOL, (ea, ew, plain)
    report("gemm grid", worst_with_floor=worst, worst_fp32_grade_range=worst_plain)


def test_ffn_float64_magnitude_grid(rt):
    """masr_ffn_tc_f16x2 (D = 256, F = 512) with A ~ 2^ea and both weights ~ 2^ew (rms 2^ew / sqrt(fan-in)), biases and the
    residual at the scale of their sums, for hidden activations up to about 1e3, against float64 of the pairs it is given.
    Bound: the first GEMM's error carried through SiLU (slope <= 1.1) and the hidden pair, plus the second GEMM's, each
    with its split floor.  Observed (H100): at most 2.0 (s_A = 2^-8, s_W = 2^-16), elsewhere below 0.4."""
    M, Fh = 130, 512
    worst = 0.0
    for ea, ew in grid_cells(limit_y=8):
        g = torch.Generator().manual_seed(2000 + 37 * ea + ew)
        sa, sw = 2.0 ** ea, 2.0 ** ew
        A = torch.randn(M, D, generator=g) * sa
        W1 = torch.randn(Fh, D, generator=g) / math.sqrt(D) * sw
        b1 = torch.randn(Fh, generator=g) * 0.1 * sa * sw
        W2 = torch.randn(D, Fh, generator=g) / math.sqrt(Fh) * sw
        b2 = torch.randn(D, generator=g) * 0.1 * sa * sw * sw
        x = torch.full((M + 2, D), float("nan"))
        x[:M] = torch.randn(M, D, generator=g) * sa * sw * sw
        Ap, W1p, W2p = split(rt, A.to(rt.dev)), split(rt, W1.to(rt.dev)), split(rt, W2.to(rt.dev))
        xd, b1d, b2d = x.to(rt.dev), b1.to(rt.dev), b2.to(rt.dev)
        rt.call("masr_ffn_tc_f16x2", P(Ap[0]), P(Ap[1]), D, P(W1p[0]), P(W1p[1]), P(b1d), P(W2p[0]), P(W2p[1]), P(b2d), P(xd), D, M, D,
                Fh, 0.5, rt.st())
        torch.cuda.synchronize()
        out = xd.cpu()
        assert torch.isnan(out[M:]).all()
        y1 = A.double() @ W1.double().t() + b1.double()
        hid = F.silu(y1)
        e_hid = 1.1 * (gemm_scale(A, W1, y1) + floor_scale(A, W1)) + 8 * U32 * hid.abs()
        e_hid = e_hid + REL * hid.abs() + FLOOR                  # the hidden activation's own pair
        y2 = hid @ W2.double().t() + b2.double()
        want = x[:M].double() + 0.5 * y2
        bnd = 0.5 * (gemm_scale(hid, W2, y2) + floor_scale(hid, W2) + e_hid @ W2.double().abs().t()) + 2 * U32 * want.abs()
        r = ratio(out[:M], want, bnd + 1e-300)
        report(f"ffn grid s_A=2^{ea} s_W=2^{ew}", ratio=r)
        worst = max(worst, r)
        assert r < RATIO_TOL, (ea, ew, r)
    report("ffn grid", worst=worst)


def test_ctc_head_float64_magnitude_grid(rt):
    """masr_ctc_head_argmax_tc_f16x2 (V = 4233) with A ~ 2^ea, W ~ 2^ew for logits from ~2^-32 (uniform posterior) to
    ~2^8 (one-hot): ids equal the float64 argmax where the top-two margin exceeds 16 row error scales (with the floor);
    maxp within the row's error scale plus its float32 summation error (16 u maxp).  Observed (H100): at most 0.65."""
    M, V, K = 300, 4233, 256
    worst = 0.0
    for ea, ew in grid_cells(limit_y=8):
        g = torch.Generator().manual_seed(3000 + 37 * ea + ew)
        sa, sw = 2.0 ** ea, 2.0 ** ew
        A = torch.randn(M, K, generator=g) * sa
        W = torch.randn(V, K, generator=g) * (3.0 / math.sqrt(K)) * sw
        b = torch.randn(V, generator=g) * sa * sw
        (Ah, Al), (Wh, Wl) = split(rt, A.to(rt.dev)), split(rt, W.to(rt.dev))
        bd = b.to(rt.dev)
        ws = torch.empty(3 * ((V + 31) // 32) * M * 4, dtype=torch.uint8, device=rt.dev)
        ids = torch.full((M + 3,), -7, dtype=torch.int32, device=rt.dev)
        mp = nan((M + 3,), rt.dev)
        rt.call("masr_ctc_head_argmax_tc_f16x2", P(Ah), P(Al), K, P(Wh), P(Wl), P(bd), M, V, K, P(ws), ws.numel(), P(ids), P(mp), rt.st())
        torch.cuda.synchronize()
        ids, mp = ids.cpu(), mp.cpu()
        assert torch.all(ids[M:] == -7) and torch.isnan(mp[M:]).all()
        y = A.double() @ W.double().t() + b.double()
        row = (gemm_scale(A, W, y) + floor_scale(A, W)).max(1).values
        top2 = y.topk(2, dim=1).values
        sure = (top2[:, 0] - top2[:, 1]) > 16 * row
        assert torch.equal(ids[:M][sure].long(), y.argmax(1)[sure])
        pmax = torch.softmax(y, 1).max(1).values
        r = ratio(mp[:M], pmax, row + 16 * U32 * pmax)
        report(f"ctc grid s_A=2^{ea} s_W=2^{ew}", maxp_ratio=r, ids_checked=float(sure.float().mean()))
        worst = max(worst, r)
        assert r < RATIO_TOL, (ea, ew, r)
    report("ctc grid", worst=worst)


RNN_RMS = [-14, -12, -10, -8, -6, -4]          # log2 of the W_hh rms


def final_state_pair(ws, T, nb, RH):
    """The (h, l) pair of h_T the H = 2048 recurrence leaves in its workspace (rt_store_pair, lstm.cu): buffer T % 2 of
    the two [nb][H * 64] ping-pong buffers, unit u / lane col at ((u/16)*4 + col/8)*256 + ((col%8)*4 + (u%8)/2)*4 +
    ((u%16)/8)*2 + u%2, l 128 halves after h -> h, l [nb * 32, H] (lane-major)."""
    buf = ws[:2 * nb * RH * 64 * 2].view(torch.float16).cpu().view(2, nb, RH * 64)[T % 2]
    u = torch.arange(RH)[:, None]
    col = torch.arange(32)[None, :]
    k = u % 16
    o = ((u // 16) * 4 + col // 8) * 256 + ((col % 8) * 4 + (k % 8) // 2) * 4 + (k // 8) * 2 + k % 2
    h = buf[:, o].permute(0, 2, 1).reshape(nb * 32, RH)
    l = buf[:, o + 128].permute(0, 2, 1).reshape(nb * 32, RH)
    return h, l


@pytest.mark.parametrize("cell", ["lstm", "gru"])
def test_recurrence_float64_magnitude_grid(rt, cell):
    """masr_{lstm,gru}_seq_tc_f16x2 (H = 2048, both directions, ragged lengths) with W_hh ~ N(0, rms^2) for rms 2^-14 ..
    2^-4, against float64 torch.nn.LSTM / GRU.  The recurrence's pairs are the split of its fp32 values bit for bit: the
    output pair of every valid row, and the h_T pair it keeps in its workspace for the next step.

    Bound: one step's pre-activation W_hh.h_{t-1} carries the GEMM error, gemm_scale + floor_scale of (h_{t-1}, W_hh)
    (float64 trajectory), the cell adds its float32 rounding, 4u (1 + |gates_x| + |W_hh.h|); the ratio is the maximum
    error of the outputs and final states over the largest such per-step term, after up to 24 steps.
    Observed (H100): LSTM 0.13 - 1.0, GRU 0.14 - 1.6 (the largest at rms 2^-4, where ||W_hh|| ~ 6 amplifies earlier steps'
    errors).  At H = 2048 the cell's float32 rounding dominates the per-step term at every rms on the grid, so the floor term
    changes the ratio by under 1 %: the recurrence's W_hh.h has K = 2048 terms of |h| ~ 0.5, far above the floor."""
    from test_gpu_family_kernels import from_T, to_T
    from test_gpu_wide_deepspeech2 import H as RH, _Run, _problem, _reference
    B, T = 9, 24
    for e in RNN_RMS:
        pb = _problem(cell, B, T, seed=4000 + 17 * (e + 20) + (cell == "gru"))
        g = torch.Generator().manual_seed(5000 + e)
        pb["w_hh"] = torch.randn(2, pb["G"] * RH, RH, generator=g) * 2.0 ** e
        ref_out, ref_h, ref_c = _reference(pb)
        run = _Run(rt, pb)
        nbytes = ctypes.c_int64()
        rt.call("masr_rnn_seq_tc_workspace_bytes", B, RH, ctypes.byref(nbytes))
        nb = (B + 31) // 32
        fn = "masr_lstm_seq_tc_f16x2" if cell == "lstm" else "masr_gru_seq_tc_f16x2"
        err_all, step_b, step_b0 = 0.0, 0.0, 0.0
        for d in range(2):
            h0T = to_T(pb["h0"][d], 30 + d).to(rt.dev)
            hNT = nan(h0T.shape, rt.dev)
            c = pb["c0"][d].clone().to(rt.dev)
            ws = torch.zeros(nbytes.value, dtype=torch.uint8, device=rt.dev)
            Tk = max(pb["lens"])
            rt.call(fn, P(run.gx[d]), pb["G"] * RH, run.bstride, P(run.packed[d]), P(h0T), P(hNT), P(run.aux(d, c)), P(run.out),
                    P(run.oh), P(run.ol), 2 * RH, d * RH, P(run.lens), B, RH, Tk, d, P(ws), nbytes.value, rt.st())
            torch.cuda.synchronize()
            hN = from_T(hNT, B)
            fh, fl = final_state_pair(ws, Tk, nb, RH)
            check_pair(fh[:B], fl[:B], hN.numpy(), f"{cell} rms=2^{e} d={d}: h_T pair in the workspace")
            err_all = max(err_all, (hN.double() - ref_h[d]).abs().max().item())
            if cell == "lstm":
                err_all = max(err_all, (c.cpu().double() - ref_c[d]).abs().max().item())
            # per-step error terms along the float64 trajectory: h_{t-1} of every valid (lane, step)
            prev, gxs = [], []
            for i, n in enumerate(pb["lens"]):
                for t in range(n):
                    tp = t - 1 if d == 0 else t + 1
                    first = t == 0 if d == 0 else t == n - 1
                    prev.append(pb["h0"][d, i].double() if first else ref_out[i, tp, d * RH:(d + 1) * RH])
                    gxs.append(pb["gx"][d, i, t].double())
            if prev:
                hp, gx = torch.stack(prev), torch.stack(gxs)
                W = pb["w_hh"][d]
                z = hp @ W.double().t()
                cell_term = 4 * U32 * (1 + gx.abs() + z.abs())
                s0 = gemm_scale(hp, W, z)
                step_b = max(step_b, (s0 + floor_scale(hp, W) + cell_term).max().item())
                step_b0 = max(step_b0, (s0 + cell_term).max().item())
        out = run.out.cpu().view(B, run.bstride, 2 * RH)
        oh = run.oh.cpu().view(B, run.bstride, 2 * RH)
        ol = run.ol.cpu().view(B, run.bstride, 2 * RH)
        for i, n in enumerate(pb["lens"]):
            if n:
                err_all = max(err_all, (out[i, :n].double() - ref_out[i, :n]).abs().max().item())
                check_pair(oh[i, :n], ol[i, :n], out[i, :n].numpy(), f"{cell} rms=2^{e}: output pair")
            assert torch.isnan(out[i, n:]).all()
        r = err_all / step_b
        report(f"{cell} recurrence W_hh rms=2^{e}", err=err_all, ratio=r, fp32_scale_only=err_all / step_b0)
        assert r < RATIO_TOL, (cell, e, r)


# ---- 4. peaked attention ---------------------------------------------------------------------------------------------------

def peaked_attn(lens, where, peak, seed):
    """Queries share a direction e (per utterance): q = b e + noise.  Keys are small noise except a winner key
    k = c e (score ~ +peak), a runner-up (c - d) e 30 below it in an earlier key block (later when the winner is key 0),
    and 'anti' keys -c e (score ~ -peak).  `where`: the winner is the first valid key, the first key of a middle 64-key
    block (the last key below 65 keys) or the last valid key."""
    g = torch.Generator().manual_seed(seed)
    B, T = len(lens), max(lens)
    qkv = garbage((B, T, 3 * D), seed)
    beta = math.sqrt(peak / 8.0)                                      # |e_head|^2 ~ 64, / sqrt(d_k) = 8
    for i, n in enumerate(lens):
        if not n:
            continue
        e = torch.randn(D, generator=g)
        qkv[i, :n, :D] = beta * e + 0.1 * torch.randn(n, D, generator=g)
        qkv[i, :n, D:2 * D] = 0.05 * torch.randn(n, D, generator=g)
        qkv[i, :n, 2 * D:] = torch.randn(n, D, generator=g)
        w = {"first": 0, "middle": min(n - 1, max(64, n // 2 // 64 * 64)), "last": n - 1}[where]
        r = 0 if w > 0 else n - 1
        for j in range(min(n, 6)):
            a = (7 * j + 3) % n
            if a not in (w, r):
                qkv[i, a, D:2 * D] = -beta * e
        if r != w:
            qkv[i, r, D:2 * D] = (beta - 30.0 / (8 * beta)) * e
        qkv[i, w, D:2 * D] = beta * e
    ptab = garbage((TABLE_ROWS, D), seed + 1)
    ptab[:T] = 0.1 * torch.randn(T, D, generator=g)
    pu, pv = torch.randn(H, DK, generator=g) * 0.1, torch.randn(H, DK, generator=g) * 0.1
    a = Attn(qkv, ptab, pu, pv, lens)
    a.winner, a.peak = [], peak
    for n in lens:
        w = {"first": 0, "middle": min(n - 1, max(64, n // 2 // 64 * 64)), "last": n - 1}[where]
        a.winner.append((w, 0 if w > 0 else n - 1))
    return a


def assert_peaked(a):
    """The construction is what the test claims, from the float64 scores of every query and head (the pos_u / pos_v and
    linear_pos terms included): the maximum is the winner key at 0.5 - 2 x peak, the runner-up key is second, 10 - 60 below
    it and in an earlier 32-key tile (earlier 64-key block past 64 keys) when the winner is not key 0, and the minimum is
    below -0.5 x peak."""
    for i, n in enumerate(a.lens):
        heads = lambda t: t.double().reshape(n, H, DK).transpose(0, 1)
        q, k, p = heads(a.qkv[i, :n, :D]), heads(a.qkv[i, :n, D:2 * D]), heads(a.ptab[:n])
        s = ((q + a.pu.double()[:, None]) @ k.transpose(1, 2) + (q + a.pv.double()[:, None]) @ p.transpose(1, 2)) / math.sqrt(DK)
        w, r = a.winner[i]
        top = s.max(-1)
        assert torch.all(top.indices == w), "the winner key is not the maximum everywhere"
        assert torch.all(top.values > 0.5 * a.peak) and torch.all(top.values < 2 * a.peak), top.values.aminmax()
        if n > 1:
            two = s.topk(2, dim=-1)
            gap = two.values[..., 0] - two.values[..., 1]
            assert torch.all(two.indices[..., 1] == r), "the runner-up key is not second everywhere"
            assert torch.all(gap > 10) and torch.all(gap < 60), gap.aminmax()
            assert s.min() < -0.5 * a.peak
        if w > 0 and n > 32:
            assert r // 32 < w // 32 and (n <= 64 or r // 64 < w // 64), (n, w, r)


PEAK_LENS = [1, 63, 64, 65, 256, 257]
PEAK_TOL = {"masr_relpos_attention_f32": 1e-7, "masr_relpos_attention_tc": 1e-6, "masr_relpos_attention_tc5": 1e-6}


@pytest.mark.parametrize("peak", [100.0, 1000.0])
@pytest.mark.parametrize("where", ["first", "middle", "last"])
@pytest.mark.parametrize("fn", ATTN_FNS)
def test_peaked_attention(rt, fn, where, peak):
    """Scores near +-peak (a nearly one-hot softmax) with the winner in the first, a middle or the last key block and a
    runner-up 30 below it earlier (the running maximum jumps by ~30 there), lengths 1, 63, 64, 65, 256, 257 (_tc also 1500),
    garbage past every length, against float64.  Observed (H100): f32 1.4e-8, tc and tc5 2.4e-7 (the fp16 pairs of K, V
    and P); tolerances about 4x those."""
    lens = [n for n in PEAK_LENS if fn != "masr_relpos_attention_tc5" or n <= 256]
    if fn == "masr_relpos_attention_tc":
        lens = lens + [1500]
    a = peaked_attn(lens, where, peak, int(peak) + len(where) + len(fn))
    assert_peaked(a)
    e = a.error(a.run(rt, fn))
    report(f"peaked {fn} winner={where} peak={peak}", out=e)
    assert e < PEAK_TOL[fn]


# ---- 5. overflow is never silent -----------------------------------------------------------------------------------------

BIG = 70000.0


def test_gemm_overflow_poisons_its_row_and_column(rt):
    """One A element and one weight element at 70000 (>= 65520: h = inf, l = -inf): every epilogue's row i0 and column j0
    are non-finite (ReLU included: a NaN must not become 0), every other element is bit-identical to the run without the
    outliers.  The pair output carries the same poison."""
    M, N, K = 150, 160, 256
    i0, k0, j0, k1 = 77, 5, 100, 200
    g = torch.Generator().manual_seed(51)
    A = torch.randn(M, K, generator=g)
    W = torch.randn(N, K, generator=g) / math.sqrt(K)
    b = torch.randn(N, generator=g)
    R = torch.randn(M, N, generator=g)
    A2, W2 = A.clone(), W.clone()
    A2[i0, k0] = BIG
    W2[j0, k1] = -BIG
    bd, Rd = b.to(rt.dev), R.to(rt.dev)
    pairs = [(split(rt, A.to(rt.dev)), split(rt, W.to(rt.dev))), (split(rt, A2.to(rt.dev)), split(rt, W2.to(rt.dev)))]
    hA = pairs[1][0][0].cpu()
    assert torch.isinf(hA[i0, k0]) and torch.isinf(pairs[1][0][1].cpu()[i0, k0])
    mask = torch.ones(M, N, dtype=torch.bool)
    mask[i0] = False
    mask[:, j0] = False
    for epi in range(6):
        No = N // 2 if epi == 3 else N
        outs = []
        for (ah, al), (wh, wl) in pairs:
            C = nan((M, No), rt.dev)
            Ch, Cl = nan((M, No), rt.dev, torch.float16), nan((M, No), rt.dev, torch.float16)
            rt.call("masr_gemm_tc_f16x2", P(ah), P(al), K, P(wh), P(wl), P(bd), P(Rd), N, P(C), P(Ch), P(Cl), No, M, N, K, epi, 0.5,
                    rt.st())
            torch.cuda.synchronize()
            outs.append((C.cpu(), pair_value(Ch, Cl)))
        (c0, p0), (c1, p1) = outs
        jj = j0 // 2 if epi == 3 else j0
        m = mask[:, 0::2] if epi == 3 else mask
        if epi == 3:
            m = m.clone()
            m[:, jj] = False
        assert torch.isfinite(c0).all()
        assert not torch.isfinite(c1[i0]).any(), f"epilogue {epi}: the overflowed A row is finite somewhere"
        assert not torch.isfinite(c1[:, jj]).any(), f"epilogue {epi}: the overflowed weight's column is finite somewhere"
        assert not torch.isfinite(p1[i0]).any() and not torch.isfinite(p1[:, jj]).any(), f"epilogue {epi}: pair output"
        assert torch.equal(c1[m], c0[m]) and torch.equal(p1[m], p0[m]), f"epilogue {epi}: unaffected outputs changed"


def test_ffn_overflow_poisons_its_row_and_column(rt):
    """masr_ffn_tc_f16x2: an A element at 70000 poisons its row, a W2 element its output column, a W1 element (a hidden
    unit every output sums over) every output; all else bit-identical to the run without the outlier."""
    M, Fh = 70, 512
    i0, d0 = 33, 17
    g = torch.Generator().manual_seed(53)
    A = torch.randn(M, D, generator=g)
    W1 = torch.randn(Fh, D, generator=g) / math.sqrt(D)
    b1 = torch.randn(Fh, generator=g) * 0.1
    W2 = torch.randn(D, Fh, generator=g) / math.sqrt(Fh)
    b2 = torch.randn(D, generator=g) * 0.1
    x = torch.randn(M, D, generator=g)

    def run(a, w1, w2):
        xd, b1d, b2d = x.to(rt.dev), b1.to(rt.dev), b2.to(rt.dev)
        Ap, W1p, W2p = split(rt, a.to(rt.dev)), split(rt, w1.to(rt.dev)), split(rt, w2.to(rt.dev))
        rt.call("masr_ffn_tc_f16x2", P(Ap[0]), P(Ap[1]), D, P(W1p[0]), P(W1p[1]), P(b1d), P(W2p[0]), P(W2p[1]), P(b2d), P(xd), D, M, D,
                Fh, 0.5, rt.st())
        torch.cuda.synchronize()
        return xd.cpu()

    base = run(A, W1, W2)
    assert torch.isfinite(base).all()
    A2, W22, W12 = A.clone(), W2.clone(), W1.clone()
    A2[i0, 9] = BIG
    W22[d0, 300] = -BIG
    W12[200, 7] = BIG
    out = run(A2, W1, W22)
    mask = torch.ones(M, D, dtype=torch.bool)
    mask[i0] = False
    mask[:, d0] = False
    assert not torch.isfinite(out[i0]).any() and not torch.isfinite(out[:, d0]).any()
    assert torch.equal(out[mask], base[mask])
    assert not torch.isfinite(run(A, W12, W2)).any(), "an overflowed W1 element feeds every output"


def test_ctc_head_overflow_gives_nan_maxp_and_id_zero(rt):
    """masr_ctc_head_argmax_tc_f16x2 and the unfused masr_gemm_tc_f16x2 + masr_ctc_frame_argmax_f32: a frame whose logits
    hold a NaN has an undefined posterior (the reference's softmax row is all NaN, and np.argmax of it is 0): maxp NaN and
    id 0, never a plausible token.  An A element at 70000 poisons its frame only (all other frames bit-identical to the
    run without it); a weight element at 70000 poisons one logit of every frame, hence every frame."""
    M, V, K = 200, 4233, 256
    i0 = 123
    g = torch.Generator().manual_seed(57)
    A = torch.randn(M, K, generator=g)
    W = torch.randn(V, K, generator=g) * (3.0 / math.sqrt(K))
    b = torch.randn(V, generator=g)
    bd = b.to(rt.dev)
    Vp = rup(V, 16)

    def run(a, w):
        (ah, al), (wh, wl) = split(rt, a.to(rt.dev)), split(rt, w.to(rt.dev))
        ws = torch.empty(3 * ((V + 31) // 32) * M * 4, dtype=torch.uint8, device=rt.dev)
        ids, mp = torch.full((M,), -7, dtype=torch.int32, device=rt.dev), nan((M,), rt.dev)
        rt.call("masr_ctc_head_argmax_tc_f16x2", P(ah), P(al), K, P(wh), P(wl), P(bd), M, V, K, P(ws), ws.numel(), P(ids), P(mp), rt.st())
        logits = nan((M, Vp), rt.dev)
        rt.call("masr_gemm_tc_f16x2", P(ah), P(al), K, P(wh), P(wl), P(bd), None, 0, P(logits), None, None, Vp, M, V, K, 0, 1.0, rt.st())
        ids0, mp0 = torch.full((M,), -7, dtype=torch.int32, device=rt.dev), nan((M,), rt.dev)
        rt.call("masr_ctc_frame_argmax_f32", P(logits), Vp, M, V, P(ids0), P(mp0), None, V, rt.st())
        torch.cuda.synchronize()
        return ids.cpu(), mp.cpu(), ids0.cpu(), mp0.cpu()

    base = run(A, W)
    assert torch.isfinite(base[1]).all() and torch.equal(base[0], base[2])
    A2 = A.clone()
    A2[i0, 40] = BIG
    ids, mp, ids0, mp0 = run(A2, W)
    keep = torch.arange(M) != i0
    for i, p, what in ((ids, mp, "fused head"), (ids0, mp0, "frame argmax")):
        assert torch.isnan(p[i0]) and i[i0] == 0, f"{what}: poisoned frame gave id {i[i0].item()}, maxp {p[i0].item()}"
    assert torch.equal(ids[keep], base[0][keep]) and torch.equal(mp[keep], base[1][keep])
    assert torch.equal(ids0[keep], base[2][keep]) and torch.equal(mp0[keep], base[3][keep])
    W2 = W.clone()
    W2[1234, 77] = BIG
    ids, mp, ids0, mp0 = run(A, W2)
    for i, p, what in ((ids, mp, "fused head"), (ids0, mp0, "frame argmax")):
        assert torch.isnan(p).all() and torch.all(i == 0), f"{what}: a NaN logit column must poison every frame"
