"""GPU (-m gpu): the kernels whose model width is a compile-time parameter, one C-ABI entry point at a time against float64
CPU references, at C = 512 (the wide Conformer) and, with the same code and bounds, at C = 256:

  masr_layernorm_split_f16 (256) or masr_layernorm_f32 + masr_split_f16 (512), masr_layernorm2_split_f16
                                                         LayerNorm(s) -> fp16 (h, l) operand pair
  masr_dwconv_ln_silu_f32                                depthwise Conv1d (k = 7 / 15 / 31) -> LayerNorm -> SiLU
  masr_conv1_cmvn_relu_planes_f16 + masr_conv2_tc_f16x2   convolution subsampling (conv-2 as an implicit GEMM)

Conventions of tests/kernel_contract.py: garbage past every valid length, NaN-filled outputs with sentinel rows that must
stay NaN.  Bounds are those of tests/test_gpu_conformer_kernels.py / tests/test_gpu_kernels.py for the 256-wide kernels;
conv-2 at C = 512 sums twice as many products per output and gets twice the bound.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from kernel_contract import P, assert_pair_reconstructs, err, garbage, nan, pair_value, report, runtime

pytestmark = pytest.mark.gpu

WIDTHS = [256, 512]


@pytest.fixture(scope="module")
def rt():
    return runtime()


def all_nan(t):
    return bool(torch.isnan(t.cpu().float()).all())


def split(rt, x):
    x = x.contiguous()
    h = torch.empty(x.shape, dtype=torch.float16, device=rt.dev)
    l = torch.empty_like(h)
    rt.call("masr_split_f16", P(x), P(h), P(l), x.numel(), rt.st())
    return h, l


def ln64(x, ga, be):
    return F.layer_norm(x.double(), (x.shape[-1],), ga.double(), be.double(), 1e-5)


LN_TOL = 4e-6          # fp32 LayerNorm of O(1) rows against float64


@pytest.mark.parametrize("M", [1, 7, 8, 9, 7936])
@pytest.mark.parametrize("D", WIDTHS)
def test_layernorm_to_pair_float64(rt, D, M):
    """LayerNorm -> operand pair as the engine runs it (`ConformerEngine._ln_split`): masr_layernorm_split_f16 at D = 256;
    at D = 512, where that entry point has no instantiation, masr_layernorm_f32 + masr_split_f16.  One warp per row, 8 rows
    per CTA: M = 1, 7, 8, 9 are the partial / full / spilling CTA, 7936 the headline batch.  The input has a row pitch of
    D + 8 with garbage in the gap; 3 sentinel rows past M stay NaN."""
    g = torch.Generator().manual_seed(D + M)
    ldx = D + 8
    xf = garbage((M, ldx), M)
    xf[:, :D] = torch.randn(M, D, generator=g) * 2 + 0.5
    ga, be = 1 + 0.1 * torch.randn(D, generator=g), 0.1 * torch.randn(D, generator=g)
    xd, gd, bd = xf.to(rt.dev), ga.to(rt.dev), be.to(rt.dev)
    yh, yl = nan((M + 3, D), rt.dev, torch.float16), nan((M + 3, D), rt.dev, torch.float16)
    if D == 256:
        rt.call("masr_layernorm_split_f16", P(xd), ldx, P(gd), P(bd), P(yh), P(yl), D, M, D, 1e-5, rt.st())
    else:
        y = nan((M + 3, D), rt.dev)
        rt.call("masr_layernorm_f32", P(xd), ldx, P(gd), P(bd), P(y), D, M, D, 1e-5, rt.st())
        rt.call("masr_split_f16", P(y), P(yh), P(yl), M * D, rt.st())
        assert all_nan(y[M:])
    torch.cuda.synchronize()
    ref = ln64(xf[:, :D], ga, be)
    got = pair_value(yh[:M], yl[:M])
    assert torch.isfinite(got).all()
    e = (got - ref).abs()
    assert torch.all(e <= 2.0 ** -21 * ref.abs() + LN_TOL), e.max().item()
    assert all_nan(yh[M:]) and all_nan(yl[M:])
    report(f"layernorm -> pair D={D} M={M}", pair=e.max().item())


@pytest.mark.parametrize("M", [1, 7, 8, 9, 7936])
@pytest.mark.parametrize("D", WIDTHS)
def test_layernorm2_split_float64(rt, D, M):
    """y1 = LN1(x) in place, y2 = LN2(y1) as fp32 and as the operand pair, against two float64 LayerNorms."""
    g = torch.Generator().manual_seed(2 * D + M)
    x = torch.randn(M, D, generator=g) * 3 - 1
    g1, b1 = 1 + 0.1 * torch.randn(D, generator=g), 0.1 * torch.randn(D, generator=g)
    g2, b2 = 1 + 0.1 * torch.randn(D, generator=g), 0.1 * torch.randn(D, generator=g)
    d = lambda t: t.contiguous().to(rt.dev)
    xin, g1d, b1d, g2d, b2d = d(x), d(g1), d(b1), d(g2), d(b2)
    y2 = nan((M + 3, D), rt.dev)
    yh, yl = nan((M + 3, D), rt.dev, torch.float16), nan((M + 3, D), rt.dev, torch.float16)
    rt.call("masr_layernorm2_split_f16", P(xin), D, P(g1d), P(b1d), P(xin), P(g2d), P(b2d), P(y2), P(yh), P(yl), D, M, D, 1e-5, rt.st())
    torch.cuda.synchronize()
    r1 = ln64(x, g1, b1)
    r2 = ln64(r1, g2, b2)
    e1, e2 = err(xin, r1), err(y2[:M], r2)
    assert_pair_reconstructs(yh[:M], yl[:M], y2[:M])
    assert all_nan(y2[M:]) and all_nan(yh[M:]) and all_nan(yl[M:])
    report(f"layernorm2_split D={D} M={M}", ln1=e1, ln2=e2)
    assert e1 < LN_TOL and e2 < 2 * LN_TOL


@pytest.mark.parametrize("mode", ["causal", "noncausal", "chunk"])
@pytest.mark.parametrize("ks", [7, 15, 31])
@pytest.mark.parametrize("C", WIDTHS)
def test_dwconv_ln_silu_float64(rt, C, ks, mode):
    """Whole-utterance causal (left padding = `pad_vec`, lpad = k - 1) and non-causal (zeros, lpad = (k - 1) / 2) forms and
    the streaming-chunk form (lpad = 0 over [cache ++ chunk] rows).  Ragged `in_lens` including 0 and 1, rows past each
    length garbage (they must read as zeros); `out_rows` = 37 is not a multiple of the 16 frames of a CTA; fp32 and pair
    outputs in one call; 3 sentinel rows per utterance past `out_rows` stay NaN.  k = 31 at C = 512 is the instantiation
    whose weight tile is dynamic shared memory.  Bound 2e-5 (SiLU on the SFU), as tests/test_gpu_kernels.py."""
    g = torch.Generator().manual_seed(1000 * C + 10 * ks + len(mode))
    out_rows = 37
    lpad = {"causal": ks - 1, "noncausal": (ks - 1) // 2, "chunk": 0}[mode]
    in_rows = out_rows + (ks - 1 if mode == "chunk" else 0)
    lens = [in_rows, 0, 1, 9, in_rows - 5]
    B, ldg, ldy, yb = len(lens), C + 4, C + 8, out_rows + 3
    x = garbage((B, in_rows, ldg), C + ks)
    for i, n in enumerate(lens):
        x[i, :n, :C] = torch.randn(n, C, generator=g)
    w = torch.randn(C, 1, ks, generator=g) / math.sqrt(ks)
    b = torch.randn(C, generator=g) * 0.1
    ga, be = 1 + 0.1 * torch.randn(C, generator=g), 0.1 * torch.randn(C, generator=g)
    pad = torch.randn(C, generator=g)
    d = lambda t: t.contiguous().to(rt.dev)
    xd, wd, bd, gd, bed, padd = d(x), d(w.reshape(C, ks)), d(b), d(ga), d(be), d(pad)
    ld = torch.tensor(lens, dtype=torch.int32, device=rt.dev)
    y = nan((B, yb, ldy), rt.dev)
    yh, yl = nan((B, yb, ldy), rt.dev, torch.float16), nan((B, yb, ldy), rt.dev, torch.float16)
    rt.call("masr_dwconv_ln_silu_f32", P(xd), ldg, in_rows, P(wd), P(bd), P(gd), P(bed), P(padd) if mode == "causal" else None,
            P(y), P(yh), P(yl), ldy, yb, P(ld), B, C, ks, lpad, out_rows, 1e-5, rt.st())
    torch.cuda.synchronize()
    y, yh, yl = y.cpu(), yh.cpu(), yl.cpu()
    e = 0.0
    for i, n in enumerate(lens):
        # the rows the kernel sees at tau = -lpad .. out_rows - lpad + ks - 2
        rows = torch.zeros(out_rows + ks - 1, C, dtype=torch.float64)
        if mode == "causal":
            rows[:lpad] = pad.double()
        hi = min(n, out_rows - lpad + ks - 1)
        rows[lpad:lpad + hi] = x[i, :hi, :C].double()
        r = F.conv1d(rows.t()[None], w.double(), b.double(), groups=C)[0].t()
        ref = F.silu(ln64(r, ga, be))
        e = max(e, err(y[i, :out_rows, :C], ref))
        assert_pair_reconstructs(yh[i, :out_rows, :C], yl[i, :out_rows, :C], y[i, :out_rows, :C])
    for t in (y, yh, yl):
        assert all_nan(t[:, out_rows:]) and all_nan(t[:, :, C:]), "write outside out_rows rows / C columns"
    report(f"dwconv_ln_silu C={C} k={ks} {mode}", y=e)
    assert e < 2e-5


def test_dwconv_rejects_unsupported_widths(rt):
    from masr_b200._lib import MasrB200Error
    z = torch.zeros(16, 512, device=rt.dev)
    ld = torch.tensor([16], dtype=torch.int32, device=rt.dev)
    with pytest.raises(MasrB200Error, match="C=384"):
        rt.call("masr_dwconv_ln_silu_f32", P(z), 384, 16, P(z), P(z), P(z), P(z), None, P(z), None, None, 384, 16, P(ld), 1, 384, 15,
                7, 16, 1e-5, rt.st())
    with pytest.raises(MasrB200Error, match="C=512"):       # the strided (EfficientConformer) form is 256-wide only
        rt.call("masr_dwconv_ln_silu_strided_f32", P(z), 512, 16, P(z), P(z), P(z), P(z), None, P(z), None, None, 512, 8, P(ld), 1,
                512, 15, 7, 2, 8, 1e-5, rt.st())
    with pytest.raises(MasrB200Error, match="C=512"):       # and so is the BatchNorm (Squeezeformer) form
        rt.call("masr_dwconv_bn_silu_f32", P(z), 512, 16, P(z), P(z), P(z), P(z), None, P(z), None, None, 512, 16, P(ld), 1, 512, 15,
                7, 16, rt.st())


@pytest.mark.parametrize("B,T2", [(1, 1), (3, 1), (3, 5), (1, 6), (3, 6), (3, 7), (1, 248)])
@pytest.mark.parametrize("C", WIDTHS)
def test_conv_subsampling_float64(rt, C, B, T2):
    """conv-1 into parity planes + conv-2 implicit GEMM against float64 conv2d: T2 = 1, 5, 6, 7 (below, at and above one
    6-row time tile; with B = 3 a partial tile's spare rows fall on the next utterance's rows and must not be written)
    and 248 (the 10 s shape).  At C = 512 a tap is 16 K-blocks = two 256-K accumulation chunks and N is four column tiles.
    fp32 and pair outputs; rows past B*T2*19 stay NaN."""
    Fm = 2 * (2 * T2 + 1 + T2 % 2) + 1                # odd F1 for even T2, even F1 for odd T2
    g = torch.Generator().manual_seed(B * 1000 + Fm + C)
    idim = 80
    feats = torch.randn(B, Fm, idim, generator=g) * 3 + 20
    mean = torch.randn(idim, generator=g) + 20
    istd = torch.rand(idim, generator=g) * 0.3 + 0.2
    w1, b1 = torch.randn(C, 1, 3, 3, generator=g) / 3, torch.randn(C, generator=g) / 3
    s2 = 3 * math.sqrt(C)
    w2, b2 = torch.randn(C, C, 3, 3, generator=g) / s2, torch.randn(C, generator=g) / s2
    F1, W1 = (Fm - 1) // 2, (idim - 1) // 2
    assert (F1 - 1) // 2 == T2
    W2, TH = (W1 - 1) // 2, (F1 + 1) // 2
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
    report(f"conv subsampling C={C} B={B} T2={T2}", conv1=e1, conv2=e2)
    assert e1 < 6e-6 and e2 < 7e-6 * (C // 256)


def test_conv2_rejects_other_widths(rt):
    from masr_b200._lib import MasrB200Error
    z = torch.zeros(4 * 2 * 20 * 384, dtype=torch.float16, device=rt.dev)
    o = torch.zeros(19, 384, device=rt.dev)
    with pytest.raises(MasrB200Error, match="C=384"):
        rt.call("masr_conv2_tc_f16x2", P(z), P(z), P(z), P(z), None, P(o), None, None, 1, 3, 1, 384, rt.st())
