"""GPU (-m gpu): each C-ABI kernel against a plain torch float32 CPU reference of the same op."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def rt():
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
    return None if t is None else t.data_ptr()


def maxdiff(a, b):
    return (a.detach().float().cpu() - b.detach().float().cpu()).abs().max().item()


def test_layernorm(rt):
    g = torch.Generator().manual_seed(1)
    x = torch.randn(517, 256, generator=g) * 3 + 1; ga = torch.randn(256, generator=g); be = torch.randn(256, generator=g)
    xd, gd, bd = x.to(rt.dev), ga.to(rt.dev), be.to(rt.dev)
    y = torch.empty_like(xd)
    rt.call("masr_layernorm_f32", P(xd), 256, P(gd), P(bd), P(y), 256, 517, 256, 1e-5, rt.st())
    assert maxdiff(y, F.layer_norm(x, (256,), ga, be, 1e-5)) < 1e-5
    rt.call("masr_layernorm_f32", P(xd), 256, P(gd), P(bd), P(xd), 256, 517, 256, 1e-5, rt.st())   # in place
    assert maxdiff(xd, y) == 0.0


@pytest.mark.parametrize("fn", ["masr_relpos_attention_f32", "masr_relpos_attention_tc", "masr_relpos_attention_tc5"])
@pytest.mark.parametrize("lens", [[5], [64, 1], [130, 77, 129], [200], [33, 248], [256, 0, 128, 255]])
def test_relpos_attention(rt, lens, fn):
    g = torch.Generator().manual_seed(sum(lens))
    B, T, H, dk = len(lens), max(lens), 4, 64
    d = H * dk
    qkv = torch.randn(B, T, 3 * d, generator=g)
    Ptab = torch.randn(T + 3, d, generator=g)
    u = torch.randn(H, dk, generator=g) * 0.3; v = torch.randn(H, dk, generator=g) * 0.3
    qd, pd, ud, vd = qkv.to(rt.dev), Ptab.to(rt.dev), u.to(rt.dev), v.to(rt.dev)
    ld = torch.tensor(lens, dtype=torch.int32, device=rt.dev)
    out = torch.full((B, T, d), float("nan"), device=rt.dev)
    if fn in ("masr_relpos_attention_tc", "masr_relpos_attention_tc5"):
        def split(x):
            x = x.contiguous()
            h = torch.empty(x.shape, dtype=torch.float16, device=rt.dev); l = torch.empty_like(h)
            rt.call("masr_split_f16", P(x), P(h), P(l), x.numel(), rt.st())
            return h, l
        qh, ql = split(qd)
        ph, pl = split(pd)
        extra = (Ptab.shape[0],) if fn.endswith("tc5") else ()
        oh = torch.full((B, T, d), float("nan"), dtype=torch.float16, device=rt.dev); ol = torch.full_like(oh, float("nan"))
        rt.call(fn, P(qd), 3 * d, T, qh.data_ptr() + 2 * d, ql.data_ptr() + 2 * d, qh.data_ptr() + 4 * d, ql.data_ptr() + 4 * d,
                3 * d, T, P(ph), P(pl), d, *extra, P(ud), P(vd), P(out), P(oh), P(ol), d, T, P(ld), P(ld), B, H, dk, T, rt.st())
        torch.cuda.synchronize()
        assert maxdiff(oh.float() + ol.float() / 2048.0, out) < 2e-6          # the (h,l) pair output reconstructs the fp32 one
    else:
        rt.call(fn, P(qd), 3 * d, T, qd.data_ptr() + 4 * d, qd.data_ptr() + 8 * d, 3 * d, T,
                P(pd), d, P(ud), P(vd), P(out), None, None, d, T, P(ld), P(ld), B, H, dk, T, rt.st())
    out = out.cpu()
    for b, n in enumerate(lens):
        if n == 0:
            assert torch.all(out[b] == 0)
            continue
        q = qkv[b, :n, :d].view(n, H, dk); k = qkv[b, :n, d:2 * d].view(n, H, dk).transpose(0, 1)
        vv = qkv[b, :n, 2 * d:].view(n, H, dk).transpose(0, 1)
        p = Ptab[:n].view(n, H, dk).transpose(0, 1)
        s = ((q + u).transpose(0, 1) @ k.transpose(1, 2) + (q + v).transpose(0, 1) @ p.transpose(1, 2)) / math.sqrt(dk)
        ref = (torch.softmax(s, -1) @ vv).transpose(0, 1).reshape(n, d)
        assert maxdiff(out[b, :n], ref) < 2e-5
        assert torch.all(out[b, n:] == 0)     # padded queries are written as zeros


@pytest.mark.parametrize("ks,causal", [(15, True), (15, False), (7, False), (31, True)])
def test_dwconv_ln_silu(rt, ks, causal):
    g = torch.Generator().manual_seed(ks)
    lens = [37, 9, 64]
    B, T, C = len(lens), max(lens), 256
    x = torch.randn(B, T, C, generator=g)
    w = torch.randn(C, 1, ks, generator=g) / math.sqrt(ks); b = torch.randn(C, generator=g) * 0.1
    ga = 1 + 0.1 * torch.randn(C, generator=g); be = 0.1 * torch.randn(C, generator=g)
    pad = torch.randn(C, generator=g)
    d = lambda t: t.contiguous().to(rt.dev)
    xd, wd, bd, gd, bed, padd = d(x), d(w.reshape(C, ks)), d(b), d(ga), d(be), d(pad)
    ld = torch.tensor(lens, dtype=torch.int32, device=rt.dev)
    y = torch.empty(B, T, C, device=rt.dev)
    lpad = ks - 1 if causal else (ks - 1) // 2
    rt.call("masr_dwconv_ln_silu_f32", P(xd), C, T, P(wd), P(bd), P(gd), P(bed), P(padd) if causal else None, P(y), None, None, C, T,
            P(ld), B, C, ks, lpad, T, 1e-5, rt.st())
    y = y.cpu()
    for i, n in enumerate(lens):
        xi = x[i, :n].t()[None]                                        # [1,C,n]
        if causal:
            xi = torch.cat([pad[None, :, None].expand(1, C, lpad), xi], dim=2)
            r = F.conv1d(xi, w, b, groups=C)
        else:
            r = F.conv1d(xi, w, b, padding=lpad, groups=C)
        ref = F.silu(F.layer_norm(r[0].t(), (C,), ga, be, 1e-5))
        assert maxdiff(y[i, :n], ref) < 2e-5


@pytest.mark.parametrize("lens,threads", [([160000] * 32, 8), ([5, 0, 400001, 17, 262144, 1], 4), ([1000], 8), ([300000] * 3, 1)])
def test_stage_waves(rt, lens, threads):
    """masr_stage_waves_f32: separate host arrays -> pinned buffer -> device, bit-identical to a plain concatenate."""
    import ctypes as C
    rng = np.random.default_rng(len(lens))
    waves = [rng.standard_normal(n).astype(np.float32) for n in lens]
    total = sum(lens)
    pinned = torch.empty(total + 16, dtype=torch.float32, pin_memory=True)
    dev = torch.full((total + 16,), float("nan"), device=rt.dev)
    ptrs = (C.c_void_p * len(lens))(*[w.ctypes.data for w in waves])
    lc = (C.c_int64 * len(lens))(*lens)
    rt.call("masr_stage_waves_f32", ptrs, lc, len(lens), pinned.data_ptr(), dev.data_ptr(), threads, rt.st())
    torch.cuda.synchronize()
    ref = np.concatenate(waves)
    assert np.array_equal(dev[:total].cpu().numpy(), ref)
    assert np.array_equal(pinned[:total].numpy(), ref)
    assert torch.isnan(dev[total:]).all()


def test_layernorm2_is_two_layernorms(rt):
    """masr_layernorm2_split_f16 == masr_layernorm_f32 followed by masr_layernorm_split_f16, bit for bit (in place too)."""
    g = torch.Generator().manual_seed(11)
    M, D = 1003, 256
    x = (torch.randn(M, D, generator=g) * 3 + 0.5).to(rt.dev)
    g1, b1, g2, b2 = (torch.randn(D, generator=g).to(rt.dev) for _ in range(4))
    y1 = torch.empty_like(x)
    rt.call("masr_layernorm_f32", P(x), D, P(g1), P(b1), P(y1), D, M, D, 1e-5, rt.st())
    y2 = torch.empty_like(x)
    rt.call("masr_layernorm_f32", P(y1), D, P(g2), P(b2), P(y2), D, M, D, 1e-5, rt.st())
    rh = torch.empty(M, D, dtype=torch.float16, device=rt.dev); rl = torch.empty_like(rh)
    rt.call("masr_layernorm_split_f16", P(y1), D, P(g2), P(b2), P(rh), P(rl), D, M, D, 1e-5, rt.st())
    xin = x.clone()
    o2 = torch.full_like(x, float("nan"))
    oh = torch.empty_like(rh); ol = torch.empty_like(rl)
    rt.call("masr_layernorm2_split_f16", P(xin), D, P(g1), P(b1), P(xin), P(g2), P(b2), P(o2), P(oh), P(ol), D, M, D, 1e-5, rt.st())
    torch.cuda.synchronize()
    assert torch.equal(xin, y1) and torch.equal(o2, y2) and torch.equal(oh, rh) and torch.equal(ol, rl)
    ref = F.layer_norm(F.layer_norm(x.cpu(), (D,), g1.cpu(), b1.cpu()), (D,), g2.cpu(), b2.cpu())
    assert maxdiff(o2, ref) < 2e-5


def test_stream_cache_bookkeeping(rt):
    """masr_stream_append_rows / masr_stream_shift_cache against plain indexing (fp16 pair form and fp32 form)."""
    g = torch.Generator().manual_seed(3)
    S, C, cap, d = 5, 16, 64, 256
    base = torch.tensor([0, 16, 32, 3, 48], dtype=torch.int32)
    cnt = torch.tensor([16, 0, 5, 16, 1], dtype=torch.int32)
    src_h = torch.randn(S * C, 3 * d, generator=g).half().to(rt.dev); src_l = torch.randn(S * C, 3 * d, generator=g).half().to(rt.dev)
    dst_h = torch.zeros(S * cap, 2 * d, dtype=torch.float16, device=rt.dev); dst_l = torch.zeros_like(dst_h)
    bd, cd = base.to(rt.dev), cnt.to(rt.dev)
    rt.call("masr_stream_append_rows", P(src_h), P(src_l), 3 * d * 2, d * 2, 2 * d * 2, P(dst_h), P(dst_l), 2 * d * 2, cap, P(bd), P(cd), C, S, rt.st())
    want_h = torch.zeros_like(dst_h); want_l = torch.zeros_like(dst_l)
    for s in range(S):
        for t in range(int(cnt[s])):
            want_h[s * cap + int(base[s]) + t] = src_h[s * C + t, d:]
            want_l[s * cap + int(base[s]) + t] = src_l[s * C + t, d:]
    assert torch.equal(dst_h, want_h) and torch.equal(dst_l, want_l)
    src32 = torch.randn(S * C, 2 * d, generator=g).to(rt.dev)
    dst32 = torch.zeros(S * cap, 2 * d, device=rt.dev)
    rt.call("masr_stream_append_rows", P(src32), None, 2 * d * 4, 0, 2 * d * 4, P(dst32), None, 2 * d * 4, cap, P(bd), P(cd), C, S, rt.st())
    for s in range(S):
        n = int(cnt[s])
        assert torch.equal(dst32[s * cap + int(base[s]): s * cap + int(base[s]) + n], src32[s * C: s * C + n])
    # slide the conv left context: rows [0, lorder) <- rows [n, n + lorder), overlapping moves included
    lorder, LC = 14, 30
    x = torch.randn(S, LC, d, generator=g).to(rt.dev)
    ref = x.clone()
    for s in range(S):
        n = int(cnt[s])
        if n:
            ref[s, :lorder] = x[s, n:n + lorder]
    y = x.clone()
    rt.call("masr_stream_shift_cache", P(y), None, LC, lorder, d * 4, P(cd), S, rt.st())
    assert torch.equal(y, ref)
    xh, xl = x.half(), (x * 3).half()
    rh, rl = xh.clone(), xl.clone()
    for s in range(S):
        n = int(cnt[s])
        if n:
            rh[s, :lorder] = xh[s, n:n + lorder]; rl[s, :lorder] = xl[s, n:n + lorder]
    rt.call("masr_stream_shift_cache", P(xh), P(xl), LC, lorder, d * 2, P(cd), S, rt.st())
    assert torch.equal(xh, rh) and torch.equal(xl, rl)
