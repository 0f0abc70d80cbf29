"""Squeezeformer engine (configs/squeezeformer.yml; masr/model_utils/squeezeformer/encoder.py:20-216).

Post-norm blocks MHA -> LN -> FFN -> LN -> Conv -> LN -> FFN -> LN with an adaptive scale/bias in front of every
sub-module, BatchNorm1d (eval) in the conv module, depthwise kernel 31, a stride-2 time reduction before block 5 and
a recovery (upsample + linear + skip) before block 11.  Whole-utterance (batched) path, tensor-core GEMMs; every row
of a ragged batch is computed as if alone (B=1 API semantics)."""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Dict, List

import torch

from ._lib import EPI_BIAS, EPI_BIAS_GLU, EPI_RESIDUAL
from .engine import ConformerEngine, _p, subsampled_len
from .weights import check_supported, sinusoid_table


@dataclass
class SqueezeLayer:
    att_ada: tuple = None
    wqkv: torch.Tensor = None
    bqkv: torch.Tensor = None
    wpos: torch.Tensor = None
    pos_u: torch.Tensor = None
    pos_v: torch.Tensor = None
    wo: torch.Tensor = None
    bo: torch.Tensor = None
    ln1: tuple = None
    ffn1_ada: tuple = None
    ffn1: tuple = None
    ln2: tuple = None
    conv_ada: tuple = None
    pw1: torch.Tensor = None
    pw1_b: torch.Tensor = None
    glu_pad: torch.Tensor = None
    dw: torch.Tensor = None
    dw_b: torch.Tensor = None
    bn: tuple = None            # folded (scale, shift)
    pw2: torch.Tensor = None
    pw2_b: torch.Tensor = None
    ln3: tuple = None
    ffn2_ada: tuple = None
    ffn2: tuple = None
    ln4: tuple = None
    ptab: torch.Tensor = None
    kernel: int = 31


@dataclass
class SqueezeWeights:
    d_model: int
    heads: int
    ffn: int
    kernel: int
    idim: int
    vocab: int
    max_len: int
    cmvn_mean: torch.Tensor = None
    cmvn_istd: torch.Tensor = None
    conv1_w: torch.Tensor = None
    conv1_b: torch.Tensor = None
    conv2_w: torch.Tensor = None
    conv2_b: torch.Tensor = None
    embed_w: torch.Tensor = None
    embed_b: torch.Tensor = None
    pe: torch.Tensor = None
    preln: tuple = None
    layers: List[SqueezeLayer] = field(default_factory=list)
    tr_dw: torch.Tensor = None
    tr_dw_b: torch.Tensor = None
    tr_pw: torch.Tensor = None
    tr_pw_b: torch.Tensor = None
    rec_w: torch.Tensor = None
    rec_b: torch.Tensor = None
    ctc_w: torch.Tensor = None
    ctc_b: torch.Tensor = None


def pack_squeezeformer(sd: Dict[str, torch.Tensor], device, max_len: int = 5000, bn_eps: float = 1e-5) -> SqueezeWeights:
    dev = torch.device(device)
    check_supported(sd, "squeezeformer")

    def D(t):
        return t.contiguous().to(dev)

    d = sd["encoder.preln.weight"].shape[0]
    h = sd["encoder.encoders.0.self_attn.pos_bias_u"].shape[0]
    ffn = sd["encoder.encoders.0.ffn1.w_1.weight"].shape[0]
    kernel = int(sd["encoder.encoders.0.conv_module.depthwise_conv.weight"].shape[2])
    idim = sd["encoder.global_cmvn.mean"].shape[0]
    vocab = sd["ctc.ctc_lo.weight"].shape[0]
    nblocks = 1 + max(int(k.split(".")[2]) for k in sd if k.startswith("encoder.encoders."))
    w = SqueezeWeights(d_model=d, heads=h, ffn=ffn, kernel=kernel, idim=idim, vocab=vocab, max_len=max_len)
    w.cmvn_mean, w.cmvn_istd = D(sd["encoder.global_cmvn.mean"]), D(sd["encoder.global_cmvn.istd"])
    w.conv1_w, w.conv1_b = D(sd["encoder.embed.pw_conv.weight"].reshape(d, 9)), D(sd["encoder.embed.pw_conv.bias"])
    assert sd["encoder.embed.dw_conv.weight"].shape[1] == d, "dw_stride=True subsampling is not supported"
    w.conv2_w = D(sd["encoder.embed.dw_conv.weight"].permute(0, 2, 3, 1).reshape(d, 9 * d))
    w.conv2_b = D(sd["encoder.embed.dw_conv.bias"])
    f2 = ((idim - 1) // 2 - 1) // 2
    ew = sd["encoder.embed.input_proj.0.weight"]
    # x*sqrt(d) is applied before input_proj (subsampling.py:74-75): fold the exact power-of-two scale into the weight
    xs = math.sqrt(d)
    assert xs == int(xs) and (int(xs) & (int(xs) - 1)) == 0, "sqrt(d_model) must be a power of two to fold exactly"
    w.embed_w = D((ew * xs).reshape(d, d, f2).permute(0, 2, 1).reshape(d, f2 * d))
    w.embed_b = D(sd["encoder.embed.input_proj.0.bias"])
    w.pe = D(sinusoid_table(d, max_len))

    def ln(name):
        return D(sd[name + ".weight"]), D(sd[name + ".bias"])

    def ada(p):
        return D(sd[p + "ada_scale"].reshape(d)), D(sd[p + "ada_bias"].reshape(d))

    def ffn_w(p):
        return (D(sd[p + "w_1.weight"]), D(sd[p + "w_1.bias"]), D(sd[p + "w_2.weight"]), D(sd[p + "w_2.bias"]))

    w.preln = ln("encoder.preln")
    for i in range(nblocks):
        p = f"encoder.encoders.{i}."
        a = p + "self_attn."
        L = SqueezeLayer()
        L.att_ada = ada(a)
        L.wqkv = D(torch.cat([sd[a + "linear_q.weight"], sd[a + "linear_k.weight"], sd[a + "linear_v.weight"]], 0))
        L.bqkv = D(torch.cat([sd[a + "linear_q.bias"], sd[a + "linear_k.bias"], sd[a + "linear_v.bias"]], 0))
        L.wpos, L.pos_u, L.pos_v = D(sd[a + "linear_pos.weight"]), D(sd[a + "pos_bias_u"]), D(sd[a + "pos_bias_v"])
        L.wo, L.bo = D(sd[a + "linear_out.weight"]), D(sd[a + "linear_out.bias"])
        L.ln1, L.ln2, L.ln3, L.ln4 = (ln(p + f"layer_norm{j}") for j in (1, 2, 3, 4))
        L.ffn1_ada, L.ffn1 = ada(p + "ffn1."), ffn_w(p + "ffn1.")
        L.ffn2_ada, L.ffn2 = ada(p + "ffn2."), ffn_w(p + "ffn2.")
        c = p + "conv_module."
        L.conv_ada = ada(c)
        pw1 = sd[c + "pointwise_conv1.weight"].reshape(2 * d, d)
        pb1 = sd[c + "pointwise_conv1.bias"]
        L.pw1 = D(torch.stack([pw1[:d], pw1[d:]], dim=1).reshape(2 * d, d))
        L.pw1_b = D(torch.stack([pb1[:d], pb1[d:]], dim=1).reshape(2 * d))
        L.glu_pad = D(torch.nn.functional.glu(pb1.reshape(1, 2 * d, 1), dim=1).reshape(d))
        L.kernel = int(sd[c + "depthwise_conv.weight"].shape[2])
        L.dw, L.dw_b = D(sd[c + "depthwise_conv.weight"].reshape(d, L.kernel)), D(sd[c + "depthwise_conv.bias"])
        scale = sd[c + "norm.weight"] / torch.sqrt(sd[c + "norm.running_var"] + bn_eps)
        L.bn = (D(scale), D(sd[c + "norm.bias"] - sd[c + "norm.running_mean"] * scale))
        L.pw2, L.pw2_b = D(sd[c + "pointwise_conv2.weight"].reshape(d, d)), D(sd[c + "pointwise_conv2.bias"])
        w.layers.append(L)
    t = "encoder.time_reduction_layer."
    w.tr_dw = D(sd[t + "dw_conv.weight"].reshape(d, -1))
    w.tr_dw_b = D(sd[t + "dw_conv.bias"])
    w.tr_pw, w.tr_pw_b = D(sd[t + "pw_conv.weight"].reshape(d, d)), D(sd[t + "pw_conv.bias"])
    w.rec_w, w.rec_b = D(sd["encoder.time_recover_layer.weight"]), D(sd["encoder.time_recover_layer.bias"])
    w.ctc_w, w.ctc_b = D(sd["ctc.ctc_lo.weight"]), D(sd["ctc.ctc_lo.bias"])
    return w


class SqueezeformerEngine(ConformerEngine):
    REDUCE, RECOVER = 5, 11

    def __init__(self, weights_src, streaming: bool = True, device: str = "cuda", max_len: int = 5000, gemm: str = "tc",
                 use_graphs: bool = True):
        if gemm != "tc":
            raise ValueError("SqueezeformerEngine implements the tensor-core path only")
        super().__init__(weights_src, streaming, device, max_len, gemm, use_graphs)

    def _half_rate(self, i: int) -> bool:
        return self.REDUCE <= i < self.RECOVER    # reduced-rate blocks see pos_emb[:, ::2] (encoder.py:194)

    def _embed_epilogue(self):
        return EPI_BIAS, 1.0                      # pack_squeezeformer folds the sqrt(d) scale into the embed weight

    def _pack(self, sd, max_len):
        return pack_squeezeformer(sd, self.device, max_len)

    def _split_weights(self):
        w, t = self.w, self._tcw
        t["conv2"], t["embed"], t["ctc"] = self._split(w.conv2_w), self._split(w.embed_w), self._split(w.ctc_w)
        t["tr_pw"], t["rec"] = self._split(w.tr_pw), self._split(w.rec_w)
        for i, L in enumerate(w.layers):
            t[i, "qkv"], t[i, "wo"] = self._split(L.wqkv), self._split(L.wo)
            t[i, "f1a"], t[i, "f1b"] = self._split(L.ffn1[0]), self._split(L.ffn1[2])
            t[i, "f2a"], t[i, "f2b"] = self._split(L.ffn2[0]), self._split(L.ffn2[2])
            t[i, "pw1"], t[i, "pw2"] = self._split(L.pw1), self._split(L.pw2)
        torch.cuda.synchronize(self.device)

    def new_stream(self, max_frames: int = 3000, keep_probs: bool = False):
        """Streaming state of one utterance (``InferencePredictor`` att/cnn caches + offset): a one-slot stream pool."""
        from .stream_pool import PoolStream, SqueezeformerStreamPool
        return PoolStream(SqueezeformerStreamPool(self, 1, max_frames, keep_probs=keep_probs))

    def encode_chunk(self, feats_chunk, st, required_cache_size: int = -1, want_probs: bool = False):
        """``SqueezeformerModel.get_encoder_out_chunk`` for one stream (encoder.py:240-361): feats_chunk [n<=67, 80] on device
        -> (ids, max-prob) device tensors of length ((n-1)//2-1)//2."""
        if want_probs and st.pool.probs is None:
            raise ValueError("create the stream with new_stream(keep_probs=True) to get the chunk posteriors")
        return st.encode_chunk(feats_chunk, required_cache_size)

    def _ln_ada(self, x, gb, y, ada, yp, M):
        self._k("layernorm", "masr_layernorm_ada_split_f16", _p(x), self.d, _p(gb[0]), _p(gb[1]), _p(y),
                None if ada is None else _p(ada[0]), None if ada is None else _p(ada[1]), _p(yp[0]), _p(yp[1]), self.d, M,
                self.d, 1e-5)

    def _dwconv(self, L, g, g_rows: int, lens, B: int, out_rows: int, out, cached: bool = False, stride: int = 1):
        """The conv module's depthwise conv + BatchNorm (eval) + SiLU (masr_dwconv_bn_silu_f32) -> the fp16 pair `out`."""
        assert stride == 1, "the Squeezeformer conv module has no strided form"
        d = self.d
        pad, lpad = self._dw_context(L, cached)
        self._k("dwconv_bn_silu", "masr_dwconv_bn_silu_f32", _p(g), d, g_rows, _p(L.dw), _p(L.dw_b), _p(L.bn[0]), _p(L.bn[1]),
                pad, None, _p(out[0]), _p(out[1]), d, out_rows, _p(lens), B, d, L.kernel, lpad, out_rows)

    def _encode_tc(self, feats, ws, tl, tlens, B, Fmax, T, M):
        w, d, tw = self.w, self.d, self._tcw
        x, g, qkv, y = ws["x"], ws["g"], ws["qkv"], ws["t1"]        # y: pre-LayerNorm sums
        t0p, t1p, hidp = ws["t0p"], ws["t1p"], self._hidp(ws)
        T2 = (T + 1) // 2
        if "tlens2" not in ws:
            ws["tlens2"] = torch.zeros(B, device=self.device, dtype=torch.int32)
            ws["saved"] = torch.empty(max(1, M), d, device=self.device, dtype=torch.float32)
        tlens2, saved = ws["tlens2"], ws["saved"]
        torch.div(tlens + 1, 2, rounding_mode="floor", out=tlens2)
        self._subsample(feats, ws, B, Fmax, T, y)
        # preln -> x (fp32 residual stream) + pair(ada_att0(x))
        self._ln_ada(y, w.preln, x, w.layers[0].att_ada, t0p, M)
        cur_T, cur_M, cur_lens = T, M, tlens
        nl = len(w.layers)
        for i, L in enumerate(w.layers):
            if i == self.REDUCE:
                # save the full-rate stream, reduce time by 2 (time_reduction.py), re-derive the attention input pair
                saved[:cur_M].copy_(x[:cur_M])
                k = w.tr_dw.shape[1]
                self._k("time_reduce", "masr_time_reduce_dw_split_f16", _p(x), cur_T, _p(w.tr_dw), _p(w.tr_dw_b), _p(t1p[0]),
                        _p(t1p[1]), T2, _p(cur_lens), B, T2, k, 0 if k == 1 else 3, d)
                M2 = B * T2
                self._tc(t1p, d, tw["tr_pw"], w.tr_pw_b, M2, d, d, EPI_BIAS, C=x, ldc=d, tag="time_reduce_pw")
                self._k("affine_split", "masr_affine_split_f16", _p(x), _p(L.att_ada[0]), _p(L.att_ada[1]), _p(t0p[0]),
                        _p(t0p[1]), M2, d)
                cur_T, cur_M, cur_lens = T2, M2, tlens2
            if i == self.RECOVER:
                # x (half rate) -> Linear -> upsample x2 + saved skip (encoder.py:198-204)
                self._k("affine_split", "masr_affine_split_f16", _p(x), None, None, _p(t1p[0]), _p(t1p[1]), cur_M, d)
                self._tc(t1p, d, tw["rec"], w.rec_b, cur_M, d, d, EPI_BIAS, C=y, ldc=d, tag="time_recover")
                self._k("upsample_add", "masr_upsample2_add_f32", _p(saved), _p(y), _p(x), T, T2, B, T, d)
                cur_T, cur_M, cur_lens = T, M, tlens
                self._k("affine_split", "masr_affine_split_f16", _p(x), _p(L.att_ada[0]), _p(L.att_ada[1]), _p(t0p[0]),
                        _p(t0p[1]), cur_M, d)
            Mi, Ti = cur_M, cur_T
            # MHA (input pair = ada(x) in t0p) -> y = x + out_proj(att) -> x = LN1(y), pair(ada_ffn1(x))
            self._tc(t0p, d, tw[i, "qkv"], L.bqkv, Mi, 3 * d, d, C=qkv, Cp=ws["qkvp"], ldc=3 * d, tag="qkv_proj")
            self._attention_tc(L, qkv, ws["qkvp"], t1p, Ti, cur_lens, B)
            self._tc(t1p, d, tw[i, "wo"], L.bo, Mi, d, d, EPI_RESIDUAL, 1.0, x, d, C=y, ldc=d, tag="out_proj")
            self._ln_ada(y, L.ln1, x, L.ffn1_ada, t0p, Mi)
            self._ffn_gemms(t0p, tw[i, "f1a"], L.ffn1[1], tw[i, "f1b"], L.ffn1[3], Mi, x, y, 1.0, hidp)
            self._ln_ada(y, L.ln2, x, L.conv_ada, t0p, Mi)
            # conv module
            self._tc(t0p, d, tw[i, "pw1"], L.pw1_b, Mi, 2 * d, d, EPI_BIAS_GLU, C=g, ldc=d, tag="pw1_glu")
            self._dwconv(L, g, Ti, cur_lens, B, Ti, t1p)
            self._tc(t1p, d, tw[i, "pw2"], L.pw2_b, Mi, d, d, EPI_RESIDUAL, 1.0, x, d, C=y, ldc=d, tag="pw2")
            self._ln_ada(y, L.ln3, x, L.ffn2_ada, t0p, Mi)
            self._ffn_gemms(t0p, tw[i, "f2a"], L.ffn2[1], tw[i, "f2b"], L.ffn2[3], Mi, x, y, 1.0, hidp)
            nxt = w.layers[i + 1].att_ada if (i + 1 < nl and i + 1 not in (self.REDUCE, self.RECOVER)) else None
            self._ln_ada(y, L.ln4, x, nxt, t0p, Mi)     # last block: pair(x) feeds the CTC head
        ws["tlens"] = cur_lens
        ws["tl_host"] = None
        return x[:cur_M], tl, cur_T, ws
