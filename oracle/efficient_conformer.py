"""Oracle (test infrastructure): EfficientConformer inference forward, restated as plain torch-CPU
functions over a ``state_dict`` (full-context pass; B=1 semantics).

Follows masr/model_utils/efficient_conformer/:
  * ``EfficientConformerEncoder.forward``            encoder.py:213-265 (grouped attention in blocks 0-3, strided conv
                                                     block 3, kernel 15 -> 7, pos_emb/masks re-strided :253-258)
  * ``StrideConformerEncoderLayer.forward``          encoder.py:454-545 (AvgPool1d(2,2,ceil_mode) on the residual :520-523)
  * ``GroupedRelPositionMultiHeadedAttention``       attention.py:35-69 (pad4group: the ``view`` regroups the [t,h,d_k]
                                                     memory of 3 consecutive frames into 4 heads x 192), :120-182
  * ``ConvolutionModule.forward`` (stride)           convolution.py:73-134
The un-grouped blocks and the FFN / subsampling are the Conformer ones (oracle/conformer.py).
Config trap (SURVEY.md §5): ``encoder_conf.efficient_conf`` is swallowed by ``**kwargs``; the constructor
defaults apply (stride_layer_idx=3, stride=2, group_layer_idx=(0,1,2,3), group_size=3, stride_kernel=True).
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Optional

import torch
import torch.nn.functional as F

from . import conformer as oc


@dataclass
class EfficientConfig(oc.ConformerConfig):
    stride_layer: int = 3
    stride: int = 2
    group_layers: tuple = (0, 1, 2, 3)
    group_size: int = 3

    def kernel_of(self, i: int) -> int:
        return self.kernel if i <= self.stride_layer else self.kernel // self.stride


def grouped_attention(sd, p, cfg: EfficientConfig, x, pos_emb):
    """x [B,T,d]; pos_emb [1,T,d] -> [B,T,d] (no cache, full mask)."""
    B, T, d = x.shape
    h, dk, g = cfg.heads, cfg.d_model // cfg.heads, cfg.group_size
    q = F.linear(x, sd[p + "linear_q.weight"], sd[p + "linear_q.bias"])
    k = F.linear(x, sd[p + "linear_k.weight"], sd[p + "linear_k.bias"])
    v = F.linear(x, sd[p + "linear_v.weight"], sd[p + "linear_v.bias"])
    pos = F.linear(pos_emb, sd[p + "linear_pos.weight"])
    pad = (g - T % g) % g
    # [B,T,d] rows of h*dk floats; zero-pad time to a multiple of g and regroup 3 frames x 256 -> 4 heads x 192
    def regroup(t):
        t = F.pad(t, (0, 0, 0, pad))
        return t.reshape(t.shape[0], -1, h, dk * g).transpose(1, 2)          # [B,h,T/g,dk*g]
    qg, kg, vg, pg = regroup(q), regroup(k), regroup(v), regroup(pos)
    qu = qg + sd[p + "pos_bias_u"][None, :, None, :]
    qv = qg + sd[p + "pos_bias_v"][None, :, None, :]
    scores = (qu @ kg.transpose(-2, -1) + qv @ pg.transpose(-2, -1)) / math.sqrt(dk * g)
    ctx = torch.softmax(scores, dim=-1) @ vg                                 # [B,h,T/g,dk*g]
    ctx = ctx.transpose(1, 2).reshape(B, -1, d)
    if pad:
        ctx = ctx[:, :ctx.shape[1] - pad]
    return F.linear(ctx, sd[p + "linear_out.weight"], sd[p + "linear_out.bias"])


def conv_module(sd, p, cfg: EfficientConfig, x, kernel: int, stride: int):
    xt = x.transpose(1, 2)
    lorder = kernel - 1 if cfg.causal else 0
    if lorder > 0:
        xt = F.pad(xt, (lorder, 0))
    y = F.glu(F.conv1d(xt, sd[p + "pointwise_conv1.weight"], sd[p + "pointwise_conv1.bias"]), dim=1)
    y = F.conv1d(y, sd[p + "depthwise_conv.weight"], sd[p + "depthwise_conv.bias"], stride=stride,
                 padding=0 if lorder > 0 else (kernel - 1) // 2, groups=cfg.d_model)
    y = F.silu(F.layer_norm(y.transpose(1, 2), (cfg.d_model,), sd[p + "norm.weight"], sd[p + "norm.bias"], 1e-5)).transpose(1, 2)
    y = F.conv1d(y, sd[p + "pointwise_conv2.weight"], sd[p + "pointwise_conv2.bias"])
    return y.transpose(1, 2)


def encoder_layer(sd, i, cfg: EfficientConfig, x, pos_emb):
    p = f"encoder.encoders.{i}."
    eps = cfg.ln_eps
    x = x + 0.5 * oc._ffn(sd, p + "feed_forward_macaron", oc._ln(sd, p + "norm_ff_macaron", x, eps))
    xn = oc._ln(sd, p + "norm_mha", x, eps)
    if i in cfg.group_layers:
        a = grouped_attention(sd, p + "self_attn.", cfg, xn, pos_emb)
    else:
        a, _ = oc.rel_attention(sd, p + "self_attn.", cfg, xn, pos_emb, None, None)
    x = x + a
    strided = i == cfg.stride_layer
    c = conv_module(sd, p + "conv_module.", cfg, oc._ln(sd, p + "norm_conv", x, eps), cfg.kernel_of(i),
                    cfg.stride if strided else 1)
    res = x
    if strided:
        res = F.avg_pool1d(x.transpose(1, 2), cfg.stride, cfg.stride, 0, ceil_mode=True, count_include_pad=False).transpose(1, 2)
    x = res + c
    x = x + 0.5 * oc._ffn(sd, p + "feed_forward", oc._ln(sd, p + "norm_ff", x, eps))
    return oc._ln(sd, p + "norm_final", x, eps)


def encode(sd, cfg: EfficientConfig, feats: torch.Tensor, taps: Optional[dict] = None) -> torch.Tensor:
    x = oc.subsample(sd, cfg, feats)
    pos_emb = oc.sinusoid_table(cfg).to(x.dtype)[None, :x.shape[1]]
    for i in range(cfg.blocks):
        x = encoder_layer(sd, i, cfg, x, pos_emb)
        if i == cfg.stride_layer:
            pos_emb = pos_emb[:, ::cfg.stride]
        if taps is not None:
            taps[f"layer{i}"] = x.clone()
    return oc._ln(sd, "encoder.after_norm", x, cfg.ln_eps)


def get_encoder_out(sd, cfg, feats: torch.Tensor) -> torch.Tensor:
    return oc.ctc_probs(sd, encode(sd, cfg, feats))


# ---- chunk (streaming) forward ------------------------------------------------------------------------------------
@dataclass
class ChunkState:
    offset: int = 0                            # in OUTPUT frames (80 ms): inference_predictor.py:93 adds probs.shape[1]
    att_cache: Optional[torch.Tensor] = None   # [blocks, h, t, 2*dk], every block stored at the full (40 ms) frame rate
    cnn_cache: Optional[torch.Tensor] = None   # [blocks, 1, d, kernel-1], left-padded with zeros for the k=7 blocks


def grouped_attention_chunk(sd, p, cfg: EfficientConfig, x, pos_emb, cache):
    """attention.py:120-182 with a K|V cache: keys = [cache ++ chunk] are zero-padded to a multiple of 3 and regrouped
    from key index 0, queries from the first frame of the chunk; returns (out, new_cache [1,h,t,2*dk])."""
    B, T, d = x.shape
    h, dk, g = cfg.heads, cfg.d_model // cfg.heads, cfg.group_size
    q = F.linear(x, sd[p + "linear_q.weight"], sd[p + "linear_q.bias"]).view(B, T, h, dk).transpose(1, 2)
    k = F.linear(x, sd[p + "linear_k.weight"], sd[p + "linear_k.bias"]).view(B, T, h, dk).transpose(1, 2)
    v = F.linear(x, sd[p + "linear_v.weight"], sd[p + "linear_v.bias"]).view(B, T, h, dk).transpose(1, 2)
    pos = F.linear(pos_emb, sd[p + "linear_pos.weight"])                     # [1, key_size, d]
    if cache is not None and cache.numel() > 0:
        k = torch.cat([cache[..., :dk], k], dim=2)
        v = torch.cat([cache[..., dk:], v], dim=2)
    new_cache = torch.cat((k, v), dim=-1)

    def regroup(t):                                                          # [B,h,t,dk] -> [B,h,ceil(t/g),dk*g]
        pad = (g - t.shape[2] % g) % g
        t = F.pad(t, (0, 0, 0, pad))
        return t.transpose(1, 2).contiguous().view(B, -1, h, dk * g).transpose(1, 2), pad
    qg, pad_q = regroup(q)
    kg, _ = regroup(k)
    vg, _ = regroup(v)
    pad_p = (g - pos.shape[1] % g) % g
    pg = F.pad(pos, (0, 0, 0, pad_p)).view(1, -1, h, dk * g).transpose(1, 2)
    qu = qg + sd[p + "pos_bias_u"][None, :, None, :]
    qv = qg + sd[p + "pos_bias_v"][None, :, None, :]
    scores = (qu @ kg.transpose(-2, -1) + qv @ pg.transpose(-2, -1)) / math.sqrt(dk * g)
    ctx = (torch.softmax(scores, dim=-1) @ vg).transpose(1, 2).contiguous().view(B, -1, d)
    if pad_q:
        ctx = ctx[:, :ctx.shape[1] - pad_q]
    return F.linear(ctx, sd[p + "linear_out.weight"], sd[p + "linear_out.bias"]), new_cache


def conv_module_chunk(sd, p, cfg: EfficientConfig, x, kernel: int, stride: int, cache):
    """convolution.py:73-134 with a left-context cache (only its last kernel-1 columns are used, :101-104)."""
    xt = x.transpose(1, 2)
    lorder = kernel - 1
    if cache is None or cache.numel() == 0:
        xt = F.pad(xt, (lorder, 0))
    else:
        xt = torch.cat((cache[:, :, -lorder:], xt), dim=2)
    new_cache = xt[:, :, -lorder:]
    y = F.glu(F.conv1d(xt, sd[p + "pointwise_conv1.weight"], sd[p + "pointwise_conv1.bias"]), dim=1)
    y = F.conv1d(y, sd[p + "depthwise_conv.weight"], sd[p + "depthwise_conv.bias"], stride=stride, groups=cfg.d_model)
    y = F.silu(F.layer_norm(y.transpose(1, 2), (cfg.d_model,), sd[p + "norm.weight"], sd[p + "norm.bias"], 1e-5)).transpose(1, 2)
    y = F.conv1d(y, sd[p + "pointwise_conv2.weight"], sd[p + "pointwise_conv2.bias"])
    return y.transpose(1, 2), new_cache


def get_encoder_out_chunk(sd, cfg: EfficientConfig, feats_chunk: torch.Tensor, st: ChunkState, required_cache_size: int = -1):
    """``EfficientConformerModel.get_encoder_out_chunk`` = ``EfficientConformerEncoder.forward_chunk`` (encoder.py:267-392)
    + CTC softmax + the caller's ``offset += T_out`` (inference_predictor.py:80-94).  feats_chunk [1,<=67,80] -> probs [1,t,V]."""
    assert cfg.causal, "chunk decoding needs the streaming model"
    eps = cfg.ln_eps
    offset = st.offset * cfg.stride                      # encoder.py:306: back to 40 ms frames
    x = oc.subsample(sd, cfg, feats_chunk)
    chunk = x.shape[1]
    cache_t1 = 0 if st.att_cache is None else st.att_cache.shape[2]
    key_size = cache_t1 + chunk
    pos_emb = oc.sinusoid_table(cfg).to(x.dtype)[None, offset - cache_t1: offset - cache_t1 + key_size]
    if required_cache_size < 0:
        start = 0
    elif required_cache_size == 0:
        start = key_size
    else:
        start = max(key_size - required_cache_size, 0)
    atts, cnns = [], []
    max_att_len = max_cnn_len = 0
    for i in range(cfg.blocks):
        f = cfg.stride if i > cfg.stride_layer else 1
        p = f"encoder.encoders.{i}."
        ac = None if st.att_cache is None else st.att_cache[i:i + 1, :, ::f, :]
        cc = None if st.cnn_cache is None else st.cnn_cache[i]
        x = x + 0.5 * oc._ffn(sd, p + "feed_forward_macaron", oc._ln(sd, p + "norm_ff_macaron", x, eps))
        xn = oc._ln(sd, p + "norm_mha", x, eps)
        if i in cfg.group_layers:
            a, na = grouped_attention_chunk(sd, p + "self_attn.", cfg, xn, pos_emb, ac)
        else:
            a, na = oc.rel_attention(sd, p + "self_attn.", cfg, xn, pos_emb, ac, None)
        x = x + a
        strided = i == cfg.stride_layer
        c, nc = conv_module_chunk(sd, p + "conv_module.", cfg, oc._ln(sd, p + "norm_conv", x, eps), cfg.kernel_of(i),
                                  cfg.stride if strided else 1, cc)
        res = x
        if strided:
            res = F.avg_pool1d(x.transpose(1, 2), cfg.stride, cfg.stride, 0, ceil_mode=True, count_include_pad=False).transpose(1, 2)
        x = res + c
        x = x + 0.5 * oc._ffn(sd, p + "feed_forward", oc._ln(sd, p + "norm_ff", x, eps))
        x = oc._ln(sd, p + "norm_final", x, eps)
        if strided:
            pos_emb = pos_emb[:, ::cfg.stride]
        na = na[:, :, start // f:, :].repeat_interleave(f, dim=2)
        nc = F.pad(nc.unsqueeze(0), (cfg.kernel - 1 - nc.shape[2], 0))
        if i == 0:
            max_att_len, max_cnn_len = na.shape[2], nc.shape[3]
        atts.append(na[:, :, -max_att_len:, :])
        cnns.append(nc[:, :, :, -max_cnn_len:])
    x = oc._ln(sd, "encoder.after_norm", x, eps)
    st.att_cache = torch.cat(atts, dim=0)
    st.cnn_cache = torch.cat(cnns, dim=0)
    probs = oc.ctc_probs(sd, x)
    st.offset += probs.shape[1]
    return probs
