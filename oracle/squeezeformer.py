"""Oracle (test infrastructure): Squeezeformer inference forward (full-context pass, B=1 semantics),
restated as plain torch-CPU functions over a ``state_dict``.

Follows masr/model_utils/squeezeformer/:
  * ``DepthwiseConv2DSubsampling4.forward``  subsampling.py:60-76  (x sqrt(d) is applied to the 4864-vector *before*
                                             ``input_proj``; ``dw_conv`` is a full Conv2d because dw_stride=False :44-45)
  * ``SqueezeformerEncoder.forward``         encoder.py:168-216    (preln; time reduce before block 5, recover before 11)
  * ``SqueezeformerEncoderLayer.forward``    encoder.py:412-463    (post-norm: MHA -> LN -> FFN -> LN -> Conv -> LN -> FFN -> LN)
  * ``RelPositionMultiHeadedAttention``      attention.py:88-167   (ada scale/bias on the q/k/v input, no rel_shift)
  * ``PositionwiseFeedForward.forward``      positionwise.py:49-59 (ada scale/bias, SiLU)
  * ``ConvolutionModule.forward``            convolution.py:92-148 (ada scale/bias, k=31, BatchNorm1d in eval mode)
  * ``TimeReductionLayer1D/Stream.forward``  time_reduction.py:53-76,174-197
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Optional

import torch
import torch.nn.functional as F

from . import conformer as oc


@dataclass
class SqueezeformerConfig:
    input_dim: int = 80
    d_model: int = 256
    heads: int = 4
    ffn: int = 2048
    blocks: int = 12
    kernel: int = 31
    causal: bool = True          # streaming: causal conv + 'stream' time reduction (squeezeformer/model.py:35-41)
    reduce_idx: int = 5
    recover_idx: int = 11
    max_len: int = 5000
    ln_eps: float = 1e-5
    bn_eps: float = 1e-5


def subsample(sd, cfg, feats):
    x = (feats - sd["encoder.global_cmvn.mean"]) * sd["encoder.global_cmvn.istd"]
    x = x.unsqueeze(1)
    x = F.relu(F.conv2d(x, sd["encoder.embed.pw_conv.weight"], sd["encoder.embed.pw_conv.bias"], stride=2))
    x = F.relu(F.conv2d(x, sd["encoder.embed.dw_conv.weight"], sd["encoder.embed.dw_conv.bias"], stride=2))
    b, c, t, f = x.shape
    x = x.permute(0, 2, 1, 3).contiguous().view(b, t, c * f)
    x = x * math.sqrt(cfg.d_model)
    return F.linear(x, sd["encoder.embed.input_proj.0.weight"], sd["encoder.embed.input_proj.0.bias"])


def _ln(sd, name, x, eps=1e-5):
    return F.layer_norm(x, (x.shape[-1],), sd[name + ".weight"], sd[name + ".bias"], eps)


def _ada(sd, p, x):
    return sd[p + "ada_scale"] * x + sd[p + "ada_bias"]


def attention(sd, p, cfg, x, pos_emb, cache=None, want_cache=False):
    """``cache`` [1,h,t,2*dk] = K|V of earlier chunks (attention.py:131-137); pos_emb covers cache + chunk."""
    B, T, d = x.shape
    h, dk = cfg.heads, cfg.d_model // cfg.heads
    xin = _ada(sd, p, x)
    q = F.linear(xin, sd[p + "linear_q.weight"], sd[p + "linear_q.bias"]).view(B, T, h, dk)
    k = F.linear(xin, sd[p + "linear_k.weight"], sd[p + "linear_k.bias"]).view(B, T, h, dk).transpose(1, 2)
    v = F.linear(xin, sd[p + "linear_v.weight"], sd[p + "linear_v.bias"]).view(B, T, h, dk).transpose(1, 2)
    if cache is not None and cache.numel() > 0:
        k = torch.cat([cache[..., :dk], k], dim=2)
        v = torch.cat([cache[..., dk:], v], dim=2)
    new_cache = torch.cat((k, v), dim=-1)
    pos = F.linear(pos_emb, sd[p + "linear_pos.weight"]).view(1, -1, h, dk).transpose(1, 2)
    qu = (q + sd[p + "pos_bias_u"]).transpose(1, 2)
    qv = (q + sd[p + "pos_bias_v"]).transpose(1, 2)
    scores = (qu @ k.transpose(-2, -1) + qv @ pos.transpose(-2, -1)) / math.sqrt(dk)
    ctx = (torch.softmax(scores, dim=-1) @ v).transpose(1, 2).reshape(B, T, d)
    out = F.linear(ctx, sd[p + "linear_out.weight"], sd[p + "linear_out.bias"])
    return (out, new_cache) if want_cache else out


def ffn(sd, p, x):
    x = _ada(sd, p, x)
    return F.linear(F.silu(F.linear(x, sd[p + "w_1.weight"], sd[p + "w_1.bias"])), sd[p + "w_2.weight"], sd[p + "w_2.bias"])


def conv_module(sd, p, cfg, x, cache=None, want_cache=False):
    """``cache`` [1,d,lorder]: the previous chunk's last (ada-scaled) input columns (convolution.py:119-127)."""
    xt = _ada(sd, p, x).transpose(1, 2)
    lorder = cfg.kernel - 1 if cfg.causal else 0
    if lorder > 0:
        if cache is None or cache.numel() == 0:
            xt = F.pad(xt, (lorder, 0))
        else:
            xt = torch.cat((cache, xt), dim=2)
    new_cache = xt[:, :, -lorder:] if lorder > 0 else xt.new_zeros(0, 0, 0)
    y = F.glu(F.conv1d(xt, sd[p + "pointwise_conv1.weight"], sd[p + "pointwise_conv1.bias"]), dim=1)
    y = F.conv1d(y, sd[p + "depthwise_conv.weight"], sd[p + "depthwise_conv.bias"],
                 padding=0 if lorder > 0 else (cfg.kernel - 1) // 2, groups=cfg.d_model)
    y = F.batch_norm(y, sd[p + "norm.running_mean"], sd[p + "norm.running_var"], sd[p + "norm.weight"], sd[p + "norm.bias"],
                     training=False, eps=cfg.bn_eps)
    y = F.conv1d(F.silu(y), sd[p + "pointwise_conv2.weight"], sd[p + "pointwise_conv2.bias"])
    return (y.transpose(1, 2), new_cache) if want_cache else y.transpose(1, 2)


def encoder_layer(sd, i, cfg, x, pos_emb):
    p = f"encoder.encoders.{i}."
    x = _ln(sd, p + "layer_norm1", x + attention(sd, p + "self_attn.", cfg, x, pos_emb))
    x = _ln(sd, p + "layer_norm2", x + ffn(sd, p + "ffn1.", x))
    x = _ln(sd, p + "layer_norm3", x + conv_module(sd, p + "conv_module.", cfg, x))
    return _ln(sd, p + "layer_norm4", x + ffn(sd, p + "ffn2.", x))


def time_reduce(sd, cfg, x):
    p = "encoder.time_reduction_layer."
    T = x.shape[1]
    xt = x.transpose(1, 2)
    if cfg.causal:      # TimeReductionLayerStream: k=1, s=2, p=0
        y = F.conv1d(xt, sd[p + "dw_conv.weight"], sd[p + "dw_conv.bias"], stride=2, groups=cfg.d_model)
    else:               # TimeReductionLayer1D: k=5, s=2, p=3
        y = F.conv1d(xt, sd[p + "dw_conv.weight"], sd[p + "dw_conv.bias"], stride=2, padding=3, groups=cfg.d_model)
    y = F.conv1d(y, sd[p + "pw_conv.weight"], sd[p + "pw_conv.bias"]).transpose(1, 2)
    L = (T + 1) // 2    # mask_pad[:, :, ::2]
    if y.shape[1] > L:
        y = y[:, :L]
    elif y.shape[1] < L:
        y = torch.cat([y, y.new_zeros(y.shape[0], L - y.shape[1], y.shape[2])], dim=1)
    return y


def encode(sd, cfg: SqueezeformerConfig, feats: torch.Tensor, taps: Optional[dict] = None) -> torch.Tensor:
    x = subsample(sd, cfg, feats)
    T = x.shape[1]
    pos_emb = oc.sinusoid_table(oc.ConformerConfig(d_model=cfg.d_model, max_len=cfg.max_len)).to(x.dtype)[None, :T]
    x = _ln(sd, "encoder.preln", x)
    saved = None
    for i in range(cfg.blocks):
        if i == cfg.reduce_idx:
            saved = (x, pos_emb)
            x = time_reduce(sd, cfg, x)
            pos_emb = pos_emb[:, ::2]
        if i == cfg.recover_idx:
            rec_x, rec_pos = saved
            x = torch.repeat_interleave(x, 2, dim=1)
            x = F.linear(x, sd["encoder.time_recover_layer.weight"], sd["encoder.time_recover_layer.bias"])
            x = rec_x + x[:, :rec_x.shape[1]]
            pos_emb = rec_pos
        x = encoder_layer(sd, i, cfg, x, pos_emb)
        if taps is not None:
            taps[f"layer{i}"] = x.clone()
    return x


def get_encoder_out(sd, cfg, feats: torch.Tensor) -> torch.Tensor:
    return oc.ctc_probs(sd, encode(sd, cfg, feats))


# ---- chunk (streaming) forward ------------------------------------------------------------------------------------
@dataclass
class ChunkState:
    offset: int = 0
    att_cache: Optional[torch.Tensor] = None   # [blocks, h, t, 2*dk], every block at the FULL frame rate (encoder.py:349-356)
    cnn_cache: Optional[torch.Tensor] = None   # [blocks, 1, d, lorder]


def _factor(cfg, i):
    """``calculate_downsampling_factor`` (encoder.py:222-238) for one reduce / one recover index."""
    return 2 if cfg.reduce_idx <= i < cfg.recover_idx else 1


def encoder_layer_chunk(sd, i, cfg, x, pos_emb, att_cache, cnn_cache):
    p = f"encoder.encoders.{i}."
    a, new_att = attention(sd, p + "self_attn.", cfg, x, pos_emb, att_cache, want_cache=True)
    x = _ln(sd, p + "layer_norm1", x + a)
    x = _ln(sd, p + "layer_norm2", x + ffn(sd, p + "ffn1.", x))
    c, new_cnn = conv_module(sd, p + "conv_module.", cfg, x, cnn_cache, want_cache=True)
    x = _ln(sd, p + "layer_norm3", x + c)
    return _ln(sd, p + "layer_norm4", x + ffn(sd, p + "ffn2.", x)), new_att, new_cnn


def get_encoder_out_chunk(sd, cfg: SqueezeformerConfig, feats_chunk: torch.Tensor, st: ChunkState, required_cache_size: int = -1):
    """``SqueezeformerModel.get_encoder_out_chunk`` = ``SqueezeformerEncoder.forward_chunk`` (encoder.py:240-361) + CTC
    softmax, plus the caller's ``offset += T`` (inference_predictor.py:80-94).  feats_chunk [1, <=67, 80] -> probs [1,t,V].
    The reference keeps every block's K|V cache at the full frame rate: reduced blocks read it with ``[::2]`` and write it
    back with ``repeat_interleave(2)`` trimmed to block 0's length (:339-356)."""
    assert cfg.causal, "chunk decoding needs the streaming model"
    x = subsample(sd, cfg, feats_chunk)
    chunk = x.shape[1]
    cache_t1 = 0 if st.att_cache is None else st.att_cache.shape[2]
    key_size = cache_t1 + chunk
    pe = oc.sinusoid_table(oc.ConformerConfig(d_model=cfg.d_model, max_len=cfg.max_len)).to(x.dtype)
    pos_emb = pe[None, st.offset - cache_t1: st.offset - cache_t1 + key_size]
    if required_cache_size < 0:
        start = 0
    elif required_cache_size == 0:
        start = key_size
    else:
        start = max(key_size - required_cache_size, 0)
    x = _ln(sd, "encoder.preln", x)
    atts, cnns = [], []
    saved = None
    max_att_len = 0
    for i in range(cfg.blocks):
        if i == cfg.reduce_idx:
            saved = (x, pos_emb)
            x = time_reduce(sd, cfg, x)
            pos_emb = pos_emb[:, ::2]
        if i == cfg.recover_idx:
            rec_x, rec_pos = saved
            x = torch.repeat_interleave(x, 2, dim=1)
            x = F.linear(x, sd["encoder.time_recover_layer.weight"], sd["encoder.time_recover_layer.bias"])
            x = rec_x + x[:, :rec_x.shape[1]]
            pos_emb = rec_pos
        f = _factor(cfg, i)
        ac = None
        if st.att_cache is not None:
            ac = st.att_cache[i:i + 1][:, :, ::f, :][:, :, :pos_emb.shape[1] - x.shape[1], :]
        cc = None if st.cnn_cache is None else st.cnn_cache[i]
        x, na, nc = encoder_layer_chunk(sd, i, cfg, x, pos_emb, ac, cc)
        cached = na[:, :, start // f:, :].repeat_interleave(f, dim=2)
        if i == 0:
            max_att_len = cached.shape[2]
        atts.append(cached[:, :, :max_att_len, :])
        cnns.append(nc)
    st.att_cache = torch.cat(atts, dim=0)
    st.cnn_cache = torch.stack(cnns, dim=0)
    probs = oc.ctc_probs(sd, x)
    st.offset += probs.shape[1]
    return probs
