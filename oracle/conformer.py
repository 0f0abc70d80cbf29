"""Oracle (test infrastructure): the reference Conformer inference forward, restated as plain
functions over a ``state_dict`` with torch CPU float32 ops (the reference's own arithmetic
library — ATen/oneDNN on CPU — so this is also the honest CPU baseline, ``kind: "port"``).

Follows:
  * ``GlobalCMVN.forward``                         masr/model_utils/utils/cmvn.py:21-32
  * ``Conv2dSubsampling4.forward``                 masr/model_utils/conformer/subsampling.py:93-112
  * ``PositionalEncoding.__init__`` (pe table)     masr/model_utils/conformer/embedding.py:10-37
  * ``RelPositionalEncoding.forward`` / ``position_encoding``  embedding.py:73-101,56-70
  * ``PositionwiseFeedForward.forward``            masr/model_utils/conformer/positionwise.py:30-37
  * ``RelPositionMultiHeadedAttention.forward`` + ``forward_attention``  conformer/attention.py:190-251,81-119
  * ``ConvolutionModule.forward``                  masr/model_utils/conformer/convolution.py:76-132
  * ``ConformerEncoderLayer.forward``              masr/model_utils/conformer/encoder.py:82-163
  * ``ConformerEncoder.forward`` / ``forward_chunk`` encoder.py:305-346,348-420
  * ``CTCLoss.softmax``                            masr/model_utils/loss/ctc.py:62-70
  * ``ConformerModel.get_encoder_out[_chunk]``     masr/model_utils/conformer/model.py:152-190

Semantics note (SURVEY.md §7 "hard parts"): the reference *API* is single-utterance; its padded
batch path differs slightly from its B=1 path.  The parity target is the B=1 semantics, so
``encode_batch`` here runs each utterance on its own, un-padded.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, List, Optional, Tuple

import torch
import torch.nn.functional as F


@dataclass
class ConformerConfig:
    input_dim: int = 80
    d_model: int = 256
    heads: int = 4
    ffn: int = 2048
    blocks: int = 12
    kernel: int = 15
    causal: bool = True          # configs/conformer.yml `streaming: True` -> causal conv (model.py:35-39)
    max_len: int = 5000
    ln_eps: float = 1e-5


def sinusoid_table(cfg: ConformerConfig) -> torch.Tensor:
    """embedding.py:31-37: pe[p, 2i] = sin(p * w_i), pe[p, 2i+1] = cos(p * w_i), float32."""
    pos = torch.arange(0, cfg.max_len, dtype=torch.float32).unsqueeze(1)
    div = torch.exp(torch.arange(0, cfg.d_model, 2, dtype=torch.float32) * -(math.log(10000.0) / cfg.d_model))
    pe = torch.zeros(cfg.max_len, cfg.d_model)
    pe[:, 0::2] = torch.sin(pos * div)
    pe[:, 1::2] = torch.cos(pos * div)
    return pe


def subsample(sd, cfg: ConformerConfig, feats: torch.Tensor) -> torch.Tensor:
    """[B, F, 80] raw log-mel -> [B, T, d] (CMVN, two stride-2 convs + ReLU, linear, x sqrt(d))."""
    x = (feats - sd["encoder.global_cmvn.mean"]) * sd["encoder.global_cmvn.istd"]
    x = x.unsqueeze(1)
    x = F.relu(F.conv2d(x, sd["encoder.embed.conv.0.weight"], sd["encoder.embed.conv.0.bias"], stride=2))
    x = F.relu(F.conv2d(x, sd["encoder.embed.conv.2.weight"], sd["encoder.embed.conv.2.bias"], stride=2))
    b, c, t, f = x.shape
    x = x.transpose(1, 2).reshape(b, t, c * f)
    x = F.linear(x, sd["encoder.embed.out.0.weight"], sd["encoder.embed.out.0.bias"])
    return x * math.sqrt(cfg.d_model)


def _ln(sd, name, x, eps):
    return F.layer_norm(x, (x.shape[-1],), sd[name + ".weight"], sd[name + ".bias"], eps)


def _ffn(sd, p, x):
    return F.linear(F.silu(F.linear(x, sd[p + ".w_1.weight"], sd[p + ".w_1.bias"])),
                    sd[p + ".w_2.weight"], sd[p + ".w_2.bias"])


def rel_attention(sd, p, cfg, x, pos_emb, att_cache: Optional[torch.Tensor], key_mask: Optional[torch.Tensor]):
    """x [B,T,d]; pos_emb [1,Tk,d]; att_cache [B,h,Tc,2*dk] or None; key_mask bool [B,Tk] or None.
    Returns (out [B,T,d], new_cache [B,h,Tk,2dk])."""
    B, T, d = x.shape
    h, dk = cfg.heads, cfg.d_model // cfg.heads
    q = F.linear(x, sd[p + "linear_q.weight"], sd[p + "linear_q.bias"]).view(B, T, h, dk)
    k = F.linear(x, sd[p + "linear_k.weight"], sd[p + "linear_k.bias"]).view(B, T, h, dk).transpose(1, 2)
    v = F.linear(x, sd[p + "linear_v.weight"], sd[p + "linear_v.bias"]).view(B, T, h, dk).transpose(1, 2)
    if att_cache is not None and att_cache.numel() > 0:
        k = torch.cat([att_cache[..., :dk], k], dim=2)
        v = torch.cat([att_cache[..., dk:], v], dim=2)
    new_cache = torch.cat([k, v], dim=-1)
    pos = F.linear(pos_emb, sd[p + "linear_pos.weight"]).view(1, -1, h, dk).transpose(1, 2)
    qu = (q + sd[p + "pos_bias_u"]).transpose(1, 2)
    qv = (q + sd[p + "pos_bias_v"]).transpose(1, 2)
    # no rel_shift (attention.py:245-247): the positional term is indexed by *key* position
    scores = (qu @ k.transpose(-2, -1) + qv @ pos.transpose(-2, -1)) / math.sqrt(dk)
    if key_mask is not None:
        m = ~key_mask[:, None, None, :]
        attn = torch.softmax(scores.masked_fill(m, -float("inf")), dim=-1).masked_fill(m, 0.0)
    else:
        attn = torch.softmax(scores, dim=-1)
    ctx = (attn @ v).transpose(1, 2).reshape(B, T, d)
    return F.linear(ctx, sd[p + "linear_out.weight"], sd[p + "linear_out.bias"]), new_cache


def conv_module(sd, p, cfg, x, cnn_cache: Optional[torch.Tensor]):
    """x [B,T,d] (already norm_conv'ed).  Causal: the 14-frame left context (zeros or the cache)
    is prepended *before* pointwise_conv1, so padded frames contribute GLU(bias), not zero
    (convolution.py:101-109).  Returns (y [B,T,d], new_cache [B,d,lorder])."""
    xt = x.transpose(1, 2)
    lorder = cfg.kernel - 1 if cfg.causal else 0
    if lorder > 0:
        if cnn_cache is None or cnn_cache.numel() == 0:
            xt = F.pad(xt, (lorder, 0))
        else:
            xt = torch.cat([cnn_cache, xt], dim=2)
        new_cache = xt[:, :, -lorder:]
    else:
        new_cache = xt.new_zeros(0, 0, 0)
    y = F.conv1d(xt, sd[p + "pointwise_conv1.weight"], sd[p + "pointwise_conv1.bias"])
    y = F.glu(y, dim=1)
    y = F.conv1d(y, sd[p + "depthwise_conv.weight"], sd[p + "depthwise_conv.bias"],
                 padding=0 if lorder > 0 else (cfg.kernel - 1) // 2, groups=cfg.d_model)
    y = F.silu(_ln(sd, p + "norm", y.transpose(1, 2), 1e-5)).transpose(1, 2)
    y = F.conv1d(y, sd[p + "pointwise_conv2.weight"], sd[p + "pointwise_conv2.bias"])
    return y.transpose(1, 2), new_cache


def encoder_layer(sd, i, cfg, x, pos_emb, att_cache=None, cnn_cache=None, key_mask=None):
    p = f"encoder.encoders.{i}."
    eps = cfg.ln_eps
    x = x + 0.5 * _ffn(sd, p + "feed_forward_macaron", _ln(sd, p + "norm_ff_macaron", x, eps))
    a, new_att = rel_attention(sd, p + "self_attn.", cfg, _ln(sd, p + "norm_mha", x, eps), pos_emb, att_cache, key_mask)
    x = x + a
    c, new_cnn = conv_module(sd, p + "conv_module.", cfg, _ln(sd, p + "norm_conv", x, eps), cnn_cache)
    x = x + c
    x = x + 0.5 * _ffn(sd, p + "feed_forward", _ln(sd, p + "norm_ff", x, eps))
    return _ln(sd, p + "norm_final", x, eps), new_att, new_cnn


def encode(sd, cfg: ConformerConfig, feats: torch.Tensor, taps: Optional[dict] = None) -> torch.Tensor:
    """Full-context forward of ONE un-padded utterance batch ([B,F,80], all rows the same
    length): ``ConformerEncoder.forward(decoding_chunk_size=-1)`` -> [B,T,d] after ``after_norm``."""
    x = subsample(sd, cfg, feats)
    T = x.shape[1]
    pos_emb = sinusoid_table(cfg).to(x.dtype)[None, :T]      # (float32 table, widened for a float64 run)
    if taps is not None:
        taps["embed"] = x.clone()
    for i in range(cfg.blocks):
        x, _, _ = encoder_layer(sd, i, cfg, x, pos_emb)
        if taps is not None:
            taps[f"layer{i}"] = x.clone()
    return _ln(sd, "encoder.after_norm", x, cfg.ln_eps)


def ctc_probs(sd, enc: torch.Tensor) -> torch.Tensor:
    """loss/ctc.py:70."""
    return torch.softmax(F.linear(enc, sd["ctc.ctc_lo.weight"], sd["ctc.ctc_lo.bias"]), dim=2)


def get_encoder_out(sd, cfg, feats: torch.Tensor) -> torch.Tensor:
    """``ConformerModel.get_encoder_out`` for un-padded input -> probs [B,T,V]."""
    return ctc_probs(sd, encode(sd, cfg, feats))


def encode_batch(sd, cfg, feat_list: List[torch.Tensor]) -> List[torch.Tensor]:
    """B=1 semantics for a ragged batch: each utterance alone -> list of probs [T_i, V]."""
    return [get_encoder_out(sd, cfg, f[None])[0] for f in feat_list]


@dataclass
class ChunkState:
    offset: int = 0
    att_cache: Optional[torch.Tensor] = None   # [blocks, h, t, 2*dk]
    cnn_cache: Optional[torch.Tensor] = None   # [blocks, 1, d, lorder]


def get_encoder_out_chunk(sd, cfg, feats_chunk: torch.Tensor, st: ChunkState, required_cache_size: int = -1):
    """``ConformerModel.get_encoder_out_chunk`` + the caller's ``offset += T`` bookkeeping
    (inference_predictor.py:80-94).  feats_chunk [1, <=67, 80] -> probs [1, t, V]; updates ``st``."""
    x = subsample(sd, cfg, feats_chunk)
    chunk = x.shape[1]
    cache_t1 = 0 if st.att_cache is None else st.att_cache.shape[2]
    key_size = cache_t1 + chunk
    pe = sinusoid_table(cfg).to(x.dtype)           # (float32 table; the input's dtype so a float64 run stays float64)
    pos_emb = pe[None, st.offset - cache_t1: st.offset - cache_t1 + key_size]
    if required_cache_size < 0:
        start = 0
    elif required_cache_size == 0:
        start = key_size
    else:
        start = max(key_size - required_cache_size, 0)
    atts, cnns = [], []
    for i in range(cfg.blocks):
        ac = None if st.att_cache is None else st.att_cache[i:i + 1]
        cc = None if st.cnn_cache is None else st.cnn_cache[i]
        x, na, nc = encoder_layer(sd, i, cfg, x, pos_emb, ac, cc)
        atts.append(na[:, :, start:, :])
        cnns.append(nc)
    x = _ln(sd, "encoder.after_norm", x, cfg.ln_eps)
    st.att_cache = torch.cat(atts, dim=0)
    st.cnn_cache = torch.stack(cnns, dim=0)
    probs = ctc_probs(sd, x)
    st.offset += probs.shape[1]
    return probs
