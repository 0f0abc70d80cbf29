"""Load the reference's weight formats and repack them for the CUDA kernels.

Accepted inputs (SURVEY.md §8b "weight / config formats"):
  * ``inference.pt`` — the TorchScript archive written by ``MASRTrainer.export``
    (masr/trainer.py:684-689); ``torch.jit.load(p).state_dict()`` yields the tensors;
  * ``model.pt`` — a plain ``state_dict`` checkpoint (masr/trainer.py:266-321);
  * an in-memory ``dict`` name -> tensor / ndarray (used with :mod:`masr_b200.synth`).

Repacking done once at load time (all of it layout, none of it arithmetic on activations):
  * conv #2 weight [co,ci,kh,kw] -> [co,kh,kw,ci]  (K-contiguous for the implicit GEMM);
  * ``embed.out`` weight columns (c*19+f) -> (f*256+c)  (conv #2 output is channels-last, so the
    ``transpose(1,2).reshape`` of subsampling.py:110 disappears);
  * q/k/v projection weights stacked into one [768,256] matrix;
  * ``pointwise_conv1`` rows interleaved (value_j, gate_j) for the GLU epilogue;
  * the sinusoid table ``pe`` is regenerated (it is a plain attribute, absent from the
    state_dict — embedding.py:31-37) with the *same torch CPU ops* as the reference, and
    ``linear_pos(pe)`` is precomputed per layer on the GPU (it is input-independent).
"""
from __future__ import annotations

import math
import os
from dataclasses import dataclass, field
from typing import Dict, List, Optional

import numpy as np
import torch


def load_state_dict(src) -> Dict[str, torch.Tensor]:
    """``src``: path to inference.pt / model.pt, or a mapping of tensors / ndarrays."""
    if isinstance(src, (str, os.PathLike)):
        if not os.path.exists(src):
            raise Exception("模型文件不存在，请检查{}是否存在！".format(src))  # predict.py:76-77
        try:
            sd = torch.jit.load(src, map_location="cpu").state_dict()
        except Exception:
            sd = torch.load(src, map_location="cpu")
            if isinstance(sd, dict) and "state_dict" in sd:
                sd = sd["state_dict"]
    else:
        sd = src
    out = {}
    for k, v in sd.items():
        if isinstance(v, np.ndarray):
            v = torch.from_numpy(np.ascontiguousarray(v))
        out[k] = v.detach().to(torch.float32).cpu().contiguous() if torch.is_floating_point(v) else v.detach().cpu()
    return out


def sinusoid_table(d_model: int, max_len: int) -> torch.Tensor:
    """embedding.py:31-37, same op sequence on the CPU -> bit-identical table."""
    position = torch.arange(0, max_len, dtype=torch.float32).unsqueeze(1)
    div_term = torch.exp(torch.arange(0, d_model, 2, dtype=torch.float32) * -(math.log(10000.0) / d_model))
    pe = torch.zeros(max_len, d_model)
    pe[:, 0::2] = torch.sin(position * div_term)
    pe[:, 1::2] = torch.cos(position * div_term)
    return pe


@dataclass
class ConformerLayerWeights:
    ln_ffm: tuple = None
    ffm: tuple = None           # (w1, b1, w2, b2)
    ln_mha: tuple = None
    wqkv: torch.Tensor = None
    bqkv: torch.Tensor = None
    wpos: torch.Tensor = None
    pos_u: torch.Tensor = None
    pos_v: torch.Tensor = None
    wo: torch.Tensor = None
    bo: torch.Tensor = None
    ln_conv: tuple = None
    pw1: torch.Tensor = None    # interleaved [2d, d]
    pw1_b: torch.Tensor = None
    glu_pad: torch.Tensor = None
    dw: torch.Tensor = None     # [d, k]
    dw_b: torch.Tensor = None
    cn: tuple = None            # conv-module LayerNorm
    pw2: torch.Tensor = None
    pw2_b: torch.Tensor = None
    ln_ff: tuple = None
    ff: tuple = None
    ln_final: tuple = None
    ptab: torch.Tensor = None   # linear_pos(pe) [max_len, d], filled by the engine
    kernel: int = 15            # depthwise kernel size of this block
    grouped: bool = False       # EfficientConformer grouped attention (pos_bias [h, group*d_k])


@dataclass
class ConformerWeights:
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
    layers: List[ConformerLayerWeights] = field(default_factory=list)
    after_norm: tuple = None
    ctc_w: torch.Tensor = None
    ctc_b: torch.Tensor = None


class UnsupportedConfig(ValueError):
    """The checkpoint comes from a reference configuration this build has no kernels for."""


def check_supported(sd: Dict[str, torch.Tensor], family: str = "conformer") -> None:
    """Fail loudly on supported-by-the-reference variants this build does not implement, instead of mis-packing them
    (the packers read architecture from tensor names and shapes): ``cnn_module_norm='batch_norm'`` in a Conformer /
    EfficientConformer (convolution.py:60-63: same ``conv_module.norm.weight`` key as the LayerNorm variant, plus running
    statistics), ``input_layer`` conv2d6 / conv2d8 (subsampling.py:115-236: extra ``embed.conv.4``), attention heads that
    are not 64 wide, model widths without kernels (Conformer: 256 and 512; Squeezeformer, EfficientConformer: 256).  A DeepSpeech2 checkpoint is an LSTM one (``encoder.rnns.{l}.rnn.*``, 4H gate rows) or a GRU one
    (``use_gru: True``: the reference's ``GRU`` wrapper nests ``nn.GRU`` one level deeper, ``encoder.rnns.{l}.rnn.rnn.*``,
    3H gate rows; deepspeech2/encoder.py:24-33, gru.py:6-15); 3H-row tensors under the LSTM names are no layout the
    reference writes."""
    keys = sd.keys()
    if family in ("conformer", "efficient_conformer") and any(k.endswith("conv_module.norm.running_mean") for k in keys):
        raise UnsupportedConfig("unsupported config: cnn_module_norm='batch_norm' (this build implements the shipped "
                                "layer_norm conv module for conformer / efficient_conformer)")
    if any(k.startswith("encoder.embed.conv.4.") for k in keys):
        raise UnsupportedConfig("unsupported config: input_layer conv2d6/conv2d8 (this build implements conv2d = Conv2dSubsampling4)")
    if family == "deepspeech2":
        hh = sd.get("encoder.rnns.0.rnn.weight_hh_l0")
        if hh is not None and hh.shape[0] != 4 * hh.shape[1]:          # GRU: 3 gates, LSTM: 4
            raise UnsupportedConfig(f"unsupported layout: {hh.shape[0]}-row recurrent weights under the LSTM key names "
                                    "(use_gru=True checkpoints keep their GRU under encoder.rnns.{l}.rnn.rnn.*)")
        hh = sd.get("encoder.rnns.0.rnn.rnn.weight_hh_l0")
        if hh is not None and hh.shape[0] != 3 * hh.shape[1]:
            raise UnsupportedConfig(f"unsupported layout: {hh.shape[0]}-row recurrent weights under the GRU key names "
                                    "(use_gru=True: 3 gates)")
        return
    dn = sd.get("encoder.after_norm.weight", sd.get("encoder.preln.weight"))
    u = sd.get("encoder.encoders.0.self_attn.pos_bias_u")
    if u is not None and dn is not None:
        d = dn.shape[0]
        if d % u.shape[0] or d // u.shape[0] != 64:
            raise UnsupportedConfig(f"unsupported config: attention heads of width {d / u.shape[0]:g} (this build: d_k = 64, "
                                    "e.g. output_size 256 / attention_heads 4)")
    if dn is not None:
        d = dn.shape[0]
        widths = (256, 512) if family == "conformer" else (256,)
        if d not in widths:
            raise UnsupportedConfig(f"unsupported config: output_size {d} for {family} (this build has kernels for "
                                    f"output_size {' and '.join(str(x) for x in widths)})")


def pack_conformer(sd: Dict[str, torch.Tensor], device, max_len: int = 5000, family: str = "conformer") -> ConformerWeights:
    dev = torch.device(device)
    check_supported(sd, family)

    def D(t):
        return t.contiguous().to(dev)

    d = sd["encoder.after_norm.weight"].shape[0]
    h = sd["encoder.encoders.0.self_attn.pos_bias_u"].shape[0]
    ffn = sd["encoder.encoders.0.feed_forward.w_1.weight"].shape[0]
    kernel = sd["encoder.encoders.0.conv_module.depthwise_conv.weight"].shape[2]
    idim = sd["encoder.global_cmvn.mean"].shape[0]
    vocab = sd["ctc.ctc_lo.weight"].shape[0]
    nblocks = 1 + max(int(k.split(".")[2]) for k in sd if k.startswith("encoder.encoders."))
    w = ConformerWeights(d_model=d, heads=h, ffn=ffn, kernel=kernel, idim=idim, vocab=vocab, max_len=max_len)
    w.cmvn_mean = D(sd["encoder.global_cmvn.mean"])
    w.cmvn_istd = D(sd["encoder.global_cmvn.istd"])
    w.conv1_w = D(sd["encoder.embed.conv.0.weight"].reshape(d, 9))
    w.conv1_b = D(sd["encoder.embed.conv.0.bias"])
    w.conv2_w = D(sd["encoder.embed.conv.2.weight"].permute(0, 2, 3, 1).reshape(d, 9 * d))
    w.conv2_b = D(sd["encoder.embed.conv.2.bias"])
    f2 = ((idim - 1) // 2 - 1) // 2
    ew = sd["encoder.embed.out.0.weight"]                      # [d, c*f2 + f]
    w.embed_w = D(ew.reshape(d, d, f2).permute(0, 2, 1).reshape(d, f2 * d))
    w.embed_b = D(sd["encoder.embed.out.0.bias"])
    w.pe = D(sinusoid_table(d, max_len))

    def ln(name):
        return D(sd[name + ".weight"]), D(sd[name + ".bias"])

    def ffn_w(p):
        return (D(sd[p + ".w_1.weight"]), D(sd[p + ".w_1.bias"]), D(sd[p + ".w_2.weight"]), D(sd[p + ".w_2.bias"]))

    for i in range(nblocks):
        p = f"encoder.encoders.{i}."
        L = ConformerLayerWeights()
        L.ln_ffm = ln(p + "norm_ff_macaron")
        L.ffm = ffn_w(p + "feed_forward_macaron")
        L.ln_mha = ln(p + "norm_mha")
        a = p + "self_attn."
        L.wqkv = D(torch.cat([sd[a + "linear_q.weight"], sd[a + "linear_k.weight"], sd[a + "linear_v.weight"]], 0))
        L.bqkv = D(torch.cat([sd[a + "linear_q.bias"], sd[a + "linear_k.bias"], sd[a + "linear_v.bias"]], 0))
        L.wpos = D(sd[a + "linear_pos.weight"])
        L.pos_u = D(sd[a + "pos_bias_u"])
        L.pos_v = D(sd[a + "pos_bias_v"])
        L.wo = D(sd[a + "linear_out.weight"])
        L.bo = D(sd[a + "linear_out.bias"])
        L.ln_conv = ln(p + "norm_conv")
        c = p + "conv_module."
        pw1 = sd[c + "pointwise_conv1.weight"].reshape(2 * d, d)
        pb1 = sd[c + "pointwise_conv1.bias"]
        L.pw1 = D(torch.stack([pw1[:d], pw1[d:]], dim=1).reshape(2 * d, d))
        L.pw1_b = D(torch.stack([pb1[:d], pb1[d:]], dim=1).reshape(2 * d))
        # what a zero (left-padding) input frame becomes after pointwise_conv1 + GLU (convolution.py:103,117-118)
        L.glu_pad = D(torch.nn.functional.glu(pb1.reshape(1, 2 * d, 1), dim=1).reshape(d))
        L.kernel = int(sd[c + "depthwise_conv.weight"].shape[2])
        L.grouped = int(sd[a + "pos_bias_u"].shape[1]) != d // h
        L.dw = D(sd[c + "depthwise_conv.weight"].reshape(d, L.kernel))
        L.dw_b = D(sd[c + "depthwise_conv.bias"])
        L.cn = ln(c + "norm")
        L.pw2 = D(sd[c + "pointwise_conv2.weight"].reshape(d, d))
        L.pw2_b = D(sd[c + "pointwise_conv2.bias"])
        L.ln_ff = ln(p + "norm_ff")
        L.ff = ffn_w(p + "feed_forward")
        L.ln_final = ln(p + "norm_final")
        w.layers.append(L)
    w.after_norm = ln("encoder.after_norm")
    w.ctc_w = D(sd["ctc.ctc_lo.weight"])
    w.ctc_b = D(sd["ctc.ctc_lo.bias"])
    return w
