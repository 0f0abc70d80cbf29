"""Oracle (test infrastructure): DeepSpeech2 with ``encoder_conf.use_gru: True``, restated as plain torch-CPU functions over a
``state_dict`` (B=1 semantics; whole utterance and chunked with carried state), beside the LSTM form in
``oracle/deepspeech2.py`` whose front-end (``subsample``) and configuration (``DS2Config``) it shares.

Follows masr/model_utils/deepspeech2/:
  * ``RNN`` with ``use_gru``              encoder.py:24-33 -> the ``GRU`` wrapper of gru.py:6-22 (keys one level deeper:
                                          ``encoder.rnns.{l}.rnn.rnn.*``)
  * ``GRU.forward``                       gru.py:18-22 (the incoming c is ignored; the returned c is h)
  * ``DeepSpeech2Model.get_encoder_out[_chunk]``  model.py:65-77
The GRU cell is written out explicitly (PyTorch gate order r, z, n) rather than calling ``nn.GRU``, so the restatement is
independent of cuDNN/oneDNN fused kernels; it is pinned against the reference in the golden tests.
"""
from __future__ import annotations

from typing import Optional, Tuple

import torch
import torch.nn.functional as F

from .deepspeech2 import DS2Config, subsample


def gru_direction(x, w_ih, w_hh, b_ih, b_hh, h0, reverse: bool):
    """x [T, in] -> (out [T, H], h_T); order (r, z, n), b_hn inside the product with r:
    n = tanh(W_in x + b_in + r * (W_hn h + b_hn)), h' = n + z * (h - n) (ATen's form of (1 - z) n + z h)."""
    T, H = x.shape[0], w_hh.shape[1]
    gx = F.linear(x, w_ih, b_ih)
    h = h0
    out = x.new_zeros(T, H)
    steps = range(T - 1, -1, -1) if reverse else range(T)
    for t in steps:
        gh = F.linear(h, w_hh, b_hh)
        r = torch.sigmoid(gx[t, :H] + gh[:H])
        z = torch.sigmoid(gx[t, H:2 * H] + gh[H:2 * H])
        n = torch.tanh(gx[t, 2 * H:] + r * gh[2 * H:])
        h = n + z * (h - n)
        out[t] = h
    return out, h


def encode(sd, cfg: DS2Config, feats: torch.Tensor, state: Optional[Tuple[torch.Tensor, torch.Tensor]] = None):
    """feats [1, F, 80] -> (enc [T, H or 2H], (h [L, dirs, H], c [L, dirs, H])) with c = h, as the reference returns it;
    only state[0] (h) is read."""
    x = subsample(sd, feats)[0]
    H = cfg.hidden
    dirs = 2 if cfg.bidirectional else 1
    hs = []
    for l in range(cfg.layers):
        p = f"encoder.rnns.{l}.rnn.rnn."
        outs, hl = [], []
        for dname, rev in (("", False), ("_reverse", True))[:dirs]:
            di = 1 if rev else 0
            h0 = x.new_zeros(H) if state is None else state[0][l, di]
            o, h = gru_direction(x, sd[p + "weight_ih_l0" + dname], sd[p + "weight_hh_l0" + dname],
                                 sd[p + "bias_ih_l0" + dname], sd[p + "bias_hh_l0" + dname], h0, rev)
            outs.append(o); hl.append(h)
        x = torch.cat(outs, dim=1)
        x = F.layer_norm(x, (x.shape[1],), sd[f"encoder.rnns.{l}.layer_norm.weight"], sd[f"encoder.rnns.{l}.layer_norm.bias"], 1e-5)
        hs.append(torch.stack(hl))
    h = torch.stack(hs)
    return x, (h, h)


def get_encoder_out(sd, cfg, feats, state=None):
    """-> (probs [T, V], new state)."""
    enc, st = encode(sd, cfg, feats, state)
    return torch.softmax(F.linear(enc, sd["decoder.ctc_lo.weight"], sd["decoder.ctc_lo.bias"]), dim=1), st
