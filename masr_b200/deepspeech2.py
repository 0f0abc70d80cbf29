"""DeepSpeech2 engine (configs/deepspeech2.yml; masr/model_utils/deepspeech2/{conv,encoder,model}.py):
CMVN -> Conv2d(1,32,3,2)+ReLU -> Conv2d(32,32,3,2)+ReLU -> 5 x [LSTM(H) or GRU(H) (use_gru), uni (streaming) / bi ->
LayerNorm] -> CTC, H = encoder_conf.rnn_size (1024; 2048 for large data).

Input projections and the CTC head are tensor-core GEMMs (FP16x2 split); the first projection (K = 608) runs on the fp32
FMA pipe.  The recurrence is one persistent launch per layer and direction: on the fp32 FMA pipe up to H = 1024, on the
tensor cores (FP16x2 split) at H = 2048; with MASR_LSTM_PERSISTENT=0, or at other widths, one launch per time step.
Whole-utterance batches and the chunked streaming path with carried state (inference_predictor.py:66-78: (h, c) for the
LSTM, h for the GRU) are both implemented.  The cell type comes from the weights, as in the reference."""
from __future__ import annotations

import os
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch

from . import _lib
from ._lib import EPI_BIAS, call
from .engine import ConformerEngine, _p, subsampled_len

TC_HIDDEN = 2048      # the width of the tensor-core persistent recurrence (masr_{lstm,gru}_seq_tc_f16x2)


@dataclass
class DS2Weights:
    d_model: int          # encoder output width (H * dirs)
    heads: int
    ffn: int
    kernel: int
    idim: int
    vocab: int
    max_len: int
    hidden: int = 1024
    dirs: int = 1
    cmvn_mean: torch.Tensor = None
    cmvn_istd: torch.Tensor = None
    conv1_w: torch.Tensor = None
    conv1_b: torch.Tensor = None
    conv2_w: torch.Tensor = None
    conv2_b: torch.Tensor = None
    layers: list = field(default_factory=list)      # unused (ConformerEngine plumbing)
    rnn: List[dict] = field(default_factory=list)   # per layer: {"wih": [dirs], "whh": [dirs], "bias": [dirs], "ln": (g, b)}
                                                    # (+ "bhn": [dirs] for the GRU)
    cell: str = "lstm"                              # "lstm" or "gru" (encoder_conf.use_gru)
    gates: int = 4                                  # gate rows per hidden unit: 4 (LSTM) / 3 (GRU)
    ctc_w: torch.Tensor = None
    ctc_b: torch.Tensor = None
    pe: torch.Tensor = None


def pack_deepspeech2(sd: Dict[str, torch.Tensor], device) -> DS2Weights:
    dev = torch.device(device)

    def D(t):
        return t.contiguous().to(dev)

    idim = sd["encoder.global_cmvn.mean"].shape[0]
    C = sd["encoder.conv.conv.0.weight"].shape[0]
    from .weights import check_supported
    check_supported(sd, "deepspeech2")
    gru = "encoder.rnns.0.rnn.rnn.weight_hh_l0" in sd       # the reference's GRU wrapper (gru.py:6-15)
    rp = "rnn.rnn." if gru else "rnn."
    G = 3 if gru else 4
    H = sd[f"encoder.rnns.0.{rp}weight_hh_l0"].shape[1]
    dirs = 2 if f"encoder.rnns.0.{rp}weight_hh_l0_reverse" in sd else 1
    nl = 1 + max(int(k.split(".")[2]) for k in sd if k.startswith("encoder.rnns."))
    vocab = sd["decoder.ctc_lo.weight"].shape[0]
    w = DS2Weights(d_model=H * dirs, heads=1, ffn=0, kernel=0, idim=idim, vocab=vocab, max_len=0, hidden=H, dirs=dirs,
                   cell="gru" if gru else "lstm", gates=G)
    w.cmvn_mean, w.cmvn_istd = D(sd["encoder.global_cmvn.mean"]), D(sd["encoder.global_cmvn.istd"])
    w.conv1_w, w.conv1_b = D(sd["encoder.conv.conv.0.weight"].reshape(C, 9)), D(sd["encoder.conv.conv.0.bias"])
    w.conv2_w = D(sd["encoder.conv.conv.2.weight"].permute(0, 2, 3, 1).reshape(C, 9 * C))
    w.conv2_b = D(sd["encoder.conv.conv.2.bias"])
    f2 = ((idim - 1) // 2 - 1) // 2
    for l in range(nl):
        p = f"encoder.rnns.{l}.{rp}"
        ent = {"wih": [], "whh": [], "bias": []}
        if gru:
            ent["bhn"] = []
        for suf in ("", "_reverse")[:dirs]:
            wih = sd[p + "weight_ih_l0" + suf]
            if l == 0:   # conv output is channels-last here: permute the (c*19+f) input columns to (f*32+c)
                wih = wih.reshape(G * H, C, f2).permute(0, 2, 1).reshape(G * H, f2 * C)
            ent["wih"].append(D(wih))
            ent["whh"].append(D(sd[p + "weight_hh_l0" + suf]))
            bih, bhh = sd[p + "bias_ih_l0" + suf], sd[p + "bias_hh_l0" + suf]
            if gru:      # b_hr, b_hz fold into the input projection; b_hn is multiplied by r inside the cell
                ent["bias"].append(D(bih + torch.cat([bhh[:2 * H], torch.zeros_like(bhh[2 * H:])])))
                ent["bhn"].append(D(bhh[2 * H:]))
            else:
                ent["bias"].append(D(bih + bhh))
        ent["ln"] = (D(sd[f"encoder.rnns.{l}.layer_norm.weight"]), D(sd[f"encoder.rnns.{l}.layer_norm.bias"]))
        w.rnn.append(ent)
    w.ctc_w, w.ctc_b = D(sd["decoder.ctc_lo.weight"]), D(sd["decoder.ctc_lo.bias"])
    return w


class DeepSpeech2Stream:
    """The recurrent state of the 5 layers carried between chunks (inference_predictor.py:45-46,97-99), for `n` streams side
    by side (one for ``predict_stream``, one per slot for ``DeepSpeech2StreamPool``): stream s is lane s % 32 of lane group
    s // 32 of every layer's h, in the kernels' transposed layout ``[ceil(n/32)][H][32]``, and for the LSTM row s of every
    layer's c ``[n][H]``.  A GRU carries h only (its c is h again, gru.py:21), so ``c`` is None for a GRU model.
    ``hT[l, cur[l]]`` holds layer l's state; the persistent recurrence updates it in place, the per-step form ping-pongs
    through ``hT[l, 1 - cur[l]]``."""

    def __init__(self, eng: "DeepSpeech2Engine", n: int = 1):
        self.eng = eng
        H, nl = eng.H, len(eng.w.rnn)
        self.hT = torch.zeros(nl, 2, (n + 31) // 32, H, 32, device=eng.device, dtype=torch.float32)
        self.c = torch.zeros(nl, n, H, device=eng.device, dtype=torch.float32) if eng.w.cell == "lstm" else None
        self.cur = [0] * nl

    def reset(self):
        self.hT.zero_()
        if self.c is not None:
            self.c.zero_()
        self.cur = [0] * len(self.cur)


class DeepSpeech2Engine(ConformerEngine):
    def __init__(self, weights_src, streaming: bool = True, device: str = "cuda", max_len: int = 5000, gemm: str = "tc",
                 use_graphs: bool = True):
        if gemm != "tc":
            raise ValueError("DeepSpeech2Engine implements the tensor-core projection path only")
        super().__init__(weights_src, streaming, device, max_len, gemm, use_graphs)
        self.H = self.w.hidden
        self.dirs = self.w.dirs
        # one persistent launch per layer and direction (masr_lstm_seq_f32 / masr_gru_seq_f32) instead of one launch per
        # time step; the switch covers both cells
        self.persistent_lstm = os.environ.get("MASR_LSTM_PERSISTENT", "1") != "0"
        if bool(streaming) != (self.dirs == 1):
            raise Exception("streaming DeepSpeech2 needs forward-only recurrent weights, non-streaming bidirectional ones")
        self.G = self.w.gates
        self._seq_fn, self._step_fn = (("masr_gru_seq_f32", "masr_gru_step_f32") if self.w.cell == "gru" else
                                       ("masr_lstm_seq_f32", "masr_lstm_step_f32"))
        self._seq_tc_fn = f"masr_{self.w.cell}_seq_tc_f16x2"
        if self.H == TC_HIDDEN:
            self._pack_rnn_tc()

    @property
    def rnn_form(self) -> str:
        """Which recurrence kernel runs: the fp32 persistent one ("seq", W_hh slices resident in shared memory) up to
        H = 1024, the tensor-core persistent one ("seq_tc", W_hh partly resident, partly streamed from L2 every step) at
        H = 2048, and one launch per time step ("step") at any other width or with ``persistent_lstm`` off."""
        H = self.H
        if not self.persistent_lstm:
            return "step"
        return "seq" if H % 128 == 0 and H <= 1024 else "seq_tc" if H == TC_HIDDEN else "step"

    def _pack_rnn_tc(self):
        """W_hh of every layer and direction in the fragment order of the tensor-core recurrence (masr_rnn_tc_pack_f16x2)."""
        for l, ent in enumerate(self.w.rnn):
            packed = []
            for whh in ent["whh"]:
                buf = torch.empty(whh.numel() * 4, device=self.device, dtype=torch.uint8)
                call("masr_rnn_tc_pack_f16x2", _p(whh), _p(buf), self.G, self.H, self._stream())
                packed.append(buf)
            self._tcw[l, "whh_tc"] = packed
        torch.cuda.synchronize(self.device)

    def _pack(self, sd, max_len):
        return pack_deepspeech2(sd, self.device)

    def _precompute_pos(self):
        pass

    def _split_weights(self):
        t = self._tcw
        t["ctc"] = self._split(self.w.ctc_w)
        for l, ent in enumerate(self.w.rnn):
            if l > 0:
                t[l, "wih"] = [self._split(x) for x in ent["wih"]]
        torch.cuda.synchronize(self.device)

    def _alloc_workspace(self, B: int, Fmax: int):
        dev, f32, f16 = self.device, torch.float32, torch.float16
        F1 = (Fmax - 1) // 2
        T = subsampled_len(Fmax)
        M = max(1, B * T)
        C = self.w.conv1_w.shape[0]
        D = self.H * self.dirs
        nb = (B + 31) // 32
        ws = {
            "c1": torch.empty(B * max(1, F1) * self.w1_cols * C, device=dev, dtype=f32),
            "c2": torch.empty(M, self.f2 * C, device=dev, dtype=f32),
            "gx": torch.empty(M, self.G * self.H, device=dev, dtype=f32),
            "out": torch.zeros(M, D, device=dev, dtype=f32),
            "t0": torch.empty(M, D, device=dev, dtype=f32),
            "xp": (torch.empty(M, D, device=dev, dtype=f16), torch.empty(M, D, device=dev, dtype=f16)),
            "hT": torch.zeros(2, nb, self.H, 32, device=dev, dtype=f32),
            "c": torch.zeros(B, self.H, device=dev, dtype=f32) if self.w.cell == "lstm" else None,
            "logits": torch.empty(M, self.Vpad, device=dev, dtype=f32),
            "ids": torch.empty(M, device=dev, dtype=torch.int32),
            "maxp": torch.empty(M, device=dev, dtype=f32),
        }
        self._alloc_out_pack(ws, B, T)
        ws["t0p"] = ws["xp"]
        return ws

    # ------------------------------------------------------------------------------------------------
    def _rnn_stack(self, ws, B, T, M, tlens, hT_init=None, c_init=None, stream: Optional[DeepSpeech2Stream] = None):
        """x = ws['c2'] [M, 608] -> ws['xp'] pair of the last LayerNorm output (and ws['t0'] fp32)."""
        w, H, dirs, D, GH = self.w, self.H, self.dirs, self.H * self.dirs, self.G * self.H
        out, gx, xp = ws["out"], ws["gx"], ws["xp"]
        for l, ent in enumerate(w.rnn):
            for di in range(dirs):
                if l == 0:
                    K0 = ws["c2"].shape[1]
                    self._gemm(ws["c2"], K0, ent["wih"][di], ent["bias"][di], gx, GH, M, GH, K0, EPI_BIAS, tag="lstm_xproj")
                else:
                    self._tc(xp, D, self._tcw[l, "wih"][di], ent["bias"][di], M, GH, D, EPI_BIAS, C=gx, ldc=GH, tag="lstm_xproj")
                if stream is None:
                    hT, c = ws["hT"], ws["c"]
                    hT.zero_()
                    if c is not None:
                        c.zero_()
                    cur = 0
                else:
                    hT, cur = stream.hT[l], stream.cur[l]
                    c = None if stream.c is None else stream.c[l]
                # the cell's per-unit operand: the LSTM's cell state c [B][H] (updated in place), the GRU's b_hn [H]
                aux = ent["bhn"][di] if w.cell == "gru" else c
                if self.rnn_form == "seq":
                    # the whole recurrence of this layer / direction in one persistent launch (W_hh slices resident in shared memory).
                    # The state is updated in place (h0_T == hN_T), so it never changes buffers: a captured pool step reads in the
                    # next replay what it wrote in this one.
                    if ws.get("lstm_ws") is None:
                        nbytes = _lib.C.c_int64(0)
                        call("masr_lstm_seq_workspace_bytes", B, H, _lib.C.byref(nbytes))
                        ws["lstm_ws"] = torch.empty(nbytes.value, device=self.device, dtype=torch.uint8)
                    self._k(f"{w.cell}_seq", self._seq_fn, _p(gx), GH, T, _p(ent["whh"][di]), _p(hT[cur]), _p(hT[cur]), _p(aux),
                            _p(out), None, None, D, di * H, _p(tlens), B, H, T, di, _p(ws["lstm_ws"]), ws["lstm_ws"].numel())
                elif self.rnn_form == "seq_tc":
                    # the same in-place persistent launch on the tensor cores (H = 2048)
                    if ws.get("rnn_tc_ws") is None:
                        nbytes = _lib.C.c_int64(0)
                        call("masr_rnn_seq_tc_workspace_bytes", B, H, _lib.C.byref(nbytes))
                        ws["rnn_tc_ws"] = torch.empty(nbytes.value, device=self.device, dtype=torch.uint8)
                    self._k(f"{w.cell}_seq", self._seq_tc_fn, _p(gx), GH, T, _p(self._tcw[l, "whh_tc"][di]), _p(hT[cur]),
                            _p(hT[cur]), _p(aux), _p(out), None, None, D, di * H, _p(tlens), B, H, T, di, _p(ws["rnn_tc_ws"]),
                            ws["rnn_tc_ws"].numel())
                else:
                    for s in range(T):
                        self._k(f"{w.cell}_step", self._step_fn, _p(gx), GH, T, _p(ent["whh"][di]), _p(hT[cur]), _p(hT[1 - cur]),
                                _p(aux), _p(out), None, None, D, di * H, _p(tlens), B, H, s, di)
                        cur = 1 - cur
                if stream is not None:
                    stream.cur[l] = cur
            self._k("layernorm", "masr_layernorm_split_f16", _p(out), D, _p(ent["ln"][0]), _p(ent["ln"][1]), _p(xp[0]), _p(xp[1]),
                    D, M, D, 1e-5)
        last = w.rnn[-1]["ln"]
        self._k("layernorm", "masr_layernorm_f32", _p(out), D, _p(last[0]), _p(last[1]), _p(ws["t0"]), D, M, D, 1e-5)

    def _front(self, feats, ws, B, Fmax, F1, T):
        w = self.w
        C = w.conv1_w.shape[0]
        self._k("conv1", "masr_conv1_cmvn_relu_f32", _p(feats), _p(w.cmvn_mean), _p(w.cmvn_istd), _p(w.conv1_w), _p(w.conv1_b),
                _p(ws["c1"]), B, Fmax, w.idim, F1, self.w1_cols, C)
        self._k("conv2", "masr_conv2_s2_relu_f32", _p(ws["c1"]), _p(w.conv2_w), _p(w.conv2_b), _p(ws["c2"]), B, F1, self.w1_cols,
                T, self.f2, C)

    def encode(self, feats: torch.Tensor, feat_lens: Sequence[int], tlens_dev: Optional[torch.Tensor] = None):
        B, Fmax = feats.shape[0], feats.shape[1]
        F1 = (Fmax - 1) // 2
        T = subsampled_len(Fmax)
        tl = [subsampled_len(int(f)) for f in feat_lens]
        ws = self._workspace(B, Fmax)
        if T == 0:
            return ws["t0"][:0], tl, 0, ws
        M = B * T
        if tlens_dev is not None:
            ws["tlens"], ws["tl_host"] = tlens_dev, None
        elif ws.get("tl_host") != tl:
            ws["tlens"] = torch.tensor(tl, dtype=torch.int32, device=self.device)
            ws["tl_host"] = list(tl)
        self._front(feats, ws, B, Fmax, F1, T)
        self._rnn_stack(ws, B, T, M, ws["tlens"])
        return ws["t0"][:M], tl, T, ws

    def _ctc_operand(self, ws):
        return ws["xp"], self.H * self.dirs

    # ---- streaming ----------------------------------------------------------------------------------
    def new_stream(self, n: int = 1) -> DeepSpeech2Stream:
        """The carried recurrent state of `n` streams (``DeepSpeech2StreamPool`` keeps one for all its slots)."""
        if self.dirs != 1:
            raise Exception("chunk decoding needs a streaming (forward-only) model")
        return DeepSpeech2Stream(self, n)

    def encode_chunk(self, feats_chunk: torch.Tensor, st: DeepSpeech2Stream, required_cache_size: int = -1,
                     want_probs: bool = False):
        """``DeepSpeech2Model.get_encoder_out_chunk`` for one stream (model.py:70-77): feats [n, 80] on device ->
        (ids, max-prob[, posteriors]) for ((n-1)//2-1)//2 frames; the recurrent state is carried in ``st``."""
        n = int(feats_chunk.shape[0])
        T = subsampled_len(n)
        if T == 0:
            return None
        ws = self._workspace(1, n)
        if ws.get("tl_host") != [T]:
            ws["tlens"] = torch.tensor([T], dtype=torch.int32, device=self.device)
            ws["tl_host"] = [T]
        self._front(feats_chunk.reshape(1, n, -1), ws, 1, n, (n - 1) // 2, T)
        self._rnn_stack(ws, 1, T, T, ws["tlens"], stream=st)
        probs = torch.empty(T, self.V, device=self.device, dtype=torch.float32) if want_probs else None
        logits = self._ctc_argmax(ws, T, probs)
        st.last_logits = logits[:T]                    # (the streaming beam search reads the chunk's logits)
        return ws["ids"][:T], ws["maxp"][:T], probs
