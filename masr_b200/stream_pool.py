"""Many live streams on one GPU: batched chunk decoding for the streaming Conformer, Squeezeformer, EfficientConformer and
DeepSpeech2 (``DeepSpeech2StreamPool``: every slot's LSTM state advanced in one pass per layer).

The reference's streaming API is one stream per ``MASRPredictor`` (predict.py:237-343; ``forward_chunk`` asserts
batch 1, conformer/encoder.py:378) and `infer_server.py` effectively serves one stream at a time.  BASELINE.json
config 3/5 ask for dozens to hundreds of concurrent streams.  ``ConformerStreamPool`` keeps N slots of streaming state
(attention K|V caches as fp16 pairs, conv left contexts, offsets) in one set of device buffers and advances every slot
that has a chunk ready in ONE pass of tensor-core GEMMs (M = slots x 16 rows) — each slot computed exactly like the
single-stream ``encode_chunk`` / reference ``forward_chunk`` with ``required_cache_size < 0`` (all history kept, which
is what ``predict_stream`` passes).  ``StreamPool`` adds the per-stream host logic of ``predict_stream`` (sample
carry-over with in-place dB renormalisation, 67/64/3 feature windowing, greedy history) and, with ``beam=...``, the
streaming CTC prefix beam search of every slot (``PoolBeam``: two more launches per chunk step, inside its CUDA graph).
"""
from __future__ import annotations

import gc
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch

from ._lib import EPI_BIAS, EPI_BIAS_GLU, EPI_RESIDUAL
from .audio import pcm_bytes_to_float32, samples_to_float32
from .beam import POOL, BeamSearch, check_n_best
from .hotwords import HotwordBuffer, graph_or_none
from .engine import ConformerEngine, _p, greedy_score, nbest_lists, subsampled_len
from .predict import CACHED_FEATURE_NUM, DECODING_WINDOW, FRAME_SHIFT, chunk_starts
from .resample import MODEL_RATE, output_length
from .text import ids_to_text, nbest_dicts
from . import timestamps as ts

CHUNK_FRAMES = DECODING_WINDOW          # 67 feature frames -> 16 encoder frames
CHUNK_OUT = 16


class _PoolBase:
    """Shared machinery of the batched chunk-decoding pools.

    Everything that varies from step to step is DEVICE DATA (one int32 table `meta`, refreshed by a single small H2D copy):
    per slot the valid query rows, key rows and cache fill at the full and at the halved frame rate.  The launch sequence
    of a step is therefore fixed, and after one eager step it is captured into a CUDA graph and replayed (a chunk step is
    ~150-250 small launches: launch-bound otherwise).  K|V rows are appended and conv left contexts slid by two
    bookkeeping kernels (csrc/stream.cu) instead of host-built index lists."""

    # rows of `meta`
    QLEN, KLEN, BASE, QLEN2, KLEN2, BASE2 = range(6)
    OUT_ROWS = CHUNK_OUT          # output frames per slot and chunk (8 for the EfficientConformer)

    def _init_common(self, eng, n_slots: int, use_graph: bool, keep_probs: bool = False):
        self.eng, self.S = eng, n_slots
        # keep_probs: also write the CTC posteriors of every output frame ([S * OUT_ROWS, V], `self.probs`) — the
        # `InferencePredictor.predict_chunk_conformer` seam (inference_predictor.py:80-94) returns them
        self.probs = (torch.zeros(n_slots * self.OUT_ROWS, eng.V, device=eng.device, dtype=torch.float32) if keep_probs else None)
        dev = eng.device
        self.meta = torch.zeros(6, n_slots, device=dev, dtype=torch.int32)
        self.meta_host = torch.zeros(6, n_slots, dtype=torch.int32, pin_memory=True)
        self.feats_in = torch.zeros(n_slots, CHUNK_FRAMES, 80, device=dev, dtype=torch.float32)
        self.lens_host = [0] * n_slots
        self.use_graph = bool(use_graph) and eng.use_graphs
        self.beam = None              # PoolBeam: the prefix beam search runs after every step (captured with it)
        self._graph = None
        self._graph_launches = 0
        self._warm = False
        self._meta_ev = None          # the previous step's H2D copy out of `meta_host` (pinned) has completed

    def _m(self, row):
        return self.meta[row].data_ptr()

    def frame_bounds(self):
        """(cap, max_len): a slot may hold at most `cap` encoder frames since its reset (its K|V cache rows), and fewer than
        `max_len` (the rows of the engine's relative-position table).  None: no such bound."""
        return self.cap, self.eng.w.max_len

    def _prepare(self, nframes: Sequence[int], short_ok_once: bool):
        eng, S, C = self.eng, self.S, CHUNK_OUT
        tout = [subsampled_len(int(n)) for n in nframes]
        tout2 = [(t + 1) // 2 for t in tout]
        cap, max_len = self.frame_bounds()
        for s in range(S):
            if short_ok_once and tout[s] and self.lens_host[s] % C:
                raise AssertionError(f"stream slot {s}: a short (final) chunk was already decoded; reset the stream first")
            n = self.lens_host[s] + tout[s]
            if (cap is not None and n > cap) or (max_len is not None and n >= max_len):
                raise AssertionError(f"stream slot {s}: {n} cached frames exceed the pool capacity")
        if self._meta_ev is not None:
            self._meta_ev.synchronize()
        mh = self.meta_host.numpy()
        mh[self.QLEN] = tout
        mh[self.BASE] = self.lens_host
        mh[self.KLEN] = mh[self.BASE] + mh[self.QLEN]
        mh[self.QLEN2] = tout2
        mh[self.BASE2] = mh[self.BASE] // 2
        mh[self.KLEN2] = mh[self.BASE2] + mh[self.QLEN2]
        self.meta.copy_(self.meta_host, non_blocking=True)
        self._meta_ev = torch.cuda.Event()
        self._meta_ev.record(torch.cuda.current_stream(eng.device))
        return tout, tout2

    def _run(self):
        """Eager on the first step (one-time setup: function attributes, tables), then capture once and replay."""
        eng = self.eng
        if not self.use_graph:
            self._step_body()
            return
        if not self._warm:
            self._step_body()
            self._warm = True
            return
        if self._graph is None:
            n0 = eng.launches
            g = torch.cuda.CUDAGraph()
            # no garbage collection inside the capture: a collected object that owns a CUDA graph (e.g. a dropped pool in a
            # reference cycle) would destroy it here, which is not permitted while a stream captures and invalidates this graph
            gc_on = gc.isenabled()
            gc.disable()
            try:
                with torch.cuda.graph(g, capture_error_mode="thread_local"):
                    self._step_body()
            finally:
                if gc_on:
                    gc.enable()
            self._graph_launches = eng.launches - n0
            eng.launches = n0
            self._graph = g
        self._graph.replay()
        eng.launches += self._graph_launches

    def _step_body(self):
        self._body()
        if self.beam is not None:
            self.beam.launch()

    def _append_pair(self, src, ld_src_elems, col0_elems, ncols, dst, cap, base_row, cnt_row, rows_per_slot, elem_bytes=2):
        """dst pair rows (s*cap + base[s] + t) <- src pair rows (s*rows_per_slot + t), columns [col0, col0+ncols)."""
        s1, d1 = (None, None) if not isinstance(src, tuple) else (src[1], dst[1])
        s0, d0 = (src, dst) if not isinstance(src, tuple) else (src[0], dst[0])
        self.eng._k("stream_append", "masr_stream_append_rows", _p(s0), _p(s1), ld_src_elems * elem_bytes, col0_elems * elem_bytes,
                    ncols * elem_bytes, _p(d0), _p(d1), d0.shape[-1] * elem_bytes, cap, self._m(base_row), self._m(cnt_row),
                    rows_per_slot, self.S)

    def _shift(self, x0, x1, rows_per_slot, lorder, row_bytes, cnt_row):
        self.eng._k("stream_shift", "masr_stream_shift_cache", _p(x0), _p(x1), rows_per_slot, lorder, row_bytes, self._m(cnt_row), self.S)

    def _rate(self, half: bool):
        """(chunk rows per slot, cache rows per slot, `meta` rows of the query count, key count and cache fill) of the blocks
        at the full or at the halved frame rate."""
        if half:
            return CHUNK_OUT // 2, self.cap2, self.QLEN2, self.KLEN2, self.BASE2
        return CHUNK_OUT, self.cap, self.QLEN, self.KLEN, self.BASE

    def _cached_attention(self, i: int, L, rate, out):
        """Append the chunk's K|V rows (pair b["qkvp"]) to every slot's layer-i cache, then rel-pos attention of the chunk's
        queries (b["qkv"]) over [cache ++ chunk] -> the fp16 pair `out`."""
        eng, d, b = self.eng, self.eng.d, self.b
        Ci, cap, rq, rk, rb = rate
        kvh, kvl = self.kv[i]
        self._append_pair(b["qkvp"], 3 * d, d, 2 * d, (kvh, kvl), cap, rb, rq, Ci)
        ph, pl, _ = eng._ptab_pair(L)
        eng._k("attention", "masr_relpos_attention_tc", _p(b["qkv"]), 3 * d, Ci, kvh.data_ptr(), kvl.data_ptr(), kvh.data_ptr() + 2 * d,
               kvl.data_ptr() + 2 * d, 2 * d, cap, _p(ph), _p(pl), d, _p(L.pos_u), _p(L.pos_v), None, _p(out[0]), _p(out[1]), d, Ci,
               self._m(rq), self._m(rk), self.S, eng.h, eng.dk, Ci)

    def _cached_conv(self, i: int, L, rate, cache, clen, out, A=None, stride: int = 1):
        """Conv module middle over every slot's [cache ++ chunk] rows `cache` ([S, kernel - 1 + chunk rows, d]: fp32, or an
        fp16 pair): pw1 + GLU from the pair `A` (default: `cache` itself), the depthwise stage (in_lens `clen`) -> the fp16
        pair `out`, then each slot's new left context = the last kernel - 1 valid rows."""
        eng, d = self.eng, self.eng.d
        Ci, rq = rate[0], rate[2]
        lorder = L.kernel - 1
        g = self.b["g"]
        x0, x1 = cache if isinstance(cache, tuple) else (cache, None)
        eng._tc(cache if A is None else A, d, eng._tcw[i, "pw1"], L.pw1_b, self.S * (lorder + Ci), 2 * d, d, EPI_BIAS_GLU, C=g,
                ldc=d, tag="pw1_glu")
        eng._dwconv(L, g, lorder + Ci, clen, self.S, Ci // stride, out, cached=True, stride=stride)
        self._shift(x0, x1, lorder + Ci, lorder, d * x0.element_size(), rq)

    def step(self, feats: torch.Tensor, nframes: Sequence[int]):
        """feats [S, 67, 80] raw log-mel (device), nframes[s] = valid feature frames of slot s this round (0 = idle).
        -> (ids [S, OUT_ROWS] int32, maxp [S, OUT_ROWS], valid output frames per slot)."""
        tout, tout2 = self._prepare(nframes, self.SHORT_ONCE)
        if feats.data_ptr() != self.feats_in.data_ptr():
            self.feats_in.copy_(feats)
        self._run()
        for s in range(self.S):
            self.lens_host[s] += tout[s]
        R = self.OUT_ROWS
        return self.b["ids"].view(self.S, R), self.b["maxp"].view(self.S, R), (tout if R == CHUNK_OUT else tout2)


class ConformerStreamPool(_PoolBase):
    """Device state + one batched chunk step for `n_slots` streams."""

    SHORT_ONCE = False            # every block runs at the full frame rate: short chunks may be followed by more chunks

    def __init__(self, eng: ConformerEngine, n_slots: int, max_frames: int = 3000, use_graph: bool = True, keep_probs: bool = False):
        if not eng.causal:
            raise Exception("chunk decoding needs a streaming (causal) model")
        if eng.gemm_path != "tc":
            raise Exception("the stream pool runs on the tensor-core path")
        self._init_common(eng, n_slots, use_graph, keep_probs)
        self.cap = max_frames
        dev, d, w = eng.device, eng.d, eng.w
        f16, f32 = torch.float16, torch.float32
        nl = len(w.layers)
        S, C = n_slots, CHUNK_OUT
        self.lorder = w.kernel - 1
        M = S * C
        self.kv = [(torch.zeros(S * self.cap, 2 * d, device=dev, dtype=f16), torch.zeros(S * self.cap, 2 * d, device=dev, dtype=f16))
                   for _ in range(nl)]
        self.xcat = torch.zeros(nl, S, self.lorder + C, d, device=dev, dtype=f32)
        self.b = {
            **eng._subsample_planes(S, CHUNK_FRAMES),
            "x": torch.empty(M, d, device=dev, dtype=f32), "t0": torch.empty(M, d, device=dev, dtype=f32),
            "t0p": (torch.empty(M, d, device=dev, dtype=f16), torch.empty(M, d, device=dev, dtype=f16)),
            "t1p": (torch.empty(M, d, device=dev, dtype=f16), torch.empty(M, d, device=dev, dtype=f16)),
            "hidp": (torch.empty(M, w.ffn, device=dev, dtype=f16), torch.empty(M, w.ffn, device=dev, dtype=f16)),
            "qkv": torch.empty(M, 3 * d, device=dev, dtype=f32),
            "qkvp": (torch.empty(M, 3 * d, device=dev, dtype=f16), torch.empty(M, 3 * d, device=dev, dtype=f16)),
            "xcp": (torch.empty(S * (self.lorder + C), d, device=dev, dtype=f16), torch.empty(S * (self.lorder + C), d, device=dev, dtype=f16)),
            "g": torch.empty(S * (self.lorder + C), d, device=dev, dtype=f32),
            "logits": torch.empty(M, eng.Vpad, device=dev, dtype=f32),
            "ids": torch.empty(M, device=dev, dtype=torch.int32), "maxp": torch.empty(M, device=dev, dtype=f32),
            "clen": torch.full((S,), self.lorder + C, device=dev, dtype=torch.int32),
        }

    def reset(self, slot: int):
        """``InferencePredictor.reset_stream`` for one slot (inference_predictor.py:97-102)."""
        self.lens_host[slot] = 0
        self.xcat[:, slot].zero_()

    def _body(self):
        """One batched ``forward_chunk`` over all slots (fixed launch sequence; per-slot lengths come from `meta`)."""
        eng, S, C = self.eng, self.S, CHUNK_OUT
        w, d, tw, b = eng.w, eng.d, eng._tcw, self.b
        M = S * C
        rate = self._rate(False)
        x, t0, t0p, t1p, hidp, qkv, qkvp, xcp = b["x"], b["t0"], b["t0p"], b["t1p"], b["hidp"], b["qkv"], b["qkvp"], b["xcp"]
        eng._ln_tmp = t0                              # scratch of eng._ln_split at d = 512: t0 is live only from norm_conv to its copy into xcat
        eng._subsample(self.feats_in, b, S, CHUNK_FRAMES, C, x)
        for i, L in enumerate(w.layers):
            eng._ln_split(x, L.ln_ffm, t0p, M)
            eng._ffn_gemms(t0p, tw[i, "ffm1"], L.ffm[1], tw[i, "ffm2"], L.ffm[3], M, x, x, 0.5, hidp)
            eng._ln_split(x, L.ln_mha, t0p, M)
            eng._tc(t0p, d, tw[i, "qkv"], L.bqkv, M, 3 * d, d, C=qkv, Cp=qkvp, ldc=3 * d)
            self._cached_attention(i, L, rate, t1p)
            # conv module over [cache ++ chunk] per slot (convolution.py:101-109): t0 <- norm_conv(x + out_proj(att))
            eng._tc(t1p, d, tw[i, "wo"], L.bo, M, d, d, EPI_RESIDUAL, 1.0, x, d, C=x, ldc=d)
            eng._ln(x, L.ln_conv, t0, M)
            xc = self.xcat[i]                                   # [S, 14+16, d]
            xc[:, self.lorder:].copy_(t0.view(S, C, d))
            eng._k("affine_split", "masr_affine_split_f16", _p(xc), None, None, _p(xcp[0]), _p(xcp[1]), S * (self.lorder + C), d)
            self._cached_conv(i, L, rate, xc, b["clen"], t1p, A=xcp)
            eng._tc(t1p, d, tw[i, "pw2"], L.pw2_b, M, d, d, EPI_RESIDUAL, 1.0, x, d, C=x, ldc=d)
            eng._ln_split(x, L.ln_ff, t0p, M)
            eng._ffn_gemms(t0p, tw[i, "ff1"], L.ff[1], tw[i, "ff2"], L.ff[3], M, x, x, 0.5, hidp)
            eng._ln(x, L.ln_final, x, M)
        eng._ln_split(x, w.after_norm, t0p, M)
        eng._ctc_argmax(b, M, self.probs)


class SqueezeformerStreamPool(_PoolBase):
    """``ConformerStreamPool`` for the streaming Squeezeformer (``SqueezeformerEncoder.forward_chunk``,
    masr/model_utils/squeezeformer/encoder.py:240-361, with ``required_cache_size < 0`` as ``predict_stream`` passes).

    Blocks 5..10 run at half the frame rate: 16 chunk frames -> 8 (``TimeReductionLayerStream``: kernel 1, stride 2), and
    their K|V caches are kept at that rate (the reference stores them ``repeat_interleave``d to the full rate and reads them
    back with ``[::2]``, :339-356 — a round trip).  The conv-module left context (30 rows of the ada-scaled input,
    convolution.py:119-127) is kept as the fp16 (h,l) operand pair the pointwise GEMM consumes.  A chunk shorter than 67
    frames (the last one of a stream) is supported once per stream: afterwards the slot must be reset."""

    SHORT_ONCE = True

    def __init__(self, eng, n_slots: int, max_frames: int = 3000, use_graph: bool = True, keep_probs: bool = False):
        if not eng.causal:
            raise Exception("chunk decoding needs a streaming (causal) model")
        self._init_common(eng, n_slots, use_graph, keep_probs)
        self.cap = (max_frames + 15) // 16 * 16
        self.cap2 = self.cap // 2
        dev, d, w = eng.device, eng.d, eng.w
        f16, f32 = torch.float16, torch.float32
        nl = len(w.layers)
        S, C = n_slots, CHUNK_OUT
        C2 = C // 2
        self.lorder = w.kernel - 1
        M = S * C
        LC = self.lorder + C
        self.reduced = [eng.REDUCE <= i < eng.RECOVER for i in range(nl)]
        self.kv = [(torch.zeros(S * (self.cap2 if r else self.cap), 2 * d, device=dev, dtype=f16),
                    torch.zeros(S * (self.cap2 if r else self.cap), 2 * d, device=dev, dtype=f16)) for r in self.reduced]
        # [cache ++ chunk] input rows of every block's conv module, as fp16 pairs
        self.xcat = [(torch.zeros(S, self.lorder + (C2 if r else C), d, device=dev, dtype=f16),
                      torch.zeros(S, self.lorder + (C2 if r else C), d, device=dev, dtype=f16)) for r in self.reduced]
        self.b = {
            **eng._subsample_planes(S, CHUNK_FRAMES),
            "x": torch.zeros(M, d, device=dev, dtype=f32), "y": torch.zeros(M, d, device=dev, dtype=f32),
            "saved": torch.zeros(M, d, device=dev, dtype=f32),
            "t0p": (torch.zeros(M, d, device=dev, dtype=f16), torch.zeros(M, d, device=dev, dtype=f16)),
            "t1p": (torch.zeros(M, d, device=dev, dtype=f16), torch.zeros(M, d, device=dev, dtype=f16)),
            "hidp": (torch.empty(M, w.ffn, device=dev, dtype=f16), torch.empty(M, w.ffn, device=dev, dtype=f16)),
            "qkv": torch.zeros(M, 3 * d, device=dev, dtype=f32),
            "qkvp": (torch.zeros(M, 3 * d, device=dev, dtype=f16), torch.zeros(M, 3 * d, device=dev, dtype=f16)),
            "g": torch.empty(S * LC, d, device=dev, dtype=f32),
            "logits": torch.empty(M, eng.Vpad, device=dev, dtype=f32),
            "ids": torch.empty(M, device=dev, dtype=torch.int32), "maxp": torch.empty(M, device=dev, dtype=f32),
            "clen": torch.full((S,), self.lorder + C, device=dev, dtype=torch.int32),
            "clen2": torch.full((S,), self.lorder + C2, device=dev, dtype=torch.int32),
        }

    def reset(self, slot: int):
        """``InferencePredictor.reset_stream`` for one slot (inference_predictor.py:97-102)."""
        self.lens_host[slot] = 0
        for xh, xl in self.xcat:
            xh[slot].zero_()
            xl[slot].zero_()

    def _body(self):
        eng, S, C = self.eng, self.S, CHUNK_OUT
        C2 = C // 2
        w, d, tw, b = eng.w, eng.d, eng._tcw, self.b
        M, M2 = S * C, S * C2
        x, y, saved, t0p, t1p, hidp, qkv, qkvp = b["x"], b["y"], b["saved"], b["t0p"], b["t1p"], b["hidp"], b["qkv"], b["qkvp"]
        eng._subsample(self.feats_in, b, S, CHUNK_FRAMES, C, y)
        eng._ln_ada(y, w.preln, x, w.layers[0].att_ada, t0p, M)
        nl = len(w.layers)
        full = (M, b["clen"], self._rate(False))
        half = (M2, b["clen2"], self._rate(True))
        Mi, clen, rate = full
        for i, L in enumerate(w.layers):
            if i == eng.REDUCE:
                saved.copy_(x)
                eng._k("time_reduce", "masr_time_reduce_dw_split_f16", _p(x), C, _p(w.tr_dw), _p(w.tr_dw_b), _p(t1p[0]), _p(t1p[1]),
                       C2, self._m(self.QLEN), S, C2, int(w.tr_dw.shape[1]), 0, d)
                eng._tc(t1p, d, tw["tr_pw"], w.tr_pw_b, M2, d, d, EPI_BIAS, C=x, ldc=d)
                eng._k("affine_split", "masr_affine_split_f16", _p(x), _p(L.att_ada[0]), _p(L.att_ada[1]), _p(t0p[0]), _p(t0p[1]), M2, d)
                Mi, clen, rate = half
            if i == eng.RECOVER:
                eng._k("affine_split", "masr_affine_split_f16", _p(x), None, None, _p(t1p[0]), _p(t1p[1]), M2, d)
                eng._tc(t1p, d, tw["rec"], w.rec_b, M2, d, d, EPI_BIAS, C=y, ldc=d)
                eng._k("upsample_add", "masr_upsample2_add_f32", _p(saved), _p(y), _p(x), C, C2, S, C, d)
                Mi, clen, rate = full
                eng._k("affine_split", "masr_affine_split_f16", _p(x), _p(L.att_ada[0]), _p(L.att_ada[1]), _p(t0p[0]), _p(t0p[1]), Mi, d)
            Ci = rate[0]
            # MHA over [cache ++ chunk] keys
            eng._tc(t0p, d, tw[i, "qkv"], L.bqkv, Mi, 3 * d, d, C=qkv, Cp=qkvp, ldc=3 * d)
            self._cached_attention(i, L, rate, t1p)
            eng._tc(t1p, d, tw[i, "wo"], L.bo, Mi, d, d, EPI_RESIDUAL, 1.0, x, d, C=y, ldc=d)
            eng._ln_ada(y, L.ln1, x, L.ffn1_ada, t0p, Mi)
            eng._ffn_gemms(t0p, tw[i, "f1a"], L.ffn1[1], tw[i, "f1b"], L.ffn1[3], Mi, x, y, 1.0, hidp)
            eng._ln_ada(y, L.ln2, x, L.conv_ada, t0p, Mi)
            # conv module over [cache ++ chunk] per slot
            xh, xl = self.xcat[i]
            xh[:, self.lorder:].copy_(t0p[0][:Mi].view(S, Ci, d))
            xl[:, self.lorder:].copy_(t0p[1][:Mi].view(S, Ci, d))
            self._cached_conv(i, L, rate, (xh, xl), clen, t1p)
            eng._tc(t1p, d, tw[i, "pw2"], L.pw2_b, Mi, d, d, EPI_RESIDUAL, 1.0, x, d, C=y, ldc=d)
            eng._ln_ada(y, L.ln3, x, L.ffn2_ada, t0p, Mi)
            nxt = w.layers[i + 1].att_ada if (i + 1 < nl and i + 1 not in (eng.REDUCE, eng.RECOVER)) else None
            eng._ffn_gemms(t0p, tw[i, "f2a"], L.ffn2[1], tw[i, "f2b"], L.ffn2[3], Mi, x, y, 1.0, hidp)
            eng._ln_ada(y, L.ln4, x, nxt, t0p, Mi)           # (last block: pair(x) feeds the CTC head)
        eng._ctc_argmax(b, M, self.probs)


class EfficientConformerStreamPool(_PoolBase):
    """Batched chunk decoding for the streaming EfficientConformer (``EfficientConformerEncoder.forward_chunk``,
    masr/model_utils/efficient_conformer/encoder.py:267-392, ``required_cache_size < 0``).

    Blocks 0-3 run at 40 ms frames with grouped attention over a float32 K|V cache (keys regrouped from key 0, queries from
    the first chunk frame, attention.py:44-60); block 3's conv module strides by 2 (16 -> 8 frames, AvgPool residual);
    blocks 4-11 run at 80 ms frames (depthwise kernel 7) over fp16-pair K|V caches kept at that rate — the reference stores
    them ``repeat_interleave``d and reads them back with ``[::2]`` (:344,372), a round trip.  The caller's offset counts
    output frames and is doubled inside (:306).  One chunk yields 8 output frames.  A short final chunk is supported once
    per stream (reset afterwards)."""

    SHORT_ONCE = True
    OUT_ROWS = CHUNK_OUT // 2

    def __init__(self, eng, n_slots: int, max_frames: int = 3000, use_graph: bool = True, keep_probs: bool = False):
        if not eng.causal:
            raise Exception("chunk decoding needs a streaming (causal) model")
        self._init_common(eng, n_slots, use_graph, keep_probs)
        self.cap = (max_frames + 15) // 16 * 16
        self.cap2 = self.cap // 2
        dev, d, w = eng.device, eng.d, eng.w
        f16, f32 = torch.float16, torch.float32
        S, C = n_slots, CHUNK_OUT
        C2 = C // 2
        self.SL = eng.STRIDE_LAYER
        M = S * C
        self.kv32 = {i: torch.zeros(S * self.cap, 2 * d, device=dev, dtype=f32) for i, L in enumerate(w.layers) if L.grouped}
        self.kv = {i: (torch.zeros(S * (self.cap if i <= self.SL else self.cap2), 2 * d, device=dev, dtype=f16),
                       torch.zeros(S * (self.cap if i <= self.SL else self.cap2), 2 * d, device=dev, dtype=f16))
                   for i, L in enumerate(w.layers) if not L.grouped}
        self.xcat = [(torch.zeros(S, (L.kernel - 1) + (C if i <= self.SL else C2), d, device=dev, dtype=f16),
                      torch.zeros(S, (L.kernel - 1) + (C if i <= self.SL else C2), d, device=dev, dtype=f16))
                     for i, L in enumerate(w.layers)]
        LCmax = max(x[0].shape[1] for x in self.xcat)
        self.b = {
            **eng._subsample_planes(S, CHUNK_FRAMES),
            "x": torch.zeros(M, d, device=dev, dtype=f32), "t0": torch.zeros(M, d, device=dev, dtype=f32),
            "t0p": (torch.zeros(M, d, device=dev, dtype=f16), torch.zeros(M, d, device=dev, dtype=f16)),
            "t1p": (torch.zeros(M, d, device=dev, dtype=f16), torch.zeros(M, d, device=dev, dtype=f16)),
            "hidp": (torch.empty(M, w.ffn, device=dev, dtype=f16), torch.empty(M, w.ffn, device=dev, dtype=f16)),
            "qb": torch.zeros(M, d, device=dev, dtype=f32), "kvn": torch.zeros(M, 2 * d, device=dev, dtype=f32),
            "qkv": torch.zeros(M, 3 * d, device=dev, dtype=f32),
            "qkvp": (torch.zeros(M, 3 * d, device=dev, dtype=f16), torch.zeros(M, 3 * d, device=dev, dtype=f16)),
            "g": torch.empty(S * LCmax, d, device=dev, dtype=f32),
            "logits": torch.empty(S * C2, eng.Vpad, device=dev, dtype=f32),
            "ids": torch.empty(S * C2, device=dev, dtype=torch.int32), "maxp": torch.empty(S * C2, device=dev, dtype=f32),
            "clen": torch.full((S,), LCmax, device=dev, dtype=torch.int32),
        }

    def reset(self, slot: int):
        self.lens_host[slot] = 0
        for xh, xl in self.xcat:
            xh[slot].zero_()
            xl[slot].zero_()

    def _body(self):
        eng, S, C = self.eng, self.S, CHUNK_OUT
        C2 = C // 2
        w, d, tw, b = eng.w, eng.d, eng._tcw, self.b
        M, M2 = S * C, S * C2
        x, t0, t0p, t1p, hidp, qkv, qkvp, qb, kvn = (b["x"], b["t0"], b["t0p"], b["t1p"], b["hidp"], b["qkv"], b["qkvp"], b["qb"],
                                                      b["kvn"])
        eng._subsample(self.feats_in, b, S, CHUNK_FRAMES, C, x)
        for i, L in enumerate(w.layers):
            half = i > self.SL
            rate = self._rate(half)
            Ci, cap, rq, rk, rb = rate
            Mi = S * Ci
            lorder = L.kernel - 1
            eng._ln_split(x, L.ln_ffm, t0p, Mi)
            eng._ffn_gemms(t0p, tw[i, "ffm1"], L.ffm[1], tw[i, "ffm2"], L.ffm[3], Mi, x, x, 0.5, hidp)
            eng._ln_split(x, L.ln_mha, t0p, Mi)
            if L.grouped:
                wh, wl = tw[i, "qkv"]
                eng._tc(t0p, d, (wh[:d], wl[:d]), L.bqkv[:d], Mi, d, d, C=qb, ldc=d)
                eng._tc(t0p, d, (wh[d:], wl[d:]), L.bqkv[d:], Mi, 2 * d, d, C=kvn, ldc=2 * d)
                kc = self.kv32[i]
                self._append_pair(kvn, 2 * d, 0, 2 * d, kc, cap, rb, rq, Ci, elem_bytes=4)
                eng._k("attention", "masr_grouped_attention_cache_f32", _p(qb), d, Ci, kc.data_ptr(), kc.data_ptr() + 4 * d, 2 * d, cap,
                       _p(L.ptab), _p(L.pos_u), _p(L.pos_v), None, _p(t1p[0]), _p(t1p[1]), self._m(rq), self._m(rk), S, eng.h, eng.dk,
                       eng.GROUP, Ci)
            else:
                eng._tc(t0p, d, tw[i, "qkv"], L.bqkv, Mi, 3 * d, d, C=qkv, Cp=qkvp, ldc=3 * d)
                self._cached_attention(i, L, rate, t1p)
            eng._tc(t1p, d, tw[i, "wo"], L.bo, Mi, d, d, EPI_RESIDUAL, 1.0, x, d, C=x, ldc=d)
            # conv module over [cache ++ chunk] per slot (convolution.py:93-111)
            eng._ln_split(x, L.ln_conv, t0p, Mi)
            xh, xl = self.xcat[i]
            xh[:, lorder:].copy_(t0p[0][:Mi].view(S, Ci, d))
            xl[:, lorder:].copy_(t0p[1][:Mi].view(S, Ci, d))
            if i == self.SL:
                self._cached_conv(i, L, rate, (xh, xl), b["clen"], t1p, stride=2)
                eng._k("avgpool", "masr_avgpool2_time_f32", _p(x), C, _p(t0), C2, self._m(self.QLEN), S, C2, d)
                Mo, res = M2, t0
            else:
                self._cached_conv(i, L, rate, (xh, xl), b["clen"], t1p)
                Mo, res = Mi, x
            eng._tc(t1p, d, tw[i, "pw2"], L.pw2_b, Mo, d, d, EPI_RESIDUAL, 1.0, res, d, C=x, ldc=d)
            eng._ln_split(x, L.ln_ff, t0p, Mo)
            eng._ffn_gemms(t0p, tw[i, "ff1"], L.ff[1], tw[i, "ff2"], L.ff[3], Mo, x, x, 0.5, hidp)
            eng._ln(x, L.ln_final, x, Mo)
        eng._ln_split(x, w.after_norm, t0p, M2)
        eng._ctc_argmax(b, M2, self.probs)


class DeepSpeech2StreamPool(_PoolBase):
    """Batched chunk decoding for the streaming (forward-only) DeepSpeech2 (``DeepSpeech2Model.get_encoder_out_chunk``,
    masr/model_utils/deepspeech2/model.py:70-77, with the (h, c) state carried as inference_predictor.py:66-78 does).

    One step is the launch sequence of ``DeepSpeech2Engine.encode_chunk`` over every slot at once (M = slots x 16 rows):
    CMVN + conv1, conv2, per layer the input projection, the recurrence (16 steps over the `meta` lengths row: a lane past
    its slot's valid frames is frozen, so an idle slot keeps its state byte for byte) and the LayerNorm, then the CTC head
    and argmax.  No stage's result for a row or lane depends on the batch, so every slot equals ``encode_chunk`` on a
    ``DeepSpeech2Stream`` bit for bit.  The state of all slots is one ``DeepSpeech2Stream`` in pool-owned buffers that stay
    put across rounds, as a CUDA graph replay needs: the persistent recurrence updates it in place, and the per-step form
    (``MASR_LSTM_PERSISTENT=0``) ping-pongs 16 times per round, so it ends where it started.

    The persistent recurrences need all their CTAs co-resident (a grid barrier per step): H / 8 for the fp32 form at
    H <= 1024, H / 16 = 128 with 216 KiB of shared memory each for the tensor-core form at H = 2048 (the host checks the
    occupancy and refuses to launch a grid that cannot be resident).  The pool launches on the engine's stream like every
    other engine call; do not run its steps on a second stream beside another persistent launch.

    There is no position table and the state has a constant size, so a greedy slot decodes any length; with a beam search
    attached, `max_frames` sizes each slot's prefix trie and bounds the slot.  A short chunk may be followed by more."""

    SHORT_ONCE = False

    def __init__(self, eng, n_slots: int, max_frames: int = 3000, use_graph: bool = True, keep_probs: bool = False):
        self.state = eng.new_stream(n_slots)
        self._init_common(eng, n_slots, use_graph, keep_probs)
        self.cap = max_frames
        # pool-owned (not the engine's per-shape cache, which frees buffers a captured step still uses)
        self.b = eng._alloc_workspace(n_slots, CHUNK_FRAMES)

    def frame_bounds(self):
        return (self.cap if self.beam is not None else None), None

    def reset(self, slot: int):
        """``InferencePredictor.reset_stream`` for one slot: zero state (inference_predictor.py:97-99)."""
        self.lens_host[slot] = 0
        self.state.hT[:, :, slot // 32, :, slot % 32].zero_()
        if self.state.c is not None:                       # (a GRU carries h only)
            self.state.c[:, slot].zero_()

    def _body(self):
        eng, S, C, ws = self.eng, self.S, CHUNK_OUT, self.b
        eng._front(self.feats_in, ws, S, CHUNK_FRAMES, (CHUNK_FRAMES - 1) // 2, C)
        eng._rnn_stack(ws, S, C, S * C, self.meta[self.QLEN], stream=self.state)
        eng._ctc_argmax(ws, S * C, self.probs)


class PoolStream:
    """One stream = a one-slot pool behind the single-stream interface ``MASRPredictor.predict_stream`` uses
    (``eng.new_stream()`` / ``eng.encode_chunk(chunk, stream)``)."""

    def __init__(self, pool):
        self.pool = pool
        self.batch = torch.zeros(1, CHUNK_FRAMES, 80, device=pool.eng.device, dtype=torch.float32)

    def reset(self):
        self.pool.reset(0)

    def encode_chunk(self, feats_chunk: torch.Tensor, required_cache_size: int = -1):
        if required_cache_size >= 0:
            raise NotImplementedError("bounded attention caches (required_cache_size >= 0) are not implemented for this model; "
                                      "predict_stream always asks for the whole history")
        n = int(feats_chunk.shape[0])
        if n > CHUNK_FRAMES:
            raise ValueError(f"a chunk has at most {CHUNK_FRAMES} feature frames")
        if subsampled_len(n) == 0:
            return None
        self.batch[0, :n].copy_(feats_chunk)
        ids, maxp, tout = self.pool.step(self.batch, [n])
        probs = None if self.pool.probs is None else self.pool.probs[:tout[0]]
        self.last_logits = self.pool.b["logits"][:tout[0]]      # (the streaming beam search reads the chunk's logits)
        return ids[0, :tout[0]], maxp[0, :tout[0]], probs


def make_pool(eng, n_slots: int, max_frames: int = 3000):
    """The batched chunk-decoding pool that matches the engine's model family."""
    from .deepspeech2 import DeepSpeech2Engine
    from .engine import EfficientConformerEngine
    from .squeezeformer import SqueezeformerEngine
    if isinstance(eng, DeepSpeech2Engine):
        return DeepSpeech2StreamPool(eng, n_slots, max_frames)
    if isinstance(eng, SqueezeformerEngine):
        return SqueezeformerStreamPool(eng, n_slots, max_frames)
    if isinstance(eng, EfficientConformerEngine):
        return EfficientConformerStreamPool(eng, n_slots, max_frames)
    if type(eng) is ConformerEngine:
        return ConformerStreamPool(eng, n_slots, max_frames)
    raise NotImplementedError(f"no stream pool for {type(eng).__name__}")


class PoolBeam(BeamSearch):
    """Streaming CTC prefix beam search of EVERY slot of a chunk-decoding pool (``engine.StreamBeam`` for many streams; the
    reference's ``BeamSearchDecoder.decode_chunk / reset_decoder`` per stream, beam_search_decoder.py:75-96).

    Each pool step adds two launches, captured into the step's CUDA graph with the encoder: the top-k candidates of all
    ``S * OUT_ROWS`` CTC-head rows (``pool.b["logits"]``), then the pool form of the prefix beam search with one CTA per slot
    over that slot's valid rows (the length row of the pool's device ``meta``).  Slots without frames in a step are not
    touched.  Per slot the beam, its trie and the trie's hash stay on the device, so after every step a slot's best
    prefix equals the whole-utterance search over its frames since the last ``reset`` — what ``predict_stream`` returns.
    The trie is sized by ``beam_size`` and the pool's frame capacity (at most ``beam_size`` new prefixes per frame), so
    no stream the pool accepts can overflow it.  ``lm`` / ``alpha`` / ``beta``: character- or word-LM shallow fusion as in
    ``StreamBeam``; the reported score is then approx_ctc.

    Hotwords (``hotwords``: the pool default, a ``HotwordGraph`` or None; ``max_hotword_nodes``: the room per slot): one
    device buffer (``hotwords.HotwordBuffer``) with a region of ``max(max_hotword_nodes, default nodes)`` nodes per slot and
    one for the default, allocated here, so a slot's graph never moves while the slot is live and the captured step graph
    stays valid.  ``set_hotwords`` points a slot at the default, at no hotwords or at its own list.  With neither a
    default nor room per slot the pool searches without the hotword instantiations, exactly as before."""

    def __init__(self, pool, beam_size: int = 300, cutoff_prob: float = 0.99, cutoff_top_n: int = 40, lm=None,
                 alpha: float = 0.0, beta: float = 0.0, hotwords=None, max_hotword_nodes: int = 0):
        beam_size = int(beam_size)
        if not 1 <= beam_size <= 512:
            raise ValueError(f"beam_size={beam_size} out of range (1..512)")
        S, R = pool.S, pool.OUT_ROWS
        # beam frames one slot can reach: the pool's cap at its output rate (+1: the EfficientConformer halves an odd final chunk up)
        frames = pool.cap * R // CHUNK_OUT + 1
        buf, roots, self.default_hotwords = None, None, hotwords
        if hotwords is not None or max_hotword_nodes > 0:
            buf = HotwordBuffer(pool.eng.device, S + 1, max(int(max_hotword_nodes), 0 if hotwords is None else hotwords.nodes))
            if hotwords is not None:
                buf.put(S, hotwords)
            roots = torch.full((S,), -1 if hotwords is None else buf.root(S), device=pool.eng.device, dtype=torch.int32)
        super().__init__(pool.eng.device, POOL, S, S * R, frames, beam_size, cutoff_prob, cutoff_top_n, lm, alpha, beta,
                         buf, roots)
        # what the launches read from the pool (the pool holds this object: no reference back to it, so dropping a pool frees
        # its CUDA graph at once instead of in a later garbage collection, which may fall inside another pool's capture)
        self.eng, self.R, self.logits = pool.eng, R, pool.b["logits"]
        self._own_lm = lm                                        # (the search itself holds the LM only weakly)
        self.lens = pool._m(pool.QLEN if R == CHUNK_OUT else pool.QLEN2)          # valid rows per slot (device meta row)

    def reset(self, slot: int):
        """``reset_decoder`` for one slot: start it at the root on its next frames (the kernel clears the flag) with an empty
        prefix hash."""
        cap = self.trie_cap
        self.fresh[slot] = 1
        self.trie_par[slot * cap + cap // 5:(slot + 1) * cap].fill_(-1)

    def set_hotwords(self, slot: int, graph, default: bool = False):
        """Slot ``slot`` searches with ``graph`` (copied into its own region), with the pool default (``default``), or
        without hotwords (graph None, not default).  Outside graph capture, while the slot has no frames since its reset."""
        if self.hot is None:
            raise ValueError("this pool was built without hotwords: create it with hotwords or max_hotword_nodes > 0")
        if default:
            root = -1 if self.default_hotwords is None else self.hot.root(self.slots)
        elif graph is None:
            root = -1
        else:
            self.hot.put(slot, graph)
            root = self.hot.root(slot)
        self.slot_root[slot] = root

    def launch(self):
        """The two launches of one pool step (device inputs only: safe to capture and replay)."""
        self.topk(self.eng, self.logits, self.eng.Vpad, self.slots * self.R)
        self.search(self.eng, self.lens, self.slots, self.R)

    def results(self, slots: Sequence[int], frames: Sequence[int], onsets: bool = False,
                n_best: Optional[int] = None) -> Dict[int, tuple]:
        """slot -> (token ids of its best prefix, score) after the last step: one D2H copy of every slot's count and score,
        then one of the token rows spanning `slots`.  ``frames[slot]``: the slot's encoder frames since its reset; a slot
        without any gets ([], 0.0), as ``predict_stream`` does.  ``onsets``: each with a third element, the tokens' onset
        frames since the slot's reset (one read-out launch here, outside the step graph, and one more copy).  ``n_best``
        (1..beam_size): each with a last element, the slot's ``n_best`` best (token ids, score), best first, entry 0 the
        first two (``engine.nbest_lists``: one read-out launch here, outside the step graph; none for n_best = 1)."""
        slots = list(slots)
        if not slots:
            return {}
        eng = self.eng
        oh = self.out.cpu()
        n = oh[1].view(torch.int32).numpy()
        score = oh[0].numpy()
        had = [s for s in slots if frames[s] > 0]
        nmax = max((int(n[s]) for s in had), default=0)
        lo, hi = (min(had), max(had) + 1) if had else (0, 0)
        toks = self.out_tok[lo:hi, :nmax].cpu().numpy() if nmax else None
        fr = self.frames(eng, hi)[lo:hi, :nmax].cpu().numpy() if onsets and nmax else None
        eng.d2h_bytes += oh.numel() * 4 + (0 if toks is None else toks.size * 4) + (0 if fr is None else fr.size * 4)
        out = {}
        for s in slots:
            if frames[s] == 0:
                out[s] = ([], 0.0)
            else:
                out[s] = (toks[s - lo, :n[s]].tolist() if n[s] else [], float(score[s]))
            if onsets:
                out[s] += (fr[s - lo, :len(out[s][0])].tolist() if out[s][0] else [],)
        if n_best is not None:
            nb = nbest_lists(self if had else None, eng, hi, n_best, [out.get(s, ([], 0.0))[0] for s in range(hi)],
                             [out.get(s, ([], 0.0))[1] for s in range(hi)])
            for s in slots:
                out[s] += (nb[s] if frames[s] > 0 else [([], 0.0)],)
        return out


class StreamPool:
    """`predict_stream` for many streams at once (same per-stream results as one ``MASRPredictor`` per stream).

    Host work per push is O(slots) integer bookkeeping: the un-consumed feature frames of every slot live in ONE device
    ring ``[S, RING, 80]`` (appended and windowed with two batched index ops per push / per round instead of per-slot
    tensor ops), and the greedy history is folded incrementally — the reference re-collapses the whole history on every
    chunk (ctc_greedy_decoder.py:81-88), which yields the same tokens and the same left-to-right float32 score sum."""

    RING = 1024                    # feature frames kept per slot (un-consumed frames never exceed one push + one window)

    def __init__(self, eng: ConformerEngine, vocab: Sequence[str], n_slots: int, use_db_normalization: bool = True,
                 target_db: float = -20.0, max_frames: int = 3000, beam: Optional[dict] = None, use_graph: bool = True,
                 resample: bool = False, timestamps: bool = False, hotword_score: float = 1.5, n_best: Optional[int] = None):
        """``beam``: None decodes greedily (``ctc_greedy``); a dict ``{beam_size, cutoff_prob, cutoff_top_n, lm, alpha,
        beta}`` (``MASRPredictor``'s ``ctc_beam_search`` settings; ``lm`` a ``CharLM``, ``WordLM`` or None) runs the streaming prefix
        beam search of every slot on the GPU (``PoolBeam``), and every result is the beam's, as ``predict_stream`` with
        ``decoder: ctc_beam_search`` returns it.  ``use_graph=False`` launches every step eagerly instead of replaying
        its CUDA graph (same results).  ``resample``: accept pushes at other sample rates (``push(..., sample_rate=)``) and
        resample them on the GPU as ``predict_stream`` does; False makes such a push a per-slot error.  ``timestamps``:
        every result also carries ``'tokens'`` (+ ``'words'``) timed since the slot's reset, as ``predict_stream(...,
        timestamps=True)`` returns them, plus ``t0[slot]`` seconds (0 after a reset; a caller that cuts a longer stream
        into utterances sets it to the utterance's start).

        Hotwords (beam search only): ``beam`` may also carry ``hotwords`` (the pool default, a ``HotwordGraph``) and
        ``max_hotword_nodes`` (automaton nodes each slot's own list may take; ``HotwordBuffer.bytes_per_node`` bytes of
        device memory per node, per slot).  ``set_hotwords`` gives a slot its own list, scored ``hotword_score`` per token.

        ``n_best`` (beam search only, 1..beam_size): every result also carries ``'n_best'``, the slot's ``n_best`` best
        hypotheses so far as ``[{'text', 'score'}, ...]``, best first, entry 0 the result's own text and score (one
        read-out launch per push, outside the step graph; scores as ``'score'``: approx_ctc with an LM, so they need not
        decrease down the list)."""
        if n_best is not None:
            if beam is None:
                raise ValueError("n_best needs the prefix beam search (decoder: ctc_beam_search)")
            check_n_best(n_best, beam.get("beam_size", 300))
        self.eng, self.vocab, self.S = eng, list(vocab), n_slots
        self.timestamps, self.dt, self.t0 = bool(timestamps), ts.frame_seconds(eng), [0.0] * n_slots
        self.resample = bool(resample)
        self.pool = make_pool(eng, n_slots, max_frames)
        if not use_graph:
            self.pool.use_graph = False
        self.beam = None
        if beam is not None:
            self.beam = PoolBeam(self.pool, **beam)
            self.pool.beam = self.beam
        self.hotword_score = hotword_score
        self.n_best = None if n_best is None else int(n_best)
        self.use_db, self.target_db = use_db_normalization, target_db
        self.remained: List[Optional[np.ndarray]] = [None] * n_slots
        dev = eng.device
        # row S*RING is an all-zero frame: the source of window rows beyond a slot's chunk
        self.ring = torch.zeros(n_slots * self.RING + 1, 80, device=dev, dtype=torch.float32)
        self.head = [0] * n_slots      # absolute index of the first un-consumed frame
        self.count = [0] * n_slots     # un-consumed frames in the ring
        self._reset_hist(range(n_slots))

    def _reset_hist(self, slots):
        if not hasattr(self, "toks"):
            self.toks = [[] for _ in range(self.S)]
            self.prev = np.full(self.S, -1, np.int64)          # last frame id per slot (-1: none yet)
            self.acc = np.zeros(self.S, np.float32)            # left-to-right float32 sum of the non-blank max-probabilities
            self.nprob = np.zeros(self.S, np.int64)
            self.seen = np.zeros(self.S, np.int64)             # encoder frames since the reset
            self.t_start = [[] for _ in range(self.S)]         # per token: its first frame, and the end of its run so far
            self.t_end = [[] for _ in range(self.S)]
        for s in slots:
            self.toks[s], self.t_start[s], self.t_end[s] = [], [], []
            self.prev[s], self.acc[s], self.nprob[s], self.seen[s] = -1, np.float32(0.0), 0, 0

    def _fold(self, ids_h: np.ndarray, mp_h: np.ndarray, tout: Sequence[int]):
        """Incremental ``greedy_decoder_chunk`` (ctc_greedy_decoder.py:70-89) for every slot at once: collapse repeats against
        the previous frame, drop blanks, and keep the score as the reference's left-to-right float32 sum — one vectorised
        float32 add per frame column (16 columns), so each slot's sum sees its terms in order with float32 rounding at
        every step, exactly like a scalar per-slot loop."""
        S, C = ids_h.shape
        tout = np.asarray(tout, np.int64)
        if not tout.any():
            return
        ids = ids_h.astype(np.int64)
        valid = np.arange(C)[None, :] < tout[:, None]
        prev_col = np.concatenate([self.prev[:, None], ids[:, :-1]], axis=1)
        nonblank = valid & (ids != 0)
        new_tok = nonblank & (ids != prev_col)
        acc = self.acc
        for t in range(C):
            col = nonblank[:, t]
            if col.any():
                acc = np.where(col, (acc + mp_h[:, t]).astype(np.float32), acc)
        self.acc = acc.astype(np.float32)
        self.nprob += nonblank.sum(1)
        for s in np.nonzero(new_tok.any(1))[0]:
            self.toks[s].extend(ids[s, new_tok[s]].tolist())
        if self.timestamps:                      # a non-blank frame starts a token or continues the last token's run
            for s in np.nonzero(nonblank.any(1))[0]:
                base = int(self.seen[s])
                for t in np.nonzero(nonblank[s])[0]:
                    if new_tok[s, t]:
                        self.t_start[s].append(base + int(t))
                        self.t_end[s].append(base + int(t) + 1)
                    else:
                        self.t_end[s][-1] = base + int(t) + 1
        self.seen += tout
        has = tout > 0
        last = np.take_along_axis(ids, np.maximum(tout - 1, 0)[:, None], axis=1)[:, 0]
        self.prev = np.where(has, last, self.prev)

    def reset_stream(self, slot: int):
        self.pool.reset(slot)
        if self.beam is not None:
            self.beam.reset(slot)
        self.remained[slot] = None
        self.head[slot], self.count[slot], self.t0[slot] = 0, 0, 0.0
        self._reset_hist([slot])

    def set_hotwords(self, slot: int, hotwords):
        """The hotwords slot ``slot`` boosts from its next frames on: a list of strings (its own list, which must fit the
        pool's ``max_hotword_nodes``), ``[]`` (none) or None (back to the pool default).  Legal only while the slot has had no
        frames since its reset (a ValueError otherwise); the list stays with the slot across later resets until it is set
        again.  Raises ValueError for a pool that decodes greedily or was built without hotwords."""
        if self.beam is None:
            raise ValueError("hotwords need the prefix beam search (decoder: ctc_beam_search)")
        if not 0 <= slot < self.S:
            raise ValueError(f"slot {slot} out of range (0..{self.S - 1})")
        if self.pool.lens_host[slot] != 0:
            raise ValueError(f"slot {slot} has decoded frames since its reset: set its hotwords right after a reset")
        if hotwords is None:
            self.beam.set_hotwords(slot, None, default=True)
        else:
            self.beam.set_hotwords(slot, graph_or_none(hotwords, self.vocab, self.hotword_score))

    def _dev_index(self, idx: np.ndarray) -> torch.Tensor:
        return torch.from_numpy(idx).to(self.eng.device, non_blocking=False)

    def _grow_ring(self, need: int):
        """Re-allocate the feature ring with room for `need` un-consumed frames per slot (a single message longer than the
        ring — about 10 s — is legal: the reference's `predict_stream` accepts any message length)."""
        R0, S = self.RING, self.S
        R1 = R0
        while R1 < need:
            R1 *= 2
        ring = torch.zeros(S * R1 + 1, 80, device=self.eng.device, dtype=torch.float32)
        src, dst = [], []
        for s in range(S):
            if self.count[s]:
                f = np.arange(self.count[s], dtype=np.int64)
                src.append(s * R0 + (self.head[s] + f) % R0)
                dst.append(s * R1 + f)
            self.head[s] = 0
        if src:
            ring.index_copy_(0, self._dev_index(np.concatenate(dst)), self.ring.index_select(0, self._dev_index(np.concatenate(src))))
        self.ring, self.RING = ring, R1

    def push(self, audio: Dict[int, object], is_end: bool = False, channels: int = 1, samp_width: int = 2,
             on_error: str = "raise", sample_rate=MODEL_RATE):
        """audio: slot -> np.ndarray | PCM bytes (one push per slot).  -> slot -> {'text','score'} | None, exactly what
        ``MASRPredictor.predict_stream(chunk, is_end, sample_rate=...)`` would return for that stream.  ``sample_rate``: one
        rate for every slot, or a ``{slot: rate}`` dict (missing slots: 16 kHz); off 16 kHz needs ``resample=True``.

        Per-slot isolation: every slot is validated (decodable input, gain within 300 dB, pool / position-table capacity,
        no chunk after a short final chunk) BEFORE any state changes; a slot that fails keeps its previous state, is left
        out of the batched rounds and its exception lands in ``self.last_errors[slot]`` — the other slots of the push are
        decoded normally, as the reference only fails the offending connection (infer_server.py:130-137).
        ``on_error="raise"`` then raises ``StreamSlotError`` (carrying ``errors`` and the healthy slots' ``results``);
        ``on_error="return"`` returns the healthy slots' results only."""
        eng, S = self.eng, self.S
        self.last_errors = {}
        errors = self.last_errors
        cand = {}
        for s in sorted(audio):
            a = audio[s]
            try:
                new = samples_to_float32(a) if isinstance(a, np.ndarray) else pcm_bytes_to_float32(a, channels, samp_width)
            except Exception as e:                    # undecodable message: only this slot fails
                errors[s] = e
                continue
            cand[s] = new if self.remained[s] is None else np.concatenate([self.remained[s], new])
        rates = {s: int(sample_rate.get(s, MODEL_RATE) if isinstance(sample_rate, dict) else sample_rate) for s in cand}
        off = []
        for s in sorted(cand):
            if rates[s] == MODEL_RATE:
                continue
            try:
                if not self.resample:
                    raise Exception(f"masr_b200: resampling is off for this pool (got {rates[s]} Hz, model expects "
                                    f"{MODEL_RATE} Hz)")
                output_length(len(cand[s]), rates[s])
                off.append(s)
            except Exception as e:                    # rate not accepted, or too few samples to resample: this slot only
                errors[s] = e
                del cand[s]
        if off:
            # predict.py:267-274 per slot: the carried-over tail plus the new chunk, labelled with the chunk's rate, resampled
            for s, y in zip(off, eng.resample([cand[s] for s in off], [rates[s] for s in off])):
                cand[s] = y
        slots = sorted(cand)
        out: Dict[int, Optional[dict]] = {}
        if slots:
            # one batched fbank over every slot's un-consumed samples; the tail keeps the gain (predict.py:274)
            feats, frames, status = eng.fbank([cand[s] for s in slots], self.use_db, self.target_db)
            gains = eng.last_gain.cpu().numpy() if self.use_db else np.ones(len(slots), np.float32)
            status_h = status.cpu().numpy()
            Fmax = feats.shape[1]
            pool = self.pool
            lens_host = getattr(pool, "lens_host", None)
            cap, max_len = pool.frame_bounds() if lens_host is not None else (None, None)
            short_once = bool(getattr(pool, "SHORT_ONCE", False))
            good, pending = [], {}
            for j, s in enumerate(slots):
                if status_h[j] != 0:
                    errors[s] = ValueError("无法将段规范化到目标dB，音频增益已经超过max_gain_db (300.0dB)")
                    continue
                total = self.count[s] + frames[j]
                starts = chunk_starts(total, is_end)
                if lens_host is not None and starts:
                    new_out = sum(subsampled_len(min(c + CHUNK_FRAMES, total) - c) for c in starts)
                    have = lens_host[s]
                    if short_once and have % CHUNK_OUT and new_out:
                        errors[s] = AssertionError(f"stream slot {s}: a short (final) chunk was already decoded; reset the stream first")
                        continue
                    if (cap is not None and have + new_out > cap) or (max_len is not None and have + new_out >= max_len):
                        errors[s] = AssertionError("offset: {} + x.shape[1]: {} is larger than the max_len: {}".format(
                            have, new_out, min(v for v in (cap, max_len) if v is not None)))
                        continue
                good.append((j, s))
                pending[s] = starts
            need = max((self.count[s] + frames[j] for j, s in good), default=0)
            if need > self.RING:
                self._grow_ring(need)
            R = self.RING
            # ---- commit: nothing below can fail for a validated slot ----
            for j, s in good:
                tail = cand[s][FRAME_SHIFT * frames[j]:]
                self.remained[s] = (tail * np.float32(gains[j])).astype(np.float32) if self.use_db else tail
            # append the new frames of every slot to the ring: one gather + one scatter, index lists built without a per-slot loop
            gj = np.asarray([j for j, _ in good], np.int64)
            gs = np.asarray([s for _, s in good], np.int64)
            nf = np.asarray([frames[j] for j, _ in good], np.int64)
            if nf.sum() > 0:
                seg = np.repeat(np.arange(len(good)), nf)
                off = np.arange(int(nf.sum()), dtype=np.int64) - np.repeat(np.cumsum(nf) - nf, nf)
                start = np.asarray([self.head[s] + self.count[s] for s in gs], np.int64)
                src = gj[seg] * Fmax + off
                dst = gs[seg] * R + (start[seg] + off) % R
                self.ring.index_copy_(0, self._dev_index(dst), feats.view(-1, 80).index_select(0, self._dev_index(src)))
            for j, s in good:
                self.count[s] += frames[j]
            live = [s for _, s in good]
            ends = {}
            rounds = max((len(v) for v in pending.values()), default=0)
            zero_row = S * R
            win = np.arange(CHUNK_FRAMES, dtype=np.int64)
            for r in range(rounds):
                nfr = [0] * S
                act = [s for s in live if r < len(pending[s])]
                idx = np.full((S, CHUNK_FRAMES), zero_row, np.int64)
                if act:
                    a = np.asarray(act, np.int64)
                    cur = np.asarray([pending[s][r] for s in act], np.int64)
                    cnt = np.asarray([self.count[s] for s in act], np.int64)
                    n = np.minimum(cur + CHUNK_FRAMES, cnt) - cur
                    hd = np.asarray([self.head[s] for s in act], np.int64)
                    rows = a[:, None] * R + (hd[:, None] + cur[:, None] + win[None, :]) % R
                    idx[a] = np.where(win[None, :] < n[:, None], rows, zero_row)
                    for s, c_, n_ in zip(act, cur, n):
                        nfr[s] = int(n_)
                        ends[s] = int(c_ + n_)
                batch = self.ring.index_select(0, self._dev_index(idx.reshape(-1))).view(S, CHUNK_FRAMES, 80)
                ids, maxp, tout = self.pool.step(batch, nfr)
                if self.beam is None:                # (the beam's state stays on the device: no copy per round)
                    self._fold(ids.cpu().numpy(), maxp.cpu().numpy(), tout)
            beam_out = self.beam.results([s for s in live if pending[s]], self.pool.lens_host, self.timestamps,
                                         self.n_best) if self.beam is not None else None
            for s in live:
                if not pending[s]:
                    out[s] = None
                    continue
                consumed = ends[s] - CACHED_FEATURE_NUM              # predict.py:330: keep the last 3 frames of the window
                self.head[s] = (self.head[s] + consumed) % R
                self.count[s] -= consumed
                if beam_out is not None:
                    toks, score = beam_out[s][:2]
                    out[s] = {"text": ids_to_text(toks, self.vocab), "score": score}
                    if self.timestamps:
                        ts.beam_result(out[s], toks, beam_out[s][2], self.vocab, self.dt, self.t0[s])
                    if self.n_best is not None:
                        out[s]["n_best"] = nbest_dicts(beam_out[s][-1], self.vocab)
                else:
                    out[s] = {"text": ids_to_text(self.toks[s], self.vocab), "score": greedy_score(self.acc[s], int(self.nprob[s]))}
                    if self.timestamps:
                        ts.attach(out[s], self.toks[s], self.t_start[s], self.t_end[s], self.vocab, self.dt, self.t0[s])
        if errors and on_error == "raise":
            raise StreamSlotError(errors, out)
        return out


class StreamSlotError(Exception):
    """Some slots of a ``StreamPool.push`` failed: ``errors`` maps slot -> exception, ``results`` holds what the healthy
    slots returned (their state advanced normally)."""

    def __init__(self, errors: Dict[int, Exception], results: Dict[int, Optional[dict]]):
        self.errors, self.results = dict(errors), dict(results)
        first = next(iter(self.errors.values()))
        super().__init__(f"{len(self.errors)} stream slot(s) failed: slot {next(iter(self.errors))}: {first}")
