"""Long-form recognition support (SURVEY.md §8 f4): the segmentation half of ``MASRPredictor.predict_long``.

The reference runs the silero VAD network (an ONNX model shipped next to masr/infer_utils/vad_predictor.py, evaluated with
onnxruntime on the CPU, one 512-sample window per session call) and turns its per-window speech probabilities into
speech segments with a hysteresis state machine (vad_predictor.py:106-175).  Here the network runs on the GPU
(``GpuSileroVAD``): the model file is read and packed by ``masr_b200.silero``, one launch encodes every window of the
recording in parallel and one persistent single-CTA launch runs the LSTM across all windows (csrc/vad.cu).
``SileroVAD`` keeps the reference's onnxruntime form for hosts that have it.  The state machine is restated here
(``speech_timestamps_from_probs``) and pinned to the reference's own implementation by
tests/golden/vad_timestamps_golden.json; any object with the reference's ``get_speech_timestamps(samples,
sampling_rate)`` method can be plugged into ``MASRPredictor.predict_long``.
The streaming half of the reference's VADPredictor (``reset_states`` / ``__call__`` / ``stream_vad``,
vad_predictor.py:73-104, 177-213) runs on the GPU too: ``GpuSileroVAD`` carries the (h, c) state of every stream on the
device, and ``GpuSileroVAD.slots(n)`` advances many independent streams with one encoder and one recurrence launch
(csrc/vad.cu, one CTA per stream).  Its hysteresis is restated in ``stream_vad_step``, pinned to the reference by
tests/golden/stream_vad_golden.json.
The recognition half then sends all segments of a recording through ONE batched pass (``predict_batch``) instead of the
reference's one-``predict``-per-segment loop (predict.py:216-224).
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Optional, Sequence

import numpy as np


def speech_timestamps_from_probs(speech_probs: Sequence[float], audio_length_samples: int, sampling_rate: int = 16000,
                                 threshold: float = 0.5, min_speech_duration_ms: int = 250, min_silence_duration_ms: int = 100,
                                 window_size_samples: int = 512, speech_pad_ms: int = 30) -> List[Dict[str, int]]:
    """vad_predictor.py:114-175: per-window speech probabilities -> [{'start', 'end'}] in samples.

    A segment opens at the first window with p >= threshold, closes once p has stayed below threshold - 0.15 for
    ``min_silence_duration_ms`` (the close point is where the silence began), is kept if longer than
    ``min_speech_duration_ms``; afterwards segments are padded by ``speech_pad_ms`` (or share the gap when it is shorter
    than two pads)."""
    min_speech_samples = sampling_rate * min_speech_duration_ms / 1000
    min_silence_samples = sampling_rate * min_silence_duration_ms / 1000
    speech_pad_samples = sampling_rate * speech_pad_ms / 1000
    W = window_size_samples
    triggered = False
    speeches: List[Dict[str, int]] = []
    cur: Dict[str, int] = {}
    neg_threshold = threshold - 0.15
    temp_end = 0
    for i, p in enumerate(speech_probs):
        if p >= threshold and temp_end:
            temp_end = 0
        if p >= threshold and not triggered:
            triggered = True
            cur["start"] = W * i
            continue
        if p < neg_threshold and triggered:
            if not temp_end:
                temp_end = W * i
            if W * i - temp_end < min_silence_samples:
                continue
            cur["end"] = temp_end
            if cur["end"] - cur["start"] > min_speech_samples:
                speeches.append(cur)
            temp_end = 0
            cur = {}
            triggered = False
    if cur and (audio_length_samples - cur["start"]) > min_speech_samples:
        cur["end"] = audio_length_samples
        speeches.append(cur)
    for i, sp in enumerate(speeches):
        if i == 0:
            sp["start"] = int(max(0, sp["start"] - speech_pad_samples))
        if i != len(speeches) - 1:
            silence = speeches[i + 1]["start"] - sp["end"]
            if silence < 2 * speech_pad_samples:
                sp["end"] += int(silence // 2)
                speeches[i + 1]["start"] = int(max(0, speeches[i + 1]["start"] - silence // 2))
            else:
                sp["end"] = int(min(audio_length_samples, sp["end"] + speech_pad_samples))
                speeches[i + 1]["start"] = int(max(0, speeches[i + 1]["start"] - speech_pad_samples))
        else:
            sp["end"] = int(min(audio_length_samples, sp["end"] + speech_pad_samples))
    return speeches


class StreamVADState:
    """The per-stream state of the reference's ``stream_vad``: ``triggered``, ``temp_end`` and ``current_sample``."""

    def __init__(self):
        self.reset()

    def reset(self):
        self.triggered, self.temp_end, self.current_sample = False, 0, 0


def stream_vad_step(st, speech_prob: float, sampling_rate: int, threshold: float = 0.5,
                    min_silence_duration_ms: int = 100, speech_pad_ms: int = 30, return_seconds: bool = False):
    """vad_predictor.py:194-213: one window's speech probability -> ``{'start': ...}``, ``{'end': ...}`` or None.

    ``st`` (``StreamVADState`` or any object with its three fields) must already count this window in
    ``current_sample``.  A start is announced at ``current_sample - pad``; the first window below ``threshold - 0.15``
    while triggered sets ``temp_end = current_sample``, a window at or above ``threshold`` clears it, and once
    ``current_sample - temp_end`` reaches ``min_silence`` the end is announced at ``temp_end + pad``.  The arithmetic is the
    reference's: float sample counts, ``int()`` (or seconds rounded to 0.1) on the way out."""
    min_silence_samples = sampling_rate * min_silence_duration_ms / 1000
    speech_pad_samples = sampling_rate * speech_pad_ms / 1000
    if (speech_prob >= threshold) and st.temp_end:
        st.temp_end = 0
    if (speech_prob >= threshold) and not st.triggered:
        st.triggered = True
        speech_start = st.current_sample - speech_pad_samples
        return {'start': int(speech_start) if not return_seconds else round(speech_start / sampling_rate, 1)}
    if (speech_prob < threshold - 0.15) and st.triggered:
        if not st.temp_end:
            st.temp_end = st.current_sample
        if st.current_sample - st.temp_end < min_silence_samples:
            return None
        speech_end = st.temp_end + speech_pad_samples
        st.temp_end = 0
        st.triggered = False
        return {'end': int(speech_end) if not return_seconds else round(speech_end / sampling_rate, 1)}
    return None


class ProbabilityVAD:
    """Adapter: a callable ``window_probs(samples float32[n], sampling_rate) -> sequence of per-window speech probabilities``
    (one per ``window_size_samples`` window, the last one zero-padded) behind the reference's ``get_speech_timestamps``."""

    def __init__(self, window_probs, threshold: float = 0.5, min_speech_duration_ms: int = 250, min_silence_duration_ms: int = 100,
                 window_size_samples: int = 512, speech_pad_ms: int = 30):
        self.window_probs = window_probs
        self.kw = dict(threshold=threshold, min_speech_duration_ms=min_speech_duration_ms,
                       min_silence_duration_ms=min_silence_duration_ms, window_size_samples=window_size_samples,
                       speech_pad_ms=speech_pad_ms)

    def get_speech_timestamps(self, audio: np.ndarray, sampling_rate: int):
        probs = self.window_probs(np.asarray(audio, np.float32), sampling_rate)
        return speech_timestamps_from_probs(list(probs), len(audio), sampling_rate, **self.kw)


class SileroVAD(ProbabilityVAD):
    """The reference's VADPredictor (vad_predictor.py:11-104): the silero ONNX network on the host through onnxruntime,
    512-sample windows with the LSTM state carried across windows.  Needs ``onnxruntime`` and the model file."""

    def __init__(self, path: str, **kw):
        try:
            import onnxruntime
        except ImportError as e:                                    # not part of this image: fail loudly, no fallback
            raise RuntimeError("SileroVAD needs the `onnxruntime` package (the reference's VAD runs the silero ONNX model on "
                               "the CPU); pass another `vad_predictor` to predict_long or install it") from e
        self.session = onnxruntime.InferenceSession(path)
        super().__init__(self._probs, **kw)

    def _probs(self, audio: np.ndarray, sr: int):
        if sr != 16000 and sr % 16000 == 0:
            audio, sr = audio[::sr // 16000], 16000
        if sr not in (8000, 16000):
            raise ValueError("Supported sampling rates: [8000, 16000] (or multiply of 16000)")
        W = self.kw["window_size_samples"]
        h = np.zeros((2, 1, 64), np.float32)
        c = np.zeros((2, 1, 64), np.float32)
        out = []
        for s in range(0, len(audio), W):
            chunk = audio[s:s + W]
            if len(chunk) < W:
                chunk = np.pad(chunk, (0, W - len(chunk)))
            o, h, c = self.session.run(None, {"input": chunk[None].astype(np.float32), "h": h, "c": c,
                                              "sr": np.array(sr, dtype=np.int64)})
            out.append(float(np.asarray(o).item()))
        return out


class GpuSileroVAD(ProbabilityVAD):
    """The reference's VADPredictor with the silero network on the GPU (csrc/vad.cu): the model file's 16 kHz branch is
    checked and packed once (``masr_b200.silero``), then each recording costs two launches, the window-parallel encoder
    and the single-CTA recurrence, whatever its length.  ``window_size_samples`` is 512, 1024 or 1536.

    The reference's streaming interface is here as well: ``reset_states``, ``__call__`` on one window per stream
    (``[W]`` or ``[B, W]``, the (h, c) of every stream kept on the device) and ``stream_vad``; ``slots(n)`` keeps the
    state of ``n`` streams that advance by any number of samples at a time."""

    def __init__(self, path: str, device="cuda", **kw):
        import torch
        from . import _lib, silero
        super().__init__(self._probs, **kw)
        W = self.kw["window_size_samples"]
        if W not in (512, 1024, 1536):
            raise ValueError(f"window_size_samples = {W}: the 16 kHz silero network takes 512, 1024 or 1536")
        if not torch.cuda.is_available():
            raise _lib.MasrB200Error("GpuSileroVAD needs a CUDA device (there is no CPU fallback)")
        packed = silero.load_silero_16k(path)
        sizes = (C.c_int64 * 4)()
        _lib.call("masr_silero_vad_layout", sizes)
        want = {"basis": sizes[0], "enc": sizes[1], "rec": sizes[2]}
        for k, n in want.items():
            if packed[k].size != n:
                raise _lib.MasrB200Error(f"packed silero buffer {k} has {packed[k].size} floats, the kernels read {n}")
        self.gate_width = int(sizes[3])
        self.device = torch.device(device)
        self.weights = {k: torch.from_numpy(v).to(self.device) for k, v in packed.items()}
        self._init_stream_state()

    def _init_stream_state(self):
        # VADPredictor.__init__ (vad_predictor.py:40-51)
        kw = self.kw
        self.threshold, self.min_speech_duration_ms = kw["threshold"], kw["min_speech_duration_ms"]
        self.min_silence_duration_ms, self.window_size_samples = kw["min_silence_duration_ms"], kw["window_size_samples"]
        self.speech_pad_ms = kw["speech_pad_ms"]
        self.sample_rates = [8000, 16000]
        self.reset_states()

    def _stream(self):
        import torch
        return torch.cuda.current_stream(self.device).cuda_stream

    def encode(self, samples, window: Optional[int] = None):
        """Layer-1 LSTM gate inputs ``W_ih1 x + b1`` [N * T, 256] (rows i, f, g, o) of 16 kHz ``samples`` (a float32
        array or CUDA tensor)."""
        import torch
        from . import _lib
        x = torch.as_tensor(samples, dtype=torch.float32).to(self.device).contiguous()
        W = self.kw["window_size_samples"] if window is None else int(window)
        n_windows = (x.numel() + W - 1) // W
        gx = torch.empty(n_windows * (W // 512), self.gate_width, dtype=torch.float32, device=self.device)
        _lib.call("masr_silero_vad_encode_f32", x.data_ptr(), x.numel(), W, self.weights["basis"].data_ptr(),
                  self.weights["enc"].data_ptr(), gx.data_ptr(), self._stream())
        return gx

    def recur_slots(self, gx, win_off: Sequence[int], state, window: Optional[int] = None):
        """Per-window speech probabilities [win_off[-1]] of several streams from the gate inputs of ``encode`` (CUDA
        tensor): stream s owns windows [win_off[s], win_off[s+1]) and starts from ``state[s]`` ([n, 4, 64] CUDA float32:
        h1, c1, h2, c2), which is advanced in place.  A stream without windows keeps its state.  One launch."""
        import torch
        from . import _lib
        W = self.kw["window_size_samples"] if window is None else int(window)
        T = W // 512
        n = len(win_off) - 1
        if state.shape != (n, 4, 64) or state.dtype != torch.float32 or not state.is_contiguous():
            raise ValueError(f"state must be a contiguous float32 [{n}, 4, 64] tensor")
        total = int(win_off[-1])
        gx = gx.contiguous()
        if gx.shape[0] != total * T:
            raise ValueError(f"gate inputs have {gx.shape[0]} rows, the windows need {total * T}")
        off = torch.tensor(np.asarray(win_off, np.int32), device=self.device)
        logits = torch.empty(max(total * T, 1), dtype=torch.float32, device=self.device)
        probs = torch.empty(max(total, 1), dtype=torch.float32, device=self.device)
        if total:
            _lib.call("masr_silero_vad_recur_slots_f32", gx.data_ptr(), off.data_ptr(), n, W, self.weights["rec"].data_ptr(),
                      state.data_ptr(), logits.data_ptr(), probs.data_ptr(), self._stream())
        return probs[:total]

    def slots(self, n: int) -> "VadSlots":
        """Device state of ``n`` independent streams (``VadSlots``)."""
        return VadSlots(self, n)

    # ---- the reference's streaming interface (vad_predictor.py:54-104, 177-213) ------------------------------------
    def _validate_input(self, x, sr: int):
        """vad_predictor.py:54-71, as written: 1-D input becomes one row; at a multiple of 16 kHz ``x[::step]`` keeps every
        step-th ROW of the batch (the samples are not decimated) and the rate is taken as 16 kHz."""
        x = np.asarray(x)
        if len(x.shape) == 1:
            x = x[np.newaxis, :]
        if len(x.shape) > 2:
            raise ValueError(f"Too many dimensions for input audio chunk {x.ndim}")
        if sr != 16000 and (sr % 16000 == 0):
            step = sr // 16000
            x = x[::step]
            sr = 16000
        if sr not in self.sample_rates:
            raise ValueError(f"Supported sampling rates: {self.sample_rates} (or multiply of 16000)")
        if sr / x.shape[1] > 31.25:
            raise ValueError("Input audio chunk is too short")
        return x, sr

    def reset_states(self, batch_size: int = 1):
        """vad_predictor.py:73-81: zero (h, c) for ``batch_size`` streams and the ``stream_vad`` state."""
        self._state_batch, self._slots = batch_size, None          # (device state made on the next call)
        self._last_sr = 0
        self._last_batch_size = 0
        self.triggered = False
        self.temp_end = 0
        self.current_sample = 0

    def __call__(self, x, sr: int):
        """vad_predictor.py:83-104: one window per stream (``[W]`` or ``[B, W]``, W = 512, 1024 or 1536 at 16 kHz) ->
        speech probabilities [B, 1].  Each row continues its own (h, c); the state is reset when the batch size or the
        rate changes, and on the first call after ``reset_states``."""
        x, sr = self._validate_input(x, sr)
        batch_size = x.shape[0]
        if not self._last_batch_size:
            self.reset_states(batch_size)
        if self._last_sr and (self._last_sr != sr):
            self.reset_states(batch_size)
        if self._last_batch_size and (self._last_batch_size != batch_size):
            self.reset_states(batch_size)
        out = self._run_windows(x, sr)
        self._last_sr = sr
        self._last_batch_size = batch_size
        return out

    def _run_windows(self, x: np.ndarray, sr: int) -> np.ndarray:
        """The network on one window per row of ``x`` [B, W], each row from its own carried state -> [B, 1]."""
        if sr == 8000:
            raise ValueError("GpuSileroVAD runs the silero network's 16 kHz branch only; resample 8 kHz audio to 16 kHz")
        B, W = x.shape
        if W not in (512, 1024, 1536):
            raise ValueError(f"window of {W} samples: the 16 kHz silero network on the GPU takes 512, 1024 or 1536")
        if self._slots is None or self._slots.n != B:
            self._slots = VadSlots(self, B)
        gx = self.encode(np.ascontiguousarray(x, np.float32).reshape(-1), window=W)
        probs = self.recur_slots(gx, list(range(B + 1)), self._slots.state, window=W)
        return probs.cpu().numpy().reshape(B, 1)

    def stream_vad(self, x, sampling_rate, return_seconds=False):
        """vad_predictor.py:177-213: one window of a live stream -> ``{'start'}``, ``{'end'}`` or None (``stream_vad_step``).
        As in the reference, ``current_sample`` is advanced before the network runs, so the reset of the first call
        after ``reset_states`` clears that window's count."""
        if len(x) < self.window_size_samples:
            return None
        window_size_samples = len(x[0]) if len(x.shape) == 2 else len(x)
        self.current_sample += window_size_samples
        speech_prob = self(x, sampling_rate).item()
        return stream_vad_step(self, speech_prob, sampling_rate, self.threshold, self.min_silence_duration_ms,
                               self.speech_pad_ms, return_seconds)

    def recur(self, gx):
        """Per-window speech probabilities [N] from the gate inputs of ``encode`` (CUDA tensor)."""
        import torch
        from . import _lib
        W = self.kw["window_size_samples"]
        T = W // 512
        gx = gx.contiguous()
        n_windows = gx.shape[0] // T
        logits = torch.empty(gx.shape[0], dtype=torch.float32, device=self.device)
        probs = torch.empty(n_windows, dtype=torch.float32, device=self.device)
        _lib.call("masr_silero_vad_recur_f32", gx.data_ptr(), n_windows, W, self.weights["rec"].data_ptr(),
                  logits.data_ptr(), probs.data_ptr(), self._stream())
        return probs

    def _probs(self, audio: np.ndarray, sr: int):
        if sr != 16000 and sr % 16000 == 0:
            audio, sr = audio[::sr // 16000], 16000
        if sr == 8000:
            raise ValueError("GpuSileroVAD runs the silero network's 16 kHz branch only; resample 8 kHz audio to 16 kHz")
        if sr != 16000:
            raise ValueError("Supported sampling rates: [8000, 16000] (or multiply of 16000)")
        if len(audio) == 0:
            return []
        return self.recur(self.encode(np.ascontiguousarray(audio, np.float32))).cpu().numpy().tolist()


class VadSlots:
    """The silero state of ``n`` independent live streams (slots) on the device: ``state`` [n, 4, 64] (h1, c1, h2, c2
    per slot) and, per slot, the samples received since the last complete window.

    ``advance({slot: samples})`` cuts each listed slot's carry plus its new samples into complete windows of
    ``window_size_samples``, gathers every slot's complete windows into one buffer and runs ONE encoder launch (each window
    is encoded on its own, so its gate inputs do not depend on where it lands) and ONE recurrence launch (one CTA per slot,
    each resuming from its state).  A slot's probabilities therefore equal one pass over its whole stream, however its
    samples were split across calls."""

    def __init__(self, vad: GpuSileroVAD, n: int):
        import torch
        if n < 1:
            raise ValueError(f"n = {n}: at least one slot")
        self.vad, self.n, self.W = vad, int(n), int(vad.kw["window_size_samples"])
        self.state = torch.zeros(self.n, 4, 64, dtype=torch.float32, device=vad.device)
        self.carry: List[np.ndarray] = [np.zeros(0, np.float32) for _ in range(self.n)]

    def reset(self, slot: int):
        """Start ``slot`` over: zero state, no carried samples."""
        self.state[slot].zero_()
        self.carry[slot] = np.zeros(0, np.float32)

    def advance(self, samples: Dict[int, np.ndarray]) -> Dict[int, np.ndarray]:
        """slot -> 16 kHz float32 samples  ->  slot -> the speech probabilities of the windows they completed (float32,
        possibly empty).  Slots not listed are not touched."""
        W = self.W
        parts, counts = [], np.zeros(self.n, np.int64)
        for s in sorted(samples):
            if not 0 <= s < self.n:
                raise IndexError(f"slot {s} out of range (0..{self.n - 1})")
            x = np.asarray(samples[s], np.float32).reshape(-1)
            buf = np.concatenate([self.carry[s], x]) if len(self.carry[s]) else x
            k = len(buf) // W
            counts[s] = k
            if k:
                parts.append(buf[:k * W])
            self.carry[s] = np.array(buf[k * W:], np.float32)
        off = np.concatenate([[0], np.cumsum(counts)])
        if off[-1] == 0:
            return {s: np.zeros(0, np.float32) for s in samples}
        gx = self.vad.encode(np.concatenate(parts))
        probs = self.vad.recur_slots(gx, off.tolist(), self.state).cpu().numpy()
        return {s: probs[off[s]:off[s + 1]] for s in samples}
