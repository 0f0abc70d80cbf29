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
The recognition half then sends all segments of a recording through ONE batched pass (``predict_batch``) instead of the
reference's one-``predict``-per-segment loop (predict.py:216-224).
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Sequence

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
    and the single-CTA recurrence, whatever its length.  ``window_size_samples`` is 512, 1024 or 1536."""

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

    def _stream(self):
        import torch
        return torch.cuda.current_stream(self.device).cuda_stream

    def encode(self, samples):
        """Layer-1 LSTM gate inputs ``W_ih1 x + b1`` [N * T, 256] (rows i, f, g, o) of 16 kHz ``samples`` (a float32
        array or CUDA tensor)."""
        import torch
        from . import _lib
        x = torch.as_tensor(samples, dtype=torch.float32).to(self.device).contiguous()
        W = self.kw["window_size_samples"]
        n_windows = (x.numel() + W - 1) // W
        gx = torch.empty(n_windows * (W // 512), self.gate_width, dtype=torch.float32, device=self.device)
        _lib.call("masr_silero_vad_encode_f32", x.data_ptr(), x.numel(), W, self.weights["basis"].data_ptr(),
                  self.weights["enc"].data_ptr(), gx.data_ptr(), self._stream())
        return gx

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
