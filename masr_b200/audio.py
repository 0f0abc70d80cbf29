"""Host-side sample ingestion with the reference's conventions (no arithmetic on the hot path
beyond integer->float scaling, which is exact).

Mirrors the parts of ``masr.data_utils.audio.AudioSegment`` that ``MASRPredictor`` touches:
  * ``AudioSegment.__init__`` / ``_convert_samples_to_float32``   audio.py:24-32,532-546
  * ``from_ndarray`` :142-152, ``from_pcm_bytes`` :122-139 (+ ``buf_to_float`` data_utils/utils.py:382-411)
  * ``from_file`` / ``from_bytes`` for PCM WAV containers (the reference uses soundfile/PyAV,
    which are not part of the path's arithmetic; only RIFF/WAVE PCM is supported here).
dB normalisation, int16 quantisation and fbank happen on the GPU (csrc/fbank.cu).
Resampling (resampy kaiser_best, audio.py:306-317) runs on the GPU (``masr_b200.resample``, csrc/resample.cu) when the
predictor is built with ``resample=True``; otherwise a sample-rate mismatch raises.
"""
from __future__ import annotations

import io
import wave
from io import BufferedReader

import numpy as np

_INT_TYPES = (np.int8, np.int16, np.int32, np.int64)
_FLOAT_TYPES = (np.float16, np.float32, np.float64)


def samples_to_float32(samples: np.ndarray) -> np.ndarray:
    """Integers are scaled to [-1, 1) by 2^-(bits-1); multi-channel input is averaged over channels."""
    samples = np.asarray(samples)
    if samples.dtype == np.float32 and samples.ndim == 1 and samples.flags.c_contiguous:
        return samples               # already in the internal format: no copy (the engine never writes into it)
    out = samples.astype(np.float32)
    if samples.dtype in _INT_TYPES:
        out *= np.float32(1.0 / 2 ** (np.iinfo(samples.dtype).bits - 1))
    elif samples.dtype not in _FLOAT_TYPES:
        raise TypeError("Unsupported sample type: %s." % samples.dtype)
    if out.ndim >= 2:
        out = np.mean(out, 1)
    return np.ascontiguousarray(out, dtype=np.float32)


def pcm_bytes_to_float32(data: bytes, channels: int = 1, samp_width: int = 2) -> np.ndarray:
    scale = 1.0 / float(1 << ((8 * samp_width) - 1))
    x = scale * np.frombuffer(data, "<i{:d}".format(samp_width)).astype(np.float32)
    if channels > 1:
        x = x.reshape(-1, channels)
    return samples_to_float32(x)


def _read_wav(fobj):
    with wave.open(fobj, "rb") as w:
        sr, ch, sw, n = w.getframerate(), w.getnchannels(), w.getsampwidth(), w.getnframes()
        raw = w.readframes(n)
    if sw == 1:   # 8-bit WAV is unsigned
        x = (np.frombuffer(raw, np.uint8).astype(np.float32) - 128.0) / 128.0
        if ch > 1:
            x = x.reshape(-1, ch).mean(1)
        return np.ascontiguousarray(x, np.float32), sr
    return pcm_bytes_to_float32(raw, ch, sw), sr


def load_audio(audio_data, sample_rate: int = 16000):
    """``MASRPredictor._load_audio`` (predict.py:147-164): path / file object / ndarray / bytes of a
    complete file -> (float32 mono samples, sample rate)."""
    if isinstance(audio_data, str):
        with open(audio_data, "rb") as f:
            return _read_wav(f)
    if isinstance(audio_data, BufferedReader):
        return _read_wav(audio_data)
    if isinstance(audio_data, np.ndarray):
        return samples_to_float32(audio_data), sample_rate
    if isinstance(audio_data, bytes):
        return _read_wav(io.BytesIO(audio_data))
    raise Exception(f'不支持该数据类型，当前数据类型为：{type(audio_data)}')
