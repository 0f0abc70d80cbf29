"""Resampling to the model rate on the GPU: ``AudioSegment.resample`` (masr/data_utils/audio.py:306-317), i.e.
``resampy.resample(x, sr, 16000, filter='kaiser_best')``, which ``AudioFeaturizer.featurize`` calls before anything
else when the audio is not at ``preprocess_conf.sample_rate`` (audio_featurizer.py:45-47).

The kernel is ``masr_resample_f32`` (csrc/resample.cu); this module holds the host side of its contract: the filter
table, the output-length rule and the launch over a packed ragged batch."""
from __future__ import annotations

from typing import Sequence

import numpy as np
import torch

MODEL_RATE = 16000               # the rate the fbank kernel implements (preprocess_conf.sample_rate of every config)

NUM_ZEROS = 64                   # kaiser_best: zero crossings of the right wing
NUM_TABLE = 2 ** 9               # table entries per zero crossing (resampy precision = 9)
ROLLOFF = 0.9475937167399596
BETA = 14.769656459379492

_table = None
_dev_tables = {}


def kaiser_best_table() -> np.ndarray:
    """Right wing of the kaiser_best interpolation filter, 32769 float64 entries, built once per process from the
    parameters resampy documents for it."""
    global _table
    if _table is None:
        n = NUM_TABLE * NUM_ZEROS
        _table = ROLLOFF * np.sinc(ROLLOFF * np.linspace(0, NUM_ZEROS, num=n + 1)) * np.kaiser(2 * n + 1, BETA)[n:]
    return _table


def device_table(device: torch.device) -> torch.Tensor:
    """The table on ``device``, uploaded once per device."""
    t = _dev_tables.get(device)
    if t is None:
        t = torch.from_numpy(kaiser_best_table()).to(device)
        _dev_tables[device] = t
    return t


def output_length(n: int, sr_orig: int, sr_new: int = MODEL_RATE) -> int:
    """resampy's output length, ``int(n * sr_new / sr_orig)``; ValueError, as resampy raises it, when that is 0.
    A row already at ``sr_new`` is not resampled and keeps its length."""
    if sr_orig == sr_new:
        return n
    if sr_orig <= 0:
        raise ValueError(f"sample rate must be positive, got {sr_orig}")
    n_out = int(n * sr_new / sr_orig)
    if n_out < 1:
        raise ValueError("Input signal length={} is too small to resample from {}->{}".format(n, sr_orig, sr_new))
    return n_out


def needs_resampling(rates) -> bool:
    """True when some row of a batch is not at the model rate (a batch at the model rate runs no resampling)."""
    return rates is not None and any(int(r) != MODEL_RATE for r in rates)


def launch(eng, x: torch.Tensor, x_offs: torch.Tensor, rates_dev: torch.Tensor, y: torch.Tensor, y_offs: torch.Tensor,
           rates: Sequence[int], out_lengths: Sequence[int]) -> None:
    """Enqueue ``masr_resample_f32`` on ``eng``'s current stream: packed ``x`` (offsets ``x_offs``, per-row rates
    ``rates_dev`` int32) -> packed ``y`` at the model rate (offsets ``y_offs``).  ``rates`` / ``out_lengths`` are the
    host copies that bound the launch."""
    tab = device_table(eng.device)
    eng._k("resample", "masr_resample_f32", x.data_ptr(), x_offs.data_ptr(), rates_dev.data_ptr(), MODEL_RATE,
           len(out_lengths), tab.data_ptr(), tab.numel(), y.data_ptr(), y_offs.data_ptr(), max(out_lengths),
           max(int(r) for r in rates))


def offsets(lengths: Sequence[int]) -> np.ndarray:
    offs = np.zeros(len(lengths) + 1, np.int64)
    np.cumsum(lengths, out=offs[1:])
    return offs
