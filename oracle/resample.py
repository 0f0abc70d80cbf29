"""``resampy.resample(x, sr_orig, sr_new, filter='kaiser_best')`` (the call of AudioSegment.resample,
masr/data_utils/audio.py:306-317) restated in numpy, operation for operation, for a 1-D float32 signal.

resampy is not a dependency of this project, so its interpolation loop is specified here and the GPU kernel
(``masr_resample_f32``, csrc/resample.cu) must equal this function bit for bit:

* ``ratio = float(sr_new) / sr_orig``; ``n_out = int(n * sr_new / sr_orig)``; ValueError when ``n_out < 1``;
* the filter table is ``WIN * ratio`` when ``ratio < 1`` else ``WIN``, and ``delta = diff(win, append=win[-1])``;
* ``scale = min(1, ratio)``, ``index_step = int(scale * 512)``, ``t_out = arange(n_out) * (1.0 / ratio)``;
* per output (float64): ``n = int(t)``, ``frac = scale * (t - n)``, ``idx = frac * 512``, ``offset = int(idx)``,
  ``eta = idx - offset``; the left wing adds ``(win[j] + eta * delta[j]) * x[n - i]`` for
  ``i < min(n + 1, (nwin - offset) // index_step)``, ``j = offset + i * index_step``; then ``frac = scale - frac`` and
  the right wing adds the same over ``x[n + k + 1]`` for ``k < min(n_orig - n - 1, (nwin - offset) // index_step)``;
* the accumulator is float32, rounded after every tap (``y = float32(float64(y) + w * float64(x))``), and no product
  is fused into an add (numba, which runs resampy's loop, does not contract for a float32 signal).

``WIN`` is the right wing of kaiser_best regenerated from the parameters resampy documents (64 zero crossings,
2**9 entries per crossing, rolloff 0.9475937167399596, Kaiser beta 14.769656459379492).  Whether it equals the table
shipped in resampy's ``kaiser_best.npz`` is UNVERIFIED (DESIGN.md §2).

The loop over output samples is vectorised: for each tap index, every output that still has that tap is updated at
once, so each output's own taps are still added in the order above.
"""
import numpy as np

NUM_ZEROS = 64
PRECISION = 9
NUM_TABLE = 2 ** PRECISION
ROLLOFF = 0.9475937167399596
BETA = 14.769656459379492

_WIN = None


def kaiser_best_table() -> np.ndarray:
    """The 32769 float64 entries of the kaiser_best filter's right wing (``WIN[0] == ROLLOFF``)."""
    global _WIN
    if _WIN is None:
        n = NUM_TABLE * NUM_ZEROS
        _WIN = ROLLOFF * np.sinc(ROLLOFF * np.linspace(0, NUM_ZEROS, num=n + 1)) * np.kaiser(2 * n + 1, BETA)[n:]
    return _WIN


def output_length(n: int, sr_orig: int, sr_new: int) -> int:
    n_out = int(n * sr_new / sr_orig)
    if n_out < 1:
        raise ValueError("Input signal length={} is too small to resample from {}->{}".format(n, sr_orig, sr_new))
    return n_out


def resample(x: np.ndarray, sr_orig: int, sr_new: int = 16000) -> np.ndarray:
    x = np.asarray(x, dtype=np.float32)
    assert x.ndim == 1
    n_orig = x.shape[0]
    n_out = output_length(n_orig, sr_orig, sr_new)
    ratio = float(sr_new) / sr_orig
    win = kaiser_best_table()
    if ratio < 1:
        win = win * ratio
    delta = np.diff(win, append=win[-1])
    nwin = win.shape[0]
    scale = min(1.0, ratio)
    index_step = int(scale * NUM_TABLE)
    t_out = np.arange(n_out) * (1.0 / ratio)
    x64 = x.astype(np.float64)
    y = np.zeros(n_out, np.float32)

    n = t_out.astype(np.int64)
    frac = scale * (t_out - n)
    for right in (False, True):
        if right:
            frac = scale - frac
        idx = frac * NUM_TABLE
        offset = idx.astype(np.int64)
        eta = idx - offset
        reach = (nwin - offset) // index_step
        taps = np.minimum(n_orig - n - 1, reach) if right else np.minimum(n + 1, reach)
        for i in range(int(taps.max(initial=0))):
            m = taps > i
            j = offset[m] + i * index_step
            w = win[j] + eta[m] * delta[j]
            xi = x64[n[m] + i + 1] if right else x64[n[m] - i]
            y[m] = (y[m].astype(np.float64) + w * xi).astype(np.float32)
    return y
