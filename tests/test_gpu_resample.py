"""GPU (-m gpu): resampling to 16 kHz (``masr_resample_f32``, csrc/resample.cu) bit for bit against the restatement of
resampy's kaiser_best loop (oracle/resample.py), and ``MASRPredictor(..., resample=True)`` end to end: every entry point
at other rates equals the 16 kHz call on the oracle-resampled samples, the streaming / long-form control flow matches the
reference predictor frozen in predictor_golden_resample.json, and 16 kHz input runs exactly what it ran without the
option."""
import io
import json
import os
import wave

import numpy as np
import pytest
import torch
import yaml

from conftest import GOLDEN, synth_weights
from masr_b200 import _lib, synth
from masr_b200.resample import MODEL_RATE, device_table, offsets
from oracle.resample import resample as oracle_resample

pytestmark = pytest.mark.gpu

SCORE_TOL = 1e-3
RATES = [8000, 11025, 22050, 24000, 32000, 44100, 48000, 96000]


def kernel(waves, rates, dev="cuda"):
    """One masr_resample_f32 launch over a packed ragged batch; outputs pre-filled with NaN sentinels."""
    lengths = [len(w) for w in waves]
    out = [n if r == MODEL_RATE else int(n * MODEL_RATE / r) for n, r in zip(lengths, rates)]
    xo, yo = offsets(lengths), offsets(out)
    x = torch.from_numpy(np.concatenate(waves).astype(np.float32)).to(dev)
    y = torch.full((int(yo[-1]) + 64,), float("nan"), device=dev)
    tab = device_table(torch.device(dev, torch.cuda.current_device()))
    xo_d, yo_d = torch.from_numpy(xo).to(dev), torch.from_numpy(yo).to(dev)
    r_d = torch.tensor(rates, dtype=torch.int32, device=dev)
    _lib.call("masr_resample_f32", x.data_ptr(), xo_d.data_ptr(), r_d.data_ptr(), MODEL_RATE, len(waves), tab.data_ptr(),
              tab.numel(), y.data_ptr(), yo_d.data_ptr(), max(out), max(rates), None)
    yh = y.cpu().numpy()
    assert np.all(np.isnan(yh[int(yo[-1]):]))                 # nothing written past the last row
    return [yh[yo[i]:yo[i + 1]] for i in range(len(waves))]


def same_bits(a, b):
    return a.shape == b.shape and np.array_equal(a.view(np.int32), b.view(np.int32))


@pytest.mark.parametrize("sr", RATES)
def test_kernel_bit_identical_to_oracle(sr):
    rng = np.random.default_rng(sr)
    one = -(-sr // MODEL_RATE)                                 # fewest samples that give one output
    lengths = [one, 37, 173, sr, 10 * sr]                      # 1 output, shorter than one filter wing, 1 s, 10 s
    waves = [synth.speechlike_audio(int(rng.integers(1 << 20)), n) for n in lengths]
    waves[1] = (rng.standard_normal(37) * 0.5).astype(np.float32)
    got = kernel(waves, [sr] * len(waves))
    for w, g in zip(waves, got):
        want = oracle_resample(w, sr)
        assert len(want) == len(g) and (len(w) != one or sr < MODEL_RATE or len(g) == 1)
        assert same_bits(g, want), (sr, len(w), np.flatnonzero(g != want)[:5])


def test_kernel_30s_at_44k1():
    x = synth.speechlike_audio(5, 30 * 44100)
    assert same_bits(kernel([x], [44100])[0], oracle_resample(x, 44100))


def test_kernel_ragged_mixed_batch_copies_16k_rows_verbatim():
    rng = np.random.default_rng(64)
    rates = [int(r) for r in rng.choice(RATES + [MODEL_RATE, MODEL_RATE], 64)]
    lengths = [int(rng.integers(-(-r // MODEL_RATE), 2 * r)) for r in rates]
    waves = [(rng.standard_normal(n) * 0.3).astype(np.float32) for n in lengths]
    got = kernel(waves, rates)
    assert MODEL_RATE in rates
    for w, r, g in zip(waves, rates, got):
        assert same_bits(g, w if r == MODEL_RATE else oracle_resample(w, r)), (r, len(w))


def test_kernel_rejects_bad_launch_arguments():
    x = torch.zeros(16, device="cuda")
    o = torch.tensor([0, 16], dtype=torch.int64, device="cuda")
    r = torch.tensor([48000], dtype=torch.int32, device="cuda")
    tab = device_table(x.device)
    with pytest.raises(_lib.MasrB200Error, match="rates must be positive"):
        _lib.call("masr_resample_f32", x.data_ptr(), o.data_ptr(), r.data_ptr(), 0, 1, tab.data_ptr(), tab.numel(),
                  x.data_ptr(), o.data_ptr(), 5, 48000, None)
    with pytest.raises(_lib.MasrB200Error, match="more than 512 x"):
        _lib.call("masr_resample_f32", x.data_ptr(), o.data_ptr(), r.data_ptr(), 16000, 1, tab.data_ptr(), tab.numel(),
                  x.data_ptr(), o.data_ptr(), 5, 16000 * 513, None)


# ---- predictor ---------------------------------------------------------------------------------------------------------

def build(tmp, use_model="conformer", decoder="ctc_greedy", resample=True, lm_path="lm/none.klm", wseed=0):
    from masr_b200.predict import MASRPredictor
    sd = {"conformer": lambda: synth_weights(wseed), "efficient_conformer": lambda: synth.efficient_conformer_state_dict(wseed),
          "squeezeformer": lambda: synth.squeezeformer_state_dict(wseed),
          "deepspeech2": lambda: synth.deepspeech2_state_dict(wseed, streaming=True)}[use_model]()
    mp, vp, mi = str(tmp / f"{use_model}.pt"), str(tmp / "vocabulary.txt"), str(tmp / "mean_istd.json")
    torch.save(synth.to_torch(sd), mp)
    synth.write_vocabulary(vp)
    synth.write_mean_istd(mi, wseed)
    cfg = {"use_model": use_model, "streaming": True, "decoder": decoder,
           "preprocess_conf": {"feature_method": "fbank", "n_mels": 80, "sample_rate": 16000, "use_dB_normalization": True,
                               "target_dB": -20},
           "dataset_conf": {"dataset_vocab": vp, "mean_istd_path": mi},
           "ctc_beam_search_decoder_conf": {"alpha": 2.2, "beta": 4.3, "beam_size": 20, "cutoff_prob": 0.99, "cutoff_top_n": 40,
                                            "language_model_path": lm_path}}
    p = str(tmp / f"{use_model}.yml")
    with open(p, "w", encoding="utf-8") as f:
        yaml.safe_dump(cfg, f)
    return MASRPredictor(configs=p, model_path=mp, use_gpu=True, resample=resample)


def wav_bytes(pcm, sr):
    buf = io.BytesIO()
    with wave.open(buf, "wb") as w:
        w.setnchannels(1)
        w.setsampwidth(2)
        w.setframerate(sr)
        w.writeframes(pcm.tobytes())
    return buf.getvalue()


def clips(seed=0):
    """(rate, int16 PCM, float32 samples as the WAV reader returns them) at several rates, 1.3 - 2.9 s."""
    out = []
    for i, (sr, secs) in enumerate([(8000, 2.1), (44100, 1.3), (48000, 2.9), (16000, 1.7), (22050, 2.4)]):
        x = synth.speechlike_audio(300 + 10 * seed + i, int(sr * secs))
        pcm = (np.clip(x, -1, 1) * 32767).astype("<i2")
        out.append((sr, pcm, pcm.astype(np.float32) * np.float32(1.0 / 32768)))
    return out


@pytest.mark.parametrize("use_model,decoder", [(m, d) for m in ("conformer", "efficient_conformer", "squeezeformer", "deepspeech2")
                                               for d in ("ctc_greedy", "ctc_beam_search")])
def test_predict_entry_points_equal_16k_calls_on_oracle_resampled_input(tmp_path, use_model, decoder):
    pred = build(tmp_path, use_model, decoder)
    cl = clips()
    want = [pred.predict(audio_data=oracle_resample(x, sr) if sr != MODEL_RATE else x) for sr, _, x in cl]
    assert any(w["text"] for w in want)
    for (sr, _, x), w in zip(cl, want):
        assert pred.predict(audio_data=x.copy(), sample_rate=sr) == w, sr
    wavs = [wav_bytes(pcm, sr) for sr, pcm, _ in cl]
    assert pred.predict_batch(wavs) == want                              # mixed rates in one batch
    assert pred.predict_batch([x for sr, _, x in cl if sr == 48000], sample_rate=48000) == [want[2]]
    outs = list(pred.predict_batches([wavs[:2], wavs[2:], [wavs[3]], wavs]))
    assert outs == [want[:2], want[2:], [want[3]], want]


def test_beam_with_char_lm_equals_16k_calls(tmp_path):
    p = str(tmp_path / "o3.arpa")
    synth.character_lm_arpa(p, seed=3, order=3, n_chars=4200, n_sentences=600)
    pred = build(tmp_path, "conformer", "ctc_beam_search", lm_path=p)
    assert pred.lm is not None
    cl = clips(1)
    want = [pred.predict(audio_data=oracle_resample(x, sr) if sr != MODEL_RATE else x) for sr, _, x in cl]
    wavs = [wav_bytes(pcm, sr) for sr, pcm, _ in cl]
    assert [pred.predict(audio_data=w) for w in wavs] == want
    assert pred.predict_batch(wavs) == want
    assert list(pred.predict_batches([wavs[:3], wavs[3:]])) == [want[:3], want[3:]]


def test_wav_path_bytes_and_file_object_equal_ndarray(tmp_path):
    pred = build(tmp_path)
    sr, pcm, x = clips(2)[2]
    assert sr == 48000
    want = pred.predict(audio_data=x.copy(), sample_rate=sr)
    assert want["text"]
    path = str(tmp_path / "a48k.wav")
    with open(path, "wb") as f:
        f.write(wav_bytes(pcm, sr))
    assert pred.predict(audio_data=path) == want
    with open(path, "rb") as f:
        assert pred.predict(audio_data=f.read()) == want
    with open(path, "rb") as f:
        assert pred.predict(audio_data=f) == want
    with pytest.raises(ValueError, match="too small to resample"):
        pred.predict(audio_data=np.zeros(2, np.float32), sample_rate=48000)
    off = build(tmp_path, resample=False)
    with pytest.raises(Exception, match="resampling"):
        off.predict(audio_data=path)


def test_16k_input_runs_exactly_what_it_ran_without_the_option(tmp_path):
    for decoder in ("ctc_greedy", "ctc_beam_search"):
        on, off = build(tmp_path, decoder=decoder, resample=True), build(tmp_path, decoder=decoder, resample=False)
        cl = [c for c in clips(3) if c[0] == MODEL_RATE] + [(MODEL_RATE, None, synth.speechlike_audio(9, 16000 * 3 + 77))]
        xs = [x for _, _, x in cl]

        def run(p):
            n0 = p.predictor.launches
            r = [p.predict(audio_data=x.copy()) for x in xs]
            r.append(p.predict_batch([x.copy() for x in xs]))
            r.append(list(p.predict_batches([[xs[0]], xs, [xs[1]]])))
            pcm = (np.clip(xs[1], -1, 1) * 32767).astype("<i2")
            p.reset_stream()
            r.append([p.predict_stream(pcm[s:s + 8000].tobytes(), is_end=s + 8000 >= len(pcm)) for s in range(0, len(pcm), 8000)])
            return r, p.predictor.launches - n0
        assert run(on) == run(off), decoder


# ---- streaming and long-form control flow against the reference predictor -------------------------------------------

@pytest.fixture(scope="module")
def golden():
    with open(os.path.join(GOLDEN, "predictor_golden_resample.json"), encoding="utf-8") as f:
        return json.load(f)


@pytest.fixture(scope="module")
def conformer(tmp_path_factory, golden):
    return build(tmp_path_factory.mktemp("rs"), wseed=golden["wseed"])


# Audio upsampled from 8 kHz has nothing above 4 kHz: its upper mel bins hold only the int16 quantisation noise of the
# front-end, so a 1-ulp difference of the dB gain (GPU vs numpy) moves them by up to ~0.6 in log-mel where 16 kHz audio
# moves by ~2e-3.  Scores of such streams are compared at this looser bound; the text must still match exactly.
UPSAMPLED_SCORE_TOL = 0.05


def _same(r, w, rate=MODEL_RATE):
    if w is None:
        return r is None
    tol = UPSAMPLED_SCORE_TOL if rate < MODEL_RATE else SCORE_TOL
    return r is not None and r["text"] == w["text"] and abs(r["score"] - w["score"]) < tol


def _stream_chunks(case):
    x = synth.speechlike_audio(case["aseed"], case["samples"])
    pcm = (np.clip(x, -1, 1) * 32767).astype("<i2")
    p = case["push"]
    return [pcm[s:s + p].tobytes() for s in range(0, len(pcm), p)]


def test_whole_and_long_match_reference_golden(conformer, golden):
    for case in golden["whole"]:
        x = synth.speechlike_audio(case["aseed"], case["samples"])
        assert _same(conformer.predict(audio_data=x, sample_rate=case["rate"]), case["result"]), case["rate"]

    class ScriptedVAD:
        seen = []

        def get_speech_timestamps(self, samples, sampling_rate):
            self.seen.append([len(samples), sampling_rate])
            return [dict(s) for s in lg["stamps"]]
    lg = golden["long"]
    v = ScriptedVAD()
    x = synth.speechlike_audio(lg["aseed"], lg["samples"])
    r = conformer.predict_long(x, sample_rate=lg["rate"], vad_predictor=v)
    assert v.seen == [lg["vad_saw"]]
    assert r["text"] == lg["result"]["text"] and abs(r["score"] - lg["result"]["score"]) <= 0.011


def test_predict_stream_matches_reference_golden_push_by_push(conformer, golden):
    for case in golden["streams"]:
        conformer.reset_stream()
        chunks = _stream_chunks(case)
        got = [conformer.predict_stream(c, is_end=i == len(chunks) - 1, sample_rate=case["rate"]) for i, c in enumerate(chunks)]
        assert len(got) == len(case["pushes"])
        for i, (r, w) in enumerate(zip(got, case["pushes"])):
            assert _same(r, w, case["rate"]), (case["rate"], i, r, w)
    conformer.reset_stream()


def test_pool_with_mixed_rates_matches_predict_stream_and_golden(conformer, golden):
    g48, g8 = golden["streams"]
    extra = []
    for sr, seed, push in [(16000, 51, 16000), (44100, 52, 22050)]:
        x = synth.speechlike_audio(seed, int(sr * 3.3))
        pcm = (np.clip(x, -1, 1) * 32767).astype("<i2")
        extra.append((sr, [pcm[s:s + push].tobytes() for s in range(0, len(pcm), push)]))
    streams = {0: extra[0], 1: (8000, _stream_chunks(g8)), 2: extra[1], 3: (48000, _stream_chunks(g48))}
    rates = {s: sr for s, (sr, _) in streams.items()}
    # each stream alone through predict_stream
    alone = {}
    for s, (sr, chunks) in streams.items():
        conformer.reset_stream()
        alone[s] = [conformer.predict_stream(c, is_end=i == len(chunks) - 1, sample_rate=sr) for i, c in enumerate(chunks)]
    conformer.reset_stream()
    assert all(_same(r, w, 8000) for r, w in zip(alone[1], g8["pushes"]))
    assert all(_same(r, w) for r, w in zip(alone[3], g48["pushes"]))
    pool = conformer.create_stream_pool(4)
    got = {s: [] for s in streams}
    for rnd in range(max(len(c) for _, c in streams.values()) - 1):
        batch = {s: c[rnd] for s, (_, c) in streams.items() if rnd < len(c) - 1}
        for s, r in pool.push(batch, sample_rate=rates).items():
            got[s].append(r)
    for s, r in pool.push({s: c[-1] for s, (_, c) in streams.items()}, is_end=True, sample_rate=rates).items():
        got[s].append(r)
    for s in streams:                       # the pool's batched chunk encoder agrees with predict_stream's to float32 level
        assert len(got[s]) == len(alone[s]) and all(_same(r, w) for r, w in zip(got[s], alone[s])), s
    # without the option a push off 16 kHz fails for its slot only
    plain = conformer.create_stream_pool(2)
    plain.resample = False
    out = plain.push({0: streams[0][1][0], 1: streams[1][1][0]}, sample_rate={1: 8000}, on_error="return")
    assert 1 in plain.last_errors and 0 in out
