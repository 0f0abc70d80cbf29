"""CPU: the wide Conformer (``output_size: 512``, ``attention_heads: 8``).  The oracle at d_model=512 / heads=8 is pinned
to the reference's frozen outputs (tests/golden/conformer_wide_golden.npz, predictor_golden_wide.json, made by
tests/golden/make_wide_golden.py from the unmodified reference), and ``weights.check_supported`` names the widths each
family has kernels for."""
import json
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN, load_npz, make_audio
from masr_b200 import synth
from masr_b200.predict import CACHED_FEATURE_NUM, DECODING_WINDOW, chunk_starts
from oracle import conformer as oc, ctc as octc, fbank as ob

WIDE = {"output_size": 512, "attention_heads": 8}
_SD = {}


def wide_weights(seed):
    if seed not in _SD:
        _SD[seed] = synth.conformer_state_dict(seed, **WIDE)
    return _SD[seed]


def wide_config(causal=True):
    return oc.ConformerConfig(d_model=512, heads=8, causal=causal)


def test_wide_oracle_matches_reference():
    """Same tolerances as tests/test_oracle_golden.py uses for the 256-wide model."""
    z, meta = load_npz("conformer_wide_golden.npz")
    vocab = synth.vocabulary()
    for m in meta:
        sd = synth.to_torch(wide_weights(m["wseed"]))
        cfg = wide_config(m["streaming"])
        feat = torch.from_numpy(z[m["name"] + "/feat"])[None]
        with torch.no_grad():
            enc = oc.encode(sd, cfg, feat)
            probs = oc.ctc_probs(sd, enc)[0].numpy()
        assert enc.shape[2] == 512
        assert np.abs(enc[0].numpy() - z[m["name"] + "/enc"]).max() < 1e-5
        ids, _ = octc.best_path(probs)
        assert np.array_equal(ids, z[m["name"] + "/ids"])
        got = np.take_along_axis(probs, z[m["name"] + "/top_i"].astype(np.int64), axis=1)
        assert np.abs(got - z[m["name"] + "/top_p"]).max() < 1e-6
        score, text, _ = octc.greedy_decode(probs, vocab)
        assert text == m["text"]
        assert abs(score - m["score"]) < 1e-4


def test_wide_oracle_chunk_path_reproduces_reference_predict_stream():
    """``MASRPredictor.predict_stream`` (predict.py:237-343) on top of the oracle's chunk forward, push by push."""
    with open(os.path.join(GOLDEN, "predictor_golden_wide.json"), encoding="utf-8") as f:
        g = json.load(f)
    assert (g["output_size"], g["attention_heads"]) == (512, 8)
    sd, cfg, vocab = synth.to_torch(wide_weights(g["wseed"])), wide_config(), synth.vocabulary()
    x = make_audio(g["kind"], g["aseed"], g["samples"])
    pcm = (np.clip(x, -1, 1) * 32767).astype("<i2")
    st, gs = oc.ChunkState(), octc.GreedyStream()
    remained, cached, got = None, None, []
    for s in range(0, len(pcm), g["push"]):
        is_end = s + g["push"] >= len(pcm)
        new = ob.pcm_bytes_to_float32(pcm[s:s + g["push"]].tobytes())
        remained = new if remained is None else np.concatenate([remained, new])
        xn, _ = ob.normalize_gain(remained.copy())
        feat = ob.kaldi_fbank(ob.to_int16(xn))
        cached = feat if cached is None else np.concatenate([cached, feat], axis=0)
        remained = xn[160 * feat.shape[0]:]
        starts = chunk_starts(cached.shape[0], is_end)
        if not starts:
            got.append(None)
            continue
        for cur in starts:
            end = min(cur + DECODING_WINDOW, cached.shape[0])
            with torch.no_grad():
                probs = oc.get_encoder_out_chunk(sd, cfg, torch.from_numpy(cached[cur:end])[None], st, -16)[0].numpy()
            res = gs.push(probs, vocab)
        cached = cached[end - CACHED_FEATURE_NUM:]
        got.append({"text": res[1], "score": res[0]})
    assert st.att_cache.shape[1:] == (8, st.att_cache.shape[2], 128) and st.cnn_cache.shape[2:] == (512, 14)
    assert len(got) == len(g["pushes_pcm"])
    for r, w in zip(got, g["pushes_pcm"]):
        assert (r is None) == (w is None)
        if r is not None:
            assert r["text"] == w["text"] and abs(r["score"] - w["score"]) < 1e-3


def _tiny(sd_fn, **kw):
    """Shape-only stand-in: check_supported reads names and shapes, so two blocks are enough."""
    return synth.to_torch(sd_fn(0, vocab_size=32, **kw))


def test_check_supported_widths():
    from masr_b200.weights import UnsupportedConfig, check_supported
    check_supported(_tiny(synth.conformer_state_dict, num_blocks=2, linear_units=64, **WIDE), "conformer")
    check_supported(_tiny(synth.conformer_state_dict, num_blocks=2, linear_units=64), "conformer")
    with pytest.raises(UnsupportedConfig, match="384"):
        check_supported(_tiny(synth.conformer_state_dict, num_blocks=2, linear_units=64, output_size=384, attention_heads=6),
                        "conformer")
    with pytest.raises(UnsupportedConfig, match="512"):
        check_supported(_tiny(synth.squeezeformer_state_dict, d=512, heads=8, ffn=64, num_blocks=2), "squeezeformer")
    check_supported(_tiny(synth.squeezeformer_state_dict, ffn=64, num_blocks=2), "squeezeformer")
    eff = _tiny(synth.conformer_state_dict, num_blocks=2, linear_units=64, **WIDE)
    with pytest.raises(UnsupportedConfig, match="512"):
        check_supported(eff, "efficient_conformer")
