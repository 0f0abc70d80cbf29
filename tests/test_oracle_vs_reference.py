"""CPU: the oracle against the unmodified reference, through outputs of the reference frozen in
tests/golden/reference_chunks_golden.npz (tests/golden/make_reference_chunks.py): featurizer outputs, the full-utterance
encoder output and every chunk's probabilities and caches.  Large tensors are compared on a fixed, seeded sample of
elements plus the per-frame argmax."""
import os
import sys

import numpy as np
import pytest
import torch

from conftest import GOLDEN, make_audio, synth_weights
from masr_b200 import synth
from oracle import conformer as oc, fbank as ob

sys.path.insert(0, GOLDEN)
from make_reference_chunks import sample_index  # noqa: E402


@pytest.fixture(scope="module")
def ref():
    return np.load(os.path.join(GOLDEN, "reference_chunks_golden.npz"))


def check(ref, name, got, tol, argmax=False):
    """`got` (torch / numpy) against the stored reference tensor `name`: shape, sampled elements within tol, argmax."""
    a = np.asarray(got.detach().cpu().numpy() if hasattr(got, "detach") else got, dtype=np.float32)
    assert tuple(a.shape) == tuple(ref[name + ".shape"]), (name, a.shape)
    if name in ref:
        assert np.abs(a - ref[name]).max() < tol, name
        return
    got_s = a.reshape(-1)[sample_index(name, a.size)]
    assert np.abs(got_s - ref[name + ".val"]).max() < tol, name
    if argmax:
        assert np.array_equal(a.argmax(-1), ref[name + ".argmax"]), name


def test_featurizer_matches(ref):
    for kind, seed, n in [("noise", 5, 20000), ("speech", 6, 33333)]:
        check(ref, f"fbank.{kind}{seed}", ob.featurize(make_audio(kind, seed, n).copy()), 5e-4)
    pcm = (make_audio("speech", 7, 8000) * 20000).astype(np.int16)
    check(ref, "fbank.pcm7", ob.featurize(ob.pcm_bytes_to_float32(pcm.tobytes())), 5e-4)


def test_full_and_chunk_forward_match(ref):
    sd = synth.to_torch(synth_weights(0))
    cfg = oc.ConformerConfig()
    feat = torch.from_numpy(ob.featurize(make_audio("speech", 8, 16000 * 3)))[None]
    with torch.no_grad():
        check(ref, "conformer.full", oc.get_encoder_out(sd, cfg, feat), 1e-6, argmax=True)
        st = oc.ChunkState()
        i = 0
        for cur in range(0, feat.shape[1] - 67 + 1, 64):
            pm = oc.get_encoder_out_chunk(sd, cfg, feat[:, cur:cur + 67], st, -16)
            check(ref, f"conformer.{i}.probs", pm, 1e-6, argmax=True)
            check(ref, f"conformer.{i}.att", st.att_cache, 1e-6)
            check(ref, f"conformer.{i}.cnn", st.cnn_cache, 1e-6)
            i += 1
        assert i == int(ref["conformer.chunks"][0])


def _chunk_walk(ref, prefix, step, feat):
    nf = feat.shape[1]
    i = 0
    for cur in range(0, nf - 7 + 1, 64):
        step(i, feat[:, cur:min(cur + 67, nf)])
        i += 1
    assert i == int(ref[f"{prefix}.chunks"][0])


def test_squeezeformer_chunk_forward_matches(ref):
    """oracle/squeezeformer.get_encoder_out_chunk against the reference's TorchScript-able chunk method, chunk by
    chunk (probabilities and both caches), including a short final chunk."""
    from oracle import squeezeformer as osq
    sd = synth.to_torch(synth.squeezeformer_state_dict(0, streaming=True))
    cfg = osq.SqueezeformerConfig(causal=True)
    feat = torch.from_numpy(ob.featurize(make_audio("speech", 9, 16000 * 3 + 4000)))[None]
    st = osq.ChunkState()

    def step(i, ch):
        pm = osq.get_encoder_out_chunk(sd, cfg, ch, st, -16)
        check(ref, f"squeezeformer.{i}.probs", pm, 5e-6, argmax=True)          # fp32 summation-order noise (different operand strides)
        check(ref, f"squeezeformer.{i}.att", st.att_cache, 2e-5)
        check(ref, f"squeezeformer.{i}.cnn", st.cnn_cache, 2e-5)
    with torch.no_grad():
        _chunk_walk(ref, "squeezeformer", step, feat)


def test_efficient_conformer_chunk_forward_matches(ref):
    """oracle/efficient_conformer.get_encoder_out_chunk against the reference, chunk by chunk (probabilities and
    both caches), including a short final chunk."""
    from oracle import efficient_conformer as oe
    sd = synth.to_torch(synth.efficient_conformer_state_dict(0))
    cfg = oe.EfficientConfig()
    feat = torch.from_numpy(ob.featurize(make_audio("speech", 13, 16000 * 3 + 4000)))[None]
    st = oe.ChunkState()

    def step(i, ch):
        pm = oe.get_encoder_out_chunk(sd, cfg, ch, st, -16)
        check(ref, f"efficient.{i}.probs", pm, 5e-6, argmax=True)
        check(ref, f"efficient.{i}.att", st.att_cache, 2e-5)
        check(ref, f"efficient.{i}.cnn", st.cnn_cache, 2e-5)
    with torch.no_grad():
        _chunk_walk(ref, "efficient", step, feat)


def test_deepspeech2_chunk_forward_matches(ref):
    """oracle/deepspeech2.get_encoder_out with a carried (h, c) state against the reference's
    ``get_encoder_out_chunk`` (deepspeech2/model.py:70-77), window by window."""
    from oracle import deepspeech2 as od
    sd = synth.to_torch(synth.deepspeech2_state_dict(0, streaming=True))
    cfg = od.DS2Config(bidirectional=False)
    feat = torch.from_numpy(ob.featurize(make_audio("speech", 14, 16000 * 3 + 4000)))[None]
    state = [None]

    def step(i, ch):
        pm, state[0] = od.get_encoder_out(sd, cfg, ch, state[0])
        assert pm.shape[0] == int(ref[f"deepspeech2.{i}.lens"][0])
        check(ref, f"deepspeech2.{i}.probs", pm, 5e-6, argmax=True)
        h_ref, c_ref = f"deepspeech2.{i}.att", f"deepspeech2.{i}.cnn"                 # the reference's (h, c) chunk state
        for name, got in ((h_ref, state[0][0]), (c_ref, state[0][1])):
            n = int(np.prod(ref[name + ".shape"]))
            flat = got.reshape(-1).detach().cpu().numpy()
            assert flat.size == n, name
            assert np.abs(flat[sample_index(name, n)] - ref[name + ".val"]).max() < 2e-5, name
    with torch.no_grad():
        _chunk_walk(ref, "deepspeech2", step, feat)
