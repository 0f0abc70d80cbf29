"""CPU: the product's ONNX reader (masr_b200/silero.py) on a ModelProto encoded by hand here, the packing of the real
silero model and the rejection of other graphs, the float64 graph interpreter (oracle/silero_vad.py), and, where
onnxruntime is installed, the interpreter against it."""
import os
import struct

import numpy as np
import pytest

from masr_b200 import silero
from oracle import silero_vad as sv

needs_model = pytest.mark.skipif(not os.path.exists(sv.MODEL_PATH),
                                 reason="oracle/_ref/silero_vad.onnx is fetched by build() from the reference tree")


# ---- a minimal protobuf encoder, independent of both decoders ------------------------------------------------------
def _varint(v):
    v &= (1 << 64) - 1
    out = bytearray()
    while True:
        b = v & 0x7F
        v >>= 7
        out.append(b | (0x80 if v else 0))
        if not v:
            return bytes(out)


def _key(field, wire):
    return _varint(field << 3 | wire)


def _ld(field, payload):
    return _key(field, 2) + _varint(len(payload)) + payload


def _vi(field, v):
    return _key(field, 0) + _varint(v)


def _value_info(name):
    return _ld(1, name.encode())


def test_reader_decodes_a_hand_encoded_model():
    raw = np.arange(6, dtype="<f4") * 0.5
    t_raw = _ld(1, _varint(2) + _varint(3)) + _vi(2, 1) + _ld(8, b"w") + _ld(9, raw.tobytes())           # packed dims
    t_int = _vi(1, 3) + _vi(2, 7) + _ld(8, b"idx") + _vi(7, 5) + _vi(7, -2) + _vi(7, 1 << 40)              # int64_data
    t_flt = _vi(1, 2) + _vi(2, 1) + _ld(8, b"f") + _ld(4, struct.pack("<2f", 1.5, -3.25))                  # float_data
    sub = _ld(1, _ld(1, b"w") + _ld(2, b"z") + _ld(4, b"Identity")) + _ld(2, b"sub") + _ld(12, _value_info("z"))
    attrs = (_ld(5, _ld(1, b"pads") + _ld(8, _varint(2) + _varint(-1 & (2 ** 64 - 1))) + _vi(20, 7)) +
             _ld(5, _ld(1, b"strides") + _vi(8, 64) + _vi(20, 7)) +
             _ld(5, _ld(1, b"alpha") + _key(2, 5) + struct.pack("<f", 0.25) + _vi(20, 1)) +
             _ld(5, _ld(1, b"mode") + _ld(4, b"reflect") + _vi(20, 3)) +
             _ld(5, _ld(1, b"group") + _vi(3, 258) + _vi(20, 2)) +
             _ld(5, _ld(1, b"then_branch") + _ld(6, sub) + _vi(20, 5)))
    node = _ld(1, b"x") + _ld(1, b"w") + _ld(1, b"") + _ld(2, b"y") + _ld(3, b"n0") + _ld(4, b"Conv") + attrs
    graph = (_ld(1, node) + _ld(2, b"g") + _ld(5, t_raw) + _ld(5, t_int) + _ld(5, t_flt) +
             _ld(11, _value_info("x")) + _ld(12, _value_info("y")))
    model = _vi(1, 8) + _ld(2, b"pytorch") + _ld(7, graph) + _ld(8, _ld(1, b"") + _vi(2, 16))
    g = silero.read_model(model)
    assert g.name == "g" and g.inputs == ["x"] and g.outputs == ["y"]
    np.testing.assert_array_equal(g.initializers["w"], raw.reshape(2, 3))
    assert g.initializers["w"].dtype == np.float32
    np.testing.assert_array_equal(g.initializers["idx"], np.array([5, -2, 1 << 40], np.int64))
    np.testing.assert_array_equal(g.initializers["f"], np.array([1.5, -3.25], np.float32))
    (n,) = g.nodes
    assert (n.op, n.name, n.inputs, n.outputs) == ("Conv", "n0", ["x", "w", ""], ["y"])
    assert n.attrs["pads"] == [2, -1] and n.attrs["strides"] == [64] and n.attrs["alpha"] == 0.25
    assert n.attrs["mode"] == "reflect" and n.attrs["group"] == 258
    sg = n.attrs["then_branch"]
    assert sg.name == "sub" and sg.nodes[0].op == "Identity" and sg.outputs == ["z"]
    with pytest.raises(silero.UnsupportedVadModel):
        silero.read_model(_vi(1, 8) + _ld(7, graph)[:-5])        # truncated inside the graph
    with pytest.raises(silero.UnsupportedVadModel, match="silero"):
        silero.pack_silero_16k(g)                               # a valid model, but not the silero network


@needs_model
def test_real_model_packs_with_the_listed_shapes():
    from masr_b200 import _lib
    with open(sv.MODEL_PATH, "rb") as fh:
        g = silero.read_model(fh.read())
    p = silero.pack_silero_16k(g)
    assert p["basis"].shape == (258, 256) and all(v.dtype == np.float32 for v in p.values())
    sizes = (__import__("ctypes").c_int64 * 4)()
    _lib.call("masr_silero_vad_layout", sizes)
    assert (p["basis"].size, p["enc"].size, p["rec"].size, 256) == tuple(sizes)
    assert p["enc"].size == sum(n for _, n in silero.ENC_LAYOUT) and p["rec"].size == sum(n for _, n in silero.REC_LAYOUT)
    # against the oracle's independent decoding of the same file: the basis, and the LSTM gates moved to i, f, g, o
    og = sv.load(sv.MODEL_PATH)
    np.testing.assert_array_equal(p["basis"], og.inits["model.feature_extractor.forward_basis_buffer"][:, 0])
    (W1, R1, b1), (W2, R2, b2) = sv.lstm_weights(og)
    perm = np.concatenate([np.arange(64) + 64 * k for k in (0, 2, 3, 1)])
    enc = dict(zip([n for n, _ in silero.ENC_LAYOUT], np.split(p["enc"], np.cumsum([n for _, n in silero.ENC_LAYOUT])[:-1])))
    rec = dict(zip([n for n, _ in silero.REC_LAYOUT], np.split(p["rec"], np.cumsum([n for _, n in silero.REC_LAYOUT])[:-1])))
    np.testing.assert_array_equal(enc["wih1t"].reshape(64, 256), W1[perm].T.astype(np.float32))
    np.testing.assert_allclose(enc["b1"], b1[perm], rtol=0, atol=1e-6)
    np.testing.assert_array_equal(rec["whh1"].reshape(256, 64), R1[perm].astype(np.float32))
    np.testing.assert_array_equal(rec["wih2"].reshape(256, 64), W2[perm].astype(np.float32))
    np.testing.assert_array_equal(rec["whh2"].reshape(256, 64), R2[perm].astype(np.float32))
    np.testing.assert_allclose(rec["b2"], b2[perm], rtol=0, atol=1e-6)
    np.testing.assert_array_equal(enc["log"], [1048576.0, 1.0])


@needs_model
def test_other_graphs_are_rejected():
    with open(sv.MODEL_PATH, "rb") as fh:
        data = fh.read()
    g = silero.read_model(data)
    b16 = g.nodes[1].attrs["then_branch"]
    name = "model.encoder.3.0.pw_conv.0.weight"
    keep = b16.initializers.get(name, g.initializers.get(name))
    g.initializers[name] = np.zeros((48, 16, 1), np.float32)
    with pytest.raises(silero.UnsupportedVadModel, match="pw_conv"):
        silero.pack_silero_16k(g)
    g.initializers[name] = keep
    silero.pack_silero_16k(g)
    sr_const = g.nodes[0].inputs[1]
    g.initializers[sr_const] = np.array(8000, np.int64)         # an export whose If selects another rate
    with pytest.raises(silero.UnsupportedVadModel, match="16000"):
        silero.pack_silero_16k(g)
    g.initializers[sr_const] = np.array(16000, np.int64)
    b16.nodes.pop(b16.nodes.index(next(n for n in b16.nodes if n.op == "Sigmoid")))
    with pytest.raises(silero.UnsupportedVadModel, match="16 kHz branch"):
        silero.pack_silero_16k(g)


@needs_model
def test_interpreter_is_deterministic_and_carries_state():
    from conftest import make_audio
    g = sv.load()
    a = make_audio("speech", 7, 16000 + 200)
    p1, k1 = sv.speech_probs(g, a, keep=(sv.LSTM_INPUT,))
    p2, k2 = sv.speech_probs(g, a, keep=(sv.LSTM_INPUT,))
    assert len(p1) == 32 and np.array_equal(p1, p2)
    assert all(np.array_equal(x[sv.LSTM_INPUT], y[sv.LSTM_INPUT]) for x, y in zip(k1, k2))
    assert k1[0][sv.LSTM_INPUT].shape == (1, 1, 64)
    # the state is carried: the second window's probability depends on the first window
    q, _ = sv.speech_probs(g, a[512:1024])
    assert q[0] != p1[1]
    # the LSTM restated from the traced LSTM inputs gives the graph's own probabilities
    (W1, _, b1), _ = sv.lstm_weights(g)
    gx = np.concatenate([k[sv.LSTM_INPUT][:, 0] @ W1.T + b1 for k in k1])
    dec_w = g.inits["model.decoder.decoder.1.weight"].reshape(64)
    dec_b = float(g.inits["model.decoder.decoder.1.bias"][0])
    np.testing.assert_allclose(sv.lstm_f64(gx, sv.lstm_weights(g), 1, dec_w, dec_b), p1, rtol=0, atol=1e-12)


@needs_model
def test_interpreter_matches_onnxruntime():
    ort = pytest.importorskip("onnxruntime")
    from conftest import make_audio
    g = sv.load()
    sess = ort.InferenceSession(sv.MODEL_PATH)
    for W in (512, 1024, 1536):
        a = make_audio("speech", 11, 3 * 16000 + 77)
        want, _ = sv.speech_probs(g, a, window=W)
        h = np.zeros((2, 1, 64), np.float32)
        c = np.zeros((2, 1, 64), np.float32)
        got = []
        for s in range(0, len(a), W):
            chunk = np.pad(a[s:s + W], (0, max(0, W - len(a[s:s + W]))))
            o, h, c = sess.run(None, {"input": chunk[None], "h": h, "c": c, "sr": np.array(16000, np.int64)})
            got.append(float(np.asarray(o).item()))
        np.testing.assert_allclose(got, want, rtol=0, atol=1e-5)
