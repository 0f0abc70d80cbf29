"""Reader and weight packer for the silero VAD model (``silero_vad.onnx``, the model the reference's ``VADPredictor``
runs, masr/infer_utils/vad_predictor.py).

``read_model`` decodes the protobuf wire format of the parts of ModelProto, GraphProto, NodeProto, AttributeProto
(subgraphs included) and TensorProto (float / int64, raw or repeated data) that an ONNX export uses; the ``onnx``
package is not needed.  ``pack_silero_16k`` takes the model's 16 kHz branch (``If sr == 16000`` at the top level),
checks that it is the network the kernels of csrc/vad.cu implement — op sequence, initializer shapes, conv attributes
and the front-end constants — and packs its weights into the three float32 buffers the kernels read:

* ``basis``  [258, 256]: the STFT basis, rows 0..128 the real part, 129..257 the imaginary part;
* ``enc``    the front-end and encoder convs followed by the layer-1 LSTM input weights, transposed (``W_ih1^T``
  [64, 256], so that the threads of one gate row each read consecutive words), and the summed biases ``Wb1 + Rb1``
  [256], in the order of ``ENC_LAYOUT``;
* ``rec``    ``W_hh1``, ``W_ih2``, ``W_hh2`` (each [256, 64]), ``Wb2 + Rb2`` [256], the decoder's weight [64] and bias.

The LSTM gate rows are permuted from ONNX's order (i, o, f, c) to i, f, g, o, the order the kernels use.
Any other graph (an 8 kHz-only export, silero v4/v5 with another layout) is refused with ``UnsupportedVadModel``.
"""
from __future__ import annotations

import struct
from typing import Dict, List, Tuple

import numpy as np


class UnsupportedVadModel(ValueError):
    pass


# ---- protobuf -------------------------------------------------------------------------------------------------------
class _Reader:
    def __init__(self, buf: bytes):
        self.buf, self.pos = memoryview(buf), 0

    def varint(self) -> int:
        shift = val = 0
        while True:
            if self.pos >= len(self.buf):
                raise UnsupportedVadModel("truncated protobuf varint")
            byte = self.buf[self.pos]
            self.pos += 1
            val |= (byte & 0x7F) << shift
            if not byte & 0x80:
                return val
            shift += 7

    def __iter__(self):
        while self.pos < len(self.buf):
            tag = self.varint()
            field, wire = tag >> 3, tag & 7
            if wire == 0:
                yield field, wire, self.varint()
            elif wire in (1, 5):
                n = 8 if wire == 1 else 4
                yield field, wire, bytes(self.buf[self.pos:self.pos + n])
                self.pos += n
            elif wire == 2:
                n = self.varint()
                if self.pos + n > len(self.buf):
                    raise UnsupportedVadModel("truncated protobuf field")
                yield field, wire, bytes(self.buf[self.pos:self.pos + n])
                self.pos += n
            else:
                raise UnsupportedVadModel(f"protobuf wire type {wire} does not occur in an ONNX model")


def _signed(v: int) -> int:
    return v - (1 << 64) if v & (1 << 63) else v


def _repeated_ints(wire: int, val) -> List[int]:
    if wire == 0:
        return [_signed(val)]
    r, out = _Reader(val), []
    while r.pos < len(r.buf):
        out.append(_signed(r.varint()))
    return out


def _repeated_floats(wire: int, val) -> List[float]:
    return list(struct.unpack(f"<{len(val) // 4}f", val))


_NP = {1: "<f4", 6: "<i4", 7: "<i8", 9: "?", 11: "<f8"}


def read_tensor(buf: bytes) -> Tuple[str, np.ndarray]:
    """TensorProto -> (name, array): float32 / int64 (also int32, bool, double) from raw_data or the typed fields."""
    name, dims, dtype, raw, floats, ints = "", [], 1, None, [], []
    for f, w, v in _Reader(buf):
        if f == 1:
            dims += _repeated_ints(w, v)
        elif f == 2:
            dtype = v
        elif f == 8:
            name = v.decode()
        elif f == 9:
            raw = v
        elif f == 4:
            floats += _repeated_floats(w, v)
        elif f in (5, 7):
            ints += _repeated_ints(w, v)
    if dtype not in _NP:
        raise UnsupportedVadModel(f"tensor {name!r}: data type {dtype} is not supported")
    if raw is not None:
        arr = np.frombuffer(raw, _NP[dtype]).copy()
    else:
        arr = np.array(floats if dtype == 1 else ints, _NP[dtype])
    if arr.size != int(np.prod(dims, dtype=np.int64)):
        raise UnsupportedVadModel(f"tensor {name!r}: {arr.size} values for dims {dims}")
    return name, arr.reshape(dims)


class OnnxNode:
    __slots__ = ("op", "name", "inputs", "outputs", "attrs")

    def __init__(self):
        self.op, self.name, self.inputs, self.outputs, self.attrs = "", "", [], [], {}


class OnnxGraph:
    __slots__ = ("name", "nodes", "initializers", "inputs", "outputs")

    def __init__(self):
        self.name, self.nodes, self.initializers, self.inputs, self.outputs = "", [], {}, [], []


def read_attribute(buf: bytes):
    name, scalar, ints, floats = "", None, [], []
    for f, w, v in _Reader(buf):
        if f == 1:
            name = v.decode()
        elif f == 2:
            scalar = struct.unpack("<f", v)[0]
        elif f == 3:
            scalar = _signed(v)
        elif f == 4:
            scalar = v.decode("utf-8", "replace")
        elif f == 5:
            scalar = read_tensor(v)[1]
        elif f == 6:
            scalar = read_graph(v)
        elif f == 7:
            floats += _repeated_floats(w, v) if w == 2 else [struct.unpack("<f", v)[0]]
        elif f == 8:
            ints += _repeated_ints(w, v)
    return name, scalar if scalar is not None else (ints or floats)


def read_node(buf: bytes) -> OnnxNode:
    n = OnnxNode()
    for f, w, v in _Reader(buf):
        if f == 1:
            n.inputs.append(v.decode())
        elif f == 2:
            n.outputs.append(v.decode())
        elif f == 3:
            n.name = v.decode()
        elif f == 4:
            n.op = v.decode()
        elif f == 5:
            k, a = read_attribute(v)
            n.attrs[k] = a
    return n


def _value_info_name(buf: bytes) -> str:
    for f, _, v in _Reader(buf):
        if f == 1:
            return v.decode()
    return ""


def read_graph(buf: bytes) -> OnnxGraph:
    g = OnnxGraph()
    for f, w, v in _Reader(buf):
        if f == 1:
            g.nodes.append(read_node(v))
        elif f == 2:
            g.name = v.decode()
        elif f == 5:
            k, t = read_tensor(v)
            g.initializers[k] = t
        elif f == 11:
            g.inputs.append(_value_info_name(v))
        elif f == 12:
            g.outputs.append(_value_info_name(v))
    return g


def read_model(data: bytes) -> OnnxGraph:
    """ModelProto bytes -> its main graph (field 7)."""
    for f, w, v in _Reader(data):
        if f == 7 and w == 2:
            return read_graph(v)
    raise UnsupportedVadModel("no graph in the ONNX model")


# ---- the silero 16 kHz network --------------------------------------------------------------------------------------
# Op sequence of the 16 kHz branch of silero_vad.onnx (PyTorch 1.12 export, opset 16).
BRANCH_OPS = (
    "Shape", "Gather", "Unsqueeze", "Gather", "Unsqueeze", "Concat", "Reshape", "Unsqueeze", "Pad", "Shape", "Gather",
    "Equal", "If", "Conv", "Slice", "Pow", "Slice", "Pow", "Add", "Sqrt", "Mul", "Add", "Log", "Shape", "Shape",
    "Gather", "Squeeze", "Equal", "If", "ReduceMean", "Slice", "Slice", "Slice", "Slice", "Concat", "Conv",
    "ReduceMean", "Neg", "Add", "Concat", "Conv", "Relu", "Conv", "Conv", "Add", "Relu", "Conv", "Relu", "Conv",
    "Relu", "Conv", "Conv", "Add", "Relu", "Conv", "Relu", "Conv", "Relu", "Conv", "Add", "Relu", "Conv", "Relu",
    "Conv", "Relu", "Conv", "Conv", "Add", "Relu", "Conv", "Relu", "Transpose", "Transpose", "Shape", "Gather",
    "Squeeze", "Cast", "If", "Transpose", "Relu", "Conv", "Sigmoid", "Shape", "Gather", "Equal", "If", "ReduceMean",
    "Unsqueeze")

# The 18 Conv nodes of the branch, in graph order: (role, weight shape, group, stride, pads).  The unnamed 1x1 convs
# between the encoder blocks are the exporter's fusions of each block's trailing conv + batch norm.
CONVS = (
    ("stft", (258, 1, 256), 1, 64, (0, 0)),
    ("norm", (1, 1, 7), 1, 1, (0, 0)),
    ("dw0", (258, 1, 5), 258, 1, (2, 2)), ("pw0", (16, 258, 1), 1, 1, (0, 0)), ("pj0", (16, 258, 1), 1, 1, (0, 0)),
    ("c1", (16, 16, 1), 1, 2, (0, 0)),
    ("dw3", (16, 1, 5), 16, 1, (2, 2)), ("pw3", (32, 16, 1), 1, 1, (0, 0)), ("pj3", (32, 16, 1), 1, 1, (0, 0)),
    ("c2", (32, 32, 1), 1, 2, (0, 0)),
    ("dw7", (32, 1, 5), 32, 1, (2, 2)), ("pw7", (32, 32, 1), 1, 1, (0, 0)),
    ("c3", (32, 32, 1), 1, 2, (0, 0)),
    ("dw11", (32, 1, 5), 32, 1, (2, 2)), ("pw11", (64, 32, 1), 1, 1, (0, 0)), ("pj11", (64, 32, 1), 1, 1, (0, 0)),
    ("c4", (64, 64, 1), 1, 1, (0, 0)),
    ("dec", (1, 64, 1), 1, 1, (0, 0)),
)

# Named initializers the branch must carry, with their shapes.
NAMED = {
    "model.feature_extractor.forward_basis_buffer": (258, 1, 256),
    "model.adaptive_normalization.filter_": (1, 1, 7),
    "model.first_layer.0.dw_conv.0.weight": (258, 1, 5), "model.first_layer.0.dw_conv.0.bias": (258,),
    "model.first_layer.0.pw_conv.0.weight": (16, 258, 1), "model.first_layer.0.pw_conv.0.bias": (16,),
    "model.first_layer.0.proj.weight": (16, 258, 1), "model.first_layer.0.proj.bias": (16,),
    "model.encoder.3.0.dw_conv.0.weight": (16, 1, 5), "model.encoder.3.0.pw_conv.0.weight": (32, 16, 1),
    "model.encoder.3.0.proj.weight": (32, 16, 1),
    "model.encoder.7.0.dw_conv.0.weight": (32, 1, 5), "model.encoder.7.0.pw_conv.0.weight": (32, 32, 1),
    "model.encoder.11.0.dw_conv.0.weight": (32, 1, 5), "model.encoder.11.0.pw_conv.0.weight": (64, 32, 1),
    "model.encoder.11.0.proj.weight": (64, 32, 1),
    "model.decoder.decoder.1.weight": (1, 64, 1), "model.decoder.decoder.1.bias": (1,),
}

HIDDEN = 64
REFLECT_PAD = 96           # samples of reflect padding on each side of a window
LOG_MUL, LOG_ADD = 1048576.0, 1.0

# float32 element counts of the packed encoder buffer, in order (mirrored by the offsets in csrc/vad.cu)
ENC_LAYOUT = (
    ("dw0.w", 258 * 5), ("dw0.b", 258), ("pw0.w", 16 * 258), ("pw0.b", 16), ("pj0.w", 16 * 258), ("pj0.b", 16),
    ("c1.w", 16 * 16), ("c1.b", 16),
    ("dw3.w", 16 * 5), ("dw3.b", 16), ("pw3.w", 32 * 16), ("pw3.b", 32), ("pj3.w", 32 * 16), ("pj3.b", 32),
    ("c2.w", 32 * 32), ("c2.b", 32),
    ("dw7.w", 32 * 5), ("dw7.b", 32), ("pw7.w", 32 * 32), ("pw7.b", 32),
    ("c3.w", 32 * 32), ("c3.b", 32),
    ("dw11.w", 32 * 5), ("dw11.b", 32), ("pw11.w", 64 * 32), ("pw11.b", 64), ("pj11.w", 64 * 32), ("pj11.b", 64),
    ("c4.w", 64 * 64), ("c4.b", 64),
    ("norm.w", 7), ("log", 2),
    ("wih1t", 64 * 256), ("b1", 256),
)
REC_LAYOUT = (("whh1", 256 * 64), ("wih2", 256 * 64), ("whh2", 256 * 64), ("b2", 256), ("dec.w", 64), ("dec.b", 1))

# ONNX gate blocks (i, o, f, c) -> the kernels' order (i, f, g, o)
GATE_ORDER = (0, 2, 3, 1)


def _reorder_gates(a: np.ndarray) -> np.ndarray:
    blocks = a.reshape(4, HIDDEN, *a.shape[1:])
    return np.concatenate([blocks[k] for k in GATE_ORDER]).astype(np.float32)


def _const(env: Dict[str, np.ndarray], name: str) -> np.ndarray:
    if name not in env:
        raise UnsupportedVadModel(f"constant {name!r} is not an initializer")
    return env[name]


def _branch_16k(g: OnnxGraph) -> OnnxGraph:
    ops = [n.op for n in g.nodes]
    if ops != ["Equal", "If"] or g.inputs[:4] != ["input", "sr", "h", "c"]:
        raise UnsupportedVadModel("not the silero VAD v3/v4 graph (expected inputs input, sr, h, c and a top-level "
                                  f"If on the sample rate; found ops {ops[:8]} and inputs {g.inputs})")
    eq, br = g.nodes
    rate = g.initializers.get(eq.inputs[1])
    if eq.inputs[0] != "sr" or rate is None or int(np.asarray(rate).reshape(-1)[0]) != 16000:
        raise UnsupportedVadModel("the top-level If does not select on sr == 16000")
    return br.attrs["then_branch"]


def pack_silero_16k(g: OnnxGraph) -> Dict[str, np.ndarray]:
    """Check the 16 kHz branch and pack it: {'basis', 'enc', 'rec'} float32 buffers (see the module docstring)."""
    b16 = _branch_16k(g)
    env = dict(g.initializers)
    env.update(b16.initializers)
    ops = tuple(n.op for n in b16.nodes)
    if ops != BRANCH_OPS:
        raise UnsupportedVadModel(f"the 16 kHz branch has {len(ops)} nodes that are not the silero v3/v4 network "
                                  f"({len(BRANCH_OPS)} expected)")
    for name, shape in NAMED.items():
        if name not in env:
            raise UnsupportedVadModel(f"initializer {name} is missing")
        if tuple(env[name].shape) != shape:
            raise UnsupportedVadModel(f"initializer {name} has shape {tuple(env[name].shape)}, expected {shape}")

    convs = [n for n in b16.nodes if n.op == "Conv"]
    w: Dict[str, Tuple[np.ndarray, np.ndarray]] = {}
    for n, (role, shape, group, stride, pads) in zip(convs, CONVS):
        wt = _const(env, n.inputs[1])
        if tuple(wt.shape) != shape:
            raise UnsupportedVadModel(f"conv {role} ({n.inputs[1]}) has weight shape {tuple(wt.shape)}, expected {shape}")
        attrs = (n.attrs.get("group", 1), list(n.attrs.get("strides", [1])), list(n.attrs.get("pads", [0, 0])),
                 list(n.attrs.get("dilations", [1])))
        if attrs != (group, [stride], list(pads), [1]):
            raise UnsupportedVadModel(f"conv {role} has (group, strides, pads, dilations) {attrs}")
        bias = _const(env, n.inputs[2]) if len(n.inputs) > 2 and n.inputs[2] else None
        if bias is not None and tuple(bias.shape) != (shape[0],):
            raise UnsupportedVadModel(f"conv {role} has bias shape {tuple(bias.shape)}")
        w[role] = (wt.astype(np.float32), None if bias is None else bias.astype(np.float32))
    if w["stft"][1] is not None or w["norm"][1] is not None or any(w[r][1] is None for r in w if r not in ("stft", "norm")):
        raise UnsupportedVadModel("unexpected conv biases")

    pad = next(n for n in b16.nodes if n.op == "Pad")
    pads = [int(v) for v in _const(env, pad.inputs[1]).reshape(-1)]
    if pad.attrs.get("mode") != "reflect" or pads != [0, 0, 0, REFLECT_PAD, 0, 0, 0, REFLECT_PAD]:
        raise UnsupportedVadModel(f"window padding is {pad.attrs.get('mode')} {pads}, expected reflect by {REFLECT_PAD}")
    sl = [n for n in b16.nodes if n.op == "Slice"][:2]
    bounds = [[int(_const(env, k).reshape(-1)[0]) for k in n.inputs[1:5]] for n in sl]
    if bounds != [[129, 2 ** 63 - 1, 1, 1], [0, 129, 1, 1]]:
        raise UnsupportedVadModel(f"STFT real / imaginary split is {bounds}")
    for n in (m for m in b16.nodes if m.op == "Pow"):
        if float(_const(env, n.inputs[1])) != 2.0:
            raise UnsupportedVadModel("magnitude is not sqrt(re^2 + im^2)")
    mul = next(n for n in b16.nodes if n.op == "Mul")
    add = b16.nodes[ops.index("Mul") + 1]
    log_mul = float(_const(env, mul.inputs[1]))
    log_add = float(_const(env, add.inputs[0]))

    inner = b16.nodes[ops.index("Cast") + 1].attrs["then_branch"]
    lstms = [n for n in inner.nodes if n.op == "LSTM"]
    if len(lstms) != 2:
        raise UnsupportedVadModel(f"{len(lstms)} LSTM layers, expected 2")
    layers = []
    for n in lstms:
        if (n.attrs.get("hidden_size"), n.attrs.get("direction", "forward"), n.attrs.get("layout", 0),
                n.attrs.get("input_forget", 0), "activations" in n.attrs, "clip" in n.attrs) != (HIDDEN, "forward", 0, 0, False, False):
            raise UnsupportedVadModel("LSTM attributes are not a plain forward LSTM with hidden_size 64")
        W, R, B = (_const(inner.initializers, k) for k in n.inputs[1:4])
        if W.shape != (1, 4 * HIDDEN, HIDDEN) or R.shape != (1, 4 * HIDDEN, HIDDEN) or B.shape != (1, 8 * HIDDEN):
            raise UnsupportedVadModel(f"LSTM weights have shapes {W.shape}, {R.shape}, {B.shape}")
        layers.append((W[0], R[0], B[0, :4 * HIDDEN].astype(np.float64) + B[0, 4 * HIDDEN:]))

    parts = {
        "dw0.w": w["dw0"][0], "dw0.b": w["dw0"][1], "pw0.w": w["pw0"][0], "pw0.b": w["pw0"][1],
        "pj0.w": w["pj0"][0], "pj0.b": w["pj0"][1], "c1.w": w["c1"][0], "c1.b": w["c1"][1],
        "dw3.w": w["dw3"][0], "dw3.b": w["dw3"][1], "pw3.w": w["pw3"][0], "pw3.b": w["pw3"][1],
        "pj3.w": w["pj3"][0], "pj3.b": w["pj3"][1], "c2.w": w["c2"][0], "c2.b": w["c2"][1],
        "dw7.w": w["dw7"][0], "dw7.b": w["dw7"][1], "pw7.w": w["pw7"][0], "pw7.b": w["pw7"][1],
        "c3.w": w["c3"][0], "c3.b": w["c3"][1],
        "dw11.w": w["dw11"][0], "dw11.b": w["dw11"][1], "pw11.w": w["pw11"][0], "pw11.b": w["pw11"][1],
        "pj11.w": w["pj11"][0], "pj11.b": w["pj11"][1], "c4.w": w["c4"][0], "c4.b": w["c4"][1],
        "norm.w": w["norm"][0], "log": np.array([log_mul, log_add]),
        "wih1t": _reorder_gates(layers[0][0]).T, "b1": _reorder_gates(layers[0][2]),
    }
    rec_parts = {
        "whh1": _reorder_gates(layers[0][1]), "wih2": _reorder_gates(layers[1][0]), "whh2": _reorder_gates(layers[1][1]),
        "b2": _reorder_gates(layers[1][2]), "dec.w": w["dec"][0], "dec.b": w["dec"][1],
    }

    def flat(layout, src):
        out = []
        for name, size in layout:
            a = np.asarray(src[name], np.float32).reshape(-1)
            assert a.size == size, (name, a.size, size)
            out.append(a)
        return np.ascontiguousarray(np.concatenate(out))

    return {"basis": np.ascontiguousarray(w["stft"][0].reshape(258, 256)), "enc": flat(ENC_LAYOUT, parts),
            "rec": flat(REC_LAYOUT, rec_parts)}


def load_silero_16k(path: str) -> Dict[str, np.ndarray]:
    with open(path, "rb") as fh:
        return pack_silero_16k(read_model(fh.read()))
