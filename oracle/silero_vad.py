"""The silero VAD network of the reference's ``VADPredictor`` (masr/infer_utils/vad_predictor.py), executed in float64
from the model file's own ONNX graph — TEST INFRASTRUCTURE, NOT PRODUCT CODE.

``silero_vad.onnx`` is a PyTorch 1.12 export whose top level is an ``If`` on ``sr == 16000``.  This module decodes
the protobuf wire format itself (the ``onnx`` package is not a dependency) and interprets the graph node by node,
subgraphs included, for the op set the model uses.  Every tensor is float64 (int64 for shapes and indices), so the
interpreter is the float64 restatement the GPU kernels (csrc/vad.cu) are measured against.

It has its own protobuf decoder on purpose: the product's reader (``masr_b200/silero.py``) decodes the same file,
and a shared decoder would let one decoding bug pass both sides.

``speech_probs`` drives the graph the way ``VADPredictor.get_speech_timestamps`` does (vad_predictor.py:113-126):
the state ``h``, ``c`` (both ``[2, 1, 64]``) starts at zero for each recording and is carried from window to window,
one call per ``window`` samples, and the last window is zero-padded to full length.
"""
from __future__ import annotations

import hashlib
import os
import struct
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

MODEL_SHA256 = "a35ebf52fd3ce5f1469b2a36158dba761bc47b973ea3382b3186ca15b1f5af28"
MODEL_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref", "silero_vad.onnx")


# ---- protobuf wire format ------------------------------------------------------------------------------------------
def _varint(b: bytes, p: int) -> Tuple[int, int]:
    r = s = 0
    while True:
        x = b[p]
        p += 1
        r |= (x & 0x7F) << s
        s += 7
        if x < 0x80:
            return r, p


def _fields(b: bytes):
    p, n = 0, len(b)
    while p < n:
        key, p = _varint(b, p)
        f, w = key >> 3, key & 7
        if w == 0:
            v, p = _varint(b, p)
        elif w == 1:
            v, p = b[p:p + 8], p + 8
        elif w == 5:
            v, p = b[p:p + 4], p + 4
        elif w == 2:
            ln, p = _varint(b, p)
            v, p = b[p:p + ln], p + ln
        else:
            raise ValueError(f"protobuf wire type {w} is not used by ONNX")
        yield f, w, v


def _int64(v: int) -> int:
    return v - (1 << 64) if v >= 1 << 63 else v


def _ints(w: int, v) -> List[int]:
    if w != 2:
        return [_int64(v)]
    out, p = [], 0
    while p < len(v):
        x, p = _varint(v, p)
        out.append(_int64(x))
    return out


_DTYPES = {1: np.float32, 6: np.int32, 7: np.int64, 9: np.bool_, 11: np.float64}


def _tensor(b: bytes) -> Tuple[str, np.ndarray]:
    dims, dt, name, raw, fl, il = [], 1, "", None, [], []
    for f, w, v in _fields(b):
        if f == 1:
            dims += _ints(w, v)
        elif f == 2:
            dt = v
        elif f == 8:
            name = v.decode()
        elif f == 9:
            raw = bytes(v)
        elif f == 4:
            fl += list(np.frombuffer(v, "<f4")) if w == 2 else [struct.unpack("<f", v)[0]]
        elif f == 7:
            il += _ints(w, v)
    if raw is not None:
        a = np.frombuffer(raw, np.dtype(_DTYPES[dt]).newbyteorder("<")).copy()
    else:
        a = np.array(fl if dt == 1 else il, _DTYPES[dt])
    a = a.reshape(dims)
    return name, a.astype(np.float64) if a.dtype.kind == "f" else a.astype(np.int64) if a.dtype.kind in "iu" else a


class Node:
    def __init__(self, b: bytes):
        self.inputs: List[str] = []
        self.outputs: List[str] = []
        self.op, self.name, self.attrs = "", "", {}
        for f, w, v in _fields(b):
            if f == 1:
                self.inputs.append(v.decode())
            elif f == 2:
                self.outputs.append(v.decode())
            elif f == 3:
                self.name = v.decode()
            elif f == 4:
                self.op = v.decode()
            elif f == 5:
                k, a = _attribute(v)
                self.attrs[k] = a


def _attribute(b: bytes):
    name, val, ints, floats = "", None, [], []
    for f, w, v in _fields(b):
        if f == 1:
            name = v.decode()
        elif f == 2:
            val = struct.unpack("<f", v)[0]
        elif f == 3:
            val = _int64(v)
        elif f == 4:
            val = bytes(v).decode()
        elif f == 5:
            val = _tensor(v)[1]
        elif f == 6:
            val = Graph(v)
        elif f == 7:
            floats += list(np.frombuffer(v, "<f4")) if w == 2 else [struct.unpack("<f", v)[0]]
        elif f == 8:
            ints += _ints(w, v)
    if val is None:
        val = ints if ints else floats
    return name, val


class Graph:
    def __init__(self, b: bytes):
        self.nodes: List[Node] = []
        self.inits: Dict[str, np.ndarray] = {}
        self.inputs: List[str] = []
        self.outputs: List[str] = []
        for f, w, v in _fields(b):
            if f == 1:
                self.nodes.append(Node(v))
            elif f == 5:
                k, a = _tensor(v)
                self.inits[k] = a
            elif f in (11, 12):
                nm = next(bytes(x).decode() for g, _, x in _fields(v) if g == 1)
                (self.inputs if f == 11 else self.outputs).append(nm)


def load(path: str = MODEL_PATH) -> Graph:
    with open(path, "rb") as fh:
        b = fh.read()
    for f, w, v in _fields(b):
        if f == 7:
            return Graph(v)
    raise ValueError(f"{path}: no graph in the ModelProto")


# ---- interpreter ---------------------------------------------------------------------------------------------------
def _conv(x, w, b, a):
    (pl, pr), s, g = a.get("pads", [0, 0]), a.get("strides", [1])[0], a.get("group", 1)
    assert a.get("dilations", [1]) == [1] and x.ndim == 3
    x = np.pad(x, ((0, 0), (0, 0), (pl, pr)))
    K = w.shape[2]
    L = (x.shape[2] - K) // s + 1
    cols = np.lib.stride_tricks.sliding_window_view(x, K, axis=2)[:, :, ::s][:, :, :L]    # [B, C, L, K]
    ci, co = x.shape[1] // g, w.shape[0] // g
    y = np.concatenate([np.einsum("bclk,ock->bol", cols[:, i * ci:(i + 1) * ci], w[i * co:(i + 1) * co])
                        for i in range(g)], axis=1)
    return y if b is None else y + b[None, :, None]


def _lstm(x, W, R, B, h0, c0, a):
    assert a.get("direction", "forward") == "forward" and a.get("layout", 0) == 0 and not a.get("input_forget", 0)
    H = a["hidden_size"]
    W, R = W[0], R[0]
    bias = B[0, :4 * H] + B[0, 4 * H:]
    h, c = h0[0], c0[0]
    ys = []
    sig = lambda v: 1.0 / (1.0 + np.exp(-v))
    for t in range(x.shape[0]):
        z = x[t] @ W.T + h @ R.T + bias                       # gates in ONNX order i, o, f, c
        i, o, f, g = sig(z[:, :H]), sig(z[:, H:2 * H]), sig(z[:, 2 * H:3 * H]), np.tanh(z[:, 3 * H:])
        c = f * c + i * g
        h = o * np.tanh(c)
        ys.append(h)
    return np.stack(ys)[:, None], h[None], c[None]


def _slice(x, starts, ends, axes=None, steps=None):
    axes = range(len(starts)) if axes is None else axes
    steps = [1] * len(starts) if steps is None else steps
    sl = [slice(None)] * x.ndim
    for s, e, ax, st in zip(starts, ends, axes, steps):
        n = x.shape[ax]
        s, e = int(s), int(e)
        s = s + n if s < 0 else s
        e = e + n if e < 0 else e
        if st > 0:
            s, e = min(max(s, 0), n), min(max(e, 0), n)
        else:
            s, e = min(max(s, -1), n - 1), min(max(e, -1), n - 1)
        sl[ax] = slice(s, e if e >= 0 else None, int(st))
    return x[tuple(sl)]


def _pad(x, pads, mode):
    r = x.ndim
    width = [(int(pads[i]), int(pads[i + r])) for i in range(r)]
    return np.pad(x, width, mode={"constant": "constant", "reflect": "reflect", "edge": "edge"}[mode])


def _reshape(x, shape):
    shape = [x.shape[i] if s == 0 else int(s) for i, s in enumerate(shape)]
    return x.reshape(shape)


class Interpreter:
    """Executes a Graph; ``trace`` (when a dict) receives every tensor computed, by name, subgraphs included."""

    def __init__(self, graph: Graph):
        self.graph = graph

    def run(self, feeds: Dict[str, np.ndarray], trace: Optional[dict] = None) -> List[np.ndarray]:
        return self._run(self.graph, dict(feeds), trace)

    def _run(self, g: Graph, scope: dict, trace) -> List[np.ndarray]:
        env = dict(scope)
        env.update(g.inits)
        for n in g.nodes:
            ins = [env[i] if i else None for i in n.inputs]
            outs = self._op(n, ins, env, trace)
            for k, v in zip(n.outputs, outs):
                env[k] = v
                if trace is not None:
                    trace[k] = v
        return [env[o] for o in g.outputs]

    def _op(self, n: Node, x, env, trace):
        a, op = n.attrs, n.op
        if op == "If":
            return self._run(a["then_branch"] if bool(np.asarray(x[0]).reshape(-1)[0]) else a["else_branch"], env, trace)
        if op == "Conv":
            return [_conv(x[0], x[1], x[2] if len(x) > 2 else None, a)]
        if op == "LSTM":
            return list(_lstm(x[0], x[1], x[2], x[3], x[5], x[6], a))
        if op == "Pad":
            return [_pad(x[0], x[1], a.get("mode", "constant"))]
        if op == "Slice":
            return [_slice(x[0], *[v for v in x[1:]])]
        if op == "Concat":
            return [np.concatenate(x, axis=a["axis"])]
        if op == "Reshape":
            return [_reshape(x[0], x[1])]
        if op == "Transpose":
            return [np.transpose(x[0], a["perm"])]
        if op == "Squeeze":
            return [np.squeeze(x[0], axis=tuple(int(v) for v in x[1]))]
        if op == "Unsqueeze":
            y = x[0]
            for ax in sorted(int(v) % (np.ndim(y) + len(x[1])) for v in x[1]):
                y = np.expand_dims(y, ax)
            return [y]
        if op == "Shape":
            return [np.array(np.shape(x[0])[a.get("start", 0):], np.int64)]
        if op == "Gather":
            return [np.take(x[0], x[1], axis=a.get("axis", 0))]
        if op == "ConstantOfShape":
            return [np.full([int(v) for v in x[0]], a["value"].reshape(-1)[0], a["value"].dtype)]
        if op == "ReduceMean":
            return [np.mean(x[0], axis=tuple(a["axes"]), keepdims=bool(a.get("keepdims", 1)))]
        if op == "Cast":
            return [np.asarray(x[0]).astype({9: np.bool_, 7: np.int64, 1: np.float64, 11: np.float64}[a["to"]])]
        unary = {"Sqrt": np.sqrt, "Log": np.log, "Neg": np.negative, "Relu": lambda v: np.maximum(v, 0.0),
                 "Sigmoid": lambda v: 1.0 / (1.0 + np.exp(-v)), "Identity": lambda v: v}
        if op in unary:
            return [unary[op](x[0])]
        binary = {"Pow": np.power, "Mul": np.multiply, "Add": np.add, "Equal": np.equal}
        if op in binary:
            return [binary[op](x[0], x[1])]
        raise NotImplementedError(f"ONNX op {op} is not interpreted")


def speech_probs(graph: Graph, audio: np.ndarray, sr: int = 16000, window: int = 512,
                 keep: Sequence[str] = ()) -> Tuple[np.ndarray, List[Dict[str, np.ndarray]]]:
    """Per-window speech probabilities of ``audio`` (float64 [N]), plus the tensors named in ``keep`` for each window."""
    it = Interpreter(graph)
    audio = np.asarray(audio, np.float32)
    h = np.zeros((2, 1, 64))
    c = np.zeros((2, 1, 64))
    probs, kept = [], []
    for s in range(0, len(audio), window):
        chunk = audio[s:s + window]
        if len(chunk) < window:
            chunk = np.pad(chunk, (0, window - len(chunk)))
        trace = {} if keep else None
        out, h, c = it.run({"input": chunk[None].astype(np.float64), "sr": np.array(sr, np.int64), "h": h, "c": c}, trace)
        probs.append(float(np.asarray(out).reshape(-1)[0]))
        if keep:
            kept.append({k: trace[k] for k in keep})
    return np.array(probs), kept


# Name of the 16 kHz branch's LSTM input sequence [T, 1, 64], which the encoder kernel's test compares against.
LSTM_INPUT = "284"


def lstm_weights(graph: Graph):
    """The two 16 kHz LSTM layers' (W [256, 64], R [256, 64], Wb + Rb [256]) in ONNX gate order i, o, f, c, taken from
    the branch the graph runs when ``h`` is passed (the reference always passes it)."""
    top_if = next(n for n in graph.nodes if n.op == "If")
    g16 = top_if.attrs["then_branch"]
    inner = next(n for n in g16.nodes if n.op == "If" and any(m.op == "LSTM" for m in n.attrs["then_branch"].nodes))
    br = inner.attrs["then_branch"]
    out = []
    for n in (m for m in br.nodes if m.op == "LSTM"):
        W, R, B = (br.inits[k] for k in n.inputs[1:4])
        out.append((W[0], R[0], B[0, :256] + B[0, 256:]))
    return out


def lstm_f64(gx: np.ndarray, layers, steps_per_window: int, dec_w: np.ndarray, dec_b: float) -> np.ndarray:
    """float64 recurrence from given layer-1 input projections ``gx`` [S, 256] (ONNX gate order, bias included):
    layer-1 recurrence, layer 2, decoder, sigmoid, mean over each window's steps -> probs [S / steps_per_window]."""
    (_, R1, _), (W2, R2, b2) = layers
    sig = lambda v: 1.0 / (1.0 + np.exp(-v))
    h1 = c1 = h2 = c2 = np.zeros(64)
    p = np.empty(len(gx))
    for t in range(len(gx)):
        for layer in (1, 2):
            z = gx[t] + R1 @ h1 if layer == 1 else W2 @ h1 + R2 @ h2 + b2
            i, o, f, g = sig(z[:64]), sig(z[64:128]), sig(z[128:192]), np.tanh(z[192:])
            if layer == 1:
                c1 = f * c1 + i * g
                h1 = o * np.tanh(c1)
            else:
                c2 = f * c2 + i * g
                h2 = o * np.tanh(c2)
        p[t] = sig(dec_w @ np.maximum(h2, 0.0) + dec_b)
    return p.reshape(-1, steps_per_window).mean(axis=1)


# ---- model file recipe ---------------------------------------------------------------------------------------------
def fetch_model(reference_root: Optional[str] = None, dest: str = MODEL_PATH) -> Optional[str]:
    """Copy the reference's ``masr/infer_utils/silero_vad.onnx`` to ``oracle/_ref/`` (kept out of git) when the
    reference tree is present, after checking its sha256.  Returns the copied path, or None without a reference tree."""
    if reference_root is None:
        reference_root = os.environ.get("MASR_REFERENCE_ROOT", "/root/reference")
    src = os.path.join(reference_root, "masr", "infer_utils", "silero_vad.onnx")
    if not os.path.exists(src):
        return dest if os.path.exists(dest) else None
    with open(src, "rb") as fh:
        b = fh.read()
    digest = hashlib.sha256(b).hexdigest()
    if digest != MODEL_SHA256:
        raise RuntimeError(f"{src}: sha256 {digest} is not the recorded silero VAD model ({MODEL_SHA256})")
    os.makedirs(os.path.dirname(dest), exist_ok=True)
    if not os.path.exists(dest) or open(dest, "rb").read() != b:
        tmp = dest + ".tmp"
        with open(tmp, "wb") as fh:
            fh.write(b)
        os.replace(tmp, dest)
    return dest
