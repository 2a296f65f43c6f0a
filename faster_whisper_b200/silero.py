"""Silero VAD v6 (16 kHz) weights straight from its ONNX file, without onnx, onnxruntime or google.protobuf.

``read_graph(path)`` decodes the protobuf wire format of ModelProto -> GraphProto into nodes (op type, inputs, outputs,
attributes) and float32/int64 initializers.  ``load_weights(path)`` checks that graph against the one network the GPU
kernels implement (csrc/vad.cu) and returns its weights; any other graph — another Silero version, the 8 kHz branch, a
re-export with different padding or strides — raises ``ValueError`` naming the first node that differs, so it is refused
rather than run wrongly.  A truncated or non-ONNX file raises ``ValueError`` as well.

The network, as the graph states it (input ``[N, 576]``: each 512-sample window after the previous window's last 64):

  Pad(reflect, 128 | 128) -> Unsqueeze(1) -> Conv(basis [258, 1, 256], stride 128): 5 frames
  -> Slice rows 0..128 / 129..257 of frames 1..4 (frame 0 dropped) -> sqrt(re^2 + im^2): [N, 129, 4]
  -> 4 x (Conv k3 pad 1 + Relu): 129->128 s1, 128->64 s2, 64->64 s2, 64->128 s1: [N, 128, 1]
  -> Transpose(0, 2, 1) -> LSTM(hidden 128, forward, gates i,o,f,c) over the N windows as one sequence of batch 1,
     state h, c [1, 1, 128] in and out -> Squeeze(1) -> Relu -> Transpose(1, 2, 0) -> Conv 1x1 128->1 -> Sigmoid -> Reshape(-1)
"""

from __future__ import annotations

import struct
from dataclasses import dataclass, field
from typing import Dict, List, Tuple

import numpy as np

INT64_MAX = 2**63 - 1

# ---- protobuf wire format -------------------------------------------------------------------------------------------


def _varint(b: bytes, i: int) -> Tuple[int, int]:
    r = s = 0
    while True:
        if i >= len(b) or s > 63:
            raise ValueError("not an ONNX file: truncated or malformed varint")
        x = b[i]
        i += 1
        r |= (x & 0x7F) << s
        s += 7
        if x < 0x80:
            return r, i


def _fields(b: bytes) -> List[Tuple[int, int, object]]:
    """(field number, wire type, value) of one message; value is an int (varint), or bytes (fixed32/64, length-delimited)."""
    out, i = [], 0
    while i < len(b):
        key, i = _varint(b, i)
        f, w = key >> 3, key & 7
        if f == 0:
            raise ValueError("not an ONNX file: field number 0")
        if w == 0:
            v, i = _varint(b, i)
        elif w in (1, 5):
            n = 8 if w == 1 else 4
            v, i = b[i : i + n], i + n
        elif w == 2:
            n, i = _varint(b, i)
            v, i = b[i : i + n], i + n
        else:
            raise ValueError(f"not an ONNX file: wire type {w}")
        if i > len(b):
            raise ValueError("not an ONNX file: truncated message")
        out.append((f, w, v))
    return out


def _ints(fields, num) -> List[int]:
    """A repeated int64 field, packed or not (two's complement for negatives)."""
    out = []
    for f, w, v in fields:
        if f != num:
            continue
        if w == 0:
            out.append(v)
        elif w == 2:
            i = 0
            while i < len(v):
                x, i = _varint(v, i)
                out.append(x)
        else:
            raise ValueError("not an ONNX file: bad repeated int")
    return [x - (1 << 64) if x >= 1 << 63 else x for x in out]


def _str(fields, num) -> List[str]:
    return [v.decode("utf-8", "replace") for f, w, v in fields if f == num and w == 2]


# ---- ONNX messages ----------------------------------------------------------------------------------------------------
_FLOAT, _INT64 = 1, 7  # TensorProto.DataType


@dataclass
class Node:
    name: str
    op: str
    inputs: List[str]
    outputs: List[str]
    attrs: Dict[str, object] = field(default_factory=dict)


@dataclass
class Graph:
    nodes: List[Node]
    initializers: Dict[str, np.ndarray]
    inputs: List[str]
    outputs: List[str]


def _tensor(b: bytes) -> Tuple[str, np.ndarray]:
    fs = _fields(b)
    dims = _ints(fs, 1)
    dtype = _ints(fs, 2)
    name = (_str(fs, 8) or [""])[0]
    raw = [v for f, w, v in fs if f == 9 and w == 2]
    if not dtype or dtype[0] not in (_FLOAT, _INT64):
        raise ValueError(f"initializer {name!r}: unsupported data type {dtype}")
    dt = np.dtype("<f4") if dtype[0] == _FLOAT else np.dtype("<i8")
    if raw:
        data = raw[0]
    elif dtype[0] == _FLOAT:  # float_data: packed, or one fixed32 per entry
        data = b"".join(v for f, w, v in fs if f == 4)
    else:
        data = np.array(_ints(fs, 7), "<i8").tobytes()
    n = int(np.prod(dims)) if dims else 1
    if len(data) != n * dt.itemsize:
        raise ValueError(f"initializer {name!r}: {len(data)} bytes for shape {dims}")
    return name, np.frombuffer(data, dt).reshape(dims).copy()


def _attr(b: bytes) -> Tuple[str, object]:
    fs = _fields(b)
    name = (_str(fs, 1) or [""])[0]
    kind = (_ints(fs, 20) or [0])[0]
    if kind == 1:  # FLOAT
        return name, struct.unpack("<f", [v for f, w, v in fs if f == 2][0])[0]
    if kind == 2:  # INT
        return name, _ints(fs, 3)[0]
    if kind == 3:  # STRING
        return name, [v for f, w, v in fs if f == 4][0].decode()
    if kind == 7:  # INTS
        return name, _ints(fs, 8)
    if kind == 8:  # STRINGS
        return name, _str(fs, 9)
    if kind == 6:  # FLOATS
        vals = [v for f, w, v in fs if f == 7]
        return name, [x for v in vals for x in struct.unpack("<%df" % (len(v) // 4), v)]
    return name, ("unsupported attribute type", kind)


def read_graph(path: str) -> Graph:
    """The main graph of an ONNX file: nodes in order, initializers as arrays, graph input and output names."""
    with open(path, "rb") as f:
        data = f.read()
    model = _fields(data)
    graphs = [v for f, w, v in model if f == 7 and w == 2]
    if len(graphs) != 1 or not any(f == 1 and w == 0 for f, w, _ in model):
        raise ValueError(f"{path}: not an ONNX model (no ir_version or graph)")
    g = _fields(graphs[0])
    nodes = []
    for f, w, v in g:
        if f == 1 and w == 2:
            nf = _fields(v)
            nodes.append(Node(name=(_str(nf, 3) or [""])[0], op=(_str(nf, 4) or [""])[0], inputs=_str(nf, 1), outputs=_str(nf, 2),
                              attrs=dict(_attr(a) for ff, ww, a in nf if ff == 5 and ww == 2)))
    inits = dict(_tensor(v) for f, w, v in g if f == 5 and w == 2)
    names = lambda num: [(_str(_fields(v), 1) or [""])[0] for f, w, v in g if f == num and w == 2]  # ValueInfoProto.name
    return Graph(nodes=nodes, initializers=inits, inputs=names(11), outputs=names(12))


# ---- the one graph the kernels implement ------------------------------------------------------------------------------
_CONVS = [(129, 128, 1), (128, 64, 2), (64, 64, 2), (64, 128, 1)]  # (in, out, stride), kernel 3, pad 1
_OPS = (["Pad", "Unsqueeze", "Conv", "Slice", "Slice", "Pow", "Pow", "Add", "Sqrt"] + ["Conv", "Relu"] * 4 +
        ["Transpose", "LSTM", "Squeeze", "Relu", "Transpose", "Conv", "Sigmoid", "Reshape"])
# each node's data inputs: a name, or k for "the first output of node k"
_DATA_IN = {0: ["input"], 1: [0], 2: [1], 3: [2], 4: [2], 5: [3], 6: [4], 7: [5, 6], 8: [7], 9: [8], 10: [9], 11: [10], 12: [11],
            13: [12], 14: [13], 15: [14], 16: [15], 17: [16], 18: [17], 19: [18], 20: [19], 21: [20], 22: [21], 23: [22], 24: [23]}


def load_weights(path: str) -> Dict[str, np.ndarray]:
    """Checks the graph in ``path`` and returns its weights as float32 arrays:

    ``basis [258, 256]`` (STFT rows: 129 real then 129 imaginary), ``conv{0..3}.weight [out, in, 3]`` and ``.bias [out]``,
    ``lstm.w_ih [512, 128]``, ``lstm.w_hh [512, 128]`` and ``lstm.bias [512]`` (= b_ih + b_hh; gate blocks i, o, f, c in ONNX
    order), ``decoder.weight [128]``, ``decoder.bias [1]``."""
    g = read_graph(path)
    return check_graph(g)


def check_graph(g: Graph) -> Dict[str, np.ndarray]:
    init = g.initializers

    def node_err(k: int, what: str):
        n = g.nodes[k] if k < len(g.nodes) else None
        label = f"node {k} ({n.op} {n.name or n.outputs[:1]})" if n else f"node {k}"
        return ValueError(f"unsupported Silero VAD graph: {label}: {what}")

    def const(k: int, slot: int, what: str) -> np.ndarray:
        n = g.nodes[k]
        if slot >= len(n.inputs) or n.inputs[slot] not in init:
            raise node_err(k, f"{what} is not an initializer")
        return init[n.inputs[slot]]

    def expect_const(k: int, slot: int, what: str, want):
        got = const(k, slot, what).tolist()
        if got != (list(want) if isinstance(want, (list, tuple)) else want):
            raise node_err(k, f"{what} is {got}, expected {want}")

    def weight(k: int, slot: int, what: str, shape) -> np.ndarray:
        w = const(k, slot, what)
        if w.dtype != np.float32 or tuple(w.shape) != tuple(shape):
            raise node_err(k, f"{what} has shape {tuple(w.shape)} {w.dtype}, expected {tuple(shape)} float32")
        return w

    def expect_attr(k: int, name: str, want, default=None):
        got = g.nodes[k].attrs.get(name, default)
        if got != want:
            raise node_err(k, f"attribute {name} is {got!r}, expected {want!r}")

    def conv(k: int, kernel: int, stride: int, pad: int):
        extra = set(g.nodes[k].attrs) - {"kernel_shape", "strides", "pads", "group", "dilations"}
        if extra:
            raise node_err(k, f"unexpected attributes {sorted(extra)}")
        expect_attr(k, "kernel_shape", [kernel])
        expect_attr(k, "strides", [stride], [1])
        expect_attr(k, "pads", [pad, pad], [0, 0])
        expect_attr(k, "group", 1, 1)
        expect_attr(k, "dilations", [1], [1])

    if [n.op for n in g.nodes] != _OPS:
        ops = [n.op for n in g.nodes]
        k = next((i for i, (a, b) in enumerate(zip(ops, _OPS)) if a != b), min(len(ops), len(_OPS)))
        raise node_err(k, f"op sequence {ops[k:k + 3]} where {_OPS[k:k + 3]} was expected ({len(ops)} nodes, expected {len(_OPS)})")
    if g.inputs[:3] != ["input", "h", "c"] or g.outputs[:3] != ["speech_probs", "hn", "cn"]:
        raise ValueError(f"unsupported Silero VAD graph: inputs {g.inputs}, outputs {g.outputs}")
    for k, srcs in _DATA_IN.items():
        for slot, s in enumerate(srcs):
            want = s if isinstance(s, str) else g.nodes[s].outputs[0]
            if g.nodes[k].inputs[slot] != want:
                raise node_err(k, f"input {slot} is {g.nodes[k].inputs[slot]!r}, expected {want!r}")

    expect_attr(0, "mode", "reflect", "constant")
    expect_const(0, 1, "pads", [0, 128, 0, 128])
    if len(g.nodes[0].inputs) > 2 and g.nodes[0].inputs[2]:
        raise node_err(0, "unexpected constant value or axes")
    expect_const(1, 1, "axes", [1])
    conv(2, 256, 128, 0)
    basis = weight(2, 1, "STFT basis", (258, 1, 256))
    if len(g.nodes[2].inputs) > 2 and g.nodes[2].inputs[2]:
        raise node_err(2, "unexpected bias")
    for k, starts, ends in ((3, [0, 1], [129, INT64_MAX]), (4, [129, 1], [INT64_MAX, INT64_MAX])):
        expect_const(k, 1, "starts", starts)
        expect_const(k, 2, "ends", ends)
        expect_const(k, 3, "axes", [1, 2])
        if len(g.nodes[k].inputs) > 4:
            expect_const(k, 4, "steps", [1, 1])
    for k in (5, 6):
        expect_const(k, 1, "exponent", 2.0)
    out = {"basis": basis.reshape(258, 256)}
    for i, (cin, cout, stride) in enumerate(_CONVS):
        k = 9 + 2 * i
        conv(k, 3, stride, 1)
        out[f"conv{i}.weight"] = weight(k, 1, f"conv{i} weight", (cout, cin, 3))
        out[f"conv{i}.bias"] = weight(k, 2, f"conv{i} bias", (cout,))
    expect_attr(17, "perm", [0, 2, 1])
    lstm = g.nodes[18]
    expect_attr(18, "hidden_size", 128)
    expect_attr(18, "direction", "forward", "forward")
    expect_attr(18, "activations", ["Sigmoid", "Tanh", "Tanh"], ["Sigmoid", "Tanh", "Tanh"])
    expect_attr(18, "input_forget", 0, 0)
    expect_attr(18, "layout", 0, 0)
    for a in ("clip", "activation_alpha", "activation_beta"):
        if a in lstm.attrs:
            raise node_err(18, f"unexpected attribute {a}")
    if (lstm.inputs + [""] * 8)[4:8] != ["", "h", "c", ""] or lstm.outputs[:3] != [g.nodes[19].inputs[0], "hn", "cn"]:
        raise node_err(18, f"inputs {lstm.inputs} / outputs {lstm.outputs}: expected (x, W, R, B, '', h, c) -> (Y, hn, cn)")
    w_ih = weight(18, 1, "W", (1, 512, 128))
    w_hh = weight(18, 2, "R", (1, 512, 128))
    b = weight(18, 3, "B", (1, 1024))
    out["lstm.w_ih"], out["lstm.w_hh"] = w_ih[0], w_hh[0]
    out["lstm.bias"] = b[0, :512] + b[0, 512:]
    expect_const(19, 1, "axes", [1])
    expect_attr(21, "perm", [1, 2, 0])
    conv(22, 1, 1, 0)
    out["decoder.weight"] = weight(22, 1, "decoder weight", (1, 128, 1)).reshape(128)
    out["decoder.bias"] = weight(22, 2, "decoder bias", (1,))
    expect_const(24, 1, "shape", [-1])
    if g.nodes[24].outputs[0] != "speech_probs":
        raise node_err(24, "does not produce speech_probs")
    return {k: np.ascontiguousarray(v, np.float32) for k, v in out.items()}


WEIGHT_SHAPES = {
    "basis": (258, 256),
    **{f"conv{i}.weight": (o, c, 3) for i, (c, o, _) in enumerate(_CONVS)},
    **{f"conv{i}.bias": (o,) for i, (_, o, _) in enumerate(_CONVS)},
    "lstm.w_ih": (512, 128), "lstm.w_hh": (512, 128), "lstm.bias": (512,),
    "decoder.weight": (128,), "decoder.bias": (1,),
}
