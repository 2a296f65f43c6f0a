"""Float64 references of the Silero VAD v6 network (faster_whisper_b200/silero.py states the graph).

* ``probs(weights, audio)``: the network restated in NumPy from the weight dict ``silero.load_weights`` returns, window
  preparation included (``SileroVADModel.__call__``'s context and last-window tail quirk).  The GPU kernels are pinned to it.
* ``run_graph(graph, x, h, c)``: a second, independent reading — a generic executor of the stored ONNX graph node by node,
  for the 13 op types it uses, following the ONNX operator definitions (Pad, Conv, Slice, LSTM with gates i,o,f,c and
  B = [Wb, Rb], ...).  A CPU test pins ``probs`` to it.  Neither is pinned against onnxruntime, which is not available here.
* ``synthetic_weights(seed)``: Silero-shaped weights whose probabilities spread over (0, 1), for tests without the asset.
"""

from __future__ import annotations

from typing import Dict, Tuple

import numpy as np

WINDOW, CONTEXT = 512, 64


def windows(audio: np.ndarray) -> np.ndarray:
    """[N, 576] float64 network inputs of a padded signal, exactly as SileroVADModel builds them: every window after the last
    64 samples of the previous one (zeros before the first), and the last window's own final 64 samples zeroed."""
    assert audio.ndim == 1 and audio.shape[0] % WINDOW == 0 and audio.shape[0] > 0
    frames = np.asarray(audio, np.float32).astype(np.float64).reshape(-1, WINDOW).copy()
    frames[-1, -CONTEXT:] = 0
    ctx = np.concatenate([np.zeros((1, CONTEXT)), frames[:-1, -CONTEXT:]], axis=0)
    return np.concatenate([ctx, frames], axis=1)


def _sigmoid(x):
    return 1.0 / (1.0 + np.exp(-x))


def _conv3(x: np.ndarray, w: np.ndarray, b: np.ndarray, stride: int) -> np.ndarray:
    """x [N, cin, L], w [cout, cin, 3], pad 1 -> relu(conv) [N, cout, L_out]"""
    L = x.shape[2]
    xp = np.pad(x, ((0, 0), (0, 0), (1, 1)))
    lout = (L + 2 - 3) // stride + 1
    y = np.zeros((x.shape[0], w.shape[0], lout))
    for t in range(lout):
        y[:, :, t] = np.tensordot(xp[:, :, t * stride : t * stride + 3], w, axes=([1, 2], [1, 2]))
    return np.maximum(y + b[None, :, None], 0.0)


def features(weights: Dict[str, np.ndarray], x: np.ndarray) -> np.ndarray:
    """[N, 576] window inputs -> [N, 128] LSTM inputs (STFT magnitude of frames 1..4 and the four conv + ReLU layers)."""
    W = {k: np.asarray(v, np.float64) for k, v in weights.items()}
    xp = np.pad(x, ((0, 0), (128, 128)), mode="reflect")                     # [N, 832]
    frames = np.stack([xp[:, 128 * f : 128 * f + 256] for f in range(1, 5)], axis=1)  # frame 0 is dropped
    spec = frames @ W["basis"].T                                             # [N, 4, 258]
    mag = np.sqrt(spec[:, :, :129] ** 2 + spec[:, :, 129:] ** 2).transpose(0, 2, 1)  # [N, 129, 4]
    a = mag
    for i, stride in enumerate((1, 2, 2, 1)):
        a = _conv3(a, W[f"conv{i}.weight"], W[f"conv{i}.bias"], stride)
    return a[:, :, 0]


def probs(weights: Dict[str, np.ndarray], audio: np.ndarray, h=None, c=None, return_state: bool = False):
    """One speech probability per 512-sample window of ``audio`` (length a positive multiple of 512), float64."""
    W = {k: np.asarray(v, np.float64) for k, v in weights.items()}
    gx = features(weights, windows(audio)) @ W["lstm.w_ih"].T + W["lstm.bias"]  # [N, 512], gate blocks i, o, f, c
    h = np.zeros(128) if h is None else np.asarray(h, np.float64).copy()
    c = np.zeros(128) if c is None else np.asarray(c, np.float64).copy()
    H = np.empty((gx.shape[0], 128))
    R = W["lstm.w_hh"]
    for n in range(gx.shape[0]):
        g = gx[n] + R @ h
        i, o, f, cc = _sigmoid(g[:128]), _sigmoid(g[128:256]), _sigmoid(g[256:384]), np.tanh(g[384:])
        c = f * c + i * cc
        h = o * np.tanh(c)
        H[n] = h
    p = _sigmoid(np.maximum(H, 0.0) @ W["decoder.weight"] + W["decoder.bias"][0])
    return (p, h, c) if return_state else p


# ---- generic executor of the stored graph -----------------------------------------------------------------------------


def _conv_nd1(x, w, b, attrs):
    """ONNX Conv for 1-D spatial input: x [N, C, L], w [M, C/group, k]."""
    assert attrs.get("group", 1) == 1 and attrs.get("dilations", [1]) == [1]
    k = w.shape[2]
    assert attrs.get("kernel_shape", [k]) == [k]
    s = attrs.get("strides", [1])[0]
    p0, p1 = attrs.get("pads", [0, 0])
    xp = np.pad(x, ((0, 0), (0, 0), (p0, p1)))
    lout = (xp.shape[2] - k) // s + 1
    cols = np.stack([xp[:, :, t * s : t * s + k] for t in range(lout)], axis=2)  # [N, C, lout, k]
    y = np.tensordot(cols, w, axes=([1, 3], [1, 2])).transpose(0, 2, 1)
    return y + (b[None, :, None] if b is not None else 0.0)


def _slice(x, starts, ends, axes, steps):
    idx = [slice(None)] * x.ndim
    for s, e, a, st in zip(starts, ends, axes, steps):
        d = x.shape[a]
        s = max(0, min(d, s + d if s < 0 else s))
        e = max(0, min(d, e + d if e < 0 else e))
        idx[a] = slice(s, e, st)
    return x[tuple(idx)]


def _lstm(X, Wt, Rt, Bt, h0, c0, attrs):
    """ONNX LSTM, forward, default activations: X [T, B, I], W [1, 4H, I], R [1, 4H, H], B [1, 8H]; gates i, o, f, c."""
    assert attrs.get("direction", "forward") == "forward" and attrs.get("layout", 0) == 0
    Hs = attrs["hidden_size"]
    W, R = Wt[0], Rt[0]
    Wb, Rb = Bt[0, : 4 * Hs], Bt[0, 4 * Hs :]
    h, c = h0[0], c0[0]
    Y = np.empty((X.shape[0], 1, X.shape[1], Hs))
    for t in range(X.shape[0]):
        g = X[t] @ W.T + h @ R.T + Wb + Rb
        i, o, f, cc = (g[:, k * Hs : (k + 1) * Hs] for k in range(4))
        i, o, f, cc = _sigmoid(i), _sigmoid(o), _sigmoid(f), np.tanh(cc)
        c = f * c + i * cc
        h = o * np.tanh(c)
        Y[t, 0] = h
    return Y, h[None], c[None]


def run_graph(graph, x: np.ndarray, h: np.ndarray, c: np.ndarray) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """Executes ``graph`` (silero.read_graph) in float64 on inputs x [N, 576], h, c [1, 1, 128]: (speech_probs, hn, cn)."""
    env = {k: (v.astype(np.float64) if v.dtype == np.float32 else v) for k, v in graph.initializers.items()}
    env.update(input=np.asarray(x, np.float64), h=np.asarray(h, np.float64), c=np.asarray(c, np.float64))
    for n in graph.nodes:
        a = [env[i] if i else None for i in n.inputs]
        at = n.attrs
        if n.op == "Pad":
            pads = a[1].tolist()
            r = len(pads) // 2
            mode = {"reflect": "reflect", "constant": "constant", "edge": "edge"}[at.get("mode", "constant")]
            out = [np.pad(a[0], list(zip(pads[:r], pads[r:])), mode=mode)]
        elif n.op == "Unsqueeze":
            out = [np.expand_dims(a[0], tuple(a[1].tolist()))]
        elif n.op == "Squeeze":
            out = [np.squeeze(a[0], tuple(a[1].tolist()))]
        elif n.op == "Conv":
            out = [_conv_nd1(a[0], a[1], a[2] if len(a) > 2 else None, at)]
        elif n.op == "Slice":
            steps = a[4].tolist() if len(a) > 4 and a[4] is not None else [1] * len(a[1])
            out = [_slice(a[0], a[1].tolist(), a[2].tolist(), a[3].tolist(), steps)]
        elif n.op == "Pow":
            out = [np.power(a[0], a[1])]
        elif n.op == "Add":
            out = [a[0] + a[1]]
        elif n.op == "Sqrt":
            out = [np.sqrt(a[0])]
        elif n.op == "Relu":
            out = [np.maximum(a[0], 0.0)]
        elif n.op == "Sigmoid":
            out = [_sigmoid(a[0])]
        elif n.op == "Transpose":
            out = [np.transpose(a[0], at["perm"])]
        elif n.op == "Reshape":
            out = [a[0].reshape(a[1].tolist())]
        elif n.op == "LSTM":
            out = list(_lstm(a[0], a[1], a[2], a[3], a[5], a[6], at))
        else:
            raise NotImplementedError(n.op)
        for name, v in zip(n.outputs, out):
            env[name] = v
    return env["speech_probs"], env["hn"], env["cn"]


def graph_probs(graph, audio: np.ndarray) -> np.ndarray:
    """The graph executor driven as SileroVADModel drives the ONNX session (blocks of 10000 windows, state carried)."""
    x = windows(audio)
    h = c = np.zeros((1, 1, 128))
    outs = []
    for lo in range(0, x.shape[0], 10000):
        p, h, c = run_graph(graph, x[lo : lo + 10000], h, c)
        outs.append(p)
    return np.concatenate(outs)


def synthetic_weights(seed: int) -> Dict[str, np.ndarray]:
    """Silero-shaped float32 weights: a Hann-windowed DFT basis and random layers scaled so activations stay O(1) and the
    probabilities spread over (0, 1) on speech-like and noise input."""
    rng = np.random.default_rng(seed)
    k = np.arange(256)
    win = 0.5 - 0.5 * np.cos(2 * np.pi * k / 256)
    f = np.arange(129)[:, None]
    basis = np.concatenate([np.cos(2 * np.pi * f * k / 256) * win, -np.sin(2 * np.pi * f * k / 256) * win]).astype(np.float32)
    w = {"basis": basis}
    scale_in = 2.0  # keeps conv0's output O(1) on the magnitude spectrum of 0.1-level audio
    for i, (cin, cout) in enumerate(((129, 128), (128, 64), (64, 64), (64, 128))):
        w[f"conv{i}.weight"] = (rng.standard_normal((cout, cin, 3)) * np.sqrt(2.0 / (3 * cin)) / (scale_in if i == 0 else 1)).astype(np.float32)
        w[f"conv{i}.bias"] = (0.1 * rng.standard_normal(cout)).astype(np.float32)
    w["lstm.w_ih"] = (rng.standard_normal((512, 128)) * 4.0 / np.sqrt(128)).astype(np.float32)
    w["lstm.w_hh"] = (rng.standard_normal((512, 128)) * 1.0 / np.sqrt(128)).astype(np.float32)
    w["lstm.bias"] = (0.2 * rng.standard_normal(512)).astype(np.float32)
    w["decoder.weight"] = (rng.standard_normal(128) * 12.0 / np.sqrt(128)).astype(np.float32)
    w["decoder.bias"] = np.zeros(1, np.float32)
    return w


# ---- a Silero-v6-shaped ONNX file from a weight dict ------------------------------------------------------------------
# The same 25 nodes, attributes, initializer names and field order as the v6 asset, so the reader, its structure check and the
# GPU path can be tested without the asset.  Protobuf wire format written by hand (no onnx package).


def _pb_varint(n: int) -> bytes:
    n &= (1 << 64) - 1
    out = bytearray()
    while True:
        b, n = n & 0x7F, n >> 7
        out.append(b | (0x80 if n else 0))
        if not n:
            return bytes(out)


def _pb_int(field: int, n: int) -> bytes:
    return _pb_varint(field << 3) + _pb_varint(n)


def _pb_bytes(field: int, data) -> bytes:
    data = data.encode() if isinstance(data, str) else bytes(data)
    return _pb_varint((field << 3) | 2) + _pb_varint(len(data)) + data


def _pb_tensor(name: str, arr: np.ndarray) -> bytes:
    dtype = 1 if arr.dtype == np.float32 else 7
    raw = np.ascontiguousarray(arr, "<f4" if dtype == 1 else "<i8").tobytes()
    return b"".join(_pb_int(1, d) for d in arr.shape) + _pb_int(2, dtype) + _pb_bytes(8, name) + _pb_bytes(9, raw)


def _pb_attr(name: str, value) -> bytes:
    if isinstance(value, str):
        return _pb_bytes(1, name) + _pb_bytes(4, value) + _pb_int(20, 3)
    if isinstance(value, int):
        return _pb_bytes(1, name) + _pb_int(3, value) + _pb_int(20, 2)
    return _pb_bytes(1, name) + b"".join(_pb_int(8, v) for v in value) + _pb_int(20, 7)


def _pb_node(name: str, op: str, inputs, outputs, attrs=()) -> bytes:
    return (b"".join(_pb_bytes(1, i) for i in inputs) + b"".join(_pb_bytes(2, o) for o in outputs) + _pb_bytes(3, name) +
            _pb_bytes(4, op) + b"".join(_pb_bytes(5, _pb_attr(k, v)) for k, v in attrs))


def write_onnx(weights: Dict[str, np.ndarray], path: str, seed: int = 0) -> None:
    """Writes ``weights`` (the dict ``silero.load_weights`` returns) as a Silero VAD v6 ONNX graph.  The LSTM bias is stored as
    B = [Wb, Rb] with a seeded split of ``lstm.bias`` between the two halves."""
    rng = np.random.default_rng(seed)
    rb = (0.1 * rng.standard_normal(512)).astype(np.float32)
    i64 = lambda v: np.array(v, np.int64)  # noqa: E731
    big = 2**63 - 1
    inits = [
        ("encoder.feature_extractor.forward_basis_buffer", weights["basis"].reshape(258, 1, 256)),
        *[(f"encoder.conv_layers.{i}.{p}", weights[f"conv{i}.{p}"]) for i in range(4) for p in ("weight", "bias")],
        ("decoder.conv1d.weight", weights["decoder.weight"].reshape(1, 128, 1)), ("decoder.conv1d.bias", weights["decoder.bias"]),
        ("onnx::LSTM_209", weights["lstm.w_ih"][None]), ("onnx::LSTM_210", weights["lstm.w_hh"][None]),
        ("onnx::LSTM_211", np.concatenate([weights["lstm.bias"] - rb, rb])[None]),
        ("shape_m1", i64([-1])), ("axes_1", i64([1])), ("two", np.array(2.0, np.float32)), ("pads", i64([0, 128, 0, 128])),
        ("re_starts", i64([0, 1])), ("re_ends", i64([129, big])), ("slice_axes", i64([1, 2])), ("slice_steps", i64([1, 1])),
        ("im_starts", i64([129, 1])), ("im_ends", i64([big, big])),
    ]
    conv = lambda k, s, p: [("dilations", [1]), ("group", 1), ("kernel_shape", [k]), ("pads", [p, p]), ("strides", [s])]  # noqa: E731
    fe = "/encoder/feature_extractor/"
    nodes = [
        _pb_node(fe + "padding/Pad", "Pad", ["input", "pads"], ["pad"], [("mode", "reflect")]),
        _pb_node(fe + "Unsqueeze", "Unsqueeze", ["pad", "axes_1"], ["unsq"]),
        _pb_node(fe + "Conv", "Conv", ["unsq", "encoder.feature_extractor.forward_basis_buffer"], ["stft"], conv(256, 128, 0)),
        _pb_node(fe + "Slice", "Slice", ["stft", "re_starts", "re_ends", "slice_axes", "slice_steps"], ["re"]),
        _pb_node(fe + "Slice_1", "Slice", ["stft", "im_starts", "im_ends", "slice_axes", "slice_steps"], ["im"]),
        _pb_node(fe + "Pow", "Pow", ["re", "two"], ["re2"]),
        _pb_node(fe + "Pow_1", "Pow", ["im", "two"], ["im2"]),
        _pb_node(fe + "Add", "Add", ["re2", "im2"], ["power"]),
        _pb_node(fe + "Sqrt", "Sqrt", ["power"], ["mag"]),
    ]
    x = "mag"
    for i, stride in enumerate((1, 2, 2, 1)):
        relu = "/encoder/relu" + ("" if i == 0 else f"_{i}") + "/Relu"
        nodes += [_pb_node(f"/encoder/conv_layers.{i}/Conv", "Conv", [x, f"encoder.conv_layers.{i}.weight", f"encoder.conv_layers.{i}.bias"],
                           [f"conv{i}"], conv(3, stride, 1)),
                  _pb_node(relu, "Relu", [f"conv{i}"], [f"relu{i}"])]
        x = f"relu{i}"
    nodes += [
        _pb_node("/Transpose", "Transpose", [x], ["seq"], [("perm", [0, 2, 1])]),
        _pb_node("/decoder/rnn/LSTM", "LSTM", ["seq", "onnx::LSTM_209", "onnx::LSTM_210", "onnx::LSTM_211", "", "h", "c"],
                 ["Y", "hn", "cn"], [("hidden_size", 128)]),
        _pb_node("/decoder/rnn/Squeeze", "Squeeze", ["Y", "axes_1"], ["Ysq"]),
        _pb_node("/decoder/relu/Relu", "Relu", ["Ysq"], ["Yr"]),
        _pb_node("/decoder/Transpose", "Transpose", ["Yr"], ["Yt"], [("perm", [1, 2, 0])]),
        _pb_node("/decoder/conv1d/Conv", "Conv", ["Yt", "decoder.conv1d.weight", "decoder.conv1d.bias"], ["logit"], conv(1, 1, 0)),
        _pb_node("/decoder/sigmoid/Sigmoid", "Sigmoid", ["logit"], ["sig"]),
        _pb_node("/Reshape", "Reshape", ["sig", "shape_m1"], ["speech_probs"]),
    ]
    graph = (b"".join(_pb_bytes(1, n) for n in nodes) + _pb_bytes(2, "main_graph") +
             b"".join(_pb_bytes(5, _pb_tensor(name, np.asarray(a))) for name, a in inits) +
             b"".join(_pb_bytes(11, _pb_bytes(1, n)) for n in ("input", "h", "c")) +
             b"".join(_pb_bytes(12, _pb_bytes(1, n)) for n in ("speech_probs", "hn", "cn")))
    model = _pb_int(1, 8) + _pb_bytes(2, "silero_oracle") + _pb_bytes(7, graph) + _pb_bytes(8, _pb_bytes(1, "") + _pb_int(2, 18))
    with open(path, "wb") as f:
        f.write(model)
