"""Minimal ONNX (protobuf wire format) reader/writer - just enough to ingest the reference's model files
without the ``onnx`` package (absent in this image; field numbers from onnx.proto3, SURVEY.md Appendix E).

Readers:
  * ``head_from_onnx``      - wake-word heads of the DNN family the reference trains/exports
                               (openwakeword/train.py:56-83,144-165, torch.onnx.export opset 13):
                               Flatten -> Gemm|MatMul+Add -> [LayerNorm] -> Relu -> ... -> Gemm -> Sigmoid | (Relu ->) Softmax.
                               LayerNorm may be the fused ``LayerNormalization`` op (opset >= 17) or the decomposed
                               ReduceMean/Sub/Pow/ReduceMean/Add/Sqrt/Div/Mul/Add chain (opset 13).
  * ``embedding_from_onnx`` - the speech-embedding CNN as 20 Conv + 19 BatchNormalization nodes in graph order
                               (best effort: the released file could not be inspected here).
Anything else raises ``ValueError`` - the CUDA kernels implement this family only, and nothing falls back to a CPU
interpreter.  The writer (``write_head_onnx`` / ``write_embedding_onnx``) exists so the tests can round-trip files
of the same structure.  Only float32 tensors (raw_data or float_data) and int64 attributes are handled.
"""
import struct

import numpy as np

from . import weights as _weights


# ------------------------------------------------------------------ wire format
def _varint(buf, i):
    r, s = 0, 0
    while True:
        b = buf[i]
        i += 1
        r |= (b & 0x7F) << s
        if not b & 0x80:
            return r, i
        s += 7


def _fields(buf):
    """Yield (field_number, wire_type, value) for one message; value is int or memoryview."""
    i, n = 0, len(buf)
    while i < n:
        key, i = _varint(buf, i)
        fn, wt = key >> 3, key & 7
        if wt == 0:
            v, i = _varint(buf, i)
        elif wt == 1:
            v = bytes(buf[i:i + 8]); i += 8
        elif wt == 2:
            ln, i = _varint(buf, i)
            v = buf[i:i + ln]; i += ln
        elif wt == 5:
            v = bytes(buf[i:i + 4]); i += 4
        else:
            raise ValueError(f"unsupported protobuf wire type {wt}")
        yield fn, wt, v


def _enc_varint(v):
    out = bytearray()
    v &= (1 << 64) - 1
    while True:
        b = v & 0x7F
        v >>= 7
        out.append(b | (0x80 if v else 0))
        if not v:
            return bytes(out)


def _ld(fn, payload):
    return _enc_varint((fn << 3) | 2) + _enc_varint(len(payload)) + payload


def _vi(fn, v):
    return _enc_varint(fn << 3) + _enc_varint(v)


# ------------------------------------------------------------------ parse
def _tensor(buf):
    dims, dtype, name, raw, floats, ints = [], 0, "", None, [], []
    for fn, wt, v in _fields(buf):
        if fn == 1:
            if wt == 0:
                dims.append(v)
            else:                                   # packed
                j = 0
                while j < len(v):
                    d, j = _varint(v, j); dims.append(d)
        elif fn == 2:
            dtype = v
        elif fn == 8:
            name = bytes(v).decode()
        elif fn == 9:
            raw = bytes(v)
        elif fn == 4:
            floats += list(struct.unpack(f"<{len(v) // 4}f", bytes(v))) if wt == 2 else [struct.unpack("<f", v)[0]]
        elif fn == 7:
            if wt == 0:
                ints.append(v)
            else:
                j = 0
                while j < len(v):
                    d, j = _varint(v, j); ints.append(d)
    if dtype == 1:
        a = np.frombuffer(raw, "<f4") if raw is not None else np.asarray(floats, np.float32)
    elif dtype == 7:
        a = np.frombuffer(raw, "<i8") if raw is not None else np.asarray(ints, np.int64)
    else:
        return name, None
    return name, a.reshape(dims).copy()


def _attr(buf):
    name, val = "", None
    for fn, wt, v in _fields(buf):
        if fn == 1:
            name = bytes(v).decode()
        elif fn == 2:
            val = struct.unpack("<f", v)[0]
        elif fn == 3:
            val = v if v < (1 << 63) else v - (1 << 64)
        elif fn == 8:
            if wt == 0:
                val = (val or []) + [v]
            else:
                j, lst = 0, []
                while j < len(v):
                    d, j = _varint(v, j); lst.append(d if d < (1 << 63) else d - (1 << 64))
                val = lst
        elif fn == 5:
            val = _tensor(v)[1]
    return name, val


def _value_info(buf):
    name, shape = "", []
    for fn, _, v in _fields(buf):
        if fn == 1:
            name = bytes(v).decode()
        elif fn == 2:
            for f2, _, t in _fields(v):
                if f2 == 1:                          # tensor_type
                    for f3, _, sh in _fields(t):
                        if f3 == 2:                  # shape
                            for f4, _, dim in _fields(sh):
                                if f4 == 1:
                                    dv = None
                                    for f5, _, x in _fields(dim):
                                        if f5 == 1:
                                            dv = x
                                    shape.append(dv)
    return name, shape


def parse_onnx(path):
    buf = memoryview(open(path, "rb").read())
    graph = None
    for fn, _, v in _fields(buf):
        if fn == 7:
            graph = v
    if graph is None:
        raise ValueError(f"{path}: no GraphProto found")
    nodes, inits, inputs, outputs = [], {}, [], []
    for fn, _, v in _fields(graph):
        if fn == 1:
            ins, outs, op, attrs = [], [], "", {}
            for f2, _, x in _fields(v):
                if f2 == 1:
                    ins.append(bytes(x).decode())
                elif f2 == 2:
                    outs.append(bytes(x).decode())
                elif f2 == 4:
                    op = bytes(x).decode()
                elif f2 == 5:
                    k, val = _attr(x)
                    attrs[k] = val
            nodes.append({"op": op, "in": ins, "out": outs, "attrs": attrs})
        elif fn == 5:
            name, arr = _tensor(v)
            inits[name] = arr
        elif fn == 11:
            inputs.append(_value_info(v))
        elif fn == 12:
            outputs.append(_value_info(v))
    for nd in nodes:                                  # Constant nodes act as initialisers
        if nd["op"] == "Constant" and "value" in nd["attrs"]:
            inits[nd["out"][0]] = nd["attrs"]["value"]
    inputs = [(n, s) for n, s in inputs if n not in inits]
    return {"nodes": nodes, "initializers": inits, "inputs": inputs, "outputs": outputs}


# ------------------------------------------------------------------ heads
_PASS = ("Identity", "Cast", "Reshape", "Flatten", "Squeeze", "Unsqueeze", "Dropout")


class _Graph:
    """Producer map + helpers to walk a head graph backwards from its output."""

    def __init__(self, path, g):
        self.path, self.init, self.nodes = path, g["initializers"], g["nodes"]
        self.prod = {}
        for nd in self.nodes:
            for o in nd["out"]:
                self.prod[o] = nd
        self.input = g["inputs"][0][0]

    def fail(self, msg):
        raise ValueError(f"{self.path}: {msg}")

    def const(self, name):
        return self.init.get(name)

    def producer(self, name):
        if name == self.input:
            return None
        if name not in self.prod:
            self.fail(f"tensor '{name}' has no producer")
        return self.prod[name]

    def data_inputs(self, nd):
        return [i for i in nd["in"] if i and self.const(i) is None]


def _walk_layernorm_decomposed(G, add_beta):
    """Add(beta) <- Mul(gamma) <- Div(c, sqrt(var+eps)) ; c = Sub(x, ReduceMean(x)).  Returns (x, gamma, beta)."""
    beta = next((G.const(i) for i in add_beta["in"] if G.const(i) is not None), None)
    mul = G.producer(G.data_inputs(add_beta)[0])
    if mul is None or mul["op"] != "Mul":
        return None
    gamma = next((G.const(i) for i in mul["in"] if G.const(i) is not None), None)
    div = G.producer(G.data_inputs(mul)[0]) if G.data_inputs(mul) else None
    if div is None or div["op"] != "Div" or gamma is None or beta is None or gamma.size < 2:
        return None
    sub = G.producer(div["in"][0])
    sq = G.producer(div["in"][1])
    if sub is None or sub["op"] != "Sub" or sq is None or sq["op"] != "Sqrt":
        G.fail("unrecognised LayerNorm decomposition")
    add_eps = G.producer(sq["in"][0])
    eps = next((G.const(i) for i in add_eps["in"] if G.const(i) is not None), None) if add_eps and add_eps["op"] == "Add" else None
    if eps is None or abs(float(np.asarray(eps).ravel()[0]) - 1e-5) > 1e-7:
        G.fail("LayerNorm epsilon must be 1e-5")
    rm = G.producer(sub["in"][1])
    if rm is None or rm["op"] != "ReduceMean" or rm["in"][0] != sub["in"][0]:
        G.fail("unrecognised LayerNorm decomposition (mean)")
    return sub["in"][0], gamma.astype(np.float32).ravel(), beta.astype(np.float32).ravel()


def _walk_branch(G, name):
    """Walk one DNN branch backwards from tensor `name` to the graph input, enforcing the op ORDER of the reference's
    family (train.py:56-83): Flatten, then (Linear [LayerNorm] Relu)*, Linear, then one of {nothing, Sigmoid, Relu,
    Softmax, Relu+Softmax}.  Returns a head dict."""
    ops = []                       # reversed list of ("linear", W, b) | ("ln", g, b) | ("relu",) | ("sigmoid",) | ("softmax",)
    cur = name
    while True:
        nd = G.producer(cur)
        if nd is None:
            break
        op = nd["op"]
        if op in _PASS:
            cur = G.data_inputs(nd)[0]
        elif op == "Relu":
            ops.append(("relu",)); cur = nd["in"][0]
        elif op == "Sigmoid":
            ops.append(("sigmoid",)); cur = nd["in"][0]
        elif op == "Softmax":
            ops.append(("softmax",)); cur = nd["in"][0]
        elif op == "Gemm":
            Wm = G.const(nd["in"][1])
            b = G.const(nd["in"][2]) if len(nd["in"]) > 2 else None
            if Wm is None:
                G.fail("Gemm without constant weights")
            if nd["attrs"].get("transA", 0):
                G.fail("Gemm transA not supported")
            if nd["attrs"].get("transB", 0):
                Wm = Wm.T
            if nd["attrs"].get("alpha", 1.0) != 1.0 or nd["attrs"].get("beta", 1.0) != 1.0:
                G.fail("Gemm alpha/beta != 1 not supported")
            ops.append(("linear", np.ascontiguousarray(Wm, np.float32),
                        np.zeros(Wm.shape[1], np.float32) if b is None else b.astype(np.float32).ravel()))
            cur = nd["in"][0]
        elif op == "Add":
            ln = _walk_layernorm_decomposed(G, nd)
            if ln is not None:
                cur = ln[0]; ops.append(("ln", ln[1], ln[2]))
                continue
            c = next((G.const(i) for i in nd["in"] if G.const(i) is not None), None)
            mm = G.producer(G.data_inputs(nd)[0]) if len(G.data_inputs(nd)) == 1 else None
            if c is None or mm is None or mm["op"] != "MatMul" or G.const(mm["in"][1]) is None:
                G.fail("Add that is neither a Linear bias nor a LayerNorm shift")
            Wm = G.const(mm["in"][1])
            ops.append(("linear", np.ascontiguousarray(Wm, np.float32), c.astype(np.float32).ravel()))
            cur = mm["in"][0]
        elif op == "MatMul":
            Wm = G.const(nd["in"][1])
            if Wm is None:
                G.fail("MatMul without constant weights")
            ops.append(("linear", np.ascontiguousarray(Wm, np.float32), np.zeros(Wm.shape[1], np.float32)))
            cur = nd["in"][0]
        elif op == "LayerNormalization":
            gm = G.const(nd["in"][1])
            bt = G.const(nd["in"][2]) if len(nd["in"]) > 2 else None
            if gm is None:
                G.fail("LayerNormalization without constant scale")
            if abs(nd["attrs"].get("epsilon", 1e-5) - 1e-5) > 1e-7:
                G.fail("LayerNorm epsilon must be 1e-5")
            ops.append(("ln", gm.astype(np.float32).ravel(),
                        np.zeros(gm.size, np.float32) if bt is None else bt.astype(np.float32).ravel()))
            cur = nd["in"][0]
        else:
            G.fail(f"op '{op}' is outside the DNN head family the b200 backend implements")
    ops.reverse()
    # ---- grammar check on the forward op sequence ----
    i, layers = 0, []
    while i < len(ops):
        if ops[i][0] != "linear":
            break
        lay = {"W": ops[i][1], "b": ops[i][2], "ln": None}
        i += 1
        if i < len(ops) and ops[i][0] == "ln" and i + 1 < len(ops) and ops[i + 1][0] == "relu" and \
                any(o[0] == "linear" for o in ops[i + 2:]):
            lay["ln"] = (ops[i][1], ops[i][2]); i += 2
        elif i < len(ops) and ops[i][0] == "relu" and any(o[0] == "linear" for o in ops[i + 1:]):
            i += 1
        layers.append(lay)
    tail = tuple(o[0] for o in ops[i:])
    finals = {(): "none", ("sigmoid",): "sigmoid", ("relu",): "relu", ("softmax",): "softmax", ("relu", "softmax"): "relu_softmax"}
    if not layers:
        G.fail("no Linear layers found")
    if tail not in finals:
        G.fail(f"op order {[o[0] for o in ops]} is not Linear [LayerNorm] Relu ... Linear (Sigmoid | Relu | [Relu] Softmax)")
    for a, b in zip(layers[:-1], layers[1:]):
        if a["W"].shape[1] != b["W"].shape[0]:
            G.fail("Linear layer shapes do not chain")
    for lay in layers[:-1]:
        if lay["ln"] is not None and lay["ln"][0].size != lay["W"].shape[1]:
            G.fail("LayerNorm width does not match its Linear layer")
    if any(l["ln"] is not None for l in layers[:-1]) and any(l["ln"] is None for l in layers[:-1]):
        G.fail("LayerNorm on only some hidden layers is not supported")
    return {"layers": layers, "final": finals[tail]}


def head_from_onnx(path):
    """-> head dict, or a gated pair {"main", "verifier", "threshold"} for graphs of the released hey_jarvis structure:
    two parallel DNN branches p1, p2 on the same input joined by  Where(Greater(p1, t), p2, p1)  (or the equivalent
    Where(LessOrEqual/Less(p1, t) | Not(Greater), p1, p2)): docs/models/hey_jarvis.md:9,38."""
    g = parse_onnx(path)
    if len(g["inputs"]) != 1:
        raise ValueError(f"{path}: expected one graph input, found {len(g['inputs'])}")
    shape = g["inputs"][0][1]
    if len(shape) != 3 or shape[2] != 96 or not shape[1]:
        raise ValueError(f"{path}: head input must be [batch, n_frames, 96], found {shape}")
    n_in = int(shape[1])
    if len(g["outputs"]) != 1:
        raise ValueError(f"{path}: expected one graph output, found {len(g['outputs'])}")
    G = _Graph(path, g)
    out = g["outputs"][0][0]
    nd = G.producer(out)
    while nd is not None and nd["op"] in _PASS:
        out = G.data_inputs(nd)[0]; nd = G.producer(out)

    def finish(h):
        if h["layers"][0]["W"].shape[0] != n_in * 96:
            raise ValueError(f"{path}: first Linear takes {h['layers'][0]['W'].shape[0]} inputs, expected {n_in * 96}")
        h["n_in"] = n_in
        return h

    if nd is not None and nd["op"] == "Where":
        cond = G.producer(nd["in"][0])
        neg = False
        while cond is not None and cond["op"] == "Not":
            neg = not neg; cond = G.producer(cond["in"][0])
        if cond is None or cond["op"] not in ("Greater", "GreaterOrEqual", "Less", "LessOrEqual"):
            G.fail("Where without a score comparison: not the conditional-verifier structure")
        thr = G.const(cond["in"][1])
        if thr is None:
            G.fail("the gate compares against a non-constant")
        p_cmp = cond["in"][0]
        greater = cond["op"] in ("Greater", "GreaterOrEqual")
        if neg:
            greater = not greater
        x_true, x_false = nd["in"][1], nd["in"][2]
        main_t, ver_t = (x_false, x_true) if greater else (x_true, x_false)
        if main_t != p_cmp:
            G.fail("the gate must compare the main network's own score")
        main, ver = finish(_walk_branch(G, main_t)), finish(_walk_branch(G, ver_t))
        for h in (main, ver):
            if h["layers"][-1]["W"].shape[1] != 1:
                G.fail("gated networks must be single-output")
        return {"main": main, "verifier": ver, "threshold": float(np.asarray(thr).ravel()[0]), "n_in": n_in}
    return finish(_walk_branch(G, out))


def embedding_from_onnx(path):
    g = parse_onnx(path)
    init = g["initializers"]
    convs = [nd for nd in g["nodes"] if nd["op"] == "Conv"]
    bns = [nd for nd in g["nodes"] if nd["op"] == "BatchNormalization"]
    if len(convs) != 20 or len(bns) != 19:
        raise ValueError(f"{path}: expected 20 Conv + 19 BatchNormalization nodes (unfolded speech-embedding graph), found "
                         f"{len(convs)} + {len(bns)}; convert the weights with openwakeword_b200.weights.save_embedding instead")
    conv, bn = [], []
    for li, nd in enumerate(convs):
        w = init.get(nd["in"][1])
        kh, kw, cin, cout, _, _ = _weights.EMBEDDING_LAYERS[li]
        if w is None or w.shape != (cout, cin, kh, kw):
            raise ValueError(f"{path}: Conv #{li} weight shape {None if w is None else w.shape} != {(cout, cin, kh, kw)}")
        if len(nd["in"]) > 2 and nd["in"][2] in init and np.any(init[nd["in"][2]] != 0):
            raise ValueError(f"{path}: Conv #{li} has a bias; the reference graph is bias-free")
        conv.append(np.ascontiguousarray(w.transpose(2, 3, 1, 0), np.float32))          # OIHW -> HWIO
    for li, nd in enumerate(bns):
        ps = [init.get(n) for n in nd["in"][1:5]]
        if any(p is None for p in ps):
            raise ValueError(f"{path}: BatchNormalization #{li} without constant parameters")
        eps = nd["attrs"].get("epsilon", 1e-5)
        if abs(eps - _weights.BN_EPS) > 1e-6:
            raise ValueError(f"{path}: BatchNormalization epsilon {eps} != {_weights.BN_EPS}")
        bn.append(tuple(p.astype(np.float32) for p in ps))
    return {"conv": conv, "bn": bn}


# ------------------------------------------------------------------ writer (tests)
def _tensor_proto(name, arr):
    arr = np.asarray(arr)
    dt = 1 if arr.dtype == np.float32 else 7
    out = b"".join(_vi(1, d) for d in arr.shape) + _vi(2, dt) + _ld(8, name.encode())
    return out + _ld(9, arr.astype("<f4" if dt == 1 else "<i8").tobytes())


def _node(op, ins, outs, **attrs):
    out = b"".join(_ld(1, i.encode()) for i in ins) + b"".join(_ld(2, o.encode()) for o in outs) + _ld(4, op.encode())
    for k, v in attrs.items():
        a = _ld(1, k.encode())
        if isinstance(v, float):
            a += _enc_varint((2 << 3) | 5) + struct.pack("<f", v) + _vi(20, 1)
        elif isinstance(v, int):
            a += _vi(3, v) + _vi(20, 2)
        else:
            a += b"".join(_vi(8, x) for x in v) + _vi(20, 7)
        out += _ld(5, a)
    return _ld(1, out)


def _vinfo(fn, name, shape):
    dims = b"".join(_ld(1, (_vi(1, d) if isinstance(d, int) else _ld(2, str(d).encode()))) for d in shape)
    ttype = _vi(1, 1) + _ld(2, dims)
    return _ld(fn, _ld(1, name.encode()) + _ld(2, _ld(1, ttype)))


def _model(graph_body, opset):
    return _vi(1, 8) + _ld(8, _ld(1, b"") + _vi(2, opset)) + _ld(7, graph_body)


def _head_body(head, fused_layernorm, use_matmul, pre, out_name):
    """Nodes + initialisers of one DNN branch reading the graph input; tensor names carry the prefix `pre`."""
    body, x = b"", pre + "flat"
    body += _node("Flatten", ["onnx::Flatten_0"], [x], axis=1)
    L = head["layers"]
    for i, lay in enumerate(L):
        W, b = np.asarray(lay["W"], np.float32), np.asarray(lay["b"], np.float32)
        if use_matmul:
            body += _ld(5, _tensor_proto(f"{pre}W{i}", W)) + _ld(5, _tensor_proto(f"{pre}b{i}", b))
            body += _node("MatMul", [x, f"{pre}W{i}"], [f"{pre}mm{i}"]) + _node("Add", [f"{pre}mm{i}", f"{pre}b{i}"], [f"{pre}lin{i}"])
        else:
            body += _ld(5, _tensor_proto(f"{pre}W{i}", np.ascontiguousarray(W.T))) + _ld(5, _tensor_proto(f"{pre}b{i}", b))
            body += _node("Gemm", [x, f"{pre}W{i}", f"{pre}b{i}"], [f"{pre}lin{i}"], alpha=1.0, beta=1.0, transB=1)
        x = f"{pre}lin{i}"
        if i == len(L) - 1:
            break
        if lay.get("ln") is not None:
            g_, h_ = lay["ln"]
            body += _ld(5, _tensor_proto(f"{pre}g{i}", np.asarray(g_, np.float32))) + _ld(5, _tensor_proto(f"{pre}h{i}", np.asarray(h_, np.float32)))
            if fused_layernorm:
                body += _node("LayerNormalization", [x, f"{pre}g{i}", f"{pre}h{i}"], [f"{pre}ln{i}"], axis=-1, epsilon=1e-5)
            else:
                body += _ld(5, _tensor_proto(f"{pre}two{i}", np.asarray(2.0, np.float32))) + _ld(5, _tensor_proto(f"{pre}eps{i}", np.asarray(1e-5, np.float32)))
                body += _node("ReduceMean", [x], [f"{pre}mu{i}"], axes=[-1])
                body += _node("Sub", [x, f"{pre}mu{i}"], [f"{pre}c{i}"])
                body += _node("Pow", [f"{pre}c{i}", f"{pre}two{i}"], [f"{pre}sq{i}"])
                body += _node("ReduceMean", [f"{pre}sq{i}"], [f"{pre}var{i}"], axes=[-1])
                body += _node("Add", [f"{pre}var{i}", f"{pre}eps{i}"], [f"{pre}ve{i}"])
                body += _node("Sqrt", [f"{pre}ve{i}"], [f"{pre}sd{i}"])
                body += _node("Div", [f"{pre}c{i}", f"{pre}sd{i}"], [f"{pre}nrm{i}"])
                body += _node("Mul", [f"{pre}nrm{i}", f"{pre}g{i}"], [f"{pre}sc{i}"])
                body += _node("Add", [f"{pre}sc{i}", f"{pre}h{i}"], [f"{pre}ln{i}"])
            x = f"{pre}ln{i}"
        body += _node("Relu", [x], [f"{pre}act{i}"])
        x = f"{pre}act{i}"
    fin = head["final"]
    if fin == "sigmoid":
        body += _node("Sigmoid", [x], [out_name])
    elif fin == "relu_softmax":
        body += _node("Relu", [x], [pre + "pre"]) + _node("Softmax", [pre + "pre"], [out_name], axis=1)
    elif fin == "softmax":
        body += _node("Softmax", [x], [out_name], axis=1)
    elif fin == "relu":
        body += _node("Relu", [x], [out_name])
    else:
        body += _node("Identity", [x], [out_name])
    return body


def write_head_onnx(path, head, fused_layernorm=False, use_matmul=False):
    """torch.onnx.export-shaped graph of a head dict (opset 13 decomposed LayerNorm by default).  A gated pair is
    written as two branches joined by Greater + Where (the conditional-verifier structure of hey_jarvis)."""
    if "verifier" in head:
        body = _head_body(head["main"], fused_layernorm, use_matmul, "m_", "p_main")
        body += _head_body(head["verifier"], fused_layernorm, use_matmul, "v_", "p_ver")
        body += _ld(5, _tensor_proto("gate_thr", np.asarray(head["threshold"], np.float32)))
        body += _node("Greater", ["p_main", "gate_thr"], ["gate"]) + _node("Where", ["gate", "p_ver", "p_main"], ["out"])
        n_in, n_out = head["main"]["n_in"], 1
    else:
        body = _head_body(head, fused_layernorm, use_matmul, "", "out")
        n_in, n_out = head["n_in"], head["layers"][-1]["W"].shape[1]
    body += _ld(2, b"head") + _vinfo(11, "onnx::Flatten_0", [1, n_in, 96]) + _vinfo(12, "out", [1, n_out])
    open(path, "wb").write(_model(body, 17 if fused_layernorm else 13))


def write_embedding_onnx(path, weights):
    """20 Conv (OIHW) + 19 BatchNormalization nodes in graph order (structure only; activations omitted)."""
    body, x = b"", "input_1"
    for li, w in enumerate(weights["conv"]):
        body += _ld(5, _tensor_proto(f"k{li}", np.ascontiguousarray(np.asarray(w, np.float32).transpose(3, 2, 0, 1))))
        body += _node("Conv", [x, f"k{li}"], [f"c{li}"])
        x = f"c{li}"
        if li < len(weights["bn"]):
            for nm, p in zip(("s", "b", "m", "v"), weights["bn"][li]):
                body += _ld(5, _tensor_proto(f"{nm}{li}", np.asarray(p, np.float32)))
            body += _node("BatchNormalization", [x, f"s{li}", f"b{li}", f"m{li}", f"v{li}"], [f"n{li}"], epsilon=float(_weights.BN_EPS))
            x = f"n{li}"
    body += _ld(2, b"embedding") + _vinfo(11, "input_1", ["batch", 76, 32, 1]) + _vinfo(12, x, ["batch", 1, 1, 96])
    open(path, "wb").write(_model(body, 13))
