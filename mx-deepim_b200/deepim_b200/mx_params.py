"""Reader / writer for MXNet `.params` checkpoints (`mx.nd.save` of a name -> NDArray dict), so the published DeepIM
weights (README.md:184, `<prefix>-%04d.params`) can be loaded without MXNet (SURVEY 8(f) row 1).

Mirrors lib/utils/load_model.py:10-30 (`load_checkpoint`: keys are "arg:<name>" / "aux:<name>").

The container format lives in MXNet (not vendored; README pins 1.2.0) -- restated from its NDArray serialiser
(src/ndarray/ndarray.cc, `NDArray::Save/Load` and the list container of `MXNDArraySave`):

    uint64  0x112  (list magic)      uint64 0 (reserved)
    uint64  n_arrays ; n_arrays x NDArray
    uint64  n_names  ; n_names x (uint64 length, bytes)

    NDArray (V2, MXNet >= 1.0):  uint32 0xF993FAC9, int32 storage type (0 = dense),
                                 uint32 ndim, int64 dims[ndim], int32 dev_type, int32 dev_id, int32 type_flag, raw data
    NDArray (V1):                uint32 0xF993FAC8, then as V2 without the storage type
    NDArray (legacy, < 0.12):    uint32 ndim, uint32 dims[ndim], int32 dev_type, int32 dev_id, int32 type_flag, raw data

PARITY UNPINNED: the reference ships no `.params` file and MXNet cannot be installed here, so the reader is pinned only
against this module's own writer and a hand-assembled byte string in tests/test_capi_and_host.py."""
from __future__ import annotations

import struct

import numpy as np

LIST_MAGIC = 0x112
V2_MAGIC, V1_MAGIC = 0xF993FAC9, 0xF993FAC8
DTYPES = {0: np.float32, 1: np.float64, 2: np.float16, 3: np.uint8, 4: np.int32, 5: np.int8, 6: np.int64}
FLAGS = {np.dtype(v): k for k, v in DTYPES.items()}


class _Reader:
    def __init__(self, buf):
        self.b, self.o = memoryview(buf), 0

    def take(self, fmt):
        try:
            v = struct.unpack_from("<" + fmt, self.b, self.o)
        except struct.error:
            raise ValueError("truncated .params file") from None
        self.o += struct.calcsize("<" + fmt)
        return v if len(v) > 1 else v[0]

    def raw(self, n):
        v = self.b[self.o:self.o + n]
        if len(v) != n:
            raise ValueError("truncated .params file")
        self.o += n
        return v


def _read_ndarray(r):
    magic = r.take("I")
    if magic == V2_MAGIC:
        stype = r.take("i")
        if stype != 0:
            raise NotImplementedError("sparse NDArray (storage type %d) in .params" % stype)
        ndim = r.take("I")
        shape = [r.take("q") for _ in range(ndim)]
    elif magic == V1_MAGIC:
        ndim = r.take("I")
        shape = [r.take("q") for _ in range(ndim)]
    else:  # legacy: the word just read is ndim
        ndim = magic
        if ndim > 32:
            raise ValueError("not an MXNet NDArray record (magic 0x%08x)" % magic)
        shape = [r.take("I") for _ in range(ndim)]
    if ndim == 0:
        return np.zeros((0,), np.float32)
    r.take("ii")  # context: dev_type, dev_id
    flag = r.take("i")
    if flag not in DTYPES:
        raise ValueError("unknown MXNet type flag %d" % flag)
    dt = np.dtype(DTYPES[flag])
    n = int(np.prod(shape, dtype=np.int64))
    return np.frombuffer(r.raw(n * dt.itemsize), dtype=dt).reshape(shape).copy()


def load(path_or_bytes):
    """mx.nd.load: returns {name: ndarray} (or a list when the file carries no names)."""
    buf = path_or_bytes if isinstance(path_or_bytes, (bytes, bytearray, memoryview)) else open(path_or_bytes, "rb").read()
    r = _Reader(buf)
    if r.take("Q") != LIST_MAGIC:
        raise ValueError("not an MXNet NDArray list file")
    r.take("Q")
    arrays = [_read_ndarray(r) for _ in range(r.take("Q"))]
    names = [bytes(r.raw(r.take("Q"))).decode("utf-8") for _ in range(r.take("Q"))]
    if not names:
        return arrays
    if len(names) != len(arrays):
        raise ValueError("name / array count mismatch")
    return dict(zip(names, arrays))


def save(path, params: dict):
    """mx.nd.save of a dict (V2 records, cpu(0) context)."""
    out = [struct.pack("<QQQ", LIST_MAGIC, 0, len(params))]
    for a in params.values():
        a = np.ascontiguousarray(a)
        out.append(struct.pack("<IiI", V2_MAGIC, 0, a.ndim))
        out.append(struct.pack("<%dq" % a.ndim, *a.shape))
        out.append(struct.pack("<iii", 1, 0, FLAGS[a.dtype]))
        out.append(a.tobytes())
    out.append(struct.pack("<Q", len(params)))
    for k in params:
        kb = k.encode("utf-8")
        out.append(struct.pack("<Q", len(kb)) + kb)
    data = b"".join(out)
    if path is not None:
        with open(path, "wb") as f:
            f.write(data)
    return data


def load_checkpoint(prefix, epoch):
    """lib/utils/load_model.py:10-30: (arg_params, aux_params) as dicts of numpy arrays."""
    d = load("%s-%04d.params" % (prefix, epoch))
    arg, aux = {}, {}
    for k, v in d.items():
        tp, name = k.split(":", 1)
        (arg if tp == "arg" else aux if tp == "aux" else {})[name] = v
    return arg, aux


def save_checkpoint(prefix, epoch, arg_params, aux_params=None):
    d = {"arg:" + k: v for k, v in arg_params.items()}
    d.update({"aux:" + k: v for k, v in (aux_params or {}).items()})
    save("%s-%04d.params" % (prefix, epoch), d)


def input_depth_of(arg_params) -> bool:
    """Which network a checkpoint belongs to, from its flow_conv1_weight: (64, 8, 7, 7) = RGB (INPUT_MASK), (64, 10, 7, 7) =
    RGB-D (INPUT_DEPTH + INPUT_MASK, deepIM_flownet.py:33-51).  Anything else raises ValueError."""
    shape = tuple(np.shape(arg_params["flow_conv1_weight"]))
    if shape == (64, 8, 7, 7):
        return False
    if shape == (64, 10, 7, 7):
        return True
    raise ValueError("flow_conv1_weight has shape %s: expected (64, 8, 7, 7) (RGB) or (64, 10, 7, 7) (RGB-D)" % (shape,))


def network_of(arg_params) -> dict:
    """Which network a checkpoint belongs to, as Context keyword arguments, from its flow_conv1_weight: (64, 8, 7, 7) = RGB
    (INPUT_MASK) -> {input_depth: False, input_mask: True}; (64, 10, 7, 7) = RGB-D (INPUT_DEPTH + INPUT_MASK) -> input_depth
    True; (64, 6, 7, 7) = image-only (INPUT_MASK: False, deepIM_flownet.py:53-62, e.g. a FlowNetS-initialised model) ->
    input_mask False.  Anything else raises ValueError."""
    shape = tuple(np.shape(arg_params["flow_conv1_weight"]))
    nets = {(64, 8, 7, 7): (False, True), (64, 10, 7, 7): (True, True), (64, 6, 7, 7): (False, False)}
    if shape not in nets:
        raise ValueError("flow_conv1_weight has shape %s: expected (64, 8, 7, 7) (RGB), (64, 10, 7, 7) (RGB-D) or (64, 6, 7, 7) "
                         "(image-only)" % (shape,))
    depth, mask = nets[shape]
    return {"input_depth": depth, "input_mask": mask}


# ----------------------------------------------------------------------------------------- <prefix>-symbol.json
# MXNet writes the network graph next to the checkpoint (`Module.save_checkpoint` -> `<prefix>-symbol.json`): a JSON object
# {"nodes": [{"op": "null" | "<Operator>", "name": ..., "attrs" (>= 1.0) | "attr" | "param" (older): {str: str},
#             "inputs": [[node_id, output_index, version], ...]}, ...],
#  "arg_nodes": [ids of the "null" nodes = variables], "node_row_ptr": [...], "heads": [[node_id, index, version], ...],
#  "attrs": {"mxnet_version": ["int", 10200]}}.
# The CUDA path does not execute the graph (it IS the FlowNetS tower of deepim/symbols/deepIM_flownet.py:53-116); reading the
# file serves to CHECK that a checkpoint belongs to this architecture before its tensors are repacked.
def load_symbol_json(path_or_text):
    import json
    import os
    text = open(path_or_text).read() if os.path.exists(str(path_or_text)) else path_or_text
    g = json.loads(text)
    if "nodes" not in g or "arg_nodes" not in g:
        raise ValueError("not an MXNet symbol file (no 'nodes' / 'arg_nodes')")
    nodes = []
    for n in g["nodes"]:
        attrs = n.get("attrs", n.get("attr", n.get("param", {}))) or {}
        nodes.append({"op": n["op"], "name": n["name"], "attrs": {str(k): str(v) for k, v in attrs.items()},
                      "inputs": [int(i[0]) for i in n.get("inputs", [])]})
    return {"nodes": nodes, "arg_nodes": [int(i) for i in g["arg_nodes"]], "heads": [int(h[0]) for h in g.get("heads", [])],
            "arguments": [nodes[int(i)]["name"] for i in g["arg_nodes"]]}


def _tuple_attr(v):
    return tuple(int(x) for x in v.strip("()[] ").replace(" ", "").split(",") if x != "")


def check_flownet_symbol(sym, conv_specs=None):
    """Raise ValueError unless every Convolution of the FlowNetS tower (name, num_filter, kernel, stride, pad as in
    deepIM_flownet.py:63-107) and fc6 / fc7 (FullyConnected, 256 hidden) are present in the symbol with those attributes."""
    from . import synth
    conv_specs = conv_specs or synth.CONV_SPECS
    by_name = {n["name"]: n for n in sym["nodes"]}
    for name, cout, cin, k, s, p in conv_specs:
        n = by_name.get(name)
        if n is None or n["op"] != "Convolution":
            raise ValueError("symbol has no Convolution named %r" % name)
        a = n["attrs"]
        got = (int(a.get("num_filter", -1)), _tuple_attr(a.get("kernel", "()")), _tuple_attr(a.get("stride", "(1,1)")),
               _tuple_attr(a.get("pad", "(0,0)")))
        if got != (cout, (k, k), (s, s), (p, p)):
            raise ValueError("%s: symbol says %r, FlowNetS expects %r" % (name, got, (cout, (k, k), (s, s), (p, p))))
        if name + "_weight" not in sym["arguments"]:
            raise ValueError("%s_weight is not an argument of the symbol" % name)
    for name in ("fc6", "fc7"):
        n = by_name.get(name)
        if n is None or n["op"] != "FullyConnected" or int(n["attrs"].get("num_hidden", -1)) != 256:
            raise ValueError("symbol has no FullyConnected %r with 256 hidden units" % name)
    return True


def save_symbol_json(path, conv_specs=None):
    """Write the FAST_TEST inference graph (tower + fc6 / fc7 + rot / trans heads) in MXNet's symbol-file layout (testing aid)."""
    import json
    from . import synth
    conv_specs = conv_specs or synth.CONV_SPECS
    nodes, args = [], []

    def var(name):
        nodes.append({"op": "null", "name": name, "inputs": []})
        args.append(len(nodes) - 1)
        return len(nodes) - 1

    def op(kind, name, inputs, attrs):
        nodes.append({"op": kind, "name": name, "attrs": attrs, "inputs": [[i, 0, 0] for i in inputs]})
        return len(nodes) - 1

    x = var("data")
    for name, cout, cin, k, s, p in conv_specs:
        w, b = var(name + "_weight"), var(name + "_bias")
        x = op("Convolution", name, [x, w, b], {"num_filter": str(cout), "kernel": "(%d, %d)" % (k, k), "stride": "(%d, %d)" % (s, s),
                                                 "pad": "(%d, %d)" % (p, p)})
        x = op("LeakyReLU", "ReLU_" + name, [x], {"act_type": "leaky", "slope": "0.1"})
    x = op("Flatten", "flatten", [x], {})
    for name in ("fc6", "fc7"):
        w, b = var(name + "_weight"), var(name + "_bias")
        x = op("FullyConnected", name, [x, w, b], {"num_hidden": "256"})
        x = op("LeakyReLU", "ReLU_" + name, [x], {"act_type": "leaky", "slope": "0.1"})
    heads = []
    for name, nh in (("rot", 4), ("trans", 3)):
        w, b = var(name + "_weight"), var(name + "_bias")
        heads.append(op("FullyConnected", name, [x, w, b], {"num_hidden": str(nh)}))
    g = {"nodes": nodes, "arg_nodes": args, "node_row_ptr": list(range(len(nodes) + 1)), "heads": [[h, 0, 0] for h in heads],
         "attrs": {"mxnet_version": ["int", 10200]}}
    with open(path, "w") as f:
        json.dump(g, f)
    return path
