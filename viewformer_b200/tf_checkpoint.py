"""TensorFlow checkpoint container (TensorBundle + object graph) reader / writer in pure Python — no TensorFlow needed.

The reference restores its transformer with Keras ``model.load_weights(<dir>/model)`` (viewformer/utils/tensorflow.py:20-63): a TF2
object-graph checkpoint, i.e. two files

    model.index                 an SSTable (LevelDB table format, uncompressed blocks) mapping
                                  ""                              -> BundleHeaderProto
                                  "_CHECKPOINTABLE_OBJECT_GRAPH"  -> BundleEntryProto of a DT_STRING tensor holding a TrackableObjectGraph
                                  "<path>/.ATTRIBUTES/VARIABLE_VALUE" -> BundleEntryProto (dtype, shape, shard, offset, size, crc32c)
    model.data-00000-of-00001   the raw little-endian tensor bytes

Variables are resolved by WALKING THE OBJECT GRAPH along attribute names (``h`` -> ``0`` -> ``attn`` -> ``c_attn`` -> ``weight``), the way
Keras itself matches a checkpoint to a model, so the spelling of the checkpoint keys does not matter.  Those attribute paths are the
reference's layer attribute names (models/migt.py:284-315: wte, wpe, pose_embedding, pose_classifier, h[i].{ln_1, attn.{c_attn,c_proj},
ln_2, mlp.{c_fc,c_proj}}, ln_f) = the state_dict key names of viewformer_b200.MIGT with '.' for '/'.

``write_checkpoint`` produces the same container (used by ``MIGT.save_weights`` and by the tests: there is no TensorFlow in this image
to produce a file with, so the reader is validated against this writer and against the format rules above — see DESIGN.md).
"""
import os
import struct

import numpy as np

_MAGIC = 0xDB4775248B80FB57
_DTYPES = {1: np.float32, 2: np.float64, 3: np.int32, 4: np.uint8, 5: np.int16, 6: np.int8, 9: np.int64, 10: np.bool_, 19: np.float16}
_DTYPE_CODES = {np.dtype(v): k for k, v in _DTYPES.items()}
OBJECT_GRAPH_KEY = "_CHECKPOINTABLE_OBJECT_GRAPH"
VAR_SUFFIX = "/.ATTRIBUTES/VARIABLE_VALUE"
SLOT_INFIX = "/.OPTIMIZER_SLOT/"                           # key of a slot variable: <variable path>/.OPTIMIZER_SLOT/<owner path>/<slot name>


# ----------------------------------------------------------------------------------------------- varint / protobuf wire helpers
def _varint(buf, pos):
    r, s = 0, 0
    while True:
        b = buf[pos]
        pos += 1
        r |= (b & 0x7F) << s
        if not b & 0x80:
            return r, pos
        s += 7


def _put_varint(v):
    out = bytearray()
    v &= (1 << 64) - 1
    while True:
        b = v & 0x7F
        v >>= 7
        if v:
            out.append(b | 0x80)
        else:
            out.append(b)
            return bytes(out)


def _fields(buf):
    """Yield (field_number, wire_type, value) of one protobuf message; length-delimited values come back as bytes."""
    pos, n = 0, len(buf)
    while pos < n:
        tag, pos = _varint(buf, pos)
        fn, wt = tag >> 3, tag & 7
        if wt == 0:
            v, pos = _varint(buf, pos)
        elif wt == 1:
            v = struct.unpack_from("<Q", buf, pos)[0]
            pos += 8
        elif wt == 2:
            ln, pos = _varint(buf, pos)
            v = bytes(buf[pos:pos + ln])
            pos += ln
        elif wt == 5:
            v = struct.unpack_from("<I", buf, pos)[0]
            pos += 4
        else:
            raise ValueError(f"unsupported protobuf wire type {wt}")
        yield fn, wt, v


def _msg(*parts):
    return b"".join(parts)


def _f_varint(fn, v):
    return _put_varint(fn << 3) + _put_varint(v)


def _f_bytes(fn, b):
    return _put_varint((fn << 3) | 2) + _put_varint(len(b)) + b


def _f_fixed32(fn, v):
    return _put_varint((fn << 3) | 5) + struct.pack("<I", v)


# ----------------------------------------------------------------------------------------------- crc32c (Castagnoli), masked as in TF / LevelDB
_CRC_TABLE = None


def _crc_table():
    global _CRC_TABLE
    if _CRC_TABLE is None:
        t = []
        for i in range(256):
            c = i
            for _ in range(8):
                c = (c >> 1) ^ 0x82F63B78 if c & 1 else c >> 1
            t.append(c)
        _CRC_TABLE = t
    return _CRC_TABLE


def crc32c(data, crc=0):
    t = _crc_table()
    c = crc ^ 0xFFFFFFFF
    for b in bytes(data):
        c = t[(c ^ b) & 0xFF] ^ (c >> 8)
    return c ^ 0xFFFFFFFF


def masked_crc(data):
    c = crc32c(data)
    return (((c >> 15) | (c << 17)) + 0xA282EAD8) & 0xFFFFFFFF


# ----------------------------------------------------------------------------------------------- SSTable (LevelDB table) reader
def _block_entries(block):
    """Entries of one uncompressed table block: prefix-compressed keys, restart array at the end."""
    n_restarts = struct.unpack_from("<I", block, len(block) - 4)[0]
    end = len(block) - 4 - 4 * n_restarts
    pos, key = 0, b""
    while pos < end:
        shared, pos = _varint(block, pos)
        non_shared, pos = _varint(block, pos)
        vlen, pos = _varint(block, pos)
        key = key[:shared] + bytes(block[pos:pos + non_shared])
        pos += non_shared
        yield key, bytes(block[pos:pos + vlen])
        pos += vlen


def _read_block(data, offset, size, verify=False):
    """Block contents; every block is followed by a 5-byte trailer: compression type + masked crc32c(contents + type)."""
    if offset + size + 5 > len(data):
        raise ValueError("SSTable block handle points past the end of the file")
    ctype = data[offset + size]
    if ctype != 0:
        raise NotImplementedError("compressed SSTable block (type %d): TensorFlow writes checkpoint indices uncompressed" % ctype)
    if verify and struct.unpack_from("<I", data, offset + size + 1)[0] != masked_crc(data[offset:offset + size + 1]):
        raise ValueError(f"SSTable block at offset {offset}: crc32c mismatch")
    return data[offset:offset + size]


def read_index(prefix, verify=False):
    """``<prefix>.index`` -> {key: value bytes} (values are serialized BundleHeaderProto / BundleEntryProto).  ``verify`` checks the
    crc32c trailer of every table block (LevelDB's ``verify_checksums``; off by default as in TensorFlow's BundleReader)."""
    with open(prefix + ".index", "rb") as f:
        data = f.read()
    if len(data) < 48 or struct.unpack_from("<Q", data, len(data) - 8)[0] != _MAGIC:
        raise ValueError(f"{prefix}.index is not an SSTable (bad magic)")
    footer = data[-48:]
    pos = 0
    _, pos = _varint(footer, pos)          # metaindex handle
    _, pos = _varint(footer, pos)
    ioff, pos = _varint(footer, pos)       # index block handle
    isize, pos = _varint(footer, pos)
    out = {}
    for _, handle in _block_entries(_read_block(data, ioff, isize, verify)):
        boff, p = _varint(handle, 0)
        bsize, p = _varint(handle, p)
        for k, v in _block_entries(_read_block(data, boff, bsize, verify)):
            out[k.decode("utf-8", "surrogateescape")] = v
    return out


def parse_entry(buf):
    """BundleEntryProto -> dict(dtype, shape, shard_id, offset, size, crc32c)."""
    e = dict(dtype=0, shape=[], shard_id=0, offset=0, size=0, crc32c=None)
    for fn, wt, v in _fields(buf):
        if fn == 1:
            e["dtype"] = v
        elif fn == 2:
            for f2, _, v2 in _fields(v):
                if f2 == 2:                                   # TensorShapeProto.dim
                    size = 0
                    for f3, _, v3 in _fields(v2):
                        if f3 == 1:
                            size = v3 if v3 < (1 << 63) else v3 - (1 << 64)
                    e["shape"].append(size)
        elif fn == 3:
            e["shard_id"] = v
        elif fn == 4:
            e["offset"] = v
        elif fn == 5:
            e["size"] = v
        elif fn == 6:
            e["crc32c"] = v
    return e


class Checkpoint:
    """Random access to the tensors of a TensorBundle checkpoint."""

    def __init__(self, prefix):
        self.prefix = prefix
        self.raw = read_index(prefix)
        if "" not in self.raw:
            raise ValueError("checkpoint index has no header entry")
        self.num_shards, self.little_endian = 1, True
        for fn, _, v in _fields(self.raw[""]):
            if fn == 1:
                self.num_shards = v
            elif fn == 2:
                self.little_endian = v == 0
        if not self.little_endian:
            raise NotImplementedError("big-endian checkpoint")
        self.entries = {k: parse_entry(v) for k, v in self.raw.items() if k != ""}

    def keys(self):
        return list(self.entries.keys())

    def _shard(self, i):
        return "%s.data-%05d-of-%05d" % (self.prefix, i, self.num_shards)

    def read_bytes(self, key):
        e = self.entries[key]
        with open(self._shard(e["shard_id"]), "rb") as f:
            f.seek(e["offset"])
            return f.read(e["size"])

    def tensor(self, key, verify_crc=False):
        e = self.entries[key]
        raw = self.read_bytes(key)
        if verify_crc and e["crc32c"] is not None and masked_crc(raw) != e["crc32c"]:
            raise ValueError(f"crc32c mismatch for {key}")
        if e["dtype"] == 7:                                   # DT_STRING: varint lengths, a masked crc of them, then the bytes
            n = int(np.prod(e["shape"])) if e["shape"] else 1
            pos, lens = 0, []
            for _ in range(n):
                ln, pos = _varint(raw, pos)
                lens.append(ln)
            pos += 4
            out = []
            for ln in lens:
                out.append(raw[pos:pos + ln])
                pos += ln
            return out[0] if not e["shape"] else out
        if e["dtype"] not in _DTYPES:
            raise NotImplementedError(f"dtype code {e['dtype']} of {key}")
        return np.frombuffer(raw, dtype=_DTYPES[e["dtype"]]).reshape(e["shape"]).copy()

    # --- object graph -----------------------------------------------------------------------------------------
    def object_graph(self):
        """TrackableObjectGraph -> list of nodes: dict(children={local_name: node_id}, attributes={name: checkpoint_key},
        slots={(original_variable_node_id, slot_name): slot_variable_node_id}) — the last on the node that owns the slots (an optimizer)."""
        blob = self.tensor(OBJECT_GRAPH_KEY)
        nodes = []
        for fn, _, v in _fields(blob):
            if fn != 1:
                continue
            node = dict(children={}, attributes={}, slots={})
            for f2, _, v2 in _fields(v):
                if f2 == 1:                                   # ObjectReference
                    nid, name = 0, ""
                    for f3, _, v3 in _fields(v2):
                        if f3 == 1:
                            nid = v3
                        elif f3 == 2:
                            name = v3.decode()
                    node["children"][name] = nid
                elif f2 == 2:                                 # SerializedTensor
                    aname, ckey = "", ""
                    for f3, _, v3 in _fields(v2):
                        if f3 == 1:
                            aname = v3.decode()
                        elif f3 == 3:
                            ckey = v3.decode()
                    node["attributes"][aname] = ckey
                elif f2 == 3:                                 # SlotVariableReference
                    orig, sname, snid = 0, "", 0
                    for f3, _, v3 in _fields(v2):
                        if f3 == 1:
                            orig = v3
                        elif f3 == 2:
                            sname = v3.decode()
                        elif f3 == 3:
                            snid = v3
                    node["slots"][(orig, sname)] = snid
            nodes.append(node)
        return nodes

    @staticmethod
    def _walk(path, nodes):
        nid = 0
        for part in path.split("/"):
            ch = nodes[nid]["children"]
            if part not in ch:
                raise KeyError(f"checkpoint object graph has no '{part}' under '{path}'")
            nid = ch[part]
        return nid

    def resolve(self, path, nodes=None):
        """Attribute path ('h/0/attn/c_attn/weight') -> checkpoint key of its VARIABLE_VALUE, via the object graph."""
        nodes = self.object_graph() if nodes is None else nodes
        attrs = nodes[self._walk(path, nodes)]["attributes"]
        if "VARIABLE_VALUE" not in attrs:
            raise KeyError(f"'{path}' is not a variable in the checkpoint")
        return attrs["VARIABLE_VALUE"]

    def slot(self, path, slot_name, owner="optimizer", nodes=None):
        """Checkpoint key of the slot variable ``slot_name`` ('m', 'v') that the object at ``owner`` keeps for the variable at ``path``."""
        nodes = self.object_graph() if nodes is None else nodes
        ref = (self._walk(path, nodes), slot_name)
        slots = nodes[self._walk(owner, nodes)]["slots"]
        if ref not in slots or "VARIABLE_VALUE" not in nodes[slots[ref]]["attributes"]:
            raise KeyError(f"'{owner}' keeps no slot '{slot_name}' for '{path}'")
        return nodes[slots[ref]]["attributes"]["VARIABLE_VALUE"]


def object_paths(key):
    """Object-graph paths under which the reference's Keras MIGT tracks the variable of state_dict key ``key`` — the Python attribute
    names a TF2 object-based checkpoint is keyed by — most specific first (checked against the attributes of the real model object in
    tests/test_reference_on_shim.py).  Almost always 'a.b.c' -> 'a/b/c' (h/<i>/attn/c_attn/weight, ln_f/gamma, wte/weight ...); two are not:
      * ``wpe.embeddings``: MIGT.build does ``self.wpe = self.add_weight(name="embeddings", ...)`` on the MODEL (migt.py:305-315), so the
        variable hangs directly off the root, as 'wpe' (attribute) and 'embeddings' (add_weight's dependency name);
      * ``pose_classifier.*``: the MLP is owned by ``self.pose_criterion`` (QuaternionPoseRepresentation, migt.py:136, :277).
    The literal 'a/b/c' form stays last so that files written by earlier versions of this package still load."""
    base = key.replace(".", "/")
    if key == "wpe.embeddings":
        return ["wpe", "embeddings", base]
    if key.startswith("pose_classifier."):
        return ["pose_criterion/" + base, base]
    return [base]


def load_state_dict(prefix, expected_keys, strict=True):
    """{state_dict key: torch tensor} for ``expected_keys`` ('h.0.attn.c_attn.weight' <-> object path 'h/0/attn/c_attn/weight', see
    ``object_paths``).  Falls back to the literal checkpoint key '<path>/.ATTRIBUTES/VARIABLE_VALUE' when the file carries no object graph."""
    import torch
    ck = Checkpoint(prefix)
    nodes = ck.object_graph() if OBJECT_GRAPH_KEY in ck.entries else None
    out, missing = {}, []
    for k in expected_keys:
        for path in object_paths(k):
            try:
                key = ck.resolve(path, nodes) if nodes is not None else path + VAR_SUFFIX
                if key not in ck.entries:
                    raise KeyError(key)
                out[k] = torch.from_numpy(ck.tensor(key))
                break
            except KeyError:
                continue
        else:
            missing.append(k)
    if missing and strict:
        raise RuntimeError(f"Missing keys in TF checkpoint {prefix}: {missing[:8]}{' ...' if len(missing) > 8 else ''}")
    return out


# ----------------------------------------------------------------------------------------------- optimizer entries
# Where the reference's compiled Keras model keeps what MIGTTrainer.optimizer_state() holds.  'optimizer' (the model's attribute),
# 'iter' (OptimizerV2.iterations' weight name), the schedule under 'learning_rate' with WarmUp's 'offset' attribute and the Adam slot
# names 'm' / 'v' are the names the reference's AdamWeightDecay / WarmUp / MIGT objects carry (tests/test_trainer_state_formats.py walks
# them).  The names below the wrapper that --fp16 adds (mixed_precision.LossScaleOptimizer: the wrapped optimizer as 'base_optimizer',
# the scale as 'loss_scale' with weights 'current_loss_scale' / 'good_steps') are TF 2.4's as far as known, and whether TF 2.4 tracks a
# LearningRateSchedule's variables at all could not be checked either — see INTEGRATION.md.  Keras does not checkpoint the model's
# _train_counter; it and the dropout seed travel under a child of the root that Keras does not know and skips under expect_partial().
OPTIMIZER_SCALARS = {                                       # optimizer_state() key -> (path below the Adam optimizer's node, dtype)
    "iterations": ("iter", np.int64),
    "schedule_offset": ("learning_rate/offset", np.int64),
}
LOSS_SCALE_SCALARS = {                                      # ... -> (path below the LossScaleOptimizer's node, dtype)
    "loss_scale": ("loss_scale/current_loss_scale", np.float32),
    "loss_scale_counter": ("loss_scale/good_steps", np.int64),
}
EXTRA_SCALARS = {"train_counter": ("viewformer_b200/train_counter", np.int64), "seed": ("viewformer_b200/seed", np.int64)}
OPTIMIZER_ROOT, BASE_OPTIMIZER, SLOT_NAMES = "optimizer", "base_optimizer", ("m", "v")


def optimizer_entries(state):
    """MIGTTrainer.optimizer_state() -> (tensors, slots) for ``write_checkpoint``, next to the weights written under ``object_paths``."""
    bf16 = state["precision"] == "bf16"
    adam = OPTIMIZER_ROOT + ("/" + BASE_OPTIMIZER if bf16 else "")
    tensors = {adam + "/" + path: np.asarray(state[k], dt) for k, (path, dt) in OPTIMIZER_SCALARS.items()}
    if bf16:
        tensors.update({OPTIMIZER_ROOT + "/" + path: np.asarray(state[k], dt) for k, (path, dt) in LOSS_SCALE_SCALARS.items()})
    tensors.update({path: np.asarray(state[k], dt) for k, (path, dt) in EXTRA_SCALARS.items()})
    slots = {(adam, slot, object_paths(key)[0]): t.numpy() for slot in SLOT_NAMES for key, t in state[slot].items()}
    return tensors, slots


def load_optimizer_state(prefix, expected_keys):
    """The optimizer entries of a checkpoint as MIGTTrainer.optimizer_state() lays them out, or None when the file carries none."""
    import torch
    ck = Checkpoint(prefix)
    if OBJECT_GRAPH_KEY not in ck.entries:
        return None
    nodes = ck.object_graph()

    def scalar(path):
        try:
            return ck.tensor(ck.resolve(path, nodes)).item()
        except KeyError:
            return None

    for adam, precision in ((OPTIMIZER_ROOT, "fp32"), (OPTIMIZER_ROOT + "/" + BASE_OPTIMIZER, "bf16")):
        if scalar(adam + "/" + OPTIMIZER_SCALARS["iterations"][0]) is not None:
            break
    else:
        return None
    state = dict(precision=precision)
    tables = [(adam, OPTIMIZER_SCALARS), ("", EXTRA_SCALARS)] + ([(OPTIMIZER_ROOT, LOSS_SCALE_SCALARS)] if precision == "bf16" else [])
    for base, table in tables:
        for k, (path, _) in table.items():
            val = scalar((base + "/" if base else "") + path)
            if val is not None:
                state[k] = val
    for slot in SLOT_NAMES:
        state[slot] = {}
        for key in expected_keys:
            for path in object_paths(key):
                try:
                    state[slot][key] = torch.from_numpy(ck.tensor(ck.slot(path, slot, adam, nodes)))
                    break
                except KeyError:
                    continue
    return state


# ----------------------------------------------------------------------------------------------- writer
def _build_block(items, restart_interval=16):
    out, restarts, prev, n = bytearray(), [], b"", 0
    for k, v in items:
        if n % restart_interval == 0:
            restarts.append(len(out))
            shared = 0
        else:
            shared = 0
            while shared < min(len(prev), len(k)) and prev[shared] == k[shared]:
                shared += 1
        out += _put_varint(shared) + _put_varint(len(k) - shared) + _put_varint(len(v)) + k[shared:] + v
        prev = k
        n += 1
    if not restarts:
        restarts = [0]
    for r in restarts:
        out += struct.pack("<I", r)
    out += struct.pack("<I", len(restarts))
    return bytes(out)


def _emit_block(f, block):
    off = f.tell()
    f.write(block)
    trailer = b"\x00"
    f.write(trailer + struct.pack("<I", masked_crc(block + trailer)))
    return off, len(block)


def write_checkpoint(prefix, tensors, slots=None):
    """Write {attribute path ('h/0/ln_1/gamma'): numpy array} as a TF2 object-graph checkpoint (<prefix>.index + one data shard).
    ``slots``: {(owner path, slot name, variable path): numpy array} — slot variables as an optimizer keeps them: a node of its own per
    slot, reachable only through the owner's ``slot_variables`` (no child edge), stored under the variable's path + SLOT_INFIX + owner +
    slot name.  Owner and variable must be paths of ``tensors``' graph."""
    os.makedirs(os.path.dirname(os.path.abspath(prefix)), exist_ok=True)
    # object graph: one node per path component, variables are leaf nodes with a VARIABLE_VALUE attribute
    nodes = [dict(children={}, attributes={}, slots=[])]

    def node_for(parts):
        nid = 0
        for p in parts:
            ch = nodes[nid]["children"]
            if p not in ch:
                nodes.append(dict(children={}, attributes={}, slots=[]))
                ch[p] = len(nodes) - 1
            nid = ch[p]
        return nid

    entries = {}
    data = bytearray()
    work = [(path, None, arr) for path, arr in tensors.items()]
    for path, _, _ in work:                                   # the whole variable graph first, so that slot nodes come after it
        node_for(path.split("/"))
    work += [(var + SLOT_INFIX + owner + "/" + name, (owner, name, var), arr) for (owner, name, var), arr in (slots or {}).items()]
    for path, slot, arr in work:
        arr = np.asarray(arr)
        if arr.ndim and not arr.flags.c_contiguous:
            arr = np.ascontiguousarray(arr)
        key = path + VAR_SUFFIX
        if slot is None:
            nid = node_for(path.split("/"))
        else:
            owner, name, var = slot
            if var not in tensors or not any(t.startswith(owner + "/") for t in tensors):
                raise KeyError(f"slot '{name}' of '{var}' kept by '{owner}': both must be paths of the variable graph")
            nodes.append(dict(children={}, attributes={}, slots=[]))
            nid = len(nodes) - 1
            nodes[node_for(owner.split("/"))]["slots"].append((node_for(var.split("/")), name, nid))
        nodes[nid]["attributes"]["VARIABLE_VALUE"] = key
        raw = arr.tobytes()
        shape = _msg(*[_f_bytes(2, _f_varint(1, d)) for d in arr.shape])
        entries[key] = _msg(_f_varint(1, _DTYPE_CODES[arr.dtype]), _f_bytes(2, shape), _f_varint(4, len(data)) if len(data) else b"",
                            _f_varint(5, len(raw)), _f_fixed32(6, masked_crc(raw)))
        data += raw
    graph = b""
    for n in nodes:
        body = b""
        for name, nid in n["children"].items():
            body += _f_bytes(1, _msg(_f_varint(1, nid) if nid else b"", _f_bytes(2, name.encode())))
        for name, key in n["attributes"].items():
            body += _f_bytes(2, _msg(_f_bytes(1, name.encode()), _f_bytes(2, key.encode()), _f_bytes(3, key.encode())))
        for orig, name, nid in n["slots"]:
            body += _f_bytes(3, _msg(_f_varint(1, orig), _f_bytes(2, name.encode()), _f_varint(3, nid)))
        graph += _f_bytes(1, body)
    lens = _put_varint(len(graph))
    sraw = lens + struct.pack("<I", masked_crc(lens)) + graph
    entries[OBJECT_GRAPH_KEY] = _msg(_f_varint(1, 7), _f_bytes(2, b""), _f_varint(4, len(data)), _f_varint(5, len(sraw)),
                                     _f_fixed32(6, masked_crc(sraw)))
    data += sraw
    with open(prefix + ".data-00000-of-00001", "wb") as f:
        f.write(bytes(data))
    header = _msg(_f_varint(1, 1), _f_bytes(3, _msg(_f_varint(1, 1))))            # num_shards = 1, little endian (default), version.producer = 1
    items = sorted([(b"", header)] + [(k.encode(), v) for k, v in entries.items()])
    with open(prefix + ".index", "wb") as f:
        handles = []
        for i in range(0, len(items), 64):                                          # several data blocks, as a real table has
            chunk = items[i:i + 64]
            off, size = _emit_block(f, _build_block(chunk))
            handles.append((chunk[-1][0], _put_varint(off) + _put_varint(size)))
        moff, msize = _emit_block(f, _build_block([]))                             # empty metaindex
        ioff, isize = _emit_block(f, _build_block(handles, restart_interval=1))
        footer = _put_varint(moff) + _put_varint(msize) + _put_varint(ioff) + _put_varint(isize)
        f.write(footer + b"\x00" * (40 - len(footer)) + struct.pack("<Q", _MAGIC))
