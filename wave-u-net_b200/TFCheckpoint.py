"""TensorFlow V2 checkpoint ("tensor bundle") reader / writer - replaces the tf.train.Saver calls of the reference
(Training.py:92-98,113 save/restore of tf.global_variables(); Evaluate.py:55-57 restore for prediction) so that
checkpoints written by the reference (e.g. the published M4 / M5 / M6 models, README.md:106-111) load into this engine
and checkpoints written here load back into the reference.  No TensorFlow needed.

Format (restated from the published TensorFlow / LevelDB sources - tensorflow/core/util/tensor_bundle,
tensorflow/core/lib/io/{table,block,format}; TensorFlow itself is not installable here, so this module is pinned by
known-answer vectors of its primitives (CRC-32C RFC 3720 vectors, LevelDB mask constant, varint / protobuf wire bytes,
table magic), by Google's own code where this image carries it - TensorBoard's TensorFlow stub for CRC-32C and its mask, the
protobuf runtime over TensorBoard's generated TensorShapeProto / DataType / VersionDef for the two bundle protos (byte for byte)
and the `checkpoint` state file - and by its own round trip, NOT by a checkpoint written by TensorFlow: the table layout of the
.index stays unpinned - tests/test_tf_checkpoint.py says the same):

  <prefix>.index                  a LevelDB-format sorted string table, uncompressed:
      key ""            -> BundleHeaderProto  { num_shards = 1; endianness = LITTLE; version { producer = 1 } }
      key <tensor name> -> BundleEntryProto   { dtype; shape; shard_id; offset; size; crc32c (masked, of the tensor bytes) }
      data blocks: entries  varint32 shared | varint32 non_shared | varint32 value_len | key suffix | value,
                   a restart (shared = 0) every 16 entries, then fixed32 restart offsets + fixed32 count;
                   every block is followed by a 5-byte trailer: compression type (0) + fixed32 masked CRC-32C of
                   block + type.  Then the (empty) metaindex block, the index block (last key of each data block ->
                   BlockHandle varint64 offset, varint64 size) and the 48-byte footer
                   (metaindex handle, index handle, zero padding to 40 bytes, magic 0xdb4775248b80fb57 little-endian).
  <prefix>.data-00000-of-00001    the raw little-endian tensor bytes, in key order, no padding.
  checkpoint                      text proto naming the latest prefix (what Saver.save also writes).

Names the reference's graph produces (Training.py:66-77, UnetAudioSeparator.py:92, InterpolationLayer.py:19):
  separator/conv1d{,_1,...}/{kernel,bias}, separator/interp_<level>            model variables (kernel = [k, C_in, C_out])
  separator_solver/<variable>/Adam, .../Adam_1                                 Adam slots m, v   [TF naming, from memory]
  separator_solver/beta1_power, separator_solver/beta2_power                   float32 scalars   [TF naming, from memory]
  global_step                                                                  int64 scalar
The loader therefore matches optimizer state by SUFFIX, so either scoping convention restores.
"""
import os
import struct
from collections import OrderedDict

import numpy as np

import wun

TABLE_MAGIC = 0xdb4775248b80fb57
MASK_DELTA = 0xa282ead8
RESTART_INTERVAL = 16
BLOCK_SIZE = 262144          # table::Options::block_size default in TensorFlow's copy of the table code

# tensorflow/core/framework/types.proto
DT_FLOAT, DT_DOUBLE, DT_INT32, DT_UINT8, DT_INT16, DT_INT8, DT_STRING, DT_INT64, DT_BOOL = 1, 2, 3, 4, 5, 6, 7, 9, 10
DT_UINT16, DT_HALF, DT_UINT32, DT_UINT64, DT_BFLOAT16 = 17, 19, 22, 23, 14
_DT_TO_NP = {DT_FLOAT: np.float32, DT_DOUBLE: np.float64, DT_INT32: np.int32, DT_UINT8: np.uint8, DT_INT16: np.int16,
             DT_INT8: np.int8, DT_INT64: np.int64, DT_BOOL: np.bool_, DT_UINT16: np.uint16, DT_HALF: np.float16,
             DT_UINT32: np.uint32, DT_UINT64: np.uint64}
_NP_TO_DT = {np.dtype(v): k for k, v in _DT_TO_NP.items()}


class CheckpointError(ValueError):
    pass


# ------------------------------------------------------------------------------------------------
# primitives
# ------------------------------------------------------------------------------------------------
def mask_crc(crc):
    """LevelDB / TensorFlow crc32c::Mask: rotate right by 15 and add a constant."""
    crc &= 0xffffffff
    return (((crc >> 15) | (crc << 17)) + MASK_DELTA) & 0xffffffff


def unmask_crc(masked):
    rot = (masked - MASK_DELTA) & 0xffffffff
    return ((rot >> 17) | (rot << 15)) & 0xffffffff


def put_varint(out, v):
    if v < 0:
        v += 1 << 64                       # protobuf int32/int64: two's complement, 10 bytes
    while v >= 0x80:
        out.append((v & 0x7f) | 0x80)
        v >>= 7
    out.append(v)


def get_varint(buf, pos):
    shift = result = 0
    while True:
        if pos >= len(buf):
            raise CheckpointError("truncated varint")
        b = buf[pos]
        pos += 1
        result |= (b & 0x7f) << shift
        if not b & 0x80:
            return result, pos
        shift += 7
        if shift > 63:
            raise CheckpointError("varint too long")


def _signed64(v):
    return v - (1 << 64) if v >= (1 << 63) else v


# ---- the three protobuf messages, hand-encoded (field numbers from tensor_bundle.proto / tensor_shape.proto) ----
def encode_header(num_shards=1):
    out = bytearray()
    out += b"\x08"; put_varint(out, num_shards)        # 1: num_shards
    # 2: endianness = LITTLE (0) is the proto3 default and is not serialised
    out += b"\x1a\x02\x08\x01"                           # 3: version { 1: producer = 1 }
    return bytes(out)


def encode_entry(dtype, shape, offset, size, crc_masked, shard_id=0):
    sh = bytearray()
    for d in shape:
        dim = bytearray(b"\x08"); put_varint(dim, int(d))            # Dim.size
        sh += b"\x12"; put_varint(sh, len(dim)); sh += dim            # TensorShapeProto.dim
    out = bytearray()
    out += b"\x08"; put_varint(out, dtype)                             # 1: dtype
    out += b"\x12"; put_varint(out, len(sh)); out += sh                # 2: shape (present even for scalars)
    if shard_id:
        out += b"\x18"; put_varint(out, shard_id)                      # 3: shard_id
    if offset:
        out += b"\x20"; put_varint(out, offset)                        # 4: offset
    if size:
        out += b"\x28"; put_varint(out, size)                          # 5: size
    if crc_masked:                                                     # (proto3: a zero scalar is not serialised)
        out += b"\x35" + struct.pack("<I", crc_masked)                 # 6: crc32c (fixed32)
    return bytes(out)


def _fields(buf):
    """Iterate (field number, wire type, value) over a protobuf message; value = int or bytes."""
    pos = 0
    while pos < len(buf):
        tag, pos = get_varint(buf, pos)
        fn, wt = tag >> 3, tag & 7
        if wt == 0:
            v, pos = get_varint(buf, pos)
        elif wt == 1:
            v = struct.unpack_from("<Q", buf, pos)[0]; pos += 8
        elif wt == 2:
            n, pos = get_varint(buf, pos)
            v = bytes(buf[pos:pos + n]); pos += n
        elif wt == 5:
            v = struct.unpack_from("<I", buf, pos)[0]; pos += 4
        else:
            raise CheckpointError("unsupported protobuf wire type %d" % wt)
        yield fn, wt, v


def decode_header(buf):
    h = {"num_shards": 0, "endianness": 0, "producer": 0}
    for fn, _, v in _fields(buf):
        if fn == 1: h["num_shards"] = v
        elif fn == 2: h["endianness"] = v
        elif fn == 3:
            for f2, _, v2 in _fields(v):
                if f2 == 1: h["producer"] = v2
    return h


def decode_entry(buf):
    e = {"dtype": 0, "shape": [], "shard_id": 0, "offset": 0, "size": 0, "crc32c": 0, "slices": 0}      # proto3 defaults
    for fn, _, v in _fields(buf):
        if fn == 1: e["dtype"] = v
        elif fn == 2:
            for f2, _, v2 in _fields(v):
                if f2 == 2:
                    size = 0
                    for f3, _, v3 in _fields(v2):
                        if f3 == 1: size = _signed64(v3)
                    e["shape"].append(size)
                elif f2 == 3 and v2:
                    raise CheckpointError("tensor of unknown rank in checkpoint")
        elif fn == 3: e["shard_id"] = v
        elif fn == 4: e["offset"] = v
        elif fn == 5: e["size"] = v
        elif fn == 6: e["crc32c"] = v
        elif fn == 7: e["slices"] += 1
    return e


# ------------------------------------------------------------------------------------------------
# table (LevelDB sstable) writer / reader
# ------------------------------------------------------------------------------------------------
class _BlockBuilder(object):
    def __init__(self):
        self.buf = bytearray()
        self.restarts = [0]
        self.count = 0
        self.last_key = b""

    def add(self, key, value):
        shared = 0
        if self.count % RESTART_INTERVAL == 0 and self.count:
            self.restarts.append(len(self.buf))
        elif self.count:
            n = min(len(key), len(self.last_key))
            while shared < n and key[shared] == self.last_key[shared]:
                shared += 1
        put_varint(self.buf, shared)
        put_varint(self.buf, len(key) - shared)
        put_varint(self.buf, len(value))
        self.buf += key[shared:]
        self.buf += value
        self.last_key = key
        self.count += 1

    def size_estimate(self):
        return len(self.buf) + 4 * len(self.restarts) + 4

    def finish(self):
        out = bytes(self.buf) + b"".join(struct.pack("<I", r) for r in self.restarts) + struct.pack("<I", len(self.restarts))
        return out


def _block_with_trailer(contents):
    trailer_type = b"\x00"                               # kNoCompression
    crc = wun.crc32c(trailer_type, wun.crc32c(contents))
    return contents + trailer_type + struct.pack("<I", mask_crc(crc))


def _handle(offset, size):
    out = bytearray()
    put_varint(out, offset)
    put_varint(out, size)
    return bytes(out)


def build_table(items, block_size=BLOCK_SIZE):
    """items: list of (key bytes, value bytes) in strictly increasing key order -> table file bytes."""
    out = bytearray()
    index = _BlockBuilder()
    blk = _BlockBuilder()
    prev = None

    def flush():
        nonlocal blk
        if blk.count == 0:
            return
        contents = blk.finish()
        index.add(blk.last_key, _handle(len(out), len(contents)))
        out.extend(_block_with_trailer(contents))
        blk = _BlockBuilder()

    for key, value in items:
        if prev is not None and not key > prev:
            raise CheckpointError("table keys must be strictly increasing")
        prev = key
        blk.add(key, value)
        if blk.size_estimate() >= block_size:
            flush()
    flush()
    meta = _BlockBuilder().finish()
    meta_handle = _handle(len(out), len(meta))
    out.extend(_block_with_trailer(meta))
    idx = index.finish()
    idx_handle = _handle(len(out), len(idx))
    out.extend(_block_with_trailer(idx))
    footer = meta_handle + idx_handle
    footer += b"\x00" * (40 - len(footer))
    footer += struct.pack("<Q", TABLE_MAGIC)
    out.extend(footer)
    return bytes(out)


def _read_block(data, offset, size, verify):
    if offset + size + 5 > len(data):
        raise CheckpointError("block handle outside the index file")
    contents = data[offset:offset + size]
    ctype = data[offset + size]
    if verify:
        stored = struct.unpack_from("<I", data, offset + size + 1)[0]
        if unmask_crc(stored) != wun.crc32c(data[offset:offset + size + 1]):
            raise CheckpointError("index block checksum mismatch at offset %d" % offset)
    if ctype != 0:
        raise CheckpointError("compressed index block (type %d): TensorFlow writes bundle indexes uncompressed; "
                              "snappy is not supported" % ctype)
    return contents


def _block_entries(contents):
    if len(contents) < 4:
        raise CheckpointError("bad block")
    nrestarts = struct.unpack_from("<I", contents, len(contents) - 4)[0]
    limit = len(contents) - 4 - 4 * nrestarts
    if limit < 0:
        raise CheckpointError("bad block restart array")
    pos = 0
    key = b""
    while pos < limit:
        shared, pos = get_varint(contents, pos)
        non_shared, pos = get_varint(contents, pos)
        vlen, pos = get_varint(contents, pos)
        if shared > len(key) or pos + non_shared + vlen > limit:
            raise CheckpointError("corrupt block entry")
        key = key[:shared] + bytes(contents[pos:pos + non_shared])
        pos += non_shared
        value = bytes(contents[pos:pos + vlen])
        pos += vlen
        yield key, value


def read_table(data, verify=True):
    """Table file bytes -> list of (key, value) in file order."""
    if len(data) < 48:
        raise CheckpointError("index file too short")
    footer = data[-48:]
    if struct.unpack("<Q", footer[40:])[0] != TABLE_MAGIC:
        raise CheckpointError("not a TensorFlow V2 checkpoint index (bad table magic)")
    pos = 0
    _, pos = get_varint(footer, pos)           # metaindex handle
    _, pos = get_varint(footer, pos)
    ioff, pos = get_varint(footer, pos)
    isize, pos = get_varint(footer, pos)
    items = []
    for _, handle in _block_entries(_read_block(data, ioff, isize, verify)):
        boff, p = get_varint(handle, 0)
        bsize, p = get_varint(handle, p)
        items.extend(_block_entries(_read_block(data, boff, bsize, verify)))
    return items


# ------------------------------------------------------------------------------------------------
# bundle level
# ------------------------------------------------------------------------------------------------
def _data_path(prefix, shard, num_shards):
    return "%s.data-%05d-of-%05d" % (prefix, shard, num_shards)


def list_variables(prefix):
    """[(name, numpy dtype, shape)] in key order (tf.train.list_variables)."""
    with open(prefix + ".index", "rb") as f:
        items = read_table(f.read())
    out = []
    for key, value in items:
        if key == b"":
            continue
        e = decode_entry(value)
        out.append((key.decode("utf-8"), _DT_TO_NP.get(e["dtype"]), tuple(e["shape"])))
    return out


def read_checkpoint(prefix, verify=True, names=None):
    """prefix -> OrderedDict name -> numpy array.  `names`: optional predicate / collection to select tensors."""
    if not os.path.exists(prefix + ".index"):
        raise CheckpointError("%s.index not found (a V2 checkpoint is named by its prefix, e.g. "
                              "checkpoints/123456/123456-2000)" % prefix)
    with open(prefix + ".index", "rb") as f:
        items = read_table(f.read(), verify)
    if not items or items[0][0] != b"":
        raise CheckpointError("checkpoint index has no header entry")
    header = decode_header(items[0][1])
    if header["endianness"] != 0:
        raise CheckpointError("big-endian checkpoint")
    num_shards = header["num_shards"]
    want = names if callable(names) or names is None else (lambda n, s=set(names): n in s)
    shards = {}
    out = OrderedDict()
    for key, value in items[1:]:
        name = key.decode("utf-8")
        if want is not None and not want(name):
            continue
        e = decode_entry(value)
        if e["slices"]:
            raise CheckpointError("%s is a partitioned (sliced) variable - not supported" % name)
        if e["dtype"] not in _DT_TO_NP:
            raise CheckpointError("%s: unsupported dtype enum %d" % (name, e["dtype"]))
        dt = np.dtype(_DT_TO_NP[e["dtype"]])
        count = int(np.prod(e["shape"], dtype=np.int64)) if e["shape"] else 1
        if count * dt.itemsize != e["size"]:
            raise CheckpointError("%s: size %d does not match shape %s" % (name, e["size"], e["shape"]))
        sid = e["shard_id"]
        if sid not in shards:
            path = _data_path(prefix, sid, num_shards)
            # (np.memmap refuses empty files - a bundle of empty tensors has a 0-byte data file)
            shards[sid] = np.memmap(path, dtype=np.uint8, mode="r") if os.path.getsize(path) > 0 else np.zeros(0, np.uint8)
        raw = shards[sid][e["offset"]:e["offset"] + e["size"]]
        if raw.size != e["size"]:
            raise CheckpointError("%s: data file truncated" % name)
        if verify and unmask_crc(e["crc32c"]) != wun.crc32c(np.asarray(raw)):
            raise CheckpointError("%s: tensor checksum mismatch" % name)
        out[name] = np.frombuffer(np.asarray(raw).tobytes(), dtype=dt.newbyteorder("<")).astype(dt).reshape(e["shape"])
    return out


def write_checkpoint(prefix, tensors, block_size=BLOCK_SIZE, update_state_file=True):
    """tensors: mapping name -> array-like.  Writes <prefix>.index, <prefix>.data-00000-of-00001 and (like Saver.save)
    the `checkpoint` state file next to them.  Returns prefix."""
    d = os.path.dirname(prefix)
    if d:
        os.makedirs(d, exist_ok=True)
    names = sorted(tensors.keys(), key=lambda n: n.encode("utf-8"))
    items = [(b"", encode_header(1))]
    offset = 0
    tmp = _data_path(prefix, 0, 1) + ".tmp"
    with open(tmp, "wb") as f:
        for name in names:
            if name == "":
                raise CheckpointError("empty tensor name")
            a = np.asarray(tensors[name])
            if np.dtype(a.dtype.type) not in _NP_TO_DT:
                raise CheckpointError("%s: dtype %s cannot be stored" % (name, a.dtype))
            shape = a.shape                                  # (np.ascontiguousarray would turn a scalar into shape (1,))
            a = np.ascontiguousarray(a.astype(a.dtype.newbyteorder("<"), copy=False))
            raw = a.view(np.uint8).reshape(-1) if a.size else np.zeros(0, np.uint8)
            f.write(raw.tobytes())
            items.append((name.encode("utf-8"),
                          encode_entry(_NP_TO_DT[np.dtype(a.dtype.type)], shape, offset, raw.size, mask_crc(wun.crc32c(raw)))))
            offset += raw.size
    os.replace(tmp, _data_path(prefix, 0, 1))
    with open(prefix + ".index.tmp", "wb") as f:
        f.write(build_table(items, block_size))
    os.replace(prefix + ".index.tmp", prefix + ".index")
    if update_state_file:
        base = os.path.basename(prefix)
        with open(os.path.join(d or ".", "checkpoint"), "w") as f:
            f.write('model_checkpoint_path: "%s"\nall_model_checkpoint_paths: "%s"\n' % (base, base))
    return prefix


def latest_checkpoint(directory):
    """tf.train.latest_checkpoint: the prefix named by <directory>/checkpoint, or None."""
    state = os.path.join(directory, "checkpoint")
    if not os.path.exists(state):
        return None
    for line in open(state):
        if line.startswith("model_checkpoint_path:"):
            p = line.split(":", 1)[1].strip().strip('"')
            return p if os.path.isabs(p) else os.path.join(directory, p)
    return None


# ------------------------------------------------------------------------------------------------
# the separator's variables <-> checkpoint tensors (Training.py:66-77,98)
# ------------------------------------------------------------------------------------------------
SOLVER_SCOPE = "separator_solver"


def separator_tensors(variables, adam_m=None, adam_v=None, global_step=0, beta1=0.9, beta2=0.999):
    """What Saver(tf.global_variables()) holds for the reference's training graph.
    variables / adam_m / adam_v: ordered mappings TF-name -> numpy array (m, v optional: inference-only checkpoint); the
    slots are written for the names adam_m holds (the trainable variables)."""
    out = OrderedDict()
    for n, a in variables.items():
        out[n] = np.asarray(a, dtype=np.float32)
    if adam_m is not None:
        for n in adam_m:
            out["%s/%s/Adam" % (SOLVER_SCOPE, n)] = np.asarray(adam_m[n], dtype=np.float32)
            out["%s/%s/Adam_1" % (SOLVER_SCOPE, n)] = np.asarray(adam_v[n], dtype=np.float32)
        # TF's Adam initialises the power accumulators to beta and multiplies once per applied step
        out[SOLVER_SCOPE + "/beta1_power"] = np.float32(beta1 ** (int(global_step) + 1))
        out[SOLVER_SCOPE + "/beta2_power"] = np.float32(beta2 ** (int(global_step) + 1))
    out["global_step"] = np.int64(global_step)
    return out


def split_separator_tensors(tensors, variable_names, slot_names=None):
    """Inverse of separator_tensors, tolerant to the optimizer's scope prefix: returns
    (variables, adam_m or None, adam_v or None, global_step).  slot_names: the variables that have Adam slots (default:
    every variable); m / v are None unless all of them have both."""
    variables = OrderedDict()
    missing = [n for n in variable_names if n not in tensors]
    if missing:
        raise CheckpointError("checkpoint lacks %d model variables, e.g. %s (has: %s ...)"
                              % (len(missing), missing[0], ", ".join(list(tensors)[:3])))
    for n in variable_names:
        variables[n] = tensors[n]

    def slot(n, suffix):
        for cand in ("%s/%s/%s" % (SOLVER_SCOPE, n, suffix), "%s/%s" % (n, suffix)):
            if cand in tensors:
                return tensors[cand]
        tail = "/%s/%s" % (n, suffix)
        hits = [k for k in tensors if k.endswith(tail)]
        return tensors[hits[0]] if len(hits) == 1 else None

    m, v = OrderedDict(), OrderedDict()
    for n in (variable_names if slot_names is None else slot_names):
        a, b = slot(n, "Adam"), slot(n, "Adam_1")
        if a is None or b is None:
            m = v = None
            break
        m[n], v[n] = a, b
    step = int(tensors["global_step"]) if "global_step" in tensors else 0
    return variables, m, v, step


# ------------------------------------------------------------------------------------------------
# Saver.save / Saver.restore for a UnetAudioSeparator facade (Training.py:92-98,113; Evaluate.py:55-57)
# ------------------------------------------------------------------------------------------------
def is_npz(path):
    """Round-1 legacy format: a numpy .npz with the same tensor names (flat Adam buffers)."""
    return path.endswith(".npz") or (not os.path.exists(path + ".index") and os.path.isfile(path))


def _slot_names(sep):
    """The variables with Adam slots: the separator's trainables when it tells them apart (the spectrogram U-Net's moving
    statistics are not trained), else every variable."""
    names = getattr(sep, "trainable_variable_names", None)
    return names() if names is not None else None


def save_separator(path, sep):
    """Write what the reference's `saver.save(sess, path, global_step)` writes; returns the checkpoint prefix."""
    table = sep.param_table()
    flat = sep.params.detach().cpu().numpy()
    slots = _slot_names(sep)
    per_var = lambda buf: OrderedDict((n, buf[o:o + c].reshape(s)) for n, s, o, c in table)
    per_slot = lambda buf: OrderedDict((n, buf[o:o + c].reshape(s)) for n, s, o, c in table if slots is None or n in slots)
    m = v = None
    if sep.adam_m is not None:
        m, v = per_slot(sep.adam_m.detach().cpu().numpy()), per_slot(sep.adam_v.detach().cpu().numpy())
    if path.endswith(".npz"):
        blob = dict(per_var(flat))
        if m is not None:
            blob["separator_solver/adam_m"] = sep.adam_m.detach().cpu().numpy()
            blob["separator_solver/adam_v"] = sep.adam_v.detach().cpu().numpy()
        blob["global_step"] = np.int64(sep.global_step)
        d = os.path.dirname(path)
        if d:
            os.makedirs(d, exist_ok=True)
        np.savez(path, **blob)
        return path
    return write_checkpoint(path, separator_tensors(per_var(flat), m, v, sep.global_step))


def restore_separator(path, sep, input_frames, with_optimizer=True):
    """`restorer.restore(sess, path)`: model variables always; Adam slots + global_step when present and wanted."""
    import torch
    names = [n for n, _, _, _ in sep.param_table(input_frames=input_frames)]
    if is_npz(path):
        ck = np.load(path)
        tensors = {k: ck[k] for k in ck.files}
        sep.load_variables({n: tensors[n] for n in names}, input_frames=input_frames)
        sep.global_step = int(tensors["global_step"]) if "global_step" in tensors else 0
        if with_optimizer and "separator_solver/adam_m" in tensors:
            sep._ensure_training_state()
            sep.adam_m.copy_(torch.from_numpy(tensors["separator_solver/adam_m"]))
            sep.adam_v.copy_(torch.from_numpy(tensors["separator_solver/adam_v"]))
        return sep
    tensors = read_checkpoint(path)
    variables, m, v, step = split_separator_tensors(tensors, names, _slot_names(sep))
    sep.load_variables(variables, input_frames=input_frames)          # asserts every shape against the plan
    sep.global_step = step
    if with_optimizer and m is not None:
        sep._ensure_training_state()
        table = sep.param_table()
        fm = np.zeros(sep.params.numel(), np.float32)
        fv = np.zeros(sep.params.numel(), np.float32)
        for n, s, o, c in table:
            if n not in m:
                continue
            if tuple(m[n].shape) != tuple(s) or tuple(v[n].shape) != tuple(s):
                raise CheckpointError("%s: Adam slot shape %s does not match the variable %s" % (n, m[n].shape, s))
            fm[o:o + c] = np.asarray(m[n], np.float32).reshape(-1)
            fv[o:o + c] = np.asarray(v[n], np.float32).reshape(-1)
        sep.adam_m.copy_(torch.from_numpy(fm))
        sep.adam_v.copy_(torch.from_numpy(fv))
    return sep
