"""Stand-alone reader / writer for TensorFlow "V2" checkpoint bundles (prefix.index + prefix.data-00000-of-00001),
the format of the reference's released snapshots (results*/Log_*/snapshots/snap-N.*), without TensorFlow.

The reference restores its variables with tf.train.Saver (utils/tester.py:60-75); here the same bytes feed ParamStore:

    params = load_params("/path/to/snapshots/snap-61")      # {'layer_0/simple_0/weights': ndarray, ...}
    enc = KPFCNN(config, params, limits)

Format (public, tensorflow/core/util/tensor_bundle + the leveldb table format it embeds):
  * .index is an immutable sorted string table: data blocks of prefix-compressed (key, value) entries with a restart
    array, an index block mapping last-keys to block handles, and a 48-byte footer (metaindex handle, index handle,
    padding, magic 0xdb4775248b80fb57). Every block is followed by a 1-byte compression tag and a masked crc32c.
  * key ""  -> BundleHeaderProto {num_shards, endianness, version}
  * key var -> BundleEntryProto  {dtype=1, shape=2, shard_id=3, offset=4, size=5, crc32c=6}
  * .data-SSSSS-of-NNNNN holds the raw little-endian tensor bytes at [offset, offset+size).
The writer emits single-block-per-entry-group tables that TensorFlow's own reader accepts (uncompressed blocks, valid
crc32c) -- it exists so that round-trip tests and synthetic fixtures need no TensorFlow either.
"""
import os
import struct

import numpy as np

_MAGIC = 0xdb4775248b80fb57
_FOOTER = 48

# tensorflow/core/framework/types.proto
_DTYPES = {1: np.float32, 2: np.float64, 3: np.int32, 4: np.uint8, 5: np.int16, 6: np.int8, 9: np.int64,
           10: np.bool_, 17: np.uint16, 19: np.float16, 22: np.uint32, 23: np.uint64}
_DTYPE_IDS = {np.dtype(v): k for k, v in _DTYPES.items()}

MODEL_SCOPE = "KernelPointNetwork/"          # models/KPFCNN_model.py: with tf.variable_scope('KernelPointNetwork')
_OPTIMIZER_SLOTS = ("/Momentum", "/Adam", "/Adam_1", "/ExponentialMovingAverage")


class CheckpointError(RuntimeError):
    pass


# ---------------------------------------------------------------------------------------------------- crc32c

def _make_crc_table():
    poly = 0x82F63B78
    tab = np.zeros(256, np.uint32)
    for i in range(256):
        c = i
        for _ in range(8):
            c = (c >> 1) ^ poly if c & 1 else c >> 1
        tab[i] = c
    return tab


_CRC_TABLE = _make_crc_table()


_CHUNK = 4096
_SHIFT = []                                 # byte tables of "feed _CHUNK zero bytes", built on first use


def _shift_tables():
    """T[i][v]: the register after _CHUNK zero bytes from register v << 8i. The map is linear over GF(2), so the
    register r goes to T[0][r & 255] ^ T[1][r >> 8 & 255] ^ T[2][r >> 16 & 255] ^ T[3][r >> 24]."""
    if not _SHIFT:
        r = (np.arange(256, dtype=np.uint32)[None, :] << (8 * np.arange(4, dtype=np.uint32))[:, None]).reshape(-1)
        for _ in range(_CHUNK):
            r = _CRC_TABLE[r & 0xFF] ^ (r >> 8)
        _SHIFT.extend(int(x) for x in r)
    return _SHIFT


def _crc_register_chunked(c, data):
    """The register after `data` (a multiple of _CHUNK bytes) from register c: every chunk's register from 0 at once
    (one table step per byte position, across all chunks), then chained: r = shift(r) ^ chunk register."""
    rows = np.frombuffer(data, np.uint8).reshape(-1, _CHUNK)
    z = np.zeros(rows.shape[0], np.uint32)
    for j in range(_CHUNK):
        z = _CRC_TABLE[(z ^ rows[:, j]) & 0xFF] ^ (z >> 8)
    T = _shift_tables()
    for v in z.tolist():
        c = T[c & 0xFF] ^ T[256 + (c >> 8 & 0xFF)] ^ T[512 + (c >> 16 & 0xFF)] ^ T[768 + (c >> 24)] ^ v
    return c


def crc32c(data, crc=0):
    """Castagnoli CRC. Table driven, byte-serial below 64 KiB; longer inputs go through _CHUNK-byte chunks whose
    registers are computed side by side in numpy and then chained (the same value, at numpy speed)."""
    tab = _CRC_TABLE
    c = (~crc) & 0xFFFFFFFF
    data = bytes(data)
    head = len(data) - len(data) % _CHUNK if len(data) >= 1 << 16 else 0
    if head:
        c = _crc_register_chunked(c, data[:head])
    for b in data[head:]:
        c = int(tab[(c ^ b) & 0xFF]) ^ (c >> 8)
    return (~c) & 0xFFFFFFFF


def _mask(crc):
    return ((((crc >> 15) | (crc << 17)) & 0xFFFFFFFF) + 0xa282ead8) & 0xFFFFFFFF


# ---------------------------------------------------------------------------------------------------- varints / protos

def _varint(buf, pos):
    out = 0
    shift = 0
    while True:
        if pos >= len(buf):
            raise CheckpointError("truncated varint")
        b = buf[pos]
        pos += 1
        out |= (b & 0x7F) << shift
        if not b & 0x80:
            return out, pos
        shift += 7
        if shift > 63:
            raise CheckpointError("varint too long")


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


def _proto_fields(buf):
    """Yields (field number, wire type, value) of one protobuf message (no schema needed for the two messages used)."""
    pos = 0
    while pos < len(buf):
        tag, pos = _varint(buf, pos)
        field, wire = tag >> 3, tag & 7
        if wire == 0:
            val, pos = _varint(buf, pos)
        elif wire == 1:
            val = struct.unpack_from("<Q", buf, pos)[0]
            pos += 8
        elif wire == 2:
            n, pos = _varint(buf, pos)
            val = bytes(buf[pos:pos + n])
            pos += n
        elif wire == 5:
            val = struct.unpack_from("<I", buf, pos)[0]
            pos += 4
        else:
            raise CheckpointError("unsupported protobuf wire type %d" % wire)
        yield field, wire, val


def _parse_shape(buf):
    dims = []
    for field, _, val in _proto_fields(buf):
        if field == 2:                      # TensorShapeProto.dim
            size = 0
            for f2, _, v2 in _proto_fields(val):
                if f2 == 1:
                    size = v2 - (1 << 64) if v2 >= (1 << 63) else v2
            dims.append(size)
    return tuple(dims)


def _parse_entry(buf):
    e = dict(dtype=0, shape=(), shard_id=0, offset=0, size=0, crc32c=None, sliced=False)
    for field, _, val in _proto_fields(buf):
        if field == 1:
            e["dtype"] = val
        elif field == 2:
            e["shape"] = _parse_shape(val)
        elif field == 3:
            e["shard_id"] = val
        elif field == 4:
            e["offset"] = val
        elif field == 5:
            e["size"] = val
        elif field == 6:
            e["crc32c"] = val
        elif field == 7:
            e["sliced"] = True
    return e


# ---------------------------------------------------------------------------------------------------- table reader

def _read_block(buf, offset, size, verify):
    if offset + size + 5 > len(buf):
        raise CheckpointError("block handle outside the index file")
    block = buf[offset:offset + size]
    ctype = buf[offset + size]
    if ctype != 0:
        raise CheckpointError("compressed index blocks (type %d) are not supported" % ctype)
    if verify:
        want = struct.unpack_from("<I", buf, offset + size + 1)[0]
        if _mask(crc32c(buf[offset:offset + size + 1])) != want:
            raise CheckpointError("index block checksum mismatch at offset %d" % offset)
    return block


def _block_entries(block):
    if len(block) < 4:
        raise CheckpointError("block too short")
    n_restarts = struct.unpack_from("<I", block, len(block) - 4)[0]
    end = len(block) - 4 - 4 * n_restarts
    if end < 0:
        raise CheckpointError("bad restart array")
    pos = 0
    key = b""
    while pos < end:
        shared, pos = _varint(block, pos)
        non_shared, pos = _varint(block, pos)
        vlen, pos = _varint(block, pos)
        key = key[:shared] + bytes(block[pos:pos + non_shared])
        pos += non_shared
        yield key, bytes(block[pos:pos + vlen])
        pos += vlen


def read_index(prefix, verify=True):
    """-> (header dict, {name: entry dict}) of prefix.index."""
    path = prefix + ".index"
    with open(path, "rb") as fh:
        buf = fh.read()
    if len(buf) < _FOOTER or struct.unpack_from("<Q", buf, len(buf) - 8)[0] != _MAGIC:
        raise CheckpointError("%s is not a tensor-bundle index (bad magic)" % path)
    foot = buf[len(buf) - _FOOTER:]
    pos = 0
    _, pos = _varint(foot, pos)             # metaindex handle (unused by bundles)
    _, pos = _varint(foot, pos)
    idx_off, pos = _varint(foot, pos)
    idx_size, pos = _varint(foot, pos)
    entries = {}
    header = None
    for _, handle in _block_entries(_read_block(buf, idx_off, idx_size, verify)):
        off, p = _varint(handle, 0)
        size, _ = _varint(handle, p)
        for key, val in _block_entries(_read_block(buf, off, size, verify)):
            if key == b"":
                header = {f: v for f, _, v in _proto_fields(val) if f in (1, 2)}
                header = dict(num_shards=header.get(1, 1), endianness=header.get(2, 0))
            else:
                entries[key.decode("utf-8")] = _parse_entry(val)
    if header is None:
        raise CheckpointError("%s has no bundle header" % path)
    if header["endianness"] != 0:
        raise CheckpointError("big-endian bundles are not supported")
    return header, entries


def read_checkpoint(prefix, names=None, verify_crc_below=1 << 16):
    """All (or the named) tensors of a bundle as numpy arrays. Tensor payload checksums are verified for tensors
    smaller than verify_crc_below bytes (the pure-Python CRC is byte-serial); index blocks always are."""
    header, entries = read_index(prefix)
    shards = {}
    out = {}
    for name, e in entries.items():
        if names is not None and name not in names:
            continue
        if e["sliced"]:
            raise CheckpointError("%s: partitioned variables are not supported" % name)
        if e["dtype"] not in _DTYPES:
            raise CheckpointError("%s: unsupported dtype enum %d" % (name, e["dtype"]))
        sid = e["shard_id"]
        if sid not in shards:
            shards[sid] = np.memmap("%s.data-%05d-of-%05d" % (prefix, sid, header["num_shards"]), dtype=np.uint8,
                                    mode="r")
        raw = shards[sid][e["offset"]:e["offset"] + e["size"]]
        dt = np.dtype(_DTYPES[e["dtype"]])
        count = int(np.prod(e["shape"], dtype=np.int64)) if e["shape"] else 1
        if raw.size != count * dt.itemsize:
            raise CheckpointError("%s: %d bytes on disk, shape %s needs %d" % (name, raw.size, e["shape"],
                                                                               count * dt.itemsize))
        if e["crc32c"] is not None and raw.size < verify_crc_below:
            if _mask(crc32c(raw.tobytes())) != e["crc32c"]:
                raise CheckpointError("%s: tensor checksum mismatch" % name)
        out[name] = np.frombuffer(raw.tobytes(), dtype=dt).reshape(e["shape"]).copy()
    if names is not None:
        missing = [n for n in names if n not in out]
        if missing:
            raise CheckpointError("not in checkpoint: %s" % ", ".join(missing))
    return out


def load_params(prefix, scope=MODEL_SCOPE):
    """Model variables of a reference snapshot keyed the way ParamStore / variable_scope look them up:
    '<layer scope>/<block>/<variable>' with the model scope stripped and optimizer slots / counters dropped."""
    out = {}
    for name, arr in read_checkpoint(prefix).items():
        if not name.startswith(scope) or name.endswith(_OPTIMIZER_SLOTS):
            continue
        out[name[len(scope):]] = arr
    if not out:
        raise CheckpointError("no variables under scope '%s' in %s" % (scope, prefix))
    return out


# ---------------------------------------------------------------------------------------------------- writer

def _block(entries, restart_interval=16):
    body = bytearray()
    restarts = []
    last = b""
    for i, (key, val) in enumerate(entries):
        if i % restart_interval == 0:
            restarts.append(len(body))
            shared = 0
        else:
            shared = 0
            while shared < min(len(last), len(key)) and last[shared] == key[shared]:
                shared += 1
        body += _put_varint(shared) + _put_varint(len(key) - shared) + _put_varint(len(val))
        body += key[shared:] + val
        last = key
    if not restarts:
        restarts = [0]
    for r in restarts:
        body += struct.pack("<I", r)
    body += struct.pack("<I", len(restarts))
    return bytes(body)


def _emit_block(fh, block):
    off = fh.tell()
    fh.write(block)
    fh.write(b"\x00")
    fh.write(struct.pack("<I", _mask(crc32c(block + b"\x00"))))
    return _put_varint(off) + _put_varint(len(block))


def _shape_proto(shape):
    out = bytearray()
    for d in shape:
        dim = b"\x08" + _put_varint(int(d))
        out += b"\x12" + _put_varint(len(dim)) + dim
    return bytes(out)


def write_checkpoint(prefix, tensors, block_entries=64):
    """Writes {name: ndarray} as a single-shard V2 bundle."""
    os.makedirs(os.path.dirname(os.path.abspath(prefix)), exist_ok=True)
    items = []
    with open(prefix + ".data-00000-of-00001", "wb") as data:
        for name in sorted(tensors, key=lambda s: s.encode("utf-8")):
            arr = np.asarray(tensors[name])
            arr = arr if arr.ndim == 0 else np.ascontiguousarray(arr)
            if arr.dtype not in _DTYPE_IDS:
                raise CheckpointError("%s: dtype %s cannot be stored" % (name, arr.dtype))
            raw = arr.astype(arr.dtype.newbyteorder("<"), copy=False).tobytes()
            off = data.tell()
            data.write(raw)
            shape = _shape_proto(arr.shape)
            entry = b"\x08" + _put_varint(_DTYPE_IDS[arr.dtype]) + b"\x12" + _put_varint(len(shape)) + shape
            if off:
                entry += b"\x20" + _put_varint(off)
            entry += b"\x28" + _put_varint(len(raw)) + b"\x35" + struct.pack("<I", _mask(crc32c(raw)))
            items.append((name.encode("utf-8"), entry))
    header = b"\x08\x01" + b"\x1a\x02\x08\x01"          # num_shards = 1, version { producer: 1 }
    items = [(b"", header)] + items
    with open(prefix + ".index", "wb") as fh:
        index = []
        for i in range(0, len(items), block_entries):
            chunk = items[i:i + block_entries]
            handle = _emit_block(fh, _block(chunk))
            index.append((chunk[-1][0], handle))
        meta_handle = _emit_block(fh, _block([]))
        index_handle = _emit_block(fh, _block(index, restart_interval=1))
        foot = meta_handle + index_handle
        fh.write(foot + b"\x00" * (40 - len(foot)) + struct.pack("<Q", _MAGIC))


# ---------------------------------------------------------------------------------------------------- optimizer slots

MOMENTUM_SLOT = "/Momentum"                 # tf.train.MomentumOptimizer's slot: '<variable>/Momentum'


def write_slots(prefix, slots, extra=None):
    """Writes the momentum accumulators {store name: ndarray} as a bundle, each under MODEL_SCOPE + name + '/Momentum'
    (the name TF gives the slot), plus the `extra` {name: ndarray} entries as they are (names outside MODEL_SCOPE)."""
    tensors = {MODEL_SCOPE + n + MOMENTUM_SLOT: np.asarray(a) for n, a in slots.items()}
    for n, a in (extra or {}).items():
        if n.startswith(MODEL_SCOPE):
            raise CheckpointError("%s: extra entries must lie outside %s" % (n, MODEL_SCOPE))
        tensors[n] = np.asarray(a)
    write_checkpoint(prefix, tensors)


def read_slots(prefix):
    """The two halves write_slots wrote: ({store name: momentum accumulator}, {other name: ndarray})."""
    slots, extra = {}, {}
    for name, arr in read_checkpoint(prefix).items():
        if name.startswith(MODEL_SCOPE) and name.endswith(MOMENTUM_SLOT):
            slots[name[len(MODEL_SCOPE):-len(MOMENTUM_SLOT)]] = arr
        else:
            extra[name] = arr
    return slots, extra
