"""Pure-Python reader (and minimal writer) for TensorFlow "tensor bundle" checkpoints
(``model.ckpt.index`` + ``model.ckpt.data-00000-of-00001``), so the reference's trained variables
(``tf.train.Saver`` files, test/create_sdf.py:180-192, README.md:31-37) can be loaded by name without TensorFlow:

    from disn_b200.tf_checkpoint import load_checkpoint
    weights = load_checkpoint("checkpoint/SDF_DISN/model.ckpt", prefixes=("vgg_16/", "sdfprediction"))
    engine.load_weights(weights)

Format (restated from TensorFlow's tensor_bundle / leveldb-table sources, which are not vendored in the
reference).  The authors' files are Dropbox downloads, so there is no TF-written bundle to pin against; the reader is
pinned instead by tests/tf_bundle_golden.py, which assembles a bundle byte by byte from the documented table layout
(prefix-compressed keys, 16-entry restart intervals, several data blocks, shortened index keys, crc32c known-answer
vectors from RFC 3720) WITHOUT using this module's writer, and by negative tests (snappy-flagged block, corrupted CRC,
truncated data shard).  Layout:
  * .index is an SSTable: data blocks of prefix-compressed (key, value) entries + restart array, a 5-byte block
    trailer (compression type, masked crc32c), an index block mapping last-keys to block handles, and a 48-byte
    footer (metaindex handle, index handle, padding, magic 0xdb4775248b80fb57);
  * key "" holds a BundleHeaderProto, every other key a BundleEntryProto
    {1: dtype, 2: shape{2: dim{1: size}}, 3: shard_id, 4: offset, 5: size, 6: crc32c};
  * .data-* files hold the raw little-endian tensor bytes.
"""
from __future__ import annotations

import os
import struct

import numpy as np

TABLE_MAGIC = 0xDB4775248B80FB57
DTYPES = {1: np.float32, 2: np.float64, 3: np.int32, 4: np.uint8, 6: np.int8, 9: np.int64, 10: np.bool_}
DTYPE_CODES = {np.dtype(v): k for k, v in DTYPES.items()}


def _varint(buf, pos):
    result = shift = 0
    while True:
        b = buf[pos]
        pos += 1
        result |= (b & 0x7F) << shift
        if not b & 0x80:
            return result, pos
        shift += 7


def _put_varint(v):
    out = bytearray()
    while True:
        b = v & 0x7F
        v >>= 7
        if v:
            out.append(b | 0x80)
        else:
            out.append(b)
            return bytes(out)


def _parse_proto(buf):
    """-> {field: [values]} with varints as int, length-delimited as bytes, fixed32/64 as int."""
    out, pos = {}, 0
    while pos < len(buf):
        tag, pos = _varint(buf, pos)
        field, wt = tag >> 3, tag & 7
        if wt == 0:
            v, pos = _varint(buf, pos)
        elif wt == 1:
            v = struct.unpack_from("<Q", buf, pos)[0]
            pos += 8
        elif wt == 2:
            n, pos = _varint(buf, pos)
            v = bytes(buf[pos:pos + n])
            pos += n
        elif wt == 5:
            v = struct.unpack_from("<I", buf, pos)[0]
            pos += 4
        else:
            raise ValueError("unsupported protobuf wire type %d" % wt)
        out.setdefault(field, []).append(v)
    return out


def _block_entries(block):
    """iterate (key, value) of one table block (contents without the 5-byte trailer)"""
    n_restarts = struct.unpack_from("<I", block, len(block) - 4)[0]
    limit = len(block) - 4 - 4 * n_restarts
    pos, key = 0, b""
    while pos < limit:
        shared, pos = _varint(block, pos)
        non_shared, pos = _varint(block, pos)
        vlen, pos = _varint(block, pos)
        key = key[:shared] + bytes(block[pos:pos + non_shared])
        pos += non_shared
        yield key, bytes(block[pos:pos + vlen])
        pos += vlen


def _read_block(data, offset, size, verify=True):
    if offset + size + 5 > len(data):
        raise ValueError("table block handle (%d, %d) points outside the file" % (offset, size))
    ctype = data[offset + size]
    if ctype != 0:
        raise NotImplementedError("compressed table blocks (type %d; 1 = snappy) are not supported; re-save the "
                                  "checkpoint uncompressed" % ctype)
    if verify:
        stored = struct.unpack_from("<I", data, offset + size + 1)[0]
        if stored != _masked_crc32c(data[offset:offset + size + 1]):
            raise ValueError("table block at offset %d fails its crc32c check (corrupt .index)" % offset)
    return data[offset:offset + size]


def read_index(index_path, with_header=False):
    """-> {tensor_name: dict(dtype, shape, shard_id, offset, size, crc32c)}; with_header=True -> (entries, header) where
    header = dict(num_shards, endianness, version) from the BundleHeaderProto stored under the empty key."""
    data = open(index_path, "rb").read()
    if len(data) < 48 or struct.unpack_from("<Q", data, len(data) - 8)[0] != TABLE_MAGIC:
        raise ValueError("%s is not a TensorFlow checkpoint index (bad table magic)" % index_path)
    footer = data[-48:]
    pos = 0
    _, pos = _varint(footer, pos)          # metaindex offset
    _, pos = _varint(footer, pos)          # metaindex size
    ioff, pos = _varint(footer, pos)
    isize, pos = _varint(footer, pos)
    entries = {}
    header = dict(num_shards=1, endianness=0, version=None)
    for _, handle in _block_entries(_read_block(data, ioff, isize)):
        boff, p = _varint(handle, 0)
        bsize, p = _varint(handle, p)
        for key, value in _block_entries(_read_block(data, boff, bsize)):
            if key == b"":                  # BundleHeaderProto {1: num_shards, 2: endianness, 3: version{1: producer}}
                h = _parse_proto(value)
                header["num_shards"] = h.get(1, [1])[0]
                header["endianness"] = h.get(2, [0])[0]
                if 3 in h:
                    header["version"] = _parse_proto(h[3][0]).get(1, [0])[0]
                if header["endianness"] != 0:
                    raise NotImplementedError("big-endian tensor bundles are not supported")
                continue
            e = _parse_proto(value)
            shape = []
            if 2 in e:
                for dim in _parse_proto(e[2][0]).get(2, []):
                    shape.append(_parse_proto(dim).get(1, [0])[0])
            entries[key.decode()] = dict(dtype=e.get(1, [0])[0], shape=tuple(shape), shard_id=e.get(3, [0])[0],
                                         offset=e.get(4, [0])[0], size=e.get(5, [0])[0], crc32c=e.get(6, [None])[0],
                                         sliced=7 in e)
    return (entries, header) if with_header else entries


# optimizer slots / moving averages / step counters a tf.train.Saver checkpoint carries next to the model variables
_SLOT_SUFFIXES = ("/Adam", "/Adam_1", "/Momentum", "/ExponentialMovingAverage", "/RMSProp", "/RMSProp_1")
_BOOKKEEPING = ("global_step", "beta1_power", "beta2_power")


def is_model_variable(name: str) -> bool:
    return not name.endswith(_SLOT_SUFFIXES) and name.split("/")[-1] not in _BOOKKEEPING


def load_checkpoint(prefix, prefixes=None, model_variables_only=True, verify_data=False):
    """Read the variables (optionally only names starting with one of `prefixes`) as numpy arrays.
    model_variables_only drops optimizer slots (`.../Adam`, `.../Adam_1`, ...) and step counters, which would otherwise
    triple the upload; verify_data=True checks every tensor's crc32c (pure Python: slow for the 554 MB of VGG-16)."""
    index, header = read_index(prefix + ".index", with_header=True)
    shards = {}
    out = {}
    num_shards = header["num_shards"]
    for name, e in index.items():
        if prefixes and not name.startswith(tuple(prefixes)):
            continue
        if model_variables_only and not is_model_variable(name):
            continue
        if e["dtype"] not in DTYPES:
            continue                        # non-numeric bookkeeping entries
        if e["sliced"]:
            raise NotImplementedError("%s is stored as slices (partitioned variable); not supported" % name)
        sid = e["shard_id"]
        if sid >= num_shards:
            raise ValueError("%s refers to shard %d of %d" % (name, sid, num_shards))
        if sid not in shards:
            shards[sid] = np.memmap("%s.data-%05d-of-%05d" % (prefix, sid, num_shards), dtype=np.uint8, mode="r")
        if e["offset"] + e["size"] > shards[sid].size:
            raise ValueError("%s: data shard %d is truncated (%d + %d > %d bytes)" % (name, sid, e["offset"], e["size"],
                                                                                    shards[sid].size))
        want = int(np.prod(e["shape"], dtype=np.int64)) * np.dtype(DTYPES[e["dtype"]]).itemsize
        if want != e["size"]:
            raise ValueError("%s: %d bytes stored for shape %s" % (name, e["size"], e["shape"]))
        raw = np.asarray(shards[sid][e["offset"]:e["offset"] + e["size"]])
        if verify_data and e["crc32c"] is not None and _masked_crc32c(raw.tobytes()) != e["crc32c"]:
            raise ValueError("%s fails its crc32c check (corrupt data shard)" % name)
        out[name] = raw.view(DTYPES[e["dtype"]]).reshape(e["shape"]).copy()
    return out


# ---------------------------------------------------------------------------------------------------------
# minimal writer (single data block per 4 KB, no compression) -- used by the tests and for exporting synthetic weights
# ---------------------------------------------------------------------------------------------------------
def _crc32c_table():
    tbl = []
    for i in range(256):
        c = i
        for _ in range(8):
            c = (c >> 1) ^ 0x82F63B78 if c & 1 else c >> 1
        tbl.append(c)
    return tbl


_CRC_TBL = _crc32c_table()


_CRC_NP = np.array(_CRC_TBL, np.uint32)
_CRC_LANE = 4096            # bytes per lane of the vectorised CRC


def _crc_op_tables(cols):
    """The four byte tables of the GF(2)-linear map whose images of the 32 unit vectors are cols."""
    t = np.zeros((4, 256), np.uint32)
    b = np.arange(256)
    for k in range(4):
        for bit in range(8):
            t[k][(b >> bit) & 1 == 1] ^= cols[8 * k + bit]
    return t


def _crc_apply(t, x):
    x = np.asarray(x, np.uint32)
    return t[0][x & 255] ^ t[1][(x >> 8) & 255] ^ t[2][(x >> 16) & 255] ^ t[3][x >> 24]


def _crc_zeros_op(nbytes):
    """Byte tables of the map that advances the CRC register over nbytes zero bytes (by squaring one zero byte)."""
    cols = np.array([1 << i for i in range(32)], np.uint32)
    one = _CRC_NP[cols & 255] ^ (cols >> 8)                 # one zero byte
    result = None
    step = _crc_op_tables(one)
    n = nbytes
    while n:
        if n & 1:
            result = step if result is None else _crc_op_tables(_crc_apply(step, _crc_apply_cols(result)))
        n >>= 1
        if n:
            step = _crc_op_tables(_crc_apply(step, _crc_apply_cols(step)))
    return result


def _crc_apply_cols(t):
    return _crc_apply(t, np.array([1 << i for i in range(32)], np.uint32))


def crc32c(data) -> int:
    """CRC-32C (Castagnoli, reflected polynomial 0x82F63B78), as in RFC 3720 appendix B.4.  Large inputs run as
    parallel lanes of 4 KB (numpy) whose registers are combined with the GF(2)-linear zero-advance maps; the result is
    the byte-serial definition's."""
    buf = np.frombuffer(bytes(data), np.uint8)
    n = buf.size
    if n < 4 * _CRC_LANE:
        c = 0xFFFFFFFF
        for b in buf.tobytes():
            c = _CRC_TBL[(c ^ b) & 0xFF] ^ (c >> 8)
        return c ^ 0xFFFFFFFF
    # register form: crc = ~(Z^n ~0 ^ R(data)) with R the register from 0; leading zero bytes leave R unchanged, so the
    # data is front-padded to whole lanes, each lane's R is formed in parallel and R = sum_i Z^(L (K-1-i)) R_i
    lanes = -(-n // _CRC_LANE)
    k = 1 << (lanes - 1).bit_length()
    padded = np.zeros(k * _CRC_LANE, np.uint8)
    padded[k * _CRC_LANE - n:] = buf
    m = np.ascontiguousarray(padded.reshape(k, _CRC_LANE).T)      # m[j] = byte j of every lane
    r = np.zeros(k, np.uint32)
    for j in range(_CRC_LANE):
        r = _CRC_NP[(r ^ m[j]) & 255] ^ (r >> 8)
    op = _crc_zeros_op(_CRC_LANE)
    while r.size > 1:
        r = _crc_apply(op, r[0::2]) ^ r[1::2]
        op = _crc_op_tables(_crc_apply(op, _crc_apply_cols(op)))
    init = int(_crc_apply(_crc_zeros_op(n), np.uint32(0xFFFFFFFF)))
    return (init ^ int(r[0])) ^ 0xFFFFFFFF


def _masked_crc32c(data):
    """leveldb / TensorFlow store crcs "masked": rotate right by 15 bits and add a constant."""
    c = crc32c(data)
    return (((c >> 15) | (c << 17)) + 0xA282EAD8) & 0xFFFFFFFF


def _field(num, wt, payload):
    return _put_varint((num << 3) | wt) + payload


def _entry_proto(dtype, shape, offset, size, crc=None):
    dims = b"".join(_field(2, 2, _put_varint(len(d)) + d) for d in (_field(1, 0, _put_varint(s)) for s in shape))
    out = (_field(1, 0, _put_varint(dtype)) + _field(2, 2, _put_varint(len(dims)) + dims) +
           _field(4, 0, _put_varint(offset)) + _field(5, 0, _put_varint(size)))
    if crc is not None:
        out += _field(6, 5, struct.pack("<I", crc))     # fixed32 crc32c (masked)
    return out


def _build_block_multi(items):
    body, restarts = bytearray(), []
    for k, v in items:
        restarts.append(len(body))
        body += _put_varint(0) + _put_varint(len(k)) + _put_varint(len(v)) + k + v
    return bytes(body) + b"".join(struct.pack("<I", r) for r in restarts) + struct.pack("<I", len(restarts))


def save_checkpoint(prefix, tensors):
    """Write {name: array} as <prefix>.index + <prefix>.data-00000-of-00001 (uncompressed, one shard)."""
    os.makedirs(os.path.dirname(os.path.abspath(prefix)), exist_ok=True)
    items = [(b"", _field(1, 0, _put_varint(1)) + _field(3, 2, _put_varint(2) + _field(1, 0, _put_varint(1))))]
    offset = 0
    with open(prefix + ".data-00000-of-00001", "wb") as f:
        for name in sorted(tensors):
            a = np.ascontiguousarray(tensors[name])
            raw = a.tobytes()
            f.write(raw)
            items.append((name.encode(), _entry_proto(DTYPE_CODES[a.dtype], a.shape, offset, len(raw), _masked_crc32c(raw))))
            offset += len(raw)
    out = bytearray()
    index_items = []
    chunk, chunk_bytes = [], 0
    def flush():
        nonlocal chunk, chunk_bytes
        if not chunk:
            return
        blk = _build_block_multi(chunk)
        index_items.append((chunk[-1][0], _put_varint(len(out)) + _put_varint(len(blk))))
        out.extend(blk + b"\x00" + struct.pack("<I", _masked_crc32c(blk + b"\x00")))
        chunk, chunk_bytes = [], 0
    for kv in items:
        chunk.append(kv)
        chunk_bytes += len(kv[0]) + len(kv[1])
        if chunk_bytes > 4096:
            flush()
    flush()
    meta = _build_block_multi([])
    meta_handle = _put_varint(len(out)) + _put_varint(len(meta))
    out.extend(meta + b"\x00" + struct.pack("<I", _masked_crc32c(meta + b"\x00")))
    idx = _build_block_multi(index_items)
    idx_handle = _put_varint(len(out)) + _put_varint(len(idx))
    out.extend(idx + b"\x00" + struct.pack("<I", _masked_crc32c(idx + b"\x00")))
    footer = meta_handle + idx_handle
    footer += b"\x00" * (40 - len(footer)) + struct.pack("<Q", TABLE_MAGIC)
    out.extend(footer)
    with open(prefix + ".index", "wb") as f:
        f.write(bytes(out))
