"""Reading (and writing) TensorFlow "tensor bundle" checkpoints without TensorFlow, and mapping their keys onto the
parameter names of this package -- SURVEY.md section 8(f) rank 3: the reference publishes its trained weights as TF
object-graph checkpoints (`README.md:61-104`, `train_chairs.py:100-119`), `model.load_params` wants
`{'fnet.conv1.kernel': array, ...}` (SURVEY Appendix B).

Format (tensorflow/core/util/tensor_bundle, tensorflow/core/lib/io/table*):
  <prefix>.index                 an SSTable (LevelDB table format, uncompressed blocks): key -> BundleEntryProto,
                                 key "" -> BundleHeaderProto
  <prefix>.data-00000-of-00001   raw little-endian tensor bytes, addressed by (offset, size) of the entry
Object-graph checkpoints name a variable `<attribute path>/.ATTRIBUTES/VARIABLE_VALUE`; children of a keras
`Sequential` appear as `layer_with_weights-N` (N counts only the layers that own weights).

PARITY NOTE: TensorFlow is not installable in this environment, so neither the reader nor the key mapping has been run
against a file written by TensorFlow itself; `tests/test_checkpoint.py` pins the reader on an index assembled byte by byte
from the format description (independent CRC, prefix compression, several restart points, two data blocks), checks that the
writer below produces exactly such bytes, round-trips files through both, and checks the key mapping on the reference's
attribute tree.
"""
import os
import struct

import numpy as np

_MAGIC = 0xdb4775248b80fb57
_SUFFIX = '/.ATTRIBUTES/VARIABLE_VALUE'
# tensorflow/core/framework/types.proto
_DTYPES = {1: np.float32, 2: np.float64, 3: np.int32, 4: np.uint8, 5: np.int16, 6: np.int8, 9: np.int64, 10: np.bool_,
           17: np.uint16, 19: np.float16, 22: np.uint32, 23: np.uint64}
_DTYPE_IDS = {np.dtype(v): k for k, v in _DTYPES.items()}


# ---- crc32c (Castagnoli), masked as LevelDB / TensorFlow store it -----------------------------------------------------
def _make_table():
    tab = []
    for i in range(256):
        c = i
        for _ in range(8):
            c = (c >> 1) ^ 0x82F63B78 if c & 1 else c >> 1
        tab.append(c)
    return tab


_CRC_TABLE = _make_table()


def crc32c(data, crc=0):
    crc ^= 0xFFFFFFFF
    tab = _CRC_TABLE
    for b in bytes(data):
        crc = tab[(crc ^ b) & 0xFF] ^ (crc >> 8)
    return crc ^ 0xFFFFFFFF


def _mask(crc):
    return ((((crc >> 15) | (crc << 17)) & 0xFFFFFFFF) + 0xa282ead8) & 0xFFFFFFFF


# ---- varints and the few protobuf messages involved -------------------------------------------------------------------
def _get_varint(buf, pos):
    shift = result = 0
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


def _parse_fields(buf):
    """Protobuf wire format -> list of (field number, wire type, value)."""
    pos, out = 0, []
    while pos < len(buf):
        tag, pos = _get_varint(buf, pos)
        field, wt = tag >> 3, tag & 7
        if wt == 0:
            v, pos = _get_varint(buf, pos)
        elif wt == 1:
            v = buf[pos:pos + 8]
            pos += 8
        elif wt == 2:
            n, pos = _get_varint(buf, pos)
            v = buf[pos:pos + n]
            pos += n
        elif wt == 5:
            v = buf[pos:pos + 4]
            pos += 4
        else:
            raise ValueError(f'unsupported protobuf wire type {wt}')
        out.append((field, wt, v))
    return out


def _parse_entry(buf):
    """BundleEntryProto: dtype=1, shape=2 (TensorShapeProto: dim=2 {size=1}), shard_id=3, offset=4, size=5, crc32c=6."""
    e = {'dtype': 0, 'shape': [], 'shard_id': 0, 'offset': 0, 'size': 0, 'crc32c': None, 'sliced': False}
    for field, _, v in _parse_fields(buf):
        if field == 1:
            e['dtype'] = v
        elif field == 2:
            for f2, _, dim in _parse_fields(v):
                if f2 == 2:
                    size = 0
                    for f3, _, x in _parse_fields(dim):
                        if f3 == 1:
                            size = x
                    e['shape'].append(size)
        elif field == 3:
            e['shard_id'] = v
        elif field == 4:
            e['offset'] = v
        elif field == 5:
            e['size'] = v
        elif field == 6:
            e['crc32c'] = struct.unpack('<I', v)[0]
        elif field == 7:
            e['sliced'] = True
    return e


def _field(num, wt, payload):
    return _put_varint(num << 3 | wt) + payload


def _encode_entry(dtype_id, shape, offset, size, crc):
    dims = b''.join(_field(2, 2, _put_varint(len(d)) + d) for d in (_field(1, 0, _put_varint(s)) for s in shape))
    msg = _field(1, 0, _put_varint(dtype_id)) + _field(2, 2, _put_varint(len(dims)) + dims)
    if offset:
        msg += _field(4, 0, _put_varint(offset))
    msg += _field(5, 0, _put_varint(size)) + _field(6, 5, struct.pack('<I', crc))
    return msg


# ---- SSTable -------------------------------------------------------------------------------------------------------
def _read_block(buf, offset, size, verify):
    data = buf[offset:offset + size]
    ctype = buf[offset + size]
    if ctype != 0:
        raise ValueError('compressed table blocks are not supported (TensorFlow writes bundle indices uncompressed)')
    if verify:
        stored = struct.unpack('<I', buf[offset + size + 1:offset + size + 5])[0]
        if _mask(crc32c(buf[offset:offset + size + 1])) != stored:
            raise ValueError('checkpoint index: block checksum mismatch')
    return data


def _block_entries(block):
    n_restarts = struct.unpack('<I', block[-4:])[0]
    end = len(block) - 4 - 4 * n_restarts
    pos, key = 0, b''
    while pos < end:
        shared, pos = _get_varint(block, pos)
        non_shared, pos = _get_varint(block, pos)
        vlen, pos = _get_varint(block, pos)
        key = key[:shared] + block[pos:pos + non_shared]
        pos += non_shared
        yield key, block[pos:pos + vlen]
        pos += vlen


def _read_table(buf, verify=True):
    if len(buf) < 48 or struct.unpack('<Q', buf[-8:])[0] != _MAGIC:
        raise ValueError('not a TensorFlow checkpoint index (bad table magic)')
    footer = buf[-48:]
    _, pos = _get_varint(footer, 0)          # metaindex handle: offset
    _, pos = _get_varint(footer, pos)        #                   size
    idx_off, pos = _get_varint(footer, pos)
    idx_size, pos = _get_varint(footer, pos)
    out = {}
    for _, handle in _block_entries(_read_block(buf, idx_off, idx_size, verify)):
        off, p = _get_varint(handle, 0)
        size, _ = _get_varint(handle, p)
        for key, value in _block_entries(_read_block(buf, off, size, verify)):
            out[bytes(key)] = bytes(value)
    return out


def _build_block(items, restart_interval=16):
    """LevelDB block: prefix-compressed entries with a restart point every `restart_interval` keys (TensorFlow's
    table builder uses 16), then the restart offsets and their count."""
    out, restarts, prev = bytearray(), [], b''
    for i, (key, value) in enumerate(items):
        shared = 0
        if i % restart_interval == 0:
            restarts.append(len(out))
        else:
            n = min(len(prev), len(key))
            while shared < n and prev[shared] == key[shared]:
                shared += 1
        out += _put_varint(shared) + _put_varint(len(key) - shared) + _put_varint(len(value)) + key[shared:] + value
        prev = key
    for r in restarts or [0]:
        out += struct.pack('<I', r)
    out += struct.pack('<I', len(restarts) or 1)
    return bytes(out)


def _emit_block(f, block):
    off = f.tell()
    f.write(block)
    f.write(b'\x00' + struct.pack('<I', _mask(crc32c(block + b'\x00'))))
    return _put_varint(off) + _put_varint(len(block))


# ---- public API ----------------------------------------------------------------------------------------------------
def read_tf_checkpoint(prefix, verify=False):
    """`{key: ndarray}` of every tensor in the checkpoint `<prefix>.index` / `<prefix>.data-*`.

    Keys are returned as stored (object-graph checkpoints: `.../.ATTRIBUTES/VARIABLE_VALUE`).  `verify=True` also checks
    the per-tensor crc32c (slow in pure Python); block checksums of the index are always checked."""
    with open(prefix + '.index', 'rb') as f:
        table = _read_table(f.read())
    header = table.pop(b'', None)
    num_shards = 1
    if header is not None:
        for field, _, v in _parse_fields(header):
            if field == 1:
                num_shards = v
            if field == 2 and v != 0:
                raise ValueError('big-endian checkpoints are not supported')
    shards = {}
    out = {}
    for key, value in sorted(table.items()):
        e = _parse_entry(value)
        name = key.decode('utf-8')
        if e['sliced']:
            raise ValueError(f'{name}: partitioned (sliced) variables are not supported')
        if e['dtype'] not in _DTYPES:
            continue                                     # strings (e.g. _CHECKPOINTABLE_OBJECT_GRAPH), variants, ...
        sid = e['shard_id']
        if sid not in shards:
            shards[sid] = np.memmap(f'{prefix}.data-{sid:05d}-of-{num_shards:05d}', dtype=np.uint8, mode='r')
        raw = shards[sid][e['offset']:e['offset'] + e['size']]
        dt = np.dtype(_DTYPES[e['dtype']])
        if int(np.prod(e['shape'], dtype=np.int64)) * dt.itemsize != e['size']:
            raise ValueError(f'{name}: shape {e["shape"]} does not match {e["size"]} bytes')
        if verify and e['crc32c'] is not None and _mask(crc32c(raw.tobytes())) != e['crc32c']:
            raise ValueError(f'{name}: tensor checksum mismatch')
        out[name] = np.frombuffer(raw.tobytes(), dtype=dt.newbyteorder('<')).reshape(e['shape']).astype(dt)
    return out


def write_tf_checkpoint(prefix, tensors):
    """Write `{key: ndarray}` as a single-shard tensor bundle (`<prefix>.index`, `<prefix>.data-00000-of-00001`)."""
    os.makedirs(os.path.dirname(os.path.abspath(prefix)), exist_ok=True)
    entries = []
    with open(prefix + '.data-00000-of-00001', 'wb') as f:
        for key in sorted(tensors, key=lambda k: k.encode('utf-8')):
            arr = np.asarray(tensors[key])                # (np.ascontiguousarray would turn a scalar into shape (1,))
            if not arr.flags.c_contiguous:
                arr = arr.copy(order='C')
            if arr.dtype not in _DTYPE_IDS:
                raise ValueError(f'{key}: unsupported dtype {arr.dtype}')
            raw = arr.astype(arr.dtype.newbyteorder('<')).tobytes()
            entries.append((key.encode('utf-8'), _encode_entry(_DTYPE_IDS[arr.dtype], arr.shape, f.tell(), len(raw),
                                                               _mask(crc32c(raw)))))
            f.write(raw)
    # BundleHeaderProto: num_shards = 1, endianness = LITTLE (0, default), version { producer = 1 }
    header = _field(1, 0, _put_varint(1)) + _field(3, 2, _put_varint(2) + _field(1, 0, _put_varint(1)))
    items = [(b'', header)] + entries
    with open(prefix + '.index', 'wb') as f:
        index_items, block, size = [], [], 0
        for key, value in items:                         # data blocks of about 4 KB, like TensorFlow's table builder
            block.append((key, value))
            size += len(key) + len(value) + 3
            if size >= 4096:
                index_items.append((key, _emit_block(f, _build_block(block))))      # separator = last key of the block
                block, size = [], 0
        if block:
            index_items.append((block[-1][0], _emit_block(f, _build_block(block))))
        meta_handle = _emit_block(f, _build_block([]))
        index_handle = _emit_block(f, _build_block(index_items, restart_interval=1))
        footer = meta_handle + index_handle
        f.write(footer + b'\x00' * (40 - len(footer)) + struct.pack('<Q', _MAGIC))


# keras Sequentials of the reference whose children do not all own weights: `layer_with_weights-N` -> child index
_SEQUENTIAL_CHILDREN = {'mask': (0, 2)}        # update.py:137-141: [Conv2D, ReLU, Conv2D]


def tf_key_to_param(key):
    """`fnet/layer2/layer_with_weights-0/downsample/layer_with_weights-1/gamma/.ATTRIBUTES/VARIABLE_VALUE`
    -> `fnet.layer2.0.downsample.1.gamma` (None for keys that are not model variables: optimizer slots, counters, the
    object graph).  A leading `model/` (tf.train.Checkpoint(model=...)) is dropped."""
    if not key.endswith(_SUFFIX):
        return None
    parts = key[:-len(_SUFFIX)].split('/')
    if parts and parts[0] == 'model':
        parts = parts[1:]
    if not parts or parts[0] not in ('fnet', 'cnet', 'update_block'):
        return None
    if '.OPTIMIZER_SLOT' in parts:
        return None
    out = []
    for i, part in enumerate(parts):
        if part.startswith('layer_with_weights-'):
            n = int(part.split('-')[1])
            parent = parts[i - 1] if i else ''
            children = _SEQUENTIAL_CHILDREN.get(parent)
            out.append(str(children[n] if children else n))
        elif part.startswith('layer-'):
            out.append(part.split('-')[1])
        else:
            out.append(part)
    return '.'.join(out)


def param_to_tf_key(name):
    """The inverse of `tf_key_to_param`: `fnet.layer2.0.downsample.1.gamma` ->
    `fnet/layer2/layer_with_weights-0/downsample/layer_with_weights-1/gamma/.ATTRIBUTES/VARIABLE_VALUE`, the key Keras's
    `save_weights` gives the variable.  Numeric components are children of a keras Sequential (`layer_with_weights-N`,
    N counting weight-owning children only, through `_SEQUENTIAL_CHILDREN`)."""
    parts, out = name.split('.'), []
    for i, part in enumerate(parts):
        if part.isdigit():
            n = int(part)
            children = _SEQUENTIAL_CHILDREN.get(parts[i - 1] if i else '')
            out.append(f'layer_with_weights-{children.index(n) if children else n}')
        else:
            out.append(part)
    return '/'.join(out) + _SUFFIX


# Keras's names for the optimiser's state in an object-graph checkpoint (OptimizerV2 `iterations`, Adam's slots)
OPTIMIZER_ITER_KEY = 'optimizer/iter' + _SUFFIX


def optimizer_slot_key(name, slot):
    """`fnet.conv1.kernel`, 'm' -> `fnet/conv1/kernel/.OPTIMIZER_SLOT/optimizer/m/.ATTRIBUTES/VARIABLE_VALUE`."""
    return param_to_tf_key(name)[:-len(_SUFFIX)] + f'/.OPTIMIZER_SLOT/optimizer/{slot}' + _SUFFIX


def load_tf_checkpoint(prefix, verify=False, expect=None):
    """Checkpoint -> `{param name: ndarray}` for `RAFT.load_params` / `SmallRAFT.load_params`.

    `expect` = the model's `state_dict()` (name -> array-like): the mapped checkpoint must then cover exactly those names
    with those shapes; anything missing, unexpected or mis-shaped is reported in ONE error instead of surfacing later as a
    `KeyError` for the first missing name."""
    params = {}
    for key, value in read_tf_checkpoint(prefix, verify).items():
        name = tf_key_to_param(key)
        if name is not None:
            params[name] = value
    if not params:
        raise ValueError(f'{prefix}: no fnet/ cnet/ update_block/ variables found')
    if expect is not None:
        want = {k: tuple(np.shape(v)) for k, v in dict(expect).items()}
        missing = sorted(set(want) - set(params))
        extra = sorted(set(params) - set(want))
        shapes = sorted(f'{k}: checkpoint {tuple(params[k].shape)} vs model {want[k]}' for k in set(want) & set(params)
                        if tuple(params[k].shape) != want[k])
        if missing or extra or shapes:
            raise ValueError(f'{prefix}: does not match the model -- missing {missing[:8]}{"..." if len(missing) > 8 else ""}, '
                             f'unexpected {extra[:8]}{"..." if len(extra) > 8 else ""}, shapes {shapes[:8]}')
    return params
