"""An independent reader and writer of the checkpoint format (DESIGN.md §5 "Checkpoints"), in numpy: an 8-byte magic,
a u32 version, then records until EOF, each a u32 name length, the name, a u8 type (0 float32, 1 int64, 2 text), a u64
element count and the payload, all little-endian."""
import struct

import numpy as np

MAGIC, VERSION = b"CNBCKPT\0", 1
DTYPES = {0: np.dtype("<f4"), 1: np.dtype("<i8"), 2: np.dtype("u1")}


def read(path):
    """{name: np.ndarray (float32 / int64) or str (text)}, in file order"""
    data = open(path, "rb").read()
    assert data[:8] == MAGIC and struct.unpack_from("<I", data, 8)[0] == VERSION
    out, pos = {}, 12
    while pos < len(data):
        (n,) = struct.unpack_from("<I", data, pos)
        name = data[pos + 4:pos + 4 + n].decode()
        typ, count = struct.unpack_from("<BQ", data, pos + 4 + n)
        pos += 4 + n + 9
        size = count * DTYPES[typ].itemsize
        payload = data[pos:pos + size]
        assert len(payload) == size, "truncated record %r" % name
        out[name] = payload.decode() if typ == 2 else np.frombuffer(payload, DTYPES[typ]).copy()
        pos += size
    return out


def write(path, records):
    """records: {name: str (text), int (int64), or an array (float32)}"""
    with open(path, "wb") as f:
        f.write(MAGIC + struct.pack("<I", VERSION))
        for name, v in records.items():
            if isinstance(v, str):
                typ, payload, count = 2, v.encode(), len(v.encode())
            elif isinstance(v, (int, np.integer)):
                typ, payload, count = 1, struct.pack("<q", int(v)), 1
            else:
                a = np.ascontiguousarray(v, dtype="<f4")
                typ, payload, count = 0, a.tobytes(), a.size
            f.write(struct.pack("<I", len(name.encode())) + name.encode() + struct.pack("<BQ", typ, count) + payload)
