"""A plain, sequential restatement of the record index (include/tfrgpu.h, RECORD INDEX) from a host frame walk: the
expectation the GPU's index_checkpoint_kernel and tfr_index_seek are tested against.

frames(data) -> the header offsets of a file's frames, or FramingError(code, offset) at its first framing error.
checkpoints(offsets, data_bytes, stride) -> [(offset, entry)] for k = 0 .. ceil(data_bytes / stride) - 1.
index_bytes(data, stride) -> the index file's bytes.
seek(offsets, data_bytes, target) -> (entry, offset) of the first frame at or after target, (n_entries, data_bytes) if none.
split(offsets, s, e) -> the entries a split [s, e) delivers: the frames whose header offset o has s <= o < e."""
import bisect
import struct

import resync_walk as RW

MAGIC = b"TFRIDX01"
HEADER = struct.Struct("<8sQQQ")


class FramingError(Exception):
    def __init__(self, code, offset):
        super().__init__(f"framing error {code} at offset {offset}")
        self.code, self.offset = code, offset


def frames(data):
    fr, q, code = RW.chain(bytes(data), 0, True)
    if code:
        raise FramingError(code, q)
    return [f[1] for f in fr]


def checkpoints(offsets, data_bytes, stride):
    out, i = [], 0
    for k in range(-(-data_bytes // stride)):
        while i < len(offsets) and offsets[i] < k * stride:
            i += 1
        out.append((offsets[i], i) if i < len(offsets) else (data_bytes, len(offsets)))
    return out


def index_bytes(data, stride):
    offs = frames(data)
    ck = checkpoints(offs, len(data), stride)
    return HEADER.pack(MAGIC, len(data), len(offs), stride) + b"".join(struct.pack("<QQ", o, e) for o, e in ck)


def seek(offsets, data_bytes, target):
    i = bisect.bisect_left(offsets, target)
    return (i, offsets[i]) if i < len(offsets) else (len(offsets), data_bytes)


def split(offsets, s, e):
    return list(range(bisect.bisect_left(offsets, s), bisect.bisect_left(offsets, e)))
