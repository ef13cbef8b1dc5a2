"""Schema inference in a parse mode (tfr_infer_create_mode) on the CPU.  TEST INFRASTRUCTURE ONLY.

Built record by record on the oracle's FAILFAST inference (`oracle.infer`, protobuf-java's parse and
TensorFlowInferSchema's verdicts), so that a record's verdict and its names are exactly what FAILFAST computes for it:

  * flags without TFR_F_DROP_MALFORMED / TFR_F_PERMISSIVE: FAILFAST, which is `oracle.infer` (no CRC is checked);
  * otherwise the frames are read as TFRecordReader reads them with its CRC check on: a framing error (TFR_E_CRC_LENGTH,
    TFR_E_RECORD_TOO_LARGE, TFR_E_TRUNCATED) ends the call with what the records before it merged.  A record whose data
    CRC fails is skipped with TFR_E_CRC_DATA; otherwise its verdict is `oracle.infer` of its frame alone, and a record
    error (TFR_E_MALFORMED_PROTO, TFR_E_KIND_MISMATCH, TFR_E_EMPTY_SCALAR) skips it.  A kept record merges the names
    `oracle.infer` gives it (max, null the identity; ArrayType(ArrayType(null)) against another type is a conflict);
  * in PERMISSIVE the entries keyed like the corrupt-record column are cut out of a record that parses before it is
    judged, in `features` / `context` and in `feature_lists`: they are neither merged nor judged.

`infer_mode` -> (status, names -> codes, [(frame index, frame offset, code)] of the skipped records).  The status is the
framing error, else TFR_E_UNSUPPORTED_TYPE for a conflict among the kept records, else 0."""
from __future__ import annotations

import struct

from oracle import oracle
from spark_tfrecord_b200 import _cabi as A


def _varint(b: bytes, p: int):
    v = s = 0
    while True:
        c = b[p]
        p += 1
        v |= (c & 0x7F) << s
        s += 7
        if c < 0x80:
            return v, p


def _fields(b: bytes):
    """(field number, wire type, start, end of the whole field, payload of a length-delimited one) of a message that
    parses; a group is one field"""
    p, out = 0, []
    while p < len(b):
        start = p
        t, p = _varint(b, p)
        f, w = t >> 3, t & 7
        val = None
        if w == 0:
            _, p = _varint(b, p)
        elif w == 1:
            p += 8
        elif w == 5:
            p += 4
        elif w == 2:
            n, p = _varint(b, p)
            val = b[p:p + n]
            p += n
        elif w == 3:
            depth = 1
            while depth:
                t2, p = _varint(b, p)
                w2 = t2 & 7
                if w2 == 3:
                    depth += 1
                elif w2 == 4:
                    depth -= 1
                elif w2 == 0:
                    _, p = _varint(b, p)
                elif w2 == 1:
                    p += 8
                elif w2 == 5:
                    p += 4
                elif w2 == 2:
                    n, p = _varint(b, p)
                    p += n
        out.append((f, w, start, p, val))
    return out


def _ld(field: int, body: bytes) -> bytes:
    out, n = bytearray([field << 3 | 2]), len(body)
    while n >= 0x80:
        out.append(n & 0x7F | 0x80)
        n >>= 7
    out.append(n)
    return bytes(out) + body


def _without_key(payload: bytes, rt: int, name: bytes) -> bytes:
    """a payload that parses, with every map entry keyed `name` cut out (the key of an entry is its last key field)"""
    out = []
    for f, w, start, end, val in _fields(payload):
        if w == 2 and (f == 1 or (f == 2 and rt == 1)):
            kept = []
            for f2, w2, s2, e2, v2 in _fields(val):
                if f2 == 1 and w2 == 2:
                    keys = [v3 for f3, w3, _, _, v3 in _fields(v2) if f3 == 1 and w3 == 2]
                    if (keys[-1] if keys else b"") == name:
                        continue
                kept.append(val[s2:e2])
            out.append(_ld(f, b"".join(kept)))
        else:
            out.append(payload[start:end])
    return b"".join(out)


def _frame(payload: bytes) -> bytes:
    hdr = struct.pack("<Q", len(payload))
    return hdr + struct.pack("<I", oracle.masked_crc32c(hdr)) + payload + struct.pack("<I", oracle.masked_crc32c(payload))


def infer_mode(data: bytes, record_type: int = 0, flags: int = 0, corrupt_name=None):
    data = bytes(data)
    if not flags & (A.TFR_F_DROP_MALFORMED | A.TFR_F_PERMISSIVE):
        rc, codes = oracle.infer(data, record_type)
        return rc, codes, []
    name = corrupt_name.encode() if isinstance(corrupt_name, str) else corrupt_name
    if not flags & A.TFR_F_PERMISSIVE:
        name = None
    merged, conflict, skipped = {}, False, []
    pos, row, rc = 0, 0, 0
    while len(data) - pos >= 8:
        left = len(data) - pos
        if left < 12:
            rc = A.TFR_E_TRUNCATED
            break
        n = struct.unpack_from("<Q", data, pos)[0]
        if oracle.masked_crc32c(data[pos:pos + 8]) != struct.unpack_from("<I", data, pos + 8)[0]:
            rc = A.TFR_E_CRC_LENGTH
            break
        if n > 0x7FFFFFFF:
            rc = A.TFR_E_RECORD_TOO_LARGE
            break
        if left < 16 + n:
            rc = A.TFR_E_TRUNCATED
            break
        payload = data[pos + 12:pos + 12 + n]
        if oracle.masked_crc32c(payload) != struct.unpack_from("<I", data, pos + 12 + n)[0]:
            err, codes = A.TFR_E_CRC_DATA, {}
        else:
            err, codes = oracle.infer(_frame(payload), record_type)
            if name is not None and err != A.TFR_E_MALFORMED_PROTO:
                err, codes = oracle.infer(_frame(_without_key(payload, record_type, name)), record_type)
        if err == A.TFR_E_UNSUPPORTED_TYPE:                   # a conflict inside the record: kept, and the call's conflict
            conflict, err = True, 0
        if err:
            skipped.append((row, pos, err))
        else:
            for k, c in codes.items():
                old = merged.get(k)
                if old is not None and old != c and 0 not in (old, c) and 10 in (old, c):
                    conflict = True
                merged[k] = c if old is None else max(old, c)
        pos += 16 + n
        row += 1
    if rc == 0 and conflict:
        rc = A.TFR_E_UNSUPPORTED_TYPE
    return rc, merged, skipped
