"""A plain, sequential restatement of the TFR_F_RESYNC rule (include/tfrgpu.h, DESIGN.md section 2): the reference the GPU's
frame index + resync_scan_kernel loop is tested against.

walk(data, is_final, H) -> (entries, consumed).  entries are the block's frames and lost regions in byte order:
    ("frame", off, end)           a frame [off, end) whose length CRC verified (its payload CRC is the decoder's business)
    ("region", o, p, code)        a lost region [o, p) and the framing error (TFR_E_*) that began it
consumed: the bytes of the block the batch takes (a non-final block leaves a partial frame, and an unresolved region, to the
next block)."""
import struct

from oracle.pyref import masked_crc32c

TFR_E_CRC_LENGTH, TFR_E_TRUNCATED, TFR_E_RECORD_TOO_LARGE = -10, -12, -13
H_MAX = 0x7FFFFFFF                         # the largest block a decoder takes


def _u32(data, p):
    return struct.unpack_from("<I", data, p)[0]


def header_ok(data, p):
    """the frame index's header predicate (frame_header_ok): length <= INT32_MAX and its masked CRC-32C verifies"""
    lo, hi = struct.unpack_from("<II", data, p)
    return hi == 0 and lo <= 0x7FFFFFFF and masked_crc32c(bytes(data[p:p + 8])) == _u32(data, p + 8)


def chain(data, s, is_final):
    """the ordinary frame chain from s -> (frames, q, code): code is the framing error at q, 0 for a clean stop at q"""
    end, q, frames = len(data), s, []
    while True:
        left = end - q
        if left < 8:                       # EOF, or 1..7 stray bytes: a clean end
            return frames, q, 0
        if left < 12:
            return frames, q, TFR_E_TRUNCATED if is_final else 0
        lo, hi = struct.unpack_from("<II", data, q)
        if masked_crc32c(bytes(data[q:q + 8])) != _u32(data, q + 8):
            return frames, q, TFR_E_CRC_LENGTH
        if hi or lo > 0x7FFFFFFF:
            return frames, q, TFR_E_RECORD_TOO_LARGE
        if left < 16 + lo:
            return frames, q, TFR_E_TRUNCATED if is_final else 0
        frames.append(("frame", q, q + 16 + lo))
        q += 16 + lo


def decisive(data, o, p, is_final, H):
    """'point' (a resync point), 'undecided' (more bytes could make p a resync point) or None"""
    end = len(data)
    if p + 16 > o + H:
        return None
    if p + 12 > end:
        return None if is_final else "undecided"
    if not header_ok(data, p):
        return None
    fe = p + 16 + _u32(data, p)
    if fe > end:
        return "undecided" if not is_final and fe - o <= H else None
    if fe - o > H:
        return None
    payload = bytes(data[p + 12:fe - 4])
    return "point" if masked_crc32c(payload) == _u32(data, fe - 4) else None


def walk(data, is_final, H=H_MAX):
    data = bytes(data)
    end, s, entries = len(data), 0, []
    while True:
        frames, o, code = chain(data, s, is_final)
        entries += frames
        if not code:
            if o == end or (is_final and end - o < 8):
                return entries, end
            return entries, o                # a partial frame (or stray bytes) carried into the next block
        for p in range(o + 1, end + 1):
            k = decisive(data, o, p, is_final, H)
            if k == "undecided":
                return entries, o            # unresolved: the next block starts at o with more bytes
            if k == "point":
                entries.append(("region", o, p, code))
                s = p
                break
        else:
            if not is_final:                 # no resync point within H of o: unresolved as well
                return entries, o
            entries.append(("region", o, end, code))
            return entries, end


def walk_blocks(data, cuts, H=H_MAX):
    """the file walked in blocks that end at the offsets `cuts` (a block loop with carry, as the readers run it; a block
    that consumes nothing grows by the next cut) -> the entries in file offsets"""
    data = bytes(data)
    out, pos = [], 0
    cuts = sorted(c for c in cuts if 0 < c < len(data)) + [len(data)]
    i = 0
    while pos < len(data):
        while cuts[i] <= pos:
            i += 1
        stop = cuts[i]
        final = stop == len(data)
        ents, used = walk(data[pos:stop], final, H)
        out += [(e[0], e[1] + pos, e[2] + pos) + e[3:] for e in ents]
        if final and used == stop - pos:
            return out
        if used == 0:
            i += 1                           # nothing decided: the same start with the next cut
            continue
        pos += used
    return out
