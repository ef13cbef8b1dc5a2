"""A plain, sequential restatement of the generated fields' rule (include/tfrgpu.h, POSITIONS) on top of resync_walk's walk:
the expectation the GPU's position_kernel is tested against.

entries(data, is_final, resync) -> (entries, consumed): the block's entries in byte order, as resync_walk.walk gives them
    (("frame", off, end) and, under TFR_F_RESYNC, ("region", o, p, code)); without TFR_F_RESYNC the frame chain up to the
    first framing stop.
rows(entries, bad, mode, n_failfast) -> the entry index of every delivered row.
positions(entries, rows, first_entry, first_offset) -> [(row index, record offset)].
extent(entries, consumed, mode, bad) -> (consumed, entries in it): what tfr_batch_extent reports.
stream(data, cuts, ...) -> the rows of a file read in blocks cut at `cuts`, each block positioned by the extents of the blocks
    before it, as a streaming reader (io.readFile, the JNI BlockIterator) does."""
import resync_walk as RW

FAILFAST, DROPMALFORMED, PERMISSIVE = "FAILFAST", "DROPMALFORMED", "PERMISSIVE"


def entries(data, is_final, resync):
    data = bytes(data)
    if resync:
        return RW.walk(data, is_final)
    frames, q, code = RW.chain(data, 0, is_final)
    end = len(data)
    if code or not (q == end or (is_final and end - q < 8)):
        return frames, q                       # a framing stop, or the partial frame carried into the next block
    return frames, end


def rows(ents, bad, mode, n_failfast=None):
    """FAILFAST: the frames in front of the first failing one (n_failfast of them); DROPMALFORMED: every entry not in `bad`;
    PERMISSIVE: every entry, `bad` ones as corrupt rows"""
    if mode == FAILFAST:
        return list(range(n_failfast))
    if mode == PERMISSIVE:
        return list(range(len(ents)))
    return [k for k in range(len(ents)) if k not in bad]


def positions(ents, rws, first_entry=0, first_offset=0):
    return [(first_entry + k, first_offset + ents[k][1]) for k in rws]


def extent(ents, consumed, mode, bad):
    """(consumed, entries): FAILFAST ends a block in front of its first failing record"""
    if mode == FAILFAST and bad:
        k = min(bad)
        return ents[k][1], k
    return consumed, len(ents)


def frame_bad(data, payload_fails):
    """the bad entries of a block: its lost regions and the frames whose payload `payload_fails`"""
    def bad(ents):
        return {k for k, e in enumerate(ents) if e[0] == "region" or payload_fails(bytes(data[e[1] + 12:e[2] - 4]), bytes(data[e[2] - 4:e[2]]))}
    return bad


def block(data, is_final, resync, mode, payload_fails, first_entry=0, first_offset=0):
    """-> (positions of the block's rows, (consumed, entries))"""
    ents, consumed = entries(data, is_final, resync)
    bad = frame_bad(data, payload_fails)(ents)
    n_ff = min(bad) if bad else len(ents)
    rws = rows(ents, bad, mode, n_ff)
    return positions(ents, rws, first_entry, first_offset), extent(ents, consumed, mode, bad)


def stream(data, cuts, resync, mode, payload_fails):
    """the rows of `data` read in blocks ending at `cuts` with carry (a block that consumes nothing grows by the next cut),
    each submitted at the (entries, offset) the extents before it add up to; FAILFAST stops after a block with an error"""
    data = bytes(data)
    out, pos, ent = [], 0, 0
    cuts = sorted(c for c in cuts if 0 < c < len(data)) + [len(data)]
    i = 0
    while pos < len(data):
        while cuts[i] <= pos:
            i += 1
        stop = cuts[i]
        final = stop == len(data)
        got, (used, n) = block(data[pos:stop], final, resync, mode, payload_fails, ent, pos)
        out += got
        ents, consumed = entries(data[pos:stop], final, resync)
        if (mode == FAILFAST and used < consumed) or (not resync and RW.chain(data[pos:stop], 0, final)[2]):
            return out                           # the reader raises the block's error (a failing record, a framing error)
        if final and used == stop - pos:
            return out
        if used == 0:
            if final:
                return out
            i += 1
            continue
        pos += used
        ent += n
    return out
