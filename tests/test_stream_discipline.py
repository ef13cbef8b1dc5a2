"""Source checks of the host runtime's concurrency rules (no GPU needed).

Spark runs several tasks per executor, each with its own decoder, encoder or inference handle on the same GPU, and every
handle's work runs on non-blocking streams.  A non-blocking stream has no ordering with the legacy default stream, so device
state a kernel reads must be written on the handle's own stream and waited for; and the opt-in shared-memory attribute of a
kernel is process-wide, so raising it is a check-then-set that must not race (DESIGN.md section 4, INTEGRATION.md
"Threading/ownership").  A task retried after an allocation failure must not leak what its handle had built, so every CUDA
resource has an owner type whose destructor frees it (DESIGN.md section 3)."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "spark-tfrecord_b200", "csrc")


def _sources():
    for f in sorted(os.listdir(CSRC)):
        if f.endswith((".cu", ".cuh", ".inc", ".h")):
            txt = open(os.path.join(CSRC, f)).read()
            yield f, re.sub(r"//[^\n]*", "", re.sub(r"/\*.*?\*/", "", txt, flags=re.S))


def _calls(code, name):
    """(line, argument text) of every call of `name`, parentheses matched"""
    for m in re.finditer(r"\b" + name + r"\s*\(", code):
        depth, i = 1, m.end()
        while depth:
            depth += {"(": 1, ")": -1}.get(code[i], 0)
            i += 1
        yield code.count("\n", 0, m.start()) + 1, code[m.end():i - 1]


def _braced_body(code, header):
    """(offset, text) of the brace-matched body that follows the regex `header` (which ends at the opening brace)"""
    m = re.search(header, code)
    assert m, f"{header} not found"
    depth, i = 1, m.end()
    while depth:
        depth += {"{": 1, "}": -1}.get(code[i], 0)
        i += 1
    return m.end(), code[m.end():i]


def _last_arg(args):
    depth, cut = 0, 0
    for i, ch in enumerate(args):
        depth += {"(": 1, ")": -1}.get(ch, 0)
        if ch == "," and depth == 0:
            cut = i + 1
    return args[cut:].strip()


def test_no_copy_or_memset_on_the_legacy_default_stream():
    """cudaMemcpy / cudaMemset run on the legacy default stream: a D2D copy or a memset returns before it is done, a pageable
    H2D copy may return before its DMA lands, and no handle stream waits for either.  Every copy and memset names a stream."""
    bad = []
    for f, code in _sources():
        for name in ("cudaMemcpy", "cudaMemset", "cudaMemcpy2D", "cudaMemcpyToSymbol", "cudaMemcpyFromSymbol"):
            bad += [f"{f}:{ln}: {name}(" for ln, _ in _calls(code, name)]
        for name in ("cudaMemcpyAsync", "cudaMemsetAsync"):
            for ln, args in _calls(code, name):
                if args.count(",") < (4 if name == "cudaMemcpyAsync" else 3) or _last_arg(args) in ("0", "nullptr", "NULL", "cudaStreamLegacy"):
                    bad.append(f"{f}:{ln}: {name} on the default stream")
    assert not bad, "synchronous or default-stream copies in csrc/:\n" + "\n".join(bad)


def test_kernel_launches_name_a_stream():
    bad = []
    for f, code in _sources():
        for m in re.finditer(r"<<<(.*?)>>>", code, flags=re.S):
            cfg = m.group(1)
            depth, parts, cur = 0, [], ""
            for ch in cfg:
                if ch == "," and depth == 0:
                    parts.append(cur); cur = ""
                    continue
                depth += {"(": 1, ")": -1}.get(ch, 0)
                cur += ch
            parts.append(cur)
            if len(parts) < 4 or parts[3].strip() in ("0", "nullptr", "NULL"):
                bad.append(f"{f}:{code.count(chr(10), 0, m.start()) + 1}: <<<{cfg}>>>")
    assert not bad, "kernel launches on the default stream:\n" + "\n".join(bad)


def test_raise_dyn_smem_checks_and_sets_under_a_lock():
    """cudaFuncSetAttribute(MaxDynamicSharedMemorySize) sets the limit, it does not take a maximum: two threads asking for
    different sizes of the same kernel must not interleave their check and their set, or the smaller one wins while the
    process believes the larger one was granted.  All the raises go through raise_dyn_smem, which holds a lock for both."""
    sets = []
    for f, code in _sources():
        sets += [(f, ln) for ln, args in _calls(code, "cudaFuncSetAttribute") if "MaxDynamicSharedMemorySize" in args]
    assert len(sets) == 1, f"every opt-in raise goes through raise_dyn_smem: {sets}"
    code = dict(_sources())["api.cu"]
    _, body = _braced_body(code, r"static\s+cudaError_t\s+raise_dyn_smem\s*\([^)]*\)\s*\{")
    assert "cudaFuncSetAttribute" in body
    lock = re.search(r"std::(lock_guard|unique_lock|scoped_lock)\s*<\s*std::mutex\s*>", body)
    assert lock, "raise_dyn_smem takes no lock"
    before_set = body[lock.end():body.index("cudaFuncSetAttribute")]
    assert "granted" in before_set, "the size is checked again under the lock, before the attribute is set"
    assert re.search(r"std::atomic\s*<\s*size_t\s*>\s+granted", body), "the unlocked fast path reads an atomic"


def test_cuda_resources_are_allocated_and_freed_only_by_their_owners():
    """Every device buffer, pinned host buffer, stream and event of a handle is held by an owner type of host_util.h whose
    destructor frees it, so a create function that returns early frees whatever it had built.  Outside host_util.h nothing
    allocates, frees, creates or destroys one by hand.  The one exception is the device copy of the CRC tables in get_ctx:
    it lives as long as the process, in static storage, where a destructor would run after the CUDA runtime has shut down.
    A block borrowed from DevPool or PinnedPool is held the same way, by a PoolBlock that gives it back when it is reset or
    destroyed: nothing outside host_util.h calls a pool's give_back, so no path can return a block twice or forget one.  An
    event borrowed from an EventPool is held by a PoolEvent in the same way: nothing outside host_util.h calls a pool's give."""
    raw = re.compile(r"\b(cuda(?:Malloc|Free|HostAlloc|StreamCreate|StreamDestroy|EventCreate|EventDestroy)\w*)\s*\(")
    api = dict(_sources())["api.cu"]
    start, body = _braced_body(api, r"static\s+int32_t\s+get_ctx\s*\([^)]*\)\s*\{")
    bad, allowed = [], []
    for f, code in _sources():
        if f == "host_util.h":
            continue
        for m in raw.finditer(code):
            where = f"{f}:{code.count(chr(10), 0, m.start()) + 1}: {m.group(1)}("
            if f == "api.cu" and m.group(1) == "cudaMalloc" and start <= m.start() < start + len(body):
                allowed.append(where)
            else:
                bad.append(where)
        bad += [f"{f}:{ln}: {name}(" for name in ("give_back", "give") for ln, _ in _calls(code, name)]
    assert not bad, "raw CUDA allocations / frees, or pool blocks or events given back, outside the owners of host_util.h:\n" + "\n".join(bad)
    assert len(allowed) == 1, f"get_ctx allocates the CRC tables once: {allowed}"
