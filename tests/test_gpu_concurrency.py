"""Many Spark task threads on one GPU, each checked bit for bit against the CPU oracle.

A Spark executor runs several tasks at once, and the reader creates one decoder per file per task
(M/TFRecordFileReader.scala:16-20); writers and schema inference do the same.  The C ABI is re-entrant: one handle per
thread, batches released from any thread, exported Arrow arrays released wherever the JVM runs their callback.  Here eight
task threads start on a barrier and each runs what a task does, several files in a row with one handle per file:

- readers stream their file in 1-8 MiB blocks the way io.TFRecordFileReader does (block t + 1 is submitted as soon as
  block t's consumed count is known, the copy-out is enqueued, then block t is waited for).  The shapes cover the uniform
  pipelined tile kernel, one-pass ragged columns, SequenceExample, ByteArray, the general path (130 fields), the
  transcoding instantiation (malformed UTF-8) and the 4 + 1 warp tiles (200-byte records).  Every block's status and
  columns, and its UnsafeRows (with partition values on one shape), must be the oracle's; one file has a flipped payload
  bit and must fail at the oracle's row while the other threads go on;
- writers encode columns and UnsafeRows of 100 B to 20 KB rows, so their shared-memory requests for the same kernels
  differ from thread to thread;
- schema inference streams files through Infer.update_block;
- a releaser thread drops batches the readers hand over: resolved ones, speculative ones never resolved, and batches
  whose exported Arrow arrays outlive the closed decoder;
- two threads fail at the same moment with different errors, and each message names its own cause.

Then every workload runs once more from one thread (a kernel whose shared-memory opt-in was lowered by a race fails there
with TFR_E_CUDA), and three fresh processes repeat both phases, so that the threads' first launches of every kernel race
each other.  The race this guards against cannot be forced: the test can pass without the fix (DESIGN.md section 4).
All expected results are computed before the threads start.

Run as a script with --child for one fresh-process round."""
import os
import queue
import subprocess
import sys
import threading
import time
import traceback

import numpy as np

TESTS = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(TESTS)
for _p in (TESTS, ROOT):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import pytest  # noqa: E402

import partition_rows as P  # noqa: E402
from oracle import unsaferow as U  # noqa: E402
from spark_tfrecord_b200 import _cabi as A  # noqa: E402
from spark_tfrecord_b200.sqltypes import *  # noqa: E402,F401,F403
from util import assert_columns_equal, record_offsets  # noqa: E402

pytestmark = pytest.mark.gpu

MiB = 1 << 20
N_TASKS = 8
INFO_KEYS = ("error_code", "error_row", "error_field", "n_rows", "consumed_bytes")


# ---------------------------------------------------------------------------------------------------------------------
# workloads (CPU only)
# ---------------------------------------------------------------------------------------------------------------------
class Block:
    __slots__ = ("pos", "take", "final", "early", "info", "cols", "rows")


class ReadFile:
    """one file a reader task streams: its bytes, block size, the oracle's result of every block it submits (up to the
    first failing one) and what the decoder's counters must show afterwards"""

    def __init__(self, name, sch, rt, data, block, rows_of_cols=None, part=None, damaged=False):
        self.name, self.sch, self.rt, self.data, self.block, self.part, self.damaged = name, sch, rt, data, block, part, damaged
        self.names = sch.names if rt != TFR_RT_BYTE_ARRAY else ["byteArray"]
        self.rows_of_cols = rows_of_cols
        self.blocks = []
        self.arrow_col = None                 # (column index) of a column checked again through Arrow after the decoder closed

    def plan(self, oracle):
        offs = record_offsets(self.data)
        pos = 0
        while True:
            b = Block()
            b.pos, b.take = pos, min(self.block, len(self.data) - pos)
            b.final = pos + b.take == len(self.data)
            # the frame index's count: every complete record of the block (a payload error is found later, in the rows)
            b.early = b.take if b.final else int(offs[np.searchsorted(offs, pos + b.take, side="right") - 1]) - pos
            want = oracle.decode(self.data[pos:pos + b.take], self.sch, self.rt, is_final=b.final)
            b.info = {k: want.info[k] for k in INFO_KEYS}
            b.cols = want.columns
            b.rows = self.rows_of_cols(b.cols, b.info["n_rows"]) if self.rows_of_cols else None
            self.blocks.append(b)
            if b.info["error_code"] or b.final:
                break
            assert b.info["consumed_bytes"] == b.early, (self.name, pos)
            pos += b.early
        assert len(self.blocks) >= 3, (self.name, len(self.data))
        assert bool(self.blocks[-1].info["error_code"]) == self.damaged, (self.name, self.blocks[-1].info)
        return self


def _generic_rows(sch):
    from test_gpu_encode_rows import rows_of

    def f(cols, n):
        data, offs = U.unsafe_rows(sch, rows_of(cols, n))
        return data, offs.astype(np.int64)
    return f


def _encoded(oracle, sch, cols, rt=0):
    data, rc, _ = oracle.encode(cols, sch, rt)
    assert rc == 0
    return np.frombuffer(data, dtype=np.uint8).copy()


def _read_files(oracle):
    from oracle.corpus import cfg2_columns, cfg4_columns, mixed_columns
    from test_gpu_fuzz import _batch, _schema
    files = {}
    # uniform columns, steady-state pipeline; rows with a file's partition values appended
    sch, cols = cfg2_columns(9000, seed=301)
    pt, pv = ["string", "int", ("decimal", 38, 6)], ["2026-10-15", 17, None]
    f = ReadFile("cfg2", sch, 0, _encoded(oracle, sch, cols), 3 * MiB, lambda c, n: P.cfg2_joined_rows(c, pt, pv),
                 part=(P.partition_row(pt, pv), P.var_flags(pt)))
    f.arrow_col = 0
    files["cfg2"] = f
    # ragged columns of a random schema (one-pass ragged kernel + look-back); a copy with one flipped payload bit
    rng = np.random.default_rng(1005)
    sch, gens = _schema(rng)
    assert any(isinstance(x.dataType, ArrayType) for x in sch.fields)
    data = _batch(oracle, sch, gens, 15000, 4242).copy()
    files["ragged"] = ReadFile("ragged", sch, 0, data, 1 * MiB, _generic_rows(sch))
    offs = record_offsets(data)
    k = int(len(offs) * 0.8)
    while int(offs[k + 1] - offs[k]) <= 16:
        k += 1
    bad = data.copy()
    bad[int(offs[k]) + 12 + int(offs[k + 1] - offs[k] - 16) // 2] ^= 0x20
    files["ragged_damaged"] = ReadFile("ragged_damaged", sch, 0, bad, 1 * MiB, _generic_rows(sch), damaged=True)
    # SequenceExample: context id + a FeatureList of float lists
    sch, cols = cfg4_columns(2600, seed=303)
    files["seq"] = ReadFile("seq", sch, TFR_RT_SEQUENCE_EXAMPLE, _encoded(oracle, sch, cols, TFR_RT_SEQUENCE_EXAMPLE), 1 * MiB,
                            _generic_rows(sch))
    # ByteArray payloads of 0 to 2000 bytes
    r = np.random.default_rng(304)
    sizes = r.integers(0, 2000, 20000)
    blob = r.integers(0, 256, int(sizes.sum()), dtype=np.uint8).tobytes()
    pos = np.concatenate([[0], np.cumsum(sizes)])
    bsch = byte_array_schema()
    bcols = A.columns_from_rows(bsch, [(blob[pos[i]:pos[i + 1]],) for i in range(len(sizes))], TFR_RT_BYTE_ARRAY)
    f = ReadFile("bytes", bsch, TFR_RT_BYTE_ARRAY, _encoded(oracle, bsch, bcols, TFR_RT_BYTE_ARRAY), 8 * MiB, _generic_rows(bsch))
    f.arrow_col = 0
    files["bytes"] = f
    # 130 fields: more than the tile kernel takes, the general path
    wsch = StructType([StructField(f"w{i:03d}", LongType() if i % 4 else StringType(), True) for i in range(130)])
    r = np.random.default_rng(305)
    rows = [tuple(None if (i + j) % 17 == 0 else (int(r.integers(-2**40, 2**40)) if i % 4 else "v" * ((i + j) % 23))
                  for i in range(130)) for j in range(1500)]
    files["wide"] = ReadFile("wide", wsch, 0, _encoded(oracle, wsch, A.columns_from_rows(wsch, rows)), 1 * MiB, _generic_rows(wsch))
    # malformed UTF-8 in ragged string columns: the transcoding instantiation of the tile kernel.  The first block is clean:
    # a decoder whose first block holds malformed UTF-8 takes the general path for it and, learning nothing, for every block
    # after it (DESIGN.md section 8)
    sch, cols = mixed_columns(9000, seed=306)
    bad_seqs = [b"\xff", b"\xc3", b"\xe2\x82", b"\xed\xa0\x80", b"\xf0\x9f\x98", b"\xc0\xaf", b"ok\x80ok", b"\xf5\x80\x80\x80"]
    for name, every in (("s", 97), ("as", 53)):
        c = cols[sch.names.index(name)]
        vals, so = c.values.copy(), c.offsets[-1]
        first = 5000                                     # a row of the second 2 MiB block; as a string index:
        for o in c.offsets[:-1]:
            first = int(o[first])
        for n_bad, i in enumerate(range(first, len(so) - 1, every)):
            seq = bad_seqs[n_bad % len(bad_seqs)]
            if so[i + 1] - so[i] >= len(seq):
                vals[so[i]:so[i] + len(seq)] = np.frombuffer(seq, np.uint8)
        cols[sch.names.index(name)] = A.HostColumn(c.elem_type, c.depth, c.n_rows, c.validity, c.offsets, vals)
    files["utf8"] = ReadFile("utf8", sch, 0, _encoded(oracle, sch, cols), 2 * MiB, _generic_rows(sch))
    # about 200-byte records: the 4 + 1 warp tiles
    small = dict(n_int=8, n_float=2, n_bytes=4, float_len=4, bytes_len=8)
    sch, cols = cfg2_columns(40000, seed=307, **small)
    f = ReadFile("small", sch, 0, _encoded(oracle, sch, cols), 2 * MiB,
                 lambda c, n: (lambda r, o: (r, o.astype(np.int64)))(*U.cfg2_rows(c, **small)))
    f.arrow_col = 0
    files["small"] = f
    for f in files.values():
        f.plan(oracle)
    return files


class WriteJob:
    def __init__(self, oracle, mean, seed, rt):
        r = np.random.default_rng(seed)
        n = int(np.clip((3 * MiB) // mean, 48, 20000))
        sizes = np.maximum(0, r.normal(mean, mean / 4, n)).astype(np.int64)
        if rt == TFR_RT_BYTE_ARRAY:
            self.sch = byte_array_schema()
            rows = [(r.integers(0, 256, int(s), dtype=np.uint8).tobytes(),) for s in sizes]
        else:
            self.sch = StructType([StructField("id", LongType()), StructField("payload", BinaryType()),
                                   StructField("vec", ArrayType(FloatType())), StructField("tag", StringType(), True)])
            rows = [(i, r.integers(0, 256, int(s), dtype=np.uint8).tobytes(),
                     [float(x) for x in r.standard_normal(int(r.integers(0, 9)), dtype=np.float32)],
                     None if i % 7 == 3 else "t" * (i % 13)) for i, s in enumerate(sizes)]
        self.rt, self.mean = rt, mean
        self.cols = A.columns_from_rows(self.sch, rows, rt)
        self.want, rc, _ = oracle.encode(self.cols, self.sch, rt)
        assert rc == 0
        self.rows, self.offs = U.unsafe_rows(self.sch, rows)


class Workload:
    def __init__(self, oracle):
        t0 = time.time()
        self.files = _read_files(oracle)
        shapes = ["cfg2", "ragged", "seq", "bytes", "wide", "utf8", "small"]
        # five readers, three files each, every shape twice or more and never the same shape on two threads at the start
        self.readers = [[shapes[(2 * k + j) % len(shapes)] for j in range(3)] for k in range(5)]
        self.readers[1].insert(1, "ragged_damaged")
        means = [(100, 4000), (20000, 1000)]             # two writer threads
        self.writers = [[WriteJob(oracle, m, 400 + 10 * w + i, rt) for i, m in enumerate(ms) for rt in (0, TFR_RT_BYTE_ARRAY)]
                        for w, ms in enumerate(means)]
        self.infer = [(nm, oracle.infer(self.files[nm].data.tobytes(), self.files[nm].rt)) for nm in ("cfg2", "seq", "ragged", "utf8")]
        for nm, (rc, _) in self.infer:
            assert rc == 0, nm
        # the two failures raised at the same moment
        self.dec_sch = StructType([StructField("x", LongType()), StructField("dec", DecimalType())])
        self.dec_data = _encoded(oracle, self.dec_sch, A.columns_from_rows(self.dec_sch, [(i, i / 4) for i in range(100)]))
        from test_gpu_encode_rows import _malformed_batch, _put, _slot
        self.bad_sch, data, offs = _malformed_batch()
        self.bad_rows, self.bad_offs = data.copy(), offs.copy()
        p, s = _slot(self.bad_rows, self.bad_offs, 50, 1)
        _put(self.bad_rows, p, ((int(offs[51] - offs[50]) + 8) << 32) | (s & 0xFFFFFFFF))    # row 50's string beyond its row
        self.prep_seconds = time.time() - t0


# ---------------------------------------------------------------------------------------------------------------------
# tasks (GPU)
# ---------------------------------------------------------------------------------------------------------------------
class Releaser:
    """drops batches handed over by their owners, on its own thread"""

    def __init__(self, errors):
        self.q, self.errors = queue.Queue(), errors
        self.t = threading.Thread(target=self._run, name="releaser")
        self.t.start()

    def put(self, batch, keep=None, arrays=None, closed=None, want=None):
        self.q.put((batch, keep, arrays, closed, want))

    def _run(self):
        while True:
            item = self.q.get()
            if item is None:
                return
            batch, keep, arrays, closed, want = item
            try:
                if closed is not None:
                    assert closed.wait(300), "the owner never closed its decoder"
                batch.release()
                if arrays is not None:                  # the arrays still hold the batch, whose decoder is closed
                    assert arrays.to_pylist() == want, "Arrow array read after its decoder was closed differs"
            except BaseException:
                self.errors.append("releaser:\n" + traceback.format_exc())
            del item, batch, keep, arrays

    def close(self):
        self.q.put(None)
        self.t.join()


def _check_block(b, f, blk, what):
    info = b.info
    for k in INFO_KEYS:
        assert info[k] == blk.info[k], (what, k, info, blk.info)
    assert_columns_equal(b.to_host(), blk.cols, f.names, what)
    if blk.rows is not None:
        rows, offs = b.unsafe_rows(True, f.part)
        assert np.array_equal(offs, blk.rows[1]) and np.array_equal(rows, blk.rows[0]), f"{what}: UnsafeRows differ"


def read_file(native, f, on_device, rel, tag):
    """one reader task's file: decoder created, the file streamed through it in blocks, the decoder closed"""
    import torch
    dev = torch.from_numpy(f.data).cuda() if on_device else None
    dec = native.Decoder(f.sch, f.rt)
    closed = threading.Event()
    try:
        pending = []

        def resolve(i, b):
            blk = f.blocks[i]
            _check_block(b, f, blk, f"{tag} {f.name} block {i}")
            if i == 0 and f.arrow_col is not None:
                c = blk.cols[f.arrow_col]
                rel.put(b, dev, b.to_arrow()[f.arrow_col], closed, [c.get(r) for r in range(c.n_rows)])
            elif i % 3 == 1:
                rel.put(b, dev)                           # waited on, released by another thread
            else:
                b.release()

        for i, blk in enumerate(f.blocks):
            src = (dev.data_ptr() + blk.pos, blk.take, 1) if on_device else f.data[blk.pos:blk.pos + blk.take]
            b = dec.submit(src, is_final=blk.final)
            assert b.consumed() == blk.early, (tag, f.name, i, blk.early)
            b.to_host_async()
            pending.append((i, b))
            if len(pending) > 1:
                resolve(*pending.pop(0))
        while pending:
            resolve(*pending.pop(0))
        st = dec.stats()
        if f.name == "wide":
            assert st["general_path_batches"] > 0, (tag, st)
        elif not f.damaged:
            assert st["general_path_batches"] == 0 and st["speculative_submits"] > 0, (tag, f.name, st)
            if f.name == "utf8":
                assert st["transcode_reruns"] > 0, (tag, st)
            # a speculative submit handed over unresolved, released after the decoder is closed
            blk = f.blocks[0]
            src = (dev.data_ptr(), blk.take, 1) if on_device else f.data[:blk.take]
            rel.put(dec.submit(src, is_final=blk.final), dev)
    finally:
        dec.close()
        closed.set()


def reader_task(native, w, files, on_device, rel, tag):
    for j, nm in enumerate(files):
        read_file(native, w.files[nm], (on_device + j) % 2 == 0, rel, tag)


def _error_round(native, w, which, state, barrier):
    if barrier is not None:
        barrier.wait(120)
    if which == 0:
        with pytest.raises(native.TfrError) as ei:
            state.unsafe_rows(True)
        assert ei.value.code == A.TFR_E_UNSUPPORTED_TYPE and "'dec'" in str(ei.value) and "DecimalType" in str(ei.value), str(ei.value)
        assert "malformed" not in str(ei.value), str(ei.value)
    else:
        with pytest.raises(native.TfrError) as ei:
            state.encode_rows(w.bad_rows, w.bad_offs)
        assert ei.value.code == A.TFR_E_INVALID_ARG and ei.value.row == 50 and "malformed UnsafeRow" in str(ei.value), str(ei.value)
        assert "DecimalType" not in str(ei.value), str(ei.value)


def writer_task(native, w, which, barrier, tag):
    """encodes its jobs' columns and rows; between jobs, fails together with the other writer (barrier), each with its own error"""
    if which == 0:
        dec = native.Decoder(w.dec_sch)
        state, _ = dec.decode(w.dec_data)
    else:
        dec, state = None, native.Encoder(w.bad_sch)
    try:
        _error_round(native, w, which, state, barrier)
        for job in w.writers[which]:
            enc = native.Encoder(job.sch, job.rt)
            try:
                got = enc.encode(job.cols)
                assert got == job.want, f"{tag}: tfr_encode of {job.mean}-byte rows (record type {job.rt}) differs"
                enc.encode_rows(job.rows, job.offs)
                assert enc.result_host() == job.want, f"{tag}: tfr_encode_rows of {job.mean}-byte rows (record type {job.rt}) differs"
            finally:
                enc.close()
            _error_round(native, w, which, state, barrier)
    finally:
        if dec is not None:
            state.release()
            dec.close()
        else:
            state.close()


def infer_task(native, w, tag):
    for nm, (_, want) in w.infer:
        f = w.files[nm]
        inf = native.Infer(f.rt)
        try:
            pos = 0
            while True:
                take = min(f.block, len(f.data) - pos)
                final = pos + take == len(f.data)
                pos += inf.update_block(f.data[pos:pos + take], final)
                if final:
                    break
            assert pos == len(f.data) and inf.result() == want, (tag, nm)
        finally:
            inf.close()


def _tasks(native, w, rel, barrier_pair):
    tasks = [(f"reader {k}", lambda k=k: reader_task(native, w, w.readers[k], k % 2, rel, f"reader {k}")) for k in range(5)]
    tasks += [(f"writer {i}", lambda i=i: writer_task(native, w, i, barrier_pair, f"writer {i}")) for i in range(2)]
    tasks.append(("inference", lambda: infer_task(native, w, "inference")))
    assert len(tasks) == N_TASKS
    return tasks


def run_threads(native, w):
    """all tasks at once, started on a barrier; -> list of failures (with tracebacks)"""
    errors = []
    rel = Releaser(errors)
    start, pair = threading.Barrier(N_TASKS), threading.Barrier(2)

    def body(name, fn):
        try:
            start.wait(120)
            fn()
        except BaseException:
            errors.append(f"{name}:\n" + traceback.format_exc())
            start.abort()
            pair.abort()

    threads = [threading.Thread(target=body, args=t, name=t[0]) for t in _tasks(native, w, rel, pair)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    rel.close()
    return errors


def run_serial(native, w):
    """every task once more from one thread: a shared-memory opt-in left lower than a size the process believes it was
    granted fails here with TFR_E_CUDA"""
    errors = []
    rel = Releaser(errors)
    try:
        for name, fn in _tasks(native, w, rel, None):
            fn()
    finally:
        rel.close()
    assert not errors, "\n".join(errors)


# ---------------------------------------------------------------------------------------------------------------------
# tests
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def native():
    from spark_tfrecord_b200 import _native
    _native.lib()
    return _native


@pytest.fixture(scope="module")
def workload(oracle):
    return Workload(oracle)


def test_task_threads_then_serial_rerun(native, workload):
    t0 = time.time()
    errors = run_threads(native, workload)
    assert not errors, "\n".join(errors)
    t1 = time.time()
    run_serial(native, workload)
    print(f"prepare {workload.prep_seconds:.1f} s, threads {t1 - t0:.1f} s, serial {time.time() - t1:.1f} s")


def test_fresh_processes(native):
    """three new processes, where no kernel's shared-memory opt-in has been raised yet: the threads' first launches race"""
    for i in range(3):
        p = subprocess.run([sys.executable, os.path.abspath(__file__), "--child"], cwd=ROOT, capture_output=True, text=True, timeout=600)
        assert p.returncode == 0 and "child ok" in p.stdout, f"child {i}: exit {p.returncode}\n{p.stdout[-4000:]}\n{p.stderr[-8000:]}"


def _child():
    from oracle import oracle
    from spark_tfrecord_b200 import _native
    oracle.build()
    _native.lib()
    w = Workload(oracle)
    errors = run_threads(_native, w)
    if errors:
        print("\n".join(errors), file=sys.stderr)
        return 1
    run_serial(_native, w)
    print("child ok")
    return 0


if __name__ == "__main__" and "--child" in sys.argv:
    sys.exit(_child())
