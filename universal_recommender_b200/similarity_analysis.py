"""Python mirror of org.apache.mahout.math.cf.SimilarityAnalysis as the reference calls it
(src/main/scala/URAlgorithm.scala:323-329, 343-346), running on the H100 through the
C ABI of include/cco_b200.h.  Same names, argument meaning and error behaviour; the arithmetic is
the hand-written sm_90a path in csrc/ -- there is no CPU implementation in this package."""
from __future__ import annotations

import ctypes as C
import os
import queue
import re
import threading
import time
import weakref
from dataclasses import dataclass
from typing import Optional, Sequence

import numpy as np

from . import _native as N
from . import events as E
from .indexed_dataset import IndexedDataset

# device staging and host buffer size of a streamed export read (CcoContext.read_events): DESIGN.md section 8 has the
# sweep it was chosen from
DEFAULT_CHUNK_BYTES = 1 << 28


def _name_part(e: Exception, paths) -> None:
    """add the part file and its 0-based line to the message of a parse error of a multi-part read (counted only here)"""
    m = re.search(r"line (\d+)", str(e))
    if m is None or len(paths) < 2:
        return
    try:
        k, line = E.locate_line([E.part_lines(p) for p in paths], int(m.group(1)))
    except (OSError, ValueError):
        return
    e.args = (f"{e.args[0]} (part {paths[k]}, line {line})",)


@dataclass
class DownsamplableCrossOccurrenceDataset:
    """org.apache.mahout.math.cf.DownsamplableCrossOccurrenceDataset as constructed at
    URAlgorithm.scala:336-340 (defaults 500 / 50 / None)."""
    iD: IndexedDataset
    maxElementsPerRow: int = 500
    maxInterestingElements: int = 50
    minLLROpt: Optional[float] = None
    parOpts: object = None   # Spark partitioning hints: meaningless here, accepted and ignored


@dataclass
class TrainStats:
    n_users: int
    nnz_in_total: int
    nnz_downsampled: list
    products: list
    distinct_cells: list
    out_nnz: list
    llr_evaluated: list
    ms_h2d: float
    ms_prepare: float
    ms_cooccurrence: float
    ms_total: float
    ms_indicator: list
    n_kernel_launches: int
    ms_prep_stage: list = None


class CcoContext:
    """One GPU context (= cco_ctx_t).  One process per GPU; for world_size > 1 pass the 128-byte NCCL id
    from `CcoContext.nccl_unique_id()` of rank 0 (distribute it with any host transport)."""

    def __init__(self, device: int = 0, rank: int = 0, world_size: int = 1, nccl_unique_id: bytes | None = None,
                 devices: Sequence[int] | None = None, result_arena: np.ndarray | None = None):
        """devices=[...]: a GROUP context over several GPUs of this process (cco_create_group): train_csr then returns the
        merged model of all of them.  result_arena: a writable uint8 array (e.g. np.memmap of a /dev/shm file) the result
        arrays are placed in (cco_config_t.result_arena)."""
        L = N.lib()
        self._L = L
        self._uid = None
        self._arena = result_arena
        self.last_stats: TrainStats | None = None
        self._pinned_addr: dict = {}
        self._logs = weakref.WeakSet()   # an event log belongs to its context: close() frees the open ones first
        if devices is not None:
            h = C.c_void_p()
            arr = (C.c_int32 * len(devices))(*devices)
            N.check(L.cco_create_group(len(devices), arr, C.byref(h)))
            self._h = h
            self.rank, self.world_size, self.device, self.devices = 0, 1, devices[0], list(devices)
            return
        cfg = N.ConfigT(device, rank, world_size, 0, None, None, 0)
        if result_arena is not None:
            cfg.result_arena = result_arena.ctypes.data
            cfg.result_arena_bytes = result_arena.nbytes
        if world_size > 1:
            if nccl_unique_id is None or len(nccl_unique_id) != 128:
                raise N.CcoInvalidArgument(N.E_INVALID_ARG, "world_size > 1 needs the 128-byte nccl_unique_id")
            self._uid = (C.c_ubyte * 128).from_buffer_copy(nccl_unique_id)
            cfg.nccl_unique_id = C.cast(self._uid, C.POINTER(C.c_ubyte))
        h = C.c_void_p()
        N.check(L.cco_create(C.byref(cfg), C.byref(h)))
        self._h = h
        self.rank, self.world_size, self.device, self.devices = rank, world_size, device, [device]

    @staticmethod
    def nccl_unique_id() -> bytes:
        buf = (C.c_ubyte * 128)()
        N.check(N.lib().cco_nccl_unique_id(buf))
        return bytes(buf)

    def close(self):
        if getattr(self, "_h", None):
            for log in list(getattr(self, "_logs", ())):
                log.free()
            self._L.cco_destroy(self._h)
            self._h = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- pinned host buffers (what the JNI shim wraps as direct ByteBuffers) -------------------------
    def host_array(self, n: int, dtype) -> np.ndarray:
        dt = np.dtype(dtype)
        p = C.c_void_p()
        N.check(self._L.cco_host_alloc(self._h, max(n, 1) * dt.itemsize, C.byref(p)))
        buf = (C.c_byte * (max(n, 1) * dt.itemsize)).from_address(p.value)
        arr = np.frombuffer(buf, dtype=dt, count=n)
        self._pinned_addr[arr.ctypes.data if n else p.value] = p
        return arr

    def host_free(self, arr: np.ndarray):
        p = self._pinned_addr.pop(arr.ctypes.data, None)
        if p is not None:
            self._L.cco_host_free(self._h, p)

    # ---- the hot path ---------------------------------------------------------------------------------------
    def _csr_array(self, mats):
        n = len(mats)
        keep = []
        cm = (N.CsrT * n)()
        for i, (nr, nc, rp, ci) in enumerate(mats):
            rp = np.ascontiguousarray(rp, dtype=np.int64)
            ci = np.ascontiguousarray(ci, dtype=np.int32)
            keep.append((rp, ci))
            cm[i] = N.as_csr_t(nr, nc, rp, ci)
        return cm, keep

    @staticmethod
    def _params_array(params):
        return (N.ParamsT * len(params))(*[N.ParamsT(int(m), int(k), 0 if ml is None else 1, 0.0 if ml is None else float(ml))
                                           for (m, k, ml) in params])

    def _collect(self, res, n, copy_arrays=True, keep=False):
        """copy_arrays: numpy copies of the result arrays (default).  keep=True: zero-copy VIEWS of the library-owned pinned
        result buffers instead; the caller must call free_result(handle) when done (returns (views, handle))."""
        L = self._L
        try:
            out = []
            for i in range(n):
                rb, re_ = C.c_int64(), C.c_int64()
                N.check(L.cco_result_row_range(res, i, C.byref(rb), C.byref(re_)))
                nr, nc = C.c_int64(), C.c_int32()
                prp, pci, pll, pcn = C.POINTER(C.c_int64)(), C.POINTER(C.c_int32)(), C.POINTER(C.c_double)(), C.POINTER(C.c_int32)()
                N.check(L.cco_result_matrix(res, i, C.byref(nr), C.byref(nc), C.byref(prp), C.byref(pci), C.byref(pll), C.byref(pcn)))
                rp = np.ctypeslib.as_array(prp, shape=(nr.value + 1,))
                if not keep:
                    rp = rp.copy()
                nnz = int(rp[-1])
                if nnz and (copy_arrays or keep):
                    ci = np.ctypeslib.as_array(pci, shape=(nnz,))
                    ll = np.ctypeslib.as_array(pll, shape=(nnz,)) if pll else np.zeros(0, np.float64)
                    cn = np.ctypeslib.as_array(pcn, shape=(nnz,)) if pcn else np.zeros(0, np.int32)
                    if not keep:
                        ci, ll, cn = ci.copy(), ll.copy(), cn.copy()
                else:
                    ci, ll, cn = np.zeros(0, np.int32), np.zeros(0, np.float64), np.zeros(0, np.int32)
                out.append((rb.value, re_.value, nc.value, rp, ci, ll, cn))
            st = N.StatsT()
            N.check(L.cco_result_stats(res, C.byref(st)))
            self.last_stats = TrainStats(st.n_users, st.nnz_in_total, list(st.nnz_downsampled)[:n], list(st.products)[:n],
                                         list(st.distinct_cells)[:n], list(st.out_nnz)[:n], list(st.llr_evaluated)[:n], st.ms_h2d, st.ms_prepare,
                                         st.ms_cooccurrence, st.ms_total, list(st.ms_indicator)[:n], st.n_kernel_launches, list(st.ms_prep_stage))
            if keep:
                h, res = res, None
                return out, h
            return out
        finally:
            if res is not None:
                L.cco_result_free(res)

    def free_result(self, handle):
        self._L.cco_result_free(handle)

    # ---- next row (SURVEY.md 8f-3): PopModel rank histograms ---------------------------------------------------------------
    def pop_model(self, mode: str, items, times_ms, n_items: int, start_ms: int, end_ms: int):
        """PopModel.calcPopular / calcTrending / calcHot (PopModel.scala:113-182) -> {item index: score} for the items the
        reference's RDD would contain."""
        code = {"popular": 0, "trending": 1, "hot": 2}[mode]
        it = np.ascontiguousarray(items, dtype=np.int32)
        tm = np.ascontiguousarray(times_ms, dtype=np.int64)
        score = np.zeros(max(n_items, 1), dtype=np.float64)
        present = np.zeros(max(n_items, 1), dtype=np.uint8)
        N.check(self._L.cco_pop_model(self._h, code, len(it), it.ctypes.data_as(C.POINTER(C.c_int32)), tm.ctypes.data_as(C.POINTER(C.c_int64)),
                                      n_items, int(start_ms), int(end_ms), score.ctypes.data_as(C.POINTER(C.c_double)),
                                      present.ctypes.data_as(C.POINTER(C.c_ubyte))))
        return {int(j): float(score[j]) for j in np.nonzero(present[:n_items])[0]}

    # ---- next row (SURVEY.md 8f-2): the model as the Elasticsearch bulk body -------------------------------------------
    @staticmethod
    def _dictionary(ids):
        """list of id strings -> (DictionaryT, keep-alive): UTF-8 bytes + offsets"""
        enc = [x.encode("utf-8") for x in ids]
        off = np.zeros(len(enc) + 1, dtype=np.int64)
        np.cumsum([len(b) for b in enc], out=off[1:])
        blob = b"".join(enc)
        buf = C.create_string_buffer(blob, max(len(blob), 1))
        return N.DictionaryT(len(enc), off.ctypes.data_as(C.POINTER(C.c_int64)), C.cast(buf, C.c_char_p)), (off, buf)

    def _format_args(self, names, row_ids, col_ids, keep):
        n = len(names)
        rd, k = self._dictionary(row_ids)
        keep.append(k)
        cds = (N.DictionaryT * n)()
        for i, ids in enumerate(col_ids):
            cds[i], k = self._dictionary(ids)
            keep.append(k)
        nm = (C.c_char_p * n)(*[x.encode("utf-8") for x in names])
        return n, nm, rd, cds

    def _take_body(self, out, ln) -> bytes:
        try:
            return C.string_at(out.value, ln.value)
        finally:
            self._L.cco_host_free(self._h, out)

    def format_es_bulk(self, handle, names, row_ids, col_ids) -> bytes:
        """cco_format_es_bulk on a kept result (train_csr(..., keep=True)): one Elasticsearch bulk index action per row,
        `{"index":{"_id":id}}\\n{"id":id,"<event>":[ordered correlator ids],...}\\n` -- what toStringMapRDD + URModel.save +
        saveToEs produce for the reference (package.scala:82-110, URModel.scala:47-102, EsClient.scala:300-313)."""
        keep = []
        n, nm, rd, cds = self._format_args(names, row_ids, col_ids, keep)
        out, ln = C.c_void_p(), C.c_int64()
        N.check(self._L.cco_format_es_bulk(self._h, handle, n, nm, C.byref(rd), cds, C.byref(out), C.byref(ln)))
        return self._take_body(out, ln)

    @staticmethod
    def _model_args(properties, rankings, keep):
        """format_model's properties / rankings arguments -> (ItemPropertiesT or None, rankings list, RankingT array)"""
        p64, p32 = C.POINTER(C.c_int64), C.POINTER(C.c_int32)
        arr = lambda x, dt: np.ascontiguousarray(x, dtype=dt)
        ptr = lambda b: b.ctypes.data if len(b) else None
        props = None
        if properties is not None:
            fields, io, ib, fi, vo, vb = properties
            io, ib, fi, vo, vb = arr(io, np.int64), arr(ib, np.uint8), arr(fi, np.int32), arr(vo, np.int64), arr(vb, np.uint8)
            if len(io) < 1 or len(vo) != len(io) or len(fi) != len(io) - 1:
                raise N.CcoInvalidArgument(N.E_INVALID_ARG, "properties need n + 1 item and value offsets and n field indices")
            fn = (C.c_char_p * max(len(fields), 1))(*[f.encode("utf-8") for f in fields])
            keep.append((io, ib, fi, vo, vb, fn))
            props = N.ItemPropertiesT(len(io) - 1, io.ctypes.data_as(p64), ptr(ib), fi.ctypes.data_as(p32), vo.ctypes.data_as(p64), ptr(vb),
                                      len(fields), fn)
        rankings = list(rankings or [])
        rk = (N.RankingT * max(len(rankings), 1))()
        for k, (name, mode, start_ms, end_ms, streams) in enumerate(rankings):
            st = (N.RankingStreamT * max(len(streams), 1))()
            for q, (io, ib, tm) in enumerate(streams):
                io, ib, tm = arr(io, np.int64), arr(ib, np.uint8), arr(tm, np.int64)
                if len(io) < 1 or len(tm) != len(io) - 1:
                    raise N.CcoInvalidArgument(N.E_INVALID_ARG, f"ranking {k}: a stream needs n + 1 offsets and n times")
                keep.append((io, ib, tm))
                st[q] = N.RankingStreamT(len(tm), io.ctypes.data_as(p64), ptr(ib), tm.ctypes.data_as(p64))
            nb = name.encode("utf-8")
            keep.append((st, nb))
            rk[k] = N.RankingT(nb, N.POP_MODES.get(mode, -1), len(streams), int(start_ms), int(end_ms), st)
        return props, rankings, rk

    def format_model(self, handle, names, row_ids, col_ids, properties=None, rankings=None, log=None) -> bytes:
        """cco_format_model: format_es_bulk plus the item properties and PopModel rankings joined in by item id, and a
        document for every item without a row that has a property or a score (URAlgorithm.scala:351-367, URModel.scala:57-102).
        properties = (field_names, item_offsets int64[n + 1], item_bytes uint8[], field int32[n], value_offsets int64[n + 1],
        value_bytes uint8[]): n (item, field, JSON text) triples, the last of a repeated (item, field) wins.
        rankings = [(field name, "popular" | "trending" | "hot" | "random", start_ms, end_ms, [(item_offsets, item_bytes,
        time_ms int64[]) per event name])].  A "random" ranking (uniqueRank) scores the items of its streams' events in
        [start_ms, end_ms) plus every property item with n · 10^-15, n a hash of the id and the window (ur_model.random_rank);
        give it every event name's stream, as calcRandom reads them all.  Id columns in the layout of encode_ids.
        log=EventLog (cco_format_model_log): the properties are the log's, aggregated on the device (`properties` must be
        None), the streams come from the log in HBM, and a ranking is (field name, mode, start_ms, end_ms, [event names]);
        a "random" one reads every event name of the log."""
        keep = []
        n, nm, rd, cds = self._format_args(names, row_ids, col_ids, keep)
        if log is not None:
            if properties is not None:
                raise N.CcoInvalidArgument(N.E_INVALID_ARG, "with log=, the properties are the log's")
            rk = self._log_rankings(rankings, keep)
            out, ln = C.c_void_p(), C.c_int64()
            N.check(self._L.cco_format_model_log(self._h, handle, n, nm, C.byref(rd), cds, log._h, len(rankings or []), rk, C.byref(out),
                                                 C.byref(ln)))
            return self._take_body(out, ln)
        props, rankings, rk = self._model_args(properties, rankings, keep)
        out, ln = C.c_void_p(), C.c_int64()
        N.check(self._L.cco_format_model(self._h, handle, n, nm, C.byref(rd), cds, C.byref(props) if props is not None else None,
                                         len(rankings), rk, C.byref(out), C.byref(ln)))
        return self._take_body(out, ln)

    @staticmethod
    def _log_rankings(rankings, keep):
        """[(field name, mode, start_ms, end_ms, [event names])] -> LogRankingT array"""
        rankings = list(rankings or [])
        rk = (N.LogRankingT * max(len(rankings), 1))()
        for k, (name, mode, start_ms, end_ms, event_names) in enumerate(rankings):
            en = [x.encode("utf-8") for x in event_names]
            arr = (C.c_char_p * max(len(en), 1))(*en)
            nb = name.encode("utf-8")
            keep.append((arr, en, nb))
            rk[k] = N.LogRankingT(nb, N.POP_MODES.get(mode, -1), len(en), int(start_ms), int(end_ms), arr)
        return rk

    def read_events(self, src, chunk_bytes: Optional[int] = None, window: Optional[E.EventWindow] = None,
                    now_ms: Optional[int] = None, keep_history: bool = False) -> "EventLog":
        """A PredictionIO event export (JSON lines, as `pio export` writes them) parsed on the device.  src is one of
          - bytes or a buffer: one read (cco_event_log_read), or chunks of chunk_bytes when it is given;
          - a file path, a directory as `pio export` writes it (its part-* files in name order; events.export_parts) or a
            sequence of paths: streamed (cco_event_log_begin / _append / _finish) through two pinned buffers of
            chunk_bytes, one filled by a reader thread while the other is appended.  A part that does not end in '\\n' is
            followed by one.  A parse error names the part and its 0-based line besides the global line;
          - an iterable of buffers (a generator, say): streamed, each appended as it comes.
        chunk_bytes defaults to DEFAULT_CHUNK_BYTES for streamed sources; it is also the device staging.  The log is the one
        cco_event_log_read of the concatenated bytes gives.
        window: the DataSource's eventWindow (events.EventWindow; cco_event_log_begin_window), applied on the device while the
        export is read: events at or before now_ms - duration expire ($set / $unset excepted), and with removeDuplicates
        equal events collapse to the latest.  now_ms defaults to the wall clock; EventLog.window_stats() counts the drops.
        keep_history: keep every training event's time and line (cco_event_log_begin_ex, CCO_LOG_KEEP_HISTORY), which
        user_queries reads; a log read without it is exactly the log read before the option existed.
        -> EventLog (free with .free(), or use it as a context manager; close() of this context frees the logs still open)."""
        whole = isinstance(src, (bytes, bytearray, memoryview, np.ndarray)) and chunk_bytes is None
        if whole and window is None and not keep_history:
            buf = np.frombuffer(src, dtype=np.uint8) if not isinstance(src, np.ndarray) else np.ascontiguousarray(src, dtype=np.uint8)
            h = C.c_void_p()
            N.check(self._L.cco_event_log_read(self._h, buf.ctypes.data if len(buf) else None, len(buf), C.byref(h)))
            return self._adopt_log(h)
        chunk = int(chunk_bytes or (max(memoryview(src).nbytes, 1) if whole else DEFAULT_CHUNK_BYTES))
        paths = None
        if isinstance(src, (str, os.PathLike)):
            p = os.fspath(src)
            paths = E.export_parts(p) if os.path.isdir(p) else [p]
        elif isinstance(src, (list, tuple)) and all(isinstance(x, (str, os.PathLike)) for x in src):
            paths = [os.fspath(x) for x in src]
        h = C.c_void_p()
        w = None
        if window is not None:
            now = now_ms if now_ms is not None else int(time.time() * 1000)
            cutoff = window.cutoff_ms(now)
            w = N.EventWindowT(-(1 << 63) if cutoff is None else cutoff, 1 if window.removeDuplicates else 0, 0)
        if keep_history:
            N.check(self._L.cco_event_log_begin_ex(self._h, chunk, C.byref(w) if w is not None else None, N.LOG_KEEP_HISTORY, C.byref(h)))
        elif w is None:
            N.check(self._L.cco_event_log_begin(self._h, chunk, C.byref(h)))
        else:
            N.check(self._L.cco_event_log_begin_window(self._h, chunk, C.byref(w), C.byref(h)))
        try:
            if paths is not None:
                self._append_files(h, paths, chunk)
            else:
                for b in ([src] if isinstance(src, (bytes, bytearray, memoryview, np.ndarray)) else src):
                    buf = np.frombuffer(b, dtype=np.uint8) if not isinstance(b, np.ndarray) else np.ascontiguousarray(b, dtype=np.uint8)
                    if len(buf):
                        N.check(self._L.cco_event_log_append(h, buf.ctypes.data, len(buf)))
            try:
                N.check(self._L.cco_event_log_finish(h))
            except N.CcoError as e:
                if paths is not None:
                    _name_part(e, paths)
                raise
        except BaseException:
            self._L.cco_event_log_free(h)
            raise
        return self._adopt_log(h)

    def _adopt_log(self, h) -> "EventLog":
        log = EventLog(self, h, None)
        self._logs.add(log)
        return log

    def _append_files(self, h, paths, chunk: int):
        """append the files in order through two pinned buffers: a reader thread fills one while the other is appended
        (readinto and the ctypes call both release the GIL)"""
        bufs = [self.host_array(chunk, np.uint8) for _ in range(2)]
        free, full = queue.Queue(), queue.Queue()
        free.put(0)
        free.put(1)

        def reader():
            try:
                for path in paths:
                    last = b"\n"
                    with open(path, "rb", buffering=0) as f:
                        while True:
                            k = free.get()
                            if k is None:
                                return
                            n = f.readinto(memoryview(bufs[k]))
                            if not n:
                                free.put(k)
                                break
                            last = bytes(bufs[k][n - 1:n])
                            full.put((k, n))
                    if last != b"\n":   # parts never join lines
                        full.put((-1, 1))
                full.put(None)
            except BaseException as e:   # handed to the appending thread
                full.put(e)

        t = threading.Thread(target=reader, daemon=True)
        t.start()
        try:
            while True:
                item = full.get()
                if item is None:
                    break
                if isinstance(item, BaseException):
                    raise item
                k, n = item
                try:
                    if k < 0:
                        N.check(self._L.cco_event_log_append(h, b"\n", 1))
                    else:
                        N.check(self._L.cco_event_log_append(h, bufs[k].ctypes.data, n))
                except N.CcoError as e:
                    _name_part(e, paths)
                    raise
                if k >= 0:
                    free.put(k)
        finally:
            free.put(None)   # a reader still waiting for a buffer stops
            t.join()
            for b in bufs:
                self.host_free(b)

    def ingest_event_log(self, log: "EventLog", names: Sequence[str], min_events_per_user: int = 0):
        """cco_event_log_ingest: ingest_strings on the log's training events of `names` (type t = names[t]), from HBM.
        -> (dataset, user ids, [item ids per type]) as ingest_strings"""
        nm = (C.c_char_p * len(names))(*[x.encode("utf-8") for x in names])
        ds = C.c_void_p()
        N.check(self._L.cco_event_log_ingest(self._h, log._h, len(names), nm, int(min_events_per_user or 0), C.byref(ds)))
        dataset = (ds, len(names))
        try:
            users = self.dataset_dictionary(dataset, -1)
            items = [self.dataset_dictionary(dataset, t) for t in range(len(names))]
        except BaseException:
            self.free_dataset(dataset)
            raise
        return dataset, users, items

    def user_queries(self, log: "EventLog", ap, query=None, users=None, now_ms: Optional[int] = None, header: str = "{}"):
        """cco_event_log_user_queries: URAlgorithm.buildQuery for every user (ur_query.py restates it), from the history of a
        log read with keep_history=True.  ap: ur_algorithm.URAlgorithmParams; query: ur_query.UserQuery (None: defaults);
        users: the user ids, or None for every user with a training event of a query event name, by first line.
        -> (body, offsets int64[n + 1]): `header\nquery\n` records, the _msearch body; record r = body[offsets[r]:offsets[r + 1]].
        With users=None -> (body, offsets, users)."""
        from . import ur_query as Q
        plan = Q.plan(ap, query or Q.UserQuery(), now_ms)
        enc = lambda xs: [x.encode("utf-8", "surrogatepass") for x in xs]
        names, black = enc(plan.names), enc(plan.blacklist)
        nm = (C.c_char_p * max(len(names), 1))(*names)
        bl = (C.c_char_p * max(len(black), 1))(*black)
        lim = np.ascontiguousarray(plan.limits, dtype=np.int32) if plan.names else np.zeros(1, np.int32)
        lo, lb = encode_ids(list(plan.blacklist_items))
        qt = N.UserQueryT(len(names), plan.n_history, nm, lim.ctypes.data_as(C.POINTER(C.c_int32)), len(black), 1 if plan.in_must else 0, bl,
                          None if plan.boost is None else plan.boost.encode(), plan.head.encode("utf-8", "surrogatepass"),
                          plan.should.encode("utf-8", "surrogatepass"), plan.must.encode("utf-8", "surrogatepass"),
                          plan.must_not.encode("utf-8", "surrogatepass"), plan.sort.encode("utf-8", "surrogatepass"),
                          header.encode("utf-8", "surrogatepass"), len(lo) - 1, lo.ctypes.data_as(C.POINTER(C.c_int64)),
                          lb.ctypes.data if len(lb) else None)
        out, ln, off, n = C.c_void_p(), C.c_int64(), C.c_void_p(), C.c_int64()
        ud = N.DictionaryT()
        if users is None:
            N.check(self._L.cco_event_log_user_queries(self._h, log._h, C.byref(qt), 0, None, None, C.byref(out), C.byref(ln), C.byref(off),
                                                       C.byref(n), C.byref(ud)))
        else:
            uo, ub = encode_ids(list(users))
            N.check(self._L.cco_event_log_user_queries(self._h, log._h, C.byref(qt), len(uo) - 1, uo.ctypes.data_as(C.POINTER(C.c_int64)),
                                                       ub.ctypes.data if len(ub) else None, C.byref(out), C.byref(ln), C.byref(off),
                                                       C.byref(n), None))
        offsets = np.ctypeslib.as_array(C.cast(off, C.POINTER(C.c_int64)), shape=(n.value + 1,)).copy()
        self._L.cco_host_free(self._h, off)
        body = self._take_body(out, ln)
        if users is not None:
            return body, offsets
        uoff = np.ctypeslib.as_array(ud.offsets, shape=(ud.n + 1,)).copy()
        addr = C.c_void_p.from_buffer(ud, N.DictionaryT.bytes.offset).value
        ids = decode_ids(uoff, C.string_at(addr, int(uoff[-1])) if uoff[-1] else b"")
        self._L.cco_host_free(self._h, C.cast(ud.offsets, C.c_void_p))
        self._L.cco_host_free(self._h, C.c_void_p(addr))
        return body, offsets, ids

    def item_queries(self, index_body: bytes, ap, query=None, items=None, now_ms: Optional[int] = None, header: str = "{}"):
        """cco_item_queries: URAlgorithm.buildQuery for item queries (ur_query.py restates it), the similar items read from a
        model index bulk body (as format_model / rerank_model write it).  ap: ur_algorithm.URAlgorithmParams; query:
        ur_query.ItemQuery (None: defaults); items: the item ids, or None for every document, in body order.
        -> (body, offsets int64[n + 1]): `header\nquery\n` records, the _msearch body; record r = body[offsets[r]:offsets[r + 1]].
        With items=None -> (body, offsets, items)."""
        from . import ur_query as Q
        p = Q.item_plan(ap, query, now_ms)
        enc = lambda x: x.encode("utf-8", "surrogatepass")
        names = [enc(n) for n in p.names]
        nm = (C.c_char_p * max(len(names), 1))(*names)
        def column(ids):   # ids compare as UTF-8 bytes, a lone surrogate in its 3-byte form
            b = [enc(x) for x in ids]
            o = np.zeros(len(b) + 1, dtype=np.int64)
            np.cumsum([len(x) for x in b], out=o[1:])
            return o, np.frombuffer(b"".join(b), dtype=np.uint8)

        def text(b: bytes) -> str:
            try:
                return b.decode("utf-8", "surrogatepass")
            except UnicodeDecodeError:
                return b.decode("utf-8", "surrogateescape")
        lo, lb = column(p.blacklist_items)
        qt = N.ItemQueryT(len(names), nm, p.max_query_events, 1 if p.in_must else 0, None if p.boost is None else p.boost.encode(),
                          1 if p.exclude_self else 0, enc(p.head), enc(p.should_head), enc(p.should), enc(p.must_head), enc(p.must),
                          enc(p.must_not), enc(p.sort), enc(header), len(lo) - 1, lo.ctypes.data_as(C.POINTER(C.c_int64)),
                          lb.ctypes.data if len(lb) else None)
        index_body = bytes(index_body)
        out, ln, off, n = C.c_void_p(), C.c_int64(), C.c_void_p(), C.c_int64()
        idd = N.DictionaryT()
        if items is None:
            N.check(self._L.cco_item_queries(self._h, index_body, len(index_body), C.byref(qt), 0, None, None, C.byref(out), C.byref(ln),
                                             C.byref(off), C.byref(n), C.byref(idd)))
        else:
            io, ib = column(list(items))
            N.check(self._L.cco_item_queries(self._h, index_body, len(index_body), C.byref(qt), len(io) - 1,
                                             io.ctypes.data_as(C.POINTER(C.c_int64)), ib.ctypes.data if len(ib) else None, C.byref(out),
                                             C.byref(ln), C.byref(off), C.byref(n), None))
        offsets = np.ctypeslib.as_array(C.cast(off, C.POINTER(C.c_int64)), shape=(n.value + 1,)).copy()
        self._L.cco_host_free(self._h, off)
        body = self._take_body(out, ln)
        if items is not None:
            return body, offsets
        ioff = np.ctypeslib.as_array(idd.offsets, shape=(idd.n + 1,)).copy()
        addr = C.c_void_p.from_buffer(idd, N.DictionaryT.bytes.offset).value
        blob = C.string_at(addr, int(ioff[-1])) if ioff[-1] else b""
        ids = [text(blob[a:b]) for a, b in zip(ioff[:-1].tolist(), ioff[1:].tolist())]
        self._L.cco_host_free(self._h, C.cast(idd.offsets, C.c_void_p))
        self._L.cco_host_free(self._h, C.c_void_p(addr))
        return body, offsets, ids

    def rerank_model(self, body: bytes, properties=None, rankings=None, log=None) -> bytes:
        """cco_rerank_model: calcPop (URAlgorithm.scala:375-399, recsModel "backfill") on an existing index.  body = the
        Elasticsearch bulk body of the current model, as format_model writes it; properties and rankings as in format_model.
        Every old document keeps its members and gets the rankings; a fresh property is added only where the old document
        has no member of that name, and an old rank member stays when the item has no score in the new ranking (include/
        cco_b200.h states the grammar, precedence and order).  Items with a property or a score but no old document are
        appended as format_model writes them.  log=EventLog: properties and rankings as in format_model(log=...)."""
        keep = []
        body = bytes(body)
        if log is not None:
            if properties is not None:
                raise N.CcoInvalidArgument(N.E_INVALID_ARG, "with log=, the properties are the log's")
            rk = self._log_rankings(rankings, keep)
            out, ln = C.c_void_p(), C.c_int64()
            N.check(self._L.cco_rerank_model_log(self._h, body, len(body), log._h, len(rankings or []), rk, C.byref(out), C.byref(ln)))
            return self._take_body(out, ln)
        props, rankings, rk = self._model_args(properties, rankings, keep)
        out, ln = C.c_void_p(), C.c_int64()
        N.check(self._L.cco_rerank_model(self._h, body, len(body), C.byref(props) if props is not None else None, len(rankings), rk,
                                         C.byref(out), C.byref(ln)))
        return self._take_body(out, ln)

    def train_csr(self, mats: Sequence[tuple[int, int, np.ndarray, np.ndarray]], params: Sequence[tuple[int, int, Optional[float]]],
                  seed: int, flags: int = 0, copy_arrays: bool = True, keep: bool = False):
        """Raw entry (cco_train): mats = [(n_rows, n_cols, row_ptr int64, col_idx int32)], params = [(m, k, minLLR|None)].
        -> list of (row_begin, row_end, n_cols, row_ptr, col_idx, llr, count) numpy copies, one per matrix
        (keep=True: zero-copy views + a handle for free_result)."""
        cm, alive = self._csr_array(mats)
        res = C.c_void_p()
        N.check(self._L.cco_train(self._h, len(mats), cm, self._params_array(params), C.c_int32(_to_i32(seed)), flags,
                                  C.byref(res)))
        return self._collect(res, len(mats), copy_arrays, keep)

    # ---- split form: matrices resident in HBM across trains ---------------------------------------------
    def upload(self, mats, flags: int = 0):
        cm, keep = self._csr_array(mats)
        ds = C.c_void_p()
        N.check(self._L.cco_dataset_upload(self._h, len(mats), cm, flags, C.byref(ds)))
        return (ds, len(mats))

    def train_dataset(self, dataset, params, seed: int, flags: int = 0, copy_arrays: bool = True, keep: bool = False):
        """cco_train_dataset on a resident dataset -> as train_csr (keep=True: zero-copy views + a handle for free_result,
        e.g. for format_es_bulk)."""
        ds, n = dataset
        res = C.c_void_p()
        N.check(self._L.cco_train_dataset(self._h, ds, self._params_array(params), C.c_int32(_to_i32(seed)), flags, C.byref(res)))
        return self._collect(res, n, copy_arrays, keep)

    def ingest(self, events, n_users_raw: int, min_events_per_user: int = 0):
        """Preparator.prepare on the device (SURVEY.md 8f-1).  events = [(users int64[], items int32[], n_items_raw)], type 0
        = primary.  -> (dataset for train_dataset, user_map int32[n_users_raw], [item_map int32[n_items_raw]])."""
        n = len(events)
        keep, ev = [], (N.EventsT * n)()
        item_maps = [np.zeros(max(ni, 1), dtype=np.int32) for (_, _, ni) in events]
        for t, (u, i, ni) in enumerate(events):
            u = np.ascontiguousarray(u, dtype=np.int64)
            i = np.ascontiguousarray(i, dtype=np.int32)
            keep.append((u, i))
            ev[t] = N.EventsT(len(u), u.ctypes.data_as(C.POINTER(C.c_int64)), i.ctypes.data_as(C.POINTER(C.c_int32)), ni)
        user_map = np.zeros(max(n_users_raw, 1), dtype=np.int32)
        maps = (C.POINTER(C.c_int32) * n)(*[m.ctypes.data_as(C.POINTER(C.c_int32)) for m in item_maps])
        ds = C.c_void_p()
        N.check(self._L.cco_ingest(self._h, n, ev, n_users_raw, min_events_per_user, user_map.ctypes.data_as(C.POINTER(C.c_int32)),
                                   maps, C.byref(ds)))
        return (ds, n), user_map[:n_users_raw], [m[:ni] for m, (_, _, ni) in zip(item_maps, events)]

    def ingest_strings(self, columns, min_events_per_user: int = 0):
        """Preparator.prepare on the device from string ids (cco_ingest_strings).  columns = one (user_offsets int64[n + 1],
        user_bytes uint8[], item_offsets int64[n + 1], item_bytes uint8[]) per event type, type 0 = primary, in the layout
        encode_ids produces (and Arrow large_string columns have).  Pinned arrays (host_array) copy at full PCIe speed.
        -> (dataset for train_dataset, user ids list[str], [item ids list[str] per type]), dictionaries in the order of
        preparator.prepare."""
        dataset = self.ingest_strings_dataset(columns, min_events_per_user)
        try:
            users = self.dataset_dictionary(dataset, -1)
            items = [self.dataset_dictionary(dataset, t) for t in range(dataset[1])]
        except BaseException:
            self.free_dataset(dataset)
            raise
        return dataset, users, items

    def ingest_strings_dataset(self, columns, min_events_per_user: int = 0):
        """ingest_strings without decoding the dictionaries: -> the resident dataset (dictionaries via dataset_dictionary)"""
        n = len(columns)
        keep, ev = [], (N.StringEventsT * n)()
        p64 = C.POINTER(C.c_int64)
        as_u8 = lambda b: np.frombuffer(b, dtype=np.uint8) if isinstance(b, (bytes, bytearray)) else np.ascontiguousarray(b, dtype=np.uint8)
        for t, (uo, ub, io, ib) in enumerate(columns):
            uo = np.ascontiguousarray(uo, dtype=np.int64)
            io = np.ascontiguousarray(io, dtype=np.int64)
            ub, ib = as_u8(ub), as_u8(ib)
            if len(uo) < 1 or len(uo) != len(io):
                raise N.CcoInvalidArgument(N.E_INVALID_ARG, f"type {t}: user and item offsets need n_events + 1 entries each")
            keep.append((uo, ub, io, ib))
            ev[t] = N.StringEventsT(len(uo) - 1, uo.ctypes.data_as(p64), ub.ctypes.data if len(ub) else None,
                                    io.ctypes.data_as(p64), ib.ctypes.data if len(ib) else None)
        ds = C.c_void_p()
        N.check(self._L.cco_ingest_strings(self._h, n, ev, int(min_events_per_user or 0), C.byref(ds)))
        return (ds, n)

    def dataset_dictionary(self, dataset, which: int) -> list[str]:
        """the user dictionary (which = -1) or the item dictionary of type `which` of a string-ingested dataset"""
        d = N.DictionaryT()
        N.check(self._L.cco_dataset_dictionary(dataset[0], which, C.byref(d)))
        off = np.ctypeslib.as_array(d.offsets, shape=(d.n + 1,)).copy()
        nb = int(off[-1])
        # the raw pointer: reading the c_char_p field would stop at the first NUL byte, and ids may contain NULs
        addr = C.c_void_p.from_buffer(d, N.DictionaryT.bytes.offset).value
        blob = C.string_at(addr, nb) if nb else b""
        return decode_ids(off, blob)

    def synth_dataset(self, types, n_users_raw: int, user_cdf: np.ndarray, user_perm: np.ndarray, min_events_per_user: int = 0,
                      raw_item_space: bool = False):
        """Bench/test utility (cco_synth_ingest): the synthetic event streams of synth.py generated in HBM and ingested there.
        types = [(n_events, seed, item_cdf float64[], item_perm int32[])].  -> resident dataset for train_dataset."""
        n = len(types)
        keep, tt = [], (N.SynthTypeT * n)()
        for t, (ne, seed, icdf, iperm) in enumerate(types):
            icdf = np.ascontiguousarray(icdf, dtype=np.float64)
            iperm = np.ascontiguousarray(iperm, dtype=np.int32)
            keep.append((icdf, iperm))
            tt[t] = N.SynthTypeT(int(ne), int(seed), len(icdf), 0, icdf.ctypes.data_as(C.POINTER(C.c_double)),
                                 iperm.ctypes.data_as(C.POINTER(C.c_int32)))
        ucdf = np.ascontiguousarray(user_cdf, dtype=np.float64)
        uperm = np.ascontiguousarray(user_perm, dtype=np.int32)
        ds = C.c_void_p()
        N.check(self._L.cco_synth_ingest(self._h, n, tt, n_users_raw, ucdf.ctypes.data_as(C.POINTER(C.c_double)),
                                         uperm.ctypes.data_as(C.POINTER(C.c_int32)), min_events_per_user, 1 if raw_item_space else 0,
                                         C.byref(ds)))
        return (ds, n)

    def dataset_shape(self, dataset, i: int):
        nr, nc, nnz = C.c_int64(), C.c_int32(), C.c_int64()
        N.check(self._L.cco_dataset_shape(dataset[0], i, C.byref(nr), C.byref(nc), C.byref(nnz)))
        return nr.value, nc.value, nnz.value

    def dataset_to_host(self, dataset, i: int, pinned: bool = True):
        """(n_rows, n_cols, row_ptr, col_idx) of matrix i of a resident dataset in (pinned) host arrays."""
        nr, nc, nnz = self.dataset_shape(dataset, i)
        rp = self.host_array(nr + 1, np.int64) if pinned else np.zeros(nr + 1, np.int64)
        ci = self.host_array(nnz, np.int32) if pinned else np.zeros(max(nnz, 1), np.int32)[:nnz]
        N.check(self._L.cco_dataset_copy_to_host(dataset[0], i, rp.ctypes.data_as(C.POINTER(C.c_int64)),
                                                 ci.ctypes.data_as(C.POINTER(C.c_int32)) if nnz else None))
        return nr, nc, rp, ci

    def dataset_matrix(self, dataset, i: int):
        """(n_rows, n_cols, row_ptr, col_idx) of matrix i of a resident dataset, copied to the host (tests)."""
        ds, _ = dataset
        nr, nc, nnz = C.c_int64(), C.c_int32(), C.c_int64()
        N.check(self._L.cco_dataset_shape(ds, i, C.byref(nr), C.byref(nc), C.byref(nnz)))
        prp, pci = C.POINTER(C.c_int64)(), C.POINTER(C.c_int32)()
        N.check(self._L.cco_dataset_download(ds, i, C.byref(prp), C.byref(pci)))
        rp = np.ctypeslib.as_array(prp, shape=(nr.value + 1,)).copy()
        ci = np.ctypeslib.as_array(pci, shape=(nnz.value,)).copy() if nnz.value else np.zeros(0, np.int32)
        self._L.cco_free(prp)
        self._L.cco_free(pci)
        return nr.value, nc.value, rp, ci

    def free_dataset(self, dataset):
        self._L.cco_dataset_free(dataset[0])

    def timer_start(self):
        N.check(self._L.cco_timer_start(self._h))

    def timer_stop(self) -> float:
        ms = C.c_float()
        N.check(self._L.cco_timer_stop(self._h, C.byref(ms)))
        return ms.value

    # ---- debug / parity entries ---------------------------------------------------------------------------
    def debug_llr(self, k11, k12, k21, k22, flags: int = 0) -> np.ndarray:
        a = [np.ascontiguousarray(x, dtype=np.int64) for x in (k11, k12, k21, k22)]
        out = np.zeros(len(a[0]), dtype=np.float64)
        p = C.POINTER(C.c_int64)
        N.check(self._L.cco_debug_llr(self._h, len(out), *[x.ctypes.data_as(p) for x in a], flags,
                                      out.ctypes.data_as(C.POINTER(C.c_double))))
        return out

    def debug_string_ids(self, offsets, data, hash_bits: int = 64) -> np.ndarray:
        """cco_debug_string_ids: dictionary id (first-appearance order) of every id of one column, hash cut to hash_bits"""
        off = np.ascontiguousarray(offsets, dtype=np.int64)
        b = np.ascontiguousarray(data, dtype=np.uint8)
        ids = np.zeros(max(len(off) - 1, 1), dtype=np.int32)
        N.check(self._L.cco_debug_string_ids(self._h, len(off) - 1, off.ctypes.data_as(C.POINTER(C.c_int64)), b.ctypes.data if len(b) else None,
                                             hash_bits, ids.ctypes.data_as(C.POINTER(C.c_int32))))
        return ids[:len(off) - 1]

    def debug_rank_text(self, values, scale: int = 0):
        """cco_debug_rank_text: the model index's rank number text of every values[i] * 10^-scale (scale 0 or 15), as the
        document kernels write it -> (offsets int64[n + 1], bytes uint8[])"""
        v = np.ascontiguousarray(values, dtype=np.int64)
        off = np.zeros(len(v) + 1, dtype=np.int64)
        b = np.zeros(max(32 * len(v), 1), dtype=np.uint8)
        N.check(self._L.cco_debug_rank_text(self._h, len(v), v.ctypes.data_as(C.POINTER(C.c_int64)), scale,
                                            off.ctypes.data_as(C.POINTER(C.c_int64)), b.ctypes.data))
        return off, b[:off[-1]]

    def debug_downsample(self, n_rows, n_cols, row_ptr, col_idx, max_interactions: int, seed: int, flags: int = 0):
        rp = np.ascontiguousarray(row_ptr, dtype=np.int64)
        ci = np.ascontiguousarray(col_idx, dtype=np.int32)
        m = N.as_csr_t(n_rows, n_cols, rp, ci)
        orp, oci = C.POINTER(C.c_int64)(), C.POINTER(C.c_int32)()
        raw = np.zeros(max(n_cols, 1), np.int32)
        new = np.zeros(max(n_cols, 1), np.int32)
        N.check(self._L.cco_debug_downsample(self._h, C.byref(m), max_interactions, _to_i32(seed), flags, C.byref(orp),
                                             C.byref(oci), raw.ctypes.data_as(C.POINTER(C.c_int32)),
                                             new.ctypes.data_as(C.POINTER(C.c_int32))))
        r = np.ctypeslib.as_array(orp, shape=(n_rows + 1,)).copy()
        nnz = int(r[-1])
        c = np.ctypeslib.as_array(oci, shape=(nnz,)).copy() if nnz else np.zeros(0, np.int32)
        self._L.cco_free(orp)
        self._L.cco_free(oci)
        return r, c, raw[:n_cols], new[:n_cols]

    def debug_downsample_block(self, n_rows, n_cols, row_ptr, col_idx, row_lo: int, row_hi: int, raw_col_counts,
                               max_interactions: int, seed: int, flags: int = 0):
        """cco_debug_downsample_block: users [row_lo, row_hi) sampled as the rank owning them samples them, with the whole
        matrix's raw column counts -> (kept per user int64[n_rows], the block's kept columns, its post-sample column counts)."""
        rp = np.ascontiguousarray(row_ptr, dtype=np.int64)
        ci = np.ascontiguousarray(col_idx, dtype=np.int32)
        m = N.as_csr_t(n_rows, n_cols, rp, ci)
        raw = np.zeros(max(n_cols, 1), np.int32)
        raw[:n_cols] = raw_col_counts
        kept = np.zeros(max(n_rows, 1), np.int64)
        new = np.zeros(max(n_cols, 1), np.int32)
        oci = C.POINTER(C.c_int32)()
        N.check(self._L.cco_debug_downsample_block(self._h, C.byref(m), row_lo, row_hi, raw.ctypes.data_as(C.POINTER(C.c_int32)),
                                                   max_interactions, _to_i32(seed), flags, kept.ctypes.data_as(C.POINTER(C.c_int64)),
                                                   C.byref(oci), new.ctypes.data_as(C.POINTER(C.c_int32))))
        n = int(kept[row_lo:row_hi].sum())
        c = np.ctypeslib.as_array(oci, shape=(n,)).copy() if n else np.zeros(0, np.int32)
        self._L.cco_free(oci)
        return kept[:n_rows], c, new[:n_cols]

    def debug_cooccurrence(self, a, b):
        """a, b = (n_rows, n_cols, row_ptr, col_idx) canonical binary matrices -> (row_ptr, col_idx, count) of A^T B."""
        keep = []
        cs = []
        for (nr, nc, rp, ci) in (a, b):
            rp = np.ascontiguousarray(rp, dtype=np.int64)
            ci = np.ascontiguousarray(ci, dtype=np.int32)
            keep.append((rp, ci))
            cs.append(N.as_csr_t(nr, nc, rp, ci))
        orp, oci, ocn = C.POINTER(C.c_int64)(), C.POINTER(C.c_int32)(), C.POINTER(C.c_int32)()
        N.check(self._L.cco_debug_cooccurrence(self._h, C.byref(cs[0]), C.byref(cs[1]), C.byref(orp), C.byref(oci), C.byref(ocn)))
        r = np.ctypeslib.as_array(orp, shape=(a[1] + 1,)).copy()
        nnz = int(r[-1])
        c = np.ctypeslib.as_array(oci, shape=(nnz,)).copy() if nnz else np.zeros(0, np.int32)
        n = np.ctypeslib.as_array(ocn, shape=(nnz,)).copy() if nnz else np.zeros(0, np.int32)
        for p in (orp, oci, ocn):
            self._L.cco_free(p)
        return r, c, n


@dataclass
class EventLogInfo:
    n_lines: int
    names: list          # distinct event names, first appearance order
    n_training: list     # per name
    n_ranking: list      # per name
    n_property_events: int
    n_property_items: int    # items whose aggregated properties exist (each gets a document)
    n_property_fields: int
    n_ignored: int


class EventLog:
    """A PredictionIO event export resident on one GPU (cco_event_log_t), from CcoContext.read_events."""

    def __init__(self, ctx: CcoContext, h, pinned: Optional[np.ndarray]):
        self._ctx, self._h, self._pinned = ctx, h, pinned

    def _info(self):
        i = N.EventLogInfoT()
        N.check(self._ctx._L.cco_event_log_info(self._h, C.byref(i)))
        return i

    def info(self) -> EventLogInfo:
        i = self._info()
        g = i.names.n
        off = np.ctypeslib.as_array(i.names.offsets, shape=(g + 1,)).copy() if g else np.zeros(1, np.int64)
        addr = C.c_void_p.from_buffer(i.names, N.DictionaryT.bytes.offset).value
        names = decode_ids(off, C.string_at(addr, int(off[-1])) if off[-1] else b"")
        per = lambda p: np.ctypeslib.as_array(p, shape=(g,)).tolist() if g else []
        return EventLogInfo(i.n_lines, names, per(i.n_training), per(i.n_ranking), i.n_property_events, i.n_property_items,
                            i.n_property_fields, i.n_ignored)

    def window_stats(self) -> tuple[int, int]:
        """(expired, duplicates): the lines the eventWindow dropped (both 0 for a read without one)"""
        x, d = C.c_int64(), C.c_int64()
        N.check(self._ctx._L.cco_event_log_window_stats(self._h, C.byref(x), C.byref(d)))
        return x.value, d.value

    def free(self):
        if getattr(self, "_h", None):
            self._ctx._L.cco_event_log_free(self._h)
            self._h = None
            self._ctx._logs.discard(self)
            if self._pinned is not None:
                self._ctx.host_free(self._pinned)
                self._pinned = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.free()


def encode_ids(ids: Sequence[str]) -> tuple[np.ndarray, np.ndarray]:
    """id strings -> (offsets int64[n + 1], bytes uint8[]): UTF-8, id i = bytes[offsets[i]:offsets[i + 1]] (the Arrow
    large_string layout cco_ingest_strings takes)."""
    ids = ids if isinstance(ids, list) else list(ids)
    joined = "".join(ids)
    if joined.isascii():   # one byte per character: lengths are str lengths, one encode for the whole column
        lens = np.fromiter(map(len, ids), dtype=np.int64, count=len(ids))
        blob = joined.encode("ascii")
    else:
        enc = [x.encode("utf-8") for x in ids]
        lens = np.fromiter(map(len, enc), dtype=np.int64, count=len(enc))
        blob = b"".join(enc)
    off = np.zeros(len(ids) + 1, dtype=np.int64)
    np.cumsum(lens, out=off[1:])
    return off, np.frombuffer(blob, dtype=np.uint8)


def decode_ids(offsets: np.ndarray, blob: bytes) -> list[str]:
    """inverse of encode_ids (bytes that are not UTF-8 decode with surrogateescape, so they round-trip too)"""
    off = np.asarray(offsets, dtype=np.int64)
    base = int(off[0]) if len(off) else 0
    if blob.isascii():
        text = blob.decode("ascii")
        return [text[a - base:b - base] for a, b in zip(off[:-1].tolist(), off[1:].tolist())]
    return [blob[a - base:b - base].decode("utf-8", "surrogateescape") for a, b in zip(off[:-1].tolist(), off[1:].tolist())]


def _to_i32(seed: int) -> int:
    """`.toInt` of a Long seed as in URAlgorithm.scala:325,345 (wraps)."""
    s = int(seed) & 0xffffffff
    return s - (1 << 32) if s & 0x80000000 else s


_default_ctx: CcoContext | None = None


def default_context() -> CcoContext:
    """Process-wide single-GPU context on device 0 (multi-GPU jobs build theirs with distributed.context_from_env)."""
    global _default_ctx
    if _default_ctx is None:
        _default_ctx = CcoContext(device=0)
    return _default_ctx


class SimilarityAnalysis:
    """Drop-in for the two static calls of URAlgorithm.calcAll."""

    @staticmethod
    def crossOccurrenceDownsampled(datasets: Sequence[DownsamplableCrossOccurrenceDataset], randomSeed: int = 0xdeadbeef,
                                   ctx: CcoContext | None = None, flags: int = 0) -> list[IndexedDataset]:
        """URAlgorithm.scala:343-346.  datasets[0] is the primary (A).  Returns one IndexedDataset per input,
        rowIDs = A.columnIDs, columnIDs = B_i.columnIDs, values = LLR, rows sorted (llr desc, col asc)."""
        if len(datasets) == 0:
            raise N.CcoInvalidArgument(N.E_INVALID_ARG, "datasets is empty")
        ctx = ctx or default_context()
        a = datasets[0].iD
        mats = [(d.iD.n_rows, d.iD.n_cols, d.iD.row_ptr, d.iD.col_idx) for d in datasets]
        params = [(d.maxElementsPerRow, d.maxInterestingElements, d.minLLROpt) for d in datasets]
        res = ctx.train_csr(mats, params, randomSeed, flags)
        out = []
        for d, (rb, re_, nc, rp, ci, ll, cn) in zip(datasets, res):
            if ctx.world_size == 1:
                out.append(a.create(rp, ci, a.column_ids, d.iD.column_ids, ll, cn))
            else:   # this rank's row slice, padded to the full primary-item row space
                full = np.zeros(a.n_cols + 1, dtype=np.int64)
                full[rb + 1:re_ + 1] = rp[1:]
                full[re_ + 1:] = rp[-1]
                out.append(a.create(full, ci, a.column_ids, d.iD.column_ids, ll, cn))
        return out

    @staticmethod
    def cooccurrencesIDSs(indexedDatasets: Sequence[IndexedDataset], randomSeed: int = 0xdeadbeef,
                          maxInterestingItemsPerThing: int = 50, maxNumInteractions: int = 500,
                          ctx: CcoContext | None = None, flags: int = 0) -> list[IndexedDataset]:
        """URAlgorithm.scala:323-329: one global (k, m) for every matrix."""
        ds = [DownsamplableCrossOccurrenceDataset(i, maxNumInteractions, maxInterestingItemsPerThing, None)
              for i in indexedDatasets]
        return SimilarityAnalysis.crossOccurrenceDownsampled(ds, randomSeed, ctx, flags)
