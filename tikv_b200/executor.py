"""Host-side mirror of the reference's operator interface on top of the C ABI.

`BatchExecutor` follows trait BatchExecutor (components/tidb_query_executors/src/interface.rs:36-97):
schema(), next_batch(scan_rows) -> BatchExecuteResult, collect_exec_stats(), can_be_cached().
`DagHandler.handle_request()` follows BatchDagHandler (src/coprocessor/dag/mod.rs:155-192) and
`checksum()` follows ChecksumContext::handle_request (src/coprocessor/checksum.rs:59-98).
"""
import ctypes as C

import numpy as np

from . import ffi
from .plan import key_ranges


class B2Error(Exception):
    def __init__(self, status, message, mysql_code=0, entry_index=None):
        super().__init__(f"[status {status}] {message}")
        self.status, self.message, self.mysql_code, self.entry_index = status, message, mysql_code, entry_index


def _decimal_to_int(raw40):
    """b2_decimal (40 raw bytes, integer decimals) -> python int, independent of the C++ code."""
    int_cnt, frac_cnt, _, neg = raw40[0], raw40[1], raw40[2], raw40[3]
    words = np.frombuffer(raw40[4:40], dtype="<u4")
    n = (int_cnt + 8) // 9
    v = 0
    for i in range(n):
        v = v * 10 ** 9 + int(words[i])
    assert frac_cnt == 0
    return -v if neg else v


def _decimal_value(raw40):
    """b2_decimal -> python int (no fraction digits) or decimal.Decimal."""
    import decimal
    int_cnt, frac_cnt, neg = raw40[0], raw40[1], raw40[3]
    if frac_cnt == 0:
        return _decimal_to_int(raw40)
    words = np.frombuffer(raw40[4:40], dtype="<u4")
    iw, fw = (int_cnt + 8) // 9, (frac_cnt + 8) // 9
    v = 0
    for w in words[:iw + fw]:
        v = v * 10 ** 9 + int(w)
    v //= 10 ** (fw * 9 - frac_cnt)
    return decimal.Decimal(-v if neg else v).scaleb(-frac_cnt, decimal.Context(prec=200))


def raw_cell_values(kind, data, offsets, non_null):
    """Cells of a BYTES / JSON (heap + offsets) or TIME / DURATION / DECIMAL (fixed cells) column as python values:
    bytes, the u64 CoreTime bit field, i64 nanoseconds, int / decimal.Decimal; None = NULL."""
    n = len(non_null)
    if kind in (ffi.COL_BYTES, ffi.COL_JSON):
        return [bytes(data[offsets[i]:offsets[i + 1]]) if non_null[i] else None for i in range(n)]
    if kind == ffi.COL_DECIMAL:
        return [_decimal_value(bytes(data[40 * i:40 * i + 40])) if non_null[i] else None for i in range(n)]
    a = np.frombuffer(data, dtype="<u8" if kind == ffi.COL_TIME else "<i8", count=n)
    return [int(a[i]) if non_null[i] else None for i in range(n)]


class BatchResult:
    """BatchExecuteResult with compacted, decoded columns (logical_rows is the identity)."""

    def __init__(self, columns, kinds, field_types, is_drained, error=None):
        self.columns, self.kinds, self.field_types, self.is_drained, self.error = columns, kinds, field_types, is_drained, error

    @property
    def n_rows(self):
        return len(self.columns[0]) if self.columns else 0

    def rows(self):
        return list(zip(*self.columns)) if self.columns else []


def _read_batch(b, location):
    assert location == ffi.LOC_HOST, "python helpers read host output only"
    cols, kinds, fts = [], [], []
    n = b.n_rows
    for i in range(b.n_columns):
        c = b.columns[i]
        kinds.append(c.kind)
        fts.append((c.field_tp, c.field_flag))
        if n == 0:
            cols.append([])
            continue
        words = (n + 63) // 64
        bm = np.ctypeslib.as_array(C.cast(c.null_bitmap, C.POINTER(C.c_uint64)), shape=(words,))
        nn = ((bm[np.arange(n) >> 6] >> (np.arange(n) & 63).astype(np.uint64)) & np.uint64(1)).astype(bool)
        if c.kind in (ffi.COL_BYTES, ffi.COL_JSON):
            offs = np.ctypeslib.as_array(C.cast(c.offsets, C.POINTER(C.c_int64)), shape=(n + 1,))
            heap = C.string_at(c.data, int(offs[n])) if offs[n] else b""
            vals = raw_cell_values(c.kind, heap, [int(x) for x in offs], list(nn))
        elif c.kind in (ffi.COL_TIME, ffi.COL_DURATION):
            vals = raw_cell_values(c.kind, C.string_at(c.data, 8 * n), None, list(nn))
        elif c.kind == ffi.COL_I64:
            a = np.ctypeslib.as_array(C.cast(c.data, C.POINTER(C.c_int64)), shape=(n,))
            vals = [int(a[j]) if nn[j] else None for j in range(n)]
        elif c.kind == ffi.COL_F64:
            a = np.ctypeslib.as_array(C.cast(c.data, C.POINTER(C.c_double)), shape=(n,))
            vals = [float(a[j]) if nn[j] else None for j in range(n)]
        else:
            raw = np.ctypeslib.as_array(C.cast(c.data, C.POINTER(C.c_uint8)), shape=(n * 40,)).tobytes()
            vals = [_decimal_value(raw[40 * j:40 * j + 40]) if nn[j] else None for j in range(n)]
        cols.append(vals)
    return cols, kinds, fts


class BatchExecutor:
    def __init__(self, plan, ranges, region, output=ffi.LOC_HOST, stream=0, jit=ffi.JIT_AUTO, deadline_ns=0):
        self._L = ffi.lib()
        self._plan, self._region = plan, region  # keep ctypes memory alive
        self._kr, self._keep = key_ranges(ranges)
        cfg = ffi.ExecConfig()
        cfg.output_location, cfg.cuda_stream, cfg.jit, cfg.deadline_ns = output, stream, jit, deadline_ns
        self._out_loc = output
        self._h = C.c_void_p()
        rc = self._L.b2_exec_open(C.byref(plan.c), self._kr, len(ranges), C.byref(region.c), C.byref(cfg), C.byref(self._h))
        if rc != ffi.B2_OK:
            raise B2Error(rc, self._L.b2_last_error_message().decode())

    def schema(self):
        n = C.c_uint32(64)
        tps, flags = (C.c_int32 * 64)(), (C.c_uint32 * 64)()
        self._L.b2_exec_schema(self._h, tps, flags, C.byref(n))
        return [(tps[i], flags[i]) for i in range(n.value)]

    def next_batch_raw(self, scan_rows):
        b = ffi.Batch()
        rc = self._L.b2_exec_next_batch(self._h, scan_rows, C.byref(b))
        return rc, b

    def next_batch(self, scan_rows):
        rc, b = self.next_batch_raw(scan_rows)
        cols, kinds, fts = _read_batch(b, self._out_loc)
        err = None
        if rc != ffi.B2_OK:
            e = self.last_error()
            err = B2Error(e.status, e.message.decode(), e.mysql_code, e.entry_index)
        return BatchResult(cols, kinds, fts, b.is_drained != ffi.DRAIN_REMAIN, err)

    def next_batch_async(self, scan_rows):
        """Start a batch without blocking (interface.rs:53 `async fn next_batch`); poll() collects it."""
        rc = self._L.b2_exec_next_batch_async(self._h, scan_rows)
        if rc != ffi.B2_OK:
            raise B2Error(rc, self._L.b2_last_error_message().decode())

    def poll(self):
        """None while the batch is in flight, else the BatchResult b2_exec_next_batch would have returned."""
        b = ffi.Batch()
        rc = self._L.b2_exec_poll(self._h, C.byref(b))
        if rc == ffi.B2_PENDING:
            return None
        cols, kinds, fts = _read_batch(b, self._out_loc)
        err = None
        if rc != ffi.B2_OK:
            e = self.last_error()
            err = B2Error(e.status, e.message.decode(), e.mysql_code, e.entry_index)
        r = BatchResult(cols, kinds, fts, b.is_drained != ffi.DRAIN_REMAIN, err)
        r.n_warnings = b.n_warnings
        return r

    def warnings(self):
        """(warning_cnt, [(mysql_code, message)]) of the request so far (EvalWarnings, expr/ctx.rs:180-215)."""
        out = (ffi.Warning * 64)()
        n = C.c_uint64()
        self._L.b2_exec_warnings(self._h, out, 64, C.byref(n))
        return n.value, [(out[i].mysql_code, out[i].message.decode()) for i in range(min(n.value, 64))]

    def take_scanned_range(self):
        """(lower_inclusive, upper_exclusive) raw keys covered since the previous call (scanner.rs:204-229)."""
        lo, hi, ln, hn = C.c_void_p(), C.c_void_p(), C.c_uint32(), C.c_uint32()
        rc = self._L.b2_exec_take_scanned_range(self._h, C.byref(lo), C.byref(ln), C.byref(hi), C.byref(hn))
        if rc != ffi.B2_OK:
            raise B2Error(rc, self._L.b2_last_error_message().decode())
        return C.string_at(lo, ln.value) if ln.value else b"", C.string_at(hi, hn.value) if hn.value else b""

    def collect_scanned_rows_per_range(self):
        n = C.c_uint32(4096)
        rows = (C.c_uint64 * 4096)()
        self._L.b2_exec_collect_scanned_rows_per_range(self._h, rows, C.byref(n))
        return [rows[i] for i in range(n.value)]

    def encode_batch(self, encode_type):
        """Chunk.rows_data of the batch just returned (runner.rs:1051-1088), encoded on the device, as bytes."""
        out = ffi.EncodedChunk()
        rc = self._L.b2_exec_encode_batch(self._h, encode_type, ffi.LOC_HOST, C.byref(out))
        if rc != ffi.B2_OK:
            raise B2Error(rc, self._L.b2_last_error_message().decode())
        return C.string_at(out.rows_data, out.len) if out.len else b""

    def last_error(self):
        e = ffi.ErrorInfo()
        self._L.b2_exec_last_error(self._h, C.byref(e))
        return e

    def collect_exec_stats(self):
        s = ffi.ExecStats()
        self._L.b2_exec_collect_stats(self._h, C.byref(s))
        return s

    def can_be_cached(self):
        return bool(self._L.b2_exec_can_be_cached(self._h))

    def close(self):
        if self._h:
            self._L.b2_exec_close(self._h)
            self._h = C.c_void_p()

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()


class DagResult:
    def __init__(self, status, message, mysql_code, columns, kinds, stats, can_be_cached):
        self.status, self.message, self.mysql_code = status, message, mysql_code
        self.columns, self.kinds, self.stats, self.can_be_cached = columns, kinds, stats, can_be_cached

    @property
    def n_rows(self):
        return len(self.columns[0]) if self.columns else 0

    def rows(self):
        return list(zip(*self.columns)) if self.columns else []


class DagHandler:
    """RequestHandler for a DAG request: handle_request() runs the executors to drain."""

    def __init__(self, plan, ranges, region, batch_rows=1 << 22, jit=None):
        self.plan, self.ranges, self.region, self.batch_rows, self.jit = plan, ranges, region, batch_rows, jit

    def handle_request(self):
        try:
            ex = BatchExecutor(self.plan, self.ranges, self.region) if self.jit is None else BatchExecutor(self.plan, self.ranges, self.region, jit=self.jit)
        except B2Error as e:
            return DagResult(e.status, e.message, 0, [], [], None, False)
        with ex:
            cols, kinds = None, []
            status, message, mysql = ffi.B2_OK, "", 0
            while True:
                r = ex.next_batch(self.batch_rows)
                if cols is None:
                    cols, kinds = [list(c) for c in r.columns], r.kinds
                else:
                    for a, c in zip(cols, r.columns):
                        a.extend(c)
                if r.error is not None:
                    status, message, mysql = r.error.status, r.error.message, r.error.mysql_code
                    break
                if r.is_drained:
                    break
            st = ex.collect_exec_stats()
            return DagResult(status, message, mysql, cols or [], kinds, st, ex.can_be_cached())


def checksum(ranges, region, old_prefix=b"", new_prefix=b"", stream=0, want_stats=False):
    """ChecksumContext::handle_request -> (status, (checksum, total_kvs, total_bytes[, exec stats]), message)."""
    L = ffi.lib()
    kr, keep = key_ranges(ranges)
    out, st = ffi.ChecksumResponse(), ffi.ExecStats()
    cfg = ffi.ExecConfig()
    cfg.cuda_stream = stream
    rc = L.b2_checksum_handle(kr, len(ranges), old_prefix, len(old_prefix), new_prefix, len(new_prefix), C.byref(region.c), C.byref(cfg) if stream else None,
                              C.byref(out), C.byref(st))
    msg = L.b2_last_error_message().decode() if rc else ""
    res = (out.checksum, out.total_kvs, out.total_bytes) + ((st,) if want_stats else ())
    return rc, res, msg


class DeviceRegion:
    """A region source whose CF_WRITE / CF_DEFAULT blocks live in HBM (torch tensors own the memory)."""

    def __init__(self, host_region, device=0):
        import torch
        self._t = []
        dev = torch.device("cuda", device)

        def up(arr):
            t = torch.from_numpy(np.ascontiguousarray(arr)).to(dev)
            self._t.append(t)
            return t.data_ptr()

        def blocks(hbs):
            arr = (ffi.CfBlock * len(hbs))()
            for i, hb in enumerate(hbs):
                arr[i].keys, arr[i].key_offs = up(hb.keys), up(hb.key_offs)
                arr[i].vals, arr[i].val_offs = up(hb.vals), up(hb.val_offs)
                arr[i].n = hb.n
            return arr

        self._host = host_region
        src = host_region.c
        s = ffi.RegionSource()
        C.memmove(C.byref(s), C.byref(src), C.sizeof(s))
        s.location, s.device = ffi.LOC_DEVICE, device
        self._w = blocks(host_region.wblocks)
        s.write, s.n_write = self._w, len(host_region.wblocks)
        if host_region.dblock is not None:
            self._d = blocks([host_region.dblock])
            s.dflt, s.n_dflt = self._d, 1
        torch.cuda.synchronize(dev)
        self.c = s


class SstDecoder:
    """b2_sst_decode: a run of RocksDB data blocks (prefix-compressed keys; stored plain, LZ4 / LZ4HC- or ZSTD-compressed, the
    type in each block's trailer) -> a device-resident flat CF block owned by this object.  `data` is a host buffer
    (bytes / numpy uint8 / address) or a device address."""

    def __init__(self, device=0):
        self.device, self.h = device, C.c_void_p()
        self._keep = None

    @staticmethod
    def _blocks(data, block_offs, trailer_len, key_prefix_len, key_suffix_len, d):
        """fills the b2_sst_blocks `d`; returns what must stay alive while it is used"""
        offs = np.ascontiguousarray(np.asarray(block_offs, dtype=np.uint64))
        if isinstance(data, (bytes, bytearray)):
            data = np.frombuffer(bytes(data), dtype=np.uint8)
        ptr = data.ctypes.data if isinstance(data, np.ndarray) else int(data)
        d.data, d.block_offs, d.n_blocks = ptr, offs.ctypes.data, len(offs) - 1
        d.trailer_len, d.key_prefix_len, d.key_suffix_len = trailer_len, key_prefix_len, key_suffix_len
        return data, offs

    def decode(self, data, block_offs, trailer_len=5, key_prefix_len=1, key_suffix_len=8, location=ffi.LOC_HOST):
        L = ffi.lib()
        d = ffi.SstBlocks()
        self._keep = self._blocks(data, block_offs, trailer_len, key_prefix_len, key_suffix_len, d)
        blk, st = ffi.CfBlock(), ffi.SstStats()
        rc = L.b2_sst_decode(self.device, location, C.byref(d), C.byref(self.h), C.byref(blk), C.byref(st))
        if rc != 0:
            raise B2Error(rc, L.b2_last_error_message().decode())
        return blk, st

    def merge(self, runs, snapshot_seq, global_seqs=None, location=ffi.LOC_HOST):
        """b2_sst_merge: the sorted runs of one LSM snapshot, newest first, each (data, block_offs) or a dict of decode()'s
        arguments (data, block_offs, trailer_len, key_prefix_len) -> the flat block a reader at `snapshot_seq` sees."""
        L = ffi.lib()
        arr = (ffi.SstBlocks * max(len(runs), 1))()
        keep = []
        for i, r in enumerate(runs):
            a = dict(r) if isinstance(r, dict) else dict(data=r[0], block_offs=r[1])
            keep.append(self._blocks(a["data"], a["block_offs"], a.get("trailer_len", 5), a.get("key_prefix_len", 1), 8, arr[i]))
        gs = None if global_seqs is None else (C.c_uint64 * max(len(runs), 1))(*global_seqs)
        self._keep = (keep, arr, gs)
        blk, st = ffi.CfBlock(), ffi.SstMergeStats()
        rc = L.b2_sst_merge(self.device, location, arr, len(runs), gs, snapshot_seq, C.byref(self.h), C.byref(blk), C.byref(st))
        if rc != 0:
            raise B2Error(rc, L.b2_last_error_message().decode())
        return blk, st

    def close(self):
        if self.h:
            ffi.lib().b2_sst_free(self.h)
            self.h = C.c_void_p()

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()


class SstRegion:
    """A region source whose CF_WRITE blocks arrive as RocksDB data blocks: each (data, block_offs) run, plain, LZ4 or ZSTD
    blocks as stored, is inflated and expanded on the device (b2_sst_decode) and the request reads the decoded blocks
    from HBM.  With `snapshot_seq`, `runs` are the sorted runs of one CF_WRITE LSM, newest first, each (data, offs) or
    (data, offs, global_seq), merged into one write block as a reader at that sequence number sees it (b2_sst_merge).
    The other fields follow `like`."""

    def __init__(self, like, runs, device=0, snapshot_seq=None, **fmt):
        if snapshot_seq is None:
            self._dec = [SstDecoder(device) for _ in runs]
            self.stats = []
            arr = (ffi.CfBlock * len(runs))()
            for i, (data, offs) in enumerate(runs):
                arr[i], st = self._dec[i].decode(data, offs, **fmt)
                self.stats.append(st)
        else:
            loc = fmt.pop("location", ffi.LOC_HOST)
            self._dec = [SstDecoder(device)]
            arr = (ffi.CfBlock * 1)()
            arr[0], st = self._dec[0].merge([dict(fmt, data=r[0], block_offs=r[1]) for r in runs], snapshot_seq,
                                            global_seqs=[r[2] if len(r) > 2 else 0 for r in runs], location=loc)
            self.stats = [st]
        s = ffi.RegionSource()
        C.memmove(C.byref(s), C.byref(like.c), C.sizeof(s))
        s.location, s.device = ffi.LOC_DEVICE, device
        s.write, s.n_write = arr, len(arr)
        self._w, self._like = arr, like
        if like.c.n_dflt:  # CF_DEFAULT of the model region must live where `location` says
            self._dflt = DeviceRegion(like, device)
            s.dflt, s.n_dflt = self._dflt.c.dflt, self._dflt.c.n_dflt
        self.c = s

    def close(self):
        for d in self._dec:
            d.close()
