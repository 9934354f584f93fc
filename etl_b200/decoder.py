"""Host-side mirror of the reference interface for the streaming decode path.

Reference shape (crates/etl/src/replication/apply.rs): the apply loop pulls one replication message
at a time (`events_stream.next()`, :940), converts it (`handle_replication_message`, :1687) and
appends the `Event` to a batch that is flushed to `Destination::write_events` (:1672).  Here the
same three roles are batch-shaped:

  Stager            ← EventsStream::poll_next: CopyData bodies are appended, not parsed
  Decoder.decode    ← handle_replication_message for the whole staged batch, on the GPU
  DecodedBatch      ← the Vec<Event> handed to add_event_to_batch, as columnar planes

Everything below the C ABI (include/etl_decode.h) is CUDA; this module only marshals arguments.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from . import abi


class DecodeError(RuntimeError):
    pass


@dataclass
class SchemaInfo:
    table_id: int
    n_cols: int
    n_identity: int
    snapshot_id: int
    effective_off: int
    col_kind: np.ndarray
    col_flags: np.ndarray
    col_index: np.ndarray


@dataclass
class DecodedBatch:
    """Columnar planes of one decoded batch (host copies). Field names = etl_dec_planes."""
    n_records: int
    n_cells: int
    rec_off: np.ndarray
    rec_kind: np.ndarray
    rec_flags: np.ndarray
    rec_rel: np.ndarray
    rec_schema: np.ndarray
    rec_start_lsn: np.ndarray
    rec_commit_lsn: np.ndarray
    rec_tx_ordinal: np.ndarray
    rec_cell_base: np.ndarray
    rec_tuple_bytes: np.ndarray
    rec_heap_hint: np.ndarray
    cell_tag: np.ndarray
    cell_val: np.ndarray
    cell_aux: np.ndarray
    heap: np.ndarray
    first_error: tuple   # (record_index | None, seq, code, kind)
    carry_out: tuple     # (in_tx, final_lsn, next_tx_ordinal)
    insert_bytes: int
    update_bytes: int
    delete_bytes: int
    n_events: int
    schemas: List[SchemaInfo]
    kernel_ms: float = 0.0
    h2d_ms: float = 0.0
    d2h_ms: float = 0.0
    gpu_launches: int = 0
    result_bytes: int = 0
    index_ms: float = 0.0
    emit_ms: float = 0.0
    h2d_bytes: int = 0
    d2h_bytes: int = 0
    record_index_base: int = 0
    sizing: int = 0      # abi.SIZING_* bits: how the planes were sized (diagnostic)


@dataclass
class CopyBatch:
    """Decoded COPY rows: row-major cells (cell r * n_cols + c).  A string / json cell is a span of `stream`
    (val = offset) unless bit 63 of val is set: then the low bits are an offset into `heap` (the field was unescaped)."""
    n_rows: int
    n_cols: int
    stream: np.ndarray
    cell_tag: np.ndarray
    cell_val: np.ndarray
    cell_aux: np.ndarray
    heap: np.ndarray
    first_error: tuple   # (row | None, step (0 = the row's UTF-8 check, 1 + column otherwise), code, kind)
    kernel_ms: float = 0.0
    gpu_launches: int = 0


def _make_columns(cols: Sequence[dict]):
    arr = (abi.ColumnSchema * max(1, len(cols)))()
    keep = []
    for i, c in enumerate(cols):
        nm = c["name"].encode()
        keep.append(nm)
        arr[i].name = nm
        arr[i].type_oid = c["type_oid"]
        arr[i].modifier = c.get("modifier", -1)
        arr[i].ordinal_position = c.get("ordinal_position", i + 1)
        pk = c.get("pk")
        arr[i].primary_key_ordinal_position = -1 if pk is None else pk
        arr[i].nullable = 1 if c.get("nullable", True) else 0
    return arr, keep


class Stager:
    """Pinned staging buffer + sparse anchor index + Relation-frame offsets (etl_stage_*)."""

    def __init__(self, capacity_bytes: int, anchor_stride: int = 2048):
        self._l = abi.load()
        self._h = C.c_void_p()
        rc = self._l.etl_stage_create(capacity_bytes, anchor_stride, C.byref(self._h))
        if rc:
            raise DecodeError(f"etl_stage_create failed: {rc}")

    def append(self, copydata_body: bytes):
        rc = self._l.etl_stage_append(self._h, C.cast(C.c_char_p(copydata_body), C.c_void_p), len(copydata_body))
        if rc:
            raise DecodeError(f"etl_stage_append failed: {rc}")

    def append_framed(self, framed) -> None:
        if isinstance(framed, np.ndarray):
            ptr, n = framed.ctypes.data, framed.nbytes
        else:
            self._keep = bytes(framed)
            ptr, n = C.cast(C.c_char_p(self._keep), C.c_void_p).value, len(self._keep)
        rc = self._l.etl_stage_append_framed(self._h, ptr, n)
        if rc:
            raise DecodeError(f"etl_stage_append_framed failed: {rc} (stream is not a chain of CopyData frames?)")

    def reset(self):
        self._l.etl_stage_reset(self._h)

    def view(self) -> abi.DecInput:
        inp = abi.DecInput()
        self._l.etl_stage_view(self._h, C.byref(inp))
        return inp

    def host_array(self) -> np.ndarray:
        v = self.view()
        if v.len == 0:
            return np.zeros(0, dtype=np.uint8)
        return np.ctypeslib.as_array(C.cast(v.host_buf, abi.u8p), shape=(int(v.len),))

    def close(self):
        if self._h:
            self._l.etl_stage_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def _np_from(ptr, n, dtype):
    n = int(n)
    if n == 0 or not ptr:
        return np.zeros(0, dtype=dtype)
    nbytes = n * np.dtype(dtype).itemsize
    buf = (C.c_uint8 * nbytes).from_address(ptr)
    return np.frombuffer(buf, dtype=dtype, count=n).copy()


class Decoder:
    """One decode context = one apply loop on one GPU (etl_dec_ctx)."""

    def __init__(self, device: int = 0, stream: Optional[int] = None):
        self._l = abi.load()
        self._ctx = C.c_void_p()
        rc = self._l.etl_dec_create(device, C.byref(self._ctx))
        if rc:
            raise DecodeError(f"etl_dec_create(device={device}) failed with status {rc} "
                              "(4 = no CUDA device: the decode path has no CPU fallback)")
        if stream is not None:
            self._l.etl_dec_set_stream(self._ctx, C.c_void_p(stream))

    # -- schema catalogue (what SchemaStore::get_table_schema returns) --------------------------------
    def put_table_schema(self, table_id: int, cols: Sequence[dict], snapshot_id: int = 0):
        arr, _keep = _make_columns(cols)
        rc = self._l.etl_dec_put_table_schema(self._ctx, table_id, snapshot_id, arr, len(cols))
        self._check(rc)

    def reset_relations(self):
        self._check(self._l.etl_dec_reset_relations(self._ctx))

    def _check(self, rc):
        if rc:
            raise DecodeError(f"status {rc}: {self._l.etl_dec_last_error(self._ctx).decode()}")

    # -- decode ---------------------------------------------------------------------------------------
    @staticmethod
    def _carry(inp: abi.DecInput, carry_in):
        if carry_in:
            inp.carry_in.in_tx, inp.carry_in.final_lsn, inp.carry_in.next_tx_ordinal = int(carry_in[0]), carry_in[1], carry_in[2]

    def decode_input(self, inp: abi.DecInput, to_host: bool = True, timing: bool = True) -> "BatchHandle":
        h = C.c_void_p()
        flags = (abi.RESULTS_TO_HOST if to_host else 0) | (0 if timing else abi.NO_TIMING)
        rc = self._l.etl_dec_decode(self._ctx, C.byref(inp), flags, C.byref(h))
        self._check(rc)
        return BatchHandle(self, h)

    # -- multi-GPU: the library owns the NCCL communicator and the seam / relation-update exchange ------------
    def comm_unique_id(self) -> bytes:
        buf = (C.c_uint8 * 128)()
        self._check(self._l.etl_dec_comm_unique_id(C.cast(buf, C.c_void_p), 128))
        return bytes(buf)

    def comm_init(self, unique_id: bytes, rank: int, n_ranks: int):
        buf = (C.c_uint8 * 128).from_buffer_copy(unique_id)
        self._check(self._l.etl_dec_comm_init(self._ctx, C.cast(buf, C.c_void_p), 128, rank, n_ranks))

    def comm_init_host(self, rank: int, n_ranks: int, allgather):
        """Exchange through the host: `allgather(send: bytes) -> bytes` returns the n_ranks blocks in rank order
        (e.g. torch.distributed with the gloo backend).  Same decode_sharded afterwards."""
        def _cb(_user, send, recv, nbytes):
            try:
                out = allgather(C.string_at(send, nbytes))
                if len(out) != nbytes * n_ranks:
                    return 1
                C.memmove(recv, out, len(out))
                return 0
            except Exception:  # noqa: BLE001 — reported through the status code
                return 1
        self._host_cb = abi.HOST_ALLGATHER_FN(_cb)      # keep the trampoline alive
        self._check(self._l.etl_dec_comm_init_host(self._ctx, rank, n_ranks, self._host_cb, None))

    def decode_sharded(self, inp: abi.DecInput, to_host: bool = True, timing: bool = True) -> "BatchHandle":
        """This rank's byte range of one stream: relation-update exchange, index pass, seam all-gather and fold on
        the device, record + tuple passes (etl_dec_decode_sharded)."""
        h = C.c_void_p()
        flags = (abi.RESULTS_TO_HOST if to_host else 0) | (0 if timing else abi.NO_TIMING)
        self._check(self._l.etl_dec_decode_sharded(self._ctx, C.byref(inp), flags, C.byref(h)))
        return BatchHandle(self, h)

    # -- initial-sync COPY rows (etl_dec_copy_decode; table_row.rs:25-165 for a whole buffer of rows) --------------
    def copy_decode(self, table_id: int, rows, row_offsets=None) -> "CopyBatch":
        """`rows`: bytes / uint8 array of COPY-text rows back to back (each with its LF), or a list of row chunks.
        Returns the decoded cells (host copies)."""
        if isinstance(rows, (list, tuple)):
            offs = np.zeros(len(rows) + 1, dtype=np.uint64)
            offs[1:] = np.cumsum([len(r) for r in rows])
            buf = np.frombuffer(b"".join(bytes(r) for r in rows), dtype=np.uint8)
        else:
            buf = rows if isinstance(rows, np.ndarray) else np.frombuffer(bytes(rows), dtype=np.uint8)
            offs = np.asarray(row_offsets, dtype=np.uint64)
        padded = np.zeros(buf.nbytes + 64, dtype=np.uint8)            # the kernels read whole aligned words around a value
        padded[:buf.nbytes] = buf
        inp = abi.CopyInput()
        inp.host_buf = padded.ctypes.data
        inp.len = buf.nbytes
        inp.row_offsets = offs.ctypes.data
        inp.n_rows = len(offs) - 1
        h = C.c_void_p()
        self._check(self._l.etl_dec_copy_decode(self._ctx, table_id, C.byref(inp), abi.RESULTS_TO_HOST, C.byref(h)))
        bh = BatchHandle(self, h)
        try:
            p, s = bh.planes(True), bh.summary()
            m = int(p.n_cells)
            fe = s.first_error
            return CopyBatch(n_rows=int(p.n_records), n_cols=(m // int(p.n_records)) if p.n_records else 0, stream=buf,
                             cell_tag=_np_from(p.cell_tag, m, np.uint8), cell_val=_np_from(p.cell_val, m, np.uint64),
                             cell_aux=_np_from(p.cell_aux, m, np.uint32), heap=_np_from(p.heap, p.heap_bytes, np.uint8),
                             first_error=(None if fe.record_index == 2**64 - 1 else int(fe.record_index), int(fe.seq), int(fe.code), int(fe.kind)),
                             kernel_ms=float(s.kernel_ms), gpu_launches=int(s.gpu_launches))
        finally:
            bh.free()

    def mem_info(self):
        f, t = C.c_uint64(), C.c_uint64()
        self._check(self._l.etl_dec_mem_info(self._ctx, C.byref(f), C.byref(t)))
        return int(f.value), int(t.value)

    def decode_begin(self, inp: abi.DecInput, to_host: bool = True) -> abi.Seam:
        seam = abi.Seam()
        self._check(self._l.etl_dec_decode_begin(self._ctx, C.byref(inp), abi.RESULTS_TO_HOST if to_host else 0, C.byref(seam)))
        return seam

    def decode_finish(self, carry_in: Tuple[int, int, int], record_index_base: int = 0) -> "BatchHandle":
        st = abi.StreamState()
        st.in_tx, st.final_lsn, st.next_tx_ordinal = int(carry_in[0]), carry_in[1], carry_in[2]
        h = C.c_void_p()
        self._check(self._l.etl_dec_decode_finish(self._ctx, C.byref(st), record_index_base, C.byref(h)))
        return BatchHandle(self, h)

    def decode(self, stream, carry_in=None, anchor_stride: int = 2048, max_frame_len=None) -> DecodedBatch:
        """Stage `stream` (bytes / uint8 array of CopyData-framed messages) and decode it.  `max_frame_len` overrides the
        stager's frame-length hint (tests: 0 = unknown, or a deliberately wrong bound)."""
        n = stream.nbytes if isinstance(stream, np.ndarray) else len(stream)
        st = Stager(max(n, 1), anchor_stride)
        try:
            st.append_framed(stream)
            inp = st.view()
            if max_frame_len is not None:
                inp.max_frame_len = int(max_frame_len)
            self._carry(inp, carry_in)
            with self.decode_input(inp, to_host=True) as bh:
                return bh.to_host()
        finally:
            st.close()

    def close(self):
        if self._ctx:
            self._l.etl_dec_destroy(self._ctx)
            self._ctx = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class BatchHandle:
    """Owns an etl_dec_batch (device planes + optional pinned host copy)."""

    def __init__(self, dec: Decoder, h):
        self._dec, self._l, self._h = dec, dec._l, h

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.free()

    def free(self):
        if self._h:
            self._l.etl_dec_batch_free(self._h)
            self._h = C.c_void_p()

    def summary(self) -> abi.Summary:
        s = abi.Summary()
        self._l.etl_dec_batch_summary(self._h, C.byref(s))
        return s

    def planes(self, host: bool) -> abi.Planes:
        p = abi.Planes()
        rc = self._l.etl_dec_batch_planes(self._h, 1 if host else 0, C.byref(p))
        if rc:
            raise DecodeError("planes not available (decode without RESULTS_TO_HOST?)")
        return p

    def schemas(self) -> List[SchemaInfo]:
        out = []
        for i in range(self.summary().n_schemas):
            si = abi.SchemaInfo()
            self._l.etl_dec_batch_schema(self._h, i, C.byref(si))
            n = si.n_cols
            out.append(SchemaInfo(si.table_id, n, si.n_identity, si.snapshot_id, si.effective_off,
                                  np.array([si.col_kind[k] for k in range(n)], dtype=np.uint8),
                                  np.array([si.col_flags[k] for k in range(n)], dtype=np.uint8),
                                  np.array([si.col_index[k] for k in range(n)], dtype=np.int32)))
        return out

    def to_host(self) -> DecodedBatch:
        p, s = self.planes(True), self.summary()
        n, m = p.n_records, p.n_cells
        fe = s.first_error
        nbytes = n * (8 + 1 + 1 + 4 + 4 + 8 + 8 + 8 + 8 + 4 + 4) + 8 + m * 13 + p.heap_bytes
        return DecodedBatch(
            n_records=int(n), n_cells=int(m),
            rec_off=_np_from(p.rec_off, n, np.uint64), rec_kind=_np_from(p.rec_kind, n, np.uint8),
            rec_flags=_np_from(p.rec_flags, n, np.uint8), rec_rel=_np_from(p.rec_rel, n, np.uint32),
            rec_schema=_np_from(p.rec_schema, n, np.int32), rec_start_lsn=_np_from(p.rec_start_lsn, n, np.uint64),
            rec_commit_lsn=_np_from(p.rec_commit_lsn, n, np.uint64), rec_tx_ordinal=_np_from(p.rec_tx_ordinal, n, np.uint64),
            rec_cell_base=_np_from(p.rec_cell_base, n + 1, np.uint64), rec_tuple_bytes=_np_from(p.rec_tuple_bytes, n, np.uint32),
            rec_heap_hint=_np_from(p.rec_heap_hint, n, np.uint32), cell_tag=_np_from(p.cell_tag, m, np.uint8),
            cell_val=_np_from(p.cell_val, m, np.uint64), cell_aux=_np_from(p.cell_aux, m, np.uint32),
            heap=_np_from(p.heap, p.heap_bytes, np.uint8),
            first_error=(None if fe.record_index == 2**64 - 1 else int(fe.record_index), int(fe.seq), int(fe.code), int(fe.kind)),
            carry_out=(int(s.carry_out.in_tx), int(s.carry_out.final_lsn), int(s.carry_out.next_tx_ordinal)),
            insert_bytes=int(s.insert_bytes), update_bytes=int(s.update_bytes), delete_bytes=int(s.delete_bytes),
            n_events=int(s.n_events), schemas=self.schemas(), kernel_ms=float(s.kernel_ms), h2d_ms=float(s.h2d_ms),
            d2h_ms=float(s.d2h_ms), gpu_launches=int(s.gpu_launches), result_bytes=int(nbytes),
            index_ms=float(s.index_ms), emit_ms=float(s.emit_ms), h2d_bytes=int(s.h2d_bytes), d2h_bytes=int(s.d2h_bytes),
            record_index_base=int(s.record_index_base), sizing=int(s.sizing))
