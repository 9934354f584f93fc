"""ctypes binding of include/etl_decode.h (libetl_decode.so).

This is the same binding a Rust / cgo / JNI shim would write (see INTEGRATION.md): plain pointers
and sizes, no torch types.  The library is built in-tree by etl_b200.build (nvcc, sm_90a) and the
import fails loudly if it is missing — there is no CPU fallback for the decode path.
"""
from __future__ import annotations

import ctypes as C
import os

from . import build as _build

u8p, u32p, u64p, i32p = C.POINTER(C.c_uint8), C.POINTER(C.c_uint32), C.POINTER(C.c_uint64), C.POINTER(C.c_int32)


class ColumnSchema(C.Structure):
    _fields_ = [("name", C.c_char_p), ("type_oid", C.c_uint32), ("modifier", C.c_int32),
                ("ordinal_position", C.c_int32), ("primary_key_ordinal_position", C.c_int32),
                ("nullable", C.c_uint8), ("_pad", C.c_uint8 * 7)]


class StreamState(C.Structure):
    _fields_ = [("final_lsn", C.c_uint64), ("next_tx_ordinal", C.c_uint64), ("in_tx", C.c_uint8), ("_pad", C.c_uint8 * 7)]


class FirstError(C.Structure):
    _fields_ = [("record_index", C.c_uint64), ("seq", C.c_uint32), ("code", C.c_uint32), ("kind", C.c_uint32), ("_pad", C.c_uint32)]


class DecInput(C.Structure):
    _fields_ = [("host_buf", C.c_void_p), ("dev_buf", C.c_void_p), ("len", C.c_uint64), ("anchors", C.c_void_p),
                ("dev_anchors", C.c_void_p), ("n_anchors", C.c_uint64), ("anchor_stride", C.c_uint32), ("max_frame_len", C.c_uint32),
                ("relation_offsets", C.c_void_p), ("n_relations", C.c_uint64), ("carry_in", StreamState)]


class Seam(C.Structure):
    _fields_ = [("n_records", C.c_uint64), ("n_cells", C.c_uint64), ("heap_bytes", C.c_uint64), ("lsn", C.c_uint64),
                ("ord", C.c_uint64), ("has_begin", C.c_uint8), ("closed", C.c_uint8), ("_pad", C.c_uint8 * 6)]


class CopyInput(C.Structure):
    _fields_ = [("host_buf", C.c_void_p), ("dev_buf", C.c_void_p), ("len", C.c_uint64), ("row_offsets", C.c_void_p),
                ("dev_row_offsets", C.c_void_p), ("n_rows", C.c_uint64)]


HOST_ALLGATHER_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64)


class ArrowColumn(C.Structure):
    _fields_ = [("arrow_type", C.c_uint32), ("_pad", C.c_uint32), ("validity", C.c_void_p), ("values", C.c_void_p),
                ("offsets", C.c_void_p), ("data", C.c_void_p), ("data_bytes", C.c_uint64)]


class RbIssue(C.Structure):
    _fields_ = [("row", C.c_uint64), ("column", C.c_uint32), ("element", C.c_uint32)]


class RowBinaryIssues(C.Structure):
    _fields_ = [("date_range", RbIssue), ("null_value", RbIssue), ("first_partial_update", C.c_uint64)]


class BqIssue(C.Structure):
    _fields_ = [("row", C.c_uint64), ("column", C.c_uint32), ("element", C.c_uint32), ("kind", C.c_uint32), ("_pad", C.c_uint32)]


class BigQueryIssues(C.Structure):
    _fields_ = [("value", BqIssue), ("first_invalid_record", C.c_uint64)]


class DuckLakeIssues(C.Structure):
    _fields_ = [("first_rejected_record", C.c_uint64), ("rejected_reason", C.c_uint32), ("mixed_versions", C.c_uint32),
                ("first_empty_partial_record", C.c_uint64)]


class DlSubBatch(C.Structure):
    _fields_ = [("first_mutation", C.c_uint64), ("n_mutations", C.c_uint32), ("_pad", C.c_uint32), ("fingerprint", C.c_uint64)]


class ParquetField(C.Structure):
    _fields_ = [("name", C.c_char_p), ("field_id", C.c_int32), ("element_field_id", C.c_int32), ("required", C.c_uint32),
                ("_pad", C.c_uint32)]


class ParquetMetrics(C.Structure):
    _fields_ = [("field_id", C.c_int32), ("flags", C.c_uint32), ("num_values", C.c_uint64), ("null_count", C.c_uint64),
                ("nan_count", C.c_uint64), ("compressed_bytes", C.c_uint64), ("uncompressed_bytes", C.c_uint64),
                ("min", C.c_void_p), ("min_len", C.c_uint32), ("max", C.c_void_p), ("max_len", C.c_uint32)]


class ParquetBloom(C.Structure):
    _fields_ = [("fpp", C.c_double), ("ndv", C.c_uint64), ("max_bytes", C.c_uint32), ("_pad", C.c_uint32)]


class IcebergPartitionField(C.Structure):
    _fields_ = [("source_column", C.c_uint32), ("transform", C.c_uint32), ("param", C.c_uint32), ("_pad", C.c_uint32)]


class IcebergPartitionValue(C.Structure):
    _fields_ = [("is_null", C.c_uint32), ("len", C.c_uint32), ("value", C.c_int64), ("data", C.c_void_p)]


class Planes(C.Structure):
    _fields_ = [("n_records", C.c_uint64), ("n_cells", C.c_uint64), ("heap_bytes", C.c_uint64),
                ("rec_off", C.c_void_p), ("rec_kind", C.c_void_p), ("rec_flags", C.c_void_p), ("rec_rel", C.c_void_p),
                ("rec_schema", C.c_void_p), ("rec_start_lsn", C.c_void_p), ("rec_commit_lsn", C.c_void_p),
                ("rec_tx_ordinal", C.c_void_p), ("rec_cell_base", C.c_void_p), ("rec_tuple_bytes", C.c_void_p),
                ("rec_heap_hint", C.c_void_p), ("cell_tag", C.c_void_p),
                ("cell_val", C.c_void_p), ("cell_aux", C.c_void_p), ("heap", C.c_void_p)]


class Summary(C.Structure):
    _fields_ = [("first_error", FirstError), ("carry_out", StreamState), ("insert_bytes", C.c_uint64),
                ("update_bytes", C.c_uint64), ("delete_bytes", C.c_uint64), ("n_events", C.c_uint64),
                ("n_schemas", C.c_uint32), ("gpu_launches", C.c_uint32), ("kernel_ms", C.c_float),
                ("h2d_ms", C.c_float), ("d2h_ms", C.c_float), ("index_ms", C.c_float),
                ("emit_ms", C.c_float), ("frames_ms", C.c_float), ("walk_ms", C.c_float), ("spans_ms", C.c_float), ("cells_ms", C.c_float), ("long_ms", C.c_float), ("h2d_bytes", C.c_uint64), ("d2h_bytes", C.c_uint64), ("span_bytes", C.c_uint64),
                ("record_index_base", C.c_uint64), ("abi_version", C.c_uint32), ("sizing", C.c_uint32)]


class SchemaInfo(C.Structure):
    _fields_ = [("table_id", C.c_uint32), ("n_cols", C.c_uint32), ("n_identity", C.c_uint32), ("_pad", C.c_uint32),
                ("snapshot_id", C.c_uint64), ("effective_off", C.c_uint64), ("col_kind", u8p), ("col_flags", u8p),
                ("col_index", i32p)]


# every symbol include/etl_decode.h declares (tests check the library exports all of them)
EXPORTS = [
    "etl_dec_abi_version", "etl_stage_create", "etl_stage_destroy", "etl_stage_reset", "etl_stage_append",
    "etl_stage_append_framed", "etl_stage_view", "etl_dec_create", "etl_dec_set_stream", "etl_dec_destroy",
    "etl_dec_last_error", "etl_dec_put_table_schema", "etl_dec_reset_relations", "etl_dec_decode",
    "etl_dec_decode_begin", "etl_dec_decode_finish", "etl_dec_batch_free", "etl_dec_batch_planes",
    "etl_dec_batch_summary", "etl_dec_batch_schema", "etl_dec_decode_sharded", "etl_dec_comm_unique_id", "etl_dec_comm_init", "etl_dec_comm_init_host",
    "etl_dec_kind_for_type_oid", "etl_dec_mem_info",
    "etl_dec_copy_decode", "etl_dec_arrow_emit", "etl_dec_arrow_rows", "etl_dec_arrow_cols", "etl_dec_arrow_row_records",
    "etl_dec_arrow_column", "etl_dec_arrow_list_child", "etl_dec_arrow_first_skipped", "etl_dec_arrow_free", "etl_dec_rowbinary_emit", "etl_dec_rowbinary_rows", "etl_dec_rowbinary_bytes",
    "etl_dec_rowbinary_data", "etl_dec_rowbinary_row_offsets", "etl_dec_rowbinary_row_records", "etl_dec_rowbinary_issues",
    "etl_dec_rowbinary_free", "etl_dec_rowbinary_lz4", "etl_dec_rowbinary_lz4_inserts", "etl_dec_rowbinary_lz4_insert_rows",
    "etl_dec_rowbinary_lz4_insert_offsets", "etl_dec_rowbinary_lz4_bytes", "etl_dec_rowbinary_lz4_data", "etl_dec_rowbinary_lz4_free",
    "etl_dec_bigquery_emit", "etl_dec_bigquery_rows", "etl_dec_bigquery_bytes", "etl_dec_bigquery_data",
    "etl_dec_bigquery_row_offsets", "etl_dec_bigquery_row_records", "etl_dec_bigquery_issues", "etl_dec_bigquery_free",
    "etl_dec_ducklake_emit", "etl_dec_ducklake_mutations", "etl_dec_ducklake_kinds", "etl_dec_ducklake_records",
    "etl_dec_ducklake_text", "etl_dec_ducklake_issues", "etl_dec_ducklake_sub_batches", "etl_dec_ducklake_copy_fingerprint",
    "etl_dec_ducklake_free", "etl_dec_parquet_write", "etl_dec_parquet_write_bloom", "etl_dec_parquet_size", "etl_dec_parquet_bytes", "etl_dec_parquet_metrics",
    "etl_dec_parquet_required_null", "etl_dec_parquet_free",
    "etl_dec_parquet_write_files", "etl_dec_parquet_files_count", "etl_dec_parquet_files_offsets", "etl_dec_parquet_files_bytes",
    "etl_dec_parquet_files_metrics", "etl_dec_parquet_files_required_null", "etl_dec_parquet_files_free",
    "etl_dec_iceberg_partition", "etl_dec_iceberg_partitions", "etl_dec_iceberg_partition_rows", "etl_dec_iceberg_partition_value",
    "etl_dec_iceberg_partitioned_arrow", "etl_dec_iceberg_partition_free",
    "etl_dec_batch_device_stream", "etl_shim_materialise", "etl_shim_event_count", "etl_shim_size_hint", "etl_shim_total_size_hint", "etl_shim_owned_bytes",
    "etl_shim_json_text", "etl_shim_event_list_free",
]

_lib = None


def lib_path() -> str:
    return _build.DECODE_LIB


def load(build: bool = True):
    """Load libetl_decode.so (building it first if the sources are newer). Raises if unavailable."""
    global _lib
    if _lib is not None:
        return _lib
    # an existing in-tree library is loaded as is (a copied tree need not preserve file times, so no staleness
    # check here — build() and `python -m etl_b200.build` rebuild when the sources are newer)
    path = _build.DECODE_LIB
    if build and not os.path.exists(path):
        path = _build.build_decode()
    if not os.path.exists(path):
        raise RuntimeError(f"{path} is missing: the CUDA decode library must be built (python -m etl_b200.build)")
    L = C.CDLL(path)
    vp = C.c_void_p
    L.etl_dec_abi_version.restype = C.c_uint32
    L.etl_stage_create.argtypes = [C.c_uint64, C.c_uint32, C.POINTER(vp)]
    L.etl_stage_destroy.argtypes = [vp]
    L.etl_stage_destroy.restype = None
    L.etl_stage_reset.argtypes = [vp]
    L.etl_stage_reset.restype = None
    L.etl_stage_append.argtypes = [vp, vp, C.c_uint32]
    L.etl_stage_append_framed.argtypes = [vp, vp, C.c_uint64]
    L.etl_stage_view.argtypes = [vp, C.POINTER(DecInput)]
    L.etl_dec_create.argtypes = [C.c_int, C.POINTER(vp)]
    L.etl_dec_set_stream.argtypes = [vp, vp]
    L.etl_dec_destroy.argtypes = [vp]
    L.etl_dec_destroy.restype = None
    L.etl_dec_last_error.argtypes = [vp]
    L.etl_dec_last_error.restype = C.c_char_p
    L.etl_dec_put_table_schema.argtypes = [vp, C.c_uint32, C.c_uint64, C.POINTER(ColumnSchema), C.c_uint32]
    L.etl_dec_reset_relations.argtypes = [vp]
    L.etl_dec_decode.argtypes = [vp, C.POINTER(DecInput), C.c_uint32, C.POINTER(vp)]
    L.etl_dec_decode_begin.argtypes = [vp, C.POINTER(DecInput), C.c_uint32, C.POINTER(Seam)]
    L.etl_dec_decode_finish.argtypes = [vp, C.POINTER(StreamState), C.c_uint64, C.POINTER(vp)]
    L.etl_dec_batch_free.argtypes = [vp]
    L.etl_dec_batch_free.restype = None
    L.etl_dec_batch_planes.argtypes = [vp, C.c_int, C.POINTER(Planes)]
    L.etl_dec_batch_summary.argtypes = [vp, C.POINTER(Summary)]
    L.etl_dec_batch_schema.argtypes = [vp, C.c_uint32, C.POINTER(SchemaInfo)]
    L.etl_dec_decode_sharded.argtypes = [vp, C.POINTER(DecInput), C.c_uint32, C.POINTER(vp)]
    L.etl_dec_comm_unique_id.argtypes = [vp, C.c_uint32]
    L.etl_dec_comm_init.argtypes = [vp, vp, C.c_uint32, C.c_int, C.c_int]
    L.etl_dec_comm_init_host.argtypes = [vp, C.c_int, C.c_int, HOST_ALLGATHER_FN, vp]
    L.etl_dec_kind_for_type_oid.argtypes = [C.c_uint32]
    L.etl_dec_kind_for_type_oid.restype = C.c_uint32
    L.etl_dec_mem_info.argtypes = [vp, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
    L.etl_dec_copy_decode.argtypes = [vp, C.c_uint32, C.POINTER(CopyInput), C.c_uint32, C.POINTER(vp)]
    L.etl_dec_arrow_emit.argtypes = [vp, C.c_uint32, C.c_uint32, C.c_int, C.POINTER(vp)]
    L.etl_dec_arrow_rows.argtypes = [vp]
    L.etl_dec_arrow_rows.restype = C.c_uint64
    L.etl_dec_arrow_cols.argtypes = [vp]
    L.etl_dec_arrow_cols.restype = C.c_uint32
    L.etl_dec_arrow_row_records.argtypes = [vp, C.c_int]
    L.etl_dec_arrow_row_records.restype = C.c_void_p
    L.etl_dec_arrow_column.argtypes = [vp, C.c_uint32, C.c_int, C.POINTER(ArrowColumn)]
    L.etl_dec_arrow_list_child.argtypes = [vp, C.c_uint32, C.c_int, C.POINTER(ArrowColumn), C.POINTER(C.c_uint64)]
    L.etl_dec_arrow_first_skipped.argtypes = [vp]
    L.etl_dec_arrow_first_skipped.restype = C.c_uint64
    L.etl_dec_arrow_free.argtypes = [vp]
    L.etl_dec_arrow_free.restype = None
    L.etl_dec_rowbinary_emit.argtypes = [vp, C.c_uint32, vp, C.c_uint32, C.c_int, C.POINTER(vp)]
    for f in ("etl_dec_rowbinary_rows", "etl_dec_rowbinary_bytes"):
        getattr(L, f).argtypes = [vp]
        getattr(L, f).restype = C.c_uint64
    for f in ("etl_dec_rowbinary_data", "etl_dec_rowbinary_row_offsets", "etl_dec_rowbinary_row_records"):
        getattr(L, f).argtypes = [vp, C.c_int]
        getattr(L, f).restype = C.c_void_p
    L.etl_dec_rowbinary_issues.argtypes = [vp, C.POINTER(RowBinaryIssues)]
    L.etl_dec_rowbinary_free.argtypes = [vp]
    L.etl_dec_rowbinary_free.restype = None
    L.etl_dec_rowbinary_lz4.argtypes = [vp, C.c_uint64, C.c_uint64, C.c_uint64, C.c_int, C.POINTER(vp)]
    for f in ("etl_dec_rowbinary_lz4_inserts", "etl_dec_rowbinary_lz4_bytes"):
        getattr(L, f).argtypes = [vp]
        getattr(L, f).restype = C.c_uint64
    for f in ("etl_dec_rowbinary_lz4_insert_rows", "etl_dec_rowbinary_lz4_insert_offsets", "etl_dec_rowbinary_lz4_data"):
        getattr(L, f).argtypes = [vp, C.c_int]
        getattr(L, f).restype = C.c_void_p
    L.etl_dec_rowbinary_lz4_free.argtypes = [vp]
    L.etl_dec_rowbinary_lz4_free.restype = None
    L.etl_dec_bigquery_emit.argtypes = [vp, C.c_uint32, C.c_int, C.POINTER(vp)]
    for f in ("etl_dec_bigquery_rows", "etl_dec_bigquery_bytes"):
        getattr(L, f).argtypes = [vp]
        getattr(L, f).restype = C.c_uint64
    for f in ("etl_dec_bigquery_data", "etl_dec_bigquery_row_offsets", "etl_dec_bigquery_row_records"):
        getattr(L, f).argtypes = [vp, C.c_int]
        getattr(L, f).restype = C.c_void_p
    L.etl_dec_bigquery_issues.argtypes = [vp, C.POINTER(BigQueryIssues)]
    L.etl_dec_bigquery_free.argtypes = [vp]
    L.etl_dec_bigquery_free.restype = None
    L.etl_dec_ducklake_emit.argtypes = [vp, C.c_uint32, C.POINTER(C.c_char_p), C.c_uint32, C.c_int, C.POINTER(vp)]
    L.etl_dec_ducklake_mutations.argtypes = [vp]
    L.etl_dec_ducklake_mutations.restype = C.c_uint64
    for f in ("etl_dec_ducklake_kinds", "etl_dec_ducklake_records"):
        getattr(L, f).argtypes = [vp, C.c_int]
        getattr(L, f).restype = C.c_void_p
    L.etl_dec_ducklake_text.argtypes = [vp, C.c_uint32, C.c_int, C.POINTER(vp), C.POINTER(vp), C.POINTER(C.c_uint64)]
    L.etl_dec_ducklake_issues.argtypes = [vp, C.POINTER(DuckLakeIssues)]
    L.etl_dec_ducklake_sub_batches.argtypes = [vp, C.c_char_p, C.c_uint32, C.POINTER(C.c_uint64), C.c_int, C.POINTER(vp),
                                               C.POINTER(C.c_uint64)]
    L.etl_dec_ducklake_copy_fingerprint.argtypes = [vp, C.c_char_p, C.c_uint32, C.POINTER(C.c_uint64)]
    L.etl_dec_ducklake_free.argtypes = [vp]
    L.etl_dec_ducklake_free.restype = None
    L.etl_dec_parquet_write.argtypes = [vp, C.POINTER(ParquetField), C.c_uint32, C.c_uint64, C.c_uint64, C.c_uint32, C.c_int,
                                        C.POINTER(vp)]
    L.etl_dec_parquet_write_bloom.argtypes = [vp, C.POINTER(ParquetField), C.POINTER(ParquetBloom), C.c_uint32, C.c_uint64,
                                              C.c_uint64, C.c_uint32, C.c_int, C.POINTER(vp)]
    L.etl_dec_parquet_size.argtypes = [vp]
    L.etl_dec_parquet_size.restype = C.c_uint64
    L.etl_dec_parquet_bytes.argtypes = [vp, C.c_int]
    L.etl_dec_parquet_bytes.restype = C.c_void_p
    L.etl_dec_parquet_metrics.argtypes = [vp, C.c_uint32, C.POINTER(ParquetMetrics)]
    L.etl_dec_parquet_required_null.argtypes = [vp, C.POINTER(C.c_uint32), C.POINTER(C.c_uint64)]
    L.etl_dec_parquet_free.argtypes = [vp]
    L.etl_dec_parquet_free.restype = None
    L.etl_dec_parquet_write_files.argtypes = [vp, C.POINTER(ParquetField), C.POINTER(ParquetBloom), C.c_uint32,
                                              C.POINTER(C.c_uint64), C.c_uint64, C.c_uint32, C.c_int, C.POINTER(vp)]
    L.etl_dec_parquet_files_count.argtypes = [vp]
    L.etl_dec_parquet_files_count.restype = C.c_uint64
    L.etl_dec_parquet_files_offsets.argtypes = [vp]
    L.etl_dec_parquet_files_offsets.restype = C.c_void_p
    L.etl_dec_parquet_files_bytes.argtypes = [vp, C.c_int]
    L.etl_dec_parquet_files_bytes.restype = C.c_void_p
    L.etl_dec_parquet_files_metrics.argtypes = [vp, C.c_uint64, C.c_uint32, C.POINTER(ParquetMetrics)]
    L.etl_dec_parquet_files_required_null.argtypes = [vp, C.POINTER(C.c_uint32), C.POINTER(C.c_uint64)]
    L.etl_dec_parquet_files_free.argtypes = [vp]
    L.etl_dec_parquet_files_free.restype = None
    L.etl_dec_iceberg_partition.argtypes = [vp, C.POINTER(IcebergPartitionField), C.c_uint32, C.c_uint64, C.c_uint64, C.c_int,
                                            C.POINTER(vp)]
    L.etl_dec_iceberg_partitions.argtypes = [vp]
    L.etl_dec_iceberg_partitions.restype = C.c_uint64
    L.etl_dec_iceberg_partition_rows.argtypes = [vp, C.c_int]
    L.etl_dec_iceberg_partition_rows.restype = C.c_void_p
    L.etl_dec_iceberg_partition_value.argtypes = [vp, C.c_uint64, C.c_uint32, C.POINTER(IcebergPartitionValue)]
    L.etl_dec_iceberg_partitioned_arrow.argtypes = [vp]
    L.etl_dec_iceberg_partitioned_arrow.restype = C.c_void_p
    L.etl_dec_iceberg_partition_free.argtypes = [vp]
    L.etl_dec_iceberg_partition_free.restype = None
    L.etl_dec_batch_device_stream.argtypes = [vp]
    L.etl_dec_batch_device_stream.restype = C.c_void_p
    L.etl_shim_materialise.argtypes = [vp, vp, vp, C.POINTER(vp)]
    for f in ("etl_shim_event_count", "etl_shim_total_size_hint", "etl_shim_owned_bytes"):
        getattr(L, f).argtypes = [vp]
        getattr(L, f).restype = C.c_uint64
    L.etl_shim_size_hint.argtypes = [vp, C.c_uint64]
    L.etl_shim_size_hint.restype = C.c_uint64
    L.etl_shim_json_text.argtypes = [vp, C.c_uint64, C.c_uint32, C.c_char_p, C.c_uint64]
    L.etl_shim_json_text.restype = C.c_int64
    L.etl_shim_event_list_free.argtypes = [vp]
    L.etl_shim_event_list_free.restype = None
    _lib = L
    return L


RESULTS_TO_HOST = 0x1
NO_TIMING = 0x4

# etl_dec_arrow_emit row_kinds bit: Numeric / Json columns as formatted Utf8, array columns as List (ETL_ARROW_ALL_COLUMNS)
ARROW_ALL_COLUMNS = 0x100
ARROW_LIST = 13
# row_kinds bit: append cdc_operation and sequence_number, the Iceberg CDC columns (ETL_ARROW_CDC_COLUMNS)
ARROW_CDC_COLUMNS = 0x200

# etl_bq_issue.kind (ETL_BQ_ISSUE_*)
BQ_ISSUE_ARRAY_NULL = 1
BQ_ISSUE_NUMERIC_SCALE = 2
BQ_ISSUE_JSON_INTEGER = 3

# etl_dec_ducklake_* (ETL_DL_*)
DL_INSERT, DL_UPDATE, DL_UPDATE_PARTIAL, DL_REPLACE, DL_DELETE, DL_MF_ARRAY = 1, 2, 3, 4, 5, 0x80
DL_TEXT_ROW, DL_TEXT_PREDICATE, DL_TEXT_ASSIGNMENTS = 0, 1, 2
DL_REJECT_UPDATE_NO_IDENTITY, DL_REJECT_DELETE_NO_IDENTITY, DL_REJECT_DELETE_NO_OLD_ROW, DL_REJECT_PARTIAL_KEY_MISSING = 1, 2, 3, 4

# etl_dec_parquet_write codecs (ETL_PQ_*) and etl_parquet_metrics.flags
PQ_UNCOMPRESSED, PQ_SNAPPY, PQ_ZSTD = 0, 1, 6
PQ_HAS_MIN_MAX = 1
# codec bit: dictionary-encode the eligible column chunks (ETL_PQ_DICTIONARY)
PQ_DICTIONARY = 0x100
# codec bit: write a ColumnIndex and an OffsetIndex per column chunk (ETL_PQ_PAGE_INDEX)
PQ_PAGE_INDEX = 0x400

# etl_iceberg_partition_field.transform (ETL_ICE_*) and the most fields of one spec (ETL_ICE_MAX_FIELDS)
ICE_IDENTITY, ICE_BUCKET, ICE_TRUNCATE, ICE_YEAR, ICE_MONTH, ICE_DAY, ICE_HOUR, ICE_VOID = range(8)
ICE_MAX_FIELDS = 16

# etl_dec_summary.sizing bits (ETL_SIZING_*)
SIZING_EXACT = 0x01
SIZING_OPTIMISTIC = 0x02
SIZING_RERUN_RECORDS = 0x04
SIZING_RERUN_CELLS = 0x08
SIZING_SCRATCH_RESTART = 0x10
SIZING_ARRAY_HEAP_RETRY = 0x20
SIZING_LONG_PASSES_LATE = 0x40
SIZING_NAMES = {SIZING_EXACT: "EXACT", SIZING_OPTIMISTIC: "OPTIMISTIC", SIZING_RERUN_RECORDS: "RERUN_RECORDS",
                SIZING_RERUN_CELLS: "RERUN_CELLS", SIZING_SCRATCH_RESTART: "SCRATCH_RESTART",
                SIZING_ARRAY_HEAP_RETRY: "ARRAY_HEAP_RETRY", SIZING_LONG_PASSES_LATE: "LONG_PASSES_LATE"}
