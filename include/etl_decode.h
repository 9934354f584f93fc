/*
 * etl_decode.h — C ABI of the H100 batched pgoutput (CDC) decode engine.
 *
 * This is the drop-in boundary for supabase/etl's streaming-replication hot path. The reference
 * has no FFI seam at the decoder; the entry points below are what a Rust shim in `crates/etl`
 * binds in place of:
 *
 *   reference interface replaced                                   | entry point here
 *   ---------------------------------------------------------------+-----------------------------
 *   EventsStream::poll_next  (crates/etl/src/replication/stream.rs:291-306): one parsed message
 *     per poll → raw CopyData bodies appended to a pinned staging buffer              | etl_stage_*
 *   SchemaStore / SharedTableCache lookups done per message
 *     (crates/etl/src/replication/apply.rs:2062-2079, :3324-3357)                   | etl_dec_put_table_schema
 *   ApplyLoop::handle_replication_message → handle_logical_replication_message →
 *     handle_{begin,commit,relation,insert,update,delete,truncate}_message
 *     (apply.rs:1687-2248) + conversions::event::parse_event_from_*_message
 *     (crates/etl/src/conversions/event.rs:276-543) + parse_cell_from_postgres_text
 *     (crates/etl/src/conversions/text.rs:28-173) for a whole batch at once          | etl_dec_decode
 *   Vec<Event> handed to ApplyLoopState::add_event_to_batch (apply.rs:433-439)        | etl_dec_batch_* accessors
 *
 * Conventions (SURVEY.md §8b): every function returns 0 on success and a non-zero
 * `etl_status` on infrastructure failure (CUDA, allocation, bad arguments). DATA errors are not
 * return codes: they are reported as `first_error` inside a successfully returned batch whose
 * records [0, first_error.record_index) are valid — mirroring apply.rs:1595-1599 where earlier
 * events stay in the batch and the failing message returns Err. One ctx per apply loop; calls on
 * one ctx are not re-entrant. All integers are host (little-endian) order. No torch / C++ types
 * cross this boundary.
 */
#ifndef ETL_DECODE_H
#define ETL_DECODE_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ETL_DECODE_ABI_VERSION 2u

/* ---------------------------------------------------------------- status codes */
typedef enum etl_status {
  ETL_OK = 0,
  ETL_ERR_INVALID_ARG = 1,
  ETL_ERR_CUDA = 2,
  ETL_ERR_ALLOC = 3,
  ETL_ERR_NO_DEVICE = 4,
  ETL_ERR_INTERNAL = 5,
} etl_status;

/* ---------------------------------------------------------------- record kinds
 * rec_kind is the pgoutput tag byte of the frame (XLogData 'w' frames), or 'k' for a primary
 * keepalive frame. Grammar: SURVEY.md Appendix B. */
enum {
  ETL_REC_BEGIN = 'B',
  ETL_REC_COMMIT = 'C',
  ETL_REC_ORIGIN = 'O',
  ETL_REC_RELATION = 'R',
  ETL_REC_TYPE = 'Y',
  ETL_REC_INSERT = 'I',
  ETL_REC_UPDATE = 'U',
  ETL_REC_DELETE = 'D',
  ETL_REC_TRUNCATE = 'T',
  ETL_REC_MESSAGE = 'M',
  ETL_REC_KEEPALIVE = 'k',
};

/* rec_flags bits */
enum {
  ETL_RF_OLD_FULL = 0x01,    /* 'O' image present: OldTableRow::Full   (event.rs:445-448) */
  ETL_RF_OLD_KEY = 0x02,     /* 'K' image present: OldTableRow::Key    (event.rs:441-444) */
  ETL_RF_NEW_PARTIAL = 0x04, /* UpdatedTableRow::Partial               (event.rs:662-667) */
  ETL_RF_DDL_MESSAGE = 0x08, /* 'M' whose prefix is supabase_etl_ddl   (event.rs:31)      */
  ETL_RF_EVENT = 0x80,       /* the reference emits an Event for this frame               */
};

/* ---------------------------------------------------------------- cell tags = Cell variants
 * crates/etl/src/types/cell.rs:38-76, in declaration order. */
enum {
  ETL_CELL_NULL = 0,
  ETL_CELL_BOOL = 1,        /* val = 0|1 */
  ETL_CELL_STRING = 2,      /* val = byte offset into the staged stream, aux = byte length (zero copy) */
  ETL_CELL_I16 = 3,         /* val = sign-extended value */
  ETL_CELL_I32 = 4,
  ETL_CELL_U32 = 5,
  ETL_CELL_I64 = 6,
  ETL_CELL_F32 = 7,         /* val = IEEE-754 bits (low 32) */
  ETL_CELL_F64 = 8,         /* val = IEEE-754 bits */
  ETL_CELL_NUMERIC = 9,     /* val = heap offset of etl_numeric_hdr, aux = number of base-10000 digits */
  ETL_CELL_DATE = 10,       /* val = days since 1970-01-01 (signed) */
  ETL_CELL_TIME = 11,       /* val = seconds since midnight, aux = nanoseconds (>= 1e9 only for :60 leap second) */
  ETL_CELL_TIMESTAMP = 12,  /* val = seconds since 1970-01-01T00:00:00 (naive), aux = nanoseconds */
  ETL_CELL_TIMESTAMPTZ = 13,/* val = UTC seconds since the unix epoch, aux = nanoseconds */
  ETL_CELL_UUID = 14,       /* val = heap offset of 16 big-endian bytes */
  ETL_CELL_JSON = 15,       /* val = stream byte offset, aux = byte length of the VALIDATED json text */
  ETL_CELL_BYTES = 16,      /* val = heap offset of decoded bytes, aux = length */
  ETL_CELL_ARRAY = 17,      /* val = heap offset of etl_array_hdr, aux = element count */
  ETL_CELL_MISSING = 254,   /* unresolved UnchangedToast → PartialTableRow missing index (event.rs:641-656) */
};

/* column decode classes derived from the type oid exactly as text.rs:28-173 dispatches */
enum {
  ETL_K_BOOL = 1, ETL_K_STRING = 2, ETL_K_I16 = 3, ETL_K_I32 = 4, ETL_K_U32 = 5, ETL_K_I64 = 6,
  ETL_K_F32 = 7, ETL_K_F64 = 8, ETL_K_NUMERIC = 9, ETL_K_DATE = 10, ETL_K_TIME = 11,
  ETL_K_TIMESTAMP = 12, ETL_K_TIMESTAMPTZ = 13, ETL_K_UUID = 14, ETL_K_JSON = 15, ETL_K_BYTES = 16,
  ETL_K_ARRAY = 0x20, /* ETL_K_ARRAY | element kind */
};

/* numeric heap entry: header followed by `aux` little-endian int16 base-10000 digits.
 * crates/etl/src/conversions/numeric.rs:67-88 */
typedef struct etl_numeric_hdr {
  uint8_t kind;   /* 0 value, 1 NaN, 2 +Infinity, 3 -Infinity */
  uint8_t sign;   /* 0 positive, 1 negative */
  int16_t weight;
  uint16_t scale;
  uint16_t pushed_groups; /* base-10000 groups the reference pushes onto its digit Vec before stripping zero groups
                             (numeric.rs:441-448; 0 for canonical zero and the specials, saturates at 65535): the
                             Vec's capacity — and with it the row's size hint — follows from this count */
} etl_numeric_hdr;

/* array heap entry: header followed by n_elems etl_array_elem (8-byte aligned). Element payloads
 * (unescaped strings, numerics, bytes, uuids) live in the heap at elem.val. text.rs:184-249 */
typedef struct etl_array_hdr {
  uint8_t elem_kind; /* ETL_K_* of the element type */
  uint8_t _pad[3];
  uint32_t n_elems;
} etl_array_hdr;
typedef struct etl_array_elem {
  uint64_t val;
  uint32_t aux;
  uint8_t tag;   /* ETL_CELL_* (ETL_CELL_NULL for a NULL element) */
  uint8_t _pad[3];
} etl_array_elem;

/* ---------------------------------------------------------------- data-error descriptions
 * (ErrorKind, description) pairs the path can raise. crates/etl/src/error.rs */
typedef enum etl_error_kind {
  ETL_EK_NONE = 0,
  ETL_EK_CONVERSION_ERROR = 1,
  ETL_EK_INVALID_DATA = 2,
  ETL_EK_DESERIALIZATION_ERROR = 3,
  ETL_EK_INVALID_STATE = 4,
  ETL_EK_VALIDATION_ERROR = 5,
  ETL_EK_CORRUPTED_TABLE_SCHEMA = 6,
  ETL_EK_MISSING_TABLE_SCHEMA = 7,
  ETL_EK_SOURCE_ERROR = 8, /* malformed frame: the third-party parser returns io::Error */
} etl_error_kind;

typedef enum etl_error_code {
  ETL_E_NONE = 0,
  ETL_E_UTF8 = 1,               /* ConversionError  "UTF-8 conversion failed"            error.rs:480-489 */
  ETL_E_PARSE_INT = 2,          /* ConversionError  "Integer parsing failed"             error.rs:510    */
  ETL_E_PARSE_FLOAT = 3,        /* ConversionError  "Float parsing failed"               error.rs:525    */
  ETL_E_DATETIME = 4,           /* ConversionError  "Datetime parsing failed"            error.rs:878    */
  ETL_E_NUMERIC = 5,            /* ConversionError  "Numeric parsing failed"             error.rs:893    */
  ETL_E_UUID = 6,               /* InvalidData      "UUID parsing failed"                error.rs:863    */
  ETL_E_JSON = 7,               /* DeserializationError "JSON deserialization failed"    error.rs:456-463 */
  ETL_E_BOOL = 8,               /* InvalidData      "Invalid boolean value"              bool.rs:17      */
  ETL_E_BYTEA = 9,              /* ConversionError  "Bytea hex string conversion failed" hex.rs:12-29    */
  ETL_E_BINARY_FORMAT = 10,     /* ConversionError  "Binary format not supported in tuple data" event.rs:976 */
  ETL_E_NOT_NULL = 11,          /* InvalidData      "Required column missing from tuple" event.rs:947-955 */
  ETL_E_FIELD_COUNT = 12,       /* ConversionError  "Tuple data field count does not match schema" event.rs:556,608 */
  ETL_E_FULL_ROW_MISSING = 13,  /* ConversionError  "Tuple missing source value for full row image" event.rs:568 */
  ETL_E_KEY_NO_COLUMNS = 14,    /* ConversionError  "Replica-identity tuple missing key columns" event.rs:890 */
  ETL_E_KEY_SHAPE = 15,         /* ConversionError  "Replica-identity tuple shape does not match schema" event.rs:907 */
  ETL_E_KEY_MISSING_VALUE = 16, /* ConversionError  "Replica-identity tuple missing source value" event.rs:803,847 */
  ETL_E_TX_STATE = 17,          /* InvalidState     "Invalid transaction state"          apply.rs:1955,2018,2098,... */
  ETL_E_COMMIT_LSN = 18,        /* ValidationError  "Invalid commit LSN"                 apply.rs:1960-1969 */
  ETL_E_MISSING_TABLE_STATE = 19,/* InvalidState    "Missing shared table state"         apply.rs:3328-3337 */
  ETL_E_ARRAY_SHORT = 20,       /* ConversionError  "Array input too short"              text.rs:190 */
  ETL_E_ARRAY_BRACES = 21,      /* ConversionError  "Array input missing braces"         text.rs:194 */
  ETL_E_UNKNOWN_COLUMNS = 22,   /* CorruptedTableSchema "Received columns during replication that are not in the stored table schema" error.rs:960-975 */
  ETL_E_MISSING_TABLE_SCHEMA = 23,/* MissingTableSchema  stored TableSchema absent for a Relation (apply.rs:2062-2072) */
  ETL_E_MALFORMED_FRAME = 24,   /* SourceError: truncated frame / unknown tag (postgres-replication parse error) */
  ETL_E_COPY_NOT_TERMINATED = 25, /* ConversionError "Row data not properly terminated"                  table_row.rs:88-92 */
  ETL_E_COPY_COLUMN_COUNT = 26,  /* ConversionError "Column count mismatch between schema and row"     table_row.rs:103-113,150-160 */
  ETL_E__COUNT
} etl_error_code;

typedef struct etl_first_error {
  uint64_t record_index; /* UINT64_MAX when the batch decoded cleanly */
  uint32_t seq;          /* evaluation step inside the record (old tuple cells, then new tuple cells) */
  uint32_t code;         /* etl_error_code */
  uint32_t kind;         /* etl_error_kind */
  uint32_t _pad;
} etl_first_error;

/* ---------------------------------------------------------------- schema catalogue
 * ColumnSchema — crates/etl-postgres/src/types/schema.rs:165-179 */
typedef struct etl_column_schema {
  const char* name;        /* UTF-8, NUL terminated */
  uint32_t type_oid;
  int32_t modifier;
  int32_t ordinal_position;
  int32_t primary_key_ordinal_position; /* -1 = not part of the primary key */
  uint8_t nullable;
  uint8_t _pad[7];
} etl_column_schema;

/* stream state carried between batches — ApplyLoopState {remote_final_lsn, next_tx_ordinal}
 * apply.rs:600-626 */
typedef struct etl_stream_state {
  uint64_t final_lsn;       /* valid when in_tx != 0 */
  uint64_t next_tx_ordinal;
  uint8_t in_tx;            /* remote_final_lsn.is_some() */
  uint8_t _pad[7];
} etl_stream_state;

/* ---------------------------------------------------------------- staging
 * The stager is the replacement for the per-message parse in EventsStream: each CopyData body
 * (what `copy_both_simple::<Bytes>` yields, crates/etl/src/replication/client.rs:1098-1099) is
 * appended as 'd' + int32(len+4, big-endian) + body into one pinned host buffer. While appending
 * it records, for free, (a) sparse anchors: anchors[k] = offset of the first frame that starts at
 * or after k*anchor_stride (len if none), and (b) the offsets of Relation frames. */
typedef struct etl_stager etl_stager;
int etl_stage_create(uint64_t capacity_bytes, uint32_t anchor_stride, etl_stager** out);
void etl_stage_destroy(etl_stager*);
void etl_stage_reset(etl_stager*);
int etl_stage_append(etl_stager*, const uint8_t* copydata_body, uint32_t body_len);
/* adopt an already framed stream (bench/tests): walks it once on the host to build the indexes */
int etl_stage_append_framed(etl_stager*, const uint8_t* framed, uint64_t len);

typedef struct etl_dec_input {
  const uint8_t* host_buf;       /* framed stream in host memory (pinned if from the stager) */
  const uint8_t* dev_buf;        /* optional: same bytes already resident in HBM (NULL → library copies). PRECONDITION:
                                    16-byte aligned and followed by at least 64 readable bytes after `len` — the
                                    kernels read whole aligned words / 16-byte copy granules around a cell. The
                                    library's own copy of host_buf is padded for you. */
  uint64_t len;
  const uint64_t* anchors;       /* host array, n_anchors entries, see etl_stager */
  const uint64_t* dev_anchors;   /* optional: n_anchors + 1 entries resident in HBM, last entry = len. Anchors are
                                    not trusted: the kernels clamp them to `len` and treat a non-ascending pair as an
                                    empty segment; an anchor that is not a frame start yields ETL_E_MALFORMED_FRAME. */
  uint64_t n_anchors;
  uint32_t anchor_stride;
  uint32_t max_frame_len;        /* 0 = unknown; else an upper bound of the longest frame in bytes ('d' + length field +
                                    body; the stager fills it).  A hint: when no frame can hold a 512-byte value the
                                    passes that exist for long values are skipped (and run after all if it was wrong) */
  const uint64_t* relation_offsets; /* host array: frame offsets of every 'R' frame, ascending */
  uint64_t n_relations;
  etl_stream_state carry_in;
} etl_dec_input;
int etl_stage_view(const etl_stager*, etl_dec_input* out);

/* ---------------------------------------------------------------- decoder */
typedef struct etl_dec_ctx etl_dec_ctx;
typedef struct etl_dec_batch etl_dec_batch;

/* One context = one apply loop on one GPU (the harness and the shim run one process / thread per GPU).  SURVEY §8b
 * sketched `etl_dec_create(const int* device_ids, int n_dev, …)`; with one owner per device the multi-GPU form is
 * etl_dec_create + etl_dec_comm_init(rank, n_ranks) below, which gives the context its NCCL communicator. */
int etl_dec_create(int device_id, etl_dec_ctx** out);
/* run on the caller's CUDA stream (a cudaStream_t, e.g. torch.cuda.current_stream().cuda_stream);
 * default: a private stream created by etl_dec_create */
int etl_dec_set_stream(etl_dec_ctx*, void* cuda_stream);
void etl_dec_destroy(etl_dec_ctx*);
const char* etl_dec_last_error(const etl_dec_ctx*);
uint32_t etl_dec_abi_version(void);

/* store (or replace) the TableSchema the SchemaStore would return for table_id */
int etl_dec_put_table_schema(etl_dec_ctx*, uint32_t table_id, uint64_t snapshot_id,
                             const etl_column_schema* cols, uint32_t n_cols);
/* forget replicated-schema state (new connection: Postgres re-sends Relation messages) */
int etl_dec_reset_relations(etl_dec_ctx*);
/* ETL_K_* decode class of a type oid, exactly as text.rs:28-173 dispatches (utils.rs:7-16 for unknown oids) */
uint32_t etl_dec_kind_for_type_oid(uint32_t type_oid);
/* free / total device memory as the CUDA runtime reports it (leak checks) */
int etl_dec_mem_info(etl_dec_ctx*, uint64_t* free_bytes, uint64_t* total_bytes);

/* ---------------------------------------------------------------- multi-GPU (SURVEY §8e)
 * The staged stream shards by byte range at record starts, one range per GPU of a box; the library owns the
 * exchange: an NCCL communicator over the ranks (libnccl.so.2 is resolved at run time — the copy already loaded
 * into the process if there is one).  etl_dec_decode_sharded runs
 *   relation-update exchange (the Relation frames of every range, one all-gather; apply.rs:2012-2089,
 *   table_cache.rs:36-130) → index pass → ncclAllGather of the 64-byte seam summaries ON THE DECODE STREAM →
 *   device-side fold of the ranks before this one into the carry-in (apply.rs:600-626) → record + tuple passes
 * with no host round trip between the index and the record pass.  `carry_in` of the input is the state before the
 * FIRST shard (pass the same value on every rank); summary.carry_out is the state after the LAST shard and
 * summary.record_index_base the global index of this rank's first record.  Output order = rank order. */
#define ETL_COMM_ID_BYTES 128u
int etl_dec_comm_unique_id(uint8_t* out, uint32_t cap);   /* rank 0; broadcast the bytes to the other ranks */
int etl_dec_comm_init(etl_dec_ctx*, const uint8_t* unique_id, uint32_t id_bytes, int rank, int n_ranks);
/* The same protocol with the two exchanges carried by the HOST (a box without NVLink/NCCL between the processes, tests
 * on one GPU): `fn(user, send, recv, bytes)` must fill recv with the n_ranks blocks of `bytes` in rank order, return 0. */
typedef int (*etl_host_allgather_fn)(void* user, const void* send, void* recv, uint64_t bytes);
int etl_dec_comm_init_host(etl_dec_ctx*, int rank, int n_ranks, etl_host_allgather_fn fn, void* user);

/* flags for etl_dec_decode */
enum {
  ETL_DECODE_RESULTS_TO_HOST = 0x1, /* copy result planes to pinned host memory before returning */
  ETL_DECODE_SEAM_DEFER = 0x2,      /* multi-GPU shard: carry_in unknown, run only the local scan;
                                       caller exchanges etl_dec_seam and calls etl_dec_decode_finish */
  ETL_DECODE_NO_TIMING = 0x4,       /* leave the *_ms fields of the summary at 0: the CUDA-event queries behind them cost
                                       host time on every call, which an 8 MiB batch notices */
};

/* per-shard seam summary exchanged with ONE all-gather across the GPUs of a box (SURVEY §8e) */
typedef struct etl_dec_seam {
  uint64_t n_records;
  uint64_t n_cells;
  uint64_t heap_bytes;
  uint64_t lsn;        /* final_lsn of the last Begin in the shard (valid if has_begin) */
  uint64_t ord;        /* has_begin: next_tx_ordinal at shard end; else ordinal consumers in shard */
  uint8_t has_begin;
  uint8_t closed;      /* a Commit follows the last Begin (or any Commit when !has_begin) */
  uint8_t _pad[6];
} etl_dec_seam;

/* Limits of one call: len < 1 TiB and fewer than 2^32 frames (record indices inside a batch are 32-bit: a 64 GiB
 * stream of nothing but 23-byte keepalives is still below it); a longer stream is decoded in several calls chained
 * through carry_in / carry_out, like the reference's batches. */
int etl_dec_decode(etl_dec_ctx*, const etl_dec_input*, uint32_t flags, etl_dec_batch** out);
int etl_dec_decode_sharded(etl_dec_ctx*, const etl_dec_input*, uint32_t flags, etl_dec_batch** out);
/* two-phase form: the caller exchanges the seam summaries itself (tests; hosts without NCCL) */
int etl_dec_decode_begin(etl_dec_ctx*, const etl_dec_input*, uint32_t flags, etl_dec_seam* seam_out);
int etl_dec_decode_finish(etl_dec_ctx*, const etl_stream_state* carry_in, uint64_t record_index_base,
                          etl_dec_batch** out);
void etl_dec_batch_free(etl_dec_batch*);

/* result planes. Device planes are owned by the batch. Host planes exist only when
 * ETL_DECODE_RESULTS_TO_HOST was set; they live in a pinned buffer cached on the ctx and stay
 * valid until the next decode on the same ctx. All arrays are in stream order. */
typedef struct etl_dec_planes {
  uint64_t n_records;
  uint64_t n_cells;
  uint64_t heap_bytes;
  /* record plane (n_records entries; rec_cell_base has n_records + 1) */
  const uint64_t* rec_off;
  const uint8_t* rec_kind;
  const uint8_t* rec_flags;
  const uint32_t* rec_rel;       /* relation id (R/I/U/D), relation count (T) */
  const int32_t* rec_schema;     /* schema version index (see etl_dec_batch_schema), -1 if none */
  const uint64_t* rec_start_lsn;
  const uint64_t* rec_commit_lsn;
  const uint64_t* rec_tx_ordinal;
  const uint64_t* rec_cell_base;
  const uint32_t* rec_tuple_bytes; /* DML: Σ text lengths of the frame's tuples = the ETL_ROW_SIZE_BYTES histogram sample
                                      (calculate_tuple_bytes, event.rs:260-270, :388, :462, :507); 0 for other records */
  const uint32_t* rec_heap_hint;   /* DML: Σ estimate_cell_allocated_bytes (types/table_row.rs:295-345) over the String,
                                      Bytes and Numeric cells of the event's rows — the part of Event::size_hint
                                      (types/event.rs:288-312) that depends on the data; the struct sizes and Vec<Cell>
                                      capacities follow from rec_kind / rec_flags / the schema. Json and Array payloads
                                      are estimated by whoever builds the serde_json::Value / ArrayCell. */
  /* cell plane */
  const uint8_t* cell_tag;
  const uint64_t* cell_val;
  const uint32_t* cell_aux;
  /* heap */
  const uint8_t* heap;
} etl_dec_planes;

typedef struct etl_dec_summary {
  etl_first_error first_error;
  etl_stream_state carry_out;
  uint64_t insert_bytes;  /* ETL_BYTES_PROCESSED_TOTAL{insert}: calculate_tuple_bytes event.rs:260-270 */
  uint64_t update_bytes;
  uint64_t delete_bytes;
  uint64_t n_events;      /* frames with ETL_RF_EVENT */
  uint32_t n_schemas;     /* schema versions referenced by rec_schema */
  uint32_t gpu_launches;  /* kernels launched for this batch */
  float kernel_ms;        /* CUDA-event time of the kernel sequence (resident input → resident output) */
  float h2d_ms, d2h_ms;
  float index_ms;         /* pass A: k_act_* + k_chase (frame offsets) [+ the totals-only k_records pass] */
  float emit_ms;          /* pass B+C: k_records … k_long_cells */
  float frames_ms;        /* k_records (stream-state scan + record plane) */
  float walk_ms;          /* k_bin_scan + k_perm (shape bins) */
  float spans_ms;         /* k_utf8_dead (structure-blind UTF-8 pass over segments without a frame start) */
  float cells_ms;         /* k_rows (tuples → rows: staging, walk, UTF-8, per-kind parsers, cell plane) */
  float long_ms;          /* k_long_cells (verdicts of the long text cells: line bitmap + edges) */
  uint64_t h2d_bytes, d2h_bytes; /* bytes copied host→device / device→host for this batch */
  uint64_t span_bytes;    /* bytes streamed by k_utf8_dead (its algorithmic bytes) */
  uint64_t record_index_base; /* global index of this batch's first record (sharded decode: Σ records of the ranks before) */
  uint32_t abi_version;
  uint32_t sizing;        /* ETL_SIZING_* bits: how the planes of this batch were sized, every branch the decode went through */
} etl_dec_summary;

/* etl_dec_summary.sizing — diagnostic only (the planes are the same whichever path was taken; a shim may log how often
 * the optimistic sizes miss).  The first batch of a context, decode_finish and COPY rows size the planes from exact
 * counts (EXACT).  Every later batch reserves planes from what earlier batches needed per staged byte (OPTIMISTIC); when
 * the device reports that the batch does not fit, the host counts it exactly and runs the tuple pass again
 * (RERUN_RECORDS: more records than reserved, nothing was written; RERUN_CELLS: more cells than reserved, the records
 * of the CTAs before the overflow were written and are overwritten).  More frames than the offset scratch holds
 * abandons the attempt and decodes the batch again on the exact path (SCRATCH_RESTART, together with the bits of the
 * abandoned attempt and EXACT).  An array value that did not fit its heap reservation: larger heap, tuple pass again
 * (ARRAY_HEAP_RETRY).  The frame-length hint promised no long values but there were some: the long-value passes ran
 * after the tuple pass (LONG_PASSES_LATE). */
enum {
  ETL_SIZING_EXACT = 0x01,
  ETL_SIZING_OPTIMISTIC = 0x02,
  ETL_SIZING_RERUN_RECORDS = 0x04,
  ETL_SIZING_RERUN_CELLS = 0x08,
  ETL_SIZING_SCRATCH_RESTART = 0x10,
  ETL_SIZING_ARRAY_HEAP_RETRY = 0x20,
  ETL_SIZING_LONG_PASSES_LATE = 0x40,
};

int etl_dec_batch_planes(const etl_dec_batch*, int host, etl_dec_planes* out);
int etl_dec_batch_summary(const etl_dec_batch*, etl_dec_summary* out);

/* replicated schema version i: what ReplicatedTableSchema exposes to events (schema.rs:651-900) */
typedef struct etl_dec_schema_info {
  uint32_t table_id;
  uint32_t n_cols;          /* replicated columns */
  uint32_t n_identity;
  uint32_t _pad;
  uint64_t snapshot_id;
  uint64_t effective_off;   /* stream offset of the Relation frame that installed it (0 = carried in) */
  const uint8_t* col_kind;  /* n_cols ETL_K_* */
  const uint8_t* col_flags; /* bit0 nullable, bit1 identity */
  const int32_t* col_index; /* index into the stored TableSchema's column list */
} etl_dec_schema_info;
int etl_dec_batch_schema(const etl_dec_batch*, uint32_t index, etl_dec_schema_info* out);

/* ---------------------------------------------------------------- initial-sync COPY rows (SURVEY §8f N1)
 * Replaces parse_table_row_from_postgres_copy_bytes (crates/etl/src/conversions/table_row.rs:25-165) applied row by
 * row by TableCopyStream::poll_next (crates/etl/src/replication/stream.rs:75-101) for a whole buffer of rows.
 * `buf` holds the COPY-text rows back to back exactly as the CopyData bodies arrive (each ends with its LF);
 * row_offsets has n_rows + 1 ascending entries (row r = [row_offsets[r], row_offsets[r+1])).  Same device-buffer
 * precondition as etl_dec_input.dev_buf (16-byte aligned, 64 readable bytes after len).  The table's columns are those
 * of etl_dec_put_table_schema, in order.  Result: an etl_dec_batch whose planes hold n_records = n_rows,
 * n_cells = n_rows * n_cols (row-major: cell r * n_cols + c), rec_off = the row offsets, rec_kind..rec_heap_hint NULL;
 * a string / json cell is a span of `buf` (val = offset) unless the field needed unescaping: then bit 63 of val is
 * set and the low bits are a heap offset.  first_error: record_index = row, seq = 0 for the row's UTF-8 check,
 * 1 + column otherwise; rows before it are valid. */
#define ETL_COPY_VAL_IN_HEAP (1ull << 63)
typedef struct etl_copy_input {
  const uint8_t* host_buf;
  const uint8_t* dev_buf;          /* optional, resident copy */
  uint64_t len;
  const uint64_t* row_offsets;     /* host, n_rows + 1 entries */
  const uint64_t* dev_row_offsets; /* optional, resident copy */
  uint64_t n_rows;
} etl_copy_input;
int etl_dec_copy_decode(etl_dec_ctx*, uint32_t table_id, const etl_copy_input*, uint32_t flags, etl_dec_batch** out);

/* ---------------------------------------------------------------- columnar emitter (SURVEY §8f N2)
 * The rows of ONE replicated-schema version of a decoded batch as Arrow-layout column buffers, built on the device.
 * Replaces the per-row walk of the destinations' encoders (crates/etl-destinations/src/iceberg/encoding.rs:61-330:
 * build_array_for_field and the cell_to_* converters; the DuckLake / BigQuery encoders walk the same Vec<TableRow>) for
 * the column types whose Arrow value depends on the decoded cell alone.  Numeric / Json / Array columns (cell_to_string
 * formatting in the reference) come back as ETL_ARROW_UNSUPPORTED and stay on the shim's row path unless row_kinds has
 * ETL_ARROW_ALL_COLUMNS (below): then they are built on the device too.
 * row_kinds: bit 0 inserts, bit 1 updates (new image, Full rows only), bit 2 deletes (old image, when Full); rows keep
 * stream order and etl_dec_arrow_row_records gives the record index of each (for the CDC columns).
 * A COPY batch (etl_dec_copy_decode; rec_kind == NULL in its planes) is emitted the same way: schema_index must be 0
 * (anything else is ETL_ERR_INVALID_ARG), the columns are those the batch was decoded with (a later
 * etl_dec_put_table_schema does not change them), every row of the valid prefix [0, first_error.record_index) is an
 * insert image selected by bit 0 (without it: zero rows, the columns still typed), and etl_dec_arrow_row_records gives
 * the row index.  The same type mapping, null rules and size limits apply; a String / Json cell with
 * ETL_COPY_VAL_IN_HEAP is read from the heap. */
enum {
  ETL_ARROW_UNSUPPORTED = 0,
  ETL_ARROW_BOOLEAN = 1,        /* values bit-packed like the validity bitmap */
  ETL_ARROW_INT32 = 2,          /* Cell::I16 | I32   (encoding.rs:200-206) */
  ETL_ARROW_INT64 = 3,          /* Cell::I64 | U32   (:214-220) */
  ETL_ARROW_FLOAT32 = 4,
  ETL_ARROW_FLOAT64 = 5,
  ETL_ARROW_UTF8 = 6,           /* int32 offsets[n_rows + 1] + data */
  ETL_ARROW_LARGE_BINARY = 7,   /* int64 offsets[n_rows + 1] + data */
  ETL_ARROW_DATE32 = 8,         /* days since 1970-01-01 (:257-262) */
  ETL_ARROW_TIME64_US = 9,      /* microseconds since midnight (:270-275) */
  ETL_ARROW_TIMESTAMP_US = 10,  /* naive, microseconds since the epoch (:284-289) */
  ETL_ARROW_TIMESTAMPTZ_US = 11,/* UTC, microseconds since the epoch (:297-302) */
  ETL_ARROW_UUID = 12,          /* FixedSizeBinary(16) */
  ETL_ARROW_LIST = 13,          /* List<child>: validity + int32 offsets[n_rows + 1]; values / data NULL; the child column
                                   through etl_dec_arrow_list_child (ETL_ARROW_ALL_COLUMNS only) */
};
/* row_kinds bit: build every column type of the reference's Iceberg schema (iceberg/schema.rs:9-63).  Numeric and Json
 * columns come back as ETL_ARROW_UTF8 holding cell_to_string's text (encoding.rs:338-360): PgNumeric's Display
 * (numeric.rs:503-590) and serde_json::Value's Display — compact, object keys sorted by their unescaped UTF-8 bytes, the
 * last of duplicate keys kept, numbers verbatim, strings escaped the serde_json way (third-party behaviour, parity
 * unpinned).  Array columns come back as ETL_ARROW_LIST (build_list_array, encoding.rs:386-776): a non-array or NULL cell
 * is a null list, `{}` a list of length 0, a NULL element a null child entry; child types Bool → BOOLEAN,
 * I16 / I32 → INT32, I64 / U32 → INT64, F32, F64, Date → DATE32, Time → TIME64_US, Timestamp / TimestampTz →
 * TIMESTAMP_US / TIMESTAMPTZ_US, Uuid → UUID, Bytes → LARGE_BINARY, String / Numeric / Json → UTF8 (formatted as above).
 * Without the bit the output is that of the emitter before it existed.  More than INT32_MAX elements in one List column,
 * or more than 2 GiB of text in a Utf8 child, fail like an oversize Utf8 column (ETL_ERR_INVALID_ARG: split the batch); a
 * Json value that does not parse again (the decode validated it) is ETL_ERR_INTERNAL. */
#define ETL_ARROW_ALL_COLUMNS 0x100u
/* row_kinds bit: append the two columns both Iceberg write paths add to every row (crates/etl-destinations/src/iceberg/
 * core.rs: write_table_rows :239-267, write_events :276-366), so etl_dec_arrow_cols returns n_cols + 2:
 *   column n_cols     cdc_operation:   ETL_ARROW_UTF8, never null, "INSERT" / "UPDATE" / "DELETE" from the row's record
 *                                      kind; COPY rows are "INSERT";
 *   column n_cols + 1 sequence_number: ETL_ARROW_UTF8, never null, EventSequenceKey's Display
 *                                      (crates/etl/src/types/event.rs:331-336) "{rec_commit_lsn:016x}/{rec_tx_ordinal:016x}"
 *                                      in lowercase hex; COPY rows get generate_sequence_number(0, 0)
 *                                      (etl-postgres/src/types/utils.rs:119-139) = "0000000000000000/0000000000000000".
 * Every name is 6 bytes and every key 33, so their offsets are 6 * i and 33 * i.  More than INT32_MAX bytes of keys
 * (about 65 M rows in one emit) fail like an oversize Utf8 column (ETL_ERR_INVALID_ARG: split the batch).  The column
 * names (find_unique_column_name, core.rs:679) are host metadata.  Without the bit the output is what it was before. */
#define ETL_ARROW_CDC_COLUMNS 0x200u
typedef struct etl_arrow_column {
  uint32_t arrow_type;
  uint32_t _pad;
  const uint8_t* validity;  /* bit i = row i is non-null (LSB first), ceil(n_rows / 8) bytes, zero padded to 64 */
  const void* values;       /* fixed-width values, n_rows entries (Boolean: bit-packed); NULL for var-width columns */
  const void* offsets;      /* var-width: n_rows + 1 offsets (int32 for UTF8, int64 for LARGE_BINARY) */
  const uint8_t* data;      /* var-width: the bytes */
  uint64_t data_bytes;
} etl_arrow_column;
typedef struct etl_arrow_batch etl_arrow_batch;
int etl_dec_arrow_emit(const etl_dec_batch*, uint32_t schema_index, uint32_t row_kinds, int to_host, etl_arrow_batch** out);
uint64_t etl_dec_arrow_rows(const etl_arrow_batch*);
uint32_t etl_dec_arrow_cols(const etl_arrow_batch*);
const uint64_t* etl_dec_arrow_row_records(const etl_arrow_batch*, int host);
int etl_dec_arrow_column(const etl_arrow_batch*, uint32_t column, int host, etl_arrow_column* out);
/* the child column of an ETL_ARROW_LIST column (n_elems entries; Utf8: int32 offsets, LargeBinary: int64 offsets) */
int etl_dec_arrow_list_child(const etl_arrow_batch*, uint32_t column, int host, etl_arrow_column* out, uint64_t* n_elems);
/* the smallest batch-local record index, among the records of the emitted schema version in the valid prefix, whose
 * kind row_kinds selects but which cannot become a row: an Update with ETL_RF_NEW_PARTIAL (bit 1) or a Delete without
 * ETL_RF_OLD_FULL (bit 2) — where write_events returns InvalidState (iceberg/core.rs:311-322, :336-357) while the emit
 * leaves the record out.  UINT64_MAX if there is none; always UINT64_MAX for a COPY batch. */
uint64_t etl_dec_arrow_first_skipped(const etl_arrow_batch*);
void etl_dec_arrow_free(etl_arrow_batch*);
/* ---------------------------------------------------------------- ClickHouse RowBinary emitter
 * The rows of ONE replicated-schema version of a decoded batch as the RowBinary byte stream the ClickHouse destination
 * sends in its INSERT bodies, built on the device, plus n_rows + 1 u64 row offsets (row i = [off[i], off[i+1]) of the
 * data).  Replaces the per-row host walk of crates/etl-destinations/src/clickhouse: write_events_inner /
 * flush_pending_rows (core.rs:694-863) and write_table_rows_inner (:489-521) mapping each cell through
 * cell_to_clickhouse_value (encoding.rs:50-78), expand_key_row / default_cell (core.rs:920-997), and
 * encode_to_row_binary (encoding.rs:249-273) called row by row from insert_rows (client.rs:336-379).
 * Rows, in record order, are the records of the version in the valid prefix that carry ETL_RF_EVENT: an Insert's new
 * image; an Update's new image when Full (an Update with ETL_RF_NEW_PARTIAL is no row, see first_partial_update); a
 * Delete's old image when ETL_RF_OLD_FULL, else its key image expanded column by column in schema order: a column whose
 * stored TableSchema column has a primary_key_ordinal_position takes the next key cell (NULL once they run out), a
 * source-nullable non-array column is NULL, any other column gets default_cell, on the wire all zero bytes (Bool 1;
 * I16 2; I32 / U32 / F32 / Date 4; I64 / F64 / Timestamp / TimestampTz 8; Uuid 16; String, Numeric, Time, Json, Bytes
 * and arrays 1: an empty string or array).  A COPY batch (rec_kind == NULL): every row of the valid prefix, schema_index
 * must be 0.  Each row holds the n_cols user columns, then cdc_operation (String "INSERT" / "UPDATE" / "DELETE"; COPY
 * rows "INSERT") and cdc_lsn (UInt64, the record's rec_commit_lsn; COPY rows 0).
 * nullable_flags: n_cols + 2 bytes, non-zero = the ClickHouse column is Nullable(...) (the table's actual types,
 * nullable_flags_from_clickhouse_columns, core.rs:102-142); any other n_flags is ETL_ERR_INVALID_ARG.  A flagged column
 * writes a marker byte (1 NULL, 0 value) before its value.  Values follow the cell's variant (rb_encode_value,
 * encoding.rs:201-246): Bool 1 byte; I16 / I32 / I64 / U32 and the IEEE bits of F32 / F64 little-endian; Date → Date32
 * i32 days; Timestamp / TimestampTz → i64 micros (secs * 10^6 + nanos / 1000); Uuid → high u64 LE then low u64 LE of the
 * big-endian bytes; String, and as Strings: Numeric (PgNumeric's Display), Json (serde_json's compact Display, the
 * ETL_ARROW_ALL_COLUMNS text), Time (NaiveTime's Display) and Bytes (lowercase hex) → LEB128 length + bytes; arrays →
 * LEB128 count + every element as Nullable.
 * Data issues do not fail the call; the first of each kind is reported (etl_dec_rowbinary_issues).  Every row before
 * the reported row of an issue is byte-exact; a row with an issue has consistent offsets but unspecified bytes.
 * Scratch, beside the output: 4 B per (row, column) + 4 B per row + 16 B per record of the batch, and with Json columns
 * 4 B per (row, Json column) + 8 B per such item + 17 B per input byte of Json text.  A row of 4 GiB or more is
 * ETL_ERR_INVALID_ARG; a Json value that does not parse again (the decode validated it) is ETL_ERR_INTERNAL. */
typedef struct etl_rb_issue {
  uint64_t row;      /* emitted row; UINT64_MAX = no such issue */
  uint32_t column;   /* column of the row (0 .. n_cols + 1) */
  uint32_t element;  /* array element, UINT32_MAX for a scalar */
} etl_rb_issue;
typedef struct etl_rowbinary_issues {
  etl_rb_issue date_range;       /* first Date outside 1900-01-01 ..= 2299-12-31 (ConversionError "Date out of ClickHouse
                                    Date32 range", encoding.rs:131-148), in (row, column, element) order */
  etl_rb_issue null_value;       /* first NULL in a column whose flag is clear (ConversionError "NULL value for
                                    non-nullable ClickHouse column", encoding.rs:204-212) */
  uint64_t first_partial_update; /* smallest batch-local record index of an Update with ETL_RF_NEW_PARTIAL (InvalidState
                                    "ClickHouse update requires a full new row image", core.rs:721-735); UINT64_MAX if none */
} etl_rowbinary_issues;
typedef struct etl_rowbinary_batch etl_rowbinary_batch;
int etl_dec_rowbinary_emit(const etl_dec_batch*, uint32_t schema_index, const uint8_t* nullable_flags, uint32_t n_flags,
                           int to_host, etl_rowbinary_batch** out);
uint64_t etl_dec_rowbinary_rows(const etl_rowbinary_batch*);
uint64_t etl_dec_rowbinary_bytes(const etl_rowbinary_batch*);
const uint8_t* etl_dec_rowbinary_data(const etl_rowbinary_batch*, int host);
const uint64_t* etl_dec_rowbinary_row_offsets(const etl_rowbinary_batch*, int host);   /* n_rows + 1 */
/* record index of each row (a COPY batch: the row index) */
const uint64_t* etl_dec_rowbinary_row_records(const etl_rowbinary_batch*, int host);
int etl_dec_rowbinary_issues(const etl_rowbinary_batch*, etl_rowbinary_issues* out);
void etl_dec_rowbinary_free(etl_rowbinary_batch*);

/* ---------------------------------------------------------------- ClickHouse compressed INSERT bodies
 * Rows [row_begin, row_end) of a RowBinary emit as the INSERT bodies the ClickHouse destination posts with
 * decompress=1, split and compressed on the device.  Replaces insert_rows's buffered chunks (client.rs:336-379) and
 * the clickhouse crate's LZ4 compression of each chunk into ClickHouse compressed blocks.
 * Split: insert_rows's greedy rule from row_begin: an INSERT takes rows while the bytes counted so far are below
 * max_bytes_per_insert, so the row that crosses the limit still goes into it, and the next INSERT starts after that
 * row.  insert_rows (n_inserts + 1 emit rows, [0] = row_begin, [n_inserts] = row_end): INSERT k is rows
 * [insert_rows[k], insert_rows[k+1]); its body is data[insert_offsets[k], insert_offsets[k+1]).  An empty range gives
 * zero INSERTs (one entry each).
 * Body: a sequence of ClickHouse compressed blocks whose decompressed bytes, concatenated, are the emit's
 * data[off[insert_rows[k]], off[insert_rows[k+1]]) (blocks may cut rows).  A block holds up to 16 KiB of those bytes
 * (the last of a body fewer) and is: 16 bytes of checksum, CityHash128 v1.0.2 of the 9 header bytes and the payload,
 * written as low64 then high64, each little-endian; the method byte 0x82 (LZ4); u32 LE compressed size (9 + payload);
 * u32 LE decompressed size; the payload, one LZ4 block: the last sequence is literals only, the last 5 bytes are
 * literals, no match starts within the last 12 bytes.  Deterministic: the same emit and arguments give the same bytes.
 * Not byte-identical to the clickhouse crate's own compression (lz4_flex, 256 KiB chunks); the server accepts any valid
 * LZ4 block up to 1 GiB.
 * ETL_ERR_INVALID_ARG: a NULL emit or out, max_bytes_per_insert 0 (the reference's loop never advances), row_begin >
 * row_end, row_end > n_rows.  Runs on the library's stream with three host syncs (the cuts, the output size, the end
 * of the call) and owns its output: the emit may be freed once the call returns.  Scratch, beside the output: 16 B per
 * INSERT, 16 B per block, and the compressed slots: 256/255 of the range's bytes + 56 B per block. */
typedef struct etl_rowbinary_lz4 etl_rowbinary_lz4;
int etl_dec_rowbinary_lz4(const etl_rowbinary_batch*, uint64_t row_begin, uint64_t row_end, uint64_t max_bytes_per_insert,
                          int to_host, etl_rowbinary_lz4** out);
uint64_t etl_dec_rowbinary_lz4_inserts(const etl_rowbinary_lz4*);
const uint64_t* etl_dec_rowbinary_lz4_insert_rows(const etl_rowbinary_lz4*, int host);      /* n_inserts + 1 emit rows */
const uint64_t* etl_dec_rowbinary_lz4_insert_offsets(const etl_rowbinary_lz4*, int host);   /* n_inserts + 1 byte offsets */
uint64_t etl_dec_rowbinary_lz4_bytes(const etl_rowbinary_lz4*);
const uint8_t* etl_dec_rowbinary_lz4_data(const etl_rowbinary_lz4*, int host);
void etl_dec_rowbinary_lz4_free(etl_rowbinary_lz4*);

/* ---------------------------------------------------------------- BigQuery Storage Write emitter
 * The rows of ONE replicated-schema version of a decoded batch as the serialized protobuf messages the BigQuery
 * destination puts into ProtoRows.serialized_rows, built on the device, plus n_rows + 1 u64 row offsets: row i is
 * data[off[i], off[i+1]), one message without a length prefix.  Replaces the per-row host walk of
 * crates/etl-destinations/src/bigquery: write_events (core.rs:792-970) with bigquery_update_rows /
 * bigquery_primary_key_changed (:1255-1403) and bigquery_delete_row (:1406-1524), write_table_rows (:530-546),
 * BigQueryTableRow::try_from_tagged_cells (encoding.rs:49-83) with validate_cell_for_bigquery (validation.rs) and the
 * prost serialisation (cell_encode_prost / array_cell_encode_prost, encoding.rs:151-342).
 * Fields (column_schemas_to_table_descriptor, client.rs:1292-1385): column c is field c + 1, _CHANGE_TYPE (String
 * "UPSERT" / "DELETE") field n_cols + 1, _CHANGE_SEQUENCE_NUMBER (String) field n_cols + 2, the 50 lowercase bytes
 * "{rec_commit_lsn:016x}/{rec_tx_ordinal:016x}/{ordinal:016x}" (bigquery_sequence_key, core.rs:1235).
 * Rows, in record order, come from the records of the version in the valid prefix that carry ETL_RF_EVENT:
 *   Insert → UPSERT of the new image, ordinal 0;
 *   Update → UPSERT of the new image, ordinal 0; when a primary-key cell changed, a DELETE of the old key (ordinal 0)
 *            comes first and the UPSERT has ordinal 1.  Changed: with a Full old image, any primary-key column whose
 *            old and new cells differ; with a key image, the key cells against the new image's primary-key cells in
 *            order; no old image: unchanged.  Cells compare as Cell's PartialEq: same variant, F32 / F64 by IEEE ==
 *            (a NaN key always changes, -0 equals +0), Numeric by sign, weight, scale and digits (1.0 != 1.00), Json by
 *            its canonical text (serde_json Value equality), arrays element by element;
 *   Delete → DELETE of the old key, ordinal 0.
 * A DELETE row holds only the primary-key columns (the stored TableSchema column has a primary_key_ordinal_position),
 * each under its own field, from the Full old image or from the key image taken in order.  No row, and the record
 * counts for first_invalid_record (InvalidState in write_events): an Update with ETL_RF_NEW_PARTIAL (core.rs:837-850),
 * a Delete with neither old image (:868-879), an Update or Delete with a key image when the version's identity columns
 * are not its primary-key columns (identity_matches_primary_key, :1347-1359, :1439-1451).
 * A COPY batch (rec_kind == NULL): every row of the valid prefix as an UPSERT without the sequence field (write_table_rows);
 * schema_index must be 0, and etl_dec_bigquery_row_records gives the row index.
 * Cells (prost; proto3's omission of default values does not apply, NULL writes nothing): the key is
 * varint(field << 3 | wire type).  Bool wt 0, one byte; I16 / I32 / I64 wt 0, varint of the value sign-extended to 64
 * bits; U32 wt 0, varint; F32 wt 5 / F64 wt 1, IEEE bits little-endian; Bytes wt 2, varint length + bytes; String, Uuid
 * (lowercase, hyphenated), Numeric (PgNumeric's Display), Json (serde_json's compact Display, the ETL_ARROW_ALL_COLUMNS
 * text), Date (%Y-%m-%d: years 0..=9999 as 4 digits, others with a sign and at least 4 digits), Time (%H:%M:%S%.f),
 * Timestamp (%Y-%m-%d %H:%M:%S%.f) and TimestampTz (the same + "+00:00") wt 2, varint length + UTF-8 text.  Arrays of
 * Bool / I16 / I32 / U32 / I64 / F32 / F64 are packed (one wt 2 key, the payload length, the values without keys);
 * arrays of any other kind write one wt 2 field per element; an empty array writes nothing.
 * Value issues (etl_bigquery_issues.value) do not fail the call: the first in (row, column) order over the emitted rows,
 * the key cells of DELETE rows and COPY rows included.  ARRAY_NULL: an array with a NULL element (the conversion to
 * CellNonOptional, checked first; element = the first NULL); NUMERIC_SCALE: a Numeric value, scalar or element, whose
 * Display has more than 38 fractional digits; JSON_INTEGER: a Json document, scalar or element, holding an integer
 * literal (no '.', 'e', 'E') outside i64 (starting with '-') or u64.  element is UINT32_MAX for a scalar.  Every row
 * before the reported row is byte-exact; the reported row has consistent offsets (a NULL element writes nothing).
 * to_host: also copy offsets, records and bytes to a pinned buffer (host = 1 accessors); else those return NULL.
 * Scratch, beside the output: 4 B per (row, field) + 12 B per row + 28 B per record of the batch, and with Json columns
 * 12 B per (record, Json column, image) + 17 B per input byte of Json text.  schema_index out of range, or non-zero
 * for a COPY batch, is ETL_ERR_INVALID_ARG; a row of 4 GiB or more is ETL_ERR_INVALID_ARG; a Json value that does not
 * parse again (the decode validated it) is ETL_ERR_INTERNAL. */
enum { ETL_BQ_ISSUE_ARRAY_NULL = 1, ETL_BQ_ISSUE_NUMERIC_SCALE = 2, ETL_BQ_ISSUE_JSON_INTEGER = 3 };
typedef struct etl_bq_issue {
  uint64_t row;      /* emitted row; UINT64_MAX = none */
  uint32_t column;   /* user column of the row (field column + 1) */
  uint32_t element;  /* array element, UINT32_MAX for a scalar */
  uint32_t kind;     /* ETL_BQ_ISSUE_* */
  uint32_t _pad;
} etl_bq_issue;
typedef struct etl_bigquery_issues {
  etl_bq_issue value;             /* first value issue in (row, column) order; row == UINT64_MAX: none */
  uint64_t first_invalid_record;  /* smallest batch-local record that write_events rejects with InvalidState; UINT64_MAX: none */
} etl_bigquery_issues;
typedef struct etl_bigquery_batch etl_bigquery_batch;
int etl_dec_bigquery_emit(const etl_dec_batch*, uint32_t schema_index, int to_host, etl_bigquery_batch** out);
uint64_t etl_dec_bigquery_rows(const etl_bigquery_batch*);
uint64_t etl_dec_bigquery_bytes(const etl_bigquery_batch*);
const uint8_t* etl_dec_bigquery_data(const etl_bigquery_batch*, int host);
const uint64_t* etl_dec_bigquery_row_offsets(const etl_bigquery_batch*, int host);  /* n_rows + 1 */
/* record index of each row (a COPY batch: the row index); both rows of a primary-key change carry the same record */
const uint64_t* etl_dec_bigquery_row_records(const etl_bigquery_batch*, int host);
int etl_dec_bigquery_issues(const etl_bigquery_batch*, etl_bigquery_issues* out);
void etl_dec_bigquery_free(etl_bigquery_batch*);

/* ---------------------------------------------------------------- DuckLake emitter
 * The row mutations of ONE replicated-schema version of a decoded batch, with the SQL-literal texts the DuckLake
 * destination builds for them, built on the device, and the fingerprints of its retry-safe batch identity.  Replaces
 * the host work of crates/etl-destinations/src/ducklake: write_events_inner (core.rs:715-836) with
 * validate_ducklake_replica_identity (:237-258) and key_row_from_updated_partial_row (:266-359);
 * cell_to_sql_literal_ref / table_row_to_sql_literal_ref (encoding.rs:28-272) behind delete_predicate_from_row
 * (batches.rs:1099-1186), update_assignments_from_partial_row (:1189-1269), delete_predicate_from_copy_row (:1338-1371)
 * and prepare_rows (encoding.rs:13-26); build_mutation_batch_identity / build_copy_batch_identity (batches.rs:1272-1336)
 * over the chunks of prepare_mutation_table_batches (:594-622) after retain_mutations_after_sequence_key (:806-820).
 * quoted_names: the version's n_cols column names exactly as pg_escape::quote_identifier prints them, copied verbatim
 * (any other n_names, or a NULL name, is ETL_ERR_INVALID_ARG).
 * Mutations, in record order, come from the records of the version in the valid prefix that carry ETL_RF_EVENT:
 *   Insert → INSERT (row: the new image);
 *   Update with an old image (Full or Key), Full new image → UPDATE (predicate: the old image; row: the new image);
 *   Update with an old image, ETL_RF_NEW_PARTIAL → UPDATE_PARTIAL (predicate: the old image; assignments);
 *   Update without an old image, Full new image → REPLACE (predicate: from the new row; row);
 *   Update without an old image, partial → UPDATE_PARTIAL (predicate: the identity cells of the partial row; assignments);
 *   Delete with an old image → DELETE (predicate).
 * No mutation, and the record counts for first_rejected_record with its reason: an Update / Delete when the version has
 * no identity columns (UPDATE_NO_IDENTITY / DELETE_NO_IDENTITY), a Delete without an old image (DELETE_NO_OLD_ROW), a
 * partial Update without an old image that lacks an identity column (PARTIAL_KEY_MISSING).  A partial Update without
 * any present column is still a mutation, reported in first_empty_partial_record (batches.rs:1207-1216 raises it when
 * the batch is prepared).  mixed_versions: a truncate-free run of the batch holds DML of this version's table under
 * another version; the reference then builds that table's run with the last version's schema (core.rs:737-740), so the
 * sub-batches here are not the reference's.
 * A COPY batch (rec_kind == NULL): schema_index must be 0, every row of the valid prefix is an INSERT, its predicate is
 * delete_predicate_from_copy_row: the stored TableSchema's primary-key columns (empty when there are none), and
 * etl_dec_ducklake_records gives the row index.
 * Texts (etl_dec_ducklake_text; which = ETL_DL_TEXT_*, n_mutations + 1 u64 offsets; a kind without the text has an
 * empty one):
 *   row: "(" values joined by ", " ")";
 *   predicate: the identity columns in schema order (a Full image's identity cells, a key image's cells in order),
 *              "name = lit" or "name IS NULL", joined by " AND ";
 *   assignments: the present columns ascending, "name = lit" (NULL: "name = NULL"), joined by ", ".
 * Literals: NULL; TRUE / FALSE; I16 / I32 / U32 / I64 in decimal; String quote_literal(text); Numeric
 * quote_literal(PgNumeric's Display); Uuid CAST('<lowercase hyphenated>' AS UUID); Json CAST(quote_literal(the
 * ETL_ARROW_ALL_COLUMNS text) AS JSON); Bytes from_hex('<UPPERCASE hex>'); Date DATE 'Y-m-d' (chrono's signed years);
 * Time TIME 'HH:MM:SS.ffffff' (always 6 digits, truncated; a leap second is second 60); Timestamp TIMESTAMP
 * 'Y-m-d HH:MM:SS.ffffff'; TimestampTz TIMESTAMPTZ '…ffffff+00:00'; F64 Rust's Display (the shortest round-trip
 * digits, positional, no ".0", "-0"), F32 the same of `f as f64`, NaN / ±Infinity CAST('NaN' | 'Infinity' |
 * '-Infinity' AS DOUBLE) (F32: AS FLOAT); arrays "[" elements joined by ", " "]", NULL for a NULL element.
 * quote_literal is pg_escape 0.1.1's (third-party, its source is not in the reference: parity unpinned): wrap in ',
 * double every ' and \, prefix E when the text holds a \.  Rust's shortest float digits are taken to be those of
 * Python's repr; no Rust toolchain checked that.
 * kinds: ETL_DL_* | ETL_DL_MF_ARRAY when the mutation's row image holds an array cell (prepare_rows then takes the row
 * texts as SqlLiterals instead of the appender).  The appender values are the ETL_ARROW_ALL_COLUMNS output of
 * etl_dec_arrow_emit with row_kinds = inserts | updates.
 * etl_dec_ducklake_sub_batches: with last_key = {commit_lsn, tx_ordinal}, the mutations whose (rec_commit_lsn,
 * rec_tx_ordinal) is greater (a suffix); within each truncate-free run (a Truncate event record of any table starts a
 * new one) they are cut into consecutive chunks of 16, and each chunk's fingerprint is FNV-1a 64 over what Rust's Hash
 * feeds BatchIdHasher: "mutation", the table name (a str is its bytes then 0xff), then per mutation start_lsn and
 * commit_lsn (u64, 8 bytes little-endian), the kind word ("insert", "delete", "update" for both UPDATE kinds, "replace")
 * and INSERT: row; DELETE: predicate; UPDATE / REPLACE: predicate, row; UPDATE_PARTIAL: predicate, n_cols (usize),
 * then per present column its index (usize) and its literal.  batch_id = "mutation:{first start_lsn:016x}:{last
 * commit_lsn:016x}:{fingerprint:016x}".  The result lives in the batch until the next call or etl_dec_ducklake_free;
 * ETL_ERR_INVALID_ARG for a COPY batch.
 * etl_dec_ducklake_copy_fingerprint: "copy", the table name, then per row its predicate and its row text — one serial
 * chain, computed on the host over the pinned copy: the batch must have been emitted with to_host (else, or for a
 * streaming batch, ETL_ERR_INVALID_ARG).
 * to_host: also copy records, kinds, text offsets and texts to a pinned buffer (host = 1 accessors); else those return
 * NULL (etl_dec_ducklake_text: ETL_ERR_INVALID_ARG).  Scratch, beside the output: 4 B per (text, mutation, column + 1)
 * + 4 B per mutation + 29 B per record of the batch, and with Json columns 12 B per (mutation, Json column, image) +
 * 17 B per input byte of Json text.  schema_index out of range, or non-zero for a COPY batch, is ETL_ERR_INVALID_ARG; a
 * single text of 4 GiB or more is ETL_ERR_INVALID_ARG; a Json value that does not parse again (the decode validated it)
 * is ETL_ERR_INTERNAL. */
enum { ETL_DL_INSERT = 1, ETL_DL_UPDATE = 2, ETL_DL_UPDATE_PARTIAL = 3, ETL_DL_REPLACE = 4, ETL_DL_DELETE = 5,
       ETL_DL_MF_ARRAY = 0x80 /* the mutation's row image holds a Cell::Array: prepare_rows takes SqlLiterals */ };
enum { ETL_DL_TEXT_ROW = 0, ETL_DL_TEXT_PREDICATE = 1, ETL_DL_TEXT_ASSIGNMENTS = 2 };
enum { ETL_DL_REJECT_UPDATE_NO_IDENTITY = 1, ETL_DL_REJECT_DELETE_NO_IDENTITY = 2, ETL_DL_REJECT_DELETE_NO_OLD_ROW = 3,
       ETL_DL_REJECT_PARTIAL_KEY_MISSING = 4 };
typedef struct etl_ducklake_issues {
  uint64_t first_rejected_record;      /* smallest batch-local record write_events_inner rejects; UINT64_MAX: none */
  uint32_t rejected_reason;            /* ETL_DL_REJECT_* of that record (0: none) */
  uint32_t mixed_versions;             /* non-zero: a truncate-free run holds this table's DML under another version */
  uint64_t first_empty_partial_record; /* partial update with no present column; UINT64_MAX: none */
} etl_ducklake_issues;
typedef struct etl_dl_sub_batch {
  uint64_t first_mutation;
  uint32_t n_mutations;
  uint32_t _pad;
  uint64_t fingerprint;
} etl_dl_sub_batch;
typedef struct etl_ducklake_batch etl_ducklake_batch;
int etl_dec_ducklake_emit(const etl_dec_batch*, uint32_t schema_index, const char* const* quoted_names, uint32_t n_names,
                          int to_host, etl_ducklake_batch** out);
uint64_t etl_dec_ducklake_mutations(const etl_ducklake_batch*);
const uint8_t* etl_dec_ducklake_kinds(const etl_ducklake_batch*, int host);    /* ETL_DL_* | ETL_DL_MF_ARRAY */
const uint64_t* etl_dec_ducklake_records(const etl_ducklake_batch*, int host); /* record (COPY: row) of each mutation */
int etl_dec_ducklake_text(const etl_ducklake_batch*, uint32_t which, int host,
                          const uint8_t** data, const uint64_t** offsets /* n_mutations + 1 */, uint64_t* bytes);
int etl_dec_ducklake_issues(const etl_ducklake_batch*, etl_ducklake_issues* out);
int etl_dec_ducklake_sub_batches(etl_ducklake_batch*, const uint8_t* table_name, uint32_t name_len,
                                 const uint64_t* last_key /* NULL, or {commit_lsn, tx_ordinal} */, int host,
                                 const etl_dl_sub_batch** out, uint64_t* n);
int etl_dec_ducklake_copy_fingerprint(const etl_ducklake_batch*, const uint8_t* table_name, uint32_t name_len, uint64_t* out);
void etl_dec_ducklake_free(etl_ducklake_batch*);

/* ---------------------------------------------------------------- Iceberg Parquet writer
 * Rows [row_begin, row_end) of an Arrow emit (etl_dec_arrow_emit with ETL_ARROW_ALL_COLUMNS, usually with
 * ETL_ARROW_CDC_COLUMNS) as one complete Parquet data file built on the device, plus the per-column metrics of the
 * Iceberg DataFile.  Replaces what iceberg-rust's ParquetWriter does on the host in IcebergClient::write_record_batch
 * (crates/etl-destinations/src/iceberg/client.rs:324-379, WriterProperties with Compression::SNAPPY): encode the values,
 * build the levels, compress the pages, compute the column statistics behind column_sizes, value_counts,
 * null_value_counts, nan_value_counts and lower_bounds / upper_bounds.  The shim keeps the control path: the table's
 * FileIO, the catalog transaction, file naming and the metrics mode (truncate(16) by default).
 * fields: one per emitted column, in order (n_fields == etl_dec_arrow_cols).  ETL_ERR_INVALID_ARG, before any launch:
 * another n_fields or none (an emit of a zero-column table without ETL_ARROW_CDC_COLUMNS), an ETL_ARROW_UNSUPPORTED
 * column (the emit lacked ETL_ARROW_ALL_COLUMNS), row_begin > row_end or row_end > etl_dec_arrow_rows, an unknown
 * codec (codec & 0xFF other than ETL_PQ_UNCOMPRESSED / ETL_PQ_SNAPPY / ETL_PQ_ZSTD) or a codec bit other than ETL_PQ_DICTIONARY and
 * ETL_PQ_PAGE_INDEX, a NULL or empty name or one longer than 1 KiB; with bloom, an fpp that is NaN, negative or >= 1,
 * a max_bytes that is neither 0 nor a power of two in [32, 2^27], or fpp > 0 on a Boolean leaf (Arrow C++ has no
 * filters for BOOLEAN either).
 * A null in a required column (a null list of a required List column, or a null value) is data: ETL_OK with size 0 and
 * no bytes, and etl_dec_parquet_required_null gives the smallest such column and its first null row (emit row numbers)
 * — RecordBatch::try_new in rows_to_record_batch fails there before anything is written (a ConversionError in the shim).
 * The file (parity with arrow-rs bytes and defaults is not a goal: its writer adds an ARROW:schema key and page
 * statistics; Iceberg readers resolve columns by field id and Parquet type):
 *   layout: "PAR1", the column chunks (row-group major, column minor, pages in row order), the footer, its 4-byte LE
 *           length, "PAR1".  Row groups of at most 1 048 576 rows in row order; zero rows: no row group.
 *   pages: data page V1, no CRC, no page statistics; whole rows; a page ends after the first row that
 *          brings it to 20 000 rows or to >= 1 MiB of PLAIN value bytes (Boolean: ceil(values / 8)), and at the row
 *          group's end.
 *   values: PLAIN, non-null only: Boolean bit-packed LSB first, INT32 / INT64 / FLOAT / DOUBLE little-endian,
 *           BYTE_ARRAY 4-byte LE length + bytes, FIXED_LEN_BYTE_ARRAY(16) raw.
 *   levels: only when the max level > 0, each section with a 4-byte LE length, repetition before definition; RLE /
 *           bit-packed hybrid of bit width = bits of the max level, runs cut deterministically: entries in groups of 8,
 *           a group is uniform when its (present) entries are equal; consecutive uniform groups of one value are one
 *           RLE run of their exact entry count; each maximal stretch of other groups is bit-packed runs of at most 63
 *           groups, the last group zero-padded.
 *   types: Bool BOOLEAN, Int32 INT32, Int64 INT64, Float32 FLOAT, Float64 DOUBLE, Utf8 BYTE_ARRAY STRING (UTF8),
 *          LargeBinary BYTE_ARRAY, Date32 INT32 DATE (DATE), Time64 µs INT64 TIME(MICROS, utc=false), Timestamp µs
 *          INT64 TIMESTAMP(MICROS, utc=false), Timestamptz µs INT64 TIMESTAMP(MICROS, utc=true) (TIMESTAMP_MICROS),
 *          Uuid FIXED_LEN_BYTE_ARRAY(16) UUID.  Every element carries its field id.
 *   lists: <rep> group name (LIST) { repeated group list { optional <leaf> element } }, field_id on the outer group,
 *          element_field_id on element (always optional: NestedField::list_element(…, false), iceberg/schema.rs:67-75);
 *          max definition level 3 (optional list) or 2 (required), max repetition level 1.
 *   codec: ETL_PQ_SNAPPY compresses each page's levels + values as one Snappy stream: the varint length, then the
 *          elements of independent 64 KiB fragments (no copy crosses a fragment).  Page headers are not compressed.
 *          ETL_PQ_ZSTD (Parquet's ZSTD) compresses each page's levels + values, and each dictionary page's entries, as
 *          one Zstandard frame (RFC 8878).  Frame header, 9 bytes: the magic 28 B5 2F FD, Frame_Header_Descriptor 0xA0
 *          (Single_Segment, a 4-byte Frame_Content_Size, no checksum, no dictionary id), then the Frame_Content_Size =
 *          the uncompressed page size (LE).  Blocks: exactly one per 64 KiB fragment of the payload, Last_Block set on
 *          the last one only; an empty payload is one empty last Raw block.  Every block is self-contained: no match
 *          reaches before its fragment's start, no offset is a repeat-offset code, Huffman literals always carry their
 *          own table (never Treeless), sequence modes are Predefined, RLE or FSE_Compressed (never Repeat).  A
 *          Compressed block is used only when strictly smaller than its fragment; otherwise the block is RLE when all its
 *          bytes are equal, else Raw.  The encoder has one fixed strategy (no level).  uncompressed_page_size is
 *          unchanged; compressed_page_size is the frame's length.
 *   statistics: per column chunk null_count, max_value, min_value in the type's order (signed ints / dates / times,
 *          unsigned bytewise BYTE_ARRAY / UUID, false < true), NaN excluded, a zero minimum written as -0.0 and a zero
 *          maximum as +0.0; none when the chunk has no non-NaN value or a byte-array min / max is longer than 64 bytes.
 *          column_orders: TypeDefinedOrder for every leaf.
 *   dictionary (codec | ETL_PQ_DICTIONARY; without it every chunk is PLAIN as above):
 *          eligible leaves: every leaf but Boolean (a List column's leaf is its element); each column chunk (one leaf in
 *          one row group) has its own dictionary.  Entries: the distinct PLAIN byte strings of the chunk's non-null
 *          values (fixed width: the little-endian value; Uuid: the 16 bytes; byte arrays: the bytes), floats compared
 *          bitwise (+0.0 and -0.0 are two entries, NaNs with equal bits one), in order of first occurrence in item order
 *          (the order of arrow-rs's interner), independent of thread scheduling.  Decision per chunk: its dictionary size
 *          is the sum of the entries' PLAIN sizes (byte arrays 4 + length); the chunk is dictionary-encoded iff it has a
 *          non-null value and that size is <= 1 048 576 bytes, else it is written PLAIN, byte for byte as without the
 *          flag, wherever it lands (a whole-chunk decision: arrow-rs falls back in the middle of a chunk instead).  A
 *          file in which no chunk qualifies is the file written without the flag.
 *          Dictionary page, first in the chunk: PageHeader {type DICTIONARY_PAGE (2), uncompressed / compressed size,
 *          dictionary_page_header (7) {num_values = entries, encoding PLAIN}}; payload the entries PLAIN in dictionary
 *          order, compressed as a data page is.  Data pages: the page cuts above, still on PLAIN bytes (arrow-rs cuts on
 *          encoded size); header encoding RLE_DICTIONARY (8); payload the level sections as above, one byte of bit width
 *          max(1, bits(entries - 1)) (<= 18: 1 MiB / 4-byte entries bounds entries by 262 144), then the RLE / bit-packed
 *          hybrid of the page's non-null indices without a length prefix, under the run rule of the levels (groups of 8,
 *          uniform groups of one value one RLE run of their exact count with the value in ceil(width / 8) LE bytes,
 *          other stretches bit-packed runs of at most 63 groups, LSB first, the last group zero-padded); a page without a
 *          non-null value has only the bit-width byte.
 *          Footer of a dictionary chunk: encodings [PLAIN, RLE (with levels), RLE_DICTIONARY], data_page_offset the first
 *          data page, dictionary_page_offset (11) and ColumnChunk / RowGroup file_offset the dictionary page,
 *          encoding_stats (13) [{DICTIONARY_PAGE, PLAIN, 1}, {DATA_PAGE, RLE_DICTIONARY, data pages}].  Statistics and
 *          the metrics' counts and bounds are those of the values, as without the flag.  ColumnMetaData.codec is
 *          codec & 0xFF.
 *   page index (codec | ETL_PQ_PAGE_INDEX; without it no chunk has one, and bytes [0, 4 + data end) of a file with it
 *          are the file written without it, the same codec and dictionary bit): the ColumnIndex and OffsetIndex arrow-rs
 *          writes by default, for page pruning by readers.
 *          Layout: after the last column chunk the ColumnIndex of every chunk that has one, row-group major and column
 *          minor, then the OffsetIndex of every chunk in the same order, then the footer.  Zero rows: no row group, no
 *          index.  ColumnChunk adds offset_index_offset (4, i64), offset_index_length (5, i32) and, with a ColumnIndex,
 *          column_index_offset (6, i64), column_index_length (7, i32), after meta_data; offsets are file offsets.
 *          OffsetIndex {1 page_locations: list<PageLocation>}: one per data page (not the dictionary page, so the first
 *          is data_page_offset): {1 offset: i64 of the page header, 2 compressed_page_size: i32 of the page's file bytes
 *          (header and Snappy preamble included), 3 first_row_index: i64, the page's first row relative to its row
 *          group (rows, not level entries)}.
 *          ColumnIndex {1 null_pages: list<bool> (element type 1, one byte per element: 0x01 true, 0x02 false), 2
 *          min_values, 3 max_values: list<binary>, 4 boundary_order: i32, 5 null_counts: list<i64>}, one entry per data
 *          page.  A null page has no non-null value; its bounds are empty.  Bounds: the PLAIN statistic bytes of the
 *          page's min / max under the statistics' rules (type order, NaN excluded, a zero minimum -0.0 and a zero maximum
 *          +0.0), byte arrays longer than 64 bytes truncated (arrow-rs's column_index_truncate_length; the chunk
 *          statistics keep their rule): Utf8 min the longest prefix of at most 64 bytes ending on a character boundary;
 *          Utf8 max the prefix up to the last character boundary at most 64, cut after its last character whose code
 *          point + 1 is a Unicode scalar value of the same UTF-8 length, that character incremented (none: the whole
 *          value; U+D7FF, U+FFFF, U+10FFFF and U+007F / U+07FF cannot be incremented); LargeBinary min the first 64
 *          bytes; LargeBinary max the first 64 bytes with the last one incremented, 0xFF carrying as 0x00 into the
 *          byte before (all 0xFF: the whole value).  boundary_order compares each non-null page with the previous one on
 *          the untruncated bounds: ASCENDING (1) unless a min or max is below the previous page's, else DESCENDING (2)
 *          unless one is above, else UNORDERED (0) (one page, a constant chunk or an all-null chunk: ASCENDING).
 *          null_counts: level entries minus non-null values of each page.  A chunk with a page whose non-null values
 *          are all NaN (no bounds) has no ColumnIndex, only its OffsetIndex.  Not written: level histograms and
 *          SizeStatistics, page-header statistics.  The metrics' compressed_bytes stay the chunks' page bytes (Iceberg's
 *          column_sizes); etl_dec_parquet_size counts the whole file.
 *   bloom filters (etl_dec_parquet_write_bloom, a column with fpp > 0; without one no chunk has a filter, and bytes
 *          [0, 4 + data end) of a file with filters are the file written without them, the same codec and flags): the
 *          split-block filters Arrow C++ writes (pyarrow's bloom_filter_options), for readers that skip row groups on
 *          equality predicates; readers that ignore filters read the file as before.
 *          Which chunks: every chunk (one leaf in one row group) of such a column, an all-null chunk too (its bitset all
 *          zero); a List column's leaf is its element, its filter holds the non-null elements.  Zero rows: no filter.
 *          Size: ndv = the field's ndv, or the chunk's non-null values when 0 (at least 1); bits = -8 ndv / ln(1 -
 *          fpp^(1/8)) in double, truncated, clamped to [256, 2^30], rounded up to a power of two; bytes = bits / 8, then
 *          min(bytes, max_bytes).
 *          Hash: XXH64, seed 0, of the value's PLAIN bytes without a length prefix: INT32 / INT64 / FLOAT / DOUBLE the
 *          little-endian value (floats by their bits: +0.0 and -0.0 differ, a NaN hashes as its bits), BYTE_ARRAY the
 *          bytes, UUID the 16 bytes.  Insert: blocks = bytes / 32, block ((h >> 32) × blocks) >> 32, key (uint32)h; word
 *          8 × block + i (i < 8) gets bit (uint32)(key × SALT[i]) >> 27, SALT = {0x47b6137b, 0x44974d91, 0x8824ad5b,
 *          0xa2b7289d, 0x705495c7, 0x2df1424b, 0x9efc4947, 0x5c6bfb31}; the bitset is those u32 words little-endian.
 *          Each filter: Thrift compact BloomFilterHeader {1 numBytes: i32, 2 algorithm {1 BLOCK {}}, 3 hash {1 XXHASH
 *          {}}, 4 compression {1 UNCOMPRESSED {}}} (15 bytes for 32 B of bitset, 16 for 128, 17 for 8192), then the bitset.
 *          Layout: after the last column chunk every filter, row-group major and column minor; then the page index
 *          (the same structs, behind the filters); then the footer.  ColumnMetaData adds bloom_filter_offset (14, i64,
 *          the header's file offset) and bloom_filter_length (15, i32, header + bitset) after encoding_stats.  The
 *          metrics are those of the file without filters (compressed_bytes: the chunk's pages); etl_dec_parquet_size
 *          counts the filters.
 *   footer: Thrift compact, ascending field ids: FileMetaData {version 1, schema, num_rows, row_groups, created_by,
 *          column_orders}, SchemaElement {type, type_length, repetition_type, name, num_children, converted_type,
 *          field_id, logicalType}, RowGroup {columns, total_byte_size, num_rows, file_offset, total_compressed_size,
 *          ordinal}, ColumnChunk {file_offset, meta_data[, page index fields]}, ColumnMetaData {type, encodings (PLAIN, + RLE with levels),
 *          path_in_schema, codec, num_values, total_uncompressed_size, total_compressed_size, data_page_offset,
 *          [dictionary_page_offset,] statistics[, encoding_stats][, bloom_filter_offset, bloom_filter_length]}.
 * Metrics: one record per leaf (a List column's leaf is its element), over every row group of the file; min / max are
 * the PLAIN statistic bytes, which equal Iceberg's single-value serialization of these types (before truncation).
 * to_host: also copy the file to pinned host memory (etl_dec_parquet_bytes(f, 1); else NULL).  Scratch, beside the
 * file: 36 B per (row, column), 2 B per level entry + 64 B per page, 1 bit per Boolean value, a payload slot per page (values +
 * level bound) and with Snappy a compressed slot per 64 KiB of payload (with ETL_PQ_ZSTD a slot of 64 KiB + 3 B, and 3 B
 * of literal / sequence scratch per payload byte + 8 B per fragment); with ETL_PQ_DICTIONARY also 28 B per item of an
 * eligible leaf (bounded by its level entries) + 0.5 B per item of run heads, a dictionary slot per chunk of at most
 * 1 MiB, 32 B per data page, and hash tables of at most 16 B per non-null value; with ETL_PQ_PAGE_INDEX 40 B per chunk
 * and, in the file's buffer, 189 B per page + 64 B per chunk (+ the longest row per page of a byte-array leaf with a
 * value over 64 bytes, at most its value bytes); with bloom filters 8 B per chunk, 24 B per chunk record and each
 * filtered chunk's bitset in scratch, and in the file's buffer its bitset + header (at most 19 B). */
enum { ETL_PQ_UNCOMPRESSED = 0, ETL_PQ_SNAPPY = 1, ETL_PQ_ZSTD = 6 };   /* Parquet's CompressionCodec values */
#define ETL_PQ_DICTIONARY 0x100u   /* OR-ed into codec: dictionary-encode the eligible column chunks (codec & 0xFF: compression) */
#define ETL_PQ_PAGE_INDEX 0x400u   /* OR-ed into codec: write a ColumnIndex and an OffsetIndex per column chunk */
#define ETL_PQ_HAS_MIN_MAX 1u   /* etl_parquet_metrics.flags: min / max are set */
typedef struct etl_parquet_field {
  const char* name;           /* UTF-8 column name, written verbatim into the Parquet schema */
  int32_t field_id;           /* Iceberg field id of the column */
  int32_t element_field_id;   /* ETL_ARROW_LIST columns: Iceberg field id of the list element; ignored otherwise */
  uint32_t required;          /* 1: REQUIRED (ColumnSchema nullable == false; both CDC columns), 0: OPTIONAL */
  uint32_t _pad;
} etl_parquet_field;
typedef struct etl_parquet_metrics {   /* one per leaf (= per column; a List column's leaf is its element) */
  int32_t field_id;           /* the leaf's id: field_id, or element_field_id for a List */
  uint32_t flags;             /* ETL_PQ_HAS_MIN_MAX */
  uint64_t num_values;        /* level entries (Parquet num_values), summed over row groups */
  uint64_t null_count;        /* entries whose definition level < max */
  uint64_t nan_count;         /* Float / Double leaves only */
  uint64_t compressed_bytes;  /* column-chunk bytes including page headers (and dictionary pages), summed over row groups */
  uint64_t uncompressed_bytes;
  const uint8_t* min; uint32_t min_len;   /* host memory, PLAIN-encoded statistic bytes, valid until free */
  const uint8_t* max; uint32_t max_len;
} etl_parquet_metrics;
typedef struct etl_parquet_file etl_parquet_file;
typedef struct etl_parquet_bloom {   /* one per emitted column, parallel to fields */
  double fpp;                 /* false-positive probability, 0 < fpp < 1; exactly 0: no filter for this column */
  uint64_t ndv;               /* expected distinct values per column chunk; 0: the chunk's non-null values (at least 1) */
  uint32_t max_bytes;         /* cap on one bitset: a power of two in [32, 128 MiB]; 0: 1 MiB */
  uint32_t _pad;
} etl_parquet_bloom;
int etl_dec_parquet_write(const etl_arrow_batch*, const etl_parquet_field* fields, uint32_t n_fields,
                          uint64_t row_begin, uint64_t row_end, uint32_t codec, int to_host, etl_parquet_file** out);
/* the same file with a split-block bloom filter on every column chunk of a column whose bloom[c].fpp > 0 (bloom NULL,
 * or every fpp 0: the file etl_dec_parquet_write writes) */
int etl_dec_parquet_write_bloom(const etl_arrow_batch*, const etl_parquet_field* fields, const etl_parquet_bloom* bloom,
                                uint32_t n_fields, uint64_t row_begin, uint64_t row_end, uint32_t codec, int to_host,
                                etl_parquet_file** out);
uint64_t etl_dec_parquet_size(const etl_parquet_file*);
const uint8_t* etl_dec_parquet_bytes(const etl_parquet_file*, int host);   /* the whole file, "PAR1" … "PAR1" */
int etl_dec_parquet_metrics(const etl_parquet_file*, uint32_t leaf, etl_parquet_metrics* out);
/* arrow-rs rejects a RecordBatch with a null in a non-nullable field: the smallest such column and its first null row
 * (UINT32_MAX / UINT64_MAX when there is none); no file */
int etl_dec_parquet_required_null(const etl_parquet_file*, uint32_t* column, uint64_t* row);
void etl_dec_parquet_free(etl_parquet_file*);

/* ---------------------------------------------------------------- Parquet: many files in one call
 * Every file of a partitioned write (or of a batch cut into files) in one device call: one plan, one set of allocations
 * and at most three host syncs (the plan; the sizes, offsets and metrics; with to_host the pinned copy), whatever
 * n_files is.  No per-file launch, copy or allocation.
 * Byte identity: file k is exactly the bytes etl_dec_parquet_write_bloom(a, fields, bloom, n_fields, row_offsets[k],
 * row_offsets[k + 1], codec, to_host) writes, and its metrics per leaf are that call's.  So row groups of at most
 * 1 048 576 rows restart in every file; RowGroup.ordinal, file_offset and every offset in the footer, page index and
 * bloom filters are relative to the file; each column chunk of each file has its own dictionary, statistics, page cuts
 * and bloom bitset (ndv 0: that chunk's own non-null count).
 * row_offsets: host memory, n_files + 1 non-decreasing emit rows, row_offsets[n_files] <= etl_dec_arrow_rows;
 * row_offsets[0] may be above 0.  An empty range is the zero-row file the single call writes for it.  n_files == 0 is
 * ETL_OK with no files (one offset, 0), so a partition result of zero rows can be passed as it is:
 * etl_dec_parquet_write_files(etl_dec_iceberg_partitioned_arrow(p), …, etl_dec_iceberg_partition_rows(p, 1),
 * etl_dec_iceberg_partitions(p), …).
 * Result: etl_dec_parquet_files_offsets gives n_files + 1 byte offsets (host memory); file k is bytes [offs[k],
 * offs[k + 1]) of etl_dec_parquet_files_bytes(fs, host) (host = 1: the pinned image, NULL without to_host; 0: device
 * memory), packed in order with no gaps.  etl_dec_parquet_files_metrics gives file k's record of a leaf.
 * Required nulls: a null in a required column anywhere in [row_offsets[0], row_offsets[n_files]) writes no file (every
 * offset 0, no bytes, no metrics: ETL_ERR_INVALID_ARG from _metrics) and etl_dec_parquet_files_required_null reports
 * what the single call over that whole range reports (RecordBatch::try_new fails for the whole batch before any file
 * is written); a null outside the range does not count.
 * ETL_ERR_INVALID_ARG, before any launch: everything the single call rejects, a NULL row_offsets or out, n_files >=
 * 2^32 - 1, decreasing offsets, a last offset past the emit, 2^31 column chunks or more in all (the sum over files of
 * ceil(rows / 1 048 576) times n_fields: chunk indices and the page index's length scan are 32-bit); in the accessors
 * an out-of-range file or leaf.  A CUDA failure is ETL_ERR_CUDA and leaks nothing.
 * Scratch: that of one single call over [row_offsets[0], row_offsets[n_files]) whose row groups are the files', plus
 * the terms that grow with the files.  Every file has at least one page per leaf (and with ETL_PQ_DICTIONARY a
 * dictionary slot per non-Boolean leaf), and each page costs about 0.4 KiB of scratch: its 216 B record, 32 B of slot
 * scans, 64 B of level scratch and, compressed, 8 B plus 32 B per 64 KiB fragment beyond its payload's 7/6 (its
 * compressed slot is sized by its own payload); and in the output buffer 48 B of header room (+ 189 B with
 * ETL_PQ_PAGE_INDEX).  Per file: a 72 B record, 8 B of size / offset, its footer's bound (the schema prefix + about
 * 0.3 KiB per column chunk) in the output buffer, and one metrics record per leaf (248 B on the device, its copy on
 * the host); per row group 12 B of table; once the schema prefix, leaf names and created_by.  The output buffer is
 * kept by the result until etl_dec_parquet_files_free. */
typedef struct etl_parquet_files etl_parquet_files;
int etl_dec_parquet_write_files(const etl_arrow_batch*, const etl_parquet_field* fields, const etl_parquet_bloom* bloom /* NULL: no filters */,
                                uint32_t n_fields, const uint64_t* row_offsets /* host, n_files + 1 */, uint64_t n_files,
                                uint32_t codec, int to_host, etl_parquet_files** out);
uint64_t etl_dec_parquet_files_count(const etl_parquet_files*);
const uint64_t* etl_dec_parquet_files_offsets(const etl_parquet_files*);        /* host, n_files + 1 byte offsets */
const uint8_t* etl_dec_parquet_files_bytes(const etl_parquet_files*, int host);  /* every file, back to back */
int etl_dec_parquet_files_metrics(const etl_parquet_files*, uint64_t file, uint32_t leaf, etl_parquet_metrics* out);
int etl_dec_parquet_files_required_null(const etl_parquet_files*, uint32_t* column, uint64_t* row);
void etl_dec_parquet_files_free(etl_parquet_files*);

/* ---------------------------------------------------------------- Iceberg partitioning
 * Rows [row_begin, row_end) of an Arrow emit grouped by the partition tuple of an Iceberg partition spec, on the device:
 * a permuted copy of the emit in which every partition is one contiguous row range, so that each partition's data file
 * is one etl_dec_parquet_write(_bloom) call over that range.  The reference writes unpartitioned tables only
 * (iceberg/client.rs:355-356 builds every DataFile with no partition key); this is what a partitioned table needs.
 * spec: n_fields (1 .. 16) partition fields, each a source column of the emit (table columns and both CDC columns), an
 * ETL_ICE_* transform and its parameter (bucket: N, truncate: W, both in 1 .. INT32_MAX; 0 for every other transform).
 * Transforms (Iceberg spec "Partition Transforms"; the source types are the emit's):
 *   identity     Boolean, Int32, Int64, Date32, Time64, Timestamp(tz), Utf8, LargeBinary, UUID: the value itself
 *   bucket[N]    Int32, Int64, Date32, Time64, Timestamp(tz), Utf8, LargeBinary, UUID: (murmur3_x86_32(bytes, seed 0) &
 *                INT32_MAX) % N, where bytes are (Appendix B) the value widened to a little-endian int64 for the integer
 *                types (days for Date32, micros for Time64 and timestamps), the UTF-8 bytes of Utf8, the bytes of
 *                LargeBinary and the 16 bytes of a UUID in RFC 4122 order (the order FixedSizeBinary(16) holds)
 *   truncate[W]  Int32, Int64: v - (((v % W) + W) % W) in the source's width, wrapping like two's-complement Java / Rust
 *                (truncate[10] of INT32_MIN is 2147483646); Utf8: the first W code points; LargeBinary: the first W bytes
 *   year, month  Date32, Timestamp(tz): year(d) - 1970 and (year(d) - 1970) * 12 + month(d) - 1 of the proleptic
 *                Gregorian date (iceberg-rust's and PyIceberg's formulas: 1969-12-31 is year -1 and month -1)
 *   day          Date32: the day count; Timestamp(tz): floor(micros / 86 400 000 000)
 *   hour         Timestamp(tz): floor(micros / 3 600 000 000)
 *   void         any column that is neither a List nor ETL_ARROW_UNSUPPORTED: always null
 * A Timestamptz is in UTC; a naive Timestamp is taken on its stored micros.  A null source gives a null result.  Float
 * sources are rejected for every transform but void (engines disagree on -0.0 / 0.0 and on NaN grouping).
 * Grouping: two rows share a partition when every field's null flag and result are equal (integers by value, bytes by
 * content).  Partitions come in the order of their first row; inside a partition rows keep emit order, so
 * sequence_number stays ascending inside every file.  The order depends on the input alone, not on scheduling.
 * Result:
 *   etl_dec_iceberg_partitions             P, the number of partitions (0 for zero rows);
 *   etl_dec_iceberg_partition_rows         P + 1 row offsets: partition k is rows [rows[k], rows[k + 1]) of the
 *                                          partitioned emit (host = 1: host memory, 0: device memory);
 *   etl_dec_iceberg_partition_value        partition k's result of field f: is_null, value (every integer result,
 *                                          sign-extended; Boolean 0 / 1) or len / data (Utf8, LargeBinary and UUID
 *                                          results; data in host memory owned by the result);
 *   etl_dec_iceberg_partitioned_arrow      the partitioned emit: row_end - row_begin rows, the source's columns, types,
 *                                          List children and CDC columns with the rows permuted; its
 *                                          etl_dec_arrow_row_records permuted the same way and its
 *                                          etl_dec_arrow_first_skipped the source's.  A genuine etl_arrow_batch for
 *                                          etl_dec_arrow_column / _list_child / etl_dec_parquet_write(_bloom), owned by
 *                                          the result (never etl_dec_arrow_free it); with to_host it has a host image.
 * The result owns everything it returns: the source emit may be freed right after the call.
 * ETL_ERR_INVALID_ARG, before any launch: a NULL emit, spec or out; n_fields 0 (an unpartitioned table writes the emit
 * directly) or above 16; a source column out of range, a List or ETL_ARROW_UNSUPPORTED column; a transform / type pair
 * not in the table (a float source included); an unknown transform; N or W of 0 or above INT32_MAX, or a non-zero param
 * on another transform; row_begin > row_end or row_end > etl_dec_arrow_rows; 2^32 rows or more.  A CUDA failure is
 * ETL_ERR_CUDA and leaks nothing.
 * Work: one thread per row computes every field's result and a tuple hash; a device hash table keyed by the tuple (full
 * compare on a hash match, atomicMin of the first row) finds the partitions; a scan of the first-row flags ranks them; a
 * stable radix sort of (rank, row) gives the permutation; every column, List children included, is gathered through it
 * (bits by ballot, fixed-width values, offsets from the permuted lengths, bytes a warp per row).  Host syncs: one for the
 * partition count and the representative values' sizes, then the final one.  Scratch: 13 B per (row, field), 12 B per
 * (row, field with a byte-valued result), 64–84 B per row (the hash table, ranks, the sort's keys, rows and temporary
 * storage), 4 B per row of each variable-width column and 4 B per element of each List; the output is the size of the
 * source rows it holds. */
enum { ETL_ICE_IDENTITY = 0, ETL_ICE_BUCKET = 1, ETL_ICE_TRUNCATE = 2, ETL_ICE_YEAR = 3, ETL_ICE_MONTH = 4, ETL_ICE_DAY = 5,
       ETL_ICE_HOUR = 6, ETL_ICE_VOID = 7 };
#define ETL_ICE_MAX_FIELDS 16u
typedef struct etl_iceberg_partition_field {
  uint32_t source_column;   /* column of the emit (table columns and CDC columns; not a List) */
  uint32_t transform;       /* ETL_ICE_* */
  uint32_t param;           /* bucket: N, truncate: W (1 .. INT32_MAX); 0 for every other transform */
  uint32_t _pad;
} etl_iceberg_partition_field;
typedef struct etl_iceberg_partition_value {
  uint32_t is_null, len;    /* len: bytes at data (Utf8 / LargeBinary / UUID results), else 0 */
  int64_t value;            /* every integer-valued result, sign-extended; Boolean 0 / 1 */
  const uint8_t* data;      /* host memory owned by the result, valid until free; NULL for integer results */
} etl_iceberg_partition_value;
typedef struct etl_iceberg_partitioned etl_iceberg_partitioned;
int etl_dec_iceberg_partition(const etl_arrow_batch*, const etl_iceberg_partition_field* spec, uint32_t n_fields,
                              uint64_t row_begin, uint64_t row_end, int to_host, etl_iceberg_partitioned** out);
uint64_t etl_dec_iceberg_partitions(const etl_iceberg_partitioned*);
const uint64_t* etl_dec_iceberg_partition_rows(const etl_iceberg_partitioned*, int host);   /* P + 1 entries */
int etl_dec_iceberg_partition_value(const etl_iceberg_partitioned*, uint64_t partition, uint32_t field,
                                    etl_iceberg_partition_value* out);
const etl_arrow_batch* etl_dec_iceberg_partitioned_arrow(const etl_iceberg_partitioned*);
void etl_dec_iceberg_partition_free(etl_iceberg_partitioned*);

/* device address of the staged stream a batch was decoded from (string / json cells are offsets into it); valid until
 * the next decode on the same context (library-owned copy) or as long as the caller's dev_buf lives */
const uint8_t* etl_dec_batch_device_stream(const etl_dec_batch*);

/* ---------------------------------------------------------------- shim stand-in (host only, no GPU work)
 * What the Rust shim does with the planes (INTEGRATION.md §3; replaces nothing in the reference — it is the glue that
 * rebuilds the reference's own types): materialise the AoS Vec<Event> handed to add_event_to_batch (apply.rs:433-439)
 * — one owned copy per String / Bytes / Numeric, a serde_json-style tree per Json cell, ArrayCells — and compute
 * Event::size_hint (types/event.rs:288-312, types/table_row.rs:250-345) per event.  C++ here because the image has no
 * Rust toolchain; the Rust struct sizes are parameters (pass std::mem::size_of values; NULL = x86-64 estimates). */
typedef struct etl_rust_layout {
  uint32_t size_of_cell, size_of_table_row, size_of_partial_table_row;
  uint32_t size_of_begin_event, size_of_commit_event, size_of_insert_event, size_of_update_event, size_of_delete_event,
           size_of_truncate_event, size_of_replicated_table_schema, size_of_relation_event;
  uint32_t size_of_json_value, size_of_usize;
} etl_rust_layout;
typedef struct etl_event_list etl_event_list;
/* batch must have been decoded with ETL_DECODE_RESULTS_TO_HOST; host_stream = the staged bytes (string / json spans) */
int etl_shim_materialise(const etl_dec_batch*, const uint8_t* host_stream, const etl_rust_layout*, etl_event_list** out);
uint64_t etl_shim_event_count(const etl_event_list*);
uint64_t etl_shim_size_hint(const etl_event_list*, uint64_t event_index);  /* Event::size_hint */
uint64_t etl_shim_total_size_hint(const etl_event_list*);                  /* what events_batch_bytes would hold */
uint64_t etl_shim_owned_bytes(const etl_event_list*);                      /* bytes copied into owned buffers */
/* serde_json::to_string of the Json cell at `new_row_cell` of an insert/update event (tests); returns its length */
int64_t etl_shim_json_text(const etl_event_list*, uint64_t event_index, uint32_t new_row_cell, char* buf, uint64_t cap);
void etl_shim_event_list_free(etl_event_list*);

#ifdef __cplusplus
}
#endif
#endif /* ETL_DECODE_H */
