/*
 * oracle_stream.c — CPU restatement of the streaming hot path driver.  TEST INFRASTRUCTURE ONLY.
 *
 *   frame / message parse : third-party postgres-replication 0.6.7 (git rev 31acf55, Cargo.lock:4486-4498),
 *                           not part of the reference tree → follows the PostgreSQL protocol docs
 *                           ("Logical Replication Message Formats", proto v1) and the bytes the
 *                           reference's own tests hand-encode (event.rs:1068-1146). parity unpinned
 *                           for Begin/Commit/Relation/Insert/Truncate/Message/XLogData header.
 *   state machine          : crates/etl/src/replication/apply.rs:600-626, 1687-2248
 *   relation → masks       : conversions/event.rs:325-369, etl-postgres/src/types/schema.rs:288-323,406-438,527-535,687-752
 *   tuple → rows           : conversions/event.rs:376-979
 *
 * Assumption: this worker owns every table (should_apply_changes → true, apply.rs:2257), i.e. the
 * apply worker with all tables in the Ready phase.
 */
#define _GNU_SOURCE
#include <stdlib.h>
#include <string.h>

#include "oracle_internal.h"

#define DDL_PREFIX "supabase_etl_ddl" /* event.rs:31 */

typedef struct stored_col {
  char* name;
  uint32_t type_oid;
  uint8_t nullable;
  int32_t pk;
} stored_col;
typedef struct stored_table {
  uint32_t table_id;
  uint64_t snapshot_id;
  uint32_t n_cols;
  stored_col* cols;
} stored_table;
typedef struct cached_rel { /* SharedTableCache Ready{ReplicatedTableSchema} table_cache.rs:36-130 */
  uint32_t table_id;
  orc_schema schema; /* owned arrays */
} cached_rel;

struct orc_ctx {
  stored_table* tables; uint32_t n_tables, cap_tables;
  cached_rel* rels; uint32_t n_rels, cap_rels;
};

orc_ctx* orc_create(void) { return (orc_ctx*)calloc(1, sizeof(orc_ctx)); }

static void free_schema_arrays(orc_schema* s) { free(s->col_kind); free(s->col_flags); free(s->col_index); memset(s, 0, sizeof *s); }
static void free_table(stored_table* t) {
  for (uint32_t i = 0; i < t->n_cols; i++) free(t->cols[i].name);
  free(t->cols); t->cols = NULL; t->n_cols = 0;
}
void orc_reset_relations(orc_ctx* c) {
  for (uint32_t i = 0; i < c->n_rels; i++) free_schema_arrays(&c->rels[i].schema);
  c->n_rels = 0;
}
void orc_destroy(orc_ctx* c) {
  if (!c) return;
  orc_reset_relations(c);
  for (uint32_t i = 0; i < c->n_tables; i++) free_table(&c->tables[i]);
  free(c->tables); free(c->rels); free(c);
}
int orc_put_table_schema(orc_ctx* c, uint32_t table_id, uint64_t snapshot_id,
                         const etl_column_schema* cols, uint32_t n_cols) {
  stored_table* t = NULL;
  for (uint32_t i = 0; i < c->n_tables; i++) if (c->tables[i].table_id == table_id) t = &c->tables[i];
  if (!t) {
    if (c->n_tables == c->cap_tables) { c->cap_tables = c->cap_tables ? c->cap_tables * 2 : 16; c->tables = (stored_table*)realloc(c->tables, c->cap_tables * sizeof(stored_table)); }
    t = &c->tables[c->n_tables++];
    memset(t, 0, sizeof *t);
  } else free_table(t);
  t->table_id = table_id; t->snapshot_id = snapshot_id; t->n_cols = n_cols;
  t->cols = (stored_col*)calloc(n_cols ? n_cols : 1, sizeof(stored_col));
  for (uint32_t i = 0; i < n_cols; i++) {
    t->cols[i].name = strdup(cols[i].name);
    t->cols[i].type_oid = cols[i].type_oid;
    t->cols[i].nullable = cols[i].nullable;
    t->cols[i].pk = cols[i].primary_key_ordinal_position;
  }
  return 0;
}
static stored_table* find_table(orc_ctx* c, uint32_t id) {
  for (uint32_t i = 0; i < c->n_tables; i++) if (c->tables[i].table_id == id) return &c->tables[i];
  return NULL;
}
static cached_rel* find_rel(orc_ctx* c, uint32_t id) {
  for (uint32_t i = 0; i < c->n_rels; i++) if (c->rels[i].table_id == id) return &c->rels[i];
  return NULL;
}

/* ------------------------------------------------------------------ output growth */
static void ensure_records(orc_batch* b, uint64_t n) {
  if (n <= b->cap_records) return;
  uint64_t c = b->cap_records ? b->cap_records * 2 : 1024;
  while (c < n) c *= 2;
#define GROW(f, T, extra) b->f = (T*)realloc(b->f, (c + (extra)) * sizeof(T))
  GROW(rec_off, uint64_t, 0); GROW(rec_kind, uint8_t, 0); GROW(rec_flags, uint8_t, 0);
  GROW(rec_rel, uint32_t, 0); GROW(rec_schema, int32_t, 0); GROW(rec_start_lsn, uint64_t, 0);
  GROW(rec_commit_lsn, uint64_t, 0); GROW(rec_tx_ordinal, uint64_t, 0); GROW(rec_cell_base, uint64_t, 1);
  GROW(rec_tuple_bytes, uint32_t, 0); GROW(rec_heap_hint, uint32_t, 0);
  b->cap_records = c;
}
static void ensure_cells(orc_batch* b, uint64_t n) {
  if (n <= b->cap_cells) return;
  uint64_t c = b->cap_cells ? b->cap_cells * 2 : 4096;
  while (c < n) c *= 2;
  GROW(cell_tag, uint8_t, 0); GROW(cell_val, uint64_t, 0); GROW(cell_aux, uint32_t, 0);
#undef GROW
  b->cap_cells = c;
}
static void push_cell(orc_batch* b, const orc_cell* c) {
  ensure_cells(b, b->n_cells + 1);
  b->cell_tag[b->n_cells] = c->tag; b->cell_val[b->n_cells] = c->val; b->cell_aux[b->n_cells] = c->aux;
  b->n_cells++;
}
static void push_simple(orc_batch* b, uint8_t tag, uint64_t val, uint32_t aux) {
  orc_cell c; c.tag = tag; c.val = val; c.aux = aux; push_cell(b, &c);
}
static int32_t push_schema(orc_batch* b, const orc_schema* s) {
  if (b->n_schemas == b->cap_schemas) { b->cap_schemas = b->cap_schemas ? b->cap_schemas * 2 : 16; b->schemas = (orc_schema*)realloc(b->schemas, b->cap_schemas * sizeof(orc_schema)); }
  orc_schema* d = &b->schemas[b->n_schemas];
  *d = *s;
  d->col_kind = (uint8_t*)malloc(s->n_cols ? s->n_cols : 1); memcpy(d->col_kind, s->col_kind, s->n_cols);
  d->col_flags = (uint8_t*)malloc(s->n_cols ? s->n_cols : 1); memcpy(d->col_flags, s->col_flags, s->n_cols);
  d->col_index = (int32_t*)malloc((s->n_cols ? s->n_cols : 1) * 4); memcpy(d->col_index, s->col_index, s->n_cols * 4);
  return (int32_t)b->n_schemas++;
}
void orc_batch_free(orc_batch* b) {
  if (!b) return;
  free(b->rec_off); free(b->rec_kind); free(b->rec_flags); free(b->rec_rel); free(b->rec_schema);
  free(b->rec_start_lsn); free(b->rec_commit_lsn); free(b->rec_tx_ordinal); free(b->rec_cell_base);
  free(b->rec_tuple_bytes); free(b->rec_heap_hint);
  free(b->cell_tag); free(b->cell_val); free(b->cell_aux); free(b->heap);
  for (uint32_t i = 0; i < b->n_schemas; i++) { free(b->schemas[i].col_kind); free(b->schemas[i].col_flags); free(b->schemas[i].col_index); }
  free(b->schemas);
  memset(b, 0, sizeof *b);
}

/* ------------------------------------------------------------------ wire readers (big-endian) */
static uint16_t be16(const uint8_t* p) { return (uint16_t)((p[0] << 8) | p[1]); }
static uint32_t be32(const uint8_t* p) { return ((uint32_t)p[0] << 24) | ((uint32_t)p[1] << 16) | ((uint32_t)p[2] << 8) | p[3]; }
static uint64_t be64(const uint8_t* p) { return ((uint64_t)be32(p) << 32) | be32(p + 4); }

typedef struct wcell { uint8_t tag; uint32_t len; uint64_t off; } wcell; /* off: absolute stream offset of the value bytes */
typedef struct wtuple { int32_t n; wcell* cells; } wtuple;

/* TupleData (event.rs:1068-1082 pins the layout). Returns bytes consumed or -1 if malformed. */
static int64_t parse_wtuple(const uint8_t* buf, uint64_t pos, uint64_t end, wtuple* t) {
  uint64_t p = pos;
  if (p + 2 > end) return -1;
  int16_t n = (int16_t)be16(buf + p); p += 2;
  t->n = n < 0 ? 0 : n;
  t->cells = (wcell*)calloc((size_t)(t->n ? t->n : 1), sizeof(wcell));
  for (int32_t i = 0; i < t->n; i++) {
    if (p + 1 > end) return -1;
    uint8_t tag = buf[p++];
    t->cells[i].tag = tag;
    if (tag == 'n' || tag == 'u') continue;
    if (tag != 't' && tag != 'b') return -1;
    if (p + 4 > end) return -1;
    int32_t l = (int32_t)be32(buf + p); p += 4;
    if (l < 0 || p + (uint64_t)l > end) return -1;
    t->cells[i].len = (uint32_t)l; t->cells[i].off = p;
    p += (uint64_t)l;
  }
  return (int64_t)(p - pos);
}
/* calculate_tuple_bytes event.rs:260-270 */
static uint64_t tuple_bytes(const wtuple* t) {
  uint64_t s = 0;
  for (int32_t i = 0; i < t->n; i++) if (t->cells[i].tag == 't' || t->cells[i].tag == 'b') s += t->cells[i].len;
  return s;
}
static int64_t cstr_len(const uint8_t* buf, uint64_t p, uint64_t end) {
  for (uint64_t i = p; i < end; i++) if (buf[i] == 0) return (int64_t)(i - p);
  return -1;
}

/* ------------------------------------------------------------------ error bookkeeping */
typedef struct derr { uint32_t code, seq; } derr;
#define SEQ_MALFORMED 0u
#define SEQ_STATE 1u
#define SEQ_TABLE 2u
#define SEQ_OLD_SHAPE 0x10000u
#define SEQ_OLD_CELL(i) (0x10001u + (uint32_t)(i))
#define SEQ_NEW_SHAPE 0x20000u
#define SEQ_NEW_CELL(i) (0x20001u + (uint32_t)(i))

/* Heap bytes owned by a decoded cell — estimate_cell_allocated_bytes, types/table_row.rs:295-345 — for the
 * variants whose final Rust value this path builds: String / Bytes = the buffer's capacity (= length: to_owned,
 * Vec::with_capacity hex.rs:21); Numeric = capacity of the digit Vec, which numeric.rs:441-448 grows by push from
 * Vec::new() (RawVec amortised growth 0 → 4 → 8 → 16 …, capacity survives the zero strips), × size_of::<i16>().
 * A value cloned from the old image (event.rs:958-970) allocates exactly its length.  Json / Array: the estimate
 * walks the serde_json::Value / ArrayCell, which only the materialising side builds — not counted here. */
static uint32_t vec_cap_after_pushes(uint32_t n) { uint32_t c = 4; if (!n) return 0; while (c < n) c <<= 1; return c; }
static uint32_t cell_heap_hint(const orc_cell* c, const orc_heap* heap, int cloned) {
  if (c->tag == ETL_CELL_STRING || c->tag == ETL_CELL_BYTES) return c->aux;
  if (c->tag == ETL_CELL_NUMERIC) {
    if (cloned) return 2u * c->aux;
    etl_numeric_hdr h; memcpy(&h, heap->data + c->val, sizeof h);
    return 2u * vec_cap_after_pushes(h.pushed_groups);
  }
  return 0;
}
static __thread uint64_t g_hint;   /* accumulates over the cells of the record being converted */

/* convert_tuple_data_to_cell event.rs:934-979. returns 0 ok/present, 1 missing, or sets *e */
static int convert_cell(const uint8_t* buf, const wcell* w, uint8_t kind, uint8_t nullable,
                        const orc_cell* old_value, orc_heap* heap, orc_cell* out, uint32_t* ecode) {
  switch (w->tag) {
    case 'n':
      if (nullable) { out->tag = ETL_CELL_NULL; out->val = 0; out->aux = 0; return 0; }
      *ecode = ETL_E_NOT_NULL; return -1;
    case 'u':
      if (old_value) { *out = *old_value; g_hint += cell_heap_hint(out, heap, 1); return 0; }
      return 1;
    case 't':
      if (!orc_utf8_valid(buf + w->off, w->len)) { *ecode = ETL_E_UTF8; return -1; }
      *ecode = orc_parse_text(kind, buf + w->off, w->len, w->off, heap, out);
      if (!*ecode) g_hint += cell_heap_hint(out, heap, 0);
      return *ecode ? -1 : 0;
    default: /* 'b' */
      *ecode = ETL_E_BINARY_FORMAT; return -1;
  }
}

/* convert_tuple_to_row event.rs:550-583 */
static int convert_full_row(const uint8_t* buf, const orc_schema* s, const wtuple* t, orc_heap* heap,
                            orc_cell* out, derr* e, int is_old) {
  if ((uint32_t)t->n != s->n_cols) { e->code = ETL_E_FIELD_COUNT; e->seq = is_old ? SEQ_OLD_SHAPE : SEQ_NEW_SHAPE; return -1; }
  for (uint32_t i = 0; i < s->n_cols; i++) {
    uint32_t ec = 0;
    int r = convert_cell(buf, &t->cells[i], s->col_kind[i], s->col_flags[i] & 1, NULL, heap, &out[i], &ec);
    if (r == 1) ec = ETL_E_FULL_ROW_MISSING;
    if (r != 0) { e->code = ec; e->seq = is_old ? SEQ_OLD_CELL(i) : SEQ_NEW_CELL(i); return -1; }
  }
  return 0;
}
/* normalize_key_tuple_to_row event.rs:879-919 (+ :791-860). out gets n_identity cells */
static int convert_key_row(const uint8_t* buf, const orc_schema* s, const wtuple* t, orc_heap* heap,
                           orc_cell* out, derr* e) {
  if (s->n_identity == 0) { e->code = ETL_E_KEY_NO_COLUMNS; e->seq = SEQ_OLD_SHAPE; return -1; }
  if ((uint32_t)t->n == s->n_identity) {            /* dense */
    uint32_t k = 0;
    for (uint32_t i = 0; i < s->n_cols; i++) {
      if (!(s->col_flags[i] & 2)) continue;
      uint32_t ec = 0;
      int r = convert_cell(buf, &t->cells[k], s->col_kind[i], s->col_flags[i] & 1, NULL, heap, &out[k], &ec);
      if (r == 1) ec = ETL_E_KEY_MISSING_VALUE;
      if (r != 0) { e->code = ec; e->seq = SEQ_OLD_CELL(k); return -1; }
      k++;
    }
    return 0;
  }
  if ((uint32_t)t->n == s->n_cols) {                /* full width: non-identity entries skipped undecoded */
    uint32_t k = 0;
    for (uint32_t i = 0; i < s->n_cols; i++) {
      if (!(s->col_flags[i] & 2)) continue;
      uint32_t ec = 0;
      int r = convert_cell(buf, &t->cells[i], s->col_kind[i], s->col_flags[i] & 1, NULL, heap, &out[k], &ec);
      if (r == 1) ec = ETL_E_KEY_MISSING_VALUE;
      if (r != 0) { e->code = ec; e->seq = SEQ_OLD_CELL(i); return -1; }
      k++;
    }
    return 0;
  }
  e->code = ETL_E_KEY_SHAPE; e->seq = SEQ_OLD_SHAPE; return -1;
}

/* handle_relation_message apply.rs:2012-2089: names → masks → ReplicatedTableSchema */
static int build_relation(orc_ctx* c, const uint8_t* buf, uint64_t body, uint64_t end, uint32_t rel_id,
                          uint64_t frame_off, orc_schema* out, uint32_t* ecode) {
  /* body points after 'R' + rel_id; already validated structurally by the caller */
  uint64_t p = body;
  p += (uint64_t)cstr_len(buf, p, end) + 1;          /* namespace */
  p += (uint64_t)cstr_len(buf, p, end) + 1;          /* relation name */
  uint8_t replident = buf[p++];
  int16_t ncols = (int16_t)be16(buf + p); p += 2;
  if (ncols < 0) ncols = 0;
  stored_table* t = find_table(c, rel_id);
  if (!t) { *ecode = ETL_E_MISSING_TABLE_SCHEMA; return -1; }
  uint8_t* repl = (uint8_t*)calloc(t->n_cols ? t->n_cols : 1, 1);
  uint8_t* ident = (uint8_t*)calloc(t->n_cols ? t->n_cols : 1, 1);
  int unknown = 0;
  for (int i = 0; i < ncols; i++) {
    uint8_t flags = buf[p++];
    int64_t nl = cstr_len(buf, p, end);
    const char* name = (const char*)(buf + p);
    p += (uint64_t)nl + 1 + 8;
    int found = 0;
    for (uint32_t k = 0; k < t->n_cols; k++) {
      if (strlen(t->cols[k].name) == (size_t)nl && memcmp(t->cols[k].name, name, (size_t)nl) == 0) {
        found = 1; repl[k] = 1;
        if (replident == 'f' || (flags & 1)) ident[k] = 1;   /* event.rs:351-366 */
      }
    }
    if (!found) unknown = 1;                              /* schema.rs:288-309 */
  }
  if (unknown) { free(repl); free(ident); *ecode = ETL_E_UNKNOWN_COLUMNS; return -1; }
  memset(out, 0, sizeof *out);
  out->table_id = rel_id; out->snapshot_id = t->snapshot_id; out->effective_off = frame_off;
  uint32_t n = 0;
  for (uint32_t k = 0; k < t->n_cols; k++) n += repl[k];
  out->n_cols = n;
  out->col_kind = (uint8_t*)malloc(n ? n : 1); out->col_flags = (uint8_t*)malloc(n ? n : 1); out->col_index = (int32_t*)malloc((n ? n : 1) * 4);
  uint32_t j = 0;
  for (uint32_t k = 0; k < t->n_cols; k++) {
    if (!repl[k]) continue;
    out->col_kind[j] = (uint8_t)orc_kind_for_oid(t->cols[k].type_oid);
    out->col_flags[j] = (uint8_t)((t->cols[k].nullable ? 1 : 0) | (ident[k] ? 2 : 0));
    out->col_index[j] = (int32_t)k;
    if (ident[k]) out->n_identity++;
    j++;
  }
  free(repl); free(ident);
  return 0;
}

static int cmp_rel(const void* a, const void* b) {
  uint32_t x = ((const cached_rel*)a)->table_id, y = ((const cached_rel*)b)->table_id;
  return x < y ? -1 : x > y;
}

int orc_decode(orc_ctx* c, const uint8_t* buf, uint64_t len, const etl_stream_state* carry_in,
               orc_batch* b) {
  memset(b, 0, sizeof *b);
  orc_heap heap = {0, 0, 0};
  etl_stream_state st;
  memset(&st, 0, sizeof st);
  if (carry_in) st = *carry_in;
  b->first_error.record_index = UINT64_MAX;

  /* batch-local schema list: carried-in versions first, ascending table id */
  qsort(c->rels, c->n_rels, sizeof(cached_rel), cmp_rel);
  int32_t* rel_ver = (int32_t*)malloc((c->n_rels + 1) * sizeof(int32_t));
  for (uint32_t i = 0; i < c->n_rels; i++) {
    orc_schema s = c->rels[i].schema; s.effective_off = 0;
    rel_ver[i] = push_schema(b, &s);
  }
  uint32_t rel_ver_cap = c->n_rels + 1;

  uint64_t pos = 0, rec = 0;
  derr err = {0, 0};
  orc_cell* oldc = NULL; orc_cell* newc = NULL; uint32_t cell_cap = 0;
  while (pos < len) {
    ensure_records(b, rec + 1);
    b->rec_off[rec] = pos; b->rec_kind[rec] = 0; b->rec_flags[rec] = 0; b->rec_rel[rec] = 0;
    b->rec_schema[rec] = -1; b->rec_start_lsn[rec] = 0; b->rec_commit_lsn[rec] = 0;
    b->rec_tx_ordinal[rec] = 0; b->rec_cell_base[rec] = b->n_cells;
    b->rec_tuple_bytes[rec] = 0; b->rec_heap_hint[rec] = 0;
    err.code = 0; err.seq = 0;
    wtuple t_old = {0, NULL}, t_new = {0, NULL};
    /* ---- CopyData framing written by the stager */
    if (pos + 5 > len || buf[pos] != 'd') { err.code = ETL_E_MALFORMED_FRAME; goto fail; }
    uint32_t flen = be32(buf + pos + 1);
    if (flen < 4 || pos + 1 + (uint64_t)flen > len) { err.code = ETL_E_MALFORMED_FRAME; goto fail; }
    uint64_t body = pos + 5, end = pos + 1 + flen;
    uint64_t next = end;
    if (body >= end) { err.code = ETL_E_MALFORMED_FRAME; goto fail; }
    /* ---- ReplicationMessage::parse */
    if (buf[body] == 'k') {
      if (end - body < 18) { err.code = ETL_E_MALFORMED_FRAME; goto fail; }
      b->rec_kind[rec] = ETL_REC_KEEPALIVE;
      b->rec_start_lsn[rec] = be64(buf + body + 1);      /* wal_end apply.rs:1715 */
      b->rec_rel[rec] = buf[body + 17];                  /* reply requested apply.rs:1720 */
      goto done;
    }
    if (buf[body] != 'w' || end - body < 26) { err.code = ETL_E_MALFORMED_FRAME; goto fail; }
    uint64_t start_lsn = be64(buf + body + 1);           /* wal_start apply.rs:1700 */
    uint64_t m = body + 25;                              /* pgoutput message */
    uint8_t tag = buf[m];
    uint64_t p = m + 1;
    b->rec_kind[rec] = tag;
    b->rec_start_lsn[rec] = start_lsn;
    /* ---- LogicalReplicationMessage::parse (structure first: a parse error precedes any state change) */
    uint32_t rel_id = 0; uint8_t old_tag = 0;
    switch (tag) {
      case 'B': if (end - p < 20) { err.code = ETL_E_MALFORMED_FRAME; goto fail; } break;
      case 'C': if (end - p < 25) { err.code = ETL_E_MALFORMED_FRAME; goto fail; } break;
      case 'O': if (end - p < 8 || cstr_len(buf, p + 8, end) < 0) { err.code = ETL_E_MALFORMED_FRAME; goto fail; } break;
      case 'Y': {
        if (end - p < 4) { err.code = ETL_E_MALFORMED_FRAME; goto fail; }
        int64_t a = cstr_len(buf, p + 4, end);
        if (a < 0 || cstr_len(buf, p + 4 + (uint64_t)a + 1, end) < 0) { err.code = ETL_E_MALFORMED_FRAME; goto fail; }
        break;
      }
      case 'R': {
        if (end - p < 4) { err.code = ETL_E_MALFORMED_FRAME; goto fail; }
        rel_id = be32(buf + p);
        uint64_t q = p + 4;
        int64_t a = cstr_len(buf, q, end); if (a < 0) { err.code = ETL_E_MALFORMED_FRAME; goto fail; } q += (uint64_t)a + 1;
        a = cstr_len(buf, q, end); if (a < 0) { err.code = ETL_E_MALFORMED_FRAME; goto fail; } q += (uint64_t)a + 1;
        if (q + 3 > end) { err.code = ETL_E_MALFORMED_FRAME; goto fail; }
        uint8_t ri = buf[q];
        if (ri != 'd' && ri != 'n' && ri != 'f' && ri != 'i') { err.code = ETL_E_MALFORMED_FRAME; goto fail; }
        int16_t nc = (int16_t)be16(buf + q + 1); q += 3;
        for (int i = 0; i < nc; i++) {
          if (q + 1 > end) { err.code = ETL_E_MALFORMED_FRAME; goto fail; }
          q += 1;
          a = cstr_len(buf, q, end); if (a < 0) { err.code = ETL_E_MALFORMED_FRAME; goto fail; }
          if (!orc_utf8_valid(buf + q, (uint64_t)a)) { err.code = ETL_E_MALFORMED_FRAME; goto fail; }
          q += (uint64_t)a + 1;
          if (q + 8 > end) { err.code = ETL_E_MALFORMED_FRAME; goto fail; }
          q += 8;
        }
        break;
      }
      case 'I': {
        if (end - p < 5 || buf[p + 4] != 'N') { err.code = ETL_E_MALFORMED_FRAME; goto fail; }
        rel_id = be32(buf + p);
        if (parse_wtuple(buf, p + 5, end, &t_new) < 0) { err.code = ETL_E_MALFORMED_FRAME; goto fail; }
        break;
      }
      case 'U': {
        if (end - p < 5) { err.code = ETL_E_MALFORMED_FRAME; goto fail; }
        rel_id = be32(buf + p);
        uint64_t q = p + 4;
        uint8_t tt = buf[q++];
        if (tt == 'O' || tt == 'K') {
          old_tag = tt;
          int64_t used = parse_wtuple(buf, q, end, &t_old);
          if (used < 0) { err.code = ETL_E_MALFORMED_FRAME; goto fail; }
          q += (uint64_t)used;
          if (q + 1 > end || buf[q] != 'N') { err.code = ETL_E_MALFORMED_FRAME; goto fail; }
          q++;
        } else if (tt != 'N') { err.code = ETL_E_MALFORMED_FRAME; goto fail; }
        if (parse_wtuple(buf, q, end, &t_new) < 0) { err.code = ETL_E_MALFORMED_FRAME; goto fail; }
        break;
      }
      case 'D': {
        if (end - p < 5) { err.code = ETL_E_MALFORMED_FRAME; goto fail; }
        rel_id = be32(buf + p);
        old_tag = buf[p + 4];
        if (old_tag != 'O' && old_tag != 'K') { err.code = ETL_E_MALFORMED_FRAME; goto fail; }
        if (parse_wtuple(buf, p + 5, end, &t_old) < 0) { err.code = ETL_E_MALFORMED_FRAME; goto fail; }
        break;
      }
      case 'T': {
        if (end - p < 5) { err.code = ETL_E_MALFORMED_FRAME; goto fail; }
        int32_t n = (int32_t)be32(buf + p);
        if (n > 0 && (uint64_t)n * 4 > end - p - 5) { err.code = ETL_E_MALFORMED_FRAME; goto fail; }
        break;
      }
      case 'M': {
        if (end - p < 9) { err.code = ETL_E_MALFORMED_FRAME; goto fail; }
        int64_t a = cstr_len(buf, p + 9, end);
        if (a < 0 || !orc_utf8_valid(buf + p + 9, (uint64_t)a)) { err.code = ETL_E_MALFORMED_FRAME; goto fail; }
        uint64_t q = p + 9 + (uint64_t)a + 1;
        if (q + 4 > end) { err.code = ETL_E_MALFORMED_FRAME; goto fail; }
        int32_t cl = (int32_t)be32(buf + q);
        if (cl < 0 || q + 4 + (uint64_t)cl > end) { err.code = ETL_E_MALFORMED_FRAME; goto fail; }
        break;
      }
      default: err.code = ETL_E_MALFORMED_FRAME; goto fail; /* unknown tag: parser returns io::Error */
    }
    b->rec_rel[rec] = rel_id;

    /* ---- handle_logical_replication_message apply.rs:1742-1784 */
    switch (tag) {
      case 'B': {                                          /* apply.rs:1927-1943 */
        uint64_t final_lsn = be64(buf + p);
        st.in_tx = 1; st.final_lsn = final_lsn; st.next_tx_ordinal = 0;
        b->rec_commit_lsn[rec] = final_lsn;
        b->rec_tx_ordinal[rec] = st.next_tx_ordinal++;
        b->rec_flags[rec] |= ETL_RF_EVENT;
        push_simple(b, ETL_CELL_I64, be64(buf + p + 8), 0);                 /* timestamp event.rs:286 */
        push_simple(b, ETL_CELL_U32, be32(buf + p + 16), 0);                /* xid event.rs:287 */
        break;
      }
      case 'C': {                                          /* apply.rs:1946-2006 */
        if (!st.in_tx) { err.code = ETL_E_TX_STATE; err.seq = SEQ_STATE; goto fail; }
        uint64_t remote_final = st.final_lsn;
        st.in_tx = 0;                                      /* remote_final_lsn.take() */
        uint64_t commit_lsn = be64(buf + p + 1);
        if (commit_lsn != remote_final) { err.code = ETL_E_COMMIT_LSN; err.seq = SEQ_STATE; goto fail; }
        b->rec_commit_lsn[rec] = commit_lsn;
        b->rec_tx_ordinal[rec] = st.next_tx_ordinal++;
        b->rec_flags[rec] |= ETL_RF_EVENT;
        push_simple(b, ETL_CELL_I32, (uint64_t)(int64_t)(int8_t)buf[p], 0);  /* flags event.rs:305 */
        push_simple(b, ETL_CELL_I64, be64(buf + p + 9), 0);                  /* end_lsn event.rs:306 */
        push_simple(b, ETL_CELL_I64, be64(buf + p + 17), 0);                 /* timestamp event.rs:307 */
        break;
      }
      case 'R': {                                          /* apply.rs:2012-2089 */
        if (!st.in_tx) { err.code = ETL_E_TX_STATE; err.seq = SEQ_STATE; goto fail; }
        b->rec_commit_lsn[rec] = st.final_lsn;
        b->rec_tx_ordinal[rec] = st.next_tx_ordinal++;
        orc_schema s; uint32_t ec = 0;
        if (build_relation(c, buf, p + 4, end, rel_id, pos, &s, &ec) < 0) { err.code = ec; err.seq = SEQ_TABLE; goto fail; }
        cached_rel* r = find_rel(c, rel_id);
        if (!r) {
          if (c->n_rels == c->cap_rels) { c->cap_rels = c->cap_rels ? c->cap_rels * 2 : 16; c->rels = (cached_rel*)realloc(c->rels, c->cap_rels * sizeof(cached_rel)); }
          r = &c->rels[c->n_rels++]; memset(r, 0, sizeof *r); r->table_id = rel_id;
          if (c->n_rels > rel_ver_cap) { rel_ver_cap = c->n_rels * 2; rel_ver = (int32_t*)realloc(rel_ver, rel_ver_cap * sizeof(int32_t)); }
        } else free_schema_arrays(&r->schema);
        r->schema = s;                                     /* note_ready apply.rs:2079 */
        int32_t ver = push_schema(b, &s);
        rel_ver[r - c->rels] = ver;
        b->rec_schema[rec] = ver;
        b->rec_flags[rec] |= ETL_RF_EVENT;
        break;
      }
      case 'I': case 'U': case 'D': {                      /* apply.rs:2092-2203 */
        if (!st.in_tx) { err.code = ETL_E_TX_STATE; err.seq = SEQ_STATE; goto fail; }
        b->rec_commit_lsn[rec] = st.final_lsn;
        b->rec_tx_ordinal[rec] = st.next_tx_ordinal++;
        cached_rel* r = find_rel(c, rel_id);               /* get_replicated_table_schema apply.rs:3324-3357 */
        if (!r) { err.code = ETL_E_MISSING_TABLE_STATE; err.seq = SEQ_TABLE; goto fail; }
        const orc_schema* s = &r->schema;
        b->rec_schema[rec] = rel_ver[r - c->rels];
        b->rec_flags[rec] |= ETL_RF_EVENT;
        if (s->n_cols + 1 > cell_cap) { cell_cap = s->n_cols + 64; oldc = (orc_cell*)realloc(oldc, cell_cap * sizeof(orc_cell)); newc = (orc_cell*)realloc(newc, cell_cap * sizeof(orc_cell)); }
        uint32_t n_old = 0;
        g_hint = 0;
        b->rec_tuple_bytes[rec] = (uint32_t)(tuple_bytes(&t_new) + tuple_bytes(&t_old));   /* ETL_ROW_SIZE_BYTES sample event.rs:388,462,507 */
        if (tag == 'I') {                                  /* event.rs:376-393 */
          b->insert_bytes += tuple_bytes(&t_new);
          if (convert_full_row(buf, s, &t_new, &heap, newc, &err, 0) < 0) goto fail;
          for (uint32_t i = 0; i < s->n_cols; i++) push_cell(b, &newc[i]);
          b->rec_heap_hint[rec] = (uint32_t)g_hint;
          break;
        }
        /* old image first (event.rs:429-450 / :499-520) */
        uint64_t tb = tuple_bytes(&t_old);
        if (tag == 'U') { b->update_bytes += tuple_bytes(&t_new) + (old_tag ? tb : 0); } else b->delete_bytes += tb;
        if (old_tag == 'K') {
          b->rec_flags[rec] |= ETL_RF_OLD_KEY;
          if (convert_key_row(buf, s, &t_old, &heap, oldc, &err) < 0) goto fail;
          n_old = s->n_identity;
        } else if (old_tag == 'O') {
          b->rec_flags[rec] |= ETL_RF_OLD_FULL;
          if (convert_full_row(buf, s, &t_old, &heap, oldc, &err, 1) < 0) goto fail;
          n_old = s->n_cols;
        }
        if (tag == 'U') {                                  /* convert_update_tuple_to_updated_table_row event.rs:601-671 */
          if ((uint32_t)t_new.n != s->n_cols) { err.code = ETL_E_FIELD_COUNT; err.seq = SEQ_NEW_SHAPE; goto fail; }
          uint32_t key_i = 0; int partial = 0;
          for (uint32_t i = 0; i < s->n_cols; i++) {
            int is_ident = (s->col_flags[i] & 2) != 0;
            const orc_cell* oldv = NULL;                   /* OldRowResolver::value_for_column event.rs:722-762 */
            if (old_tag == 'O') oldv = &oldc[i];
            else if (old_tag == 'K' && is_ident) oldv = &oldc[key_i++];
            uint32_t ec = 0;
            int rr = convert_cell(buf, &t_new.cells[i], s->col_kind[i], s->col_flags[i] & 1, oldv, &heap, &newc[i], &ec);
            if (rr < 0) { err.code = ec; err.seq = SEQ_NEW_CELL(i); goto fail; }
            if (rr == 1) { partial = 1; newc[i].tag = ETL_CELL_MISSING; newc[i].val = 0; newc[i].aux = 0; }
          }
          if (partial) b->rec_flags[rec] |= ETL_RF_NEW_PARTIAL;
        }
        for (uint32_t i = 0; i < n_old; i++) push_cell(b, &oldc[i]);
        if (tag == 'U') for (uint32_t i = 0; i < s->n_cols; i++) push_cell(b, &newc[i]);
        b->rec_heap_hint[rec] = (uint32_t)g_hint;
        break;
      }
      case 'T': {                                          /* apply.rs:2206-2248 */
        if (!st.in_tx) { err.code = ETL_E_TX_STATE; err.seq = SEQ_STATE; goto fail; }
        b->rec_commit_lsn[rec] = st.final_lsn;
        b->rec_tx_ordinal[rec] = st.next_tx_ordinal++;
        int32_t n = (int32_t)be32(buf + p); if (n < 0) n = 0;
        b->rec_rel[rec] = (uint32_t)n;
        push_simple(b, ETL_CELL_I32, (uint64_t)(int64_t)(int8_t)buf[p + 4], 0); /* options event.rs:540 */
        for (int32_t i = 0; i < n; i++) {
          uint32_t rid = be32(buf + p + 5 + 4 * (uint64_t)i);
          cached_rel* r = find_rel(c, rid);
          if (!r) { err.code = ETL_E_MISSING_TABLE_STATE; err.seq = SEQ_TABLE; goto fail; }
          push_simple(b, ETL_CELL_U32, rid, (uint32_t)rel_ver[r - c->rels]);
        }
        if (n > 0) b->rec_flags[rec] |= ETL_RF_EVENT;
        break;
      }
      case 'M': {                                          /* apply.rs:1808-1924: never consumes an ordinal */
        int64_t a = cstr_len(buf, p + 9, end);
        if ((size_t)a == strlen(DDL_PREFIX) && memcmp(buf + p + 9, DDL_PREFIX, (size_t)a) == 0) {
          b->rec_flags[rec] |= ETL_RF_DDL_MESSAGE;
          if (!st.in_tx) { err.code = ETL_E_TX_STATE; err.seq = SEQ_STATE; goto fail; }
        }
        break;
      }
      default: break;                                      /* Origin / Type ignored apply.rs:1771-1778 */
    }
  done:
    free(t_old.cells); free(t_new.cells);
    if (b->rec_flags[rec] & ETL_RF_EVENT) b->n_events++;
    rec++;
    pos = next;
    continue;
  fail:
    free(t_old.cells); free(t_new.cells);
    b->first_error.record_index = rec;
    b->first_error.seq = err.seq;
    b->first_error.code = err.code;
    b->first_error.kind = orc_error_kind(err.code);
    b->n_cells = b->rec_cell_base[rec]; /* drop cells of the failing record */
    break;
  }
  ensure_records(b, rec + 1);
  b->rec_cell_base[rec] = b->n_cells;
  b->n_records = rec;
  b->heap = heap.data; b->heap_bytes = heap.len;
  b->carry_out = st;
  free(oldc); free(newc); free(rel_ver);
  return 0;
}
