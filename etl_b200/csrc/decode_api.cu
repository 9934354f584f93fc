// decode_api.cu — extern "C" ABI (include/etl_decode.h) of the H100 pgoutput decode engine.
//
// Host side only does what the reference does per batch / per Relation message (rare, control
// path): staging, schema catalogue, Relation → ReplicationMask / IdentityMask
// (apply.rs:2012-2089, event.rs:325-369, etl-postgres/src/types/schema.rs:288-323,406-438,527-535),
// buffer management and kernel orchestration.  Every per-row / per-cell operation of the hot path
// runs in the sm_90a kernels of wal_kernels.cuh / rows_kernel.cuh; there is no CPU decode fallback.
//
// One decode = one host synchronisation, at the end.  The planes are sized from what the previous
// batches needed per staged byte; k_chase / k_records compare the real totals with the reservation on the device and,
// when they do not fit, every later kernel returns at once and the host re-runs the record and tuple passes
// with exact sizes (the first batch of a context takes the exact path: index pass, sync, then the rest).
// Multi-GPU: the shard seam summaries are all-gathered by NCCL on the decode stream and folded on the
// device (k_seam_fold) — nothing returns to the host between the index pass and the record pass.
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <link.h>
#include <nccl.h>   // types and prototypes only: the entry points are resolved at run time (etl_dec_comm_*)

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <string>
#include <vector>

#include "etl_decode.h"
#include "batch_internal.h"
#include "oid_classes.h"
#include "wal_kernels.cuh"

using namespace etl;

namespace {

struct StoredCol {
  std::string name;
  uint32_t type_oid;
  int32_t modifier, ordinal, pk;
  uint8_t nullable;
};
struct StoredTable {
  uint64_t snapshot_id = 0;
  std::vector<StoredCol> cols;
};
struct RelVersion {  // ReplicatedTableSchema (schema.rs:651-900)
  uint32_t table_id = 0;
  uint64_t snapshot_id = 0;
  uint64_t effective_off = 0;
  uint32_t n_ident = 0;
  std::vector<uint8_t> kind, flags;
  std::vector<int32_t> index;
};

bool kind_supported_on_device(uint32_t k) {
  if (k & ETL_K_ARRAY) k &= ~(uint32_t)ETL_K_ARRAY;   // arrays: element kinds below
  switch (k) {
    case ETL_K_BOOL: case ETL_K_STRING: case ETL_K_I16: case ETL_K_I32: case ETL_K_U32: case ETL_K_I64:
    case ETL_K_NUMERIC: case ETL_K_DATE: case ETL_K_TIME: case ETL_K_TIMESTAMP: case ETL_K_TIMESTAMPTZ:
    case ETL_K_UUID: case ETL_K_JSON: case ETL_K_BYTES: case ETL_K_F32: case ETL_K_F64:
      return true;
    default: return false;
  }
}
bool kind_has_heap(uint32_t k) { return k == ETL_K_NUMERIC || k == ETL_K_UUID || k == ETL_K_BYTES || (k & ETL_K_ARRAY); }

uint32_t error_kind_of(uint32_t code) {
  switch (code) {
    case ETL_E_NONE: return ETL_EK_NONE;
    case ETL_E_UUID: case ETL_E_BOOL: case ETL_E_NOT_NULL: return ETL_EK_INVALID_DATA;
    case ETL_E_JSON: return ETL_EK_DESERIALIZATION_ERROR;
    case ETL_E_TX_STATE: case ETL_E_MISSING_TABLE_STATE: return ETL_EK_INVALID_STATE;
    case ETL_E_COMMIT_LSN: return ETL_EK_VALIDATION_ERROR;
    case ETL_E_UNKNOWN_COLUMNS: return ETL_EK_CORRUPTED_TABLE_SCHEMA;
    case ETL_E_MISSING_TABLE_SCHEMA: return ETL_EK_MISSING_TABLE_SCHEMA;
    case ETL_E_MALFORMED_FRAME: return ETL_EK_SOURCE_ERROR;
    default: return ETL_EK_CONVERSION_ERROR;
  }
}

uint32_t rd32(const uint8_t* p) { return ((uint32_t)p[0] << 24) | ((uint32_t)p[1] << 16) | ((uint32_t)p[2] << 8) | p[3]; }
uint16_t rd16(const uint8_t* p) { return (uint16_t)((p[0] << 8) | p[1]); }

bool utf8_ok(const uint8_t* s, size_t n) {
  size_t i = 0;
  while (i < n) {
    uint8_t b = s[i];
    if (b < 0x80) { i++; continue; }
    if (b >= 0xC2 && b <= 0xDF) { if (i + 1 >= n || (s[i + 1] & 0xC0) != 0x80) return false; i += 2; }
    else if (b >= 0xE0 && b <= 0xEF) {
      if (i + 2 >= n) return false;
      uint8_t lo = b == 0xE0 ? 0xA0 : 0x80, hi = b == 0xED ? 0x9F : 0xBF;
      if (s[i + 1] < lo || s[i + 1] > hi || (s[i + 2] & 0xC0) != 0x80) return false;
      i += 3;
    } else if (b >= 0xF0 && b <= 0xF4) {
      if (i + 3 >= n) return false;
      uint8_t lo = b == 0xF0 ? 0x90 : 0x80, hi = b == 0xF4 ? 0x8F : 0xBF;
      if (s[i + 1] < lo || s[i + 1] > hi || (s[i + 2] & 0xC0) != 0x80 || (s[i + 3] & 0xC0) != 0x80) return false;
      i += 4;
    } else return false;
  }
  return true;
}

// growable device scratch; every instance registers itself with its context so that destroy releases all of them
struct DevBufBase {
  void* p = nullptr;
  size_t cap_bytes = 0;
  cudaError_t ensure_bytes(size_t n) {
    if (n <= cap_bytes) return cudaSuccess;
    if (p) cudaFree(p);
    p = nullptr; cap_bytes = 0;
    size_t want = std::max<size_t>(n + n / 4, 256);
    cudaError_t e = cudaMalloc(&p, want);
    if (e == cudaSuccess) cap_bytes = want;
    return e;
  }
  void release() { if (p) cudaFree(p); p = nullptr; cap_bytes = 0; }
};
template <typename T>
struct DevBuf : DevBufBase {
  explicit DevBuf(std::vector<DevBufBase*>& reg) { reg.push_back(this); }
  T* ptr() const { return static_cast<T*>(p); }
  cudaError_t ensure(size_t n) { return ensure_bytes(n * sizeof(T)); }
  // grow-only like ensure(); a new allocation starts out zeroed (look-back status words: epochs tell the launches apart)
  cudaError_t ensure_zeroed(size_t n, cudaStream_t st) {
    if (n * sizeof(T) <= cap_bytes) return cudaSuccess;
    cudaError_t e = ensure(n);
    return e == cudaSuccess ? cudaMemsetAsync(p, 0, cap_bytes, st) : e;
  }
};

// ---- NCCL, resolved at run time: the library already loaded into the process (PyTorch bundles its own) is
// preferred, the system libnccl.so.2 otherwise.  Linking -lnccl would pull a second copy into a torch process.
struct NcclApi {
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
  bool ok = false;
};
NcclApi& nccl_api() {
  static NcclApi api;
  static bool tried = false;
  if (tried) return api;
  tried = true;
  // the copy the process already holds (PyTorch's bundled NCCL, a host application's, …): found by walking the loaded
  // objects, re-opened by its exact path; only when there is none is the system library loaded.  RTLD_LOCAL: a second
  // NCCL must never interpose its symbols on the first.
  std::string loaded;
  dl_iterate_phdr([](struct dl_phdr_info* info, size_t, void* out) -> int {
    if (info->dlpi_name && strstr(info->dlpi_name, "libnccl.so")) { *static_cast<std::string*>(out) = info->dlpi_name; return 1; }
    return 0;
  }, &loaded);
  void* h = nullptr;
  if (!loaded.empty()) h = dlopen(loaded.c_str(), RTLD_NOW | RTLD_NOLOAD | RTLD_LOCAL);
  if (!h) h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_LOCAL);
  if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_LOCAL);
  if (!h) return api;
  api.GetUniqueId = (decltype(api.GetUniqueId))dlsym(h, "ncclGetUniqueId");
  api.CommInitRank = (decltype(api.CommInitRank))dlsym(h, "ncclCommInitRank");
  api.CommDestroy = (decltype(api.CommDestroy))dlsym(h, "ncclCommDestroy");
  api.AllGather = (decltype(api.AllGather))dlsym(h, "ncclAllGather");
  api.GetErrorString = (decltype(api.GetErrorString))dlsym(h, "ncclGetErrorString");
  api.ok = api.GetUniqueId && api.CommInitRank && api.CommDestroy && api.AllGather && api.GetErrorString;
  return api;
}

constexpr size_t kScalarWords = 16;
// device scalar block: 16 words followed by the DevCarry
//  [0] first_error key  [1..3] insert/update/delete bytes  [4] events  [5] heap_top  [7] long_count  [8] copy_count  [9] heap_overflow
//  [10] arr_top  [11] perm_len  [12] n_act (k_act_scan)  [13] ABORT_* bits (k_chase, k_records)  [14] n_frames (k_chase)  [15] CTAs of k_chase that have published their state aggregate (shards)
constexpr size_t kScalarBlockBytes = kScalarWords * 8 + sizeof(DevCarry);

}  // namespace

// ================================================================================================
struct etl_stager {
  uint8_t* buf = nullptr;   // pinned
  uint64_t cap = 0, len = 0;
  uint32_t stride = 2048;
  std::vector<uint64_t> anchors;
  std::vector<uint64_t> relations;
  size_t n_real_anchors = 0;   // anchors.size() before etl_stage_view padded the tail with `len`
  bool padded = false;
  uint64_t n_frames = 0;
  uint32_t max_frame = 0;    // longest frame ('d' + length field + body), saturating
};

struct etl_dec_batch {
  etl_dec_ctx* ctx = nullptr;
  etl_dec_planes dev{};
  etl_dec_planes host{};
  bool has_host = false;
  void* dev_block = nullptr;   // single device allocation holding all planes
  void* host_block = nullptr;  // pinned host copy (borrowed from ctx->h_result)
  size_t block_bytes = 0;
  etl_dec_summary summary{};
  std::vector<RelVersion> schemas;
  const uint8_t* dev_stream = nullptr;   // the staged bytes the planes point into
  bool copy = false;                     // COPY rows: the table and column classes they were decoded with
  uint32_t copy_table = 0;
  std::vector<uint8_t> copy_kinds;
};

struct etl_dec_ctx {
  int device = 0;
  cudaStream_t stream = nullptr;
  bool own_stream = false;
  bool lines_launched = false;
  std::string last_error;
  std::map<uint32_t, StoredTable> tables;
  std::map<uint32_t, RelVersion> current;  // SharedTableCache Ready state (table_cache.rs:36-130)
  // scratch (all registered in `bufs`)
  std::vector<DevBufBase*> bufs;
  DevBuf<uint8_t> d_stream{bufs};
  DevBuf<uint64_t> d_anchors{bufs};
  DevBuf<uint32_t> d_seg_rec_base{bufs}, d_act{bufs}, d_act_blk{bufs}, d_scan_status{bufs};
  DevBuf<uint64_t> d_frame_off{bufs};      // frame offsets in stream order (k_chase → k_records)
  DevBuf<unsigned long long> d_chase_status{bufs};
  DevBuf<ScanSlot> d_scan_slots{bufs};
  DevBuf<Summ> d_chase_summ{bufs};
  DevBuf<Summ> d_total{bufs};
  uint32_t scan_epoch = 0;
  uint32_t max_frame_hint = 0;            // etl_dec_input.max_frame_len of the batch in flight (0 = unknown)
  bool long_skipped = false;
  // ETL_TRACE=1: host wall time per phase of a decode call, printed by etl_dec_destroy (a measurement aid, not ABI)
  double tr[6] = {0, 0, 0, 0, 0, 0}; uint64_t tr_n = 0; double tr_t0 = 0;              // the long-value passes were left out of the last launch_emit_kernels
  DevBuf<uint8_t> d_tables{bufs};          // DevSchema[] | schema_by_batch[] | col_kind[] | col_flags[] | relation errors
  DevBuf<uint32_t> d_line_bad{bufs}, d_dead{bufs}, d_bin_count{bufs}, d_bin_cursor{bufs}, d_perm{bufs}, d_rec_flen{bufs};
  DevBuf<LongCell> d_long{bufs};
  DevBuf<uint8_t> d_scalars{bufs};         // kScalarBlockBytes
  DevBuf<SeamBlock> d_seam{bufs};          // [0] this rank's block, [1 .. 1+n_ranks) the gathered blocks
  DevBuf<uint8_t> d_rel_x{bufs};           // relation-update exchange: send slot | n_ranks receive slots
  void* h_result = nullptr; size_t h_result_cap = 0;  // pinned result staging, grow-only
  uint8_t* h_up = nullptr; size_t h_up_cap = 0;       // pinned staging of the small per-batch uploads
  uint8_t* h_rel_x = nullptr; size_t h_rel_x_cap = 0; // pinned staging of the relation-update exchange
  uint64_t pending_h2d_bytes = 0;
  Summ* h_total = nullptr;               // pinned
  unsigned long long* h_scalars = nullptr;  // pinned, kScalarWords + DevCarry
  cudaEvent_t ev[6]{};
  cudaEvent_t evk[4]{};
  cudaStream_t side = nullptr;           // k_utf8_dead runs here, underneath the tuple pass
  cudaEvent_t ev_in = nullptr, ev_l0 = nullptr, ev_l1 = nullptr;
  // decode in flight
  bool pending = false;
  DecodeParams P{};
  std::vector<RelVersion> pending_schemas;
  std::vector<std::pair<uint64_t, RelVersion>> pending_installs;   // (frame offset, version) of this batch's Relation frames: committed by finish
  std::vector<RelVersion> foreign_installs;                        // versions announced by the other shards (sharded decode)
  uint32_t pending_flags = 0;
  uint32_t launches = 0;
  bool tables_valid = false;             // d_tables matches `current` and no Relation frame since
  size_t n_layouts = 1;
  // what earlier batches needed per staged byte (sizing of the next one)
  double rec_per_byte = 0, cells_per_byte = 0;
  // multi-GPU
  ncclComm_t comm = nullptr;
  etl_host_allgather_fn host_allgather = nullptr;   // exchange through the host instead of NCCL (etl_dec_comm_init_host)
  void* host_user = nullptr;
  int rank = 0, n_ranks = 1;
  size_t rel_slot = 4 << 10;             // bytes per rank in the relation-update exchange (grows on demand)
  uint8_t* h_seam = nullptr; size_t h_seam_cap = 0;   // pinned copy of the gathered seam blocks
};

#define CK(call)                                                                         \
  do {                                                                                   \
    cudaError_t _e = (call);                                                             \
    if (_e != cudaSuccess) {                                                             \
      ctx->last_error = std::string(#call) + ": " + cudaGetErrorString(_e);              \
      return ETL_ERR_CUDA;                                                               \
    }                                                                                    \
  } while (0)
#define CKN(call)                                                                        \
  do {                                                                                   \
    ncclResult_t _r = (call);                                                            \
    if (_r != ncclSuccess) {                                                             \
      ctx->last_error = std::string(#call) + ": " + nccl_api().GetErrorString(_r);       \
      return ETL_ERR_CUDA;                                                               \
    }                                                                                    \
  } while (0)

static bool trace_on() { static const bool on = getenv("ETL_TRACE") != nullptr; return on; }
static double now_us() { timespec ts; clock_gettime(CLOCK_MONOTONIC, &ts); return ts.tv_sec * 1e6 + ts.tv_nsec * 1e-3; }
#define TRACE_MARK(i) do { if (trace_on()) { const double _t = now_us(); ctx->tr[i] += _t - ctx->tr_t0; ctx->tr_t0 = _t; } } while (0)

extern "C" {

uint32_t etl_dec_abi_version(void) { return ETL_DECODE_ABI_VERSION; }
uint32_t etl_dec_kind_for_type_oid(uint32_t type_oid) { return etl_oid_decode_class(type_oid); }

// ------------------------------------------------------------------------------------------------ stager
int etl_stage_create(uint64_t capacity_bytes, uint32_t anchor_stride, etl_stager** out) {
  if (!out || anchor_stride < 256 || anchor_stride > 32768 || (anchor_stride & (anchor_stride - 1))) return ETL_ERR_INVALID_ARG;
  etl_stager* s = new etl_stager();
  s->stride = anchor_stride;
  s->cap = capacity_bytes;
  // pinned when a CUDA device is usable, plain memory otherwise (the stager itself needs no GPU); 64 bytes of
  // zero padding follow the staged bytes (the kernels read whole aligned words around a cell)
  const uint64_t alloc = capacity_bytes + 64;
  if (cudaHostAlloc((void**)&s->buf, alloc, cudaHostAllocDefault) != cudaSuccess) {
    cudaGetLastError();
    s->buf = (uint8_t*)malloc(alloc);
    if (!s->buf) { delete s; return ETL_ERR_ALLOC; }
    s->cap |= (1ull << 63);  // tag: malloc'ed
  }
  memset(s->buf + capacity_bytes, 0, 64);
  *out = s;
  return ETL_OK;
}
void etl_stage_destroy(etl_stager* s) {
  if (!s) return;
  if (s->cap >> 63) free(s->buf); else cudaFreeHost(s->buf);
  delete s;
}
void etl_stage_reset(etl_stager* s) { s->len = 0; s->anchors.clear(); s->relations.clear(); s->padded = false; s->n_real_anchors = 0; s->n_frames = 0; s->max_frame = 0; }

static inline void stage_note_frame(etl_stager* s, uint64_t off, const uint8_t* body, uint32_t body_len) {
  // anchors[k] = first frame starting at or after k*stride
  if (s->padded) { s->anchors.resize(s->n_real_anchors); s->padded = false; }
  while ((uint64_t)s->anchors.size() * s->stride <= off) s->anchors.push_back(off);
  if (body_len >= 26 && body[0] == 'w' && body[25] == 'R') s->relations.push_back(off);
  s->n_frames++;
  s->max_frame = std::max<uint32_t>(s->max_frame, (uint32_t)std::min<uint64_t>(0xFFFFFFFFull, 5ull + body_len));
}
int etl_stage_append(etl_stager* s, const uint8_t* body, uint32_t body_len) {
  uint64_t cap = s->cap & ~(1ull << 63);
  if (s->len + 5ull + body_len > cap) return ETL_ERR_ALLOC;
  uint64_t off = s->len;
  uint8_t* d = s->buf + off;
  uint32_t fl = body_len + 4;
  d[0] = 'd'; d[1] = (uint8_t)(fl >> 24); d[2] = (uint8_t)(fl >> 16); d[3] = (uint8_t)(fl >> 8); d[4] = (uint8_t)fl;
  memcpy(d + 5, body, body_len);
  stage_note_frame(s, off, body, body_len);
  s->len += 5ull + body_len;
  return ETL_OK;
}
int etl_stage_append_framed(etl_stager* s, const uint8_t* framed, uint64_t len) {
  uint64_t cap = s->cap & ~(1ull << 63);
  if (s->len + len > cap) return ETL_ERR_ALLOC;
  // validate the whole chain before anything is committed: a broken chain leaves the stager untouched
  uint64_t pos = 0;
  while (pos + 5 <= len) {
    if (framed[pos] != 'd') break;
    uint32_t fl = rd32(framed + pos + 1);
    if (fl < 4 || pos + 1ull + fl > len) break;
    pos += 1ull + fl;
  }
  if (pos != len) return ETL_ERR_INVALID_ARG;
  uint64_t base = s->len;
  memcpy(s->buf + base, framed, len);
  for (pos = 0; pos < len;) {
    uint32_t fl = rd32(framed + pos + 1);
    stage_note_frame(s, base + pos, framed + pos + 5, fl - 4);
    pos += 1ull + fl;
  }
  s->len += len;
  return ETL_OK;
}
int etl_stage_view(const etl_stager* cs, etl_dec_input* out) {
  etl_stager* s = const_cast<etl_stager*>(cs);
  // blocks k*stride past the last frame start have no frame: anchors[k] = len
  if (!s->padded) { s->n_real_anchors = s->anchors.size(); s->padded = true; }
  s->anchors.resize(s->n_real_anchors);
  const uint64_t want = s->len ? (s->len + s->stride - 1) / s->stride : 0;
  while (s->anchors.size() < want) s->anchors.push_back(s->len);
  memset(out, 0, sizeof *out);
  out->host_buf = s->buf;
  out->len = s->len;
  out->anchors = s->anchors.data();
  out->n_anchors = s->anchors.size();
  out->anchor_stride = s->stride;
  out->max_frame_len = s->max_frame;
  out->relation_offsets = s->relations.data();
  out->n_relations = s->relations.size();
  return ETL_OK;
}

// ------------------------------------------------------------------------------------------------ ctx
static void ctx_release(etl_dec_ctx* ctx) {
  for (DevBufBase* b : ctx->bufs) b->release();
  if (ctx->h_result) cudaFreeHost(ctx->h_result);
  if (ctx->h_up) cudaFreeHost(ctx->h_up);
  if (ctx->h_rel_x) cudaFreeHost(ctx->h_rel_x);
  if (ctx->h_seam) cudaFreeHost(ctx->h_seam);
  if (ctx->h_total) cudaFreeHost(ctx->h_total);
  if (ctx->h_scalars) cudaFreeHost(ctx->h_scalars);
  for (auto& e : ctx->ev) if (e) cudaEventDestroy(e);
  for (auto& e : ctx->evk) if (e) cudaEventDestroy(e);
  if (ctx->ev_in) cudaEventDestroy(ctx->ev_in);
  if (ctx->ev_l0) cudaEventDestroy(ctx->ev_l0);
  if (ctx->ev_l1) cudaEventDestroy(ctx->ev_l1);
  if (ctx->side) cudaStreamDestroy(ctx->side);
  if (ctx->own_stream && ctx->stream) cudaStreamDestroy(ctx->stream);
  if (ctx->comm && nccl_api().ok) nccl_api().CommDestroy(ctx->comm);
  delete ctx;
}
int etl_dec_create(int device_id, etl_dec_ctx** out) {
  if (!out) return ETL_ERR_INVALID_ARG;
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) { cudaGetLastError(); return ETL_ERR_NO_DEVICE; }
  if (device_id < 0 || device_id >= n) return ETL_ERR_INVALID_ARG;
  etl_dec_ctx* ctx = new etl_dec_ctx();
  ctx->device = device_id;
  bool ok = cudaSetDevice(device_id) == cudaSuccess;
  // the latency-bound chain runs at the highest priority, the HBM-bound side pass at the lowest: when both have CTAs
  // pending the scheduler places the chain's first
  int prio_lo = 0, prio_hi = 0;
  ok = ok && cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi) == cudaSuccess;
  ok = ok && cudaStreamCreateWithPriority(&ctx->stream, cudaStreamNonBlocking, prio_hi) == cudaSuccess;
  ctx->own_stream = ok;
  ok = ok && cudaStreamCreateWithPriority(&ctx->side, cudaStreamNonBlocking, prio_lo) == cudaSuccess;
  for (auto& e : ctx->ev) ok = ok && cudaEventCreate(&e) == cudaSuccess;
  for (auto& e : ctx->evk) ok = ok && cudaEventCreate(&e) == cudaSuccess;
  ok = ok && cudaEventCreateWithFlags(&ctx->ev_in, cudaEventDisableTiming) == cudaSuccess;
  ok = ok && cudaEventCreate(&ctx->ev_l0) == cudaSuccess && cudaEventCreate(&ctx->ev_l1) == cudaSuccess;
  ok = ok && cudaHostAlloc((void**)&ctx->h_total, sizeof(Summ), cudaHostAllocDefault) == cudaSuccess;
  ok = ok && cudaHostAlloc((void**)&ctx->h_scalars, kScalarBlockBytes, cudaHostAllocDefault) == cudaSuccess;
  ok = ok && ctx->d_scalars.ensure(kScalarBlockBytes) == cudaSuccess && ctx->d_total.ensure(1) == cudaSuccess;
  if (ok) ok = cudaFuncSetAttribute(k_rows, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kRowsSmemBytes) == cudaSuccess;
  if (ok) ok = cudaFuncSetAttribute(k_heavy, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kHeavySmemBytes) == cudaSuccess;
  if (!ok) { cudaGetLastError(); ctx_release(ctx); return ETL_ERR_CUDA; }
  // batch planes come from the stream-ordered pool: keep freed blocks for the next batch instead of returning them to the OS
  cudaMemPool_t pool;
  if (cudaDeviceGetDefaultMemPool(&pool, device_id) == cudaSuccess) {
    uint64_t thr = UINT64_MAX;
    cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr);
  }
  *out = ctx;
  return ETL_OK;
}
int etl_dec_set_stream(etl_dec_ctx* ctx, void* s) {
  if (!ctx) return ETL_ERR_INVALID_ARG;
  if (ctx->own_stream && ctx->stream) cudaStreamDestroy(ctx->stream);
  ctx->stream = (cudaStream_t)s;
  ctx->own_stream = false;
  return ETL_OK;
}
void etl_dec_destroy(etl_dec_ctx* ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  cudaStreamSynchronize(ctx->stream);
  cudaStreamSynchronize(ctx->side);
  if (trace_on() && ctx->tr_n)
    fprintf(stderr, "[etl trace] %llu decodes, mean us: prepare %.1f | enqueue %.1f | wait %.1f | results+d2h %.1f | summary %.1f\n",
            (unsigned long long)ctx->tr_n, ctx->tr[0] / ctx->tr_n, ctx->tr[1] / ctx->tr_n, ctx->tr[2] / ctx->tr_n, ctx->tr[3] / ctx->tr_n, ctx->tr[4] / ctx->tr_n);
  ctx_release(ctx);
}
const char* etl_dec_last_error(const etl_dec_ctx* ctx) { return ctx ? ctx->last_error.c_str() : "null ctx"; }

// ---- communicator over the GPUs of one box (one process per GPU): NCCL inside the library
int etl_dec_comm_unique_id(uint8_t* out, uint32_t cap) {
  if (!out || cap < sizeof(ncclUniqueId)) return ETL_ERR_INVALID_ARG;
  if (!nccl_api().ok) return ETL_ERR_INTERNAL;
  ncclUniqueId id;
  if (nccl_api().GetUniqueId(&id) != ncclSuccess) return ETL_ERR_CUDA;
  memset(out, 0, cap);
  memcpy(out, &id, sizeof id);
  return ETL_OK;
}
int etl_dec_comm_init(etl_dec_ctx* ctx, const uint8_t* unique_id, uint32_t id_bytes, int rank, int n_ranks) {
  if (!ctx || !unique_id || id_bytes < sizeof(ncclUniqueId) || n_ranks < 1 || rank < 0 || rank >= n_ranks) return ETL_ERR_INVALID_ARG;
  if (!nccl_api().ok) { ctx->last_error = "libnccl.so.2 could not be loaded"; return ETL_ERR_INTERNAL; }
  CK(cudaSetDevice(ctx->device));
  if (ctx->comm) { nccl_api().CommDestroy(ctx->comm); ctx->comm = nullptr; }
  ncclUniqueId id;
  memcpy(&id, unique_id, sizeof id);
  CKN(nccl_api().CommInitRank(&ctx->comm, n_ranks, id, rank));
  ctx->rank = rank; ctx->n_ranks = n_ranks;
  return ETL_OK;
}

int etl_dec_comm_init_host(etl_dec_ctx* ctx, int rank, int n_ranks, etl_host_allgather_fn fn, void* user) {
  if (!ctx || !fn || n_ranks < 1 || rank < 0 || rank >= n_ranks) return ETL_ERR_INVALID_ARG;
  if (ctx->comm && nccl_api().ok) { nccl_api().CommDestroy(ctx->comm); ctx->comm = nullptr; }
  ctx->host_allgather = fn; ctx->host_user = user;
  ctx->rank = rank; ctx->n_ranks = n_ranks;
  return ETL_OK;
}
// all-gather of `bytes` per rank from d_send into d_recv (n_ranks blocks) on the decode stream: NCCL, or through the host
static int ctx_allgather(etl_dec_ctx* ctx, const void* d_send, void* d_recv, size_t bytes) {
  cudaStream_t st = ctx->stream;
  if (!ctx->host_allgather) {
    CKN(nccl_api().AllGather(d_send, d_recv, bytes, ncclUint8, ctx->comm, st));
    return ETL_OK;
  }
  std::vector<uint8_t> hs(bytes), hr(bytes * (size_t)ctx->n_ranks);
  CK(cudaMemcpyAsync(hs.data(), d_send, bytes, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  if (ctx->host_allgather(ctx->host_user, hs.data(), hr.data(), bytes) != 0) { ctx->last_error = "host all-gather callback failed"; return ETL_ERR_INTERNAL; }
  CK(cudaMemcpyAsync(d_recv, hr.data(), hr.size(), cudaMemcpyHostToDevice, st));
  CK(cudaStreamSynchronize(st));                      // hr is a local
  return ETL_OK;
}

int etl_dec_put_table_schema(etl_dec_ctx* ctx, uint32_t table_id, uint64_t snapshot_id, const etl_column_schema* cols,
                             uint32_t n_cols) {
  if (!ctx || (n_cols && !cols)) return ETL_ERR_INVALID_ARG;
  StoredTable t;
  t.snapshot_id = snapshot_id;
  for (uint32_t i = 0; i < n_cols; i++) {
    StoredCol c;
    c.name = cols[i].name ? cols[i].name : "";
    c.type_oid = cols[i].type_oid; c.modifier = cols[i].modifier; c.ordinal = cols[i].ordinal_position;
    c.pk = cols[i].primary_key_ordinal_position; c.nullable = cols[i].nullable;
    t.cols.push_back(std::move(c));
  }
  ctx->tables[table_id] = std::move(t);
  return ETL_OK;
}
int etl_dec_reset_relations(etl_dec_ctx* ctx) {
  if (!ctx) return ETL_ERR_INVALID_ARG;
  ctx->current.clear();
  ctx->tables_valid = false;
  return ETL_OK;
}

// handle_relation_message (apply.rs:2012-2089): Relation body → masks → ReplicatedTableSchema.
// returns 0 ok, else etl_error_code; *seq receives the error step.
static uint32_t build_relation(etl_dec_ctx* ctx, const uint8_t* frame, uint64_t avail, uint64_t off, RelVersion* out,
                               uint32_t* seq) {
  *seq = 0;
  if (avail < 5 || frame[0] != 'd') return ETL_E_MALFORMED_FRAME;
  uint32_t fl = rd32(frame + 1);
  if (fl < 4 || 1ull + fl > avail) return ETL_E_MALFORMED_FRAME;
  const uint8_t* end = frame + 1 + fl;
  const uint8_t* p = frame + 31;  // after 'd' len 'w' hdr 'R'
  if (p + 4 > end) return ETL_E_MALFORMED_FRAME;
  uint32_t rel_id = rd32(p); p += 4;
  auto cstr = [&](const uint8_t** q) -> const uint8_t* {
    const uint8_t* s = *q;
    const uint8_t* z = (const uint8_t*)memchr(s, 0, (size_t)(end - s));
    if (!z) return nullptr;
    *q = z + 1;
    return s;
  };
  if (!cstr(&p) || !cstr(&p)) return ETL_E_MALFORMED_FRAME;
  if (p + 3 > end) return ETL_E_MALFORMED_FRAME;
  uint8_t replident = *p++;
  if (replident != 'd' && replident != 'n' && replident != 'f' && replident != 'i') return ETL_E_MALFORMED_FRAME;
  int16_t ncols = (int16_t)rd16(p); p += 2;
  struct RC { std::string name; uint8_t flags; };
  std::vector<RC> rcols;
  for (int i = 0; i < ncols; i++) {
    if (p + 1 > end) return ETL_E_MALFORMED_FRAME;
    uint8_t flags = *p++;
    const uint8_t* nm = cstr(&p);
    if (!nm) return ETL_E_MALFORMED_FRAME;
    size_t nl = (size_t)(p - 1 - nm);
    if (!utf8_ok(nm, nl)) return ETL_E_MALFORMED_FRAME;
    if (p + 8 > end) return ETL_E_MALFORMED_FRAME;
    p += 8;
    rcols.push_back(RC{std::string((const char*)nm, nl), flags});
  }
  *seq = 2;
  auto it = ctx->tables.find(rel_id);
  if (it == ctx->tables.end()) return ETL_E_MISSING_TABLE_SCHEMA;
  const StoredTable& t = it->second;
  std::vector<uint8_t> repl(t.cols.size(), 0), ident(t.cols.size(), 0);
  for (const RC& rc : rcols) {
    bool found = false;
    for (size_t k = 0; k < t.cols.size(); k++)
      if (t.cols[k].name == rc.name) {
        found = true; repl[k] = 1;
        if (replident == 'f' || (rc.flags & 1)) ident[k] = 1;  // event.rs:351-366
      }
    if (!found) return ETL_E_UNKNOWN_COLUMNS;                  // schema.rs:288-309
  }
  out->table_id = rel_id; out->snapshot_id = t.snapshot_id; out->effective_off = off; out->n_ident = 0;
  out->kind.clear(); out->flags.clear(); out->index.clear();
  for (size_t k = 0; k < t.cols.size(); k++) {
    if (!repl[k]) continue;
    out->kind.push_back((uint8_t)etl_oid_decode_class(t.cols[k].type_oid));
    out->flags.push_back((uint8_t)((t.cols[k].nullable ? 1 : 0) | (ident[k] ? 2 : 0)));
    out->index.push_back((int32_t)k);
    if (ident[k]) out->n_ident++;
  }
  return 0;
}

static void free_batch_blocks(etl_dec_batch* b) {
  if (!b) return;
  cudaStream_t st = b->ctx ? b->ctx->stream : nullptr;
  if (b->dev_block) cudaFreeAsync(b->dev_block, st);
  b->dev_block = nullptr; b->host_block = nullptr;
}
void etl_dec_batch_free(etl_dec_batch* b) {
  if (!b) return;
  free_batch_blocks(b);
  delete b;
}

// Where the structure-blind UTF-8 pass (k_utf8_dead, HBM-bound) runs relative to the latency-bound passes.
// 0: side stream from the start of the index pass; 1: side stream from the start of the tuple pass (default);
// 2 (default): main stream after the tuple pass; 3: inside k_rows — its warps stream the dead segments after their rows.
// Measured on C5 (10 GiB): 2 is the fastest, then 0, 1 and 3: k_rows fills the register file and
// is bound by instruction issue, the UTF-8 pass needs every SM's warps to saturate HBM — sharing the SMs helps neither.
// ETL_DEAD_MODE is a tuning knob for measurement, not part of the ABI.
static int dead_mode() {
  static const int m = getenv("ETL_DEAD_MODE") ? atoi(getenv("ETL_DEAD_MODE")) : 2;
  return m;
}
// No frame of the batch can hold a text value of kCoopLen bytes (the stager's max_frame_len says so): k_rows lists no
// long cell, and the passes that exist for them — the structure-blind UTF-8 pass over dead segments, k_long_cells, the
// line bitmap — are left out.  The hint is not trusted: should k_rows list a long cell after all, run_decode runs them.
static bool long_passes_skippable(const etl_dec_ctx* ctx) {
  return ctx->max_frame_hint && ctx->max_frame_hint < (uint32_t)kCoopLen && dead_mode() == 2;
}
static uint32_t dead_grid(const DecodeParams& P) {   // 8 warps per CTA, kDeadSegsPerWarp segments per warp; surplus CTAs return at once
  const uint64_t items = (uint64_t)P.n_anchors * (P.anchor_stride > 2048u ? P.anchor_stride / 2048u : 1u);
  return (uint32_t)((items + 8u * kDeadSegsPerWarp - 1u) / (8u * kDeadSegsPerWarp)) + 1u;
}
static int sm_count(etl_dec_ctx* ctx) {
  static int sms = 0;
  if (!sms) { sms = 132; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, ctx->device); }
  return sms;
}
static cudaError_t launch_dead_side(etl_dec_ctx* ctx, cudaStream_t st) {
  cudaError_t e;
  if ((e = cudaEventRecord(ctx->ev_in, st)) != cudaSuccess) return e;
  if ((e = cudaStreamWaitEvent(ctx->side, ctx->ev_in, 0)) != cudaSuccess) return e;
  if ((e = cudaEventRecord(ctx->ev_l0, ctx->side)) != cudaSuccess) return e;
  k_utf8_dead<<<dead_grid(ctx->P), 256, 0, ctx->side>>>(ctx->P);
  if ((e = cudaEventRecord(ctx->ev_l1, ctx->side)) != cudaSuccess) return e;
  ctx->launches += 1;
  ctx->lines_launched = true;
  return cudaSuccess;
}

static int ensure_pinned(etl_dec_ctx* ctx, uint8_t** p, size_t* cap, size_t want) {
  if (*cap >= want) return ETL_OK;
  if (*p) cudaFreeHost(*p);
  *p = nullptr; *cap = 0;
  size_t n = want + want / 2 + 4096;
  CK(cudaHostAlloc((void**)p, n, cudaHostAllocDefault));
  *cap = n;
  return ETL_OK;
}

// ---- relation-update exchange (SURVEY §8e): a Relation frame in shard r changes the decode state of every
// shard after it.  Each rank contributes the raw Relation frames of its byte range; every rank builds the
// versions announced by the ranks before it (they apply from its first byte) and — at the end of the batch —
// installs all of them, in stream order, as the state the next batch starts from (apply.rs:2079 note_ready,
// table_cache.rs:36-130).  One all-gather of `rel_slot` bytes per rank; the slot grows when a shard needs more.
static int exchange_relations(etl_dec_ctx* ctx, const etl_dec_input* in, std::vector<std::vector<uint8_t>>* frames_by_rank) {
  frames_by_rank->assign(ctx->n_ranks, {});
  cudaStream_t st = ctx->stream;
  for (;;) {
    const size_t slot = ctx->rel_slot;
    CK(ctx->d_rel_x.ensure(slot * (1 + (size_t)ctx->n_ranks)));
    if (int rc = ensure_pinned(ctx, &ctx->h_rel_x, &ctx->h_rel_x_cap, slot * (1 + (size_t)ctx->n_ranks))) return rc;
    // slot: u64 payload bytes needed | u64 frames | frames back to back
    uint8_t* s = ctx->h_rel_x;
    uint64_t need = 16, nf = 0;
    for (uint64_t i = 0; i < in->n_relations; i++) {
      const uint64_t off = in->relation_offsets[i];
      if (off + 5 > in->len) continue;
      const uint64_t fl = 1ull + rd32(in->host_buf + off + 1);
      if (off + fl > in->len) continue;
      if (need + fl <= slot) memcpy(s + need, in->host_buf + off, fl);
      need += fl; nf++;
    }
    memcpy(s, &need, 8); memcpy(s + 8, &nf, 8);
    CK(cudaMemcpyAsync(ctx->d_rel_x.ptr(), s, std::min<uint64_t>(need, slot), cudaMemcpyHostToDevice, st));
    if (int rc = ctx_allgather(ctx, ctx->d_rel_x.ptr(), ctx->d_rel_x.ptr() + slot, slot)) return rc;
    CK(cudaMemcpyAsync(ctx->h_rel_x + slot, ctx->d_rel_x.ptr() + slot, slot * ctx->n_ranks, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    uint64_t max_need = 0;
    for (int r = 0; r < ctx->n_ranks; r++) { uint64_t v; memcpy(&v, ctx->h_rel_x + slot * (1 + r), 8); max_need = std::max(max_need, v); }
    if (max_need > slot) { ctx->rel_slot = (size_t)(max_need * 2); continue; }   // every rank sees the same sizes: all retry together
    for (int r = 0; r < ctx->n_ranks; r++) {
      const uint8_t* q = ctx->h_rel_x + slot * (1 + r);
      uint64_t v; memcpy(&v, q, 8);
      (*frames_by_rank)[r].assign(q + 16, q + v);
    }
    return ETL_OK;
  }
}

// ---------------------------------------------------------------- phase 0: everything known before a kernel runs
static int prepare(etl_dec_ctx* ctx, const etl_dec_input* in, uint32_t flags, bool sharded) {
  ctx->pending = false;
  const uint32_t stride = in->anchor_stride;
  if (stride < 256 || stride > 32768 || (stride & (stride - 1))) { ctx->last_error = "anchor_stride must be a power of two in [256, 32768]"; return ETL_ERR_INVALID_ARG; }
  if (in->len && (!in->host_buf && !in->dev_buf)) { ctx->last_error = "no input buffer"; return ETL_ERR_INVALID_ARG; }
  if (in->dev_buf && (reinterpret_cast<uintptr_t>(in->dev_buf) & 15u)) { ctx->last_error = "dev_buf must be 16-byte aligned"; return ETL_ERR_INVALID_ARG; }
  if (in->len >= (1ull << 40)) { ctx->last_error = "a staged batch is limited to 1 TiB"; return ETL_ERR_INVALID_ARG; }
  const uint64_t n_anchors_expected = in->len ? (in->len + stride - 1) / stride : 0;
  if (in->n_anchors != n_anchors_expected || (in->n_anchors && !in->anchors && !in->dev_anchors)) { ctx->last_error = "anchors: expected ceil(len/stride) entries"; return ETL_ERR_INVALID_ARG; }
  if (in->n_relations && (!in->relation_offsets || !in->host_buf)) { ctx->last_error = "relation_offsets require host_buf"; return ETL_ERR_INVALID_ARG; }
  if (sharded && !ctx->comm && !ctx->host_allgather) { ctx->last_error = "sharded decode needs etl_dec_comm_init / etl_dec_comm_init_host"; return ETL_ERR_INVALID_ARG; }
  CK(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  ctx->launches = 0;
  ctx->pending_flags = flags;
  ctx->pending_installs.clear();
  ctx->foreign_installs.clear();

  // ---- schema versions of this batch: carried-in (ascending table id), versions announced by earlier shards,
  // then this range's Relation frames in order
  std::vector<RelVersion> vers;
  std::map<uint32_t, RelVersion> base = ctx->current;
  if (sharded) {
    std::vector<std::vector<uint8_t>> frames;
    if (int rc = exchange_relations(ctx, in, &frames)) return rc;
    for (int r = 0; r < ctx->n_ranks; r++) {
      if (r == ctx->rank) continue;
      const std::vector<uint8_t>& fb = frames[r];
      for (size_t pos = 0; pos + 5 <= fb.size();) {
        const size_t fl = 1 + (size_t)rd32(fb.data() + pos + 1);
        RelVersion v; uint32_t seq = 0;
        if (build_relation(ctx, fb.data() + pos, fb.size() - pos, 0, &v, &seq) == 0) {
          if (r < ctx->rank) base[v.table_id] = v;               // applies from this shard's first byte
          ctx->foreign_installs.push_back(std::move(v));         // and is part of the state after the batch
          if (r > ctx->rank) ctx->foreign_installs.back().effective_off = 1;   // marker: after this shard
        }
        pos += fl;
      }
    }
  }
  const bool reuse_tables = ctx->tables_valid && in->n_relations == 0 && !sharded;
  for (auto& kv : base) { RelVersion v = kv.second; v.effective_off = 0; vers.push_back(std::move(v)); }
  std::vector<uint64_t> rel_err_off; std::vector<uint32_t> rel_err_code, rel_err_seq;
  for (uint64_t i = 0; i < in->n_relations; i++) {
    uint64_t off = in->relation_offsets[i];
    if (off >= in->len) { ctx->last_error = "relation offset out of range"; return ETL_ERR_INVALID_ARG; }
    RelVersion v; uint32_t seq = 0;
    uint32_t code = build_relation(ctx, in->host_buf + off, in->len - off, off, &v, &seq);
    if (code) { rel_err_off.push_back(off); rel_err_code.push_back(code); rel_err_seq.push_back(seq); continue; }
    ctx->pending_installs.emplace_back(off, v);   // note_ready (apply.rs:2079) happens in finish, for the valid prefix only
    vers.push_back(std::move(v));
  }
  for (const RelVersion& v : vers)
    for (uint8_t k : v.kind)
      if (!kind_supported_on_device(k)) {
        char msg[160];
        snprintf(msg, sizeof msg, "table %u: column decode class 0x%x has no device parser; refusing to decode", v.table_id, k);
        ctx->last_error = msg;
        return ETL_ERR_INVALID_ARG;
      }

  // ---- geometry
  DecodeParams& P = ctx->P;
  const void* keep_tables[6] = {P.schemas, P.schema_by_batch, P.col_kind, P.col_flags, P.rel_error_off, P.rel_error_code};
  const void* keep_seq = P.rel_error_seq;
  const uint32_t keep_counts[3] = {P.n_schemas, P.n_batch_schemas, P.n_bins};
  memset(&P, 0, sizeof P);
  P.len = in->len;
  P.n_anchors = (uint32_t)in->n_anchors;
  P.anchor_stride = stride;
  ctx->max_frame_hint = in->max_frame_len;

  // ---- uploads
  CK(cudaEventRecord(ctx->ev[0], st));
  ctx->pending_h2d_bytes = (in->dev_buf ? 0 : in->len) + (in->dev_anchors ? 0 : (in->n_anchors + 1) * 8) + kScalarBlockBytes;
  if (in->dev_buf) P.buf = in->dev_buf;
  else {
    CK(ctx->d_stream.ensure(in->len + 64));
    if (in->len) CK(cudaMemcpyAsync(ctx->d_stream.ptr(), in->host_buf, in->len, cudaMemcpyHostToDevice, st));
    CK(cudaMemsetAsync(ctx->d_stream.ptr() + in->len, 0, 64, st));
    P.buf = ctx->d_stream.ptr();
  }
  if (in->dev_anchors) P.anchors = in->dev_anchors;
  else {
    CK(ctx->d_anchors.ensure(in->n_anchors + 1));
    if (in->n_anchors) CK(cudaMemcpyAsync(ctx->d_anchors.ptr(), in->anchors, in->n_anchors * 8, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(ctx->d_anchors.ptr() + in->n_anchors, &in->len, 8, cudaMemcpyHostToDevice, st));
    P.anchors = ctx->d_anchors.ptr();
  }
  if (reuse_tables) {
    P.schemas = (const DevSchema*)keep_tables[0]; P.schema_by_batch = (const uint32_t*)keep_tables[1];
    P.col_kind = (const uint8_t*)keep_tables[2]; P.col_flags = (const uint8_t*)keep_tables[3];
    P.rel_error_off = (const uint64_t*)keep_tables[4]; P.rel_error_code = (const uint32_t*)keep_tables[5]; P.rel_error_seq = (const uint32_t*)keep_seq;
    P.n_schemas = keep_counts[0]; P.n_batch_schemas = keep_counts[1]; P.n_bins = keep_counts[2];
    P.n_rel_errors = 0;
  } else {
    // device tables sorted by (table_id, effective_off); versions with identical columns share a layout (shape bins)
    std::vector<uint32_t> order(vers.size());
    for (uint32_t i = 0; i < order.size(); i++) order[i] = i;
    std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) {
      if (vers[a].table_id != vers[b].table_id) return vers[a].table_id < vers[b].table_id;
      return vers[a].effective_off < vers[b].effective_off;
    });
    std::map<std::pair<std::vector<uint8_t>, std::vector<uint8_t>>, uint32_t> layouts;
    std::vector<DevSchema> ds; std::vector<uint8_t> ck, cf;
    for (uint32_t oi : order) {
      const RelVersion& v = vers[oi];
      DevSchema d{};
      d.table_id = v.table_id; d.n_cols = (uint32_t)v.kind.size(); d.n_ident = v.n_ident; d.col_base = (uint32_t)ck.size();
      d.effective_off = v.effective_off; d.batch_index = oi; d.has_heap = 0;
      for (uint8_t k : v.kind) if (kind_has_heap(k)) d.has_heap = 1;
      auto key = std::make_pair(v.kind, v.flags);
      auto it = layouts.find(key);
      if (it == layouts.end()) it = layouts.emplace(std::move(key), (uint32_t)layouts.size()).first;
      d.layout = it->second;
      ck.insert(ck.end(), v.kind.begin(), v.kind.end());
      cf.insert(cf.end(), v.flags.begin(), v.flags.end());
      ds.push_back(d);
    }
    ctx->n_layouts = std::max<size_t>(1, layouts.size());
    std::vector<uint32_t> sbb(ds.size() + 1, 0);
    for (uint32_t i = 0; i < ds.size(); i++) sbb[ds[i].batch_index] = i;
    auto al16 = [](size_t x) { return (x + 15) & ~(size_t)15; };
    const size_t o_ds = 0, o_sbb = al16(o_ds + (ds.size() + 1) * sizeof(DevSchema)), o_ck = al16(o_sbb + sbb.size() * 4),
                 o_cf = al16(o_ck + ck.size() + 1), o_eo = al16(o_cf + cf.size() + 1), o_ec = al16(o_eo + (rel_err_off.size() + 1) * 8),
                 o_es = al16(o_ec + (rel_err_off.size() + 1) * 4), total = al16(o_es + (rel_err_off.size() + 1) * 4);
    if (int rc = ensure_pinned(ctx, &ctx->h_up, &ctx->h_up_cap, total)) return rc;
    CK(ctx->d_tables.ensure(total));
    uint8_t* h = ctx->h_up;
    if (!ds.empty()) memcpy(h + o_ds, ds.data(), ds.size() * sizeof(DevSchema));
    memcpy(h + o_sbb, sbb.data(), sbb.size() * 4);
    if (!ck.empty()) { memcpy(h + o_ck, ck.data(), ck.size()); memcpy(h + o_cf, cf.data(), cf.size()); }
    if (!rel_err_off.empty()) {
      memcpy(h + o_eo, rel_err_off.data(), rel_err_off.size() * 8);
      memcpy(h + o_ec, rel_err_code.data(), rel_err_code.size() * 4);
      memcpy(h + o_es, rel_err_seq.data(), rel_err_seq.size() * 4);
    }
    CK(cudaMemcpyAsync(ctx->d_tables.ptr(), h, total, cudaMemcpyHostToDevice, st));   // h_up is not reused before the final sync
    ctx->pending_h2d_bytes += total;
    uint8_t* d = ctx->d_tables.ptr();
    P.schemas = (const DevSchema*)(d + o_ds); P.schema_by_batch = (const uint32_t*)(d + o_sbb);
    P.col_kind = d + o_ck; P.col_flags = d + o_cf;
    P.rel_error_off = (const uint64_t*)(d + o_eo); P.rel_error_code = (const uint32_t*)(d + o_ec); P.rel_error_seq = (const uint32_t*)(d + o_es);
    P.n_schemas = (uint32_t)ds.size(); P.n_rel_errors = (uint32_t)rel_err_off.size();
    P.n_batch_schemas = (uint32_t)vers.size();
    P.n_bins = (uint32_t)std::min<size_t>(kMaxBins, 16 * ctx->n_layouts);
    ctx->tables_valid = in->n_relations == 0 && !sharded;   // built from `current` alone: valid until a Relation arrives
  }
  CK(ctx->d_seg_rec_base.ensure(P.n_anchors + 1));
  CK(ctx->d_chase_status.ensure_zeroed((P.n_anchors + kChaseThreads - 1) / kChaseThreads + 1, st));
  P.seg_rec_base = ctx->d_seg_rec_base.ptr(); P.chase_status = ctx->d_chase_status.ptr();
  if (sharded) { CK(ctx->d_chase_summ.ensure((P.n_anchors + kChaseThreads - 1) / kChaseThreads + 1)); P.chase_summ = ctx->d_chase_summ.ptr(); }
  const size_t line_words = (in->len + 4095) / 4096 + 1;
  CK(ctx->d_line_bad.ensure(line_words)); CK(ctx->d_dead.ensure(P.n_anchors + 1));
  P.line_bad = ctx->d_line_bad.ptr(); P.dead = ctx->d_dead.ptr();
  P.long_cap = (uint32_t)(in->len / 512) + 16;        // every listed cell is at least kCoopLen (512) bytes long
  CK(ctx->d_long.ensure(P.long_cap));
  unsigned long long* sc = reinterpret_cast<unsigned long long*>(ctx->d_scalars.ptr());
  P.long_cells = ctx->d_long.ptr(); P.long_count = (unsigned int*)(sc + 7);
  P.total = ctx->d_total.ptr();
  P.first_error = sc; P.metrics = sc + 1;
  P.heap_top = sc + 5; P.heap_overflow = (unsigned int*)(sc + 9); P.arr_top = sc + 10;
  P.perm_len = (unsigned int*)(sc + 11); P.n_act = (unsigned int*)(sc + 12); P.abort_flag = (unsigned int*)(sc + 13);
  P.n_frames = (unsigned int*)(sc + 14); P.chase_done = (unsigned int*)(sc + 15);
  P.copy_count = (unsigned int*)(sc + 8);
  P.dc = reinterpret_cast<const DevCarry*>(sc + kScalarWords); P.dc_out = reinterpret_cast<DevCarry*>(sc + kScalarWords);
  const uint32_t act_blocks = (P.n_anchors + kActThreads - 1) / kActThreads;
  CK(ctx->d_act.ensure(P.n_anchors + 1)); CK(ctx->d_act_blk.ensure(act_blocks + 1));
  P.act = ctx->d_act.ptr(); P.act_blk = ctx->d_act_blk.ptr();
  CK(ctx->d_bin_count.ensure(kMaxBins)); CK(ctx->d_bin_cursor.ensure(kMaxBins));
  P.bin_count = ctx->d_bin_count.ptr(); P.bin_cursor = ctx->d_bin_cursor.ptr();
  P.rank = (uint32_t)ctx->rank; P.n_ranks = sharded ? (uint32_t)ctx->n_ranks : 1u;
  if (sharded) {
    CK(ctx->d_seam.ensure(1 + (size_t)ctx->n_ranks));
    P.seam_send = ctx->d_seam.ptr(); P.seam_all = ctx->d_seam.ptr() + 1;
  }
  if (!long_passes_skippable(ctx)) CK(cudaMemsetAsync(P.line_bad, 0, line_words * 4, st));
  ctx->pending_schemas = std::move(vers);
  ctx->lines_launched = false;
  return ETL_OK;
}

// scalars [lo, hi) ← initial values (+ the carry block when `with_carry`)
static int upload_scalars(etl_dec_ctx* ctx, size_t lo, size_t hi, const DevCarry* carry) {
  unsigned long long* h = ctx->h_scalars;
  for (size_t i = lo; i < hi; i++) h[i] = 0;
  if (lo == 0) h[0] = ~0ull;
  size_t bytes = (hi - lo) * 8;
  if (carry) { memcpy(h + kScalarWords, carry, sizeof *carry); bytes = (kScalarWords - lo) * 8 + sizeof *carry; }
  CK(cudaMemcpyAsync(ctx->d_scalars.ptr() + lo * 8, h + lo, bytes, cudaMemcpyHostToDevice, ctx->stream));
  return ETL_OK;
}

// ---------------------------------------------------------------- pass A: live segments, frame offsets
static uint32_t next_epoch(etl_dec_ctx* ctx) {
  if (ctx->scan_epoch >= (1u << 30) - 2u) {          // the status words hold 30 bits of epoch: start over on zeroed words
    if (ctx->d_chase_status.p) cudaMemsetAsync(ctx->d_chase_status.p, 0, ctx->d_chase_status.cap_bytes, ctx->stream);
    if (ctx->d_scan_status.p) cudaMemsetAsync(ctx->d_scan_status.p, 0, ctx->d_scan_status.cap_bytes, ctx->stream);
    ctx->scan_epoch = 0;
  }
  return ++ctx->scan_epoch;
}
// scratch of the record-parallel passes for up to `cap` frames
static int ensure_record_scratch(etl_dec_ctx* ctx, uint64_t cap) {
  DecodeParams& P = ctx->P;
  const size_t nb = (size_t)((cap + kRecThreads - 1) / kRecThreads) + 1;
  CK(ctx->d_frame_off.ensure(cap + 1));
  CK(ctx->d_scan_status.ensure_zeroed(nb, ctx->stream));
  CK(ctx->d_scan_slots.ensure(nb));
  P.frame_off = ctx->d_frame_off.ptr(); P.frame_cap = cap;
  P.scan_status = ctx->d_scan_status.ptr(); P.scan_slots = ctx->d_scan_slots.ptr();
  return ETL_OK;
}
// seam: a shard on the optimistic path — the walk also folds the frames' effect on the stream state and writes the seam block
static void launch_chase(etl_dec_ctx* ctx, uint32_t mode, bool seam = false) {
  DecodeParams& P = ctx->P;
  if (mode & 1u) P.scan_epoch = next_epoch(ctx);
  const uint32_t grid = (P.n_anchors + kChaseThreads - 1) / kChaseThreads;
  if (seam) k_chase<true><<<grid, kChaseThreads, 0, ctx->stream>>>(P, mode);
  else k_chase<false><<<grid, kChaseThreads, 0, ctx->stream>>>(P, mode);
  ctx->launches += 1;
}
// totals only (FULL = false) or the record plane (FULL = true); `n_max` bounds the number of frames
static void launch_records(etl_dec_ctx* ctx, bool full, uint64_t n_max) {
  DecodeParams& P = ctx->P;
  P.scan_epoch = next_epoch(ctx);
  const uint32_t grid = (uint32_t)std::max<uint64_t>(1, (n_max + kRecThreads - 1) / kRecThreads);
  if (full) k_records<true><<<grid, kRecCtaThreads, 0, ctx->stream>>>(P);
  else k_records<false><<<grid, kRecCtaThreads, 0, ctx->stream>>>(P);
  ctx->launches += 1;
}
// Optimistic (exact = false): the offset scratch is sized by the caller; one launch counts, scans and writes.
// Exact: count, read the count back, size the scratch, write.
static int launch_index(etl_dec_ctx* ctx, bool exact) {
  DecodeParams& P = ctx->P;
  cudaStream_t st = ctx->stream;
  CK(cudaEventRecord(ctx->ev[1], st));
  if (P.n_anchors) {
    if (P.n_anchors <= kActSmallSegs) { k_act_small<<<1, kActThreads, 0, st>>>(P); ctx->launches += 1; }
    else {
      const uint32_t act_blocks = (P.n_anchors + kActThreads - 1) / kActThreads;
      k_act_count<<<act_blocks, kActThreads, 0, st>>>(P);
      k_act_scan<<<1, kActThreads, 0, st>>>(P, act_blocks);
      k_act_scatter<<<act_blocks, kActThreads, 0, st>>>(P);
      ctx->launches += 3;
    }
    if (dead_mode() == 0) CK(launch_dead_side(ctx, st));   // underneath everything that follows (needs only the dead-segment list)
    if (!exact) launch_chase(ctx, 3u, P.seam_send != nullptr);
    else {
      P.frame_cap = ~0ull;
      launch_chase(ctx, 1u);
      CK(cudaMemcpyAsync(ctx->h_scalars + 14, ctx->d_scalars.ptr() + 14 * 8, 8, cudaMemcpyDeviceToHost, st));
      CK(cudaStreamSynchronize(st));
      if (int rc = ensure_record_scratch(ctx, (uint32_t)ctx->h_scalars[14])) return rc;
      launch_chase(ctx, 2u);
    }
    CK(cudaGetLastError());
  } else if (int rc = ensure_record_scratch(ctx, 0)) return rc;
  CK(cudaEventRecord(ctx->ev[2], st));
  return ETL_OK;
}
// exact totals of the batch (P.total, the seam block) without planes: a SUMMARY pass with unlimited capacities
static int launch_summary(etl_dec_ctx* ctx) {
  DecodeParams& P = ctx->P;
  const uint64_t keep_r = P.cap_records, keep_c = P.cap_cells;
  P.cap_records = ~0ull; P.cap_cells = ~0ull;
  launch_records(ctx, false, P.frame_cap);
  P.cap_records = keep_r; P.cap_cells = keep_c;
  CK(cudaGetLastError());
  return ETL_OK;
}

struct PlaneLayout { uint64_t rec_off, kind, flags, rel, schema, start, commit, ord, cbase, tb, hint, tag, val, aux, heap, total; };
static PlaneLayout plane_layout(uint64_t nr, uint64_t nc, uint64_t nh) {
  PlaneLayout L;
  uint64_t cur = 0;
  auto take = [&](uint64_t bytes) { uint64_t o = cur; cur += (bytes + 255) & ~255ull; return o; };
  L.rec_off = take(nr * 8); L.kind = take(nr); L.flags = take(nr); L.rel = take(nr * 4); L.schema = take(nr * 4);
  L.start = take(nr * 8); L.commit = take(nr * 8); L.ord = take(nr * 8); L.cbase = take((nr + 1) * 8);
  L.tb = take(nr * 4); L.hint = take(nr * 4);
  L.tag = take(nc); L.val = take(nc * 8); L.aux = take(nc * 4); L.heap = take(nh);
  L.total = cur ? cur : 256;
  return L;
}
static void fill_planes(etl_dec_planes& pl, uint8_t* bs, const PlaneLayout& L, uint64_t nr, uint64_t nc, uint64_t nh) {
  pl.n_records = nr; pl.n_cells = nc; pl.heap_bytes = nh;
  pl.rec_off = (uint64_t*)(bs + L.rec_off); pl.rec_kind = bs + L.kind; pl.rec_flags = bs + L.flags;
  pl.rec_rel = (uint32_t*)(bs + L.rel); pl.rec_schema = (int32_t*)(bs + L.schema); pl.rec_start_lsn = (uint64_t*)(bs + L.start);
  pl.rec_commit_lsn = (uint64_t*)(bs + L.commit); pl.rec_tx_ordinal = (uint64_t*)(bs + L.ord); pl.rec_cell_base = (uint64_t*)(bs + L.cbase);
  pl.rec_tuple_bytes = (uint32_t*)(bs + L.tb); pl.rec_heap_hint = (uint32_t*)(bs + L.hint);
  pl.cell_tag = bs + L.tag; pl.cell_val = (uint64_t*)(bs + L.val); pl.cell_aux = (uint32_t*)(bs + L.aux); pl.heap = bs + L.heap;
}

// ---------------------------------------------------------------- pass C into planes of capacity (cap_r, cap_c)
static int launch_emit(etl_dec_ctx* ctx, etl_dec_batch* b, uint64_t cap_r, uint64_t cap_c, uint64_t array_heap, PlaneLayout* Lout, uint64_t* scalar_heap_out) {
  DecodeParams& P = ctx->P;
  cudaStream_t st = ctx->stream;
  bool any_heap = false, any_array = false;
  for (const RelVersion& v : b->schemas) for (uint8_t k : v.kind) { any_heap = any_heap || kind_has_heap(k); any_array = any_array || (k & ETL_K_ARRAY); }
  // upper bound on Σ cell_heap_bound: numeric ≤ n/2+19, bytea ≤ n/2+7, uuid = 16 per decoded text cell.
  // Arrays reserve 16 + 44·n_elems + 1.5·len per cell: first guess 3·len, retried ×4 on overflow (≤ 48·len).
  uint64_t nh = any_heap ? (P.len / 2 + 24 * cap_c + 256) : 0;
  nh = (nh + 15) & ~15ull;
  *scalar_heap_out = nh;
  if (any_array) nh += array_heap ? array_heap : 3 * P.len + 4096;
  const PlaneLayout L = plane_layout(cap_r, cap_c, nh);
  *Lout = L;
  b->block_bytes = L.total;
  CK(cudaMallocAsync(&b->dev_block, b->block_bytes, st));
  fill_planes(b->dev, (uint8_t*)b->dev_block, L, cap_r, cap_c, nh);
  P.rec_off = (uint64_t*)b->dev.rec_off; P.rec_kind = (uint8_t*)b->dev.rec_kind; P.rec_flags = (uint8_t*)b->dev.rec_flags;
  P.rec_rel = (uint32_t*)b->dev.rec_rel; P.rec_schema = (int32_t*)b->dev.rec_schema; P.rec_start_lsn = (uint64_t*)b->dev.rec_start_lsn;
  P.rec_commit_lsn = (uint64_t*)b->dev.rec_commit_lsn; P.rec_tx_ordinal = (uint64_t*)b->dev.rec_tx_ordinal;
  P.rec_cell_base = (uint64_t*)b->dev.rec_cell_base; P.rec_tuple_bytes = (uint32_t*)b->dev.rec_tuple_bytes; P.rec_heap_hint = (uint32_t*)b->dev.rec_heap_hint;
  P.cell_tag = (uint8_t*)b->dev.cell_tag; P.cell_val = (uint64_t*)b->dev.cell_val;
  P.cell_aux = (uint32_t*)b->dev.cell_aux; P.heap = (uint8_t*)b->dev.heap;
  P.heap_cap = nh; P.arr_base = *scalar_heap_out;
  P.cap_records = cap_r; P.cap_cells = cap_c;
  const size_t perm_cap = cap_r + 32ull * P.n_bins + 256;
  CK(ctx->d_perm.ensure(perm_cap)); CK(ctx->d_rec_flen.ensure(cap_r + 1));
  P.perm = ctx->d_perm.ptr(); P.rec_flen = ctx->d_rec_flen.ptr();
  return ETL_OK;
}
static int launch_emit_kernels(etl_dec_ctx* ctx) {
  DecodeParams& P = ctx->P;
  cudaStream_t st = ctx->stream;
  const uint64_t cap_r = P.cap_records;
  const size_t perm_cap = cap_r + 32ull * P.n_bins + 256;
  CK(cudaEventRecord(ctx->ev[3], st));
  CK(cudaMemsetAsync(P.bin_count, 0, P.n_bins * 4, st));
  // k_heavy / k_fix read every cell tag: a record that failed leaves cells unwritten, and a stale tag must not look pending
  if (P.cap_cells) CK(cudaMemsetAsync(P.cell_tag, 0, P.cap_cells, st));
  ctx->long_skipped = long_passes_skippable(ctx);
  if (P.n_anchors) {
    launch_records(ctx, true, cap_r);
    cudaEventRecord(ctx->evk[0], st);
    if (dead_mode() == 1 && !ctx->lines_launched) CK(launch_dead_side(ctx, st));   // underneath the tuple pass
    P.dead_in_rows = (dead_mode() == 3 && cap_r) ? 1u : 0u;
    if (cap_r) {
      k_bin_scan<<<1, 1024, 0, st>>>(P);
      k_perm<<<(uint32_t)((cap_r + kPermThreads - 1) / kPermThreads), kPermThreads, 0, st>>>(P);
      cudaEventRecord(ctx->evk[2], st);
      const uint32_t chunks = (uint32_t)((perm_cap + kRowsThreads - 1) / kRowsThreads);
      k_rows<<<((chunks + 63u) / 64u) * 64u, kRowsThreads, kRowsSmemBytes, st>>>(P);
      k_heavy<<<std::min<uint32_t>((uint32_t)((P.cap_cells + kHeavyTile - 1) / kHeavyTile) + 1u, (uint32_t)sm_count(ctx) * 3u), kHeavyThreads, kHeavySmemBytes, st>>>(P);
      k_fix<<<sm_count(ctx) * 2, 256, 0, st>>>(P);
      ctx->launches += 5;
    } else cudaEventRecord(ctx->evk[2], st);
    cudaEventRecord(ctx->evk[1], st);
    if (ctx->lines_launched) CK(cudaStreamWaitEvent(st, ctx->ev_l1, 0));   // join: the bitmap is complete
    else if (P.dead_in_rows) { cudaEventRecord(ctx->ev_l0, st); cudaEventRecord(ctx->ev_l1, st); }   // done by k_rows
    else if (ctx->long_skipped) { cudaEventRecord(ctx->ev_l0, st); cudaEventRecord(ctx->ev_l1, st); }
    else {                                            // ETL_DEAD_MODE=2 (or a batch without DML records): the same pass on the main stream
      cudaEventRecord(ctx->ev_l0, st);
      k_utf8_dead<<<dead_grid(P), 256, 0, st>>>(P);
      cudaEventRecord(ctx->ev_l1, st);
      ctx->launches += 1;
    }
    cudaEventRecord(ctx->evk[3], st);
    if (cap_r && !ctx->long_skipped) { k_long_cells<<<sm_count(ctx) * 8, 256, 0, st>>>(P); ctx->launches += 1; }
    CK(cudaGetLastError());
  } else {
    // an empty batch: no k_records writes rec_cell_base[0] (the planes come from the pool, not zeroed)
    CK(cudaMemsetAsync(P.total, 0, sizeof(Summ), st)); CK(cudaMemsetAsync(P.rec_cell_base, 0, 8, st));
    cudaEventRecord(ctx->evk[0], st); cudaEventRecord(ctx->evk[2], st); cudaEventRecord(ctx->evk[1], st); cudaEventRecord(ctx->evk[3], st); cudaEventRecord(ctx->ev_l0, st); cudaEventRecord(ctx->ev_l1, st); }
  CK(cudaEventRecord(ctx->ev[4], st));
  CK(cudaMemcpyAsync(ctx->h_scalars, ctx->d_scalars.ptr(), kScalarWords * 8, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(ctx->h_total, P.total, sizeof(Summ), cudaMemcpyDeviceToHost, st));
  if (P.seam_all && P.n_ranks > 1) {                  // every rank's totals: the host needs them for the carry-out (and the poison check)
    if (int rc = ensure_pinned(ctx, &ctx->h_seam, &ctx->h_seam_cap, sizeof(SeamBlock) * P.n_ranks)) return rc;
    CK(cudaMemcpyAsync(ctx->h_seam, P.seam_all, sizeof(SeamBlock) * P.n_ranks, cudaMemcpyDeviceToHost, st));
  }
  return ETL_OK;
}

static Summ carry_of(const etl_stream_state* cin) {
  Summ carry = summ_identity();
  if (cin) {
    if (cin->in_tx) carry.flags = S_HAS_B;
    // final_lsn of the last Begin passes through a batch without one even outside a transaction (only read while
    // in_tx): a batch of keepalives hands on the carry it received, as one decode of the joined batches would
    carry.lsn = cin->final_lsn;
    carry.ord = cin->next_tx_ordinal;
  }
  return carry;
}

// one decode, common to every entry point.  mode 0: one-shot (optimistic sizing); 1: after decode_begin (totals known).
// `sizing`: ETL_SIZING_* bits of an abandoned attempt (scratch restart), reported together with this one's
static int run_decode(etl_dec_ctx* ctx, const etl_stream_state* carry_in, uint64_t record_index_base, bool sharded, bool totals_known,
                      etl_dec_batch** out, bool force_exact = false, uint32_t sizing = 0) {
  cudaStream_t st = ctx->stream;
  DecodeParams& P = ctx->P;
  etl_dec_batch* b = new etl_dec_batch();
  b->ctx = ctx;
  b->schemas = ctx->pending_schemas;
  auto fail = [&](int rc) { if (b->dev_block) cudaFreeAsync(b->dev_block, st); delete b; return rc; };
#define CKB(call) do { cudaError_t _e = (call); if (_e != cudaSuccess) { ctx->last_error = std::string(#call) + ": " + cudaGetErrorString(_e); return fail(ETL_ERR_CUDA); } } while (0)
  const Summ host_carry = carry_of(carry_in);
  P.host_carry = host_carry;
  DevCarry dc; dc.carry = host_carry; dc.record_index_base = record_index_base;
  auto reset_abort = [&]() -> cudaError_t {
    ctx->h_scalars[13] = 0;
    return cudaMemcpyAsync(ctx->d_scalars.ptr() + 13 * 8, ctx->h_scalars + 13, 8, cudaMemcpyHostToDevice, st);
  };

  uint64_t cap_r = 0, cap_c = 0;
  bool exact = totals_known;
  if (!totals_known) {
    if (int rc = upload_scalars(ctx, 0, kScalarWords, &dc)) return fail(rc);
    // optimistic sizes from what earlier batches needed per byte; the first batch has no history: exact path
    if (ctx->rec_per_byte > 0 && !force_exact) {
      cap_r = (uint64_t)(P.len * ctx->rec_per_byte * 1.08) + 4096;
      cap_c = (uint64_t)(P.len * ctx->cells_per_byte * 1.08) + 16384;
    } else exact = true;
    P.cap_records = exact ? ~0ull : cap_r; P.cap_cells = exact ? ~0ull : cap_c;   // k_chase / k_records decide with these
    P.rec_cell_base = nullptr;
  } else {
    if (int rc = upload_scalars(ctx, 0, 12, nullptr)) return fail(rc);           // [12] n_act, [14] n_frames survive from decode_begin
    CKB(reset_abort());
    memcpy(ctx->h_scalars + kScalarWords, &dc, sizeof dc);
    CKB(cudaMemcpyAsync(ctx->d_scalars.ptr() + kScalarWords * 8, ctx->h_scalars + kScalarWords, sizeof dc, cudaMemcpyHostToDevice, st));
  }
  sizing |= exact ? ETL_SIZING_EXACT : ETL_SIZING_OPTIMISTIC;
  PlaneLayout L{};
  uint64_t scalar_heap = 0, array_heap = 0, heap_used = 0;
  if (!totals_known && !exact) {
    // planes and offset scratch first, then the whole pipeline without a host round trip.  The scratch is cheap
    // (8 bytes per frame): twice the expected count, so that only the planes can realistically be too small.
    if (int rc = launch_emit(ctx, b, cap_r, cap_c, 0, &L, &scalar_heap)) return fail(rc);
    if (int rc = ensure_record_scratch(ctx, 2 * cap_r + 65536)) return fail(rc);
    if (int rc = launch_index(ctx, false)) return fail(rc);
    if (sharded && !P.n_anchors) { if (int rc = launch_summary(ctx)) return fail(rc); }   // (an empty range: the identity seam; otherwise k_chase wrote the seam block)
  } else if (!totals_known) {
    if (int rc = launch_index(ctx, true)) return fail(rc);
    if (int rc = launch_summary(ctx)) return fail(rc);
    if (!sharded) {
      CKB(cudaMemcpyAsync(ctx->h_total, P.total, sizeof(Summ), cudaMemcpyDeviceToHost, st));
      CKB(cudaStreamSynchronize(st));
    }
  }
  if (sharded) {
    if (int rc = ctx_allgather(ctx, P.seam_send, (void*)P.seam_all, sizeof(SeamBlock))) return fail(rc);
    k_seam_fold<<<1, 32, 0, st>>>(P);
    ctx->launches += 2;
    if (exact && !totals_known) {
      CKB(cudaMemcpyAsync(ctx->h_total, P.total, sizeof(Summ), cudaMemcpyDeviceToHost, st));
      CKB(cudaStreamSynchronize(st));
    }
  }
  std::vector<SeamBlock> seams;                        // sharded: every rank's totals (read back after the first pass)
  for (int attempt = 0;; attempt++) {
    if (exact) {
      const Summ T = *ctx->h_total;
      if (b->dev_block) { CKB(cudaFreeAsync(b->dev_block, st)); b->dev_block = nullptr; }
      if (int rc = launch_emit(ctx, b, T.n_rec, T.n_cells, array_heap, &L, &scalar_heap)) return fail(rc);
      if (attempt > 0 || totals_known) {              // a re-run of pass C: fresh scalars, the carry block stays
        if (int rc = upload_scalars(ctx, 0, 12, nullptr)) return fail(rc);
        CKB(reset_abort());
      }
    }
    if (int rc = launch_emit_kernels(ctx)) return fail(rc);
    TRACE_MARK(1);
    CKB(cudaStreamSynchronize(st));
    TRACE_MARK(2);
    if (sharded && seams.empty()) {
      seams.resize(ctx->n_ranks);
      memcpy(seams.data(), ctx->h_seam, sizeof(SeamBlock) * ctx->n_ranks);   // copied with the scalars, before the sync
    }
    if (ctx->long_skipped && ctx->h_scalars[7] && !ctx->h_scalars[13]) {
      // the frame-length hint was wrong: long values exist.  Run the passes that were left out, read the scalars again.
      ctx->long_skipped = false;
      sizing |= ETL_SIZING_LONG_PASSES_LATE;
      CKB(cudaMemsetAsync(P.line_bad, 0, ((P.len + 4095) / 4096 + 1) * 4, st));
      k_utf8_dead<<<dead_grid(P), 256, 0, st>>>(P);
      k_long_cells<<<sm_count(ctx) * 8, 256, 0, st>>>(P);
      ctx->launches += 2;
      CKB(cudaGetLastError());
      CKB(cudaMemcpyAsync(ctx->h_scalars, ctx->d_scalars.ptr(), kScalarWords * 8, cudaMemcpyDeviceToHost, st));
      CKB(cudaStreamSynchronize(st));
    }
    const uint32_t aborted = (uint32_t)ctx->h_scalars[13];
    bool scratch_short = (aborted & ABORT_SCRATCH) != 0;
    for (const SeamBlock& sb : seams) scratch_short = scratch_short || (sb.total.flags & 0x80000000u);   // some rank could not form its totals
    if (scratch_short) {
      // more frames than the offset scratch holds (2x what earlier batches needed): start over on the exact path.
      // Sharded: every rank sees the same gathered blocks, so every rank takes this branch and the exchange is repeated.
      if (force_exact) { ctx->last_error = "offset scratch overflow on the exact path"; return fail(ETL_ERR_CUDA); }
      fail(0);
      return run_decode(ctx, carry_in, record_index_base, sharded, false, out, true, sizing | ETL_SIZING_SCRATCH_RESTART);
    }
    if (aborted) {                                     // did not fit the optimistic planes: exact sizes, pass C again
      sizing |= ((aborted & ABORT_RECORDS) ? ETL_SIZING_RERUN_RECORDS : 0u) | ((aborted & ABORT_CELLS) ? ETL_SIZING_RERUN_CELLS : 0u);
      CKB(reset_abort());
      if (int rc = launch_summary(ctx)) return fail(rc);
      CKB(cudaMemcpyAsync(ctx->h_total, P.total, sizeof(Summ), cudaMemcpyDeviceToHost, st));
      CKB(cudaStreamSynchronize(st));
      exact = true;
      ctx->lines_launched = false;
      CKB(cudaMemsetAsync(P.line_bad, 0, ((P.len + 4095) / 4096 + 1) * 4, st));
      continue;
    }
    const Summ T = *ctx->h_total;
    heap_used = P.heap_cap;
    if (P.heap_cap) heap_used = std::min<uint64_t>(P.heap_cap, ctx->h_scalars[10] ? scalar_heap + ctx->h_scalars[10] : ctx->h_scalars[5]);
    if (ctx->h_scalars[9]) {                          // an array reservation did not fit: larger array region, pass C again
      if (attempt >= 4) { ctx->last_error = "array heap reservation overflow after retries"; return fail(ETL_ERR_CUDA); }
      array_heap = (P.heap_cap - scalar_heap) * 4;
      sizing |= ETL_SIZING_ARRAY_HEAP_RETRY;
      exact = true;
      ctx->lines_launched = false;
      CKB(cudaMemsetAsync(P.line_bad, 0, ((P.len + 4095) / 4096 + 1) * 4, st));
      continue;
    }
    // the planes describe exactly the batch
    b->dev.n_records = T.n_rec; b->dev.n_cells = T.n_cells; b->dev.heap_bytes = heap_used;
    break;
  }
  const Summ T = *ctx->h_total;
  if (P.len) { ctx->rec_per_byte = std::max(ctx->rec_per_byte * 0.97, (double)T.n_rec / P.len); ctx->cells_per_byte = std::max(ctx->cells_per_byte * 0.97, (double)T.n_cells / P.len); }

  uint64_t d2h_bytes = kScalarWords * 8 + sizeof(Summ);
  if (ctx->pending_flags & ETL_DECODE_RESULTS_TO_HOST) {
    // compact host image: planes laid out for the exact counts; one copy per plane, one synchronisation
    const uint64_t nr = T.n_rec, nc = T.n_cells;
    const PlaneLayout H = plane_layout(nr, nc, heap_used);
    if (ctx->h_result_cap < H.total) {
      if (ctx->h_result) cudaFreeHost(ctx->h_result);
      ctx->h_result = nullptr; ctx->h_result_cap = 0;
      size_t want = H.total + H.total / 8;
      CKB(cudaHostAlloc(&ctx->h_result, want, cudaHostAllocDefault));
      ctx->h_result_cap = want;
    }
    b->host_block = ctx->h_result;
    uint8_t* hb = (uint8_t*)b->host_block;
    const uint8_t* db = (const uint8_t*)b->dev_block;
    CKB(cudaEventRecord(ctx->ev[4], st));
    if (L.rec_off == H.rec_off && L.heap + heap_used <= H.total && L.tag == H.tag && L.heap == H.heap) {
      CKB(cudaMemcpyAsync(hb, db, H.heap + heap_used, cudaMemcpyDeviceToHost, st));
      d2h_bytes += H.heap + heap_used;
    } else {
      auto cp = [&](uint64_t ho, uint64_t dof, uint64_t bytes) { if (bytes) cudaMemcpyAsync(hb + ho, db + dof, bytes, cudaMemcpyDeviceToHost, st); d2h_bytes += bytes; };
      cp(H.rec_off, L.rec_off, nr * 8); cp(H.kind, L.kind, nr); cp(H.flags, L.flags, nr); cp(H.rel, L.rel, nr * 4); cp(H.schema, L.schema, nr * 4);
      cp(H.start, L.start, nr * 8); cp(H.commit, L.commit, nr * 8); cp(H.ord, L.ord, nr * 8); cp(H.cbase, L.cbase, (nr + 1) * 8);
      cp(H.tb, L.tb, nr * 4); cp(H.hint, L.hint, nr * 4); cp(H.tag, L.tag, nc); cp(H.val, L.val, nc * 8); cp(H.aux, L.aux, nc * 4); cp(H.heap, L.heap, heap_used);
      CKB(cudaGetLastError());
    }
    fill_planes(b->host, hb, H, nr, nc, heap_used);
    b->has_host = true;
    CKB(cudaEventRecord(ctx->ev[5], st));
    CKB(cudaStreamSynchronize(st));
  } else if (!(ctx->pending_flags & ETL_DECODE_NO_TIMING)) { CKB(cudaEventRecord(ctx->ev[5], st)); CKB(cudaEventSynchronize(ctx->ev[5])); }

  TRACE_MARK(3);
  // ---- summary
  etl_dec_summary& S = b->summary;
  memset(&S, 0, sizeof S);
  float h2d_ms = 0, index_ms = 0, emit_ms = 0, d2h_ms = 0;
  if (!(ctx->pending_flags & ETL_DECODE_NO_TIMING)) {          // ten event queries: host time an 8 MiB batch notices
    cudaEventElapsedTime(&h2d_ms, ctx->ev[0], ctx->ev[1]);
    cudaEventElapsedTime(&index_ms, ctx->ev[1], ctx->ev[2]);
    cudaEventElapsedTime(&emit_ms, ctx->ev[3], ctx->ev[4]);
    cudaEventElapsedTime(&d2h_ms, ctx->ev[4], ctx->ev[5]);
    if (ctx->pending_flags & ETL_DECODE_RESULTS_TO_HOST) { float whole = 0; cudaEventElapsedTime(&whole, ctx->ev[3], ctx->ev[5]); emit_ms = whole - d2h_ms; }
    if (P.n_anchors) {
      cudaEventElapsedTime(&S.frames_ms, ctx->ev[3], ctx->evk[0]);
      cudaEventElapsedTime(&S.walk_ms, ctx->evk[0], ctx->evk[2]);    // k_bin_scan + k_perm
      cudaEventElapsedTime(&S.cells_ms, ctx->evk[2], ctx->evk[1]);   // k_rows
      cudaEventElapsedTime(&S.spans_ms, ctx->ev_l0, ctx->ev_l1);     // k_utf8_dead
      cudaEventElapsedTime(&S.long_ms, ctx->evk[3], ctx->ev[4]);     // k_long_cells
    }
  }
  S.kernel_ms = index_ms + emit_ms;
  S.index_ms = index_ms; S.emit_ms = emit_ms;
  S.h2d_ms = h2d_ms; S.d2h_ms = d2h_ms;
  S.h2d_bytes = ctx->pending_h2d_bytes;
  // bytes k_utf8_dead streamed: the dead segments (h_scalars[12] = live segment count, left by k_act_scan)
  S.span_bytes = P.n_anchors ? std::min<uint64_t>(P.len, (uint64_t)(P.n_anchors - (uint32_t)ctx->h_scalars[12]) * P.anchor_stride) : 0;
  S.d2h_bytes = d2h_bytes;
  S.gpu_launches = ctx->launches;
  S.n_schemas = (uint32_t)b->schemas.size();
  unsigned long long key = ctx->h_scalars[0];
  uint64_t err_off = ~0ull;
  if (key == ~0ull) { S.first_error.record_index = UINT64_MAX; }
  else {
    S.first_error.record_index = key >> 24;  // global index
    S.first_error.seq = (uint32_t)((key >> 6) & 0x3FFFFu);
    S.first_error.code = (uint32_t)(key & 63u);
    S.first_error.kind = error_kind_of(S.first_error.code);
  }
  S.insert_bytes = ctx->h_scalars[1]; S.update_bytes = ctx->h_scalars[2]; S.delete_bytes = ctx->h_scalars[3]; S.n_events = ctx->h_scalars[4];
  // carry-out: this shard's end state (sharded: relative to the folded carry, read back only when asked for below)
  Summ endst = fold(host_carry, T);
  if (sharded) {                                       // the stream state after the LAST shard = fold over all seams
    const std::vector<SeamBlock>& all = seams;
    endst = host_carry;
    uint64_t base = 0;
    for (int r = 0; r < ctx->n_ranks; r++) { if (r < ctx->rank) base += all[r].total.n_rec; endst = fold(endst, all[r].total); }
    S.record_index_base = base;
  } else S.record_index_base = record_index_base;
  S.carry_out.in_tx = ((endst.flags & S_HAS_B) && !(endst.flags & S_CLOSED)) ? 1 : 0;
  S.carry_out.final_lsn = endst.lsn;
  S.carry_out.next_tx_ordinal = endst.ord;
  S.abi_version = ETL_DECODE_ABI_VERSION;
  S.sizing = sizing;

  // ---- note_ready (apply.rs:2079): the Relation frames of the valid prefix become the state of the next batch.
  // After a data error the reference has bailed out before caching anything that follows it.
  if (key != ~0ull) {
    const uint64_t local = S.first_error.record_index - S.record_index_base;
    if (local < T.n_rec) CKB(cudaMemcpy(&err_off, b->dev.rec_off + local, 8, cudaMemcpyDeviceToHost));
  }
  bool changed = false;
  for (const RelVersion& v : ctx->foreign_installs) if (v.effective_off == 0) { ctx->current[v.table_id] = v; ctx->current[v.table_id].effective_off = 0; changed = true; }
  for (auto& pr : ctx->pending_installs) if (pr.first < err_off) { ctx->current[pr.second.table_id] = pr.second; changed = true; }
  if (key == ~0ull) for (const RelVersion& v : ctx->foreign_installs) if (v.effective_off == 1) { ctx->current[v.table_id] = v; ctx->current[v.table_id].effective_off = 0; changed = true; }
  if (changed) ctx->tables_valid = false;
  ctx->pending_installs.clear(); ctx->foreign_installs.clear();
  b->dev_stream = P.buf;
  *out = b;
  TRACE_MARK(4);
  return ETL_OK;
#undef CKB
}
const uint8_t* etl_dec_batch_device_stream(const etl_dec_batch* b) { return b ? b->dev_stream : nullptr; }

int etl_dec_decode(etl_dec_ctx* ctx, const etl_dec_input* in, uint32_t flags, etl_dec_batch** out) {
  if (!ctx || !in || !out) return ETL_ERR_INVALID_ARG;
  if (trace_on()) { ctx->tr_t0 = now_us(); ctx->tr_n++; }
  if (int rc = prepare(ctx, in, flags, false)) return rc;
  TRACE_MARK(0);
  return run_decode(ctx, &in->carry_in, 0, false, false, out);
}
int etl_dec_decode_sharded(etl_dec_ctx* ctx, const etl_dec_input* in, uint32_t flags, etl_dec_batch** out) {
  if (!ctx || !in || !out) return ETL_ERR_INVALID_ARG;
  if (int rc = prepare(ctx, in, flags, true)) return rc;
  return run_decode(ctx, &in->carry_in, 0, true, false, out);
}

int etl_dec_decode_begin(etl_dec_ctx* ctx, const etl_dec_input* in, uint32_t flags, etl_dec_seam* seam_out) {
  if (!ctx || !in) return ETL_ERR_INVALID_ARG;
  if (int rc = prepare(ctx, in, flags, false)) return rc;
  DecodeParams& P = ctx->P;
  P.cap_records = ~0ull; P.cap_cells = ~0ull; P.rec_cell_base = nullptr;
  if (int rc = upload_scalars(ctx, 0, kScalarWords, nullptr)) return rc;
  if (int rc = launch_index(ctx, true)) return rc;
  if (int rc = launch_summary(ctx)) return rc;
  CK(cudaMemcpyAsync(ctx->h_total, P.total, sizeof(Summ), cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  const Summ& T = *ctx->h_total;
  if (seam_out) {
    memset(seam_out, 0, sizeof *seam_out);
    seam_out->n_records = T.n_rec; seam_out->n_cells = T.n_cells; seam_out->heap_bytes = 0;
    seam_out->lsn = T.lsn; seam_out->ord = T.ord;
    seam_out->has_begin = (T.flags & S_HAS_B) ? 1 : 0; seam_out->closed = (T.flags & S_CLOSED) ? 1 : 0;
  }
  ctx->pending = true;
  return ETL_OK;
}

int etl_dec_decode_finish(etl_dec_ctx* ctx, const etl_stream_state* carry_in, uint64_t record_index_base,
                          etl_dec_batch** out) {
  if (!ctx || !out || !ctx->pending) { if (ctx) ctx->last_error = "decode_finish without decode_begin"; return ETL_ERR_INVALID_ARG; }
  ctx->pending = false;
  CK(cudaSetDevice(ctx->device));
  return run_decode(ctx, carry_in, record_index_base, false, true, out);
}

// ---------------------------------------------------------------- COPY rows (table_row.rs:25-165 for a buffer of rows)
int etl_dec_copy_decode(etl_dec_ctx* ctx, uint32_t table_id, const etl_copy_input* in, uint32_t flags, etl_dec_batch** out) {
  if (!ctx || !in || !out) return ETL_ERR_INVALID_ARG;
  if (in->len && !in->host_buf && !in->dev_buf) { ctx->last_error = "no input buffer"; return ETL_ERR_INVALID_ARG; }
  if (in->dev_buf && (reinterpret_cast<uintptr_t>(in->dev_buf) & 15u)) { ctx->last_error = "dev_buf must be 16-byte aligned"; return ETL_ERR_INVALID_ARG; }
  if (in->n_rows && !in->row_offsets && !in->dev_row_offsets) { ctx->last_error = "row_offsets missing"; return ETL_ERR_INVALID_ARG; }
  if (in->n_rows >= (1ull << 32)) { ctx->last_error = "a COPY batch is limited to 2^32 rows"; return ETL_ERR_INVALID_ARG; }
  auto it = ctx->tables.find(table_id);
  if (it == ctx->tables.end()) { ctx->last_error = "table schema not stored"; return ETL_ERR_INVALID_ARG; }
  const StoredTable& t = it->second;
  const uint32_t n_cols = (uint32_t)t.cols.size();
  std::vector<uint8_t> kinds(n_cols);
  bool any_heap = false, any_array = false;
  for (uint32_t i = 0; i < n_cols; i++) {
    const uint32_t k = etl_oid_decode_class(t.cols[i].type_oid);
    if (!kind_supported_on_device(k)) { ctx->last_error = "column decode class has no device parser"; return ETL_ERR_INVALID_ARG; }
    kinds[i] = (uint8_t)k;
    any_heap = any_heap || kind_has_heap(k); any_array = any_array || (k & ETL_K_ARRAY);
  }
  CK(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  ctx->launches = 0;
  ctx->tables_valid = false;                          // d_tables is reused for the column classes
  etl_dec_batch* b = new etl_dec_batch();
  b->ctx = ctx;
  auto fail = [&](int rc) { if (b->dev_block) cudaFreeAsync(b->dev_block, st); delete b; return rc; };
#define CKB(call) do { cudaError_t _e = (call); if (_e != cudaSuccess) { ctx->last_error = std::string(#call) + ": " + cudaGetErrorString(_e); return fail(ETL_ERR_CUDA); } } while (0)
  DecodeParams& P = ctx->P;
  memset(&P, 0, sizeof P);
  P.len = in->len; P.anchor_stride = 2048; P.copy_cols = n_cols;
  CKB(cudaEventRecord(ctx->ev[0], st));
  uint64_t h2d = 0;
  if (in->dev_buf) P.buf = in->dev_buf;
  else {
    CKB(ctx->d_stream.ensure(in->len + 64));
    if (in->len) CKB(cudaMemcpyAsync(ctx->d_stream.ptr(), in->host_buf, in->len, cudaMemcpyHostToDevice, st));
    CKB(cudaMemsetAsync(ctx->d_stream.ptr() + in->len, 0, 64, st));
    P.buf = ctx->d_stream.ptr(); h2d += in->len;
  }
  const uint64_t nr = in->n_rows, nc = nr * n_cols;
  // planes: rec_off (row offsets) + cells + heap (unescaped text ≤ len, scalar payloads, arrays)
  uint64_t nh = in->len + 64 + (any_heap ? in->len / 2 + 24 * nc + 256 : 0);
  nh = (nh + 15) & ~15ull;
  const uint64_t scalar_heap = nh;
  uint64_t array_heap = any_array ? 3 * in->len + 4096 : 0;
  for (int attempt = 0;; attempt++) {
    const uint64_t heap_total = scalar_heap + array_heap;
    const PlaneLayout L = plane_layout(nr, nc, heap_total);
    if (b->dev_block) { CKB(cudaFreeAsync(b->dev_block, st)); b->dev_block = nullptr; }
    b->block_bytes = L.total;
    CKB(cudaMallocAsync(&b->dev_block, b->block_bytes, st));
    fill_planes(b->dev, (uint8_t*)b->dev_block, L, nr, nc, heap_total);
    uint64_t* d_rows = (uint64_t*)b->dev.rec_cell_base;             // the (n_rows + 1)-entry plane holds the row offsets
    if (in->dev_row_offsets) CKB(cudaMemcpyAsync(d_rows, in->dev_row_offsets, (nr + 1) * 8, cudaMemcpyDeviceToDevice, st));
    else if (nr) { CKB(cudaMemcpyAsync(d_rows, in->row_offsets, (nr + 1) * 8, cudaMemcpyHostToDevice, st)); h2d += (nr + 1) * 8; }
    else CKB(cudaMemsetAsync(d_rows, 0, 8, st));
    b->dev.rec_off = d_rows;
    b->dev.rec_kind = nullptr; b->dev.rec_flags = nullptr; b->dev.rec_rel = nullptr; b->dev.rec_schema = nullptr; b->dev.rec_start_lsn = nullptr;
    b->dev.rec_commit_lsn = nullptr; b->dev.rec_tx_ordinal = nullptr; b->dev.rec_tuple_bytes = nullptr; b->dev.rec_heap_hint = nullptr;
    P.rec_off = d_rows; P.rec_cell_base = d_rows;
    P.cell_tag = (uint8_t*)b->dev.cell_tag; P.cell_val = (uint64_t*)b->dev.cell_val; P.cell_aux = (uint32_t*)b->dev.cell_aux; P.heap = (uint8_t*)b->dev.heap;
    P.heap_cap = heap_total; P.arr_base = scalar_heap;
    CKB(ctx->d_tables.ensure(n_cols + 16));
    if (int rc = ensure_pinned(ctx, &ctx->h_up, &ctx->h_up_cap, n_cols + 16)) return fail(rc);
    memcpy(ctx->h_up, kinds.data(), n_cols);
    if (n_cols) CKB(cudaMemcpyAsync(ctx->d_tables.ptr(), ctx->h_up, n_cols, cudaMemcpyHostToDevice, st));
    P.col_kind = ctx->d_tables.ptr(); P.col_flags = ctx->d_tables.ptr();
    unsigned long long* sc = reinterpret_cast<unsigned long long*>(ctx->d_scalars.ptr());
    P.first_error = sc; P.metrics = sc + 1; P.heap_top = sc + 5; P.long_count = (unsigned int*)(sc + 7); P.copy_count = (unsigned int*)(sc + 8);
    P.heap_overflow = (unsigned int*)(sc + 9); P.arr_top = sc + 10; P.perm_len = (unsigned int*)(sc + 11); P.n_act = (unsigned int*)(sc + 12);
    P.abort_flag = (unsigned int*)(sc + 13);
    P.dc = reinterpret_cast<const DevCarry*>(sc + kScalarWords); P.dc_out = reinterpret_cast<DevCarry*>(sc + kScalarWords);
    P.total = ctx->d_total.ptr();
    DevCarry dc; dc.carry = summ_identity(); dc.record_index_base = 0;
    if (int rc = upload_scalars(ctx, 0, kScalarWords, &dc)) return fail(rc);
    Summ T = summ_identity(); T.n_rec = (uint32_t)nr; T.n_cells = nc;
    *ctx->h_total = T;
    CKB(cudaMemcpyAsync(P.total, ctx->h_total, sizeof(Summ), cudaMemcpyHostToDevice, st));
    P.cap_records = nr; P.cap_cells = nc;
    if (nc) CKB(cudaMemsetAsync(P.cell_tag, 0, nc, st));   // a row that failed leaves cells unwritten: k_heavy must not see stale tags
    CKB(cudaEventRecord(ctx->ev[1], st));
    if (nr) {
      k_copy_rows<<<(uint32_t)((nr + kRowsThreads - 1) / kRowsThreads), kRowsThreads, kRowsSmemBytes, st>>>(P);
      k_heavy<<<std::min<uint32_t>((uint32_t)((nc + kHeavyTile - 1) / kHeavyTile) + 1u, (uint32_t)sm_count(ctx) * 3u), kHeavyThreads, kHeavySmemBytes, st>>>(P);
      ctx->launches += 2;
      CKB(cudaGetLastError());
    }
    CKB(cudaEventRecord(ctx->ev[4], st));
    CKB(cudaMemcpyAsync(ctx->h_scalars, ctx->d_scalars.ptr(), kScalarWords * 8, cudaMemcpyDeviceToHost, st));
    CKB(cudaStreamSynchronize(st));
    if (!ctx->h_scalars[9]) break;
    if (attempt >= 4) { ctx->last_error = "array heap reservation overflow after retries"; return fail(ETL_ERR_CUDA); }
    array_heap *= 4;
  }
  const uint64_t heap_used = std::min<uint64_t>(P.heap_cap, ctx->h_scalars[10] ? scalar_heap + ctx->h_scalars[10] : ctx->h_scalars[5]);
  b->dev.heap_bytes = heap_used;
  uint64_t d2h = kScalarWords * 8;
  if (flags & ETL_DECODE_RESULTS_TO_HOST) {
    const PlaneLayout H = plane_layout(nr, nc, heap_used);
    if (ctx->h_result_cap < H.total) {
      if (ctx->h_result) cudaFreeHost(ctx->h_result);
      ctx->h_result = nullptr; ctx->h_result_cap = 0;
      size_t want = H.total + H.total / 8;
      CKB(cudaHostAlloc(&ctx->h_result, want, cudaHostAllocDefault));
      ctx->h_result_cap = want;
    }
    uint8_t* hb = (uint8_t*)ctx->h_result;
    fill_planes(b->host, hb, H, nr, nc, heap_used);
    b->host.rec_off = b->host.rec_cell_base;
    b->host.rec_kind = nullptr; b->host.rec_flags = nullptr; b->host.rec_rel = nullptr; b->host.rec_schema = nullptr; b->host.rec_start_lsn = nullptr;
    b->host.rec_commit_lsn = nullptr; b->host.rec_tx_ordinal = nullptr; b->host.rec_tuple_bytes = nullptr; b->host.rec_heap_hint = nullptr;
    CKB(cudaMemcpyAsync((void*)b->host.rec_cell_base, b->dev.rec_cell_base, (nr + 1) * 8, cudaMemcpyDeviceToHost, st));
    if (nc) {
      CKB(cudaMemcpyAsync((void*)b->host.cell_tag, b->dev.cell_tag, nc, cudaMemcpyDeviceToHost, st));
      CKB(cudaMemcpyAsync((void*)b->host.cell_val, b->dev.cell_val, nc * 8, cudaMemcpyDeviceToHost, st));
      CKB(cudaMemcpyAsync((void*)b->host.cell_aux, b->dev.cell_aux, nc * 4, cudaMemcpyDeviceToHost, st));
    }
    if (heap_used) CKB(cudaMemcpyAsync((void*)b->host.heap, b->dev.heap, heap_used, cudaMemcpyDeviceToHost, st));
    d2h += (nr + 1) * 8 + nc * 13 + heap_used;
    b->host_block = hb; b->has_host = true;
  }
  CKB(cudaEventRecord(ctx->ev[5], st));
  CKB(cudaStreamSynchronize(st));
  etl_dec_summary& S = b->summary;
  memset(&S, 0, sizeof S);
  cudaEventElapsedTime(&S.h2d_ms, ctx->ev[0], ctx->ev[1]);
  cudaEventElapsedTime(&S.emit_ms, ctx->ev[1], ctx->ev[4]);
  cudaEventElapsedTime(&S.d2h_ms, ctx->ev[4], ctx->ev[5]);
  S.kernel_ms = S.emit_ms; S.cells_ms = S.emit_ms;
  S.h2d_bytes = h2d; S.d2h_bytes = d2h; S.gpu_launches = ctx->launches; S.abi_version = ETL_DECODE_ABI_VERSION;
  S.sizing = ETL_SIZING_EXACT | (array_heap > (any_array ? 3 * in->len + 4096 : 0) ? ETL_SIZING_ARRAY_HEAP_RETRY : 0u);
  const unsigned long long key = ctx->h_scalars[0];
  if (key == ~0ull) S.first_error.record_index = UINT64_MAX;
  else {
    S.first_error.record_index = key >> 24; S.first_error.seq = (uint32_t)((key >> 6) & 0x3FFFFu);
    S.first_error.code = (uint32_t)(key & 63u); S.first_error.kind = error_kind_of(S.first_error.code);
  }
  S.n_events = nr;
  b->dev_stream = P.buf;
  b->copy = true; b->copy_table = table_id; b->copy_kinds = std::move(kinds);
  *out = b;
  return ETL_OK;
#undef CKB
}

int etl_dec_batch_planes(const etl_dec_batch* b, int host, etl_dec_planes* out) {
  if (!b || !out) return ETL_ERR_INVALID_ARG;
  if (host && !b->has_host) return ETL_ERR_INVALID_ARG;
  *out = host ? b->host : b->dev;
  return ETL_OK;
}
int etl_dec_batch_summary(const etl_dec_batch* b, etl_dec_summary* out) {
  if (!b || !out) return ETL_ERR_INVALID_ARG;
  *out = b->summary;
  return ETL_OK;
}
int etl_dec_batch_schema(const etl_dec_batch* b, uint32_t i, etl_dec_schema_info* out) {
  if (!b || !out || i >= b->schemas.size()) return ETL_ERR_INVALID_ARG;
  const RelVersion& v = b->schemas[i];
  out->table_id = v.table_id; out->n_cols = (uint32_t)v.kind.size(); out->n_identity = v.n_ident; out->_pad = 0;
  out->snapshot_id = v.snapshot_id; out->effective_off = v.effective_off;
  out->col_kind = v.kind.data(); out->col_flags = v.flags.data(); out->col_index = v.index.data();
  return ETL_OK;
}
int etl_dec_mem_info(etl_dec_ctx* ctx, uint64_t* free_bytes, uint64_t* total_bytes) {
  if (!ctx) return ETL_ERR_INVALID_ARG;
  CK(cudaSetDevice(ctx->device));
  size_t f = 0, t = 0;
  CK(cudaMemGetInfo(&f, &t));
  if (free_bytes) *free_bytes = f;
  if (total_bytes) *total_bytes = t;
  return ETL_OK;
}

}  // extern "C"

bool etl_copy_batch_columns(const etl_dec_batch* b, uint32_t* table_id, const uint8_t** col_kind, uint32_t* n_cols) {
  if (!b || !b->copy) return false;
  *table_id = b->copy_table; *col_kind = b->copy_kinds.data(); *n_cols = (uint32_t)b->copy_kinds.size();
  return true;
}
