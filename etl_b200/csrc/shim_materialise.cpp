// shim_materialise.cpp — host-side stand-in for the Rust shim's last step (INTEGRATION.md §3, SURVEY §8f N3):
// planes → the AoS `Vec<Event>` the reference hands to ApplyLoopState::add_event_to_batch (apply.rs:433-439),
// i.e. the work the device deliberately leaves to the consumer:
//   * one owned copy per String / Bytes cell and per Numeric digit vector (Rust: String::to_owned, Vec<u8>, Vec<i16>),
//   * serde_json::from_slice per Json cell → an owned tree (object keys sorted, duplicate keys: last value wins,
//     numbers kept as text: serde_json's `arbitrary_precision`, text.rs:150-158),
//   * ArrayCell construction from the heap's element lists,
//   * Event::size_hint per event (types/event.rs:288-312 over types/table_row.rs:250-345) so that the byte-budget
//     flush of the apply loop (apply.rs:1611-1624) sees the numbers the reference would have computed.
// The build needs no Rust toolchain, so this is C++ with the Rust struct sizes as parameters (etl_rust_layout:
// a real shim passes std::mem::size_of values).  Pure host code: it never touches the GPU and is timed separately
// (bench.py `e2e_materialised`).
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <map>
#include <memory>
#include <string>
#include <vector>

#include "etl_decode.h"

namespace {

struct JsonValue {
  enum T : uint8_t { Null, Bool, Number, String, Array, Object } t = Null;
  bool b = false;
  std::string s;                                         // Number (verbatim text) / String (unescaped)
  std::vector<JsonValue> arr;
  std::vector<std::pair<std::string, JsonValue>> obj;    // sorted by key (BTreeMap), unique
};

struct JsonParser {  // grammar already validated on the device; this builds the tree serde_json would build
  const uint8_t* p; const uint8_t* e;
  void ws() { while (p < e && (*p == ' ' || *p == '\t' || *p == '\n' || *p == '\r')) p++; }
  static void utf8_put(std::string& o, uint32_t c) {
    if (c < 0x80) o.push_back((char)c);
    else if (c < 0x800) { o.push_back((char)(0xC0 | (c >> 6))); o.push_back((char)(0x80 | (c & 63))); }
    else if (c < 0x10000) { o.push_back((char)(0xE0 | (c >> 12))); o.push_back((char)(0x80 | ((c >> 6) & 63))); o.push_back((char)(0x80 | (c & 63))); }
    else { o.push_back((char)(0xF0 | (c >> 18))); o.push_back((char)(0x80 | ((c >> 12) & 63))); o.push_back((char)(0x80 | ((c >> 6) & 63))); o.push_back((char)(0x80 | (c & 63))); }
  }
  static uint32_t hex4(const uint8_t* q) {
    uint32_t v = 0;
    for (int i = 0; i < 4; i++) { uint32_t c = q[i]; v = v * 16 + (c <= '9' ? c - '0' : ((c | 32) - 'a' + 10)); }
    return v;
  }
  bool str(std::string& out) {
    if (p >= e || *p != '"') return false;
    p++;
    const uint8_t* run = p;
    while (p < e && *p != '"') {
      if (*p == '\\') {
        out.append((const char*)run, (size_t)(p - run));
        if (p + 1 >= e) return false;
        uint8_t c = p[1];
        p += 2;
        switch (c) {
          case 'b': out.push_back('\b'); break; case 'f': out.push_back('\f'); break; case 'n': out.push_back('\n'); break;
          case 'r': out.push_back('\r'); break; case 't': out.push_back('\t'); break;
          case 'u': {
            if (p + 4 > e) return false;
            uint32_t u = hex4(p); p += 4;
            if (u >= 0xD800 && u <= 0xDBFF && p + 6 <= e && p[0] == '\\' && p[1] == 'u') { uint32_t lo = hex4(p + 2); p += 6; u = 0x10000 + ((u - 0xD800) << 10) + (lo - 0xDC00); }
            utf8_put(out, u);
            break;
          }
          default: out.push_back((char)c);
        }
        run = p;
      } else p++;
    }
    if (p >= e) return false;
    out.append((const char*)run, (size_t)(p - run));
    p++;
    return true;
  }
  bool value(JsonValue& v, int depth) {
    ws();
    if (p >= e || depth > 130) return false;
    switch (*p) {
      case '{': {
        v.t = JsonValue::Object; p++;
        ws();
        if (p < e && *p == '}') { p++; return true; }
        for (;;) {
          ws();
          std::string k;
          if (!str(k)) return false;
          ws();
          if (p >= e || *p != ':') return false;
          p++;
          JsonValue c;
          if (!value(c, depth + 1)) return false;
          auto it = std::lower_bound(v.obj.begin(), v.obj.end(), k, [](const std::pair<std::string, JsonValue>& a, const std::string& b) { return a.first < b; });
          if (it != v.obj.end() && it->first == k) it->second = std::move(c);      // BTreeMap::insert: key kept, value replaced
          else v.obj.insert(it, std::make_pair(std::move(k), std::move(c)));
          ws();
          if (p < e && *p == ',') { p++; continue; }
          if (p < e && *p == '}') { p++; return true; }
          return false;
        }
      }
      case '[': {
        v.t = JsonValue::Array; p++;
        ws();
        if (p < e && *p == ']') { p++; return true; }
        for (;;) {
          JsonValue c;
          if (!value(c, depth + 1)) return false;
          v.arr.push_back(std::move(c));
          ws();
          if (p < e && *p == ',') { p++; continue; }
          if (p < e && *p == ']') { p++; return true; }
          return false;
        }
      }
      case '"': v.t = JsonValue::String; return str(v.s);
      case 't': v.t = JsonValue::Bool; v.b = true; p += 4; return p <= e;
      case 'f': v.t = JsonValue::Bool; v.b = false; p += 5; return p <= e;
      case 'n': v.t = JsonValue::Null; p += 4; return p <= e;
      default: {
        const uint8_t* s = p;
        while (p < e && (*p == '-' || *p == '+' || *p == '.' || *p == 'e' || *p == 'E' || (*p >= '0' && *p <= '9'))) p++;
        if (p == s) return false;
        v.t = JsonValue::Number; v.s.assign((const char*)s, (size_t)(p - s));
        return true;
      }
    }
  }
};

struct ArrayElem;
struct OwnedCell {
  uint8_t tag = ETL_CELL_NULL;
  uint64_t val = 0;                       // fixed-width payload (ints, float bits, days, seconds)
  uint32_t aux = 0;                       // nanoseconds
  std::string text;                       // String / Bytes payload
  etl_numeric_hdr num{};
  std::vector<int16_t> digits;            // Numeric
  uint8_t uuid[16]{};
  std::unique_ptr<JsonValue> json;
  uint8_t elem_kind = 0;
  std::vector<OwnedCell> elems;           // Array
  bool cloned = false;                    // value taken from the old image (event.rs:958-970): Clone allocates len, not capacity
};
struct Row { std::vector<OwnedCell> values; std::vector<uint64_t> missing; uint64_t total_columns = 0; bool partial = false; uint64_t first_missing = 0; };
struct Event {
  uint8_t kind = 0, flags = 0;
  uint64_t start_lsn = 0, commit_lsn = 0, tx_ordinal = 0;
  uint32_t table_id = 0; int32_t schema = -1;
  int64_t timestamp = 0, end_lsn = 0; uint32_t xid = 0; int32_t commit_flags = 0; int32_t options = 0;
  std::vector<uint32_t> rel_ids;
  bool has_old = false, old_is_key = false;
  Row old_row, row;
  uint64_t size_hint = 0;
};

const etl_rust_layout kDefaultLayout = {32, 32, 72, 40, 48, 96, 176, 104, 56, 64, 40, 32, 8};

uint64_t vec_cap_after_pushes(uint64_t n) { uint64_t c = 4; if (!n) return 0; while (c < n) c <<= 1; return c; }   // RawVec::grow_amortized, elem ≤ 1 KiB
uint64_t json_bytes(const JsonValue& v, const etl_rust_layout& L) {      // estimate_json_allocated_bytes, table_row.rs:330-360
  switch (v.t) {
    case JsonValue::String: return v.s.size();
    case JsonValue::Array: { uint64_t t = vec_cap_after_pushes(v.arr.size()) * L.size_of_json_value; for (const JsonValue& c : v.arr) t += json_bytes(c, L); return t; }
    case JsonValue::Object: { uint64_t t = 0; for (const auto& kv : v.obj) t += kv.first.size() + json_bytes(kv.second, L); return t; }
    default: return 0;
  }
}
uint64_t cell_bytes(const OwnedCell& c, const etl_rust_layout& L) {      // estimate_cell_allocated_bytes, table_row.rs:295-320
  switch (c.tag) {
    case ETL_CELL_STRING: case ETL_CELL_BYTES: return c.text.size();
    case ETL_CELL_NUMERIC: return c.num.kind ? 0 : 2ull * (c.cloned ? c.digits.size() : vec_cap_after_pushes(c.num.pushed_groups));
    case ETL_CELL_JSON: return c.json ? json_bytes(*c.json, L) : 0;
    case ETL_CELL_ARRAY: {   // estimate_array_allocated_bytes, table_row.rs:362-470: capacity × size_of::<Option<T>>() + element heaps
      static const uint32_t opt_size[18] = {0, 1, 24, 4, 8, 8, 16, 8, 16, 32, 8, 12, 16, 16, 17, 32, 24, 0};
      const uint32_t k = c.elem_kind;
      uint64_t t = vec_cap_after_pushes(c.elems.size()) * (k < 18 ? opt_size[k] : 24);
      for (const OwnedCell& e : c.elems) t += cell_bytes(e, L);
      return t;
    }
    default: return 0;
  }
}
uint64_t row_bytes(const Row& r, uint64_t values_capacity, const etl_rust_layout& L) {   // estimate_table_row_allocated_bytes, table_row.rs:250-271
  uint64_t t = L.size_of_table_row + values_capacity * L.size_of_cell;
  for (const OwnedCell& c : r.values) t += cell_bytes(c, L);
  return t;
}
// capacity of `present_values` of a Partial row (event.rs:617-657): Vec::new(), reserve(n - first_missing), append(prefix), push…
uint64_t partial_values_capacity(uint64_t n_cols, uint64_t first_missing, uint64_t n_present) {
  uint64_t cap = std::max<uint64_t>(4, n_cols - first_missing), len = 0;
  auto need = [&](uint64_t want) { if (want > cap) cap = std::max<uint64_t>(std::max<uint64_t>(cap * 2, want), 4); };
  need(first_missing); len = first_missing;
  while (len < n_present) { need(len + 1); len++; }
  return cap;
}

}  // namespace

struct etl_event_list {
  std::vector<Event> events;
  etl_rust_layout layout;
  uint64_t total_hint = 0;
  uint64_t owned_bytes = 0;   // bytes copied into owned Strings / Vecs (the shim's memcpy volume)
};

extern "C" {

int etl_shim_materialise(const etl_dec_batch* batch, const uint8_t* stream, const etl_rust_layout* layout, etl_event_list** out) {
  if (!batch || !out) return ETL_ERR_INVALID_ARG;
  etl_dec_planes P;
  if (etl_dec_batch_planes(batch, 1, &P) != ETL_OK) return ETL_ERR_INVALID_ARG;   // needs ETL_DECODE_RESULTS_TO_HOST
  etl_dec_summary S;
  etl_dec_batch_summary(batch, &S);
  std::vector<etl_dec_schema_info> schemas(S.n_schemas);
  for (uint32_t i = 0; i < S.n_schemas; i++) etl_dec_batch_schema(batch, i, &schemas[i]);
  etl_event_list* L = new etl_event_list();
  L->layout = layout ? *layout : kDefaultLayout;
  const etl_rust_layout& RL = L->layout;
  const uint64_t n_valid = S.first_error.record_index == UINT64_MAX ? P.n_records
                           : std::min<uint64_t>(P.n_records, S.first_error.record_index - S.record_index_base);
  L->events.reserve(S.n_events);
  auto own = [&](uint64_t i, OwnedCell& c, bool in_array) {
    c.tag = in_array ? c.tag : P.cell_tag[i];
    const uint64_t val = in_array ? c.val : P.cell_val[i];
    const uint32_t aux = in_array ? c.aux : P.cell_aux[i];
    c.val = val; c.aux = aux;
    const uint8_t* span_src = in_array ? P.heap : stream;
    switch (c.tag) {
      case ETL_CELL_STRING: c.text.assign((const char*)span_src + val, aux); L->owned_bytes += aux; break;
      case ETL_CELL_JSON: {
        c.json.reset(new JsonValue());
        JsonParser jp{span_src + val, span_src + val + aux};
        jp.value(*c.json, 0);
        L->owned_bytes += aux;
        break;
      }
      case ETL_CELL_BYTES: c.text.assign((const char*)P.heap + val, aux); L->owned_bytes += aux; break;
      case ETL_CELL_NUMERIC:
        memcpy(&c.num, P.heap + val, sizeof c.num);
        c.digits.resize(aux);
        if (aux) memcpy(c.digits.data(), P.heap + val + 8, 2ull * aux);
        L->owned_bytes += 2ull * aux;
        break;
      case ETL_CELL_UUID: memcpy(c.uuid, P.heap + val, 16); break;
      default: break;
    }
  };
  for (uint64_t r = 0; r < n_valid; r++) {
    const uint8_t flags = P.rec_flags[r];
    if (!(flags & ETL_RF_EVENT)) continue;
    L->events.emplace_back();
    Event& ev = L->events.back();
    ev.kind = P.rec_kind[r]; ev.flags = flags;
    ev.start_lsn = P.rec_start_lsn[r]; ev.commit_lsn = P.rec_commit_lsn[r]; ev.tx_ordinal = P.rec_tx_ordinal[r];
    ev.table_id = P.rec_rel[r]; ev.schema = P.rec_schema[r];
    const uint64_t c0 = P.rec_cell_base[r], c1 = P.rec_cell_base[r + 1];
    switch (ev.kind) {
      case 'B': ev.timestamp = (int64_t)P.cell_val[c0]; ev.xid = (uint32_t)P.cell_val[c0 + 1]; ev.size_hint = RL.size_of_begin_event; break;
      case 'C': ev.commit_flags = (int32_t)P.cell_val[c0]; ev.end_lsn = (int64_t)P.cell_val[c0 + 1]; ev.timestamp = (int64_t)P.cell_val[c0 + 2]; ev.size_hint = RL.size_of_commit_event; break;
      case 'R': ev.size_hint = RL.size_of_relation_event; break;
      case 'T':
        ev.options = (int32_t)P.cell_val[c0];
        for (uint64_t i = c0 + 1; i < c1; i++) ev.rel_ids.push_back((uint32_t)P.cell_val[i]);
        ev.size_hint = RL.size_of_truncate_event + ev.rel_ids.size() * (uint64_t)RL.size_of_replicated_table_schema;
        break;
      default: {   // I / U / D
        const etl_dec_schema_info& sc = schemas[(size_t)ev.schema];
        const uint64_t n_old = (flags & ETL_RF_OLD_FULL) ? sc.n_cols : ((flags & ETL_RF_OLD_KEY) ? sc.n_identity : 0);
        auto build = [&](Row& row, uint64_t a, uint64_t b, bool is_new_of_update) {
          row.total_columns = b - a;
          for (uint64_t i = a; i < b; i++) {
            if (P.cell_tag[i] == ETL_CELL_MISSING) { if (!row.partial) { row.partial = true; row.first_missing = i - a; } row.missing.push_back(i - a); continue; }
            row.values.emplace_back();
            OwnedCell& c = row.values.back();
            own(i, c, false);
            if (c.tag == ETL_CELL_ARRAY) {
              etl_array_hdr ah; memcpy(&ah, P.heap + c.val, sizeof ah);
              c.elem_kind = ah.elem_kind;
              c.elems.resize(ah.n_elems);
              for (uint32_t k = 0; k < ah.n_elems; k++) {
                etl_array_elem e; memcpy(&e, P.heap + c.val + 8 + 16ull * k, sizeof e);
                c.elems[k].tag = e.tag; c.elems[k].val = e.val; c.elems[k].aux = e.aux;
                own(0, c.elems[k], true);
              }
            }
            // unchanged TOAST resolved from the old image (event.rs:958-970): the planes give the new cell the old cell's
            // payload location, so an identical (tag, heap offset, digits) numeric among the old cells means "cloned"
            if (is_new_of_update && n_old && c.tag == ETL_CELL_NUMERIC)
              for (uint64_t j = c0; j < c0 + n_old; j++)
                if (P.cell_tag[j] == c.tag && P.cell_val[j] == c.val && P.cell_aux[j] == c.aux) { c.cloned = true; break; }
          }
        };
        uint64_t hint = 0;
        if (n_old) {
          ev.has_old = true; ev.old_is_key = (flags & ETL_RF_OLD_KEY) != 0;
          build(ev.old_row, c0, c0 + n_old, false);
          hint += row_bytes(ev.old_row, n_old, RL);                       // Vec::with_capacity(column_count / identity len), event.rs:563,795,825
        }
        if (ev.kind == 'I' || ev.kind == 'U') {
          build(ev.row, c0 + n_old, c1, ev.kind == 'U');
          if (ev.row.partial) {                                            // PartialTableRow::new, table_row.rs:84-96,272-292
            const uint64_t cap = partial_values_capacity(sc.n_cols, ev.row.first_missing, ev.row.values.size());
            hint += RL.size_of_partial_table_row + row_bytes(ev.row, cap, RL) + vec_cap_after_pushes(ev.row.missing.size()) * RL.size_of_usize;
          } else hint += row_bytes(ev.row, sc.n_cols, RL);                 // full_values = Vec::with_capacity(column_count)
        }
        hint += ev.kind == 'I' ? RL.size_of_insert_event : (ev.kind == 'U' ? RL.size_of_update_event : RL.size_of_delete_event);
        ev.size_hint = hint;
      }
    }
    L->total_hint += ev.size_hint;
  }
  *out = L;
  return ETL_OK;
}
uint64_t etl_shim_event_count(const etl_event_list* l) { return l ? l->events.size() : 0; }
uint64_t etl_shim_size_hint(const etl_event_list* l, uint64_t i) { return (l && i < l->events.size()) ? l->events[i].size_hint : 0; }
uint64_t etl_shim_total_size_hint(const etl_event_list* l) { return l ? l->total_hint : 0; }
uint64_t etl_shim_owned_bytes(const etl_event_list* l) { return l ? l->owned_bytes : 0; }
void etl_shim_event_list_free(etl_event_list* l) { delete l; }

// canonical text of a JSON cell of event i (serde_json::to_string of the tree: keys sorted, numbers verbatim) — tests
static void json_dump(const JsonValue& v, std::string& o) {
  auto esc = [&](const std::string& s) {
    o.push_back('"');
    for (unsigned char c : s) {
      switch (c) {
        case '"': o += "\\\""; break; case '\\': o += "\\\\"; break; case '\n': o += "\\n"; break; case '\r': o += "\\r"; break;
        case '\t': o += "\\t"; break; case '\b': o += "\\b"; break; case '\f': o += "\\f"; break;
        default: if (c < 0x20) { char b[8]; snprintf(b, sizeof b, "\\u%04x", c); o += b; } else o.push_back((char)c);
      }
    }
    o.push_back('"');
  };
  switch (v.t) {
    case JsonValue::Null: o += "null"; break;
    case JsonValue::Bool: o += v.b ? "true" : "false"; break;
    case JsonValue::Number: o += v.s; break;
    case JsonValue::String: esc(v.s); break;
    case JsonValue::Array: o.push_back('['); for (size_t i = 0; i < v.arr.size(); i++) { if (i) o.push_back(','); json_dump(v.arr[i], o); } o.push_back(']'); break;
    case JsonValue::Object: o.push_back('{'); for (size_t i = 0; i < v.obj.size(); i++) { if (i) o.push_back(','); esc(v.obj[i].first); o.push_back(':'); json_dump(v.obj[i].second, o); } o.push_back('}'); break;
  }
}
int64_t etl_shim_json_text(const etl_event_list* l, uint64_t event, uint32_t new_row_cell, char* buf, uint64_t cap) {
  if (!l || event >= l->events.size()) return -1;
  const Event& ev = l->events[event];
  if (new_row_cell >= ev.row.values.size() || !ev.row.values[new_row_cell].json) return -1;
  std::string o;
  json_dump(*ev.row.values[new_row_cell].json, o);
  if (buf && cap) { const size_t n = std::min<size_t>(o.size(), cap - 1); memcpy(buf, o.data(), n); buf[n] = 0; }
  return (int64_t)o.size();
}

}  // extern "C"
