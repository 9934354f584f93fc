// host_format.cpp — TEST INFRASTRUCTURE ONLY.
// Compiles the DEVICE formatters of the columnar emitter (etl_b200/csrc/arrow_format.cuh — the very source nvcc compiles
// for sm_90a) for the host, so that the CPU suite can fuzz them against Python restatements of PgNumeric's and
// serde_json's Display (tests/test_arrow_format_cpu.py).  Nothing outside tests/ loads it.
#include <stdint.h>
#include <string.h>

#include <vector>

#define __device__
#define __host__
#define __forceinline__ inline

#include "arrow_format.cuh"

// numeric at `num` (etl_numeric_hdr + digits, as the heap holds it): Display text into out (cap bytes); returns the
// length numeric_len predicted, or -1 when numeric_write wrote a different number of bytes
extern "C" int64_t emu_numeric_text(const uint8_t* num, uint32_t nd, uint8_t* out, uint32_t cap) {
  alignas(8) static thread_local uint8_t buf[1 << 17];
  const uint32_t in_bytes = 8u + 2u * nd;
  if (in_bytes > sizeof buf) return -2;
  memcpy(buf, num, in_bytes);
  const uint32_t n = etl_fmt::numeric_len(buf, nd);
  if (n > cap) return -2;
  const uint32_t w = etl_fmt::numeric_write(buf, nd, out);
  return w == n ? (int64_t)n : -1;
}

// canonical text of one JSON document into out (n bytes of room: never longer than the input); -1 = rejected
extern "C" int64_t emu_json_canon(const uint8_t* s, uint32_t n, uint8_t* out) {
  std::vector<uint8_t> in(s, s + n);                   // exact-size copies: an overrun shows up under a sanitizer
  std::vector<uint32_t> work((size_t)etl_fmt::json_canon_work_words(n));
  const uint32_t r = etl_fmt::json_canon(in.data(), n, out, work.data());
  return r == etl_fmt::kJsonCanonBad ? -1 : (int64_t)r;
}
