// host_parquet_zstd.cpp — TEST INFRASTRUCTURE ONLY.
// Compiles the Zstandard block compressor of the Parquet writer (etl_b200/csrc/zstd_format.cuh — the very source nvcc
// compiles for sm_90a) for the host, so that the CPU suite can decode its frames with pyarrow's libzstd and compare the
// device's pages with it byte for byte (tests/test_parquet_zstd_cpu.py, tests/test_gpu_parquet_zstd.py).  Nothing
// outside tests/ loads it.
#include <stdint.h>
#include <stdlib.h>

#define __device__
#define __host__
#define __forceinline__ inline

#include "zstd_format.cuh"

static const uint32_t kFragment = 65536;   // the Parquet writer's fragment (parquet_format.cuh)

// the frame bound of n bytes: header + one block slot per fragment (one for n == 0)
extern "C" uint64_t emu_zstd_bound(uint64_t n) {
  const uint64_t nf = n ? (n + kFragment - 1) / kFragment : 1;
  return etl_zstd::kFrameHeader + n + 3 * nf;
}
// one frame of in[0..n): the header, then a block per 64 KiB fragment, Last_Block on the last; out has
// emu_zstd_bound(n) bytes.  Returns its length.
extern "C" uint64_t emu_zstd(const uint8_t* in, uint64_t n, uint8_t* out) {
  etl_zstd::Work* W = (etl_zstd::Work*)malloc(sizeof(etl_zstd::Work));
  uint8_t* lit = (uint8_t*)malloc(kFragment);
  uint64_t* seq = (uint64_t*)malloc(8 * etl_zstd::zstd_seqs(kFragment));
  uint64_t o = etl_zstd::frame_header((uint32_t)n, out);
  uint64_t off = 0;
  do {
    const uint32_t len = (uint32_t)(n - off < kFragment ? n - off : kFragment);
    o += etl_zstd::zstd_block(in + off, len, off + len >= n, out + o, *W, lit, seq);
    off += len;
  } while (off < n);
  free(seq);
  free(lit);
  free(W);
  return o;
}
