// host_cdc.cpp — TEST INFRASTRUCTURE ONLY.
// Compiles the DEVICE formatters of the emitter's CDC columns (etl_b200/csrc/arrow_format.cuh — the very source nvcc
// compiles for sm_90a) for the host, so that the CPU suite can fuzz them against a Python restatement of
// EventSequenceKey's Display (tests/test_arrow_cdc_cpu.py).  Nothing outside tests/ loads it.
#include <stdint.h>
#include <string.h>

#define __device__
#define __host__
#define __forceinline__ inline

#include "arrow_format.cuh"

// sequence key of (commit_lsn, tx_ordinal) into out (33 bytes)
extern "C" void emu_seq_key(uint64_t commit_lsn, uint64_t tx_ordinal, uint8_t* out) { etl_fmt::seq_key_write(commit_lsn, tx_ordinal, out); }
// cdc_operation of a record kind into op (6 bytes)
extern "C" void emu_cdc_op(uint32_t rec_kind, uint8_t* op) { etl_fmt::cdc_op_write(rec_kind, op); }
