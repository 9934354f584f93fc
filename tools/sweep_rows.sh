#!/bin/bash
# k_rows geometry sweep (variants built with ETL_LIB_SUFFIX / ETL_NVCC_DEFS, see etl_b200/build.py)
for v in "" _b _c; do
  for wl in "c2 1.0" "c3 0.3" "c4 0.3" "c5 0.5"; do
    echo "== variant '${v}' $wl"
    ETL_LIB_SUFFIX=$v python tools/run_decode.py $wl 5 2>&1 | tail -n 1
  done
done
