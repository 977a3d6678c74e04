#!/bin/bash
# dev tool: build A/B variants of the step kernel (launch bounds / unroll: MINB_UNR, e.g. 2_2 3_1) into scratch libs;
# run one with DRB_LIB_PATH=daisyrec_b200/lib/variants/lib_<cfg>.so
set -e
cd "$(dirname "$0")/.."
python daisyrec_b200/_build.py >/dev/null
mkdir -p daisyrec_b200/lib/variants
for cfg in "$@"; do
  mb=${cfg%%_*}; un=${cfg##*_}
  nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo -Xcompiler -fPIC -DDRB_MINB=$mb -DDRB_UNR=$un \
       -c daisyrec_b200/csrc/mf_bpr.cu -o daisyrec_b200/lib/variants/mf_bpr_${cfg}.o &
done
wait
for cfg in "$@"; do
  nvcc -gencode arch=compute_90a,code=sm_90a -shared -cudart static -o daisyrec_b200/lib/variants/lib_${cfg}.so \
       daisyrec_b200/lib/variants/mf_bpr_${cfg}.o $(ls daisyrec_b200/lib/*.o | grep -v '/mf_bpr.o$') -ldl
  rm daisyrec_b200/lib/variants/mf_bpr_${cfg}.o
done
ls daisyrec_b200/lib/variants
