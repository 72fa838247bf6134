#!/bin/bash
# usage: tools/build_variant.sh NAME [extra nvcc flags...]  ->  seekstorm_b200/libseekstorm_b200_NAME.so (experiments; select with SSB_LIB=)
N=$1; shift
cd "$(dirname "$0")/.."
C=seekstorm_b200/csrc
/usr/local/cuda/bin/nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC,-ffp-contract=off -shared -ldl "$@" \
  -o seekstorm_b200/libseekstorm_b200_$N.so $C/api.cu $C/bm25.cu $C/facets.cu $C/comm.cu $C/loader.cu $C/vec_scan.cu $C/vec_scan_tc.cu $C/vec_refine.cu $C/vec_ivf.cu 2>&1 | grep -v "warning #177\|A_BYTES\|^$\|Remark"
ls -la seekstorm_b200/libseekstorm_b200_$N.so
