#!/bin/bash
# usage: tools/build_variant.sh NAME [extra nvcc flags...]  ->  seekstorm_b200/libseekstorm_b200_NAME.so (experiments; select with SSB_LIB=)
N=$1; shift
cd "$(dirname "$0")/.."
SRCS=$(python3 -c "import __graft_entry__ as g; print(' '.join('seekstorm_b200/csrc/' + s for s in g.SOURCES))")
/usr/local/cuda/bin/nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC,-ffp-contract=off -shared -ldl "$@" \
  -o seekstorm_b200/libseekstorm_b200_$N.so $SRCS 2>&1 | grep -v "warning #177\|A_BYTES\|^$\|Remark"
ls -la seekstorm_b200/libseekstorm_b200_$N.so
