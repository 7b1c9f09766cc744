#!/bin/bash
# Instrumentation build (timeline stamps in the decode-chain kernels): vita_b200/lib/libvita_b200_trace.so
set -e
cd "$(dirname "$0")/.."
python -m vita_b200.build > /dev/null
mkdir -p /tmp/vita_trobj
for f in api attention decode_tc; do
  nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo -Xcompiler -fPIC --expt-relaxed-constexpr \
       -DVITA_TRACE -c vita_b200/csrc/$f.cu -o /tmp/vita_trobj/$f.o
done
nvcc -shared -o vita_b200/lib/libvita_b200_trace.so \
     $(ls vita_b200/lib/obj/*.o | grep -v -E "/(api|attention|decode_tc)\.o") \
     /tmp/vita_trobj/api.o /tmp/vita_trobj/attention.o /tmp/vita_trobj/decode_tc.o \
     -gencode arch=compute_90a,code=sm_90a -lcudart
echo vita_b200/lib/libvita_b200_trace.so
