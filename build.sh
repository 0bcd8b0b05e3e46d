#!/bin/bash
# Builds soilmachine_b200/lib/libsoilmachine_b200.so for sm_90a (H100), in-tree.  Variant builds (-DSM_PROFILE,
# -DSM_AUDIT_HANDOFF, passed as arguments) go where SM_LIB_OUT says.
set -e
cd "$(dirname "$0")"
mkdir -p soilmachine_b200/lib
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
# -fmad=false : no FMA contraction (bit parity with the reference's x86-64 SSE2 arithmetic)
# -dlcm=cg    : global loads go to L2 (L1 is not coherent across the SMs that share a column)
# -DSM_ACQREL : hand-off with ld.acquire/st.release instead of full fences
timeout ${SM_BUILD_TIMEOUT:-900} $NVCC -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 \
  -fmad=false -DSM_ACQREL -diag-suppress 20011,20014 -Xptxas -dlcm=cg ${SM_PTXAS_V:+-Xptxas -v} -Xcompiler -fPIC -Xcompiler -ffp-contract=off -shared \
  -o "${SM_LIB_OUT:-soilmachine_b200/lib/libsoilmachine_b200.so}" soilmachine_b200/csrc/sm_engine.cu "$@"
