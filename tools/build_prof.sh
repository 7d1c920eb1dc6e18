#!/bin/bash
# development build with clock64() accounting of the full body: jiminy_b200/libjiminy_b200_prof.so (never the product library)
cd "$(dirname "$0")/.."
/usr/local/cuda/bin/nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -Xcompiler -fPIC -shared -DJB_PROFILE_CLOCKS=1 \
    -ccbin /usr/bin/g++ -Iinclude -o jiminy_b200/libjiminy_b200_prof.so jiminy_b200/csrc/jb_capi.cu jiminy_b200/csrc/jb_plan.cpp
