#!/bin/bash
# Build every CUDA extension for sm_90a (cross-compiles without a GPU) and the CPU oracle.
set -e
cd "$(dirname "$0")"
mkdir -p vpp_b200/lib oracle/_build
nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++14 -fmad=false \
     -Xcompiler -fPIC -shared ${VPPB_NVCC_EXTRA} \
     -o vpp_b200/lib/libvppb.so vpp_b200/csrc/*.cu -ldl
gcc -O2 -ffp-contract=off -fno-fast-math -fPIC -shared -o oracle/_build/libvpp_oracle.so oracle/*.c -lm
gcc -O3 -march=native -fopenmp -DNDEBUG -ffp-contract=off -fPIC -shared -o oracle/_build/libvpp_oracle_omp.so oracle/*.c -lm
# C++14 host API tests (the reference's own tests rewritten with device kernels), run by tests/test_cpp_api.py on the GPU box
mkdir -p tests/cpp/_build
for t in core_tests algo_tests nbh_tests extruder_tests pw_bench dt_tests dm_tests sof_tests; do
  nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -std=c++14 --extended-lambda -O2 -fmad=false -I vpp_b200/include \
       -o tests/cpp/_build/$t tests/cpp/$t.cu -L vpp_b200/lib -lvppb -Xlinker -rpath -Xlinker '$ORIGIN/../../../vpp_b200/lib'
done
# the headers must also parse as plain C++14 host code (no nvcc): containers, options, algorithms
g++ -std=c++14 -fsyntax-only -I vpp_b200/include -I /usr/local/cuda/include tests/cpp/host_only.cc
g++ -std=c++14 -fsyntax-only -I vpp_b200/include -I /usr/local/cuda/include tests/cpp/dm_host_only.cc
g++ -std=c++14 -fsyntax-only -I vpp_b200/include -I /usr/local/cuda/include tests/cpp/sof_host_only.cc
echo "built vpp_b200/lib/libvppb.so oracle/_build/libvpp_oracle{,_omp}.so"
