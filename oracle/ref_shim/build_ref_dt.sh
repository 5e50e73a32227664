#!/bin/bash
# The reference's distance transforms (oracle/ref_shim/vppref_dt.cc) against the Eigen / iod stand-ins of this directory, where the
# reference tree lies under /root/reference.  Outputs only into oracle/_ref/ (git-ignored).
#   libvppref_dt.so      parity build: serial, -O2
#   libvppref_dt_omp.so  timing build: the reference's benchmark flags (benchmarks/CMakeLists.txt:10,18)
set -e
cd "$(dirname "$0")/../.."
mkdir -p oracle/_ref
g++ -std=c++14 -O2 -ffp-contract=off -fno-fast-math -fPIC -shared -w -I oracle/ref_shim -I /root/reference \
    -o oracle/_ref/libvppref_dt.so oracle/ref_shim/vppref_dt.cc
g++ -std=c++14 -O3 -march=native -fopenmp -DNDEBUG -ffp-contract=off -fPIC -shared -w -I oracle/ref_shim -I /root/reference \
    -o oracle/_ref/libvppref_dt_omp.so oracle/ref_shim/vppref_dt.cc
echo "built oracle/_ref/libvppref_dt{,_omp}.so from /root/reference"
