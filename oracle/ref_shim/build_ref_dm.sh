#!/bin/bash
# The reference's descriptor matchers (oracle/ref_shim/vppref_dm.cc) against the Eigen / iod stand-ins of this directory, where
# the reference tree lies under /root/reference.  dm/ goes first: its iod/array_view.hh also takes a pointer.  Outputs only into
# oracle/_ref/ (git-ignored).
#   libvppref_dm.so      parity build: serial, -O2
#   libvppref_dm_omp.so  timing build: the reference's benchmark flags (benchmarks/CMakeLists.txt:10,18)
set -e
cd "$(dirname "$0")/../.."
mkdir -p oracle/_ref
g++ -std=c++14 -O2 -ffp-contract=off -fno-fast-math -fPIC -shared -w -I oracle/ref_shim/dm -I oracle/ref_shim -I /root/reference \
    -o oracle/_ref/libvppref_dm.so oracle/ref_shim/vppref_dm.cc
g++ -std=c++14 -O3 -march=native -fopenmp -DNDEBUG -ffp-contract=off -fPIC -shared -w -I oracle/ref_shim/dm -I oracle/ref_shim \
    -I /root/reference -o oracle/_ref/libvppref_dm_omp.so oracle/ref_shim/vppref_dm.cc
echo "built oracle/_ref/libvppref_dm{,_omp}.so from /root/reference"
