#!/bin/bash
# Builds libgpushare_b200.so (sm_90a only) in-tree, plus the oracle's C pieces.
# Called by __graft_entry__.build(); safe to run on a GPU-less box (nvcc cross-compiles).
set -euo pipefail
cd "$(dirname "$0")"
PKG=gpushare_device_plugin_b200
SRC=$PKG/csrc
OUT=$PKG/libgpushare_b200.so
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
mkdir -p build
FLAGS="-gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -Xcompiler -fPIC,-Wall,-Wno-unused-function -cudart static"
$NVCC $FLAGS -Xptxas -v -c $SRC/hbm_probe_sm90a.cu -o build/hbm_probe_sm90a.o 2> build/ptxas_hbm_probe.log || { cat build/ptxas_hbm_probe.log; exit 1; }
$NVCC $FLAGS -c $SRC/gsb_device.cu -o build/gsb_device.o
g++ -O2 -std=c++17 -fPIC -Wall -c $SRC/gsb_wire.cc -o build/gsb_wire.o
g++ -O2 -std=c++17 -fPIC -Wall -c $SRC/gsb_fault.cc -o build/gsb_fault.o
$NVCC -shared -gencode arch=compute_90a,code=sm_90a -cudart static -o $OUT build/hbm_probe_sm90a.o build/gsb_device.o build/gsb_wire.o build/gsb_fault.o -ldl -lpthread -lrt
echo "built $OUT"
# native daemon (C++ host side: HTTP/2 + HPACK gRPC front end, kube client, manager loop) + its h2 self-test
g++ -O2 -std=c++17 -Wall -pthread -o $PKG/gsbd $SRC/daemon/gsbd.cc -L$PKG -lgpushare_b200 -lssl -lcrypto -ldl -Wl,-rpath,'$ORIGIN'
g++ -O2 -std=c++17 -Wall -pthread -o build/h2_selftest $SRC/daemon/h2_selftest.cc
g++ -O2 -std=c++17 -Wall -pthread -o $PKG/gsb_alloc_load $SRC/daemon/alloc_load.cc
g++ -O2 -std=c++17 -Wall -pthread -o $PKG/gsb_mock_kube $SRC/daemon/mock_kube.cc
echo "built $PKG/gsbd"
if [ -f oracle/Makefile ]; then make -s -C oracle; fi
