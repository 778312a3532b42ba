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
$NVCC $FLAGS -Xptxas -v -c $SRC/sm_check_sm90a.cu -o build/sm_check_sm90a.o 2> build/ptxas_sm_check.log || { cat build/ptxas_sm_check.log; exit 1; }
$NVCC $FLAGS -Xptxas -v -c $SRC/mma_operands_sm90a.cu -o build/mma_operands_sm90a.o 2> build/ptxas_mma_operands.log || { cat build/ptxas_mma_operands.log; exit 1; }
$NVCC $FLAGS -Xptxas -v -c $SRC/sm_stress_sm90a.cu -o build/sm_stress_sm90a.o 2> build/ptxas_sm_stress.log || { cat build/ptxas_sm_stress.log; exit 1; }
$NVCC $FLAGS -Xptxas -v -c $SRC/cluster_check_sm90a.cu -o build/cluster_check_sm90a.o 2> build/ptxas_cluster_check.log || { cat build/ptxas_cluster_check.log; exit 1; }
$NVCC $FLAGS -Xptxas -v -c $SRC/cluster_script_sm90a.cu -o build/cluster_script_sm90a.o 2> build/ptxas_cluster_script.log || { cat build/ptxas_cluster_script.log; exit 1; }
$NVCC $FLAGS -Xptxas -v -c $SRC/atomic_check_sm90a.cu -o build/atomic_check_sm90a.o 2> build/ptxas_atomic_check.log || { cat build/ptxas_atomic_check.log; exit 1; }
$NVCC $FLAGS -Xptxas -v -c $SRC/atomic_values_sm90a.cu -o build/atomic_values_sm90a.o 2> build/ptxas_atomic_values.log || { cat build/ptxas_atomic_values.log; exit 1; }
$NVCC $FLAGS -Xptxas -v -c $SRC/tensor_check_sm90a.cu -o build/tensor_check_sm90a.o 2> build/ptxas_tensor_check.log || { cat build/ptxas_tensor_check.log; exit 1; }
$NVCC $FLAGS -Xptxas -v -c $SRC/tensor_operands_sm90a.cu -o build/tensor_operands_sm90a.o 2> build/ptxas_tensor_operands.log || { cat build/ptxas_tensor_operands.log; exit 1; }
$NVCC $FLAGS -Xptxas -v -c $SRC/sfu_check_sm90a.cu -o build/sfu_check_sm90a.o 2> build/ptxas_sfu_check.log || { cat build/ptxas_sfu_check.log; exit 1; }
$NVCC $FLAGS -Xptxas -v -c $SRC/sfu_operands_sm90a.cu -o build/sfu_operands_sm90a.o 2> build/ptxas_sfu_operands.log || { cat build/ptxas_sfu_operands.log; exit 1; }
$NVCC $FLAGS -Xptxas -v -c $SRC/order_check_sm90a.cu -o build/order_check_sm90a.o 2> build/ptxas_order_check.log || { cat build/ptxas_order_check.log; exit 1; }
$NVCC $FLAGS -Xptxas -v -c $SRC/sparse_check_sm90a.cu -o build/sparse_check_sm90a.o 2> build/ptxas_sparse_check.log || { cat build/ptxas_sparse_check.log; exit 1; }
$NVCC $FLAGS -Xptxas -v -c $SRC/sparse_operands_sm90a.cu -o build/sparse_operands_sm90a.o 2> build/ptxas_sparse_operands.log || { cat build/ptxas_sparse_operands.log; exit 1; }
$NVCC $FLAGS -Xptxas -v -c $SRC/shared_atomic_check_sm90a.cu -o build/shared_atomic_check_sm90a.o 2> build/ptxas_shared_atomic_check.log || { cat build/ptxas_shared_atomic_check.log; exit 1; }
$NVCC $FLAGS -Xptxas -v -c $SRC/l1_check_sm90a.cu -o build/l1_check_sm90a.o 2> build/ptxas_l1_check.log || { cat build/ptxas_l1_check.log; exit 1; }
$NVCC $FLAGS -Xptxas -v -c $SRC/l1_table_sm90a.cu -o build/l1_table_sm90a.o 2> build/ptxas_l1_table.log || { cat build/ptxas_l1_table.log; exit 1; }
# the L1 and constant-cache check's kernels are a module of their own: its 64 KiB __constant__ bank fills the whole user
# bank of the module that declares it, and the kernels of libgpushare_b200.so keep their recorded SASS; their test-only
# twins (l1_table_sm90a.cu, a CUDA module of its own with its own bank) go into the same library
$NVCC -shared -gencode arch=compute_90a,code=sm_90a -cudart static -o $PKG/libgpushare_b200_l1.so build/l1_check_sm90a.o build/l1_table_sm90a.o
# the memory-ordering check's kernel is a module of its own too: the kernel set of libgpushare_b200.so and of the L1
# module is pinned with its recorded SASS (tests/golden/shipped_kernels_sass.json)
$NVCC -shared -gencode arch=compute_90a,code=sm_90a -cudart static -o $PKG/libgpushare_b200_order.so build/order_check_sm90a.o
# the SM-to-SM check's test-only twins likewise: the shipped cluster_check kernels stay in the main library, whose
# recorded kernel set the twins leave as it is; the twins are pinned in tests/golden/cluster_script_sass.json
$NVCC -shared -gencode arch=compute_90a,code=sm_90a -cudart static -o $PKG/libgpushare_b200_cluster_script.so build/cluster_script_sm90a.o
# the sparse tensor-core check's kernels and their test-only twins likewise: a module of their own, so the recorded
# kernel sets of the other libraries stay as they are
$NVCC -shared -gencode arch=compute_90a,code=sm_90a -cudart static -o $PKG/libgpushare_b200_sparse.so build/sparse_check_sm90a.o build/sparse_operands_sm90a.o
# the shared-memory atomic check's kernels likewise
$NVCC -shared -gencode arch=compute_90a,code=sm_90a -cudart static -o $PKG/libgpushare_b200_shared_atomic.so build/shared_atomic_check_sm90a.o
$NVCC $FLAGS -c $SRC/gsb_device.cu -o build/gsb_device.o
g++ -O2 -std=c++17 -fPIC -Wall -c $SRC/gsb_wire.cc -o build/gsb_wire.o
g++ -O2 -std=c++17 -fPIC -Wall -c $SRC/gsb_fault.cc -o build/gsb_fault.o
g++ -O2 -std=c++17 -fPIC -Wall -c $SRC/gsb_ecc.cc -o build/gsb_ecc.o
g++ -O2 -std=c++17 -fPIC -Wall -c $SRC/gsb_memtest.cc -o build/gsb_memtest.o
g++ -O2 -std=c++17 -fPIC -Wall -c $SRC/gsb_link.cc -o build/gsb_link.o
g++ -O2 -std=c++17 -fPIC -Wall -c $SRC/gsb_copy.cc -o build/gsb_copy.o
g++ -O2 -std=c++17 -fPIC -Wall -c $SRC/gsb_sm.cc -o build/gsb_sm.o
g++ -O2 -std=c++17 -fPIC -Wall -c $SRC/gsb_stress.cc -o build/gsb_stress.o
g++ -O2 -std=c++17 -fPIC -Wall -c $SRC/gsb_cluster.cc -o build/gsb_cluster.o
g++ -O2 -std=c++17 -fPIC -Wall -c $SRC/gsb_atomic.cc -o build/gsb_atomic.o
g++ -O2 -std=c++17 -fPIC -Wall -c $SRC/gsb_tensor.cc -o build/gsb_tensor.o
g++ -O2 -std=c++17 -fPIC -Wall -c $SRC/gsb_sfu.cc -o build/gsb_sfu.o
g++ -O2 -std=c++17 -fPIC -Wall -c $SRC/gsb_l1.cc -o build/gsb_l1.o
g++ -O2 -std=c++17 -fPIC -Wall -c $SRC/gsb_order.cc -o build/gsb_order.o
g++ -O2 -std=c++17 -fPIC -Wall -c $SRC/gsb_sparse.cc -o build/gsb_sparse.o
g++ -O2 -std=c++17 -fPIC -Wall -c $SRC/gsb_shared_atomic.cc -o build/gsb_shared_atomic.o
$NVCC -shared -gencode arch=compute_90a,code=sm_90a -cudart static -o $OUT build/hbm_probe_sm90a.o build/sm_check_sm90a.o build/mma_operands_sm90a.o build/sm_stress_sm90a.o build/cluster_check_sm90a.o build/atomic_check_sm90a.o build/atomic_values_sm90a.o build/tensor_check_sm90a.o build/tensor_operands_sm90a.o build/sfu_check_sm90a.o build/sfu_operands_sm90a.o build/gsb_device.o build/gsb_wire.o build/gsb_fault.o build/gsb_ecc.o build/gsb_memtest.o build/gsb_link.o build/gsb_copy.o build/gsb_sm.o build/gsb_stress.o build/gsb_cluster.o build/gsb_atomic.o build/gsb_tensor.o build/gsb_sfu.o build/gsb_l1.o build/gsb_order.o build/gsb_sparse.o build/gsb_shared_atomic.o -L$PKG -lgpushare_b200_l1 -lgpushare_b200_order -lgpushare_b200_cluster_script -lgpushare_b200_sparse -lgpushare_b200_shared_atomic -Xlinker -rpath,'$ORIGIN' -ldl -lpthread -lrt
echo "built $OUT"
# native daemon (C++ host side: HTTP/2 + HPACK gRPC front end, kube client, manager loop) + its h2 self-test
g++ -O2 -std=c++17 -Wall -pthread -o $PKG/gsbd $SRC/daemon/gsbd.cc -L$PKG -lgpushare_b200 -lssl -lcrypto -ldl -Wl,-rpath,'$ORIGIN'
g++ -O2 -std=c++17 -Wall -pthread -o build/h2_selftest $SRC/daemon/h2_selftest.cc
g++ -O2 -std=c++17 -Wall -pthread -o $PKG/gsb_alloc_load $SRC/daemon/alloc_load.cc
g++ -O2 -std=c++17 -Wall -pthread -o $PKG/gsb_mock_kube $SRC/daemon/mock_kube.cc
echo "built $PKG/gsbd"
if [ -f oracle/Makefile ]; then make -s -C oracle; fi
