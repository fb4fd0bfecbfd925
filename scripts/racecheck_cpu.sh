#!/bin/sh
# compute-sanitizer racecheck without a GPU: the SIMT kernels (persistent MLP, elementwise, comm, conv, and the wgmma GEMM on its functional model) compiled for the CPU
# through csrc/host_shim.h with -fsanitize=thread and run on small workloads.  Exit code 0 = no data race reported.
#   sh scripts/racecheck_cpu.sh [build-dir]
set -e
ROOT=$(cd "$(dirname "$0")/.." && pwd)
CSRC="$ROOT/colearn_federated_learning_b200/ops/csrc"
OUT=${1:-/tmp/colearn_racecheck}
mkdir -p "$OUT"
CUDA_INC=${CUDA_HOME:-/usr/local/cuda}/include
FLAGS="-std=c++20 -O1 -g -fsanitize=thread -pthread -Wno-unknown-pragmas -Wno-tsan -DCOLEARN_HOST_SHIM=1 -I$CSRC -I$CUDA_INC"
for f in simt_mlp simt_mlp_ae simt_mlp_cat simt_mlp_cw simt_mlp_opt simt_elementwise simt_comm simt_convnet simt_gemm simt_racecheck; do
  g++ $FLAGS -c "$CSRC/$f.cpp" -o "$OUT/$f.o" &
done
wait
g++ -fsanitize=thread -pthread "$OUT"/simt_mlp.o "$OUT"/simt_mlp_ae.o "$OUT"/simt_mlp_cat.o "$OUT"/simt_mlp_cw.o "$OUT"/simt_mlp_opt.o "$OUT"/simt_elementwise.o "$OUT"/simt_comm.o "$OUT"/simt_convnet.o "$OUT"/simt_gemm.o "$OUT"/simt_racecheck.o -o "$OUT/racecheck"
TSAN_OPTIONS="halt_on_error=0 exitcode=66 second_deadlock_stack=1" "$OUT/racecheck"
