#!/bin/bash
# Development build of the SAME source with the A/B knobs compiled in (-DB200_DEV_KNOBS: DevKnobs in plan.cuh reads the
# B200_* variables listed in DESIGN.md's appendix).  A/B scripts load it through B200BA_LIB; the
# product library (built by __graft_entry__.build()) reads none of them.
set -e
cd "$(dirname "$0")/../ceres_solver_b200/csrc"
nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC -shared -DB200_WITH_NCCL -DB200_DEV_KNOBS \
  -Xcompiler -fopenmp -o ../libb200ba_dev.so b200ba.cu -ldl -lgomp
echo "built ceres_solver_b200/libb200ba_dev.so"
