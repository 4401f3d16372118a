#!/bin/bash
# Build tagged variants of the library for the single-pass kernel sweep: tile K (rows per consumer thread), split S
# (ring items per column of a tile), ring depth NB (items) and resident CTAs per SM.
# usage: scripts/sweep_onepass.sh "tag:K:S:NB:CTAS" ...   e.g. k8s2n5:8:2:5:4
# then: DFD_LIB_TAG=<tag> python bench.py --no-e2e --no-cpu-baseline
set -e
cd "$(dirname "$0")/.."
for v in "$@"; do
  IFS=: read tag k s nb ctas <<< "$v"
  DFD_LIB_TAG=$tag DFD_NVCC_DEFS_ONEPASS="-DDFD_ONEPASS_K=$k -DDFD_ONEPASS_SPLIT=$s -DDFD_ONEPASS_NB=$nb -DDFD_ONEPASS_MIN_CTAS=$ctas" \
    python datafusion_distributed_b200/build.py > /dev/null &
done
wait
ls -la datafusion_distributed_b200/_lib/*.so
