#!/bin/bash
# Builds the CPU restatement of the hits aggregation (test infrastructure) into oracle/liboracle_hits.so, with the flags of oracle/build.sh.
set -e
cd "$(dirname "$0")"
g++ -std=c++17 -O3 -march=x86-64-v3 -ffp-contract=off -fPIC -shared -Wall -Wno-unused-function -pthread vlo_hits_api.cpp -o liboracle_hits.so -l:libzstd.so.1
echo built oracle/liboracle_hits.so
