#!/bin/bash
# Builds the CPU restatement of `stats ... sum(v), avg(v)` (test infrastructure) into tests/stats_oracle/liboracle_stats.so, with the flags of
# oracle/build.sh, over the oracle's headers.
set -e
cd "$(dirname "$0")"
g++ -std=c++17 -O3 -march=x86-64-v3 -ffp-contract=off -fPIC -shared -Wall -Wno-unused-function -pthread -I../../oracle vlo_stats_api.cpp -o liboracle_stats.so -l:libzstd.so.1
echo built tests/stats_oracle/liboracle_stats.so
