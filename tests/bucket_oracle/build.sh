#!/bin/bash
# Builds the CPU restatement of bucketed by-fields (test infrastructure) into tests/bucket_oracle/liboracle_bucket.so, with the flags of
# oracle/build.sh, over the oracle's headers and the sums restatement.
set -e
cd "$(dirname "$0")"
g++ -std=c++17 -O3 -march=x86-64-v3 -ffp-contract=off -fPIC -shared -Wall -Wno-unused-function -pthread -I../../oracle vlo_bucket_api.cpp -o liboracle_bucket.so -l:libzstd.so.1
echo built tests/bucket_oracle/liboracle_bucket.so
