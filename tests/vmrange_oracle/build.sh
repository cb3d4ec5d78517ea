#!/bin/bash
# Builds the CPU restatement of `stats ... histogram(v)` (test infrastructure) into tests/vmrange_oracle/liboracle_vmrange.so, with the flags
# of oracle/build.sh, over the oracle's headers and the bucketed by-fields and sums restatements.
set -e
cd "$(dirname "$0")"
g++ -std=c++17 -O3 -march=x86-64-v3 -ffp-contract=off -fPIC -shared -Wall -Wno-unused-function -pthread -I../../oracle -I../bucket_oracle vlo_vmrange_api.cpp -o liboracle_vmrange.so -l:libzstd.so.1
echo built tests/vmrange_oracle/liboracle_vmrange.so
