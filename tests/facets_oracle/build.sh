#!/bin/bash
# Builds the CPU restatement of the facets pipe (test infrastructure) into tests/facets_oracle/liboracle_facets.so, with the flags of
# oracle/build.sh, over the oracle's headers.
set -e
cd "$(dirname "$0")"
g++ -std=c++17 -O3 -march=x86-64-v3 -ffp-contract=off -fPIC -shared -Wall -Wno-unused-function -pthread -I../../oracle vlo_facets_api.cpp -o liboracle_facets.so -l:libzstd.so.1
echo built tests/facets_oracle/liboracle_facets.so
