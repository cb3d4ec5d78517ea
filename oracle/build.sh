#!/bin/bash
# Builds the CPU oracle (test infrastructure) into oracle/liboracle.so.
# -O3 -march=x86-64-v3 (AVX2; every host this runs on has it) with FP contraction off: the value parsers must round like the reference.
# zstd: linked against the image's libzstd.so.1 (prototypes declared in vlo_util.h; no zstd.h in the image).
set -e
cd "$(dirname "$0")"
g++ -std=c++17 -O3 -march=x86-64-v3 -ffp-contract=off -fPIC -shared -Wall -Wno-unused-function -pthread vlo_api.cpp -o liboracle.so -l:libzstd.so.1
echo built oracle/liboracle.so
# The same restatement linked against the REFERENCE'S OWN libzstd (v1.5.7 static library vendored under gozstd, the one the Go binary links):
# the CPU arm of bench.py then decompresses with exactly the reference's ZSTD build.  Only where the reference tree exists; output goes to
# oracle/_ref/ (git-ignored; bench.py falls back to the system libzstd build when it is absent).
REFZSTD=/root/reference/vendor/github.com/valyala/gozstd/libzstd_linux_amd64.a
if [ -f "$REFZSTD" ]; then
    mkdir -p _ref
    g++ -std=c++17 -O3 -march=x86-64-v3 -ffp-contract=off -fPIC -shared -Wall -Wno-unused-function -pthread vlo_api.cpp -o _ref/liboracle_zstd157.so "$REFZSTD"
    echo built oracle/_ref/liboracle_zstd157.so
fi
