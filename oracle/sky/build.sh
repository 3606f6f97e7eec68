#!/bin/bash
# Compiles the sky restatement (sky.cpp, test infrastructure) into oracle/sky/libsky.so with the oracle's flags.
set -euo pipefail
HERE=$(cd "$(dirname "$0")" && pwd)
g++ -std=c++17 -O2 -fPIC -shared -ffp-contract=off -fno-fast-math -mfma -mavx2 -mf16c -Wall -Wno-unused-function \
    -Wno-unused-variable -Wno-unused-but-set-variable "$HERE/sky.cpp" -o "$HERE/libsky.so"
