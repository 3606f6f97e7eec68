#!/bin/bash
# Compiles the ReSTIR PT debug-view restatement (rpt_views.cpp, test infrastructure) into oracle/rpt_views/librpt_views.so with the
# oracle's flags.
set -euo pipefail
HERE=$(cd "$(dirname "$0")" && pwd)
g++ -std=c++17 -O2 -fPIC -shared -ffp-contract=off -fno-fast-math -mfma -mavx2 -mf16c -Wall -Wno-unused-function \
    -Wno-unused-variable -Wno-unused-but-set-variable "$HERE/rpt_views.cpp" -o "$HERE/librpt_views.so"
