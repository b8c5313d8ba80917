#!/bin/sh
# Builds tests/emu/libjss_emu.so (TEST-ONLY host emulation of the CUDA library).
set -e
HERE="$(cd "$(dirname "$0")" && pwd)"
ROOT="$HERE/../.."
g++ -O1 -g -std=c++17 -ffp-contract=off -fPIC -shared -U_FORTIFY_SOURCE -D_FORTIFY_SOURCE=0 -DJSS_EMU=1 \
    -I"$HERE" -I"$ROOT/jssenv_b200/csrc" -x c++ "$ROOT/jssenv_b200/csrc/jss_api.cu" \
    -x c++ "$ROOT/jssenv_b200/csrc/jss_host.cpp" -x c++ "$HERE/emu_runtime.cpp" \
    -x c++ "$HERE/emu_selftest.cpp" -o "$HERE/libjss_emu.so" -lpthread
