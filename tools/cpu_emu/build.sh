#!/bin/bash
# Build the CPU emulation of omg_tools_b200/csrc/omg_b200.cu (test infrastructure).
#   build.sh [library name [extra compiler flags ...]]   (default: libomgb200_emu.so)
set -e
here="$(cd "$(dirname "$0")" && pwd)"
root="$(cd "$here/../.." && pwd)"
name="${1:-libomgb200_emu.so}"
shift $(( $# > 0 ? 1 : 0 ))
mkdir -p "$here/_build"
g++ -x c++ -std=c++20 -O1 -g -fPIC -shared -fno-strict-aliasing -Wno-attributes "$@" \
    -I "$here" -o "$here/_build/$name" \
    "$root/omg_tools_b200/csrc/omg_b200.cu" "$here/emu_runtime.cpp"
echo "built $here/_build/$name"
