#!/bin/bash
# Build the CPU simulator of the product library (TEST / DEVELOPMENT TOOL, see tests/host/):
#   build/libpbc_b200_sim.so  -- engine.cu + every kernel compiled for the host, same C ABI
# Use it wherever the real library would be loaded:
#   PBC_B200_LIB=$PWD/build/libpbc_b200_sim.so python -m pytest tests/test_gpu_type_a1.py -m gpu -k "not across_blocks"
set -e
cd "$(dirname "$0")/.."
mkdir -p build
python tests/host/make_host_sim.py build/host_sim.cpp "$@"
g++ -O1 -std=c++17 -shared -fPIC -Wno-unknown-pragmas -pthread -o build/libpbc_b200_sim.so build/host_sim.cpp
ls -la build/libpbc_b200_sim.so
