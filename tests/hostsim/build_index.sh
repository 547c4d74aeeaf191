#!/bin/bash
# Test infrastructure only: builds htslib_b200/csrc/cram_index.cu, with the record decoder it runs (cram_records.cu, cram_encode.cu), a
# second time FOR THE HOST (g++ -DHGPU_HOSTSIM: the slice decode and cram_index_runs_kernel become loops over the same
# __host__ __device__ code) so that tests/test_cram_index_reference.py checks the whole CRAI path against the compiled
# reference where no GPU exists.  Nothing in htslib_b200/ loads this library.
set -euo pipefail
HERE=$(cd "$(dirname "$0")" && pwd)
ROOT=$(cd "$HERE/../.." && pwd)
mkdir -p "$HERE/_build"
g++ -O1 -g -std=c++17 -fPIC -shared -DHGPU_HOSTSIM -x c++ "$ROOT/htslib_b200/csrc/cram_records.cu" "$ROOT/htslib_b200/csrc/cram_encode.cu" \
    "$ROOT/htslib_b200/csrc/cram_index.cu" -I"$ROOT/include" \
    -o "$HERE/_build/libcramidx_hostsim.so" -L"$ROOT/htslib_b200" -lhtsgpu '-Wl,-rpath,$ORIGIN/../../../htslib_b200'
echo "built $HERE/_build/libcramidx_hostsim.so"
