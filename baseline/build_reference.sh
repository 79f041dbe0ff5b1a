#!/bin/sh
# Build the UNMODIFIED reference (a pytorch/gloo checkout, given as $1) for sm_90 and install
# its benchmark binaries into baseline/_ref/bin. The reference's own arch table stops at
# sm_86 and is empty for CUDA >= 12 (cmake/Cuda.cmake:154-164), so the architecture is
# injected from outside; nothing in the source tree is touched (built from a /tmp copy).
set -e
HERE="$(cd "$(dirname "$0")" && pwd)"
SRC=${1:?usage: build_reference.sh <pytorch/gloo checkout>}
rm -rf /tmp/refsrc /tmp/refbuild
cp -r "$SRC" /tmp/refsrc
mkdir -p /tmp/refbuild "$HERE/_ref/bin"
cd /tmp/refbuild
cmake /tmp/refsrc -G Ninja -DCMAKE_BUILD_TYPE=Release -DUSE_CUDA=ON -DGLOO_USE_CUDA_TOOLKIT=ON \
  -DUSE_NCCL=ON -DBUILD_BENCHMARK=ON -DCMAKE_CUDA_ARCHITECTURES=90 \
  -DCMAKE_CUDA_COMPILER=/usr/local/cuda/bin/nvcc
ninja -j"$(nproc)"
cp gloo/benchmark/benchmark gloo/benchmark/benchmark_cuda "$HERE/_ref/bin/"
echo "installed: $HERE/_ref/bin"
# End-to-end driver (pinned host -> GPU -> stock CudaAllreduceRingChunked::run() -> pinned host)
# linked against the reference's own, unmodified static libraries.
g++ -O2 -std=c++17 "$HERE/ref_e2e.cc" -I/tmp/refsrc -I/tmp/refbuild -I/usr/local/cuda/include \
  /tmp/refbuild/gloo/libgloo_cuda.a /tmp/refbuild/gloo/libgloo.a \
  -L/usr/local/cuda/lib64 -Wl,-rpath,/usr/local/cuda/lib64 -lcudart -lnccl -lpthread -ldl \
  -o "$HERE/_ref/bin/ref_e2e"
echo "installed: $HERE/_ref/bin/ref_e2e"
