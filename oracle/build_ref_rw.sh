#!/usr/bin/env bash
# oracle/build_ref_rw.sh — compile the REFERENCE's own CUDA random walker (pyg::random_walk: its schema,
# pyg_lib/csrc/sampler/random_walk.cpp, and its CUDA kernel, sampler/cuda/random_walk_kernel.cu) straight from the
# sources where they lie under /root/reference, with nvcc for sm_90a, into oracle/_ref/libpyg_ref_rw.so.
#
# TEST INFRASTRUCTURE ONLY.  Output goes to oracle/_ref/ (git-ignored; the prebuilt .so travels to the GPU machine).
# No reference source is copied into this repo.  libpyg.so defines the same schema, so oracle/ref_random_walk.py
# loads this library in a child process.
set -euo pipefail
REF=${REF:-/root/reference}
HERE=$(cd "$(dirname "$0")" && pwd)
OUT="$HERE/_ref"
[ -d "$REF/pyg_lib/csrc" ] || { echo "no reference tree at $REF; keeping prebuilt $OUT" >&2; exit 0; }
mkdir -p "$OUT/obj"
PY=${PYTHON:-python}
CUDA_HOME=${CUDA_HOME:-/usr/local/cuda}
TORCH_DIR=$($PY -c 'import torch,os;print(os.path.dirname(torch.__file__))')
PYINC=$($PY -c 'import sysconfig;print(sysconfig.get_paths()["include"])')
ABI=$($PY -c 'import torch;print(int(torch._C._GLIBCXX_USE_CXX11_ABI))')
INC="-I$REF -I$TORCH_DIR/include -I$TORCH_DIR/include/torch/csrc/api/include -I$PYINC"
RW_CPP=pyg_lib/csrc/sampler/random_walk.cpp
RW_CU=pyg_lib/csrc/sampler/cuda/random_walk_kernel.cu
if [ ! -f "$OUT/obj/rw_schema.o" ] || [ "$REF/$RW_CPP" -nt "$OUT/obj/rw_schema.o" ]; then
  g++ -O3 -fPIC -std=c++17 -w -D_GLIBCXX_USE_CXX11_ABI=$ABI $INC -c "$REF/$RW_CPP" -o "$OUT/obj/rw_schema.o"
fi
if [ ! -f "$OUT/obj/rw_kernel.o" ] || [ "$REF/$RW_CU" -nt "$OUT/obj/rw_kernel.o" ]; then
  "$CUDA_HOME/bin/nvcc" -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -w -Xcompiler -fPIC \
    -D_GLIBCXX_USE_CXX11_ABI=$ABI $INC -c "$REF/$RW_CU" -o "$OUT/obj/rw_kernel.o"
fi
g++ -shared -o "$OUT/libpyg_ref_rw.so" "$OUT/obj/rw_schema.o" "$OUT/obj/rw_kernel.o" \
  -L"$TORCH_DIR/lib" -ltorch -ltorch_cpu -ltorch_cuda -lc10 -lc10_cuda -L"$CUDA_HOME/lib64" -lcudart \
  -Wl,-rpath,"$TORCH_DIR/lib" -Wl,-rpath,"$CUDA_HOME/lib64"
echo "built $OUT/libpyg_ref_rw.so"
