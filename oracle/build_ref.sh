#!/usr/bin/env bash
# Build the UNMODIFIED reference rasterizer extension (yikaiw/Vidu4D,
# gs/submodules/diff-surfel-rasterization) for sm_90a (H100), straight from the
# reference checkout named by REF_ROOT, into oracle/_ref/ (git-ignored build
# product).  No reference source is copied: only the compiled pybind module
# `_C.so` lands in oracle/_ref/.
#
# This is TEST/BENCH INFRASTRUCTURE (the parity checker and the "reference arm"
# of bench.py).  Nothing in vidu4d_b200/ may import it.
#
# The only deviation from the reference's own setup.py is `-include cstdint`
# (rasterizer_impl.h:24 uses std::uintptr_t / uint32_t without the header; GCC 13
# rejects that) and an explicit -gencode for sm_90a.  Device-code flags are
# nvcc defaults (-O3, -fmad=true, IEEE div/sqrt), as setup.py:30 leaves them.
set -euo pipefail
REF=${REF_ROOT:-/root/reference}/gs/submodules/diff-surfel-rasterization
HERE=$(cd "$(dirname "$0")" && pwd)
OUT=$HERE/_ref
[ -d "$REF" ] || { echo "reference not present at $REF; keeping prebuilt oracle/_ref"; exit 0; }
mkdir -p "$OUT/obj"
PY=${PYTHON:-python}
read -r TORCH_INC TORCH_LIB PY_INC <<<"$($PY - <<'PYEOF'
import torch, sysconfig, os
from torch.utils.cpp_extension import include_paths
print(":".join(include_paths()), os.path.join(os.path.dirname(torch.__file__), "lib"), sysconfig.get_paths()["include"])
PYEOF
)"
INCS=""
IFS=':' read -ra PARTS <<<"$TORCH_INC"; for p in "${PARTS[@]}"; do INCS="$INCS -I$p"; done
COMMON="-std=c++17 -include cstdint -I$REF/third_party/glm/ -I$REF $INCS -I$PY_INC -I/usr/local/cuda/include \
 -DTORCH_EXTENSION_NAME=_C -DTORCH_API_INCLUDE_EXTENSION_H -D_GLIBCXX_USE_CXX11_ABI=1"
NVFLAGS="-gencode arch=compute_90a,code=sm_90a --expt-relaxed-constexpr -Xcompiler -fPIC -lineinfo \
 -D__CUDA_NO_HALF_OPERATORS__ -D__CUDA_NO_HALF_CONVERSIONS__ -D__CUDA_NO_BFLOAT16_CONVERSIONS__ -D__CUDA_NO_HALF2_OPERATORS__"
pids=()
for f in cuda_rasterizer/forward.cu cuda_rasterizer/backward.cu cuda_rasterizer/rasterizer_impl.cu rasterize_points.cu; do
  o=$OUT/obj/$(basename "${f%.cu}").o
  if [ ! -f "$o" ] || [ "$REF/$f" -nt "$o" ]; then
    nvcc $NVFLAGS $COMMON -c "$REF/$f" -o "$o" &
    pids+=($!)
  fi
done
o=$OUT/obj/ext.o
if [ ! -f "$o" ]; then g++ -O2 -fPIC $COMMON -c "$REF/ext.cpp" -o "$o" & pids+=($!); fi
for p in "${pids[@]}"; do wait "$p"; done
g++ -shared -o "$OUT/_C.so" "$OUT"/obj/*.o -L"$TORCH_LIB" -Wl,-rpath,"$TORCH_LIB" \
  -lc10 -ltorch -ltorch_cpu -ltorch_python -lc10_cuda -ltorch_cuda -L/usr/local/cuda/lib64 -lcudart
rm -rf "$OUT/obj"
echo "built $OUT/_C.so"
