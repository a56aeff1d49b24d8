# usage: scripts/build_variant.sh NAME UNIT.cu "-DFOO=1 -DBAR=2"   -> ggrmcp_b200/variants/libggrmcp_b200_NAME.so (for GGR_LIB=...)
set -e
cd "$(dirname "$0")/.."
mkdir -p ggrmcp_b200/variants
obj=ggrmcp_b200/variants/$1_$(basename $2 .cu).o
/usr/local/cuda/bin/nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC -Iinclude $3 -c -o $obj ggrmcp_b200/csrc/$2
others=$(ls ggrmcp_b200/build/*.o | grep -v "/$(basename $2 .cu).o")
/usr/local/cuda/bin/nvcc -shared -o ggrmcp_b200/variants/libggrmcp_b200_$1.so $obj $others 2>/dev/null
ls -la ggrmcp_b200/variants/libggrmcp_b200_$1.so
