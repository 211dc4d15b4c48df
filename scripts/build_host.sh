#!/bin/bash
# Build the three host executables (TestSimulation, RunHardware, PrintSpecifications) with g++ against the
# in-tree libmm_b200.so, without CMake.
#   usage: bash scripts/build_host.sh [outdir] [float|double|half|int|...] [Multiply|Add|...] [Add|Min|...]
#   MM_STATIC_SIZES="N K M" in the environment builds the MM_DYNAMIC_SIZES=OFF flavour (sizes fixed at
#   compile time, executables take no N K M arguments), as the reference's CMake option does.
#   MM_HOST_EXACT=1 / MM_HOST_HALF_TENSOR=1 = the CMake options -DMM_EXACT=ON / -DMM_HALF_TENSOR=ON.
# MM_NUM_GPUS=G at run time splits the call over G GPUs inside libmm_b200.so (no NCCL needed).
set -e
R=$(cd "$(dirname "$0")/.." && pwd)
OUT=${1:-/tmp/hostbuild}; TYPE=${2:-float}; MAP=${3:-Multiply}; RED=${4:-Add}
mkdir -p "$OUT"
read -r SN SK SM <<< "${MM_STATIC_SIZES:-512 512 512}"
python - "$R" "$OUT" "$TYPE" "$MAP" "$RED" "$SN" "$SK" "$SM" <<'PY'
import re, sys
root, out, typ, mp, rd = sys.argv[1:6]
sn, sk, sm = map(int, sys.argv[6:9])
code = {"half": "HALF", "float": "FLOAT", "double": "DOUBLE", "int": "INT32", "unsigned": "UINT32", "uint8_t": "UINT8"}[typ]
size = {"half": 2, "float": 4, "double": 8, "int": 4, "unsigned": 4, "uint8_t": 1}[typ]
up = {"Multiply": "MULTIPLY", "Add": "ADD", "Min": "MIN", "Max": "MAX", "And": "AND"}
cfg = dict(MM_HOST_DATA_TYPE=typ, MM_DATA_TYPE=typ, MM_DTYPE_CODE="MM_DTYPE_" + code,
           MM_MAP_OP_UPPER=up[mp], MM_MAP_OP=mp, MM_REDUCE_OP_UPPER=up[rd], MM_REDUCE_OP=rd,
           MM_MEMORY_BUS_WIDTH_K=64, MM_MEMORY_BUS_WIDTH_M=64, MM_SIZE_N=sn, MM_SIZE_K=sk, MM_SIZE_M=sm,
           MM_MEMORY_TILE_SIZE_N=128, MM_MEMORY_TILE_SIZE_M=256)
t = open(root + "/gemm_hls_b200/host/Config.h.in").read()
missing = set(re.findall(r"\$\{(\w+)\}", t)) - set(cfg)
assert not missing, "Config.h.in variables without a value: %s" % sorted(missing)
import os
t = re.sub(r"\$\{(\w+)\}", lambda m: str(cfg[m.group(1)]), t)
for opt in ("MM_EXACT", "MM_HALF_TENSOR"):   # MM_HOST_EXACT=1 / MM_HOST_HALF_TENSOR=1 = the CMake options -DMM_EXACT=ON / -DMM_HALF_TENSOR=ON
    on = os.environ.get(opt.replace("MM_", "MM_HOST_"), "") not in ("", "0")
    t = t.replace("#cmakedefine " + opt, ("#define " + opt) if on else ("/* #undef %s */" % opt))
open(out + "/Config.h", "w").write(t)
PY
cd "$OUT"
DYN="-DMM_DYNAMIC_SIZES"; [ -n "$MM_STATIC_SIZES" ] && DYN=""
COMMON="-std=c++17 -O2 $DYN -I. -I$R/include -I$R/gemm_hls_b200/host -L$R/gemm_hls_b200 -lmm_b200 -Wl,-rpath,$R/gemm_hls_b200 -ldl -lpthread"
g++ $R/gemm_hls_b200/host/TestSimulation.cpp $R/gemm_hls_b200/host/KernelEntry.cpp $COMMON -o TestSimulation
g++ $R/gemm_hls_b200/host/PrintSpecifications.cpp $COMMON -o PrintSpecifications
g++ $R/gemm_hls_b200/host/RunHardware.cpp $COMMON -o RunHardware
echo "host executables in $OUT: $(ls "$OUT" | tr '\n' ' ')"
