#!/bin/bash
# A/B libraries of the Levy kernels: register budget (resident CTAs per SM the fp32 m = 8/16 instantiations are compiled
# for) and pair (f32x2 helpers) vs scalar pair arithmetic: profiles/_ab/libtsde_levy_<ctas>_<ctas_gen>_<packed>.so, selected
# at run time with TORCHSDE_B200_LIB.
set -e
cd "$(dirname "$0")/.."
F="-gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo -fmad=false -Xcompiler -fPIC -Xcompiler -fvisibility=hidden"
mkdir -p /tmp/ab profiles/_ab
rm -f profiles/_ab/*.so
for s in cabi tableau_diag tableau_general logode; do nvcc $F -c torchsde_b200/csrc/$s.cu -o /tmp/ab/$s.o & done
wait
for v in "3 3 0" "2 2 1"; do set -- $v
  nvcc $F -DTSDE_LEVY_CTAS=$1 -DTSDE_LEVY_CTAS_GEN=$2 -DTSDE_LEVY_PACKED=$3 -c torchsde_b200/csrc/brownian.cu -o /tmp/ab/brownian_$1_$2_$3.o &
done
wait
for v in "3 3 0" "2 2 1"; do set -- $v
  nvcc -shared -gencode arch=compute_90a,code=sm_90a -o profiles/_ab/libtsde_levy_$1_$2_$3.so /tmp/ab/cabi.o /tmp/ab/tableau_diag.o /tmp/ab/tableau_general.o /tmp/ab/logode.o /tmp/ab/brownian_$1_$2_$3.o
done
ls -la profiles/_ab
