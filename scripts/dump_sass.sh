#!/bin/bash
# SASS listings of the two hot BA kernels for profiles/ (instruction column only) + opcode histograms + spill counts.
# usage: scripts/dump_sass.sh r02      (after `make -C scavislam_b200/csrc`)
R=${1:-r02}
cd "$(dirname "$0")/.."
for k in ba_solve ba_build_wave; do
  o=scavislam_b200/csrc/build/$k.o
  out=profiles/${R}_sass_$k.txt
  {
    echo "# cuobjdump -sass $o  (sm_90a, -O3 -lineinfo); encodings stripped"
    echo "# opcode histogram:"
    cuobjdump -sass $o | grep -E '^\s+/\*[0-9a-f]{4,5}\*/' | sed -E 's/^\s+\/\*[0-9a-f]+\*\/\s+//; s/\s*;.*//' | sed -E 's/^@!?U?P[0-9T]+\s+//' | awk '{print $1}' | sed 's/\..*//' | sort | uniq -c | sort -rn | head -24 | sed 's/^/#   /'
    echo "# local-memory instructions (LDL/STL): $(cuobjdump -sass $o | grep -cE 'LDL|STL')   generic LD.E/ST.E: $(cuobjdump -sass $o | grep -cE ' LD\.E| ST\.E')   LDGSTS: $(cuobjdump -sass $o | grep -c LDGSTS)   DSMEM/cluster barrier (UCGABAR): $(cuobjdump -sass $o | grep -c UCGABAR)"
    nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo -Xptxas -v -c scavislam_b200/csrc/$k.cu -o /dev/null 2>&1 | grep -E "Compiling entry|registers|spill" | sed 's/^/# ptxas: /'
    cuobjdump -sass $o | grep -E '^\s+/\*[0-9a-f]{4,5}\*/|Function :' | sed -E 's/\s+\/\* 0x[0-9a-f]+ \*\/\s*$//'
  } > $out
  wc -l $out
done
