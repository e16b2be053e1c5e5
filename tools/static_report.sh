#!/bin/bash
# Static evidence for the shipped kernels (no GPU needed): ptxas resource usage per kernel and the SASS mnemonics that
# show which hardware paths the code takes (UBLKCP = 1-D bulk async copy / TMA engine, SYNCS = mbarrier,
# LDGMC / multimem = NVLS multicast loads).  Output: profiles/r02_static_report.txt
set -e
cd "$(dirname "$0")/.."
OUT=profiles/${SOD_ROUND:-r02}_static_report.txt
LIB=distributed_sod_project_b200/libsod_b200.so
TMP=$(mktemp -d)
{
  echo "# ptxas -v (registers / spills / smem per kernel), nvcc $(nvcc --version | grep -o 'V[0-9]*\.[0-9]*\.[0-9]*')"
  for f in loss sgd syncbn resample maxpool pipeline api; do
    nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Iinclude -Xptxas=-v \
         -c distributed_sod_project_b200/csrc/$f.cu -o $TMP/$f.o 2>&1 \
      | c++filt | awk '/Compiling entry function/ {name=$0; sub(/.*function ./,"",name); sub(/. for.*/,"",name)}
                       /bytes spill/ {sp=""; if ($0 !~ / 0 bytes spill stores, 0 bytes spill loads/) {sp=$0; sub(/^ */,"",sp)}}
                       /Used [0-9]+ registers/ {u=$0; sub(/.*Used /,"",u); printf "%-110.110s %s\n", name, u;
                                                if (sp != "") print "    ^ SPILL: " sp; sp=""}'
  done
  echo
  echo "# SASS mnemonic counts per kernel in the shipped $LIB (cuobjdump -sass)"
  cuobjdump -sass $LIB | c++filt | awk '
    /Function :/ {fn=$0; sub(/.*Function : /,"",fn); next}
    /UBLKCP/ {c[fn,"UBLKCP"]++; seen[fn]=1}
    /SYNCS/ {c[fn,"SYNCS"]++; seen[fn]=1}
    /LDGMC|MULTIMEM|REDG?MC/ {c[fn,"MC"]++; seen[fn]=1}
    /LDG.E.*STRONG.SYS|ST.E.*STRONG.SYS|STG.E.*STRONG.SYS/ {c[fn,"SYS"]++; seen[fn]=1}
    /BAR.SYNC/ {c[fn,"BAR"]++}
    /SHFL/ {c[fn,"SHFL"]++}
    END {printf "%-100s %7s %6s %5s %8s %4s %5s\n","kernel","UBLKCP","SYNCS","MC","sys-ld/st","BAR","SHFL";
         for (f in seen) printf "%-100.100s %7d %6d %5d %8d %4d %5d\n", f, c[f,"UBLKCP"], c[f,"SYNCS"], c[f,"MC"], c[f,"SYS"], c[f,"BAR"], c[f,"SHFL"]}' | sort
} > $OUT
rm -rf $TMP
wc -l $OUT
