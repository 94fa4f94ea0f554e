#!/bin/bash
# SASS evidence for profiles/: copy-engine / mbarrier instruction counts over the library, the TMA row-copy issue loop + one consumed
# quad of the headline forward kernel, the bulk-copied arc words of the streamed-arc backward kernel.   usage: bash tools/sass_excerpt.sh > profiles/<tag>_sass_excerpt.txt
LIB=cat_b200/libctc_crf_b200.so
T=$(mktemp -d)
cuobjdump -sass $LIB > $T/all.sass
clean() { sed 's/\/\* 0x[0-9a-f]* \*\///' | grep -v '^[[:space:]]*$' | cut -c1-96; }
echo "# SASS evidence (cuobjdump -sass $LIB)"; echo
echo "## instruction counts over the whole library"
for k in UTMALDG.2D UBLKCP SYNCS.PHASECHK.TRANS64.TRYWAIT SYNCS.ARRIVE.TRANS64 FENCE.VIEW.ASYNC R2UR "LDG.E" "REDG.E.ADD" ATOMG MUFU.EX2 MUFU.LG2 LDS.128 FFMA HMMA UTCHMMA; do printf "%-34s %s\n" "$k" "$(grep -c "$k" $T/all.sass)"; done
echo; echo "## den_forward_kernel<512,2,16,SMEM_ARCS,!HUBS,TMA,32>: the TMA row-copy issue loop and the consume path of one quad"
awk '/Function :/ {p = ($0 ~ /den_forward_kernelILi512ELi2ELi16ELb1ELb0ELb1ELi32E/)} p' $T/all.sass | clean > $T/fwd.sass
L=$(grep -n "UTMALDG" $T/fwd.sass | sed -n 3p | cut -d: -f1); sed -n "$((L-14)),$((L+32))p" $T/fwd.sass
echo; echo "## den_backward_kernel<512,2,16,!SMEM_ARCS,W1,TMA,32,STREAM> (streamed arcs): bulk copy of a batch's arc words"
awk '/Function :/ {p = ($0 ~ /den_backward_kernelILi512ELi2ELi16ELb0ELb1ELb1ELi32ELb1E/)} p' $T/all.sass | clean > $T/bwds.sass
L=$(grep -n "UBLKCP" $T/bwds.sass | sed -n 2p | cut -d: -f1); sed -n "$((L-10)),$((L+3))p" $T/bwds.sass
rm -rf $T
