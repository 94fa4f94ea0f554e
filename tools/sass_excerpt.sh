#!/bin/bash
# SASS evidence: copy-engine / mbarrier instruction counts over the library, the bulk row-copy issue + one consumed quad of the
# small-batch forward kernel, the bulk-copied arc words of the streamed-arc backward kernel.   usage: bash tools/sass_excerpt.sh
LIB=cat_b200/libctc_crf_b200.so
T=$(mktemp -d)
cuobjdump -sass $LIB > $T/all.sass
clean() { sed 's/\/\* 0x[0-9a-f]* \*\///' | grep -v '^[[:space:]]*$' | cut -c1-96; }
echo "# SASS evidence (cuobjdump -sass $LIB)"; echo
echo "## instruction counts over the whole library"
for k in UTMALDG.2D UBLKCP SYNCS.PHASECHK.TRANS64.TRYWAIT SYNCS.ARRIVE.TRANS64 FENCE.VIEW.ASYNC R2UR "LDG.E" "REDG.E.ADD" ATOMG MUFU.EX2 MUFU.LG2 LDS.128 FFMA HMMA UTCHMMA; do printf "%-34s %s\n" "$k" "$(grep -c "$k" $T/all.sass)"; done
echo; echo "## den_forward_kernel<1,16,SMEM_ARCS,!HUBS,SMALL> (small batches): one row's bulk copy (a padding row is zero-filled by STS instead), then the consume path of one quad"
awk '/Function :/ {p = ($0 ~ /den_forward_kernelILi1ELi16ELb1ELb0ELb1EE/)} p' $T/all.sass | clean > $T/fwd.sass
L=$(grep -n "UBLKCP" $T/fwd.sass | sed -n 3p | cut -d: -f1); sed -n "$((L-33)),$((L+1))p" $T/fwd.sass
echo "        ..."
C=$(awk -v l="$L" 'NR > l && /SYNCS.PHASECHK.TRANS64.TRYWAIT/ {print NR; exit}' $T/fwd.sass); sed -n "${C},$((C+17))p" $T/fwd.sass
echo; echo "## den_backward_kernel<2,16,!SMEM_ARCS,W1,!SMALL,STREAM> (streamed arcs): bulk copy of a batch's arc words"
awk '/Function :/ {p = ($0 ~ /den_backward_kernelILi2ELi16ELb0ELb1ELb0ELb1EE/)} p' $T/all.sass | clean > $T/bwds.sass
L=$(grep -n "UBLKCP" $T/bwds.sass | sed -n 2p | cut -d: -f1); sed -n "$((L-10)),$((L+3))p" $T/bwds.sass
rm -rf $T
