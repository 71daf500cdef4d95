#!/bin/bash
# SASS evidence of the Hopper-native kernels: per cubin of libpyg_b200.so, how often each tensor-core / TMA / atomic
# mnemonic occurs.
#   tools/sass_summary.sh > sass_summary.txt
set -e
LIB="$(cd "$(dirname "$0")/.." && pwd)/pyg_lib_b200/libpyg_b200.so"
T=$(mktemp -d); cd "$T"
cuobjdump -xelf all "$LIB" > /dev/null
echo "# cuobjdump -sass of $(basename "$LIB") ($(date -u +%Y-%m-%d)), occurrences per cubin"
echo "# HGMMA = wgmma.mma_async, UTMALDG = TMA tensor load, SYNCS = mbarrier operations,"
echo "# HMMA (legacy mma.sync) must be 0; ATOMG/RED = global atomics (sampler hash table)"
printf "%-34s %8s %8s %8s %6s %6s %5s\n" cubin HGMMA UTMALDG SYNCS HMMA ATOMG RED
for f in *.sm_90a.cubin; do
  cuobjdump -sass "$f" > "$f.sass"
  c() { grep -cE "$1" "$f.sass" || true; }
  printf "%-34s %8s %8s %8s %6s %6s %5s\n" "$f" "$(c 'HGMMA')" "$(c 'UTMALDG')" "$(c 'SYNCS')" "$(c '[^G]HMMA')" "$(c 'ATOMG')" "$(c '(^|[^A-Z])RED[.G]')"
done
echo
echo "# kernels containing tensor-core MMAs:"
for f in *.sm_90a.cubin; do
  awk '/Function :/ {fn=$3} /HGMMA/ {n[fn]++} END {for (k in n) printf "  %-110s HGMMA x%d\n", k, n[k]}' "$f.sass" | c++filt | cut -c1-170
done
echo
echo "# stores of the sharded sampler's exchange kernels (st.global on IPC-mapped peer pointers: k_v2_push = the all-gather of sampled edges,"
echo "# k_v2_exc = ref exceptions, k_xbarrier = flags; k_v2_sample<.., true> stores into the rank's own exchange region):"
awk '/Function :/ {fn=$3} /STG/ {n[fn]++} END {for (k in n) if (k ~ /k_v2_sample.*Lb1/ || k ~ /k_v2_push/ || k ~ /k_v2_exc/ || k ~ /k_xbarrier/) printf "  %-110s STG x%d\n", k, n[k]}' sampler.sm_90a.cubin.sass | c++filt | cut -c1-170
rm -rf "$T"
