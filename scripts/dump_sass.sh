#!/bin/bash
# cuobjdump -sass of the kernels the benches time, one file per kernel (all template instantiations), into profiles/sass/.
# Instruction encodings are dropped (address + mnemonic + operands stay).  Runs without a GPU.
# usage: scripts/dump_sass.sh [prefix]   (default prefix r2)
set -e
cd "$(dirname "$0")/.."
pfx=${1:-r2}
mkdir -p profiles/sass
cuobjdump -sass metagym_b200/libmgb200.so | python3 -c '
import re, sys
enc = re.compile(r"\s*/\* 0x[0-9a-f]+ \*/\s*$")
for line in sys.stdin:
    line = enc.sub("", line.rstrip("\n"))
    if line.strip():
        print(line)
' > /tmp/mgb_all.sass
for k in quad_step_wide_kernel quad_stream_kernel quad_step2_kernel quad_rollout_kernel maze3d_step_kernel maze3d_compose_kernel maze3d_rollout_kernel maze3d_kernel; do
    f="profiles/sass/${pfx}_$k.sass"
    awk -v k="$k" '/Function : /{f = index($0, k "I") > 0 || index($0, k "E") > 0} f' /tmp/mgb_all.sass > "$f"
    echo "$k: $(grep -c 'Function : ' $f) instantiation(s), $(wc -l < $f) lines;" \
         "UBLKCP $(grep -c UBLKCP $f || true), SYNCS $(grep -c SYNCS $f || true)," \
         "DFMA/DMUL/DADD $(grep -cE 'DFMA|DMUL|DADD' $f || true)"
done | tee "profiles/sass/${pfx}_summary.txt"
for k in quad_step2_kernel quad_rollout_kernel maze3d_compose_kernel maze3d_rollout_kernel maze3d_kernel; do gzip -nf "profiles/sass/${pfx}_$k.sass"; done
