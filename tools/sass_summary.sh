#!/bin/bash
# SASS evidence per kernel file: which Hopper-specific instructions the built library contains.
ROOT=$(cd "$(dirname "$0")/.." && pwd)
OUT=${1:-sass_summary.txt}
echo "# SASS mnemonic census of multiverso_b200/_lib/libmvb200.so (sm_90a), per object" > $OUT
for o in $ROOT/build/cuda/*.o; do
  echo "## $(basename $o .o)" >> $OUT
  cuobjdump -sass $o | grep -oE "HGMMA[A-Z0-9_.]*|WARPGROUP[A-Z0-9_.]*|UTMALDG[A-Z0-9_.]*|UTMASTG[A-Z0-9_.]*|UBLKCP[A-Z0-9_.]*|UBLKRED[A-Z0-9_.]*|SYNCS\.[A-Z0-9_.]*|RED\.E\.[A-Z0-9_.]*|REDG[A-Za-z0-9_.]*|ATOMG[A-Z0-9_.]*|LDG\.E\.128[A-Z0-9_.]*|STG\.E\.128[A-Z0-9_.]*|MEMBAR\.[A-Z0-9_.]*|LD\.E\.[A-Z0-9_.]*STRONG\.SYS|ST\.E\.[A-Z0-9_.]*STRONG\.SYS" | sort | uniq -c | sort -rn | head -24 >> $OUT
done
echo "written $OUT"
