#!/usr/bin/env bash
# BASELINE.md B2: the reference's OWN CUDA extensions, built for the H100.
# As shipped, the reference's setup.py emits sm_70/sm_80/sm_90 SASS (no PTX); sm_90 is what an H100 runs.
# This script copies the reference (path given as the first argument) to a scratch directory, changes NOTHING but the
# -gencode lines (sm_70/sm_80 dropped, to save build time), builds with --enable-cuda-ext and puts the eight
# extension modules into baseline/_ref_ext/ (git-ignored: *.so).  `bench.py --impl reference --ref-ext` and
# `bench/op_compare.py --impl reference` put that directory on sys.path; nothing of this repository is imported there.
set -euo pipefail
HERE="$(cd "$(dirname "$0")" && pwd)"
SRC="$1"
WORK="$(mktemp -d /tmp/ref_b2.XXXXXX)"
cp -r "$SRC"/. "$WORK"/
python - "$WORK/setup.py" <<'PY'
import sys
p = sys.argv[1]
s = open(p).read()
for arch in ("70", "80"):
    s = s.replace('                    "-gencode",\n                    "arch=compute_%s,code=sm_%s",\n' % (arch, arch), "")
open(p, "w").write(s)
PY
(cd "$WORK" && MAX_JOBS="${MAX_JOBS:-8}" python setup.py build_ext --inplace --enable-cuda-ext)
mkdir -p "$HERE/_ref_ext"
cp "$WORK"/unicore_fused_*.so "$HERE/_ref_ext/"
ls -la "$HERE/_ref_ext"
