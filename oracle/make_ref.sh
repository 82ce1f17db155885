#!/bin/bash
# Copy the unmodified reference (a facebookresearch/jepa checkout given as $1) into oracle/_ref (git-ignored): the source
# of tests/golden/golden_reference_step.pt (see tests/golden/make_golden_reference.py).  Plain copy, no install step:
# tools/ref_gpu.py puts oracle/_ref first on sys.path, where src/ and app/ resolve as namespace packages.
set -euo pipefail
REF=${1:?usage: oracle/make_ref.sh <jepa checkout>}
DST="$(cd "$(dirname "$0")" && pwd)/_ref"
rm -rf "$DST"
mkdir -p "$DST"
cp -r "$REF/src" "$REF/app" "$DST/"
