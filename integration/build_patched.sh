#!/bin/sh
# Builds the reference WITH the dtb200 hook from a scratch copy and stages the result (stripped) under
# oracle/_ref/patched/ (git-ignored; travels with oracle/_ref).  Needs the reference's source tree:
# $DATATABLE_REFERENCE_SRC, by default `reference` next to this repository.
set -e
HERE=$(cd "$(dirname "$0")" && pwd)
REF=${DATATABLE_REFERENCE_SRC:-$HERE/../../reference}
OUT="$HERE/../oracle/_ref/patched"
SCRATCH=${1:-${TMPDIR:-/tmp}/dthook}
rm -rf "$SCRATCH" && cp -r "$REF" "$SCRATCH"
python "$HERE/apply_hook.py" "$SCRATCH"
(cd "$SCRATCH" && python ci/ext.py build > "$SCRATCH/build.log" 2>&1) || { tail -20 "$SCRATCH/build.log"; exit 1; }
rm -rf "$OUT" && mkdir -p "$OUT"
cp -r "$SCRATCH/src/datatable" "$OUT/"
find "$OUT" -name __pycache__ -type d -prune -exec rm -rf {} +
strip -g "$OUT"/datatable/lib/_datatable*.so
PYTHONPATH="$OUT" python "$HERE/check_hook.py"
PYTHONPATH="$OUT" python "$HERE/check_hook_views.py"
