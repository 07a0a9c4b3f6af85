#!/bin/sh
# Stages an UNMODIFIED build of the reference (h2oai/datatable; source tree $DATATABLE_REFERENCE_SRC, by default
# `reference` next to this repository) under oracle/_ref/
# (git-ignored; travels to the GPU box with the snapshot).  Used only as the checker / the CPU arm:
#   tests/  -- validates the C restatement (oracle/dt_oracle.c) and generates golden vectors
#   bench.py --impl reference, cpu_baseline -- times the reference's own multithreaded CPU path
# The sources are compiled where they lie (a scratch COPY, because the reference's build backend writes
# into its tree); nothing of the reference is copied into the repository's history.
# Needs the reference's source tree.  ~2 minutes on 8 cores.
set -e
HERE=$(cd "$(dirname "$0")" && pwd)
REF=${DATATABLE_REFERENCE_SRC:-$HERE/../../reference}
[ -d "$REF" ] || { echo "oracle/build_ref.sh: no reference source tree at $REF: keeping the prebuilt oracle/_ref"; exit 0; }
SCRATCH=${1:-${TMPDIR:-/tmp}/dtref_build}
rm -rf "$SCRATCH" && cp -r "$REF" "$SCRATCH"
(cd "$SCRATCH" && python ci/ext.py build > "$SCRATCH/build.log" 2>&1) || { tail -20 "$SCRATCH/build.log"; exit 1; }
rm -rf "$HERE/_ref" && mkdir -p "$HERE/_ref"      # (drops a patched build too: build_patched.sh stages it again)
cp -r "$SCRATCH/src/datatable" "$HERE/_ref/"
find "$HERE/_ref" -name __pycache__ -type d -prune -exec rm -rf {} +
strip -g "$HERE"/_ref/datatable/lib/_datatable*.so
PYTHONPATH="$HERE/_ref" python -c "import datatable as dt; print('oracle/_ref: datatable', dt.__version__, 'nthreads', dt.options.nthreads)"
