#!/bin/sh
# Re-records tests/golden/reference_answers.json: every call the suite makes into the live
# reference (oracle/_ref, which build() makes where the reference sources are present).  Run it
# where a GPU is present so that the GPU tests' calls are recorded as well.
set -e
cd "$(dirname "$0")/../.."
test -f oracle/_ref/libguetzli_ref.so
out=tests/golden/reference_answers.json
rm -f "$out.new"
GB200_REF_RECORD="$PWD/$out.new" python -m pytest -q tests
mv "$out.new" "$out"
