#!/bin/bash
# The Go side of the JSON / XML encoder pin: every message of the golden inputs through the UNMODIFIED reference's
# -format=json and -format=xml encoders (go/goldengen -format).  Needs a Go toolchain.  Usage:
#   tests/golden/make_go_fmt_golden.sh /path/to/rtlamr-checkout
# Writes tests/golden/go_fmt_<case>.jsonl and go_fmt_<case>.xmll for the inputs make_go_golden.sh uses;
# tests/test_encoders.py then pins the C++ encoders against them.
set -euo pipefail
REF=${1:?rtlamr checkout}
HERE=$(cd "$(dirname "$0")" && pwd)
REPO=$(cd "$HERE/../.." && pwd)
WORK=$(mktemp -d)
cp -r "$REF" "$WORK/rtlamr"
cd "$WORK/rtlamr"
mkdir -p cmd/goldengen && cp "$REPO/go/goldengen/cmd/goldengen/main.go" cmd/goldengen/
if ! go list golang.org/x/xerrors >/dev/null 2>&1; then   # offline: stub the only third-party import of the path
  mkdir -p stubs && cp -r "$REPO/go/goldengen/stubs/xerrors" stubs/
  go mod edit -replace golang.org/x/xerrors=./stubs/xerrors
fi
python3 "$HERE/make_golden.py" --synthetic-inputs "$WORK"
run() {  # name input msgtypes chiplength (the cases of tests/test_encoders.py GO_FMT_CASES)
  go run ./cmd/goldengen -in "$2" -msgtype "$3" -symbollength "$4" -format json > "$HERE/go_fmt_$1.jsonl"
  go run ./cmd/goldengen -in "$2" -msgtype "$3" -symbollength "$4" -format xml > "$HERE/go_fmt_$1.xmll"
}
run sample_cl78_scm "$PWD/assets/sample.bin" scm 78
run sample_cl72_scm "$PWD/assets/sample.bin" scm 72
run synth_cl72_scm "$WORK/synth_cl72_scm.bin" scm 72
run synth_cl72_multi "$WORK/synth_cl72_multi.bin" scm,scm+,idm 72
run synth_cl72_r900 "$WORK/synth_cl72_r900.bin" r900 72
run synth_cl32_all "$WORK/synth_cl32_all.bin" scm,scm+,idm,r900 32
echo "wrote $(ls "$HERE"/go_fmt_* | wc -l) files under $HERE"
