#!/usr/bin/env bash
# Proof that a refactoring left the shipped kernels alone: snapshot the SASS of every object of the library, later compare.
#   bash tools/sass_guard.sh save  [dir]     after a build of the known-good tree     (default dir: /tmp/exl3b_sass)
#   bash tools/sass_guard.sh check [dir]     after rebuilding the modified tree: prints differing SASS lines per object
# Lines that differ only in constant-bank-4 offsets (addresses of printf format strings) and the file-name / function header lines
# are ignored.  New objects (no snapshot) are reported as such.
set -u
mode=${1:-check}; dir=${2:-/tmp/exl3b_sass}
objs=exllamav3_b200/build
mkdir -p "$dir"
norm() { grep -v "^\s*Function\|^\s*\.headerflags\|identifier" "$1" | grep -v "c\[0x4\]"; }
rc=0
for o in "$objs"/*.o; do
    b=$(basename "$o")
    if [ "$mode" = "save" ]; then
        cuobjdump -sass "$o" > "$dir/$b.sass"; echo "saved $b"
    else
        if [ ! -f "$dir/$b.sass" ]; then echo "$b: new object (no snapshot)"; continue; fi
        cuobjdump -sass "$o" > "$dir/$b.now"
        n=$(diff <(norm "$dir/$b.now") <(norm "$dir/$b.sass") | grep -c "^[<>]")
        echo "$b: $n differing SASS lines"; [ "$n" -eq 0 ] || rc=1
    fi
done
exit $rc
