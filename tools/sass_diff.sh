#!/bin/bash
# development aid: is the device code of two builds the same?   tools/sass_diff.sh <old .so or .o> <new .so or .o>
# Compares the set of kernels and, kernel by kernel, their SASS (cuobjdump -sass with the instruction addresses dropped;
# the -lineinfo line tables are not part of that listing).  Exit status 0 = same kernels, same instructions.
set -e -o pipefail
[ $# -eq 2 ] || { echo "usage: $0 <old> <new>" >&2; exit 2; }
tmp=$(mktemp -d)
trap 'rm -rf "$tmp"' EXIT
tab=$(printf '\t')
norm() {   # one line per SASS line: kernel <tab> text, kernels in name order, lines in listing order
  ${CUOBJDUMP:-cuobjdump} -sass "$1" | awk '
    /^[ \t]*Function : / { f = $3; next }
    f != "" && NF { sub(/^[ \t]*\/\*[0-9a-f]+\*\/[ \t]*/, ""); sub(/^[ \t]+/, ""); print f "\t" $0 }' | sort -s -t "$tab" -k1,1
}
norm "$1" > "$tmp/a"
norm "$2" > "$tmp/b"
cut -f1 "$tmp/a" | uniq > "$tmp/a.sym"
cut -f1 "$tmp/b" | uniq > "$tmp/b.sym"
echo "kernels: $(wc -l < "$tmp/a.sym") in $1, $(wc -l < "$tmp/b.sym") in $2"
rc=0
if ! cmp -s "$tmp/a.sym" "$tmp/b.sym"; then
  echo "kernel sets differ (< only in old, > only in new):"
  diff "$tmp/a.sym" "$tmp/b.sym" | grep '^[<>]' || true
  rc=1
fi
if cmp -s "$tmp/a" "$tmp/b"; then
  echo "SASS identical: $(wc -l < "$tmp/a") lines"
else
  echo "kernels whose SASS differs:"
  { diff "$tmp/a" "$tmp/b" || true; } | grep '^[<>]' | cut -c3- | cut -f1 | sort -u
  rc=1
fi
exit $rc
