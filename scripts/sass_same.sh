#!/bin/bash
# Is the device code of the working tree identical to that of a git ref?  (No GPU needed: a refactor whose SASS is
# unchanged needs no new parity run.)  A file that does not exist at <git-ref> is reported as new.
# usage: scripts/sass_same.sh <git-ref>
set -e
ref=${1:?git ref}
root=$(git rev-parse --show-toplevel)
wt=$(mktemp -d)
git -C "$root" worktree add -q "$wt" "$ref"
trap 'git -C "$root" worktree remove --force "$wt"' EXIT
FL="-O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -lineinfo -Xcompiler -fPIC --expt-relaxed-constexpr"
norm() { cuobjdump -sass "$1" | grep -E "^\s+/\*[0-9a-f]{4,5}\*/|Function :" | sed -E 's/\/\* 0x[0-9a-f]+ \*\///' | md5sum | cut -d' ' -f1; }
rc=0
for src in "$root"/circl_b200/csrc/*.cu; do
  b=$(basename "$src" .cu)
  if [ ! -f "$wt/circl_b200/csrc/$b.cu" ]; then echo "$b: new"; continue; fi
  nvcc $FL -c "$src" -o "$wt/$b.new.o" 2>/dev/null
  nvcc $FL -c "$wt/circl_b200/csrc/$b.cu" -o "$wt/$b.old.o" 2>/dev/null
  if [ "$(norm "$wt/$b.new.o")" = "$(norm "$wt/$b.old.o")" ]; then echo "$b: identical"; else echo "$b: DIFFERS"; rc=1; fi
done
exit $rc
