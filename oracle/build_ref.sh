#!/bin/sh
# Compiles the reference's own C conformance programs (interfaces/test/C/test_api.c,
# interfaces/test/C/test_block.c, interfaces/test/C/test_all_solvers.c, interfaces/examples/C/basic_cg.c,
# interfaces/examples/C/least_squares.c) FROM WHERE THEY LIE under /root/reference,
# against the reference's own krylov.h, and links them to libkrylov_b200.so.
# Outputs go to oracle/_ref/ only (git-ignored; travels to the GPU box).
# No reference source is copied into the repository.
set -e
HERE=$(cd "$(dirname "$0")" && pwd)
REF=${KRYLOV_REFERENCE:-/root/reference}
LIBDIR="$HERE/../krylov.jl_b200/lib"
[ -d "$REF/interfaces" ] || { echo "reference tree not present; keeping prebuilt oracle/_ref"; exit 0; }
[ -f "$LIBDIR/libkrylov_b200.so" ] || { echo "build libkrylov_b200.so first"; exit 1; }
mkdir -p "$HERE/_ref"
for prog in test/C/test_api test/C/test_block test/C/test_all_solvers examples/C/basic_cg examples/C/least_squares; do
  out="$HERE/_ref/$(basename $prog)"
  /usr/bin/gcc -O2 -o "$out" "$REF/interfaces/$prog.c" -I "$REF/interfaces/include" \
      -L "$LIBDIR" -lkrylov_b200 -Wl,-rpath,'$ORIGIN/../../krylov.jl_b200/lib' -lm
done
echo "built: $(ls $HERE/_ref)"
