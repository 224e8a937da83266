#!/bin/bash
# libreference_image_pool.so : one C export (oracle/ref_image_pool.cxx) over the reference's own ImagePool, which build_oracle.sh compiled in place into
# libreference_loader.so; this links against that library.  Outputs only into oracle/_ref/ (git-ignored).
set -euo pipefail
HERE="$(cd "$(dirname "$0")" && pwd)"
REF="${ETX_REFERENCE:-/root/reference}"
OUT="$HERE/_ref"
if [ ! -d "$REF/sources/etx" ] || [ ! -f "$OUT/libreference_loader.so" ]; then
  echo "reference or oracle/_ref/libreference_loader.so not present; the reference image pool test will skip" >&2
  exit 0
fi
T="$REF/thirdparty"
if g++ -std=c++23 -DNDEBUG -fPIC -w -O2 -include etx/core/log.hxx -I"$REF/sources" -I"$T" -I"$T/stb_image" -I"$T/tinyexr" -I"$T/enkits" \
     -shared "$HERE/ref_image_pool.cxx" -L"$OUT" -l:libreference_loader.so -Wl,-rpath,'$ORIGIN' -pthread -o "$OUT/libreference_image_pool.so"; then
  echo "built: $OUT/libreference_image_pool.so"
else
  echo "the reference image pool did not build; the test that uses it will skip" >&2
fi
