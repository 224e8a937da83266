#!/bin/bash
# Builds liboracle_vcm_adaptive_parity.so: the parity oracle with the coarse preview and the VCM's CameraAdaptive layer
# (oracle_vcm_adaptive.cxx, which compiles oracle_preview.cxx in place) from the reference's own sources WHERE THEY LIE.  Same flags and sources as build_oracle.sh's parity build.
# Outputs only into oracle/_ref/ (git-ignored, travels to the GPU box with the snapshot).
set -euo pipefail
HERE="$(cd "$(dirname "$0")" && pwd)"
REF="${ETX_REFERENCE:-/root/reference}"
OUT="$HERE/_ref"
CSRC="$HERE/../etx_tracer_b200/csrc"
if [ ! -d "$REF/sources/etx" ]; then
  echo "reference not present at $REF; keeping prebuilt oracle/_ref" >&2
  exit 0
fi
mkdir -p "$OUT"
INC="-I$REF/sources -I$REF/thirdparty/bluenoise -I$CSRC -I$HERE"
FLAGS="-std=c++23 -DNDEBUG -fPIC -w -pthread -O2 -ffp-contract=off -fno-builtin-sincos"
objs=""
for s in "$HERE/oracle_vcm_adaptive.cxx" "$HERE/layout_check.cxx" "$REF/sources/etx/render/host/spectrum.cxx" "$REF/thirdparty/bluenoise/bluenoise.cxx" \
         "$CSRC/bvh_build.cpp" "$HERE/libm_override.cxx"; do
  o="$OUT/vcm_adaptive_parity.$(basename "$s").o"
  g++ $FLAGS $INC -c "$s" -o "$o" &
  objs="$objs $o"
done
wait
g++ -shared -o "$OUT/liboracle_vcm_adaptive_parity.so" $objs -Wl,-Bsymbolic -pthread
rm -f $objs
echo "built: $OUT/liboracle_vcm_adaptive_parity.so"
