#!/usr/bin/env bash
# Build the UNMODIFIED reference (pymc-devs/pytensor) into oracle/_ref so that it can
#  (a) host the CUDALinker plugin (PyTensor is the host: graph IR, rewrites, pytensor.function), and
#  (b) act as the parity oracle / CPU baseline through its own C linker (mode='CVM').
#
# Usage: oracle/build_ref.sh <pytensor source checkout>
# `pip install --target` needs `versioneer` (imported by setup.py) and a network; this recipe does what that install would
# do offline: copy the package tree and build the one compiled extension (pytensor/scan/scan_perform.pyx,
# setup.py:24-29) with cython + gcc.  Nothing is written into the checkout; the output directory is git-ignored (it is
# NOT product source) and is all a machine without the checkout needs.
set -euo pipefail
REF=${1:?usage: build_ref.sh <pytensor source checkout>}
HERE="$(cd "$(dirname "${BASH_SOURCE[0]}")/.." && pwd)"
OUT="$HERE/oracle/_ref"
if [ ! -d "$REF/pytensor" ]; then
  echo "no pytensor package under $REF"; exit 1
fi
rm -rf "$OUT"; mkdir -p "$OUT"
cp -r "$REF/pytensor" "$OUT/pytensor"
chmod -R u+w "$OUT"   # a read-only checkout yields read-only copies; the extension is written into the copy
find "$OUT" -name '__pycache__' -type d -prune -exec rm -rf {} +
PYINC=$(python -c "import sysconfig; print(sysconfig.get_paths()['include'])")
NPINC=$(python -c "import numpy; print(numpy.get_include())")
EXT=$(python -c "import sysconfig; print(sysconfig.get_config_var('EXT_SUFFIX'))")
TMP=$(mktemp -d)
cp "$REF/pytensor/scan/scan_perform.pyx" "$TMP/"
( cd "$TMP" && python -m cython -3 scan_perform.pyx -o scan_perform.c )
gcc -O2 -shared -fPIC -fno-strict-aliasing -DNPY_NO_DEPRECATED_API=NPY_1_7_API_VERSION \
    -I"$PYINC" -I"$NPINC" "$TMP/scan_perform.c" -o "$OUT/pytensor/scan/scan_perform$EXT"
rm -rf "$TMP"
echo "reference built into $OUT"
