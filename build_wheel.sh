#!/bin/bash
# Wheels with the prebuilt sm_90a native module, one per CPython ABI found on this host
# (reference counterpart: build_manylinux_wheels.sh, which loops over cp310/cp311/cp312 inside
# a manylinux container and repairs with auditwheel).  The module links the CUDA runtime
# statically and needs no NIC libraries, so no repair step is needed; the version comes from
# `git describe` (setup.py:get_version).
#   PYTHONS="python3.10 python3.11 python3.12" ./build_wheel.sh
set -euo pipefail
cd "$(dirname "$0")"
PYTHONS=${PYTHONS:-"python3.10 python3.11 python3.12 python3"}
rm -rf dist
built=""
for py in $PYTHONS; do
    command -v "$py" >/dev/null 2>&1 || continue
    abi=$("$py" -c "import sysconfig; print(sysconfig.get_config_var('SOABI'))")
    case " $built " in *" $abi "*) continue ;; esac   # python3 may alias one of the above
    "$py" -c "import torch, pybind11, setuptools" 2>/dev/null || { echo "skip $py: needs torch, pybind11, setuptools"; continue; }
    echo "== $py ($abi)"
    rm -f infinistore_b200/_infinistore*.so
    "$py" tools/build_native.py --force
    "$py" setup.py -q bdist_wheel --dist-dir dist
    built="$built $abi"
done
python3 tools/build_native.py   # leave the tree usable with the default interpreter
ls -l dist/*.whl
