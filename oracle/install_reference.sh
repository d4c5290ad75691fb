#!/usr/bin/env bash
# Builds the reference oracle: the UNMODIFIED original project, pip-installed into oracle/_ref (git-ignored). The parity
# tests that run it live (tests/test_golden_experiment.py, bench.py --impl reference) use it when it is there.
#   bash oracle/install_reference.sh [checkout of the original project]      (default: $FLPR_REFERENCE_DIR or /root/reference)
# The original ships no setup.py / pyproject.toml, so pip refuses it directly (DESIGN.md section 6): the install is done
# from a temporary copy to which ONLY a packaging shim (package list, no source change) is added.
set -euo pipefail
REPO="$(cd "$(dirname "$0")/.." && pwd)"
SRC="${1:-${FLPR_REFERENCE_DIR:-/root/reference}}"
DST="$REPO/oracle/_ref"
TMP="$(mktemp -d)"
trap 'rm -rf "$TMP"' EXIT
cp -r "$SRC/." "$TMP/"
chmod -R u+w "$TMP"                     # (a read-only checkout yields a read-only copy the cleanup could not remove)
rm -rf "$TMP/.git"
cat > "$TMP/setup.py" <<'EOF'
from setuptools import setup, find_packages
setup(name="fedstil-reference", version="0.0.0",
      packages=find_packages(include=["analyse*", "criterions*", "datasets*", "methods*", "models*", "modules*",
                                      "tools*"]),
      py_modules=["builder", "experiment", "main"])
EOF
# packages without an __init__.py are still directories of modules the reference imports as namespace packages
for d in analyse criterions datasets methods models modules tools; do
  [ -d "$TMP/$d" ] && [ ! -f "$TMP/$d/__init__.py" ] && touch "$TMP/$d/.flpr_namespace" || true
done
rm -rf "$DST"
python -m pip install --quiet --no-index --no-build-isolation --no-deps --no-cache-dir --target "$DST" "$TMP"
# namespace directories (no __init__.py) are not picked up by find_packages: copy them verbatim
for d in analyse criterions datasets methods models modules tools; do
  if [ -d "$TMP/$d" ] && [ ! -d "$DST/$d" ]; then cp -r "$TMP/$d" "$DST/$d"; fi
done
cp -r "$TMP/configs" "$DST/configs"
find "$DST" -name .flpr_namespace -delete
echo "installed reference into $DST"
