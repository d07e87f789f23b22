#!/bin/sh
# Copy the UNMODIFIED reference hot-path sources into the git-ignored baseline/_ref/ (the reference has no setup.py, so there is
# nothing to pip-install).  Never committed.  Usage: tools/refshim/install_ref.sh REFERENCE_CHECKOUT
set -e
ROOT="$(cd "$(dirname "$0")/../.." && pwd)"
mkdir -p "$ROOT/baseline/_ref"
cp -r "$1/quant" "$1/utils" "$ROOT/baseline/_ref/"
find "$ROOT/baseline/_ref" -name __pycache__ -prune -exec rm -rf {} + 2>/dev/null || true
echo "reference copied to $ROOT/baseline/_ref (git-ignored)"
