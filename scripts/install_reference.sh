#!/bin/bash
# usage: scripts/install_reference.sh <EVcouplings checkout>
# Install the UNMODIFIED reference (pure-Python package `evcouplings`) into the git-ignored baseline/_ref/, so that the
# boundary tests can run the reference's own couplings protocol.  For a pure-Python package the install is exactly
# "unpack the package directory", which is what this script does (no build backend needed).  Nothing under
# baseline/_ref is tracked by git.
set -e
ROOT="$(cd "$(dirname "$0")/.." && pwd)"
SRC=${1:?usage: $0 <EVcouplings checkout>}
[ -d "$SRC/evcouplings" ] || { echo "reference not found at $SRC" >&2; exit 1; }
mkdir -p "$ROOT/baseline/_ref"
rm -rf "$ROOT/baseline/_ref/evcouplings"
cp -r "$SRC/evcouplings" "$ROOT/baseline/_ref/evcouplings"
find "$ROOT/baseline/_ref" -name __pycache__ -type d -prune -exec rm -rf {} +
VERSION=$(sed -n 's/^__version__ *= *"\(.*\)"/\1/p' "$SRC/evcouplings/__init__.py" | head -1)
mkdir -p "$ROOT/baseline/_ref/evcouplings-${VERSION:-0}.dist-info"
printf 'Metadata-Version: 2.1\nName: evcouplings\nVersion: %s\n' "${VERSION:-0}" > "$ROOT/baseline/_ref/evcouplings-${VERSION:-0}.dist-info/METADATA"
echo "installed evcouplings ${VERSION:-?} into $ROOT/baseline/_ref"
