#!/bin/bash
# Copies the UNMODIFIED reference package (torch_geometric 2.9.0, pure Python: nothing to compile) into oracle/_ref
# (git-ignored), where the plug-in tests and bench.py's CPU arm import it from:
#     bash oracle/install_ref.sh [<pytorch_geometric 2.9.0 source tree>]
# The source tree is the argument, else $PYG_REFERENCE_SRC, else /root/reference (where the pinned checkout is
# expected).  Without one it does nothing: those tests then skip.  Every copied file is compared with its source.
set -e
ROOT="$(cd "$(dirname "$0")/.." && pwd)"
SRC=${1:-${PYG_REFERENCE_SRC:-/root/reference}}
DST="$ROOT/oracle/_ref"
[ -d "$DST/torch_geometric" ] && exit 0
if [ ! -r "$SRC/torch_geometric/__init__.py" ]; then
    echo "no readable torch_geometric package under $SRC: oracle/_ref not installed" >&2
    exit 0
fi
TMP=$(mktemp -d "$ROOT/oracle/.ref.XXXXXX")
trap 'rm -rf "$TMP"' EXIT
(cd "$SRC" && find torch_geometric -type f ! -path '*/__pycache__/*' | sort) > "$TMP/files.txt"
(cd "$SRC" && tar cf - --exclude=__pycache__ torch_geometric) | (cd "$TMP" && tar xf -)
while read -r f; do cmp -s "$SRC/$f" "$TMP/$f" || { echo "copy of $f differs from the reference" >&2; exit 1; }; done < "$TMP/files.txt"
rm "$TMP/files.txt"
chmod -R u+w "$TMP"
rm -rf "$DST"
mv "$TMP" "$DST"
trap - EXIT
echo "oracle/_ref installed: $(find "$DST/torch_geometric" -name '*.py' | wc -l) python files identical to $SRC"
