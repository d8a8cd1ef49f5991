#!/bin/bash
# Installs the UNMODIFIED reference (uma-pi1/kge, LibKGE) into oracle/_ref, from the source tree given by
# $KGE_REFERENCE_SRC (default /root/reference).  oracle/_ref is git-ignored; it is what
#   * bench.py --impl reference      (the reference's own TrainingJob1vsAll on the host cores)
#   * the plugin tests               (unmodified reference jobs with `model: b200_<m>`)
# import as `kge`.  Nothing from the reference enters the git history.
#
# The reference's setup.py declares packages=["kge"] only (it is meant to be installed with `pip install -e .`),
# so the tree is copied module for module: every .py and .yaml file under kge/.
set -eu
cd "$(dirname "$0")/.."
REF="${KGE_REFERENCE_SRC:-/root/reference}"
[ -d "$REF/kge" ] || { echo "reference tree not found at $REF" >&2; exit 1; }
rm -rf oracle/_ref
mkdir -p oracle/_ref
(cd "$REF" && find kge -type f \( -name '*.py' -o -name '*.yaml' \) -print0) | \
  while IFS= read -r -d '' f; do
    mkdir -p "oracle/_ref/$(dirname "$f")"
    cp "$REF/$f" "oracle/_ref/$f"
    chmod u+w "oracle/_ref/$f"
  done
n_py=$(find oracle/_ref/kge -name '*.py' | wc -l); n_ref=$(find "$REF/kge" -name '*.py' | wc -l)
[ "$n_py" = "$n_ref" ] || { echo "incomplete install: $n_py of $n_ref modules" >&2; exit 1; }
echo "reference installed into oracle/_ref ($n_py modules, $(find oracle/_ref/kge -name '*.yaml' | wc -l) yaml files)"
