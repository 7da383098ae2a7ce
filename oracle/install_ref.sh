#!/usr/bin/env bash
# Installs the UNMODIFIED reference (KinWaiCheuk/nnAudio v0.3.3) into oracle/_ref (git-ignored) so that
# `bench.py --impl reference`, its `cpu_baseline` and its `reference_gpu` leg time the reference's own code.
# The reference is pure Python: its `nnAudio` package is copied as is (no pip, no build step).
#
# Source: $NNAUDIO_REF_SRC (the reference's `Installation/` directory, the one holding setup.py and
# nnAudio/) if set -- then a missing or unusable source is an error; else a checkout of the reference
# beside this repository (../reference) or at /root/reference, if one exists; else nothing is installed
# and bench.py times the NumPy oracle port instead.
set -euo pipefail
root="$(cd "$(dirname "${BASH_SOURCE[0]}")/.." && pwd)"
if [ -n "${NNAUDIO_REF_SRC:-}" ]; then
  src="$NNAUDIO_REF_SRC"
  if [ ! -f "$src/nnAudio/__init__.py" ]; then
    echo "oracle/install_ref.sh: NNAUDIO_REF_SRC=$src holds no nnAudio package" >&2
    exit 1
  fi
else
  src=""
  for cand in "$root/../reference/Installation" /root/reference/Installation; do
    if [ -f "$cand/nnAudio/__init__.py" ]; then src="$cand"; break; fi
  done
  if [ -z "$src" ]; then
    echo "oracle/install_ref.sh: no reference checkout found: reference not installed"
    exit 0
  fi
fi
tmp="$(mktemp -d)"
trap 'rm -rf "$tmp"' EXIT
cp -R "$src/nnAudio" "$tmp/nnAudio"
find "$tmp" -name __pycache__ -prune -exec rm -rf {} +
rm -rf "$root/oracle/_ref"
mkdir -p "$root/oracle/_ref"
cp -R "$tmp/nnAudio" "$root/oracle/_ref/nnAudio"
echo "installed the reference from $src into $root/oracle/_ref"
