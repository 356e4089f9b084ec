#!/usr/bin/env python
"""Installs the UNMODIFIED reference hot-path package into oracle/_ref/ (git-ignored).

`pip install` of the reference cannot work offline: habitat-lab's setup pulls gym, omegaconf, hydra-core,
habitat_sim ..., and the package `__init__`s import them.  The hot-path modules themselves only need torch / numpy, so
the install is a verbatim copy of the `habitat_baselines` python sources (byte-identical files, checked by sha256
below); they are imported through oracle/ref_shim.py (arithmetic-free stubs for the absent third-party packages).  Run
by `__graft_entry__.build()` when the reference checkout (HB200_REFERENCE_SRC, default /root/reference) is present.
Nothing under oracle/_ref is product code: only `bench.py --impl reference`, the `torch_cuda_baseline` leg of bench.py
and tests use it."""
import hashlib
import os
import shutil
import sys

SRC = os.environ.get("HB200_REFERENCE_SRC", "/root/reference")
HERE = os.path.dirname(os.path.abspath(__file__))
DST = os.path.join(HERE, "_ref")
PKG = os.path.join("habitat-baselines", "habitat_baselines")


def install(verbose=True) -> bool:
    src = os.path.join(SRC, PKG)
    if not os.path.isdir(src):
        return False
    dst = os.path.join(DST, PKG)
    n = 0
    manifest = []
    for dirpath, dirnames, files in os.walk(src):
        dirnames[:] = [d for d in dirnames if d not in ("__pycache__", "config")]
        for f in files:
            if not f.endswith(".py"):
                continue
            s = os.path.join(dirpath, f)
            rel = os.path.relpath(s, src)
            d = os.path.join(dst, rel)
            os.makedirs(os.path.dirname(d), exist_ok=True)
            if not os.path.exists(d) or open(s, "rb").read() != open(d, "rb").read():
                shutil.copyfile(s, d)
            manifest.append(f"{hashlib.sha256(open(d, 'rb').read()).hexdigest()}  {rel}")
            n += 1
    lic = os.path.join(SRC, "LICENSE")
    if os.path.exists(lic):
        shutil.copyfile(lic, os.path.join(DST, "LICENSE"))
    with open(os.path.join(DST, "MANIFEST.sha256"), "w") as f:
        f.write("\n".join(sorted(manifest)) + "\n")
    if verbose:
        print(f"reference: {n} files of {PKG} -> {dst}")
    return True


if __name__ == "__main__":
    sys.exit(0 if install() else 1)
