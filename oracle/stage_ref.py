#!/usr/bin/env python
"""Stage the UNMODIFIED reference package for the GPU box.

TEST/BENCH INFRASTRUCTURE ONLY.  The reference is pure Python and is not part of this repository.  When its checkout
is present at ``SRC``, this script copies ``src/diffusion_net/*.py`` byte for byte into ``oracle/_ref/`` (listed in
.gitignore, so the sources never enter this repository's history; the copy ships with the built tree like the .so).  ``bench.py --impl reference`` and the ``gpu_baseline`` leg then time the
reference's own modules (``cpu_baseline.kind == "reference"``); without the staged copy they fall back to the
restatement in ``oracle/dn_oracle_torch.py`` (``kind == "port"``).  ``__graft_entry__.build()`` runs this.
"""
import hashlib
import os
import shutil
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = "/root/reference/src/diffusion_net"
DST = os.path.join(HERE, "_ref", "diffusion_net")


def stage(verbose=True):
    if not os.path.isdir(SRC):
        if verbose:
            print("stage_ref: {} not present: keeping whatever is staged".format(SRC))
        return os.path.isdir(DST)
    os.makedirs(DST, exist_ok=True)
    manifest = []
    for f in sorted(os.listdir(SRC)):
        if f.endswith(".py"):
            shutil.copyfile(os.path.join(SRC, f), os.path.join(DST, f))
            with open(os.path.join(DST, f), "rb") as fh:
                manifest.append("{}  {}".format(hashlib.sha1(fh.read()).hexdigest(), f))
    with open(os.path.join(HERE, "_ref", "MANIFEST.sha1"), "w") as fh:
        fh.write("\n".join(manifest) + "\n")
    if verbose:
        print("stage_ref: staged {} files under {}".format(len(manifest), DST))
    return True


if __name__ == "__main__":
    sys.exit(0 if stage() else 1)
