#!/usr/bin/env python
"""Stage the UNMODIFIED reference functional-map head for the GPU box.

BENCH INFRASTRUCTURE ONLY.  When the reference checkout is present, this copies
``experiments/functional_correspondence/fmaps_model.py`` byte for byte to ``oracle/_ref/fmaps_model.py`` (git-ignored,
like the package ``stage_ref.py`` stages), with its sha1 in ``oracle/_ref/fmaps_model.sha1``.  ``bench_fmaps.py`` then
times the real reference head where the checkout is absent; it imports the staged package first, so the module's
``import diffusion_net`` resolves to the staged reference.  No test depends on the staged copy.
``__graft_entry__.build()`` runs this.
"""
import hashlib
import os
import shutil
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = "/root/reference/experiments/functional_correspondence/fmaps_model.py"
DST = os.path.join(HERE, "_ref", "fmaps_model.py")


def stage(verbose=True):
    if not os.path.isfile(SRC):
        if verbose:
            print("stage_ref_fmaps: {} not present: keeping whatever is staged".format(SRC))
        return os.path.isfile(DST)
    os.makedirs(os.path.dirname(DST), exist_ok=True)
    shutil.copyfile(SRC, DST)
    with open(DST, "rb") as fh:
        digest = hashlib.sha1(fh.read()).hexdigest()
    with open(os.path.join(HERE, "_ref", "fmaps_model.sha1"), "w") as fh:
        fh.write("{}  fmaps_model.py\n".format(digest))
    if verbose:
        print("stage_ref_fmaps: staged {}".format(DST))
    return True


if __name__ == "__main__":
    sys.exit(0 if stage() else 1)
