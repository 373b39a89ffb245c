"""Stage the reference project's Python package into ``oracle/_ref`` (git-ignored) for the baseline legs of bench.py.

The reference checkout is taken from ``$ALDM_REFERENCE_ROOT``, else from a directory named ``reference`` next to this
repository.  Only the ``audioldm2`` package's ``.py`` files are copied (the hot-path modules that oracle/ref_loader.py
imports with the package ``__init__`` files bypassed); nothing is compiled.  Without a checkout nothing is staged, and
bench.py's baselines run this project's restatement of those modules (oracle/functional.py), reported as kind "port".
"""
from __future__ import annotations

import os
import shutil
from typing import Optional

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
DEST = os.path.join(HERE, "_ref")


def source() -> Optional[str]:
    for cand in (os.environ.get("ALDM_REFERENCE_ROOT"), os.path.join(os.path.dirname(REPO), "reference")):
        if cand and os.path.isdir(os.path.join(cand, "audioldm2", "latent_diffusion")):
            return os.path.abspath(cand)
    return None


def stage() -> Optional[str]:
    """Copy <reference>/audioldm2/**.py to oracle/_ref/audioldm2; returns the staged root, or None without a checkout."""
    src = source()
    if src is None or os.path.abspath(src) == DEST:
        return None
    dst = os.path.join(DEST, "audioldm2")
    if os.path.isdir(dst):
        shutil.rmtree(dst)
    shutil.copytree(os.path.join(src, "audioldm2"), dst,
                    ignore=lambda d, names: [n for n in names if not n.endswith(".py") and not os.path.isdir(os.path.join(d, n))])
    return DEST


if __name__ == "__main__":
    print(stage() or "no reference checkout found: nothing staged")
