"""Copy of the reference's NYUD2-DIR evaluator for the reference-side timing of tools/nyud2_eval_bench.py -- BASELINE
INFRASTRUCTURE ONLY (nothing in the product path imports this).

nyud2-dir/util.py (Evaluator, util.py:35-133) is pure Python, so its "install" is a copy made by
__graft_entry__.build() into the git-ignored oracle/_ref/nyud2-dir/ where the reference checkout is available; a copy
of the tree carries it along.  Where it is absent the tool falls back to oracle/depth_oracle.py and says so.
"""
import os

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
UTIL = os.path.join(ROOT, "oracle", "_ref", "nyud2-dir", "util.py")


def available():
    return os.path.exists(UTIL)


def install(reference_root="/root/reference"):
    """Copy nyud2-dir/util.py into oracle/_ref (called by __graft_entry__.build())."""
    import shutil
    src = os.path.join(reference_root, "nyud2-dir", "util.py")
    if not os.path.isfile(src):
        return False
    os.makedirs(os.path.dirname(UTIL), exist_ok=True)
    shutil.copyfile(src, UTIL)
    return True
