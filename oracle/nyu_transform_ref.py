"""The reference's NYUD2-DIR transforms and loaders (nyud2-dir/nyu_transform.py, nyud2-dir/loaddata.py) for the parity
tests of the device input pipeline (imbalanced-regression_b200/loaddata.py) and the reference arm of
tools/nyud2_input_bench.py -- TEST INFRASTRUCTURE ONLY.

install() copies the two pure-Python files into the git-ignored oracle/_ref/nyud2-dir/ (next to the util.py
oracle/ref_nyud2.install() copies), as net_ref.install() does for net.py.  load() imports those copies under distinct
module names (ref_nyu_transform, ref_nyud2_loaddata), so they never shadow the package's own `loaddata`; the names the
reference imports them by (nyu_transform, util) are bound to the copies only while they load.
"""
import importlib.util
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_DIR = os.path.join(ROOT, "oracle", "_ref", "nyud2-dir")
FILES = ("nyu_transform.py", "loaddata.py")


def available():
    return all(os.path.exists(os.path.join(REF_DIR, f)) for f in FILES + ("util.py",))


def install(reference_root="/root/reference"):
    """Copy nyud2-dir/nyu_transform.py and loaddata.py into oracle/_ref (called by __graft_entry__.build())."""
    import shutil
    src = os.path.join(reference_root, "nyud2-dir")
    if not all(os.path.isfile(os.path.join(src, f)) for f in FILES):
        return False
    os.makedirs(REF_DIR, exist_ok=True)
    for f in FILES:
        shutil.copyfile(os.path.join(src, f), os.path.join(REF_DIR, f))
    return True


def _import(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


_CACHE = {}


def load():
    """-> (nyu_transform, loaddata) of the reference, from the copies install() made."""
    if "mods" not in _CACHE:
        saved = {k: sys.modules.get(k) for k in ("nyu_transform", "util")}
        try:
            nt = _import("ref_nyu_transform", os.path.join(REF_DIR, "nyu_transform.py"))
            sys.modules["nyu_transform"] = nt
            sys.modules["util"] = _import("ref_nyud2_util", os.path.join(REF_DIR, "util.py"))
            ld = _import("ref_nyud2_loaddata", os.path.join(REF_DIR, "loaddata.py"))
        finally:
            for k, v in saved.items():
                if v is None:
                    sys.modules.pop(k, None)
                else:
                    sys.modules[k] = v
        _CACHE["mods"] = (nt, ld)
    return _CACHE["mods"]
