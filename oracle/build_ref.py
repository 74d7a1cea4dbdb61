"""Build recipe for oracle/_ref: the reference's own CTC, compiled UNMODIFIED.

TEST INFRASTRUCTURE ONLY (checker / CPU baseline) -- never imported by the product path.

Compiles <reference>/ctc_fast/ctc-loss/ctc_fast.pyx (ctc_loss :13-152, decode_best_path
:154-187) and ctc_fast_blankforce.pyx (ctc_loss :13-113, decode_best_path :115-142) from where they lie, <reference>
being the checkout of the original stanford-ctc project named by $CTC_REFERENCE_DIR; outputs (generated .c and the
extension .so) go only into oracle/_ref/, which is git-ignored.  The tests do not need it (what they compare with is
stored under tests/golden/); the golden generators and bench.py's CPU baseline do.

The reference's own setup.py (ctc-loss/setup.py:1-8) uses the removed distutils/Cython.Distutils
API, so this is the modern equivalent.  language_level=2 is required: the source uses xrange,
a print statement, and C integer division in `l = (s-1)/2`.

Usage:  CTC_REFERENCE_DIR=<checkout> python oracle/build_ref.py [--force]
Without the reference sources this is a no-op: an already built .so is used.
"""
import os
import subprocess
import sys
import sysconfig

HERE = os.path.dirname(os.path.abspath(__file__))
REF_DIR = os.path.join(os.environ.get("CTC_REFERENCE_DIR", ""), "ctc_fast", "ctc-loss")
REF_PYX = os.path.join(REF_DIR, "ctc_fast.pyx")
MODULES = ("ctc_fast", "ctc_fast_blankforce")
OUT_DIR = os.path.join(HERE, "_ref")


def so_path(name="ctc_fast"):
    return os.path.join(OUT_DIR, name + sysconfig.get_config_var("EXT_SUFFIX"))


def _build_one(name, force):
    so = so_path(name)
    pyx = os.path.join(REF_DIR, name + ".pyx")
    if not os.environ.get("CTC_REFERENCE_DIR") or not os.path.exists(pyx):
        return so if os.path.exists(so) else None
    if os.path.exists(so) and not force and os.path.getmtime(so) >= os.path.getmtime(pyx):
        return so
    import importlib.util
    if importlib.util.find_spec("Cython") is None:
        print("oracle/build_ref.py: Cython is not installed; %s not built" % name, file=sys.stderr)
        return so if os.path.exists(so) else None
    import numpy as np
    c_file = os.path.join(OUT_DIR, name + ".c")
    subprocess.check_call([sys.executable, "-m", "cython", "-2", pyx, "-o", c_file])
    inc_py = sysconfig.get_paths()["include"]
    cmd = ["gcc", "-O2", "-fPIC", "-shared", "-fwrapv", "-fno-strict-aliasing",
           "-DNPY_NO_DEPRECATED_API=NPY_1_7_API_VERSION",
           "-I", inc_py, "-I", np.get_include(), c_file, "-o", so]
    subprocess.check_call(cmd)
    os.remove(c_file)  # generated C embeds reference source text: keep only the binary
    return so


def build(force=False):
    os.makedirs(OUT_DIR, exist_ok=True)
    paths = [_build_one(name, force) for name in MODULES]
    return paths[0]


if __name__ == "__main__":
    p = build(force="--force" in sys.argv)
    print("oracle/_ref:", p, so_path("ctc_fast_blankforce"))
