"""Pins the BRNN half of the oracle to the REFERENCE ITSELF: runs the reference's own NumPy BRNN,
ctc_fast/debug-utils/rnnetcpu.py (class RNNet, costAndGrad :54-150, self-test recipe
:180-193), in the authoring container and stores its inputs and outputs as tests/golden/rnnetcpu_ref.npz.

The file is Python 2 (print statements, xrange, tabs mixed with spaces), so it cannot be imported as it
lies.  It is read from the original project's checkout ($CTC_REFERENCE_DIR), converted MECHANICALLY IN MEMORY -- tabs expanded, `print x` ->
`print(x)`, `xrange` -> `range`; no arithmetic line is touched -- written to a temporary directory
(never into this repository) and imported from there with `ctc_fast` resolving to oracle/_ref, the
reference's own unmodified ctc_fast.pyx compiled by oracle/build_ref.py.

Cases: the reference's self-test recipe (seed 33, D=20, T=10, K=6, H=30, N=3, temporalLayer=2, labels
[0,1,2]; prints "COST ...") plus further shapes, incl. a net without a temporal layer and repeated labels.
tests/test_oracle.py asserts that oracle/brnn_oracle.py reproduces cost and every gradient to 1e-12.

Run from the repo root:  python tests/golden/gen_rnnetcpu_ref.py      (needs CTC_REFERENCE_DIR)
"""
import importlib.util
import os
import re
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.path.join(os.environ.get("CTC_REFERENCE_DIR", ""), "ctc_fast", "debug-utils", "rnnetcpu.py")

# name: (seed, inputDim, T, outputDim, layerSize, numLayers, temporalLayer, labels or None for the recipe's arange(3))
CASES = {
    "selftest": (33, 20, 10, 6, 30, 3, 2, None),                 # rnnetcpu.py:180-193 verbatim
    "tl1_of_2": (7, 13, 25, 11, 24, 2, 1, [3, 3, 7, 1, 10, 2]),
    "tl3_of_5": (11, 9, 40, 8, 16, 5, 3, [1, 2, 2, 2, 5, 7, 7, 3]),
    "no_temporal": (5, 10, 12, 7, 20, 3, -1, [2, 6, 1]),
    "long_T": (3, 6, 120, 5, 12, 2, 1, [1, 4, 4, 2, 3, 1, 1, 2, 4, 3]),
}


def load_reference_module():
    from oracle import build_ref
    assert build_ref.build() is not None, "oracle/_ref could not be built (CTC_REFERENCE_DIR unset or Cython missing?)"
    src = open(REF).read().expandtabs(8)
    src = re.sub(r"^(\s*)print (.+)$", r"\1print(\2)", src, flags=re.M)
    src = src.replace("xrange(", "range(")
    tmp = tempfile.mkdtemp(prefix="rnnetcpu_py3_")
    path = os.path.join(tmp, "rnnetcpu_py3.py")
    with open(path, "w") as f:
        f.write(src)
    sys.path.insert(0, build_ref.OUT_DIR)            # `import ctc_fast as ctc` -> the unmodified reference CTC
    spec = importlib.util.spec_from_file_location("rnnetcpu_py3", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def main():
    mod = load_reference_module()
    out = {}
    for name, (seed, D, T, K, H, N, tl, labels) in CASES.items():
        np.random.seed(seed)
        data = np.random.randn(D, T)                               # rnnetcpu.py:189 (drawn before initParams)
        lab = np.arange(3).astype(np.int32) if labels is None else np.array(labels, dtype=np.int32)
        net = mod.RNNet(D, K, H, N, T, temporalLayer=tl)
        net.initParams()
        stack = [[w.copy(), b.copy()] for w, b in net.stack]
        cost, grad, skip = net.costAndGrad(data, lab)
        assert not skip
        out[name + "/cfg"] = np.array([seed, D, T, K, H, N, tl], dtype=np.int64)
        out[name + "/data"] = data
        out[name + "/labels"] = lab
        out[name + "/cost"] = np.float64(cost)
        out[name + "/nstack"] = np.int64(len(stack))
        for i, ((w, b), (dw, db)) in enumerate(zip(stack, grad)):
            out["%s/w%d" % (name, i)] = w
            out["%s/b%d" % (name, i)] = b
            out["%s/dw%d" % (name, i)] = np.array(dw)
            if i <= N:                                             # the `dummy` biases carry no gradient
                out["%s/db%d" % (name, i)] = np.array(db)
        print("%-12s COST %.9f" % (name, cost))
    np.savez_compressed(os.path.join(HERE, "rnnetcpu_ref.npz"), **out)


if __name__ == "__main__":
    main()
