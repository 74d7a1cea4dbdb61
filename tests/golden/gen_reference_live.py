"""Generates tests/golden/reference_live.npz by running the compiled reference CTC modules (oracle/_ref, built by
oracle/build_ref.py from the unmodified ctc_fast.pyx / ctc_fast_blankforce.pyx) on the cases that tests/test_oracle.py
pins the C restatements to bit for bit: per group of cases (ctc: recipes.ALL_CTC, bf: recipes.ALL_BF, random_ctc /
random_bf: recipes.random_*_cases, in that order) the float64 losses, the skip flags and the SHA-256 of each float64
gradient (recipes.digest), and, for the best-path decoders, the decoded label sequences.

Run from the repo root where the reference sources exist:  python tests/golden/gen_reference_live.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import recipes  # noqa: E402
from oracle import build_ref, ctc_oracle  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))


def _put(out, group, results):
    out[group + "/nll"] = np.array([r[0] for r in results], dtype=np.float64)
    out[group + "/skip"] = np.array([r[2] for r in results], dtype=np.bool_)
    out[group + "/grad_sha256"] = np.stack([recipes.digest(r[1]) for r in results])


def main():
    assert build_ref.build() is not None, "oracle/_ref could not be built (reference sources absent?)"
    bf = ctc_oracle.ref_module("ctc_fast_blankforce")
    out = {}
    res = []
    for name in recipes.ALL_CTC:
        probs, seq = recipes.ctc_case(name)
        res.append(ctc_oracle.ref_ctc_loss(np.asfortranarray(probs.astype(np.float64)), seq))
    _put(out, "ctc", res)
    res = []
    for name in recipes.ALL_BF:
        probs, seq = recipes.bf_case(name)
        p64 = np.asfortranarray(probs.astype(np.float64))
        res.append(ctc_oracle.ref_ctc_loss_blankforce(p64, seq))
        out["bf_best_path/" + name] = np.asarray(list(bf.decode_best_path(p64)), dtype=np.int64)
    _put(out, "bf", res)
    probs, seq = recipes.bf_case("bf_small")
    p64 = np.asfortranarray(probs.astype(np.float64))
    p64[:, 4] = 0.0
    out["bf_zero_frame/skip"] = np.bool_(ctc_oracle.ref_ctc_loss_blankforce(p64, seq)[2])
    probs = np.zeros((10, 9))
    probs[[0, 3, 3, 0, 3, 1, 5, 5, 8], np.arange(9)] = 1.0
    rh, ra = ctc_oracle.ref_module().decode_best_path(np.asfortranarray(probs))
    out["best_path/hyp"], out["best_path/align"] = np.asarray(list(rh), np.int64), np.asarray(list(ra), np.int64)
    _put(out, "random_ctc", [ctc_oracle.ref_ctc_loss(p, seq) for p, seq in recipes.random_ctc_cases()])
    _put(out, "random_bf", [ctc_oracle.ref_ctc_loss_blankforce(p, seq) for p, seq in recipes.random_bf_cases()])
    np.savez_compressed(os.path.join(HERE, "reference_live.npz"), **out)
    print("%d arrays" % len(out))


if __name__ == "__main__":
    main()
