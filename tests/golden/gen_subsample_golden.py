"""Writes the config-level digests (tests/config_matrix.py) of a build of libctcb200.so from before frame subsampling
existed, for the 25,600 configs of config_matrix.MATRIX, into tests/golden/NAME.

    python tests/golden/gen_subsample_golden.py path/to/libctcb200.so [NAME]

Some answers depend on the device the library plans for (the contraction and sweep planners ask it), so there is one
file per kind of machine: subsample_configs.npz (the default NAME) written with no device visible, and
subsample_configs_h100_sxm.npz written on an H100 SXM (sm_90, 132 SMs)."""
import ctypes
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [os.path.join(ROOT, "tests"), os.path.join(ROOT, "stanford-ctc_b200")]


def main(lib_path, name="subsample_configs.npz"):
    import config_matrix
    from _ctcb import BrnnConfig
    lib = config_matrix.bind(ctypes.CDLL(os.path.abspath(lib_path)), BrnnConfig)
    d = np.array([config_matrix.digest(config_matrix.answers(lib, config_matrix.config(BrnnConfig, e)))
                  for e in config_matrix.MATRIX], dtype=np.int64)
    np.savez_compressed(os.path.join(HERE, name), digests=d)
    print("wrote %d digests" % len(d))


if __name__ == "__main__":
    main(*sys.argv[1:3])
