"""dataLoader -- reader of the reference's Kaldi-derived training files.  Class and method names follow
ctc_fast/dataLoader.py:6-95 (DataLoader, loadDataFile, loadDataFileDict,
loadDataFileAsynch, getDataAsynch) because sgd/runNNet and the reference's own tools call them.

File triple number n in a directory:
    feats<n>.bin : float32, one row of `rawsize` features per frame, utterances back to back
    keys<n>.txt  : "<utterance-key> <num_frames>" per line, in file order
    alis<n>.txt  : "<utterance-key> <label> <label> ..." per line

`loadDataFileDict` returns (data_dict, alis, keys, sizes); data_dict[key] is an (imgsize x T) float32 array
with contiguous frames (Fortran order) -- the per-utterance layout the rest of the surface expects.
The prefetch runs in a thread (the reference forks a child, dataLoader.py:22-36, which is unsafe once CUDA
is initialised; the loader only does NumPy file IO, which releases the GIL).
"""
import os
import threading

import numpy as np


def _read_alignments(path):
    table = {}
    with open(path) as fid:
        for line in fid:
            fields = line.split()
            if fields:
                table[fields[0]] = fields[1:]
    return table


def _read_keys(path):
    names, frames = [], []
    with open(path) as fid:
        for line in fid:
            fields = line.split()
            if fields:
                names.append(fields[0])
                frames.append(np.int32(fields[1]))
    return names, np.array(frames)


class DataLoader:
    def __init__(self, filedir_feat, rawsize, imgsize, filedir_ali=None, load_ali=True, load_data=True):
        self.filedir_feat = filedir_feat
        self.filedir_ali = filedir_ali if filedir_ali is not None else filedir_feat
        self.rawsize, self.imgsize = rawsize, imgsize
        self.load_ali, self.load_data = load_ali, load_data
        self.p = None            # the prefetch worker (name kept from the reference)
        self._box = None

    # -- asynchronous prefetch ---------------------------------------------------------------------
    def loadDataFileAsynch(self, filenum):
        box = {}

        def work():
            try:
                box["value"] = self.loadDataFileDict(filenum)
            except BaseException as exc:         # re-raised in the consumer
                box["error"] = exc

        self._box = box
        self.p = threading.Thread(target=work, name="dataLoader-%d" % filenum)
        self.p.start()

    def getDataAsynch(self):
        assert self.p is not None, "Error in order of asynch calls."
        self.p.join()
        self.p, box = None, self._box
        if "error" in box:
            raise box["error"]
        return box["value"]

    # -- synchronous readers -------------------------------------------------------------------------
    def _path(self, directory, stem, filenum):
        return os.path.join(directory, "%s%d.%s" % (stem, filenum, "bin" if stem == "feats" else "txt"))

    def loadDataFile(self, filenum):
        """One big (imgsize x total_frames) matrix for the whole file plus alignments, keys and sizes."""
        alis = _read_alignments(self._path(self.filedir_ali, "alis", filenum)) if self.load_ali else []
        if not self.load_data:
            return None, alis, list(alis.keys()), None
        keys = sizes = None
        keyfile = self._path(self.filedir_feat, "keys", filenum)
        if os.path.exists(keyfile):
            keys, sizes = _read_keys(keyfile)
        frames = np.fromfile(self._path(self.filedir_feat, "feats", filenum), np.float32).reshape(-1, self.rawsize)
        lo = (self.rawsize - self.imgsize) // 2       # centre crop of the context window
        frames = frames[:np.sum(sizes), lo:lo + self.imgsize]
        return frames.T, alis, keys, sizes

    def loadDataFileDict(self, filenum):
        """Like loadDataFile, with the frames split per utterance into a dictionary keyed by utterance."""
        matrix, alis, keys, sizes = self.loadDataFile(filenum)
        if not self.load_data:
            return None, alis, keys, sizes
        bounds = np.concatenate([[0], np.cumsum(sizes)])
        assert bounds[-1] == matrix.shape[1], "keys file and feature file disagree on the frame count"
        data_dict = {k: np.copy(matrix[:, bounds[i]:bounds[i + 1]]) for i, k in enumerate(keys)}
        return data_dict, alis, keys, sizes


def write_synthetic_file(dirname, filenum, num_utts, rawsize, outputDim, T_range=(150, 250), L_range=(20, 40),
                         seed=33):
    """Write one synthetic file triple in the on-disk format above (tests and examples)."""
    rng = np.random.RandomState(seed + filenum)
    os.makedirs(dirname, exist_ok=True)
    blocks, key_lines, ali_lines = [], [], []
    for u in range(num_utts):
        T = int(rng.randint(T_range[0], T_range[1] + 1))
        L = int(min(T, rng.randint(L_range[0], L_range[1] + 1)))
        key = "utt%d_%04d" % (filenum, u)
        blocks.append(rng.randn(T, rawsize).astype(np.float32))
        key_lines.append("%s %d" % (key, T))
        ali_lines.append(" ".join([key] + [str(int(x)) for x in 1 + rng.randint(0, outputDim - 1, size=L)]))
    np.concatenate(blocks, axis=0).tofile(os.path.join(dirname, "feats%d.bin" % filenum))
    for stem, lines in (("keys", key_lines), ("alis", ali_lines)):
        with open(os.path.join(dirname, "%s%d.txt" % (stem, filenum)), "w") as fid:
            fid.write("\n".join(lines) + "\n")
