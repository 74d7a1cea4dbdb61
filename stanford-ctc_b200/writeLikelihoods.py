"""writeLikelihoods -- forward-only log-likelihood dump, same function names and on-disk formats as
ctc_fast/analysis-utils/writeLikelihoods.py:8-55 (Kaldi binary "BFM" float matrix ark
+ a pickle of {key: log-prob K x T})."""
import pickle
import struct

import numpy as np


def writeUttHeader(fid, key, uttSize, numClasses):
    """Kaldi-style header per utterance; data follows as float32 in C order (rows = frames)."""
    fid.write((key + ' ').encode())
    fid.write(struct.pack('b', 0))
    fid.write(b'BFM ')
    fid.write(struct.pack('b', 4))
    fid.write(struct.pack('i', uttSize))
    fid.write(struct.pack('b', 4))
    fid.write(struct.pack('i', numClasses))


def writeLogLikes(loader, nn, fn, outDir, writePickle=False):
    data_dict, alis, keys, sizes = loader.loadDataFileDict(fn)
    lik_dict = dict()
    with open(outDir + '/loglikelihoods%d.ark' % fn, 'wb') as fid:
        for i, k in enumerate(keys):
            assert data_dict[k].shape[1] < nn.maxBatch, "Need larger max utt length."
            writeUttHeader(fid, k, int(sizes[i]), nn.outputDim)
            probs = nn.costAndGrad(data_dict[k])
            assert probs.dtype == np.float32, "Probs array malformed."
            assert probs.shape[0] == nn.outputDim, "Probs dimensions mismatch."
            with np.errstate(divide='ignore'):
                probs = np.log(probs)
            probs.T.tofile(fid)
            lik_dict[k] = probs
    if writePickle:
        with open(outDir + '/loglikelihoods_%d.pk' % fn, 'wb') as f:
            pickle.dump(lik_dict, f)
    return lik_dict
