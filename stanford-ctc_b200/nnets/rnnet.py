"""nnets.rnnet -- drop-in for ctc_fast/nnets/rnnet.py (class NNet): the uni-directional
recurrent net, computed by libctcb200 on an H100.

    NNet(inputDim, outputDim, layerSize, numLayers, maxBatch, train=True, temporalLayer=-1)   rnnet.py:8-9
    costAndGrad(data, labels=None) -> (cost, grad, skip)      training                        rnnet.py:91-191
                                   -> decode_best_path(probs) when train=False                rnnet.py:138-139

Same kernels as nnets.brnnet with one direction switched off (ctcb_brnn_config.unidirectional = 1):
stack = [[W1,b1] ... [Wout,bout], [Wt, dummy]] (rnnet.py:38-65), temporal layer
h[:,t] = clip(pre[:,t] + Wt.h[:,t-1], 0, 20) (rnnet.py:112-116), BPTT rnnet.py:162-177.  There is no L2
term in this class.  layerNorm=True normalises the ReLU hidden layers.  subsample=k runs map subsampleLayer and above at 1/k
of the frame rate; costAndGrad(train=False) best-path decodes those ceil(T / k) frames.  cell='lstm' makes the temporal layers uni-directional LSTMs (peephole=True adds their peephole connections).  numTemporal=k stacks k such layers (stack ends with [Wt_1, dummy] .. [Wt_k, dummy]).  initParams, updateParams, toFile, fromFile, check_grad and the minibatch additions
(maxUtts, costAndGradBatch, costAndGradDevice, dropout, the input masks, the weight noise, zoneout, the intermediate CTC
loss interLayer / interWeight and its selfCondition, TF32 mode tf32) are inherited.
"""
import numpy as np

import ctc_fast as ctc
from nnets import brnnet


class NNet(brnnet.NNet):

    def __init__(self, inputDim, outputDim, layerSize, numLayers, maxBatch,
                 train=True, temporalLayer=-1, maxUtts=1, maxLabels=None, device=None, numTemporal=1,
                 allowTopTemporal=False, dropout=0.0, dropoutSeed=33, cell="relu", layerNorm=False, subsample=1,
                 subsampleLayer=1, peephole=False, freqMasks=0, freqMaskWidth=0, timeMasks=0, timeMaskWidth=0,
                 timeMaskRatio=1.0, featDim=None, weightNoise=0.0, zoneoutCell=0.0, zoneoutHidden=0.0, interLayer=0,
                 interWeight=0.0, selfCondition=False, tf32=False):
        brnnet.NNet.__init__(self, inputDim, outputDim, layerSize, numLayers, maxBatch, train=train,
                             temporalLayer=temporalLayer, reg=0.0, maxUtts=maxUtts, maxLabels=maxLabels,
                             allowTopTemporal=allowTopTemporal, device=device, unidirectional=True,
                             numTemporal=numTemporal, dropout=dropout, dropoutSeed=dropoutSeed, cell=cell,
                             layerNorm=layerNorm, subsample=subsample, subsampleLayer=subsampleLayer,
                             peephole=peephole, freqMasks=freqMasks, freqMaskWidth=freqMaskWidth, timeMasks=timeMasks,
                             timeMaskWidth=timeMaskWidth, timeMaskRatio=timeMaskRatio, featDim=featDim,
                             weightNoise=weightNoise, zoneoutCell=zoneoutCell, zoneoutHidden=zoneoutHidden,
                             interLayer=interLayer, interWeight=interWeight,
                             selfCondition=selfCondition, tf32=tf32)

    def costAndGrad(self, data, labels=None):
        if not self.train:
            probs = brnnet.NNet.costAndGrad(self, data)
            return ctc.decode_best_path(np.asfortranarray(probs.astype(np.float64)))
        return brnnet.NNet.costAndGrad(self, data, labels)
