"""nnets.nnet -- drop-in for ctc_fast/nnets/nnet.py (class NNet): the feed-forward net
trained with CTC, computed by libctcb200 on an H100.

    NNet(inputDim, outputDim, layerSize, numLayers, maxBatch, train=True)     nnet.py:7
    costAndGrad(data, labels) -> (cost, grad, skip)                           nnet.py:57-113

It is the BRNN path without a temporal layer (ctcb_brnn_config.temporalLayer = 0): ReLU hidden layers
(nnet.py:67-73), softmax (:75-83), CTC (:85-87), back-propagation with sign() masks (:96-111).
stack = [[W1,b1] ... [Wout,bout]] (nnet.py:22-23).  dropout=p drops the ReLU hidden layers of training calls; layerNorm=True normalises
them; subsample=k stacks k frames into map subsampleLayer's input; freqMasks / timeMasks (with featDim) mask the input
features of training calls (SpecAugment); weightNoise=sigma adds Gaussian noise to the weight matrices of training
calls; interLayer=m, interWeight=lam adds the intermediate CTC loss of hidden layer m through the output map, and
selfCondition=True conditions the layers above m on its posteriors; tf32=True runs the tensor-core contractions in TF32
mode.  The reference's costAndGrad always trains; `train`
only sizes buffers there, here train=False additionally allows the forward-only call of nnets.brnnet.
"""
from nnets import brnnet


class NNet(brnnet.NNet):

    def __init__(self, inputDim, outputDim, layerSize, numLayers, maxBatch, train=True,
                 maxUtts=1, maxLabels=None, device=None, dropout=0.0, dropoutSeed=33, layerNorm=False, subsample=1,
                 subsampleLayer=1, freqMasks=0, freqMaskWidth=0, timeMasks=0, timeMaskWidth=0, timeMaskRatio=1.0,
                 featDim=None, weightNoise=0.0, interLayer=0, interWeight=0.0, selfCondition=False, tf32=False):
        brnnet.NNet.__init__(self, inputDim, outputDim, layerSize, numLayers, maxBatch, train=train,
                             temporalLayer=-1, reg=0.0, maxUtts=maxUtts, maxLabels=maxLabels, device=device,
                             dropout=dropout, dropoutSeed=dropoutSeed, layerNorm=layerNorm, subsample=subsample,
                             subsampleLayer=subsampleLayer, freqMasks=freqMasks, freqMaskWidth=freqMaskWidth,
                             timeMasks=timeMasks, timeMaskWidth=timeMaskWidth, timeMaskRatio=timeMaskRatio,
                             featDim=featDim, weightNoise=weightNoise, interLayer=interLayer, interWeight=interWeight,
                             selfCondition=selfCondition, tf32=tf32)

    def costAndGrad(self, data, labels=None):
        return brnnet.NNet.costAndGrad(self, data, labels)
