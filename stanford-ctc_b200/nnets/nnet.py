"""nnets.nnet -- drop-in for ctc_fast/nnets/nnet.py (class NNet): the feed-forward net
trained with CTC, computed by libctcb200 on an H100.

    NNet(inputDim, outputDim, layerSize, numLayers, maxBatch, train=True)     nnet.py:7
    costAndGrad(data, labels) -> (cost, grad, skip)                           nnet.py:57-113

It is the BRNN path without a temporal layer (ctcb_brnn_config.temporalLayer = 0): ReLU hidden layers
(nnet.py:67-73), softmax (:75-83), CTC (:85-87), back-propagation with sign() masks (:96-111).
stack = [[W1,b1] ... [Wout,bout]] (nnet.py:22-23).  The reference's costAndGrad always trains; `train`
only sizes buffers there, here train=False additionally allows the forward-only call of nnets.brnnet.
"""
from nnets import brnnet


class NNet(brnnet.NNet):

    def __init__(self, inputDim, outputDim, layerSize, numLayers, maxBatch, train=True,
                 maxUtts=1, maxLabels=None, device=None):
        brnnet.NNet.__init__(self, inputDim, outputDim, layerSize, numLayers, maxBatch, train=train,
                             temporalLayer=-1, reg=0.0, maxUtts=maxUtts, maxLabels=maxLabels, device=device)

    def costAndGrad(self, data, labels=None):
        return brnnet.NNet.costAndGrad(self, data, labels)
