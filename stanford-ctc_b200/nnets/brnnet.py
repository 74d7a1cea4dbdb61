"""nnets.brnnet -- drop-in for ctc_fast/nnets/brnnet.py (class NNet), computed by
libctcb200 on an H100.

Same constructor, attributes and methods as the reference (brnnet.py:10-11, :34, :88, :117, :251,
:258, :269, :279):

    NNet(inputDim, outputDim, layerSize, numLayers, maxBatch, train=True, temporalLayer=-1, reg=0.0)
    initParams(); paramCount(); costAndGrad(data, labels=None, sentence=None)
    updateParams(scale, update); toFile(fid); fromFile(fid); check_grad(data, labels, epsilon)
    attributes: stack, grad, reg, regcost, maxBatch, outputDim, ...

`stack` / `grad` are lists of [W, b] exactly as in the reference, but every W and b is a VIEW into one
flat fp32 device buffer (`params` / `grads`), so the optimiser and the NCCL all-reduce touch a
single contiguous vector.  New, additive surface for the minibatch/data-parallel path:

    NNet(..., maxUtts=B, maxLabels=L)        capacity for B utterances per call (micro-batch)
    NNet(..., numTemporal=k)                 k stacked temporal layers temporalLayer .. temporalLayer+k-1
    NNet(..., cell='lstm')                   LSTM temporal layers instead of the clipped-ReLU recurrence (include/ctcb200.h:
                                                the cell): each layer's affine map has ndir*4H rows, each recurrent
                                                matrix is 4H x H; 'relu' (the default) is the reference's net
    NNet(..., cell='lstm', peephole=True)    peephole connections of the LSTM cell (include/ctcb200.h: peephole): i and
                                                f also see c_{t-1}, o sees c_t, through three H-vectors per direction;
                                                one [P (3 x H), dummy] pair per direction appended to `stack` behind
                                                everything else, P = 0 at start
    NNet(..., layerNorm=True)                layer normalisation of the ReLU hidden layers (include/ctcb200.h:
                                                layerNorm): relu(gamma * layer_norm(z) + beta), one [gamma, beta] pair
                                                per normalised layer appended to `stack`, gamma = 1 and beta = 0 at start
    NNet(..., subsample=k, subsampleLayer=L) affine map L reads k consecutive frames of the layer below it (W_L is
                                                rows x k*n) and maps L and above run on ceil(T / k) frames
                                                (include/ctcb200.h: subsample); the probabilities, the CTC and the
                                                likelihood arks are at that rate
    NNet(..., dropout=p, dropoutSeed=33)     inverted dropout on the ReLU hidden layers of training calls; the mask
                                                of an utterance is drawn from (seed, the device counter dropoutStep,
                                                layer, its index in the step's minibatch, frame, unit)
    NNet(..., freqMasks=2, freqMaskWidth=15, timeMasks=2, timeMaskWidth=70, timeMaskRatio=0.2, featDim=41)
                                             SpecAugment masks of the input features of training calls
                                                (include/ctcb200.h: ctcb_brnn_set_input_masks): bands of the featDim
                                                filter-bank bins of each spliced frame slot and spans of raw frames,
                                                drawn from (seed dropoutSeed, the counter dropoutStep, the utterance's
                                                index in the step's minibatch); featDim=None is inputDim (no splicing)
    NNet(..., weightNoise=sigma)             Gaussian noise of standard deviation sigma on the weight matrices of
                                                training calls (include/ctcb200.h: ctcb_brnn_set_weight_noise): one
                                                draw per step from (seed dropoutSeed, the counter dropoutStep, the
                                                element's offset); the L2 term and the update see the clean weights
    NNet(..., cell='lstm', zoneoutCell=zc, zoneoutHidden=zh)
                                             zoneout of every LSTM layer's c and h (include/ctcb200.h: zoneout):
                                                training calls keep each unit's previous c / h with probability zc /
                                                zh, drawn from (seed dropoutSeed, the counter dropoutStep, the
                                                utterance's index, the frame, the layer, the unit); forward-only calls
                                                use the expectation, so a net for testing needs the trained values
    NNet(..., interLayer=m, interWeight=lam) an intermediate CTC loss (include/ctcb200.h: interLayer): hidden layer m's
                                                output through the net's own output map W_{N+1}, b_{N+1}, scored by a
                                                second CTC; training calls differentiate main + lam * that loss, and
                                                costAndGrad returns it.  No parameter is added and forward-only calls do
                                                not change; interCosts / interSkips hold the last batch's per-utterance
                                                intermediate nll and skips
    NNet(..., interLayer=m, interWeight=lam, selfCondition=True)
                                             self-conditioned CTC (include/ctcb200.h: selfCondition): the intermediate
                                                posteriors P = softmax(A) are projected back, X_m + W_c P + b_c, and
                                                the layers above read that, in training and forward-only calls alike;
                                                one [W_c (H x K), b_c (H x 1)] pair appended to `stack` behind
                                                everything else, both 0 at start (the net starts as the InterCTC net)
    NNet(..., tf32=True)                     TF32 mode (include/ctcb200.h: tf32): every tensor-core contraction and
                                                sweep of training and forward-only calls reads its operands rounded
                                                to TF32 and runs one MMA per product instead of three, as PyTorch's
                                                allow_tf32; no parameter or workspace changes, so checkpoints load
                                                in either mode
    costAndGradBatch(datas, labelss)         -> (costs[B], grad, skips[B])   host arrays in; more than maxUtts
                                                utterances are accumulated over micro-batches
    costAndGradDevice(batch, first, last)    -> no host sync; see DeviceBatch
    forwardBatch(datas)                      -> [K x T float32 probabilities] per utterance, in input order,
                                                micro-batches of at most maxUtts (the batched costAndGrad(train=False))

torch tensors are buffer handles only; all arithmetic is in the C ABI (include/ctcb200.h).
"""
import ctypes
import pickle

import numpy as np

import _ctcb
import parallel
from _ctcb import lib, check, ptr, BrnnConfig

CTC_MAX_LABELS = 511      # CTCB_CTC_MAX_LABELS


def utterance_labels(u, labels, maxLabels, K):
    """The label sequence of utterance u as int32, refused with a ValueError when the net cannot train on it: more than
    maxLabels labels, or a label outside [0, K) (an alignment file numbered 1..K, say).  The CTC kernel would skip such
    an utterance on the device without a word; here training stops at it."""
    l = np.asarray(labels, dtype=np.int32).reshape(-1)
    if l.shape[0] > maxLabels:
        raise ValueError("utterance %d has %d labels; this net was built for at most maxLabels=%d"
                         % (u, l.shape[0], maxLabels))
    bad = np.flatnonzero((l < 0) | (l >= K))
    if bad.size:
        raise ValueError("utterance %d has the label %d at position %d; this net has %d output classes, labels 0..%d"
                         % (u, int(l[bad[0]]), int(bad[0]), K, K - 1))
    return l


class DeviceBatch(object):
    """A minibatch staged for the device: pinned host staging buffers + device tensors.
    feats is time-major [Tmax][B][inputDim]; labels lie in [0, K)."""

    def __init__(self, torch, dev, maxT, maxB, inputDim, maxLabels, K):
        self.maxT, self.maxB, self.D = maxT, maxB, inputDim
        self.maxLabels, self.K = maxLabels, K
        self.h_feats = torch.zeros(maxT * maxB * inputDim, dtype=torch.float32).pin_memory()
        self.h_lens = torch.zeros(maxB, dtype=torch.int32).pin_memory()
        self.h_labels = torch.zeros(max(1, maxB * maxLabels), dtype=torch.int32).pin_memory()
        self.h_off = torch.zeros(maxB + 1, dtype=torch.int32).pin_memory()
        self.d_feats = torch.zeros(maxT * maxB * inputDim, dtype=torch.float32, device=dev)
        self.d_lens = torch.zeros(maxB, dtype=torch.int32, device=dev)
        self.d_labels = torch.zeros(max(1, maxB * maxLabels), dtype=torch.int32, device=dev)
        self.d_off = torch.zeros(maxB + 1, dtype=torch.int32, device=dev)
        self.B = 0
        self.Tmax = 0
        self.h2d_bytes = 0
        self._torch = torch
        self._copied = None     # event behind the last upload: the pinned buffers are free again once it completed

    def pack(self, datas, labelss):
        """datas: list of (inputDim x T_u) float32 arrays (the reference's per-utterance layout,
        dataLoader.py:88); labelss: list of int label sequences (None in forward-only mode)."""
        B = len(datas)
        Tmax = max(d.shape[1] for d in datas)
        assert B <= self.maxB, "Batch size exceeds max utterances"
        assert Tmax <= self.maxT, "Batch size exceeds max batch"      # brnnet.py:100
        if self._copied is not None:
            # an asynchronous copy out of these pinned buffers may still be queued (a step of several micro-batches
            # cycles through the two staging buffers faster than the device consumes them)
            self._copied.synchronize()
        D = self.D
        f = self.h_feats.numpy()[:Tmax * B * D].reshape(Tmax, B, D)
        lens = self.h_lens.numpy()
        for u, d in enumerate(datas):
            T = d.shape[1]
            f[:T, u, :] = d.T
            if T < Tmax:
                f[T:, u, :] = 0.0
            lens[u] = T
        off = self.h_off.numpy()
        lab = self.h_labels.numpy()
        off[0] = 0
        if labelss is not None:
            n = 0
            for u, l in enumerate(labelss):
                l = utterance_labels(u, l, self.maxLabels, self.K)
                lab[n:n + l.shape[0]] = l
                n += l.shape[0]
                off[u + 1] = n
        else:
            off[1:B + 1] = 0
        self.B, self.Tmax = B, Tmax
        return self

    def upload(self):
        n = self.Tmax * self.B * self.D
        nl = int(self.h_off[self.B])
        self.d_feats[:n].copy_(self.h_feats[:n], non_blocking=True)
        self.d_lens[:self.B].copy_(self.h_lens[:self.B], non_blocking=True)
        self.d_off[:self.B + 1].copy_(self.h_off[:self.B + 1], non_blocking=True)
        if nl:
            self.d_labels[:nl].copy_(self.h_labels[:nl], non_blocking=True)
        if self._copied is None:
            self._copied = self._torch.cuda.Event()
        self._copied.record()
        self.h2d_bytes = 4 * (n + self.B + self.B + 1 + nl)
        return self


def check_ln_pairs(got, want, n_ln, what):
    """A net with layer normalisation loads only a checkpoint with its own number of [W, b] pairs (n_ln of them the
    [gamma, beta] pairs behind the rest): zip() would otherwise leave the normalisation parameters unset."""
    if got != want:
        raise ValueError("the checkpoint's %s has %d pairs where this net (layerNorm, %d normalised layers) has %d: a "
                         "checkpoint of a net %s layer normalisation or of another shape"
                         % (what, got, n_ln, want, "without" if got < want else "with more"))


def check_cond_pairs(got, want, selfCondition, what):
    """A checkpoint of the other self-conditioning setting has the [W_c, b_c] pair more or fewer, which zip() would
    leave unset or drop."""
    if got != want:
        raise ValueError("the checkpoint's %s has %d tensors where this net (selfCondition=%s) has %d: a checkpoint of a "
                         "net %s self-conditioned CTC, or of another shape"
                         % (what, 2 * got, selfCondition, 2 * want, "with" if got > want else "without"))


def check_peephole_pairs(got, want, peephole, what):
    """An LSTM net loads only a checkpoint with its own number of [W, b] pairs: one of the other peephole setting has
    [P, dummy] pairs more or fewer, which zip() would leave unset or drop."""
    if got != want:
        raise ValueError("the checkpoint's %s has %d tensors where this net (cell='lstm', peephole=%s) has %d: a "
                         "checkpoint of an LSTM net %s peephole connections, or of another shape"
                         % (what, 2 * got, peephole, 2 * want, "with" if got > want else "without"))


class FlatList(list):
    """A stack-shaped list of [w, b] views that remembers the flat buffer it views."""

    def __init__(self, views, flat):
        list.__init__(self, views)
        self.flat = flat


class NNet:

    def __init__(self, inputDim, outputDim, layerSize, numLayers, maxBatch,
                 train=True, temporalLayer=-1, reg=0.0, maxUtts=1, maxLabels=None,
                 allowTopTemporal=False, device=None, unidirectional=False, numTemporal=1, dropout=0.0,
                 dropoutSeed=33, cell="relu", layerNorm=False, subsample=1, subsampleLayer=1, peephole=False,
                 freqMasks=0, freqMaskWidth=0, timeMasks=0, timeMaskWidth=0, timeMaskRatio=1.0, featDim=None,
                 weightNoise=0.0, zoneoutCell=0.0, zoneoutHidden=0.0, interLayer=0, interWeight=0.0,
                 selfCondition=False, tf32=False):
        # The intermediate CTC loss (include/ctcb200.h: interLayer).  The library refuses a layer outside
        # 1..numLayers-1 and a subsampled output map, with its message; a layer and a weight come only together.
        self.interLayer, self.interWeight = int(interLayer), float(interWeight)
        if self.interLayer != 0 and not (np.isfinite(self.interWeight) and self.interWeight > 0.0):
            raise ValueError("interLayer=%d needs a finite interWeight > 0; interWeight is %r" % (interLayer, interWeight))
        if self.interLayer == 0 and self.interWeight != 0.0:
            raise ValueError("interWeight=%r weighs the intermediate CTC loss; it needs interLayer >= 1" % (interWeight,))
        self.selfCondition = bool(selfCondition)
        if self.selfCondition and self.interLayer == 0:
            raise ValueError("selfCondition=True conditions on the intermediate CTC's posteriors; it needs interLayer >= 1")
        self.tf32 = bool(tf32)
        torch = _ctcb.require_cuda()
        self._torch = torch
        self.dev = torch.device("cuda", torch.cuda.current_device() if device is None else device)

        self.outputDim = outputDim
        self.inputDim = inputDim
        self.layerSize = layerSize
        self.numLayers = numLayers
        self.layerSizes = [layerSize] * numLayers
        self.maxBatch = maxBatch           # frames per utterance, as in the reference
        self.maxUtts = maxUtts             # utterances per call, i.e. per micro-batch of a step (new)
        # the CTC kernel holds at most CTC_MAX_LABELS labels per utterance (include/ctcb200.h); a reference-style
        # constructor call (no maxLabels) gets the largest capacity that exists
        self.maxLabels = min(maxBatch, CTC_MAX_LABELS) if maxLabels is None else maxLabels
        if self.maxLabels > CTC_MAX_LABELS:
            raise ValueError("maxLabels=%d: the CTC kernel supports at most %d labels per utterance"
                             % (self.maxLabels, CTC_MAX_LABELS))
        self.train = train
        self.reg = reg
        self.regcost = 0.0

        # brnnet.py:27-30.  allowTopTemporal is the documented extension that lets the LAST hidden
        # layer be the temporal one (the literal "1-layer BRNN" of BASELINE.json configs[1]).
        hi = numLayers + 1 if allowTopTemporal else numLayers
        if temporalLayer <= 0 or temporalLayer >= hi:
            self.temporalLayer = -1
        else:
            self.temporalLayer = temporalLayer
        self.maxAct = 20.0
        # numTemporal = k stacks k temporal layers, temporalLayer .. temporalLayer+k-1, each with its own recurrent
        # matrices (0 and 1: one layer, the reference's net).  A stack has to fit where one temporal layer may go.
        if numTemporal < 0:
            raise ValueError("numTemporal=%d must be >= 0" % numTemporal)
        if numTemporal > 1 and (temporalLayer <= 0 or temporalLayer + numTemporal - 1 >= hi):
            raise ValueError("numTemporal=%d from temporalLayer=%d does not fit in hidden layers 1..%d%s"
                             % (numTemporal, temporalLayer, hi - 1,
                                "" if allowTopTemporal else " (allowTopTemporal lets it end at numLayers)"))
        self.numTemporal = max(1, numTemporal) if self.temporalLayer > 0 else 0

        # unidirectional: the single forward-in-time recurrence of nnets/rnnet.py (used by nnets.rnnet.NNet)
        self.unidirectional = bool(unidirectional)
        if cell not in _ctcb.CELLS:
            raise ValueError("cell=%r must be one of %s" % (cell, ", ".join(sorted(_ctcb.CELLS))))
        self.cell = cell
        if peephole and cell != "lstm":
            raise ValueError("peephole=True needs cell='lstm'; cell is %r" % (cell,))
        self.peephole = bool(peephole)
        self.layerNorm = bool(layerNorm)
        # 0 and 1: off; the config refuses k < 0 and an L outside 1..numLayers+1 with a message (ValueError)
        self.subsample, self.subsampleLayer = int(subsample), int(subsampleLayer)
        # SpecAugment (include/ctcb200.h: ctcb_brnn_set_input_masks).  Only a net that masks lays its input out in
        # frame slots of featDim bins and reserves the masked copy, so a net without masks keeps today's workspace.
        self.freqMasks, self.freqMaskWidth = int(freqMasks), int(freqMaskWidth)
        self.timeMasks, self.timeMaskWidth, self.timeMaskRatio = int(timeMasks), int(timeMaskWidth), float(timeMaskRatio)
        self.inputMasks = self.freqMasks != 0 or self.timeMasks != 0      # negative counts: refused below
        if featDim is not None and not self.inputMasks:
            raise ValueError("featDim=%r is the layout of the input masks; it needs freqMasks or timeMasks > 0"
                             % (featDim,))
        self.featDim = (inputDim if featDim is None else int(featDim)) if self.inputMasks else None
        # Gaussian weight noise (include/ctcb200.h: ctcb_brnn_set_weight_noise).  Only a net with sigma > 0 reserves
        # the noisy copy of the parameters, so a net without noise keeps today's workspace.
        self.weightNoise = float(weightNoise)
        if not (np.isfinite(self.weightNoise) and self.weightNoise >= 0.0):
            raise ValueError("weightNoise=%r must be a finite standard deviation >= 0" % (weightNoise,))
        # Zoneout of the LSTM state (include/ctcb200.h: ctcb_brnn_set_zoneout).  Only a net with a probability > 0
        # reserves the dh carry, so a net without zoneout keeps today's workspace.
        self.zoneoutCell, self.zoneoutHidden = float(zoneoutCell), float(zoneoutHidden)
        for name, z in (("zoneoutCell", self.zoneoutCell), ("zoneoutHidden", self.zoneoutHidden)):
            if not 0.0 <= z < 1.0:
                raise ValueError("%s=%r must be in [0, 1)" % (name, z))
        self.zoneout = self.zoneoutCell > 0.0 or self.zoneoutHidden > 0.0
        if self.zoneout and cell != "lstm":
            raise ValueError("zoneoutCell / zoneoutHidden > 0 need cell='lstm'; cell is %r" % (cell,))
        self._cfg = BrnnConfig(inputDim, outputDim, layerSize, numLayers, max(self.temporalLayer, 0), maxBatch,
                               maxUtts, self.maxLabels, float(reg), float(self.maxAct), int(self.unidirectional),
                               self.numTemporal, _ctcb.CELLS[cell], int(self.layerNorm), self.subsample,
                               self.subsampleLayer, int(self.peephole), self.featDim or 0,
                               int(self.weightNoise > 0.0), int(self.zoneout), self.interLayer, self.interWeight,
                               int(self.selfCondition), int(self.tf32))
        self._h = ctypes.c_void_p()
        check(lib.ctcb_brnn_create(ctypes.byref(self._cfg), ctypes.byref(self._h)))
        self.stack = None
        self.grad = None
        # Inverted dropout (include/ctcb200.h: ctcb_brnn_set_dropout), the input masks and the weight noise.  The step
        # counter lives on the device, so a CUDA graph of an SGD step reads its current value at every replay; sgd.SGD
        # advances it once per step.  The net owns it when any of them is on.  dropoutShard = (rank, world) places
        # this process's utterances in the step's minibatch for dropout and the masks (None: from torch.distributed).
        # The weight noise is one draw per step, the same on every rank; zoneout's masks are placed like dropout's.
        self.dropout = float(dropout)
        self.dropoutSeed = int(dropoutSeed)
        self.dropoutStep = None
        self.dropoutShard = None
        if self.dropout != 0.0 and not 0.0 < self.dropout < 1.0:
            raise ValueError("dropout=%r must be in [0, 1)" % (dropout,))
        if self.dropout != 0.0 or self.inputMasks or self.weightNoise > 0.0 or self.zoneout:
            self.dropoutStep = torch.zeros(1, dtype=torch.int64, device=self.dev)
        seed = self.dropoutSeed & 0xFFFFFFFFFFFFFFFF
        if self.dropout != 0.0:
            check(lib.ctcb_brnn_set_dropout(self._h, self.dropout, seed, ptr(self.dropoutStep)))
        # called with counts 0 too, so that every value outside the limits is refused with the library's message
        check(lib.ctcb_brnn_set_input_masks(self._h, self.freqMasks, self.freqMaskWidth, self.timeMasks,
                                            self.timeMaskWidth, self.timeMaskRatio, seed, ptr(self.dropoutStep)))
        if self.weightNoise > 0.0:
            check(lib.ctcb_brnn_set_weight_noise(self._h, self.weightNoise, seed, ptr(self.dropoutStep)))
        if self.zoneout:
            check(lib.ctcb_brnn_set_zoneout(self._h, self.zoneoutCell, self.zoneoutHidden, seed,
                                            ptr(self.dropoutStep)))

    def __del__(self):
        h = getattr(self, "_h", None)
        if h:
            lib.ctcb_brnn_destroy(h)
            self._h = None

    # ------------------------------------------------------------------ parameters
    def _views(self, flat):
        out = []
        nt = lib.ctcb_brnn_num_tensors(ctypes.byref(self._cfg))
        off, r, c = ctypes.c_int64(), ctypes.c_int32(), ctypes.c_int32()
        for idx in range(nt):
            check(lib.ctcb_brnn_tensor_info(ctypes.byref(self._cfg), idx, ctypes.byref(off), ctypes.byref(r),
                                            ctypes.byref(c)))
            out.append(flat[off.value:off.value + r.value * c.value].view(r.value, c.value))
        return FlatList([[out[i], out[i + 1]] for i in range(0, nt, 2)], flat[:self.nparams])

    def initParams(self):
        """Initialize parameters using 6/sqrt(fanin+fanout) -- same shapes and the same np.random draw
        order as brnnet.py:38-41 (layer stack) and :66-70 (Wtf then Wtb).  The recurrent matrices of further
        stacked temporal layers are drawn after those, layer by layer, at the same scale.  With cell='lstm' the same
        rule and order apply to the LSTM shapes (a temporal layer's map has G = ndir*4H rows, each U is 4H x H), each
        matrix at the scale of its own shape.  With subsample=k, W_L has k*n columns and fan-in k*n."""
        torch = self._torch
        sizes = [self.inputDim] + self.layerSizes + [self.outputDim]
        cols = [n * (self.subsample if self.subsample > 1 and i + 1 == self.subsampleLayer else 1)
                for i, n in enumerate(sizes[:-1])]
        rows = [self._map_rows(i) for i in range(1, self.numLayers + 2)]
        scales = [np.sqrt(6) / np.sqrt(n + m) for n, m in zip(cols, rows)]
        host = [[np.random.rand(m, n) * 2 * s - s, np.zeros((m, 1))]
                for n, m, s in zip(cols, rows, scales)]
        H = self.layerSize
        rec_rows = 4 * H if self.cell == "lstm" else H
        for _ in range(self.numTemporal):
            scale = np.sqrt(6) / np.sqrt(rec_rows + H)
            wtf = 2 * scale * np.random.rand(rec_rows, H) - scale
            host.append([wtf, np.zeros((1, 1))])
            if not self.unidirectional:            # rnnet.py:57-61 draws a single recurrent matrix
                wtb = 2 * scale * np.random.rand(rec_rows, H) - scale
                host.append([wtb, np.zeros((1, 1))])
        # [gamma, beta] of every normalised layer, behind everything else: no draw, so the other tensors are unchanged
        host += [[np.ones((H, 1)), np.zeros((H, 1))] for _ in self.normedLayers()]
        # [P, dummy] of every direction of every peephole LSTM layer, behind those: P = 0 without a draw, so the net starts
        # out as the same net without peepholes
        host += [[np.zeros((3, H)), np.zeros((1, 1))] for _ in range(self.peepholeEntries())]
        # [W_c, b_c] of self-conditioned CTC, behind those: 0 without a draw, so the net starts as the InterCTC net
        if self.selfCondition:
            host.append([np.zeros((H, self.outputDim)), np.zeros((H, 1))])

        self.nparams = int(lib.ctcb_brnn_param_count(ctypes.byref(self._cfg)))
        self.params = torch.zeros(self.nparams, dtype=torch.float32, device=self.dev)
        self.stack = self._views(self.params)
        for (w, b), (hw, hb) in zip(self.stack, host):
            w.copy_(torch.from_numpy(hw.astype(np.float32)))
            b.copy_(torch.from_numpy(hb.astype(np.float32)))
        # the floats of the statistics tail: 4, and 6 with the intermediate CTC loss (its nll sum and skip count)
        self.statsFloats = 6 if self.interLayer else 4
        if self.train:
            # flat gradient + a 4-float tail {n_valid, sum nll, n_skipped, sweep error flag} that rides along in the
            # data-parallel all-reduce (see include/ctcb200.h: stats_out), + 4 local floats {gnorm^2, regcost, -, -}:
            # the 8 floats behind the gradient are the step's log record, read back with ONE 32-byte copy.  With the
            # intermediate CTC loss the tail has its two floats too and the record is
            # {n_valid, sum nll, n_skipped, flag, sum intermediate nll, n_skipped by it, gnorm^2, regcost}.
            ns = self.statsFloats
            self.grads_ext = torch.zeros(self.nparams + 8, dtype=torch.float32, device=self.dev)
            self.grads = self.grads_ext[:self.nparams]
            self.stats = self.grads_ext[self.nparams:self.nparams + ns]
            self.record = self.grads_ext[self.nparams:self.nparams + 8]
            self._gnorm2 = self.grads_ext[self.nparams + ns:self.nparams + ns + 1]
            self.grad = self._views(self.grads)
        else:
            self.grads = None
            self.stats = None
        # a forward-only net needs about a quarter of the training workspace (no CTC, delta or gradient buffers)
        fwd_off = ctypes.c_size_t()
        fwd_bytes = lib.ctcb_brnn_forward_workspace_bytes(ctypes.byref(self._cfg), ctypes.byref(fwd_off))
        nbytes = lib.ctcb_brnn_workspace_bytes(ctypes.byref(self._cfg)) if self.train else fwd_bytes
        self._ws = torch.zeros(nbytes, dtype=torch.uint8, device=self.dev)
        # the sweep error flag of a forward-only call, which uses the forward layout in either workspace (a training
        # call reports its flag in the statistics tail); set by the sweep kernels on a wait timeout
        self._errflag = self._ws[fwd_off.value:fwd_off.value + 4].view(torch.int32)
        self._fwd_host = None       # pinned probabilities + error flag of one forward micro-batch (forwardBatch)
        self._batch = DeviceBatch(torch, self.dev, self.maxBatch, self.maxUtts, self.inputDim, self.maxLabels,
                                  self.outputDim)
        self._batch_alt = None      # second staging buffer, created on first use by SGD.run's prefetch
        # per-utterance outputs: cost (float32) and skip (int32) share one buffer -> one D2H copy reads both
        self._out = torch.zeros(2 * self.maxUtts, dtype=torch.float32, device=self.dev)
        self._cost = self._out[:self.maxUtts]
        self._skip = self._out[self.maxUtts:].view(torch.int32)
        if self.train:
            self._regcost = self.grads_ext[self.nparams + self.statsFloats + 1:self.nparams + self.statsFloats + 2]
        else:
            self._regcost = torch.zeros(1, dtype=torch.float32, device=self.dev)
        self._out_host = torch.zeros(2 * self.maxUtts, dtype=torch.float32).pin_memory()
        self._out_all = None        # costs and skips of a step of more than maxUtts utterances (costAndGradBatch)
        self._rec_host = torch.zeros(8, dtype=torch.float32).pin_memory()
        self._probs = None
        self._comm = None
        self.interCosts = self.interSkips = None      # the intermediate nll and skips of the last costAndGradBatch
        self._inter_all = None      # their device copies, for a step of several micro-batches
        if self.interLayer and self.train:
            off = ctypes.c_size_t()
            check(lib.ctcb_brnn_activation_offset(ctypes.byref(self._cfg), 10, 0, ctypes.byref(off), None))
            self._inter_nll = self._ws[off.value:off.value + 4 * self.maxUtts].view(torch.float32)
            check(lib.ctcb_brnn_activation_offset(ctypes.byref(self._cfg), 11, 0, ctypes.byref(off), None))
            self._inter_skip = self._ws[off.value:off.value + 4 * self.maxUtts].view(torch.float32)

    def swap_batches(self):
        """Double buffering of the staging area: returns the buffer that is NOT the current one and makes it
        current (SGD.run packs minibatch i+1 into it while the device still works on minibatch i)."""
        if self._batch_alt is None:
            self._batch_alt = DeviceBatch(self._torch, self.dev, self.maxBatch, self.maxUtts, self.inputDim,
                                          self.maxLabels, self.outputDim)
        self._batch, self._batch_alt = self._batch_alt, self._batch
        return self._batch

    def _map_rows(self, i):
        """Rows of affine map i (1..numLayers+1): ndir*4H at an LSTM layer, else the width of layer i."""
        if self.cell == "lstm" and self.numTemporal and self.temporalLayer <= i < self.temporalLayer + self.numTemporal:
            return (1 if self.unidirectional else 2) * 4 * self.layerSize
        return self.layerSize if i <= self.numLayers else self.outputDim

    def normedLayers(self):
        """The layer-normalised hidden layers (layerNorm=True): every ReLU hidden layer 1..numLayers that is not
        temporal, in the order of their [gamma, beta] pairs at the end of `stack`."""
        if not self.layerNorm:
            return []
        tl, k = self.temporalLayer, self.numTemporal
        return [i for i in range(1, self.numLayers + 1) if not (k and tl <= i < tl + k)]

    def peepholeEntries(self):
        """Number of [P, dummy] pairs at the end of `stack`: one per direction of every LSTM layer with peephole=True."""
        return self.numTemporal * (1 if self.unidirectional else 2) if self.peephole else 0

    def frames(self, T):
        """Frames of the probabilities (and of the CTC) for an utterance of T input frames: ceil(T / k)."""
        return -(-T // self.subsample) if self.subsample > 1 else T

    def paramCount(self):
        return int(sum(w.numel() + b.numel() for w, b in self.stack))

    def setViews(self, batchSize):
        """Kept for interface parity (brnnet.py:96-115): buffers are sized once for maxBatch frames."""
        assert batchSize <= self.maxBatch, "Batch size exceeds max batch"

    # ------------------------------------------------------------------ compute
    def costAndGradDevice(self, batch, want_probs=False, first=True, last=True, out=None, u0=0):
        """Enqueue forward/CTC/backward for a staged DeviceBatch on the current stream.  Returns device
        tensors (cost[B], skip[B]) -- or probs [Tmax][B][K] when train=False -- without synchronising.

        Gradient accumulation over the micro-batches of one step (ctcb_brnn_cost_and_grad_part): first=False adds
        the gradient and the statistics tail into what the earlier calls left; only the last=True call exchanges
        over the ranks and adds the L2 term.  `out` optionally names the (cost[B], skip[B]) device tensors to write
        (default: the net's own per-utterance buffers).  u0: position of the batch's first utterance in this rank's
        shard of the step, which with the rank places each utterance in the minibatch for its dropout, input and zoneout
        masks."""
        if not self.train:
            return self._forward_device(batch)
        if self.dropout > 0.0 or self.inputMasks or self.zoneout:
            rank, world = self.dropoutShard or parallel.world_info()[1:]
            check(lib.ctcb_brnn_set_dropout_utts(self._h, rank + world * u0, world))
        B, Tmax = batch.B, batch.Tmax
        probs = self._probs_view(B, self.frames(Tmax)) if want_probs else None
        cost, skip = out if out is not None else (self._cost[:B], self._skip[:B])
        flags = (_ctcb.PART_FIRST if first else 0) | (_ctcb.PART_LAST if last else 0)
        check(lib.ctcb_brnn_cost_and_grad_part(
            self._h, ptr(batch.d_feats), ptr(batch.d_lens), ptr(batch.d_labels), ptr(batch.d_off), B, Tmax,
            ptr(self.params), ptr(self.grads), ptr(cost), ptr(skip), ptr(self._regcost), ptr(probs), ptr(self.stats),
            flags, ptr(self._ws), self._ws.numel(), _ctcb.current_stream()))
        return cost, skip

    def _probs_view(self, B, Tmax):
        n = Tmax * B * self.outputDim
        if self._probs is None or self._probs.numel() < n:
            self._probs = self._torch.empty(self.maxBatch * self.maxUtts * self.outputDim, dtype=self._torch.float32,
                                            device=self.dev)
        return self._probs[:n].view(Tmax, B, self.outputDim)

    def _forward_device(self, batch):
        """Forward-only call (grads = NULL, the forward workspace layout) on a staged DeviceBatch, whether or not this
        net trains: enqueues and returns the device probabilities [Tmax'][B][K] (Tmax' = frames(Tmax)) without
        synchronising."""
        probs = self._probs_view(batch.B, self.frames(batch.Tmax))
        check(lib.ctcb_brnn_cost_and_grad_part(
            self._h, ptr(batch.d_feats), ptr(batch.d_lens), None, None, batch.B, batch.Tmax, ptr(self.params), None,
            None, None, None, ptr(probs), None, _ctcb.PART_FIRST | _ctcb.PART_LAST, ptr(self._ws), self._ws.numel(),
            _ctcb.current_stream()))
        return probs

    def costAndGradBatch(self, datas, labelss):
        """Minibatch costAndGrad from host arrays: gradients of the utterances are summed.
        Returns (costs float64[B], self.grad, skips bool[B]); the L2 term is in self.regcost.
        More than maxUtts utterances are computed as consecutive micro-batches of at most maxUtts that add into the
        same gradient (parallel.micro_batches); costs and skips still cover every utterance, in input order."""
        B = len(datas)
        if B > self.maxUtts and self.train:
            return self._cost_and_grad_accumulated(datas, labelss)
        self._batch.pack(datas, labelss).upload()
        self.costAndGradDevice(self._batch)
        self._keep_inter(B, 0, B)
        # two pinned D2H copies on the stream (no kernels, no allocation), one synchronisation
        self._out_host.copy_(self._out, non_blocking=True)
        self._rec_host.copy_(self.record, non_blocking=True)
        self._torch.cuda.current_stream().synchronize()
        self._read_record()
        self._read_inter(B)
        out = self._out_host.numpy()
        costs = out[:B].astype(np.float64)
        skips = out[self.maxUtts:self.maxUtts + B].view(np.int32) != 0
        return costs, self.grad, skips

    def _read_record(self):
        rec = self._rec_host.numpy()
        if rec[3] != 0:
            raise RuntimeError("recurrent sweep: inter-CTA wait timed out (flag %d); results are invalid" % int(rec[3]))
        self.regcost = float(rec[self.statsFloats + 1])

    def _keep_inter(self, B, u0, n):
        """With the intermediate CTC loss: enqueue the copy of the last call's n intermediate nll and skips to
        positions u0.. of the step's B (the workspace holds one call's only)."""
        if not self.interLayer:
            return
        torch = self._torch
        if self._inter_all is None or self._inter_all.numel() < 2 * B:
            self._inter_all = torch.zeros(2 * B, dtype=torch.float32, device=self.dev)
        self._inter_all[u0:u0 + n].copy_(self._inter_nll[:n])
        self._inter_all[B + u0:B + u0 + n].copy_(self._inter_skip[:n])

    def _read_inter(self, B):
        if not self.interLayer:
            return
        out = self._inter_all[:2 * B].cpu().numpy()
        self.interCosts = out[:B].astype(np.float64)
        self.interSkips = out[B:2 * B].view(np.int32) != 0

    def _cost_and_grad_accumulated(self, datas, labelss):
        torch = self._torch
        B = len(datas)
        # per-utterance outputs of the whole step, apart from the net's own buffers (captured CUDA graphs of
        # sgd.SGD hold pointers into those)
        if self._out_all is None or self._out_all.numel() < 2 * B:
            self._out_all = torch.zeros(2 * B, dtype=torch.float32, device=self.dev)
            self._out_all_host = torch.zeros(2 * B, dtype=torch.float32).pin_memory()
        cost_all = self._out_all[:B]
        skip_all = self._out_all[B:2 * B].view(torch.int32)
        pieces = parallel.micro_batches(range(B), self.maxUtts)
        u0 = 0
        for k, idx in enumerate(pieces):
            batch = self.swap_batches().pack([datas[i] for i in idx],
                                             None if labelss is None else [labelss[i] for i in idx]).upload()
            n = len(idx)
            self.costAndGradDevice(batch, first=(k == 0), last=(k == len(pieces) - 1),
                                   out=(cost_all[u0:u0 + n], skip_all[u0:u0 + n]), u0=u0)
            self._keep_inter(B, u0, n)
            u0 += n
        host = self._out_all_host[:2 * B]
        host.copy_(self._out_all[:2 * B], non_blocking=True)
        self._rec_host.copy_(self.record, non_blocking=True)
        torch.cuda.current_stream().synchronize()
        self._read_record()
        self._read_inter(B)
        out = host.numpy()
        costs = out[:B].astype(np.float64)
        skips = out[B:2 * B].view(np.int32) != 0
        return costs, self.grad, skips

    def costAndGrad(self, data, labels=None, sentence=None):
        """Reference signature (brnnet.py:117): data is inputDim x T float32; returns (cost, grad, skip)
        when training, else the K x T float32 softmax outputs (K x ceil(T / k) with subsample=k).  With the
        intermediate CTC loss the cost is the objective the gradient is of, main + interWeight * intermediate nll
        (the latter left out where its CTC skips); skip is the main CTC's."""
        T = data.shape[1]
        self.setViews(T)
        if not self.train:
            self._batch.pack([data], None).upload()
            probs = self.costAndGradDevice(self._batch)
            out = np.ascontiguousarray(probs.view(self.frames(T), self.outputDim).cpu().numpy().T)
            flag = int(self._errflag.item())
            if flag != 0:
                raise RuntimeError("recurrent sweep: inter-CTA wait timed out (flag %d); results are invalid" % flag)
            return out
        costs, grad, skips = self.costAndGradBatch([data], [labels])
        cost = float(costs[0])
        if self.interLayer and not self.interSkips[0]:      # the objective the gradient is of
            cost = cost + float(np.float32(self.interWeight)) * float(self.interCosts[0])
        if self.reg > 0:
            cost = cost + self.regcost          # brnnet.py:177-183
        return cost, grad, bool(skips[0])

    def forwardBatch(self, datas):
        """The K x T float32 probabilities that costAndGrad(data) returns with train=False, for every utterance of
        `datas` (inputDim x T arrays; K x ceil(T / k) with subsample=k), in input order.  The utterances are sorted by length and cut into micro-batches
        of at most maxUtts; micro-batch i+1 is packed into the idle staging buffer while the device computes i, and
        each micro-batch ends in one synchronisation behind the copy of its probabilities and the sweep error flag
        into pinned memory.  Works on training nets too (forward-only calls fit in the training workspace)."""
        torch = self._torch
        for u, d in enumerate(datas):
            if d.shape[1] > self.maxBatch:
                raise ValueError("utterance %d has %d frames; this net was built for at most maxBatch=%d"
                                 % (u, d.shape[1], self.maxBatch))
        order = sorted(range(len(datas)), key=lambda u: datas[u].shape[1])
        pieces = parallel.micro_batches(order, self.maxUtts)
        if self._fwd_host is None:
            n = self.maxBatch * self.maxUtts * self.outputDim
            self._fwd_host = (torch.empty(n, dtype=torch.float32).pin_memory(),
                              torch.zeros(1, dtype=torch.int32).pin_memory())
        h_all, h_flag = self._fwd_host
        out = [None] * len(datas)
        batch = self.swap_batches().pack([datas[u] for u in pieces[0]], None).upload() if pieces else None
        for k, idx in enumerate(pieces):
            probs = self._forward_device(batch)
            h_probs = h_all[:probs.numel()]
            h_probs.copy_(probs.view(-1), non_blocking=True)
            h_flag.copy_(self._errflag, non_blocking=True)
            if k + 1 < len(pieces):         # host packing of the next micro-batch overlaps this one's compute
                batch = self.swap_batches().pack([datas[u] for u in pieces[k + 1]], None).upload()
            torch.cuda.current_stream().synchronize()
            flag = int(h_flag[0])
            if flag != 0:
                raise RuntimeError("recurrent sweep: inter-CTA wait timed out (flag %d); results are invalid" % flag)
            p = h_probs.numpy().reshape(probs.shape)
            for j, u in enumerate(idx):
                out[u] = np.ascontiguousarray(p[:self.frames(datas[u].shape[1]), j, :].T)
        return out

    def updateParams(self, scale, update):
        """w += scale * dw for every [w, b] (brnnet.py:251-256).  When `update` is a list of views of
        one flat buffer (grad / SGD velocity) this is a single fused axpy."""
        flat = getattr(update, "flat", None)
        if flat is not None:
            check(lib.ctcb_axpy_f32(ptr(self.params), ptr(flat), float(scale), self.nparams, _ctcb.current_stream()))
            return
        for (w, b), (dw, db) in zip(self.stack, update):
            for x, dx in ((w, dw), (b, db)):
                if x.data_ptr() == dx.data_ptr():
                    continue
                check(lib.ctcb_axpy_f32(ptr(x), ptr(dx), float(scale), x.numel(), _ctcb.current_stream()))

    # ------------------------------------------------------------------ persistence
    def toFile(self, fid):
        """Saves only the network parameters to the given fd: a pickled list of [w, b] host arrays in
        stack order, the reference's format (brnnet.py:258-267)."""
        stack = [[w.cpu().numpy(), b.cpu().numpy()] for w, b in self.stack]
        pickle.dump(stack, fid)

    def fromFile(self, fid):
        torch = self._torch
        try:
            stack = pickle.load(fid)
        except UnicodeDecodeError:          # checkpoints written by the Python-2 reference
            fid.seek(0)
            stack = pickle.load(fid, encoding="latin1")
        self.check_pair_count(stack, self.stack, "stack")
        self.check_shapes(stack, self.stack, "stack")
        for (w, b), (wi, bi) in zip(self.stack, stack):
            w.copy_(torch.from_numpy(np.ascontiguousarray(wi, dtype=np.float32).reshape(tuple(w.shape))))
            b.copy_(torch.from_numpy(np.ascontiguousarray(bi, dtype=np.float32).reshape(tuple(b.shape))))

    def check_pair_count(self, got, views, what):
        """A checkpoint's `what` (a list of [w, b]) has as many pairs as this net's: a layer-norm net refuses one with
        other [gamma, beta] pairs, an LSTM net one of the other peephole setting, a self-conditioned net one without
        [W_c, b_c], and any net one with a trailing [W_c, b_c] it does not have."""
        H, K = self.layerSize, self.outputDim
        cond_tail = (len(got) == len(views) + 1 and np.shape(got[-1][0]) == (H, K) and np.size(got[-1][1]) == H)
        if self.selfCondition or cond_tail:
            check_cond_pairs(len(got), len(views), self.selfCondition, what)
        if self.cell == "lstm" and self.numTemporal:
            check_peephole_pairs(len(got), len(views), self.peephole, what)
        if self.layerNorm:
            check_ln_pairs(len(got), len(views), len(self.normedLayers()), what)

    def check_shapes(self, got, views, what):
        """Every tensor of a checkpoint's `what` (a list of [w, b]) has the size of this net's: a checkpoint of another
        cell, subsampling (W_L is rows x k*n) or shape is refused, naming both shapes."""
        for k, ((w, b), (wi, bi)) in enumerate(zip(views, got)):
            for x, xi in ((w, wi), (b, bi)):
                if np.size(xi) != x.numel():
                    raise ValueError("checkpoint %s tensor %d has shape %s where this net (cell=%r, subsample=%d at map "
                                     "%d) has %s: a checkpoint of another cell, subsampling or shape"
                                     % (what, k, tuple(np.shape(xi)), self.cell, max(1, self.subsample),
                                        self.subsampleLayer, tuple(x.shape)))

    def check_grad(self, data, labels, epsilon=1e-3, maxChecks=10, verbose=True):
        """Finite-difference check on a small section of every weight matrix (brnnet.py:279-297).
        Returns the list of (analytic, numeric) pairs it printed.  costAndGrad never advances the dropout counter,
        so every evaluation sees the same dropout and input masks and the same weight noise (which does not depend on
        the weights' values)."""
        cost, grad, _ = self.costAndGrad(data, labels)
        out = []
        ana = [dw.clone() for dw, _ in grad]
        for (w, _), dw in zip(self.stack, ana):
            for i in range(min(w.shape[0], maxChecks)):
                for j in range(min(w.shape[1], maxChecks)):
                    w[i, j] += epsilon
                    costP, _, _ = self.costAndGrad(data, labels)
                    w[i, j] -= epsilon
                    num = (costP - cost) / epsilon
                    out.append((float(dw[i, j]), num))
                    if verbose:
                        print("Analytic %f, Numeric %f" % (out[-1][0], num))
        return out
