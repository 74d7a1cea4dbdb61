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


class DeviceBatch(object):
    """A minibatch staged for the device: pinned host staging buffers + device tensors.
    feats is time-major [Tmax][B][inputDim]."""

    def __init__(self, torch, dev, maxT, maxB, inputDim, maxLabels):
        self.maxT, self.maxB, self.D = maxT, maxB, inputDim
        self.maxLabels = maxLabels
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
                l = np.asarray(l, dtype=np.int32).reshape(-1)
                if l.shape[0] > self.maxLabels:
                    raise ValueError("utterance %d has %d labels; this net was built for at most maxLabels=%d"
                                     % (u, l.shape[0], self.maxLabels))
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


class FlatList(list):
    """A stack-shaped list of [w, b] views that remembers the flat buffer it views."""

    def __init__(self, views, flat):
        list.__init__(self, views)
        self.flat = flat


class NNet:

    def __init__(self, inputDim, outputDim, layerSize, numLayers, maxBatch,
                 train=True, temporalLayer=-1, reg=0.0, maxUtts=1, maxLabels=None,
                 allowTopTemporal=False, device=None, unidirectional=False, numTemporal=1):
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
        self._cfg = BrnnConfig(inputDim, outputDim, layerSize, numLayers, max(self.temporalLayer, 0), maxBatch,
                               maxUtts, self.maxLabels, float(reg), float(self.maxAct), int(self.unidirectional),
                               self.numTemporal)
        self._h = ctypes.c_void_p()
        check(lib.ctcb_brnn_create(ctypes.byref(self._cfg), ctypes.byref(self._h)))
        self.stack = None
        self.grad = None

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
        stacked temporal layers are drawn after those, layer by layer, at the same scale."""
        torch = self._torch
        sizes = [self.inputDim] + self.layerSizes + [self.outputDim]
        scales = [np.sqrt(6) / np.sqrt(n + m) for n, m in zip(sizes[:-1], sizes[1:])]
        host = [[np.random.rand(m, n) * 2 * s - s, np.zeros((m, 1))]
                for n, m, s in zip(sizes[:-1], sizes[1:], scales)]
        for _ in range(self.numTemporal):
            scale = np.sqrt(6) / np.sqrt(self.layerSize * 2)
            wtf = 2 * scale * np.random.rand(self.layerSize, self.layerSize) - scale
            host.append([wtf, np.zeros((1, 1))])
            if not self.unidirectional:            # rnnet.py:57-61 draws a single recurrent matrix
                wtb = 2 * scale * np.random.rand(self.layerSize, self.layerSize) - scale
                host.append([wtb, np.zeros((1, 1))])

        self.nparams = int(lib.ctcb_brnn_param_count(ctypes.byref(self._cfg)))
        self.params = torch.zeros(self.nparams, dtype=torch.float32, device=self.dev)
        self.stack = self._views(self.params)
        for (w, b), (hw, hb) in zip(self.stack, host):
            w.copy_(torch.from_numpy(hw.astype(np.float32)))
            b.copy_(torch.from_numpy(hb.astype(np.float32)))
        if self.train:
            # flat gradient + a 4-float tail {n_valid, sum nll, n_skipped, sweep error flag} that rides along in the
            # data-parallel all-reduce (see include/ctcb200.h: stats_out), + 4 local floats {gnorm^2, regcost, -, -}:
            # the 8 floats behind the gradient are the step's log record, read back with ONE 32-byte copy
            self.grads_ext = torch.zeros(self.nparams + 8, dtype=torch.float32, device=self.dev)
            self.grads = self.grads_ext[:self.nparams]
            self.stats = self.grads_ext[self.nparams:self.nparams + 4]
            self.record = self.grads_ext[self.nparams:self.nparams + 8]
            self._gnorm2 = self.grads_ext[self.nparams + 4:self.nparams + 5]
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
        self._batch = DeviceBatch(torch, self.dev, self.maxBatch, self.maxUtts, self.inputDim, self.maxLabels)
        self._batch_alt = None      # second staging buffer, created on first use by SGD.run's prefetch
        # per-utterance outputs: cost (float32) and skip (int32) share one buffer -> one D2H copy reads both
        self._out = torch.zeros(2 * self.maxUtts, dtype=torch.float32, device=self.dev)
        self._cost = self._out[:self.maxUtts]
        self._skip = self._out[self.maxUtts:].view(torch.int32)
        if self.train:
            self._regcost = self.grads_ext[self.nparams + 5:self.nparams + 6]
        else:
            self._regcost = torch.zeros(1, dtype=torch.float32, device=self.dev)
        self._out_host = torch.zeros(2 * self.maxUtts, dtype=torch.float32).pin_memory()
        self._out_all = None        # costs and skips of a step of more than maxUtts utterances (costAndGradBatch)
        self._rec_host = torch.zeros(8, dtype=torch.float32).pin_memory()
        self._probs = None
        self._comm = None

    def swap_batches(self):
        """Double buffering of the staging area: returns the buffer that is NOT the current one and makes it
        current (SGD.run packs minibatch i+1 into it while the device still works on minibatch i)."""
        if self._batch_alt is None:
            self._batch_alt = DeviceBatch(self._torch, self.dev, self.maxBatch, self.maxUtts, self.inputDim,
                                          self.maxLabels)
        self._batch, self._batch_alt = self._batch_alt, self._batch
        return self._batch

    def paramCount(self):
        return int(sum(w.numel() + b.numel() for w, b in self.stack))

    def setViews(self, batchSize):
        """Kept for interface parity (brnnet.py:96-115): buffers are sized once for maxBatch frames."""
        assert batchSize <= self.maxBatch, "Batch size exceeds max batch"

    # ------------------------------------------------------------------ compute
    def costAndGradDevice(self, batch, want_probs=False, first=True, last=True, out=None):
        """Enqueue forward/CTC/backward for a staged DeviceBatch on the current stream.  Returns device
        tensors (cost[B], skip[B]) -- or probs [Tmax][B][K] when train=False -- without synchronising.

        Gradient accumulation over the micro-batches of one step (ctcb_brnn_cost_and_grad_part): first=False adds
        the gradient and the statistics tail into what the earlier calls left; only the last=True call exchanges
        over the ranks and adds the L2 term.  `out` optionally names the (cost[B], skip[B]) device tensors to write
        (default: the net's own per-utterance buffers)."""
        if not self.train:
            return self._forward_device(batch)
        B, Tmax = batch.B, batch.Tmax
        probs = self._probs_view(B, Tmax) if want_probs else None
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
        net trains: enqueues and returns the device probabilities [Tmax][B][K] without synchronising."""
        probs = self._probs_view(batch.B, batch.Tmax)
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
        # two pinned D2H copies on the stream (no kernels, no allocation), one synchronisation
        self._out_host.copy_(self._out, non_blocking=True)
        self._rec_host.copy_(self.record, non_blocking=True)
        self._torch.cuda.current_stream().synchronize()
        self._read_record()
        out = self._out_host.numpy()
        costs = out[:B].astype(np.float64)
        skips = out[self.maxUtts:self.maxUtts + B].view(np.int32) != 0
        return costs, self.grad, skips

    def _read_record(self):
        rec = self._rec_host.numpy()
        if rec[3] != 0:
            raise RuntimeError("recurrent sweep: inter-CTA wait timed out (flag %d); results are invalid" % int(rec[3]))
        self.regcost = float(rec[5])

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
                                   out=(cost_all[u0:u0 + n], skip_all[u0:u0 + n]))
            u0 += n
        host = self._out_all_host[:2 * B]
        host.copy_(self._out_all[:2 * B], non_blocking=True)
        self._rec_host.copy_(self.record, non_blocking=True)
        torch.cuda.current_stream().synchronize()
        self._read_record()
        out = host.numpy()
        costs = out[:B].astype(np.float64)
        skips = out[B:2 * B].view(np.int32) != 0
        return costs, self.grad, skips

    def costAndGrad(self, data, labels=None, sentence=None):
        """Reference signature (brnnet.py:117): data is inputDim x T float32; returns (cost, grad, skip)
        when training, else the K x T float32 softmax outputs."""
        T = data.shape[1]
        self.setViews(T)
        if not self.train:
            self._batch.pack([data], None).upload()
            probs = self.costAndGradDevice(self._batch)
            out = np.ascontiguousarray(probs.view(T, self.outputDim).cpu().numpy().T)
            flag = int(self._errflag.item())
            if flag != 0:
                raise RuntimeError("recurrent sweep: inter-CTA wait timed out (flag %d); results are invalid" % flag)
            return out
        costs, grad, skips = self.costAndGradBatch([data], [labels])
        cost = float(costs[0])
        if self.reg > 0:
            cost = cost + self.regcost          # brnnet.py:177-183
        return cost, grad, bool(skips[0])

    def forwardBatch(self, datas):
        """The K x T float32 probabilities that costAndGrad(data) returns with train=False, for every utterance of
        `datas` (inputDim x T arrays), in input order.  The utterances are sorted by length and cut into micro-batches
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
                out[u] = np.ascontiguousarray(p[:datas[u].shape[1], j, :].T)
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
        for (w, b), (wi, bi) in zip(self.stack, stack):
            w.copy_(torch.from_numpy(np.ascontiguousarray(wi, dtype=np.float32).reshape(tuple(w.shape))))
            b.copy_(torch.from_numpy(np.ascontiguousarray(bi, dtype=np.float32).reshape(tuple(b.shape))))

    def check_grad(self, data, labels, epsilon=1e-3, maxChecks=10, verbose=True):
        """Finite-difference check on a small section of every weight matrix (brnnet.py:279-297).
        Returns the list of (analytic, numeric) pairs it printed."""
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
