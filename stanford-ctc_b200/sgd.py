"""sgd -- drop-in for ctc_fast/sgd.py (class SGD), computed by libctcb200.

Same constructor, attributes and methods as the reference (sgd.py:10-11, :36, :44, :57):

    SGD(model, maxBatch, alpha=1e-2, optimizer='nesterov', momentum=0.9, maxGradNorm=1500)
    run(data_dict, alis, keys, sizes); toFile(fid); fromFile(fid)
    attributes: alpha, it, costt, expcost, regcost, velocity, momentum, maxGNorm

New, additive: `batchSize` utterances per optimisation step (1 reproduces the reference's
per-utterance schedule exactly) and data parallelism -- when torch.distributed is initialised the
`batchSize` utterances of a step are sharded over the ranks and the flat gradient is summed with ONE
all-reduce (NCCL over NVLink) before the identical, redundant update on every rank.  The clip
threshold `maxGradNorm` applies to the norm of the summed (reduced) gradient.  A rank whose shard of a step
holds more utterances than the net's buffers (`model.maxUtts`) accumulates the gradient over micro-batches of at
most that many and then updates once (step_device_parts), so the batch size is not limited by device memory.
A net built with dropout > 0 has its device step counter advanced once per optimisation step, as the step's first
launch (inside the CUDA graph of step_device), so step `it` draws the masks of step `it` and the counter equals `it`.
`optimizer` is 'nesterov' (the reference's rule and the default), 'adagrad' (the reference's unfinished branch,
sgd.py:24-26,143-158, state `gradt`) or 'adam' (state `moment1`, `moment2`; beta1, beta2, epsilon); the rules are stated
in include/ctcb200.h.  The adaptive rules read the step number t from the same device counter (allocated here when
the net has no dropout), so graph replays see the current step.  The states follow the flat vector, so a net with
layer normalisation simply has its [gamma, beta] pairs in them too.
`emaDecay` = d in (0, 1) keeps an exponential moving average of the weights on the device, `average` (a [W, b]
FlatList of one flat vector, filled with the net's weights when the SGD is built): after each update,
a <- w + d_t (a - w) with d_t = min(d, 1 - 1/t) for the same counter t (ctcb_ema_update_f32), so it is the mean of the
iterates until 1 - 1/t reaches d and an EMA after that.  0 (the default) keeps no average and launches nothing for it.
"""
import logging
import pickle
import random

import numpy as np

import _ctcb
from _ctcb import lib, check, ptr
from nnets.brnnet import FlatList
import parallel

# the state vectors of each rule, by the attribute names that hold them as [W, b] FlatLists (velocity: sgd.py:30-33,
# gradt: sgd.py:28)
OPTIMIZERS = {"nesterov": ("velocity",), "adagrad": ("gradt",), "adam": ("moment1", "moment2")}


def pack_state(optimizer, pairs):
    """The optimiser state entry of the first pickle of params.pk.  pairs: {state name: [[W, b], ...]}.  Nesterov's is
    the reference's list of velocity pairs; the adaptive rules' is a dict that names its rule."""
    if optimizer == "nesterov":
        return pairs["velocity"]
    return dict(optimizer=optimizer, **{name: pairs[name] for name in OPTIMIZERS[optimizer]})


def unpack_state(optimizer, state):
    """{state name: [[W, b], ...]} of a pack_state entry; ValueError when it belongs to another rule."""
    saved = state.get("optimizer") if isinstance(state, dict) else "nesterov"
    if saved != optimizer:
        raise ValueError("the checkpoint holds the state of the %r optimizer; this SGD runs %r" % (saved, optimizer))
    if optimizer == "nesterov":
        return {"velocity": state}
    return {name: state[name] for name in OPTIMIZERS[optimizer]}


class SGD:

    def __init__(self, model, maxBatch, alpha=1e-2, optimizer='nesterov',
                 momentum=0.9, maxGradNorm=1500, batchSize=1, verbose=True, bucketPool=16,
                 beta1=0.9, beta2=0.999, epsilon=1e-8, emaDecay=0.0):
        if optimizer not in OPTIMIZERS:          # ctc/sgd.py:27
            raise ValueError("optimizer=%r: one of %s" % (optimizer, ", ".join(sorted(OPTIMIZERS))))
        if not 0.0 <= emaDecay < 1.0:            # NaN too
            raise ValueError("emaDecay=%r must be in [0, 1)" % (emaDecay,))
        if optimizer == "adam":
            for name, beta in (("beta1", beta1), ("beta2", beta2)):
                if not 0.0 <= beta < 1.0:
                    raise ValueError("%s=%r must be in [0, 1)" % (name, beta))
            if not (0.0 < epsilon < float("inf")):
                raise ValueError("epsilon=%r must be finite and > 0" % (epsilon,))
        torch = _ctcb.require_cuda()
        self._torch = torch
        self.model = model
        self.maxBatch = maxBatch
        self.it = 0
        self.momentum = momentum  # momentum
        self.alpha = alpha  # learning rate
        self.optimizer = optimizer
        self.beta1, self.beta2, self.epsilon = beta1, beta2, epsilon      # adam only
        self.maxGNorm = maxGradNorm  # gradient clip norm value
        self.batchSize = batchSize
        self.verbose = verbose
        # length-bucketed minibatches: pools of bucketPool * batchSize shuffled utterances sorted by length (0 = plain
        # chunks of the shuffled list); padded_frames / real_frames accumulate what the padding costs
        self.bucketPool = bucketPool
        # CUDA graphs: one launch per step instead of ~40 (see step_device)
        import os as _os
        self.useGraphs = not _os.environ.get("CTCB_NO_GRAPH")      # e.g. under a profiler that wants plain launches
        self._graphs = {}
        self._graph_seen = {}
        self._stream = None
        self.padded_frames = 0
        self.real_frames = 0

        # each state is one flat fp32 vector, exposed as the FlatList attribute OPTIMIZERS names (self.velocity, ...)
        self._flat = {}
        for name in OPTIMIZERS[optimizer]:
            self._flat[name] = torch.zeros(model.nparams, dtype=torch.float32, device=model.dev)
            setattr(self, name, FlatList(model._views(self._flat[name]), self._flat[name]))
        self._vflat = self._flat.get("velocity")
        # the weight average, started from the net's current weights so that a first step that is skipped still
        # leaves weights in it
        self.emaDecay = float(emaDecay)
        self._avg, self.average = None, None
        if self.emaDecay > 0.0:
            self._avg = model.params.clone()
            self.average = FlatList(model._views(self._avg), self._avg)
        # the optimisation step on the device: the dropout counter when the net has one, else one of our own where the
        # rule or the average reads t (a Nesterov step on a net without dropout and without an average needs none and
        # launches nothing for it)
        self._step = model.dropoutStep
        if self._step is None and (optimizer != "nesterov" or self._avg is not None):
            self._step = torch.zeros(1, dtype=torch.int64, device=model.dev)
        self._gnorm2 = model._gnorm2          # lives in the 8-float record behind the flat gradient
        self._scratch = torch.zeros(8192, dtype=torch.uint8, device=model.dev)
        # per-step log record {n_valid, sum nll, n_skipped, sweep error flag, gnorm^2, regcost, -, -} (with the
        # intermediate CTC loss its two sums sit before gnorm^2: nnets.brnnet.NNet.statsFloats): the 8 floats behind
        # the flat gradient, copied to pinned host memory on the stream right behind the step (one 32-byte D2H copy,
        # no kernel) and read one step later (two slots alternate)
        self._log_host = [torch.zeros(8, dtype=torch.float32).pin_memory() for _ in range(2)]
        self._log_event = [torch.cuda.Event() for _ in range(2)]
        self._log_slot = 0

        self.costt = []
        self.expcost = []
        self.regcost = []

    # ------------------------------------------------------------------ distributed plumbing
    def _world(self):
        return parallel.world_info()

    # ------------------------------------------------------------------ persistence (sgd.py:36-55)
    def toFile(self, fid):
        pairs = {name: [[w.cpu().numpy(), b.cpu().numpy()] for w, b in getattr(self, name)]
                 for name in OPTIMIZERS[self.optimizer]}
        pickle.dump([self.it, self.costt, self.expcost, pack_state(self.optimizer, pairs)], fid)

    def fromFile(self, fid):
        try:
            params = pickle.load(fid)
        except UnicodeDecodeError:
            fid.seek(0)
            params = pickle.load(fid, encoding="latin1")
        it, costt, expcost, state = params
        states = unpack_state(self.optimizer, state)
        if hasattr(self.model, "check_pair_count"):
            for name, stack in states.items():
                self.model.check_pair_count(stack, getattr(self, name), "optimiser state %r" % name)
        if hasattr(self.model, "check_shapes"):
            for name, stack in states.items():
                self.model.check_shapes(stack, getattr(self, name), "optimiser state %r" % name)
        self.it = it
        self.costt = costt
        self.expcost = expcost
        if self._step is not None:      # a resumed run draws the masks and takes the steps an uninterrupted one would
            self._step.fill_(int(it))
        for name, stack in states.items():
            self._copy_pairs(getattr(self, name), stack)

    def _copy_pairs(self, views, stack):
        torch = self._torch
        for (w, b), (wi, bi) in zip(views, stack):
            w.copy_(torch.from_numpy(np.ascontiguousarray(wi, dtype=np.float32).reshape(tuple(w.shape))))
            b.copy_(torch.from_numpy(np.ascontiguousarray(bi, dtype=np.float32).reshape(tuple(b.shape))))

    def averageToFile(self, fid):
        """The weight average in NNet.toFile's format (a pickled list of [w, b] host arrays), so that NNet.fromFile
        loads it as a net's weights.  runNNet writes it as the third pickle of params.pk."""
        pickle.dump([[w.cpu().numpy(), b.cpu().numpy()] for w, b in self.average], fid)

    def averageFromFile(self, fid):
        """Reads averageToFile's pickle into the average.  At the end of the file (a checkpoint written without an
        average) the average starts again from the net's current weights."""
        try:
            stack = pickle.load(fid)
        except EOFError:
            self._avg.copy_(self.model.params)
            return
        self.model.check_pair_count(stack, self.average, "weight average")
        self.model.check_shapes(stack, self.average, "weight average")
        self._copy_pairs(self.average, stack)

    # ------------------------------------------------------------------ one optimisation step
    def step_device(self, batch, mom):
        """Enqueue one full optimisation step for a staged DeviceBatch; never synchronises with the host.
        sgd.py:91-161: (Nesterov: look-ahead,) costAndGrad, (all-reduce), global norm, clip, update.
        On a non-default stream the step is captured into a CUDA graph the third time the same (buffers, B, Tmax,
        rule and its scalars, step size) combination is seen and replayed as one launch from then on (the first two
        occurrences run eagerly: first-use initialisation is not capturable)."""
        stream = _ctcb.current_stream()
        if not self.useGraphs or not stream:          # the legacy default stream cannot be captured
            return self._step_eager(batch, mom)
        import ctypes
        key = (id(batch), batch.B, batch.Tmax, float(mom), float(self.alpha), float(self.maxGNorm), stream,
               self.optimizer, float(self.beta1), float(self.beta2), float(self.epsilon), self.emaDecay)
        g = self._graphs.get(key)
        if g is None:
            seen = self._graph_seen.get(key, 0)
            if seen < 2:
                self._graph_seen[key] = seen + 1
                if len(self._graph_seen) > 4096:
                    self._graph_seen.clear()
                return self._step_eager(batch, mom)
            check(lib.ctcb_graph_capture_begin(stream))
            try:
                self._step_eager(batch, mom)
            finally:
                g = ctypes.c_void_p()
                rc = lib.ctcb_graph_capture_end(stream, ctypes.byref(g))
            check(rc)
            if len(self._graphs) >= 32:               # ragged corpora produce many (B, Tmax) pairs: keep the cache bounded
                old = next(iter(self._graphs))
                lib.ctcb_graph_destroy(self._graphs.pop(old))
            self._graphs[key] = g
        check(lib.ctcb_graph_launch(g, stream))

    def _advance_step(self, stream):
        """The step's first launch: the device step counter (dropout's and the adaptive rules' t), where one exists."""
        if self._step is not None:
            check(lib.ctcb_dropout_advance(ptr(self._step), stream))

    def _look_ahead(self, mom, stream):
        """Nesterov evaluates the gradient at w + mom*velocity (sgd.py:91-93); the adaptive rules at w."""
        m = self.model
        if self.optimizer == "nesterov":
            check(lib.ctcb_axpy_f32(ptr(m.params), ptr(self._vflat), float(mom), m.nparams, stream))

    def _update(self, mom, stream):
        """Global norm of the (reduced) gradient, then the rule's fused clip and update, then the weight average; a step
        whose utterances were all skipped (n_valid = 0, the first float of m.stats) changes nothing but Nesterov's undo
        of the look-ahead."""
        m = self.model
        # gnorm over all parameters as one vector                       sgd.py:103-107
        check(lib.ctcb_sumsq_f32(ptr(m.grads), m.nparams, ptr(self._gnorm2), ptr(self._scratch), stream))
        if self.optimizer == "nesterov":
            # undo look-ahead, clip, velocity, update                   sgd.py:97-100,130-140,161
            check(lib.ctcb_sgd_nesterov_step_f32(ptr(m.params), ptr(self._vflat), ptr(m.grads), m.nparams, float(mom),
                                                 float(self.alpha), float(self.maxGNorm), ptr(self._gnorm2),
                                                 ptr(m.stats), stream))
        elif self.optimizer == "adagrad":
            check(lib.ctcb_adagrad_step_f32(ptr(m.params), ptr(self._flat["gradt"]), ptr(m.grads), m.nparams,
                                            float(self.alpha), float(self.maxGNorm), ptr(self._gnorm2), ptr(m.stats),
                                            ptr(self._step), stream))
        else:
            check(lib.ctcb_adam_step_f32(ptr(m.params), ptr(self._flat["moment1"]), ptr(self._flat["moment2"]),
                                         ptr(m.grads), m.nparams, float(self.alpha), float(self.beta1),
                                         float(self.beta2), float(self.epsilon), float(self.maxGNorm),
                                         ptr(self._gnorm2), ptr(m.stats), ptr(self._step), stream))
        if self._avg is not None:
            check(lib.ctcb_ema_update_f32(ptr(self._avg), ptr(m.params), m.nparams, self.emaDecay, ptr(m.stats),
                                          ptr(self._step), stream))

    def _step_eager(self, batch, mom):
        m = self.model
        stream = _ctcb.current_stream()
        self._advance_step(stream)
        self._look_ahead(mom, stream)
        # forward, CTC, backward -- and, with a communicator attached (ensure_comm), the exchange: the flat gradient and
        # its statistics tail summed over ranks by libctcb200 itself (NCCL), part of it under the BPTT sweep
        m.costAndGradDevice(batch)
        self._update(mom, stream)

    def step_device_parts(self, pieces, mom):
        """One optimisation step whose shard holds more utterances than the net's buffers (model.maxUtts): the gradient
        is accumulated over consecutive micro-batches (`pieces`: lists of (data, labels) pairs, each at most maxUtts
        long), then the norm and the update run once.  Each micro-batch is packed into the staging buffer the
        device is not reading while the previous one computes; the step runs eagerly (not as a CUDA graph).  With a
        communicator attached, only the last micro-batch's call exchanges, so every rank issues the same
        collectives whatever its number of micro-batches."""
        m = self.model
        stream = _ctcb.current_stream()
        self._advance_step(stream)
        self._look_ahead(mom, stream)
        u0 = 0
        for k, piece in enumerate(pieces):
            batch = m.swap_batches().pack([d for d, _ in piece], [l for _, l in piece]).upload()
            m.costAndGradDevice(batch, first=(k == 0), last=(k == len(pieces) - 1), u0=u0)
            u0 += len(piece)
        self._update(mom, stream)

    def ensure_comm(self):
        """Data parallelism: create this process's ctcb communicator (once per model) and attach it to the net.  The
        NCCL id travels over torch.distributed, which is used for nothing else on the training path."""
        import ctypes
        dist, rank, world = self._world()
        m = self.model
        if world <= 1 or m._comm is not None:
            return
        idbuf = ctypes.create_string_buffer(128)
        if rank == 0:
            check(lib.ctcb_comm_get_unique_id(idbuf))
        box = [idbuf.raw]
        dist.broadcast_object_list(box, src=0)
        comm = ctypes.c_void_p()
        check(lib.ctcb_comm_create(box[0], rank, world, ctypes.byref(comm)))
        check(lib.ctcb_brnn_set_comm(m._h, comm))
        m._comm = comm

    def _momentum_now(self):
        return 0.5 if self.it <= 10 else self.momentum                  # sgd.py:64-74

    def _prepare(self, data_dict, alis, chunk, rank, world):
        """Host side of one step: the reference's length checks (sgd.py:76-88), sharding over ranks, packing into
        the idle staging buffer and the asynchronous H2D copy."""
        m = self.model
        used = parallel.select_step_utterances(data_dict, alis, chunk, self.maxBatch, rank, world, log=logging.info,
                                               max_labels=m.maxLabels, subsample=getattr(m, "subsample", 1))
        datas = [data_dict[k] for k in used]
        labels = [np.array(alis[k], dtype=np.int32) for k in used]     # only this rank's utterances are converted
        batch, pieces = None, None
        if len(datas) > m.maxUtts:
            # more than the buffers hold: micro-batches, packed one by one when the step is launched
            pieces = parallel.micro_batches(list(zip(datas, labels)), m.maxUtts)
        elif datas:
            batch = m.swap_batches().pack(datas, labels).upload()
        return dict(batch=batch, pieces=pieces, used=used, nlab=sum(l.shape[0] for l in labels),
                    nframes=sum(d.shape[1] for d in datas))

    def _launch(self, prep, dist):
        """Device side of one step (never synchronises), followed on the stream by the copy of its log record."""
        m = self.model
        torch = self._torch
        self.it += 1
        prep["it"] = self.it
        mom = self._momentum_now()
        if prep["batch"] is not None:
            self.step_device(prep["batch"], mom)
        elif prep["pieces"]:
            self.step_device_parts(prep["pieces"], mom)
        else:                  # this rank has no utterance this step: contribute zeros to the exchange
            st = _ctcb.current_stream()
            self._advance_step(st)
            m.grads_ext.zero_()
            check(lib.ctcb_brnn_exchange_only(m._h, ptr(m.params), ptr(m.grads), ptr(m.stats), st))
            # the look-ahead after the exchange (which reads w for the L2 term), as this branch has always done it;
            # it writes only w and the norm reads only g, so _update's norm after it gives the same bits
            self._look_ahead(mom, st)
            self._update(mom, st)
        slot = self._log_slot
        self._log_slot ^= 1
        self._log_host[slot].copy_(m.record, non_blocking=True)
        self._log_event[slot].record()
        prep["slot"] = slot

    def _finish(self, prep, rank):
        """The step's log line, as the reference prints every iteration (sgd.py:113-167), from its 28-byte record."""
        m = self.model
        self._log_event[prep["slot"]].synchronize()
        host = self._log_host[prep["slot"]].numpy().copy()
        if host[3] != 0:       # summed over ranks with the rest of the tail: every rank raises together
            raise RuntimeError("recurrent sweep: inter-CTA wait timed out (flag %d); results are invalid" % int(host[3]))
        nvalid, costsum = float(host[0]), float(host[1])
        ns = getattr(m, "statsFloats", 4)        # the tail's floats; gnorm^2 and regcost follow it
        gnorm = float(np.sqrt(host[ns]))
        m.regcost = float(host[ns + 1])
        if nvalid == 0:
            logging.info("SKIPPING: Keys=%s" % (",".join(str(k) for k in prep["used"])))
            return
        cost = costsum / nvalid + (m.regcost if m.reg > 0 else 0.0)
        if np.isfinite(cost):
            # compute exponentially weighted cost                   sgd.py:113-119
            if len(self.expcost) > 0:
                self.expcost.append(.01 * cost + .99 * self.expcost[-1])
            else:
                self.expcost.append(cost)
            self.costt.append(cost)
            if m.reg > 0.0:
                rc = m.regcost
                if len(self.regcost) > 0:
                    self.regcost.append(0.01 * rc + 0.99 * self.regcost[-1])
                else:
                    self.regcost.append(rc)
        if self.verbose and rank == 0:
            # with the intermediate CTC loss: its mean nll over the utterances its CTC kept (not in ExpCost, which
            # stays the main CTC's so that runs with and without it compare)
            inter = ""
            if ns == 6:
                kept = float(host[0]) + float(host[2]) - float(host[5])
                inter = ", InterCost=%.4f" % (float(host[4]) / kept if kept > 0 else float("nan"))
            print("Iter %d : Cost=%.4f%s, ExpCost=%.4f, GradNorm=%.4f, SeqLen=%d, NumFrames=%d."
                  % (prep["it"], cost, inter, self.expcost[-1] if self.expcost else float('nan'), gnorm,
                     prep["nlab"], prep["nframes"]))

    def run(self, data_dict, alis, keys, sizes):
        """Runs stochastic gradient descent with the optimizer's rule (nesterov acceleration by default).  Model is
        objective.
        Steps are software-pipelined: while the device works on minibatch i the host checks, packs, uploads and
        enqueues minibatch i+1 (second staging buffer); step i's log record is read after that."""
        dist, rank, world = self._world()
        self.ensure_comm()
        torch = self._torch
        if torch.cuda.current_stream().cuda_stream == 0:
            # work on a stream of our own (the legacy default stream cannot be graph-captured), ordered after whatever
            # the caller queued and joined again before returning
            if self._stream is None:
                self._stream = torch.cuda.Stream()
            self._stream.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(self._stream):
                self._run(data_dict, alis, keys, sizes, dist, rank, world)
            torch.cuda.current_stream().wait_stream(self._stream)
        else:
            self._run(data_dict, alis, keys, sizes, dist, rank, world)

    def _run(self, data_dict, alis, keys, sizes, dist, rank, world):
        # randomly select minibatch
        random.shuffle(keys)

        step = max(1, self.batchSize)
        if self.bucketPool > 0:
            # minibatches of similar length (every rank draws the same chunks: same seed, same shuffled list)
            chunks, padded, real = parallel.bucketed_chunks(keys, lambda k: data_dict[k].shape[1], step, self.bucketPool)
        else:
            chunks = [keys[k0:k0 + step] for k0 in range(0, len(keys), step)]
            ls = [[data_dict[k].shape[1] for k in c] for c in chunks]
            padded, real = sum(max(l) * len(l) for l in ls if l), sum(sum(l) for l in ls)
        self.padded_frames += padded
        self.real_frames += real
        if not chunks:
            return
        # the host is always one step ahead of the device: step i+1 is packed, uploaded and enqueued while step i
        # runs; only then is step i's log record awaited
        pending = None
        for i in range(len(chunks)):
            prep = self._prepare(data_dict, alis, chunks[i], rank, world)
            active = (prep["batch"] is not None) or bool(prep["pieces"]) or world > 1
            if active:
                self._launch(prep, dist)
            else:
                self.it += 1               # the reference counts skipped utterances too (sgd.py:71)
                self._advance_step(_ctcb.current_stream())
            if pending is not None:
                self._finish(pending, rank)
            pending = prep if active else None
        if pending is not None:
            self._finish(pending, rank)
