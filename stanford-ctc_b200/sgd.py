"""sgd -- drop-in for ctc_fast/sgd.py (class SGD), computed by libctcb200.

Same constructor, attributes and methods as the reference (sgd.py:10-11, :36, :44, :57):

    SGD(model, maxBatch, alpha=1e-2, optimizer='nesterov', momentum=0.9, maxGradNorm=1500)
    run(data_dict, alis, keys, sizes); toFile(fid); fromFile(fid)
    attributes: alpha, it, costt, expcost, regcost, velocity, momentum, maxGNorm

New, additive: `batchSize` utterances per optimisation step (1 reproduces the reference's
per-utterance schedule exactly) and data parallelism -- when torch.distributed is initialised the
`batchSize` utterances of a step are sharded over the ranks and the flat gradient is summed with ONE
all-reduce (NCCL over NVLink) before the identical, redundant update on every rank.  The clip
threshold `maxGradNorm` applies to the norm of the summed (reduced) gradient.
"""
import logging
import pickle
import random

import numpy as np

import _ctcb
from _ctcb import lib, check, ptr
from nnets.brnnet import FlatList
import parallel


class SGD:

    def __init__(self, model, maxBatch, alpha=1e-2, optimizer='nesterov',
                 momentum=0.9, maxGradNorm=1500, batchSize=1, verbose=True, bucketPool=16):
        torch = _ctcb.require_cuda()
        self._torch = torch
        self.model = model
        self.maxBatch = maxBatch
        self.it = 0
        self.momentum = momentum  # momentum
        self.alpha = alpha  # learning rate
        self.optimizer = optimizer
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
        # the reference's adagrad branch is dead code (`assert False`, sgd.py:24-26)
        assert self.optimizer == 'nesterov', "only the nesterov optimizer exists (sgd.py:24-26)"

        self._vflat = torch.zeros(model.nparams, dtype=torch.float32, device=model.dev)
        self.velocity = FlatList(model._views(self._vflat), self._vflat)
        self._gnorm2 = model._gnorm2          # lives in the 8-float record behind the flat gradient
        self._scratch = torch.zeros(8192, dtype=torch.uint8, device=model.dev)
        # per-step log record {n_valid, sum nll, n_skipped, sweep error flag, gnorm^2, regcost, -, -}: the 8 floats behind
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
        stack = [[w.cpu().numpy(), b.cpu().numpy()] for w, b in self.velocity]
        pickle.dump([self.it, self.costt, self.expcost, stack], fid)

    def fromFile(self, fid):
        torch = self._torch
        try:
            params = pickle.load(fid)
        except UnicodeDecodeError:
            fid.seek(0)
            params = pickle.load(fid, encoding="latin1")
        it, costt, expcost, stack = params
        self.it = it
        self.costt = costt
        self.expcost = expcost
        for (w, b), (wi, bi) in zip(self.velocity, stack):
            w.copy_(torch.from_numpy(np.ascontiguousarray(wi, dtype=np.float32).reshape(tuple(w.shape))))
            b.copy_(torch.from_numpy(np.ascontiguousarray(bi, dtype=np.float32).reshape(tuple(b.shape))))

    # ------------------------------------------------------------------ one optimisation step
    def step_device(self, batch, mom):
        """Enqueue one full Nesterov step for a staged DeviceBatch; never synchronises with the host.
        sgd.py:91-161: look-ahead, costAndGrad, (all-reduce), global norm, clip, velocity, update.
        On a non-default stream the step is captured into a CUDA graph the third time the same (buffers, B, Tmax,
        momentum, step size) combination is seen and replayed as one launch from then on (the first two occurrences
        run eagerly: first-use initialisation is not capturable)."""
        stream = _ctcb.current_stream()
        if not self.useGraphs or not stream:          # the legacy default stream cannot be captured
            return self._step_eager(batch, mom)
        import ctypes
        key = (id(batch), batch.B, batch.Tmax, float(mom), float(self.alpha), float(self.maxGNorm), stream)
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

    def _step_eager(self, batch, mom):
        m = self.model
        stream = _ctcb.current_stream()
        # w = w + mom*velocity (evaluate gradient at future point)      sgd.py:91-93
        check(lib.ctcb_axpy_f32(ptr(m.params), ptr(self._vflat), float(mom), m.nparams, stream))
        # forward, CTC, backward -- and, with a communicator attached (ensure_comm), the exchange: the flat gradient and
        # its statistics tail summed over ranks by libctcb200 itself (NCCL), part of it under the BPTT sweep
        m.costAndGradDevice(batch)
        # gnorm over all parameters as one vector                       sgd.py:103-107
        check(lib.ctcb_sumsq_f32(ptr(m.grads), m.nparams, ptr(self._gnorm2), ptr(self._scratch), stream))
        # undo look-ahead, clip, velocity, update                       sgd.py:97-100,130-140,161
        check(lib.ctcb_sgd_nesterov_step_f32(ptr(m.params), ptr(self._vflat), ptr(m.grads), m.nparams, float(mom),
                                             float(self.alpha), float(self.maxGNorm), ptr(self._gnorm2),
                                             ptr(m.stats), stream))

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
                                               max_labels=m.maxLabels)
        datas = [data_dict[k] for k in used]
        labels = [np.array(alis[k], dtype=np.int32) for k in used]     # only this rank's utterances are converted
        batch = None
        if datas:
            batch = m.swap_batches().pack(datas, labels).upload()
        return dict(batch=batch, used=used, nlab=sum(l.shape[0] for l in labels),
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
        else:                  # this rank has no utterance this step: contribute zeros to the exchange
            st = _ctcb.current_stream()
            m.grads_ext.zero_()
            check(lib.ctcb_brnn_exchange_only(m._h, ptr(m.params), ptr(m.grads), ptr(m.stats), st))
            check(lib.ctcb_sumsq_f32(ptr(m.grads), m.nparams, ptr(self._gnorm2), ptr(self._scratch), st))
            check(lib.ctcb_axpy_f32(ptr(m.params), ptr(self._vflat), float(mom), m.nparams, st))
            check(lib.ctcb_sgd_nesterov_step_f32(ptr(m.params), ptr(self._vflat), ptr(m.grads), m.nparams, float(mom),
                                                 float(self.alpha), float(self.maxGNorm), ptr(self._gnorm2),
                                                 ptr(m.stats), st))
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
        gnorm = float(np.sqrt(host[4]))
        m.regcost = float(host[5])
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
            print("Iter %d : Cost=%.4f, ExpCost=%.4f, GradNorm=%.4f, SeqLen=%d, NumFrames=%d."
                  % (prep["it"], cost, self.expcost[-1] if self.expcost else float('nan'), gnorm,
                     prep["nlab"], prep["nframes"]))

    def run(self, data_dict, alis, keys, sizes):
        """Runs stochastic gradient descent with nesterov acceleration.  Model is objective.
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
            active = (prep["batch"] is not None) or world > 1
            if active:
                self._launch(prep, dist)
            else:
                self.it += 1               # the reference counts skipped utterances too (sgd.py:71)
            if pending is not None:
                self._finish(pending, rank)
            pending = prep if active else None
        if pending is not None:
            self._finish(pending, rank)
