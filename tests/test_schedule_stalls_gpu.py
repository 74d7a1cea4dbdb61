"""GPU tests of the training call's two-stream schedule under forced stalls (csrc/brnn.cu, DESIGN section 3 "Step
schedule").

A training call forks its main chain (forward, CTC, delta chain, sweeps) from the caller's stream and runs the weight
gradients of the maps at and above the temporal block on a side stream; events order the two, and both are joined back
into the caller's stream.  At its natural timing on an idle card a missing edge almost never changes a byte, so each
case here runs the call three times from other data in the workspace: with CTCB_STALL off, with the main chain held for
CTCB_STALL_US right after each point where it releases the side stream (`main`: 1 + 2k stalls for k temporal layers),
and with the side stream held right after each point where it is released (`side`: 2k stalls).  `main` exposes a
side-stream read of something the main chain has not written yet; `side` a main-chain overwrite of something the side
stream has not read yet, and a caller that runs on before the join.  Every output must keep its bytes:

  * the gradient with its statistics tail, the costs, the skips, the L2 cost and the probabilities;
  * every activation and delta ctcb_brnn_activation_offset exposes for the net (what = 0..7, every layer it accepts).

The call runs on a stream the test creates; its outputs are cloned on that stream, which alone is synchronised before
they are read, so a missing join shows as an early snapshot.  A stalled eager call must also launch exactly the stall
count more kernels than the unstalled one, take at least that many stall periods of host time, and report no sweep
barrier timeout in its statistics tail.  The stall is max(500 us, 4x the unstalled call's event-timed duration), capped
at the knob's 100 ms, so the held stream waits several whole calls while the other runs as far as its edges let it.

Variants: one eager call, two micro-batches into one gradient, one captured call replayed against the eager bytes;
through the Python layer SGD.step_device_parts (five micro-batches a step, Nesterov and Adam) and SGD.step_device with
its graph replay; and two ranks where two GPUs are visible.  Each case prints one JSON line (pytest -s)."""
import ctypes
import hashlib
import json
import os
import subprocess
import sys
import time

import numpy as np
import pytest

import recipes
from test_dp_gpu import ROOT, WORKER as DP_WORKER
from test_schedule_gpu import CASES as SCHEDULE_CASES, GOLDEN as SCHEDULE_GOLDEN, make_case as schedule_case
from test_step_reductions_gpu import NETS as STEP_NETS, _batches as step_batches, _hook, _net as step_net

pytestmark = pytest.mark.gpu
MODES = ("main", "side")
STALL_MIN_US, STALL_MAX_US = 500, 100000
SWEEP_KERNELS = {0: "generic", 1: "cluster", 2: "tensor_core"}
REACHED = dict(main=False, side=False, cluster=False, tensor_core=False, generic=False, lstm=False, peephole=False,
               ln_above=False, s_side=False, parts=False, graph=False, sgd_parts=False, sgd_graph=False)

# nets of their own: the tensor-core sweep (H = 1024) and the generic cooperative sweep (CTCB_SWEEP=barrier), both with
# an L2 term, so that regcost and the L2 gradient run on the caller's stream behind the join
EXTRA_NETS = {
    "bi_tc_h1024_reg": dict(D=23, K=29, H=1024, N=2, T=24, B=4, L=6, kw=dict(temporalLayer=1, reg=1e-3)),
    "bi_barrier_stack2_reg": dict(D=23, K=30, H=128, N=4, T=32, B=8, L=6,
                                  kw=dict(temporalLayer=2, numTemporal=2, reg=1e-3), knobs={"CTCB_SWEEP": "barrier"}),
}
NAMES = list(SCHEDULE_CASES) + list(STEP_NETS) + list(EXTRA_NETS)


def _set_knob(name, value):
    from _ctcb import lib, check
    check(lib.ctcb_debug_set_knob(name.encode(), None if value is None else str(value).encode()))


class Case:
    """A net, two staged batches of other data (fixed seeds), the knobs it runs under and its number of temporal
    layers."""

    def __init__(self, name):
        self.name = name
        self.knobs = {}
        if name in SCHEDULE_CASES:
            c = SCHEDULE_CASES[name]
            self.nn, b0 = schedule_case(name)
            lens = [c["T"]] * c["B"] if name == "c2" else [48, 39, 31, 23, 20, 16, 10, 2]
            nlabs = [min(c["L"], max(1, t // 3)) for t in lens]
            datas, labelss = recipes.synth_batch(c["D"], c["K"], lens, nlabs, seed=10)
            self.batches = [b0, self.nn.swap_batches().pack(datas, labelss).upload()]
        elif name in STEP_NETS:
            c = STEP_NETS[name]
            self.nn = step_net(c)
            self.batches = []
            for seed in (41, 42):
                _, (datas, labelss) = step_batches(c, seed)
                self.batches.append(self.nn.swap_batches().pack(datas, labelss).upload())
        else:
            import nnets.brnnet as brnnet
            c = EXTRA_NETS[name]
            self.knobs = c.get("knobs", {})
            for k, v in self.knobs.items():         # before the net: workspace sizes follow the plans
                _set_knob(k, v)
            np.random.seed(6)
            self.nn = brnnet.NNet(c["D"], c["K"], c["H"], c["N"], c["T"], maxUtts=c["B"], maxLabels=c["L"], **c["kw"])
            self.nn.initParams()
            self.batches = []
            rng = np.random.RandomState(3)
            for seed in (11, 12):
                lens = [int(t) for t in rng.randint(c["T"] // 2, c["T"] + 1, size=c["B"])]
                lens[0] = c["T"]
                nlabs = [int(x) for x in rng.randint(1, c["L"] + 1, size=c["B"])]
                datas, labelss = recipes.synth_batch(c["D"], c["K"], lens, nlabs, seed=seed)
                self.batches.append(self.nn.swap_batches().pack(datas, labelss).upload())
        self.nt = self.nn.numTemporal

    def stalls(self, mode):
        """Stall launches of one call in `mode`."""
        if self.nt == 0 or mode == "off":
            return 0
        return 1 + 2 * self.nt if mode == "main" else 2 * self.nt

    def taps(self, batch):
        """{name: (byte offset, bytes)} of every activation and delta the hook exposes after a call on `batch`."""
        nn = self.nn
        Tp = nn.frames(batch.Tmax)
        maps = range(1, nn.numLayers + 2)
        temporal = range(nn.temporalLayer, nn.temporalLayer + self.nt)
        out, seen = {}, set()
        for what in range(8):
            # maps for the outputs (0) and deltas (7), the temporal layers for their directions, gates and cells
            for layer in (maps if what in (0, 7) else [0] if what == 6 else temporal):
                h = _hook(nn, what, layer)
                if h is None or h[0] in seen:
                    continue
                off, width = h
                seen.add(off)
                reduced = nn.subsample > 1 and (what == 6 or layer >= nn.subsampleLayer)
                out["w%d_l%d" % (what, layer)] = (off, 4 * (Tp if reduced else batch.Tmax) * batch.B * width)
        return out

    def sweep_family(self):
        from _ctcb import lib, check
        nn = self.nn
        if not self.nt:
            return None
        if nn.cell == "lstm":
            return "lstm"
        out = (ctypes.c_int32 * 8)()
        check(lib.ctcb_debug_sweep_plan(nn.layerSize, self.batches[0].B, 1 if nn.unidirectional else 2, out))
        return SWEEP_KERNELS[out[0]]

    def close(self):
        for k in self.knobs:
            _set_knob(k, None)


def _poison(nn):
    """NaN into every gradient tensor, the statistics tail, the L2 cost, the costs and the probabilities: an output the
    call does not write in time keeps it.  (The alignment gaps between the tensors are never written and stay 0.)"""
    for w, b in nn.grad:
        w.fill_(float("nan"))
        b.fill_(float("nan"))
    nn.stats.fill_(float("nan"))
    nn._regcost.fill_(float("nan"))
    nn._out.fill_(float("nan"))
    if nn._probs is not None:
        nn._probs.fill_(float("nan"))


def _snapshot(case, batch):
    """Clones, queued on the current stream, of every output of the last call on `batch`."""
    nn = case.nn
    B = batch.B
    snap = {"grads": nn.grads_ext[:nn.nparams + 4].clone(), "costs": nn._cost[:B].clone(),
            "skips": nn._skip[:B].clone(), "regcost": nn._regcost.clone(),
            "probs": nn._probs_view(B, nn.frames(batch.Tmax)).clone()}
    for k, (off, n) in case.taps(batch).items():
        snap[k] = nn._ws[off:off + n].clone()
    return snap


def _host(snap):
    return {k: v.cpu().numpy() for k, v in snap.items()}


def _same(a, b):
    """Names of the outputs whose bytes differ."""
    assert a.keys() == b.keys()
    return [k for k in a if a[k].tobytes() != b[k].tobytes()]


def _call(case, batch, first=True, last=True, u0=0):
    case.nn.costAndGradDevice(batch, want_probs=True, first=first, last=last, u0=u0)


def _scrub(case, stream, batch):
    """An unstalled call on other data, so that the workspace does not already hold what the next call writes."""
    _set_knob("CTCB_STALL", "off")
    _call(case, batch)
    stream.synchronize()


def _eager(case, stream, mode, us, timed=False):
    """One call on batch 0 after a scrub with batch 1: (host outputs, launches, host seconds, device ms or None)."""
    import torch
    from _ctcb import lib
    nn, b0, b1 = case.nn, case.batches[0], case.batches[1]
    _scrub(case, stream, b1)
    _poison(nn)
    _set_knob("CTCB_STALL", mode)
    _set_knob("CTCB_STALL_US", us)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    stream.synchronize()
    t0 = time.perf_counter()
    l0 = lib.ctcb_launch_count()
    if timed:
        e0.record(stream)
    _call(case, b0)
    if timed:
        e1.record(stream)
    launches = int(lib.ctcb_launch_count() - l0)
    snap = _snapshot(case, b0)
    stream.synchronize()
    dt = time.perf_counter() - t0
    _set_knob("CTCB_STALL", "off")
    return _host(snap), launches, dt, (e0.elapsed_time(e1) if timed else None)


def _parts(case, stream, mode, us):
    """Batch 0 with CTCB_PART_FIRST, then batch 1 with CTCB_PART_LAST into one gradient: (host outputs, host seconds)."""
    nn, b0, b1 = case.nn, case.batches[0], case.batches[1]
    _scrub(case, stream, b1)
    _poison(nn)
    _set_knob("CTCB_STALL", mode)
    _set_knob("CTCB_STALL_US", us)
    stream.synchronize()
    t0 = time.perf_counter()
    _call(case, b0, first=True, last=False, u0=0)
    _call(case, b1, first=False, last=True, u0=b0.B)
    snap = _snapshot(case, b1)
    stream.synchronize()
    dt = time.perf_counter() - t0
    _set_knob("CTCB_STALL", "off")
    return _host(snap), dt


def _graph(case, stream, mode, us):
    """The call on batch 0 captured under `mode`, replayed after a scrub: (host outputs, launches, host seconds)."""
    import _ctcb
    from _ctcb import lib, check
    nn, b0, b1 = case.nn, case.batches[0], case.batches[1]
    _set_knob("CTCB_STALL", mode)
    _set_knob("CTCB_STALL_US", us)
    st = _ctcb.current_stream()
    check(lib.ctcb_graph_capture_begin(st))
    try:
        _call(case, b0)
    finally:
        g = ctypes.c_void_p()
        rc = lib.ctcb_graph_capture_end(st, ctypes.byref(g))
    check(rc)
    try:
        _scrub(case, stream, b1)
        _poison(nn)
        stream.synchronize()
        t0 = time.perf_counter()
        l0 = lib.ctcb_launch_count()
        check(lib.ctcb_graph_launch(g, st))
        launches = int(lib.ctcb_launch_count() - l0)
        snap = _snapshot(case, b0)
        stream.synchronize()
        dt = time.perf_counter() - t0
    finally:
        lib.ctcb_graph_destroy(g)
        _set_knob("CTCB_STALL", "off")
    return _host(snap), launches, dt


def _digests(out):
    return {k: hashlib.sha256(out[k].tobytes()).hexdigest() for k in ("grads", "costs", "skips")}


def _reach(case):
    nn = case.nn
    fam = case.sweep_family()
    if fam:
        REACHED[fam] = True
    if nn.cell == "lstm" and nn.peephole:
        REACHED["peephole"] = True
    tl, k = nn.temporalLayer, nn.numTemporal
    if k and nn.layerNorm and any(i > tl + k - 1 for i in nn.normedLayers()):
        REACHED["ln_above"] = True
    if k and nn.subsample > 1 and nn.subsampleLayer - 1 >= tl:      # map L's weight gradient on the side stream
        REACHED["s_side"] = True


@pytest.mark.parametrize("name", NAMES)
def test_outputs_keep_their_bytes_under_stalls(name, cuda):
    torch = cuda
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        case = Case(name)
        try:
            _run_case(case, stream)
        finally:
            _set_knob("CTCB_STALL", "off")
            _set_knob("CTCB_STALL_US", None)
            case.close()


def _run_case(case, stream):
    import torch
    torch.cuda.synchronize()                     # the uploads of set-up; nothing below synchronises the device
    for b in case.batches:                       # first use: side stream, plans
        _scrub(case, stream, b)
    ref, ref_launches, ref_dt, ref_ms = _eager(case, stream, "off", 1, timed=True)
    assert ref["grads"][-1] == 0.0, "sweep error word %r" % ref["grads"][-1]
    us = int(min(STALL_MAX_US, max(STALL_MIN_US, np.ceil(4000.0 * ref_ms))))
    rep = dict(stall_us=us, call_ms=round(ref_ms, 4), launches=ref_launches, sweep=case.sweep_family(),
               outputs=len(ref))
    golden = None
    if case.name in SCHEDULE_CASES:             # the unstalled bytes are the recorded ones
        with open(SCHEDULE_GOLDEN) as f:
            g = json.load(f)
        if torch.cuda.get_device_properties(0).multi_processor_count == g["sms"]:
            golden = rep["golden"] = _digests(ref) == g["cases"][case.name]["outputs"]
    ref_parts, _ = _parts(case, stream, "off", 1)
    bad, errs, missed = {}, {}, {}
    for mode in MODES:
        n = case.stalls(mode)
        out, launches, dt, _ = _eager(case, stream, mode, us)
        parts, dt_parts = _parts(case, stream, mode, us)
        graph, g_launches, dt_graph = _graph(case, stream, mode, us)
        rep[mode] = dict(stalls=n, launches=launches, eager_s=round(dt, 4), parts_s=round(dt_parts, 4),
                         graph_s=round(dt_graph, 4))
        for what, got, want in (("eager", out, ref), ("parts", parts, ref_parts), ("graph", graph, ref)):
            diff = _same(got, want)
            if diff:
                bad["%s/%s" % (mode, what)] = diff
            if got["grads"][-1] != 0.0:           # the statistics tail's sweep error word
                errs["%s/%s" % (mode, what)] = float(got["grads"][-1])
        # every stall was launched, in the graph as well, and held its stream for its period
        period = n * us * 1e-6
        if launches != ref_launches + n or g_launches != launches or \
                not (dt >= period and dt_graph >= period and dt_parts >= 2 * period):
            missed[mode] = dict(launches=launches, graph_launches=g_launches, want=ref_launches + n, period_s=period)
        REACHED[mode] |= n > 0
    rep["differ"], rep["error_words"], rep["stalls_missed"] = bad, errs, missed
    print(json.dumps({"stalls_" + case.name: rep}))
    assert not missed, missed
    assert not errs, ("a sweep barrier timed out under the stall", errs)
    assert not bad, bad
    assert golden is not False, "the unstalled bytes differ from tests/golden/schedule_cases.json"
    REACHED["parts"] = REACHED["graph"] = True
    _reach(case)


# ------------------------------------------------------------------------------------------------ through sgd.SGD
SGD_NET = dict(STEP_NETS["bi_relu_stack2"], kw=dict(STEP_NETS["bi_relu_stack2"]["kw"], reg=1e-3))


def _sgd_pieces(c, step):
    """Five micro-batches of at most maxUtts utterances of other lengths for optimisation step `step`."""
    from test_step_reductions_gpu import D_IN, MAXB, MAXT
    rng = np.random.RandomState(100 + step)
    pieces = []
    for p in range(5):
        B = MAXB if p < 4 else 3
        lens = [int(t) for t in rng.randint(4, MAXT + 1, size=B)]
        nlabs = [int(x) for x in rng.randint(1, 4, size=B)]
        datas, labelss = recipes.synth_batch(D_IN, c["K"], lens, nlabs, seed=1000 * step + p)
        pieces.append(list(zip(datas, labelss)))
    return pieces


def _sgd_run(mode, optimizer, graphs):
    """Three steps of SGD.step_device_parts (graphs=False) or four of SGD.step_device on one batch (graphs=True, the
    third captured, the fourth a replay) under `mode` on a stream of our own: host copies of the parameters and the
    optimiser state, and the host seconds."""
    import torch
    import sgd
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        nn = step_net(SGD_NET)
        opt = sgd.SGD(nn, 40, alpha=1e-3, optimizer=optimizer, momentum=0.9, maxGradNorm=5.0, verbose=False)
        opt.useGraphs = True
        steps = [_sgd_pieces(SGD_NET, s) for s in range(3)]
        batch = None
        if graphs:
            d, l = zip(*steps[0][0])
            batch = nn.swap_batches().pack(list(d), list(l)).upload()
        torch.cuda.synchronize()
        _set_knob("CTCB_STALL", mode)
        _set_knob("CTCB_STALL_US", 2000)
        try:
            t0 = time.perf_counter()
            if graphs:
                for _ in range(4):
                    opt.step_device(batch, 0.9)
                assert len(opt._graphs) == 1, "the step was not captured"
            else:
                for pieces in steps:
                    opt.step_device_parts(pieces, 0.9)
            snap = [nn.params.clone()] + [opt._flat[k].clone() for k in sorted(opt._flat)] + [nn.stats.clone()]
            stream.synchronize()
            dt = time.perf_counter() - t0
        finally:
            _set_knob("CTCB_STALL", "off")
            _set_knob("CTCB_STALL_US", None)
            for g in opt._graphs.values():
                from _ctcb import lib
                lib.ctcb_graph_destroy(g)
            opt._graphs.clear()
    return [s.cpu().numpy() for s in snap], dt


@pytest.mark.parametrize("optimizer", ["nesterov", "adam"])
def test_sgd_step_device_parts_keeps_its_bits_under_stalls(optimizer, cuda):
    ref, _ = _sgd_run("off", optimizer, graphs=False)
    rep = {}
    for mode in MODES:
        got, dt = _sgd_run(mode, optimizer, graphs=False)
        nt = SGD_NET["kw"]["numTemporal"]
        n = 3 * 5 * (1 + 2 * nt if mode == "main" else 2 * nt)
        rep[mode] = dict(stalls=n, stall_us=2000, host_s=round(dt, 4))
        assert dt >= n * 2000e-6, (mode, dt)
        assert got[-1][3] == 0.0, (mode, "a sweep barrier timed out under the stall")
        for i, (a, b) in enumerate(zip(got, ref)):
            assert a.tobytes() == b.tobytes(), (mode, "params" if i == 0 else "state %d" % i)
    print(json.dumps({"stalls_sgd_parts_" + optimizer: rep}))
    REACHED["sgd_parts"] = True


def test_sgd_step_device_graph_replay_keeps_its_bits_under_stalls(cuda):
    ref, _ = _sgd_run("off", "nesterov", graphs=True)
    rep = {}
    for mode in MODES:
        got, dt = _sgd_run(mode, "nesterov", graphs=True)
        nt = SGD_NET["kw"]["numTemporal"]
        n = 4 * (1 + 2 * nt if mode == "main" else 2 * nt)
        rep[mode] = dict(stalls=n, stall_us=2000, host_s=round(dt, 4))
        assert dt >= n * 2000e-6, (mode, dt)
        assert got[-1][3] == 0.0, (mode, "a sweep barrier timed out under the stall")
        for i, (a, b) in enumerate(zip(got, ref)):
            assert a.tobytes() == b.tobytes(), (mode, "params" if i == 0 else "state %d" % i)
    print(json.dumps({"stalls_sgd_graph": rep}))
    REACHED["sgd_graph"] = True


# ------------------------------------------------------------------------------------------------ two ranks
def test_two_ranks_keep_their_bits_under_stalls(cuda, tmp_path):
    """The early all-reduce runs on the side stream: two ranks (the run of test_dp_gpu.py) under each stall mode end
    with parameters bit-identical to each other and to the unstalled two-rank run."""
    if cuda.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    script = tmp_path / "worker.py"
    script.write_text(DP_WORKER % ROOT)
    params = {}
    for port, mode in enumerate(("off",) + MODES):
        out = tmp_path / mode
        out.mkdir()
        env = {k: v for k, v in os.environ.items() if k not in ("RANK", "WORLD_SIZE", "LOCAL_RANK")}
        env.update(CTCB_STALL=mode, CTCB_STALL_US="2000")
        p = subprocess.Popen([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
                              "--master-addr", "127.0.0.1", "--master-port", str(29641 + port), str(script), str(out)],
                             env=env, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
        try:
            _, err = p.communicate(timeout=600)
        finally:
            if p.poll() is None:
                p.kill()
        assert p.returncode == 0, err[-2000:]
        r0, r1 = np.load(out / "params_w2_r0.npy"), np.load(out / "params_w2_r1.npy")
        assert r0.tobytes() == r1.tobytes(), mode
        params[mode] = r0
    for mode in MODES:
        assert params[mode].tobytes() == params["off"].tobytes(), mode


def test_every_stall_mode_and_schedule_path_was_reached(cuda):
    """The cases above ran both stall modes, the cluster, tensor-core and generic sweeps, the LSTM sweep with
    peepholes, a normalised map above the temporal block, a side-stream read of S, micro-batches, a graph replay and
    both SGD paths."""
    missing = [k for k, v in REACHED.items() if not v]
    assert not missing, missing
