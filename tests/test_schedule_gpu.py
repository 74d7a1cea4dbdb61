"""GPU tests of the backward pass's two-stream schedule (csrc/brnn.cu, DESIGN section 3 "Step schedule").

The weight gradients of the layers at and above the temporal block run on a side stream of the lowest priority, queued
behind the event recorded just before each BPTT sweep; the rest of a training call runs on a stream of the greatest
priority forked from the caller's, and the sweep's launch carries the greatest priority as well.  The schedule moves
only when work becomes ready, so:

  * the outputs of one training call (every gradient tensor with the statistics tail, the costs, the skips) have the
    bytes recorded in tests/golden/schedule_cases.json, and it issues the recorded number of launches, for the C2
    shape and for stacks of two and three temporal layers (bi- and uni-directional);
  * a captured call replays to the bytes of an eager one;
  * in the captured graph the main chain's nodes carry the greatest stream priority and the side stream's the least
    (a graph keeps a priority only as a per-node attribute, and runs it only when instantiated to use node priorities).

The recorded bytes depend on the split-K plans, which depend on the number of SMs: on a device with another count the
byte comparison is skipped (the count is recorded beside the digests)."""
import ctypes
import hashlib
import json
import os

import numpy as np
import pytest

import recipes

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "schedule_cases.json")

# kind: brnnet (bi) or rnnet (uni); small cases run the cluster sweep (H = 128) with ragged utterances
CASES = {
    "c2": dict(kind="bi", D=41, K=62, H=512, N=2, tl=1, k=1, T=200, B=32, L=30),
    "bi_k2": dict(kind="bi", D=13, K=11, H=128, N=4, tl=1, k=2, T=60, B=8, L=20),
    "bi_k3": dict(kind="bi", D=13, K=11, H=128, N=4, tl=1, k=3, T=60, B=8, L=20),
    "uni_k3": dict(kind="uni", D=13, K=11, H=128, N=4, tl=1, k=3, T=60, B=8, L=20),
}
RAGGED = ([50, 37, 12, 44, 29, 60, 21, 40], [9, 14, 8, 11, 5, 20, 3, 7])


def make_case(name):
    """A freshly initialised net of case `name` and its staged batch (fixed seeds)."""
    import nnets.brnnet
    import nnets.rnnet
    c = CASES[name]
    mod = nnets.rnnet if c["kind"] == "uni" else nnets.brnnet
    np.random.seed(4)
    nn = mod.NNet(c["D"], c["K"], c["H"], c["N"], c["T"], temporalLayer=c["tl"], maxUtts=c["B"], maxLabels=c["L"],
                  numTemporal=c["k"])
    nn.initParams()
    lens, nlabs = ([c["T"]] * c["B"], [c["L"]] * c["B"]) if name == "c2" else RAGGED
    datas, labelss = recipes.synth_batch(c["D"], c["K"], lens, nlabs, seed=9)
    return nn, nn._batch.pack(datas, labelss).upload()


def outputs(nn, B):
    """sha256 of the bytes of the gradient (with the statistics tail), the costs and the skips of the last call."""
    arrs = {"grads": nn.grads_ext[:nn.nparams + 4], "costs": nn._cost[:B], "skips": nn._skip[:B]}
    return {k: hashlib.sha256(v.detach().cpu().numpy().tobytes()).hexdigest() for k, v in arrs.items()}


def run_case(name):
    """One eager training call: (launches it issued, digests of its outputs)."""
    import torch
    from _ctcb import lib
    nn, batch = make_case(name)
    nn.costAndGradDevice(batch)          # first use: side stream, plans
    torch.cuda.synchronize()
    l0 = lib.ctcb_launch_count()
    nn.costAndGradDevice(batch)
    torch.cuda.synchronize()
    return int(lib.ctcb_launch_count() - l0), outputs(nn, batch.B)


def _golden():
    with open(GOLDEN) as f:
        return json.load(f)


@pytest.mark.parametrize("name", list(CASES))
def test_outputs_and_launches_match_the_recorded_schedule(name, cuda):
    g = _golden()
    launches, dig = run_case(name)
    print(json.dumps({"schedule_%s" % name: dict(launches=launches, recorded=g["cases"][name]["launches"])}))
    assert launches == g["cases"][name]["launches"]
    if cuda.cuda.get_device_properties(0).multi_processor_count != g["sms"]:
        pytest.skip("split-K plans follow the SM count: recorded on %d SMs" % g["sms"])
    assert dig == g["cases"][name]["outputs"]


@pytest.mark.parametrize("name", ["c2", "uni_k3"])
def test_captured_call_equals_eager_call(name, cuda):
    import _ctcb
    from _ctcb import lib, check
    stream = cuda.cuda.Stream()
    with cuda.cuda.stream(stream):
        nn, batch = make_case(name)
        nn.costAndGradDevice(batch)
        cuda.cuda.synchronize()
        eager = outputs(nn, batch.B)
        st = _ctcb.current_stream()
        check(lib.ctcb_graph_capture_begin(st))
        try:
            nn.costAndGradDevice(batch)
        finally:
            g = ctypes.c_void_p()
            rc = lib.ctcb_graph_capture_end(st, ctypes.byref(g))
        check(rc)
        for w, b in nn.grad:          # NaN into every tensor (the alignment gaps between them are never written)
            w.fill_(float("nan"))
            b.fill_(float("nan"))
        nn.stats.fill_(float("nan"))
        nn._cost.fill_(float("nan"))
        check(lib.ctcb_graph_launch(g, st))
        cuda.cuda.synchronize()
        lib.ctcb_graph_destroy(g)
    assert outputs(nn, batch.B) == eager


def _driver():
    cu = ctypes.CDLL("libcuda.so.1")

    def ck(rc):
        assert rc == 0, "CUDA driver call failed: %d" % rc
    return cu, ck


def test_captured_nodes_carry_the_schedule_priorities(cuda):
    cu, ck = _driver()
    least, greatest = ctypes.c_int(), ctypes.c_int()
    ck(cu.cuCtxGetStreamPriorityRange(ctypes.byref(least), ctypes.byref(greatest)))
    assert greatest.value < least.value, "the device has one stream priority"
    stream = cuda.cuda.Stream()
    with cuda.cuda.stream(stream):
        nn, batch = make_case("c2")
        nn.costAndGradDevice(batch)
        cuda.cuda.synchronize()
        h = ctypes.c_void_p(stream.cuda_stream)
        ck(cu.cuStreamBeginCapture_v2(h, 1))          # CU_STREAM_CAPTURE_MODE_THREAD_LOCAL
        try:
            nn.costAndGradDevice(batch)
        finally:
            graph = ctypes.c_void_p()
            rc = cu.cuStreamEndCapture(h, ctypes.byref(graph))
        ck(rc)
    try:
        n = ctypes.c_size_t(0)
        ck(cu.cuGraphGetNodes(graph, None, ctypes.byref(n)))
        nodes = (ctypes.c_void_p * n.value)()
        ck(cu.cuGraphGetNodes(graph, nodes, ctypes.byref(n)))

        class Params(ctypes.Structure):     # CUDA_KERNEL_NODE_PARAMS_v2
            _fields_ = [("func", ctypes.c_void_p), ("dims", ctypes.c_uint * 7), ("kernelParams", ctypes.c_void_p),
                        ("extra", ctypes.c_void_p), ("kern", ctypes.c_void_p), ("ctx", ctypes.c_void_p)]
        prio = {}
        for node in nodes:
            t = ctypes.c_int()
            ck(cu.cuGraphNodeGetType(ctypes.c_void_p(node), ctypes.byref(t)))
            if t.value != 0:                            # CU_GRAPH_NODE_TYPE_KERNEL
                continue
            val = (ctypes.c_char * 64)()                # CUlaunchAttributeValue
            ck(cu.cuGraphKernelNodeGetAttribute(ctypes.c_void_p(node), 8, val))     # CU_LAUNCH_ATTRIBUTE_PRIORITY
            p = Params()
            ck(cu.cuGraphKernelNodeGetParams_v2(ctypes.c_void_p(node), ctypes.byref(p)))
            name = ctypes.c_char_p()
            if p.func:
                ck(cu.cuFuncGetName(ctypes.byref(name), ctypes.c_void_p(p.func)))
            else:
                ck(cu.cuKernelGetName(ctypes.byref(name), ctypes.c_void_p(p.kern)))
            prio.setdefault(name.value.decode(), []).append(int.from_bytes(bytes(val[:4]), "little", signed=True))
    finally:
        cu.cuGraphDestroy(graph)
    def named(part):
        return [x for k, v in prio.items() if part in k for x in v]
    print(json.dumps({"schedule_priorities": dict(least=least.value, greatest=greatest.value, nodes=prio)}))
    # the main chain (forward and BPTT sweeps, CTC) at the greatest priority
    assert named("sweep_cluster_kernel") == [greatest.value] * 2
    assert named("ctc_par_kernel") == [greatest.value]
    # bias sums: maps 2 and 1 on the side stream (least), map 0 in the main chain's tail (greatest)
    assert sorted(named("colsum_stage2")) == sorted([least.value, least.value, greatest.value])
    # the L2 cost's reset runs on the caller's stream after the join
    assert named("set_scalar_kernel") == [0]
    assert set(x for v in prio.values() for x in v) <= {least.value, greatest.value, 0}
