"""GPU tests of zoneout on the LSTM cell (ctcb_brnn_config.zoneout = 1) on one H100.

The sweep alone (ctcb_lstm_sweep_zoneout_f32) on every plan, with and without peepholes, in training and expectation
mode, against a float64 step from its own previous state under the element-wise bounds C_FWD / C_ACT / C_BPTT of
test_lstm_plans_gpu.py (the lambdas in c64, h64 and the float64 BPTT), and its exact properties: a kept value has the bytes of the
previous one, z = 0 gives the plain (and peephole) sweep's bytes, the bytes do not depend on the plan, the error flag
stays 0.  Then whole nets against tests/net_oracle.Net (tests/net_check.py), micro-batches, emulated shards,
graph replay and resume bit for bit, forward-only probabilities against the expectation oracle, check_grad, forced
stalls and runNNet.  Each comparison prints its measured numbers as one JSON line (pytest -s)."""
import ctypes
import json
import os

import numpy as np
import pytest

import recipes
from net_check import bits as _bits, compare, rel as _rel
from net_oracle import Net, zoneout_masks
from recipes import knobs  # noqa: F401  (fixture)
from test_lstm_plans_gpu import C_ACT, C_BPTT, C_FWD, _check_bptt, _check_forward

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------ the sweep alone
class Sweep:
    """Device arrays of one sweep problem: pre-activations of a [T][B][G] layer, U and P per direction, lengths."""

    def __init__(self, T, B, H, ndir, peep, seed=3):
        import torch
        rng = np.random.RandomState(seed)
        self.T, self.B, self.H, self.ndir = T, B, H, ndir
        self.G = ndir * 4 * H
        self.lens = [T] + [int(x) for x in rng.randint(1, T + 1, size=B - 1)]
        s = 1.0 / np.sqrt(H)
        self.pre = rng.uniform(-1.5, 1.5, (T, B, self.G)).astype(np.float32)
        self.U = [rng.uniform(-2 * s, 2 * s, (4 * H, H)).astype(np.float32) for _ in range(ndir)]
        self.P = [rng.uniform(-0.5, 0.5, (3, H)).astype(np.float32) for _ in range(ndir)] if peep else None
        self.dh = rng.uniform(-1, 1, (T, B, H)).astype(np.float32)
        dev = lambda x: torch.from_numpy(x).cuda()      # noqa: E731
        self.d_len = dev(np.array(self.lens, dtype=np.int32))
        self.d_U = [dev(u) for u in self.U]
        self.d_P = [dev(p) for p in self.P] if peep else None
        self.d_dh = dev(self.dh)
        self.step = torch.tensor([5], dtype=torch.int64, device="cuda")

    def run(self, zc, zh, train, plain=False, layer=2, first=3, stride=2):
        """Forward then BPTT; returns host arrays gates, h [ndir], c [ndir], dz, and the error flag."""
        import torch
        from _ctcb import lib, check
        T, B, H, G = self.T, self.B, self.H, self.G
        gates = torch.from_numpy(self.pre.copy()).cuda()
        h = [torch.zeros(T, B, H, device="cuda") for _ in range(2)]
        c = [torch.zeros(T, B, H, device="cuda") for _ in range(2)]
        dz = torch.zeros(T, B, G, device="cuda")
        n = lib.ctcb_lstm_sweep_zoneout_workspace_bytes(H, B)
        ws = torch.zeros(n // 4 + 64, dtype=torch.float32, device="cuda")
        p = lambda t: None if t is None else t.data_ptr()      # noqa: E731
        Ub = self.d_U[1] if self.ndir == 2 else None
        Pf = self.d_P[0] if self.d_P else None
        Pb = self.d_P[1] if self.d_P and self.ndir == 2 else None
        st = torch.cuda.current_stream().cuda_stream
        for mode in (0, 1):
            if plain and Pf is None:
                rc = lib.ctcb_lstm_sweep_f32(mode, T, B, H, p(self.d_len), p(gates), p(self.d_U[0]), p(Ub), p(h[0]),
                                             p(h[1]), p(c[0]), p(c[1]), p(self.d_dh), p(dz), p(ws), n, st)
            elif plain:
                rc = lib.ctcb_lstm_sweep_peephole_f32(mode, T, B, H, p(self.d_len), p(gates), p(self.d_U[0]), p(Ub),
                                                      p(Pf), p(Pb), p(h[0]), p(h[1]), p(c[0]), p(c[1]), p(self.d_dh),
                                                      p(dz), p(ws), n, st)
            else:
                rc = lib.ctcb_lstm_sweep_zoneout_f32(mode, T, B, H, p(self.d_len), p(gates), p(self.d_U[0]), p(Ub),
                                                     p(Pf), p(Pb), p(h[0]), p(h[1]), p(c[0]), p(c[1]), p(self.d_dh),
                                                     p(dz), zc, zh, int(train), 77, p(self.step), first, stride,
                                                     layer, p(ws), n, st)
            check(rc)
            if mode == 0:
                fwd = (gates.cpu().numpy().copy(), [x.cpu().numpy() for x in h[:self.ndir]],
                       [x.cpu().numpy() for x in c[:self.ndir]])
        torch.cuda.synchronize()
        err = int(ws[:1].view(torch.int32).item())
        return fwd[0], fwd[1], fwd[2], dz.cpu().numpy(), err

    def lambdas(self, zc, zh, train, d, b, layer=2, first=3, stride=2):
        """[T][H] float64 lambdas of utterance b, direction d."""
        if not train:
            return (np.full((self.T, self.H), float(np.float32(zc))), np.full((self.T, self.H), float(np.float32(zh))))
        lc, lh = zoneout_masks(zc, zh, 77, 5, layer, d, first + stride * b, self.T, self.H)
        return lc.astype(np.float64), lh.astype(np.float64)


class _Problem:
    """The view of a Sweep that _check_forward / _check_bptt of test_lstm_plans_gpu.py read."""

    def __init__(self, sw):
        self.H, self.T, self.B, self.ndir = sw.H, sw.T, sw.B, sw.ndir
        self.lens, self.pre, self.Us, self.Ps, self.dh = np.asarray(sw.lens), sw.pre, sw.U, sw.P, sw.dh


def _lambdas(sw, zc, zh, train):
    """Per direction [T][B][H] lambda_c and lambda_h of every utterance."""
    lam = [[sw.lambdas(zc, zh, train, d, b) for b in range(sw.B)] for d in range(sw.ndir)]
    return ([np.stack([x[0] for x in per], axis=1) for per in lam], [np.stack([x[1] for x in per], axis=1) for per in lam])


PLANS = [("auto", None), ("reread", None), ("auto", 1), ("reread", 2)]
SWEEPS = {
    "h64_bi": dict(T=40, B=13, H=64, ndir=2),
    "h70_uni": dict(T=25, B=9, H=70, ndir=1),
    "h256_bi": dict(T=20, B=17, H=256, ndir=2),
    "h1024_bi": dict(T=12, B=5, H=1024, ndir=2),
    "h1024_uni": dict(T=12, B=9, H=1024, ndir=1),        # KI = 32: U in registers
}


def _plan(knobs, lstm, parts):
    knobs("CTCB_LSTM", lstm)
    knobs("CTCB_LSTM_PARTS", str(parts) if parts else "auto")


@pytest.mark.parametrize("peep", [False, True])
@pytest.mark.parametrize("name", list(SWEEPS))
def test_sweep_on_every_plan_against_float64(name, peep, knobs, cuda):
    from _ctcb import lib
    c = SWEEPS[name]
    sw = Sweep(c["T"], c["B"], c["H"], c["ndir"], peep)
    out = {}
    ref_bits = {}
    for lstm, parts in PLANS:
        _plan(knobs, lstm, parts)
        plan = (ctypes.c_int32 * 4)()
        if lib.ctcb_debug_lstm_zoneout_plan(c["H"], c["B"], c["ndir"], int(peep), plan) != 0:
            continue
        for train in (True, False):
            zc, zh = 0.3, 0.2
            gates, h, cc, dz, err = sw.run(zc, zh, train)
            assert err == 0
            r = dict(gates=gates, h=h, c=cc, dz=dz)
            lc, lh = _lambdas(sw, zc, zh, train)
            fwd = _check_forward(r, _Problem(sw), lc, lh)
            e_dz = _check_bptt(r, _Problem(sw), lc, lh)
            key = "%s_%s_%s" % (lstm, parts, "train" if train else "expect")
            out[key] = dict(KI=int(plan[0]), parts=int(plan[1]), dz=e_dz, **fwd)
            for b, Tb in enumerate(sw.lens):
                assert not any(np.any(x[Tb:, b]) for x in [gates, dz] + h + cc), "a padded frame is not 0"
            assert fwd["kept"], out[key]
            assert fwd["gates"] <= C_FWD and fwd["c"] <= C_FWD and fwd["h"] <= C_FWD, out[key]
            assert fwd["act_exact"] <= C_ACT and e_dz <= C_BPTT, out[key]
            b = [x.view(np.uint32).tobytes() for x in [gates, dz] + h + cc]
            if train in ref_bits:
                assert b == ref_bits[train], "the bits depend on the plan: " + key
            else:
                ref_bits[train] = b
    print(json.dumps({"zoneout_sweep_%s_%s" % (name, "peep" if peep else "plain"): out}))
    assert len(ref_bits) == 2


@pytest.mark.parametrize("peep", [False, True])
@pytest.mark.parametrize("name", ["h64_bi", "h70_uni", "h1024_bi", "h1024_uni"])
def test_sweep_at_zero_probabilities_has_the_plain_sweeps_bytes(name, peep, knobs, cuda):
    c = SWEEPS[name]
    sw = Sweep(c["T"], c["B"], c["H"], c["ndir"], peep)
    _plan(knobs, "auto", None)
    want = sw.run(0.0, 0.0, True, plain=True)
    for train in (True, False):
        got = sw.run(0.0, 0.0, train)
        for a, b in zip(want[:4], got[:4]):
            for x, y in zip(a if isinstance(a, list) else [a], b if isinstance(b, list) else [b]):
                assert np.array_equal(x.view(np.uint32), y.view(np.uint32)), (name, peep, train)
        assert got[4] == 0


# ------------------------------------------------------------------------------------------------ the whole net
D, K = 23, 17
NETS = {
    "h64_bi_k1": dict(H=64, N=3, tl=2, k=1, T=30, B=6, L=8),
    "h70_uni_k2_ragged": dict(H=70, N=4, tl=2, k=2, T=25, B=5, L=6, uni=True, ragged=True),
    "h64_bi_k2_ragged_peep": dict(H=64, N=4, tl=2, k=2, T=20, B=7, L=6, ragged=True, peep=True),
    "h64_bi_k1_ln_drop": dict(H=64, N=4, tl=2, k=1, T=20, B=5, L=6, ragged=True, ln=True, p=0.3),
    "h128_bi_k1_sub_below": dict(H=128, N=3, tl=2, k=1, T=24, B=4, L=4, sub=(2, 1)),
    "h64_uni_k1_sub_above_peep": dict(H=64, N=3, tl=1, k=1, T=21, B=5, L=4, uni=True, ragged=True, sub=(3, 2),
                                      peep=True),
    "h1024_bi_k1": dict(H=1024, N=2, tl=1, k=1, T=10, B=3, L=4),
    "h1024_uni_k1": dict(H=1024, N=2, tl=1, k=1, T=10, B=3, L=4, uni=True),       # KI = 32
}
ZC, ZH = 0.25, 0.15


def _kwargs(c, reg=0.0, z=(ZC, ZH)):
    k, L = c.get("sub", (1, 1))
    return dict(temporalLayer=c["tl"], numTemporal=c["k"], reg=reg, unidirectional=bool(c.get("uni")), cell="lstm",
                peephole=bool(c.get("peep")), layerNorm=bool(c.get("ln")), dropout=c.get("p", 0.0), dropoutSeed=5,
                subsample=k, subsampleLayer=L, zoneoutCell=z[0], zoneoutHidden=z[1])


def _gpu_net(c, B, reg=0.0, train=True, z=(ZC, ZH)):
    import nnets.brnnet as brnnet
    return brnnet.NNet(D, K, c["H"], c["N"], c["T"], maxUtts=B, maxLabels=c["L"], train=train, **_kwargs(c, reg, z))


def _oracle(c, reg, z=(ZC, ZH)):
    return Net(D, K, c["H"], c["N"], c["T"], **_kwargs(c, reg, z))


def _batch(c, seed=5):
    T, B, L = c["T"], c["B"], c["L"]
    k = c.get("sub", (1, 1))[0]
    if c.get("ragged"):
        rng = np.random.RandomState(seed)
        lens = [int(x) for x in rng.randint(max(1, int(0.5 * T)), T + 1, size=B)]
        lens[0] = T
        nlabs = [min(int(x), -(-n // k)) for x, n in zip(rng.randint(1, L + 1, size=B), lens)]
    else:
        lens, nlabs = [T] * B, [min(L, -(-T // k))] * B
    return lens, recipes.synth_batch(D, K, lens, nlabs, seed=33)


def _set_p(nn, on, seed=8):
    import torch
    n = nn.peepholeEntries()
    rng = np.random.RandomState(seed)
    for (w, _), (ow, _) in zip(nn.stack[len(nn.stack) - n:], on.stack[len(on.stack) - n:]):
        x = rng.uniform(-0.5, 0.5, tuple(w.shape)).astype(np.float32)
        w.copy_(torch.from_numpy(x))
        ow[...] = x


@pytest.mark.parametrize("name", list(NETS))
def test_zoneout_net_matches_float64_oracle(name, cuda):
    """The device's training call against the float64 net with the same masks (and the same dropout masks)."""
    import torch
    c = NETS[name]
    lens, (datas, labelss) = _batch(c)
    B, H, N = c["B"], c["H"], c["N"]
    reg = 1e-3
    np.random.seed(21)
    nn = _gpu_net(c, B, reg=reg)
    nn.initParams()
    np.random.seed(21)
    on = _oracle(c, reg)
    on.initParams()
    if c.get("peep"):
        _set_p(nn, on)
    nn.dropoutStep.fill_(3)
    on.dropoutStep = 3
    nn.costAndGradBatch(datas, labelss)
    torch.cuda.synchronize()
    r = compare(nn, on, datas, labelss, lens)
    assert np.array_equal(r["skips"], r["skips_own"]) and not r["skips"].any()
    fwd = dict(logits=r["fwd"]["X"][N], gates=r["fwd"]["gates"], c=r["fwd"]["c"], h=r["fwd"]["h"])
    grad_err = r["grad_given"]
    print(json.dumps({"zoneout_net_" + name: dict(cost=r["cost_own"], fwd=fwd, grad_given_frob_max=max(grad_err),
                                                  grad_given_elem_max=max(r["grad_given_elem"]))}))
    assert r["cost_own"] <= 1e-4
    assert max(fwd.values()) <= 1e-4, fwd
    assert max(grad_err) <= 1e-4, grad_err


def _small(maxUtts, z=(ZC, ZH), uni=False, peep=False, reg=1e-2):
    import nnets.brnnet
    np.random.seed(4)
    nn = nnets.brnnet.NNet(13, 11, 64, 4, 60, temporalLayer=2, reg=reg, maxUtts=maxUtts, maxLabels=20, numTemporal=2,
                           unidirectional=uni, cell="lstm", peephole=peep, zoneoutCell=z[0], zoneoutHidden=z[1])
    nn.initParams()
    return nn


def _ragged(seed=7):
    lens = [50, 37, 12, 44, 29, 60, 21, 40]
    nlabs = [9, 14, 8, 11, 5, 20, 3, 7]
    return recipes.synth_batch(13, 11, lens, nlabs, seed=seed)


@pytest.mark.parametrize("uni", [False, True])
def test_micro_batches_and_two_shards_match_one_call(uni, cuda):
    """The masks follow the utterance's minibatch index and the step, so three micro-batches and two emulated shards
    draw the masks one call draws: the gradients agree to the reordering of the sums."""
    import _ctcb
    import parallel
    from _ctcb import lib, check, ptr
    datas, labelss = _ragged()
    full = _small(8, uni=uni)
    full.dropoutStep.fill_(4)
    c1, _, _ = full.costAndGradBatch(datas, labelss)
    g1 = full.grads_ext[:full.nparams + 4].cpu().numpy().astype(np.float64)
    split = _small(3, uni=uni)
    split.dropoutStep.fill_(4)
    c2, _, _ = split.costAndGradBatch(datas, labelss)
    g2 = split.grads_ext[:split.nparams + 4].cpu().numpy().astype(np.float64)
    total, last = None, None
    for rank in range(2):
        idx = parallel.shard(list(range(8)), rank, 2)
        nn = _small(4, uni=uni)
        nn.dropoutStep.fill_(4)
        nn.dropoutShard = (rank, 2)
        check(lib.ctcb_brnn_set_deferred_l2(nn._h, 1))
        nn.costAndGradBatch([datas[i] for i in idx], [labelss[i] for i in idx])
        part = nn.grads_ext[:nn.nparams + 4].clone()
        total = part if total is None else total + part
        last = nn
    check(lib.ctcb_brnn_apply_l2_f32(last._h, ptr(last.params), ptr(total), _ctcb.current_stream()))
    g3 = total.cpu().numpy().astype(np.float64)
    e_micro, e_shard = _rel(g2[:-4], g1[:-4]), _rel(g3[:-4], g1[:-4])
    print(json.dumps({"zoneout_accum_%s" % ("uni" if uni else "bi"): dict(micro=e_micro, shards=e_shard)}))
    assert np.allclose(c1, c2, rtol=1e-6)
    assert e_micro < 1e-5 and e_shard < 1e-5


def test_masks_follow_the_step(cuda):
    datas, labelss = _ragged()
    nn = _small(8)
    out = []
    for s in (4, 5, 4):
        nn.dropoutStep.fill_(s)
        c, _, _ = nn.costAndGradBatch(datas, labelss)
        out.append((c.copy(), nn.grads_ext.cpu().numpy().copy()))
    assert np.array_equal(out[0][1], out[2][1]) and np.array_equal(out[0][0], out[2][0])
    assert not np.array_equal(out[0][1], out[1][1])


def _train(useGraphs, steps=6, z=(ZC, ZH)):
    import random
    import sgd
    import torch
    lens, nlabs = [50, 37, 44, 29, 60, 21, 40, 33], [9, 14, 11, 5, 20, 3, 7, 8]
    datas, labelss = recipes.synth_batch(13, 11, lens, nlabs, seed=9)
    keys = ["k%d" % i for i in range(len(lens))]
    dd = dict(zip(keys, datas))
    alis = dict(zip(keys, [list(map(str, l)) for l in labelss]))
    nn = _small(8, z=z, peep=True, reg=1e-3)
    random.seed(33)
    opt = sgd.SGD(nn, 60, alpha=1e-3, momentum=0.9, maxGradNorm=5.0, batchSize=8, verbose=False)
    opt.useGraphs = useGraphs
    for _ in range(steps):
        opt.run(dd, alis, list(keys), None)
    torch.cuda.synchronize()
    return nn, np.array(opt.costt), opt


def test_graph_replay_is_bit_identical_to_eager_steps(cuda):
    nn_g, c_g, opt_g = _train(True)
    nn_e, c_e, opt_e = _train(False)
    print(json.dumps({"zoneout_graph": dict(graphs=len(opt_g._graphs), costs=c_g.tolist())}))
    assert len(opt_g._graphs) >= 1
    assert np.array_equal(nn_g.params.cpu().numpy(), nn_e.params.cpu().numpy()) and np.array_equal(c_g, c_e)
    assert int(nn_g.dropoutStep.item()) == 6


def test_zoneout_config_at_zero_is_bit_identical_to_no_zoneout(cuda):
    """A net whose config has zoneout = 1 but whose probabilities are set to 0 launches what a net without zoneout
    launches and computes the same bits."""
    from _ctcb import check, lib
    datas, labelss = _ragged()
    a = _small(8, z=(0.0, 0.0), peep=True)
    b = _small(8, peep=True)
    assert a._cfg.zoneout == 0 and b._cfg.zoneout == 1
    check(lib.ctcb_brnn_set_zoneout(b._h, 0.0, 0.0, 5, None))
    b.params.copy_(a.params)
    n0 = lib.ctcb_launch_count()
    ca, _, _ = a.costAndGradBatch(datas, labelss)
    n1 = lib.ctcb_launch_count()
    cb, _, _ = b.costAndGradBatch(datas, labelss)
    n2 = lib.ctcb_launch_count()
    assert n1 - n0 == n2 - n1
    assert np.array_equal(ca, cb) and np.array_equal(_bits(a.grads_ext), _bits(b.grads_ext))


def test_forward_only_probabilities_are_the_expectation(cuda):
    for name in ("h70_uni_k2_ragged", "h64_bi_k2_ragged_peep"):
        c = NETS[name]
        lens, (datas, labelss) = _batch(c)
        np.random.seed(3)
        inf = _gpu_net(c, c["B"], train=False)
        inf.initParams()
        on = _oracle(c, 0.0)
        np.random.seed(3)
        on.initParams()
        if c.get("peep"):
            _set_p(inf, on)
        on.expectation = True
        out = inf.forwardBatch(datas)
        err = 0.0
        for u, d in enumerate(datas):
            _, _, probs = on.forward(d)
            err = max(err, float(np.max(np.abs(out[u] - probs))))
        print(json.dumps({"zoneout_forward_only_" + name: dict(prob_abs_err=err)}))
        assert err <= 1e-5


def test_nnet_refusals(cuda):
    import nnets.brnnet as brnnet
    import nnets.rnnet as rnnet
    with pytest.raises(ValueError, match="cell='lstm'"):
        brnnet.NNet(13, 11, 64, 3, 20, temporalLayer=2, zoneoutCell=0.1)
    with pytest.raises(ValueError, match="cell='lstm'"):
        rnnet.NNet(13, 11, 64, 3, 20, temporalLayer=2, zoneoutHidden=0.1)
    for kw in (dict(zoneoutCell=1.0), dict(zoneoutHidden=-0.1), dict(zoneoutCell=float("nan"))):
        with pytest.raises(ValueError, match=r"\[0, 1\)"):
            brnnet.NNet(13, 11, 64, 3, 20, temporalLayer=2, cell="lstm", **kw)
    nn = brnnet.NNet(13, 11, 64, 3, 20, temporalLayer=2, cell="lstm", zoneoutCell=0.1)
    assert nn.dropoutStep is not None


def test_check_grad(cuda):
    import nnets.brnnet as brnnet
    datas, labelss = recipes.synth_batch(13, 11, [30], [6], seed=2)
    np.random.seed(5)
    nn = brnnet.NNet(13, 11, 16, 3, 30, temporalLayer=2, cell="lstm", maxLabels=6, zoneoutCell=0.3, zoneoutHidden=0.2)
    nn.initParams()
    nn.dropoutStep.fill_(2)
    out = np.array(nn.check_grad(datas[0], labelss[0], epsilon=1e-2, maxChecks=4, verbose=False))
    err = np.abs(out[:, 0] - out[:, 1]) / np.maximum(np.abs(out[:, 1]), 5e-2)
    print(json.dumps({"zoneout_check_grad": dict(probes=len(out), rel_err_max=float(err.max()))}))
    assert float(err.max()) < 0.1


@pytest.mark.parametrize("mode", ["main", "side"])
def test_forced_stalls_keep_every_byte(mode, knobs, cuda):
    datas, labelss = _ragged()
    want = _small(8, peep=True)
    want.dropoutStep.fill_(2)
    cw, _, _ = want.costAndGradBatch(datas, labelss)
    gw = _bits(want.grads_ext)
    knobs("CTCB_STALL", mode)
    knobs("CTCB_STALL_US", "500")
    got = _small(8, peep=True)
    got.dropoutStep.fill_(2)
    cg, _, _ = got.costAndGradBatch(datas, labelss)
    assert np.array_equal(cw, cg) and np.array_equal(gw, _bits(got.grads_ext))


# ------------------------------------------------------------------------------------------------ end to end
def test_run_nnet_trains_resumes_and_tests_with_the_trained_probabilities(cuda, tmp_path):
    import dataLoader as dl
    import runNNet
    from run_utils import dump_config, load_config
    data = str(tmp_path / "data") + "/"
    for fn in (1, 2):
        dl.write_synthetic_file(data, fn, num_utts=9, rawsize=20, outputDim=9, T_range=(10, 39), L_range=(3, 6))
    args = ["--layerSize", "64", "--numLayers", "3", "--temporalLayer", "2", "--cell", "lstm", "--zoneoutCell",
            "0.15", "--zoneoutHidden", "0.05", "--epochs", "1", "--step", "1e-3", "--dataDir", data, "--numFiles", "2",
            "--inputDim", "16", "--rawDim", "20", "--outputDim", "9", "--maxUttLen", "40", "--maxLabels", "6",
            "--batchSize", "4", "--save_every", "1", "--runDir", str(tmp_path / "runs"), "--quiet"]
    opt, net = runNNet.run(args)
    assert net.zoneoutCell == 0.15 and net.zoneoutHidden == 0.05
    run_dir = os.path.join(str(tmp_path / "runs"), os.listdir(str(tmp_path / "runs"))[0])
    cfg_file = os.path.join(run_dir, "cfg.json")
    cfg = load_config(cfg_file)
    assert cfg["zoneoutCell"] == 0.15 and cfg["zoneoutHidden"] == 0.05
    p_epoch0 = net.params.cpu().numpy().copy()
    step0 = int(net.dropoutStep.item())
    assert step0 > 0
    cfg["epochs"] = 2
    dump_config(cfg, cfg_file)
    _, net2 = runNNet.run(["--cfg_file", cfg_file, "--quiet"])
    # the run resumes behind its last checkpoint: the step counter comes back as it was saved
    assert net2.zoneoutCell == 0.15 and int(net2.dropoutStep.item()) == step0
    assert np.array_equal(p_epoch0, net2.params.cpu().numpy())
    out = str(tmp_path / "arks")
    tnet = runNNet.run(["--cfg_file", cfg_file, "--test", "--dataDir", data, "--numFiles", "2", "--outDir", out,
                        "--maxUtts", "4"])
    assert not tnet.train and tnet.zoneoutCell == 0.15 and tnet.zoneoutHidden == 0.05
    for fn in (1, 2):
        assert os.path.getsize(os.path.join(out, "loglikelihoods%d.ark" % fn)) > 9 * 16
    assert np.isfinite(p_epoch0).all()
