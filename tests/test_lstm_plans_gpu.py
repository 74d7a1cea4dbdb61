"""GPU unit test of the LSTM sweep (ctcb_lstm_sweep_f32, ctcb_lstm_sweep_peephole_f32) on every plan its planner can
choose, and of the peephole weight gradients (ctcb_lstm_peephole_grad_f32), against float64.

The planner (lstm_plan, csrc/sweep_lstm.cu) picks one of twelve instantiations lstm_sweep_kernel<KI, PEEP>: U in
registers (KI = H / 32) at H = 64, 128, 256, 512 and 1024 where ndir * H / 8 CTAs fit the device at that kernel's
occupancy, else U re-read (KI = 0); and it splits the batch's 8-utterance tiles over gridDim.y partitions.  Every case
runs in both modes (plain, and peephole with P ~ U(-0.5, 0.5)), names the KI it targets, and checks the plan
ctcb_debug_lstm_plan reports for the kernel of that mode before launching: KI, partitions, CTAs per SM and tiles per
partition, against the plan that follows from the kernels' register counts and this device's SM count.  CTCB_LSTM=reread
and CTCB_LSTM_PARTS are set in process (recipes.knobs) and restored afterwards.

Forward: every output x (gates, c, h) satisfies |x - x64| <= C_FWD u S, u = 2^-24, x64 the float64 of the step computed
from the GPU's own state of the step before and S the sum of the magnitudes of the terms that make x (1 + |pre| +
|U| |h_prev| (+ |p| |c|) for a gate, |f c_prev| + |i g| for c, |o| for h); and where z is exact (h_prev = 0) the
activation alone, |a - a64| <= C_ACT u |a64|, which is what sees a less accurate exp or tanh at large |z|.  BPTT: dz
against the float64 BPTT of the GPU's own forward activations (net_oracle), |dz - dz64| <= C_BPTT u S
with S = max |dz64| of that utterance and direction, no floor: the bound is scale-free, and exact linearity in dh
(below) is what makes that sound.  Exact: padded frames 0 (outputs start as NaN), NaN guard bands around gates, h, c,
dz and the scratch unchanged, the error flag 0, a rerun gives the same bytes, dh 2^-20 gives dz 2^-20 where no dz
comes within 2^-60 of the subnormals (saturated recipes do), and the bits do not depend on the plan: KI, the
re-read path and every partition count give the same bytes, and each direction of a bi-directional launch equals a
uni-directional launch on that direction's U and pre-activations (direction 1: each utterance reversed within its own
length).  Each case prints its plan and ratios as one JSON line (pytest -s)."""
import ctypes
import json

import numpy as np
import pytest

import net_oracle
from recipes import knobs  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu
U32 = 2.0 ** -24
# Largest ratios measured on an H100 80GB HBM3 at 700 W over the cases of this file (DESIGN.md section 4): gates, c, h
# 2.2 (C_FWD as before), activations at exact pre-activations 3.3 and dz 3.95 (C_ACT, C_BPTT: 4x), dz with no growth
# in T from 1 to 1000 steps, so its bound is one constant.
C_FWD, C_ACT, C_BPTT = 8.0, 13.0, 16.0
TINY = 2.0 ** -60           # dz 2^-20 and its products with weights down to 2^-40 stay normal above this
SCALE = np.float32(2.0 ** -20)
GUARD = 64                  # NaN floats on each side of every buffer; 256 bytes keep the buffers' 16-byte alignment
NAN_BITS = np.float32(np.nan).view(np.uint32)
MODES = ("plain", "peep")
REG_H = (64, 128, 256, 512, 1024)
# CTAs of 256 threads per SM, from the registers ptxas reports for lstm_sweep_kernel<KI, PEEP> (plain / peephole):
# KI=0 128 / 124, KI=2 101 / 103, KI=4 119 / 127 -> two per SM; KI=8 142 / 148, KI=16 177 / 167, KI=32 247 / 238 -> one.
PER_SM = {0: 2, 2: 2, 4: 2, 8: 1, 16: 1, 32: 1}


# ------------------------------------------------------------------------------------------------ plans
def _sms(torch):
    return torch.cuda.get_device_properties(0).multi_processor_count


def _expect(H, B, ndir, sms, reread=False, parts=None):
    """The plan lstm_plan makes on a device of `sms` SMs, or None where it refuses."""
    slices = -(-H // 8)
    ki = H // 32 if H in REG_H and not reread else 0
    if ndir * slices > PER_SM[ki] * sms:
        ki = 0
    cap = PER_SM[ki] * sms
    if ndir * slices > cap:
        return None
    ntiles = -(-B // 8)
    p = cap // (ndir * slices)
    if parts:
        if parts > p:
            return None
        p = parts
    p = max(1, min(p, ntiles, 500))
    return dict(KI=ki, parts=p, per_sm=PER_SM[ki], tiles=-(-ntiles // p))


def _plan(H, B, ndir, peep):
    """(rc, plan) of ctcb_debug_lstm_plan for the kernel of that mode under the knobs in effect."""
    from _ctcb import lib
    out = (ctypes.c_int32 * 4)()
    rc = lib.ctcb_debug_lstm_plan(H, B, ndir, int(peep), out)
    return rc, (dict(KI=out[0], parts=out[1], per_sm=out[2], tiles=out[3]) if rc == 0 else None)


# what the cases ran: (KI, peep) instantiations, and per mode the partition edges
SEEN = dict(inst=set(), empty=set(), multi=set(), cases=0)


def _note(plan, B, peep):
    ntiles = -(-B // 8)
    tpp, parts = plan["tiles"], plan["parts"]
    SEEN["inst"].add((plan["KI"], peep))
    if tpp * (parts - 1) >= ntiles:
        SEEN["empty"].add(peep)
    last = (ntiles - 1) // tpp                  # the partition that holds the last tile
    if B % 8 and min(ntiles, (last + 1) * tpp) - last * tpp >= 2:
        SEEN["multi"].add(peep)


# ------------------------------------------------------------------------------------------------ one sweep
def _buf(torch, a):
    """A device copy of float32 array a inside NaN guard bands: (whole buffer, view of a)."""
    whole = torch.full((a.size + 2 * GUARD,), float("nan"), device="cuda")
    whole[GUARD:GUARD + a.size] = torch.from_numpy(np.ascontiguousarray(a, np.float32).ravel()).cuda()
    return whole, whole[GUARD:GUARD + a.size].view(a.shape)


def _guards_intact(whole):
    bits = whole.cpu().numpy().view(np.uint32)
    return (bits[:GUARD] == NAN_BITS).all() and (bits[-GUARD:] == NAN_BITS).all()


class Sweep:
    """Device buffers of one sweep problem; run() does the forward and the BPTT and returns the outputs (numpy)."""

    def __init__(self, torch, H, lens, pre, Us, Ps, dh):
        self.torch, self.H, self.lens = torch, H, np.asarray(lens, np.int32)
        self.T, self.B = pre.shape[:2]
        self.ndir = len(Us)
        self.pre, self.Us, self.Ps, self.dh = pre, Us, Ps, dh
        self.d_U = [torch.from_numpy(u).cuda() for u in Us]
        self.d_P = [torch.from_numpy(p).cuda() for p in Ps] if Ps is not None else None
        self.d_len = torch.from_numpy(self.lens).cuda()

    def run(self, dh=None, fwd=None):
        """Forward then BPTT on fresh buffers (fwd: a previous run whose forward activations the BPTT reads instead)."""
        from _ctcb import lib, check
        torch, H, T, B, nd = self.torch, self.H, self.T, self.B, self.ndir
        st = torch.cuda.current_stream().cuda_stream
        ws = int(lib.ctcb_lstm_sweep_workspace_bytes(H, B))
        # scratch: error flag and counters 0, the dc carry NaN (it must be written before it is read), NaN bytes behind
        scratch = torch.full((ws + 4 * GUARD,), 255, dtype=torch.uint8, device="cuda")
        scratch[:4096] = 0
        if fwd is None:
            g_all, gates = _buf(torch, self.pre)
            hw = [_buf(torch, np.full((T, B, H), np.nan, np.float32)) for _ in range(nd)]
            cw = [_buf(torch, np.full((T, B, H), np.nan, np.float32)) for _ in range(nd)]
        else:
            g_all, gates = _buf(torch, fwd["gates"])
            hw = [_buf(torch, x) for x in fwd["h"]]
            cw = [_buf(torch, x) for x in fwd["c"]]
        dz_all, dz = _buf(torch, np.full((T, B, nd * 4 * H), np.nan, np.float32))
        _, d_dh = _buf(torch, self.dh if dh is None else dh)
        p = lambda t: None if t is None else t.data_ptr()          # noqa: E731
        U, h, c = self.d_U, [x[1] for x in hw], [x[1] for x in cw]
        Ub, hB, cB = (U[1], h[1], c[1]) if nd == 2 else (None, None, None)

        def call(mode, hF, hB_, dh_, dz_):
            if self.d_P is None:
                return lib.ctcb_lstm_sweep_f32(mode, T, B, H, p(self.d_len), p(gates), p(U[0]), p(Ub), p(hF), p(hB_),
                                               p(c[0]), p(cB), p(dh_), p(dz_), p(scratch), ws, st)
            Pb = self.d_P[1] if nd == 2 else None
            return lib.ctcb_lstm_sweep_peephole_f32(mode, T, B, H, p(self.d_len), p(gates), p(U[0]), p(Ub),
                                                    p(self.d_P[0]), p(Pb), p(hF), p(hB_), p(c[0]), p(cB), p(dh_),
                                                    p(dz_), p(scratch), ws, st)
        if fwd is None:
            check(call(0, h[0], hB, None, None))
            torch.cuda.synchronize()
            err_fwd = int(scratch[:4].view(torch.int32).item())
        else:
            err_fwd = 0
        check(call(1, None, None, d_dh, dz))
        torch.cuda.synchronize()
        err = int(scratch[:4].view(torch.int32).item())
        tail = scratch[ws:].cpu().numpy()
        guards = all(_guards_intact(w) for w in [g_all, dz_all] + [x[0] for x in hw] + [x[0] for x in cw])
        return dict(gates=gates.cpu().numpy(), h=[x.cpu().numpy() for x in h], c=[x.cpu().numpy() for x in c],
                    dz=dz.cpu().numpy(), err=(err_fwd, err), guards=bool(guards and (tail == 255).all()))


def _same(a, b):
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def _same_run(r, s):
    return all(_same(r[k], s[k]) for k in ("gates", "dz")) and \
        all(_same(x, y) for k in ("h", "c") for x, y in zip(r[k], s[k]))


# ------------------------------------------------------------------------------------------------ float64
def _sig(z):
    return 1.0 / (1.0 + np.exp(-z))


def _check_forward(r, sw, lc=None, lh=None):
    """Largest |x - x64| / (u S) of the gates, c and h over the live frames, the step vectorised over the batch; and
    where z is exact (h_prev = 0: z = pre, plus p c_prev = 0 for i and f) the activation alone, |a - a64| / (u |a64|).
    Zoneout: lc, lh are per direction [T][B][H] lambdas (0 by default), c64 = lc c_prev + (1 - lc)(f c_prev + i g) with
    |lc c_prev| in S, h64 likewise; "kept" says whether every c and h with lambda = 1 has the bytes of the one before."""
    H, T, nd = sw.H, sw.T, sw.ndir
    live = np.arange(T)[:, None] < sw.lens[None, :]
    ratio = dict(gates=0.0, c=0.0, h=0.0, act_exact=0.0)
    if lc is not None:
        ratio["kept"] = True
    exact_rows = slice(0, 3 * H) if sw.Ps is not None else slice(0, 4 * H)     # peephole o: z_o + p_o c_t rounds
    for d in range(nd):
        blk = slice(d * 4 * H, (d + 1) * 4 * H)
        g, c, h = r["gates"][:, :, blk].astype(np.float64), r["c"][d].astype(np.float64), r["h"][d].astype(np.float64)
        pz = sw.pre[:, :, blk].astype(np.float64)
        U = sw.Us[d].astype(np.float64)
        Ut, aUt = U.T.copy(), np.abs(U).T.copy()
        P = sw.Ps[d].astype(np.float64) if sw.Ps is not None else np.zeros((3, H))
        hp, cp = np.zeros_like(h), np.zeros_like(c)           # the GPU's own state of the step before (0 outside)
        if d == 0:
            hp[1:], cp[1:] = h[:-1], c[:-1]
        else:
            hp[:-1], cp[:-1] = h[1:], c[1:]
        for t in range(T):
            m = live[t]
            if not m.any():
                continue
            z = pz[t, m] + hp[t, m].dot(Ut)
            S = 1.0 + np.abs(pz[t, m]) + np.abs(hp[t, m]).dot(aUt)
            ct, cpt = c[t, m], cp[t, m]
            peep = np.concatenate([P[0] * cpt, P[1] * cpt, np.zeros_like(cpt), P[2] * ct], axis=1)
            z = z + peep
            S = S + np.abs(peep)
            a64 = np.concatenate([_sig(z[:, :2 * H]), np.tanh(z[:, 2 * H:3 * H]), _sig(z[:, 3 * H:])], axis=1)
            gt = g[t, m]
            ratio["gates"] = max(ratio["gates"], float(np.max(np.abs(gt - a64) / (U32 * S))))
            ex = ~np.any(hp[t, m], axis=1)
            if ex.any():
                a, b = gt[ex, exact_rows], a64[ex, exact_rows]
                ratio["act_exact"] = max(ratio["act_exact"], float(np.max(np.abs(a - b) / (U32 * np.abs(b) + 1e-300))))
            i_, f_, g_, o_ = gt[:, :H], gt[:, H:2 * H], gt[:, 2 * H:3 * H], gt[:, 3 * H:]
            lct = np.zeros_like(ct) if lc is None else np.asarray(lc[d][t, m], np.float64)
            lht = np.zeros_like(ct) if lh is None else np.asarray(lh[d][t, m], np.float64)
            c64 = lct * cpt + (1.0 - lct) * (f_ * cpt + i_ * g_)
            Sc = np.abs(lct * cpt) + np.abs(f_ * cpt) + np.abs(i_ * g_) + 1e-30
            ratio["c"] = max(ratio["c"], float(np.max(np.abs(ct - c64) / (U32 * Sc))))
            h64 = lht * hp[t, m] + (1.0 - lht) * o_ * np.tanh(ct)
            Sh = np.abs(lht * hp[t, m]) + np.abs(o_) + 1e-30
            ratio["h"] = max(ratio["h"], float(np.max(np.abs(h[t, m] - h64) / (U32 * Sh))))
            src = t - 1 if d == 0 else t + 1
            if lc is not None and 0 <= src < T:
                for lam, x in ((lct, r["c"][d]), (lht, r["h"][d])):
                    k = lam == 1.0
                    ratio["kept"] &= bool(np.array_equal(x[t, m][k].view(np.uint32), x[src, m][k].view(np.uint32)))
    return ratio


def _check_bptt(r, sw, lc=None, lh=None):
    """Largest |dz - dz64| / (u max |dz64|) per (utterance, direction), dz64 the float64 BPTT of the GPU's own forward
    activations (through the zoneout lambdas lc, lh of _check_forward, 0 by default)."""
    H, nd = sw.H, sw.ndir
    Us = [u.astype(np.float64) for u in sw.Us]
    worst = 0.0
    for u in range(sw.B):
        Tu = int(sw.lens[u])
        dh = sw.dh[:Tu, u].T.astype(np.float64)
        for d in range(nd):
            blk = slice(d * 4 * H, (d + 1) * 4 * H)
            g = r["gates"][:Tu, u, blk].T.astype(np.float64)
            c, h = r["c"][d][:Tu, u].T.astype(np.float64), r["h"][d][:Tu, u].T.astype(np.float64)
            P = np.zeros((3, H)) if sw.Ps is None else sw.Ps[d].astype(np.float64)
            zero = np.zeros((H, Tu))
            lam = [zero if x is None else np.asarray(x[d][:Tu, u], np.float64).T for x in (lc, lh)]
            dz64 = net_oracle.lstm_direction_bptt(dh, g, c, h, Us[d], d == 1, P, *lam)[0]
            S = float(np.max(np.abs(dz64)))
            assert S > 0.0, "utterance %d direction %d has no gradient to compare" % (u, d)
            worst = max(worst, float(np.max(np.abs(r["dz"][:Tu, u, blk].T - dz64))) / (U32 * S))
    return worst


def _check_exact(r, sw):
    """Padded frames exactly 0, guard bands intact, error flag 0."""
    H, nd = sw.H, sw.ndir
    assert r["err"] == (0, 0), "error flag set: %s" % (r["err"],)
    assert r["guards"], "a guard band changed: the sweep wrote outside its arrays"
    for u in range(sw.B):
        Tu = int(sw.lens[u])
        for arr in [r["gates"][Tu:, u], r["dz"][Tu:, u]] + [x[Tu:, u] for x in r["h"] + r["c"]]:
            assert not np.any(arr), "padded frame of utterance %d not 0" % u
    for k in ("gates", "dz"):
        assert np.isfinite(r[k]).all(), k
    for x in r["h"] + r["c"]:
        assert np.isfinite(x).all()


# ------------------------------------------------------------------------------------------------ inputs
def _problem(torch, H, ndir, B, T, peep, seed, lens="ragged", mag="normal", dh="randn"):
    rng = np.random.RandomState(seed)
    G = ndir * 4 * H
    if lens == "ragged":
        L = rng.randint(1, T + 1, size=B)
        L[0] = T
    elif lens == "full":
        L = np.full(B, T)
    elif lens == "short":                       # the longest utterance is shorter than T
        L = rng.randint(1, max(2, T - 2), size=B)
    elif lens == "ones":                        # every other utterance one frame long
        L = rng.randint(1, T + 1, size=B)
        L[::2] = 1
        L[1] = T
    L = np.asarray(L, np.int32)
    s = 1.5 / np.sqrt(H)
    if mag == "normal":
        pre = rng.uniform(-1.5, 1.5, (T, B, G))
    elif mag == "saturate":                     # pre-activations up to +-30: the gates saturate
        pre = rng.uniform(-30.0, 30.0, (T, B, G))
    elif mag == "memory":                       # forget +8, input and candidate near 1: c grows about 1 per step
        pre = rng.uniform(-0.5, 0.5, (T, B, G))
        for d in range(ndir):
            pre[:, :, d * 4 * H:d * 4 * H + 3 * H] += 8.0
        s = 0.3 / np.sqrt(H)
    pre = pre.astype(np.float32)
    Us = [rng.uniform(-s, s, (4 * H, H)).astype(np.float32) for _ in range(ndir)]
    Ps = [rng.uniform(-0.5, 0.5, (3, H)).astype(np.float32) for _ in range(ndir)] if peep else None
    d = rng.randn(T, B, H).astype(np.float32)
    if dh == "last":                            # dh only at the last frame of each direction's forward order
        keep = np.zeros((T, B), bool)
        keep[L - 1, np.arange(B)] = True
        if ndir == 2:
            keep[0, :] = True
        d = d * keep[:, :, None]
    return Sweep(torch, H, L, pre, Us, Ps, d.astype(np.float32))


# ------------------------------------------------------------------------------------------------ the cases
def case(name, H, ndir, B, T, ki, lens="ragged", mag="normal", dh="randn", reread=False, parts=None):
    return dict(name=name, H=H, ndir=ndir, B=B, T=T, ki=ki, lens=lens, mag=mag, dh=dh, reread=reread, parts=parts)


CASES = []
for _H in REG_H:                                          # every width with U in registers, and re-read at that width
    for _nd in (1, 2):
        _ki = 0 if (_H == 1024 and _nd == 2) else _H // 32     # 256 CTAs do not fit one per SM on 132 SMs
        CASES.append(case("h%d_%s" % (_H, "bi" if _nd == 2 else "uni"), _H, _nd, 13, 9, _ki))
        CASES.append(case("h%d_%s_reread" % (_H, "bi" if _nd == 2 else "uni"), _H, _nd, 13, 9, 0, reread=True))
for _H in (8, 33, 70, 1000):                              # j < H warps, H % 4 != 0 state loads, < 32 lanes with work
    for _nd in (1, 2):
        CASES.append(case("h%d_%s" % (_H, "bi" if _nd == 2 else "uni"), _H, _nd, 11, 7, 0))
CASES += [
    case("b1", 256, 2, 1, 6, 8),
    case("b_1mod8", 128, 1, 33, 7, 4),
    case("multi_tile_partial", 512, 2, 125, 5, 16),      # 1 partition, 16 tiles, the last of 5 utterances
    case("empty_partition", 256, 1, 40, 6, 8),            # 4 partitions, 5 tiles: 2, 2, 1, 0
    case("forced_parts_4_empty", 64, 2, 37, 6, 2, parts=4),   # 5 tiles: 2, 2, 1, 0
    case("forced_parts_3_empty", 70, 1, 29, 5, 0, parts=3),   # 4 tiles: 2, 2 (the last of 5 utterances), 0
    case("all_padded_first_steps", 128, 2, 19, 10, 4, lens="short"),
    case("t_u_1", 64, 2, 10, 8, 2, lens="ones"),
    case("t1", 512, 1, 9, 1, 16, lens="full"),
    case("t1_bi", 70, 2, 9, 1, 0, lens="full"),
    case("long_c2", 512, 2, 32, 300, 16),
    case("long_1000", 128, 1, 6, 1000, 4),
    case("saturate", 256, 2, 12, 12, 8, mag="saturate"),
    case("saturate_h64_uni", 64, 1, 12, 4, 2, mag="saturate"),      # activations over +-30 at every KI
    case("saturate_h128_uni", 128, 1, 12, 4, 4, mag="saturate"),
    case("saturate_h512_uni", 512, 1, 12, 4, 16, mag="saturate"),
    case("saturate_h1024_uni", 1024, 1, 12, 4, 32, mag="saturate"),
    case("saturate_h1024_bi", 1024, 2, 12, 4, 0, mag="saturate"),
    case("memory", 64, 1, 9, 120, 2, mag="memory", lens="full"),
    case("memory_bi_reread", 128, 2, 9, 60, 0, mag="memory", reread=True),
    case("dh_last_only", 512, 1, 10, 40, 16, dh="last"),
    case("dh_last_only_bi", 64, 2, 10, 40, 2, dh="last"),
]
CASE_IDS = [c["name"] for c in CASES]


def _set(knobs, reread=False, parts=None):
    knobs("CTCB_LSTM", "reread" if reread else "auto")
    knobs("CTCB_LSTM_PARTS", str(parts) if parts else "auto")


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", CASE_IDS)
def test_lstm_sweep_plan(name, mode, knobs, cuda):
    torch = cuda
    c = next(x for x in CASES if x["name"] == name)
    peep = mode == "peep"
    H, nd, B, T = c["H"], c["ndir"], c["B"], c["T"]
    _set(knobs, c["reread"], c["parts"])
    want = _expect(H, B, nd, _sms(torch), c["reread"], c["parts"])
    rc, plan = _plan(H, B, nd, peep)
    assert rc == 0 and plan == want, (plan, want)
    if _sms(torch) == 132:
        assert plan["KI"] == c["ki"], "case %s targets KI=%d, planned %s" % (name, c["ki"], plan)
    _note(plan, B, peep)
    SEEN["cases"] += 1
    sw = _problem(torch, H, nd, B, T, peep, seed=H + 7 * B + T + (1 if peep else 0), lens=c["lens"], mag=c["mag"],
                  dh=c["dh"])
    r = sw.run()
    _check_exact(r, sw)
    again = sw.run()
    assert _same_run(r, again), "a rerun gave other bytes"
    # dh 2^-20 gives dz 2^-20 exactly where nothing reaches the subnormals: saturated gates (pre-activations at +-30,
    # peephole gates driven by a large c) make products of three small derivatives that do
    nz = np.abs(r["dz"][r["dz"] != 0])
    dz_min = float(nz.min()) if nz.size else 0.0
    linear = dz_min >= TINY
    if linear:
        scaled = sw.run(dh=sw.dh * SCALE, fwd=r)
        assert _same(scaled["dz"], r["dz"] * SCALE), "dz is not exactly linear in dh"
    fwd = _check_forward(r, sw)
    dz = _check_bptt(r, sw)
    cmax = float(np.max([np.abs(x[:Tu, u]).max() for x in r["c"] for u, Tu in enumerate(sw.lens)]))
    print(json.dumps({"lstm_plan_%s_%s" % (name, mode): dict(plan, H=H, ndir=nd, B=B, T=T, peephole=peep, c_max=cmax,
                                                              dz_min=dz_min, linearity_checked=linear, dz=dz,
                                                              **fwd)}))
    assert fwd["gates"] <= C_FWD and fwd["c"] <= C_FWD and fwd["h"] <= C_FWD, fwd
    assert fwd["act_exact"] <= C_ACT, fwd
    assert dz <= C_BPTT, dz


# ------------------------------------------------------------------------------------------------ plan independence
def _uni_of_direction(sw, d):
    """The uni-directional problem that direction d of bi-directional problem sw is: U_d, the pre-activations of d's
    gate block and dh, for d = 1 each utterance reversed within its own length."""
    H, T, B = sw.H, sw.T, sw.B
    pre = sw.pre[:, :, d * 4 * H:(d + 1) * 4 * H].copy()
    dh = sw.dh.copy()
    if d == 1:
        for u in range(B):
            Tu = int(sw.lens[u])
            pre[:Tu, u] = pre[:Tu, u][::-1]
            dh[:Tu, u] = dh[:Tu, u][::-1]
    Ps = None if sw.Ps is None else [sw.Ps[d]]
    return Sweep(sw.torch, H, sw.lens, pre, [sw.Us[d]], Ps, dh)


def _reverse(x, lens):
    y = x.copy()
    for u, Tu in enumerate(lens):
        y[:Tu, u] = x[:Tu, u][::-1]
    return y


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("ndir", [1, 2])
@pytest.mark.parametrize("H", [64, 70, 128, 256, 512, 1024])
def test_lstm_bits_do_not_depend_on_the_plan(H, ndir, mode, knobs, cuda):
    """The register path and the re-read path accumulate in the same lane order (k = lane + 32 i) and partitions
    change no arithmetic: the bytes of every plan at one H are those of the automatic plan.  Each direction of a
    bi-directional launch is a uni-directional launch of its own."""
    torch = cuda
    peep = mode == "peep"
    B, T = 37, 7                                           # 5 tiles: forced 4 partitions leave the last one empty
    sw = _problem(torch, H, ndir, B, T, peep, seed=3 * H + ndir)
    sms = _sms(torch)
    _set(knobs)
    _, auto = _plan(H, B, ndir, peep)
    ref = sw.run()
    _check_exact(ref, sw)
    _note(auto, B, peep)
    _, wide = _plan(H, 8 * 500, ndir, peep)                 # the partitions the device holds at this KI
    cap = wide["parts"]
    runs = {"auto": auto}
    for label, reread, parts in [("reread", True, None)] + [("parts%d" % p, False, p)
                                                             for p in sorted({1, 2, 3, 4, cap}) if p <= cap]:
        _set(knobs, reread, parts)
        rc, plan = _plan(H, B, ndir, peep)
        assert rc == 0 and plan == _expect(H, B, ndir, sms, reread, parts), (label, plan)
        r = sw.run()
        _check_exact(r, sw)
        _note(plan, B, peep)
        runs[label] = plan
        assert _same_run(r, ref), "%s gave other bytes than the automatic plan %s" % (label, auto)
    if ndir == 2:
        _set(knobs)
        for d in range(2):
            usw = _uni_of_direction(sw, d)
            u = usw.run()
            _check_exact(u, usw)
            blk = slice(d * 4 * H, (d + 1) * 4 * H)
            got = dict(gates=ref["gates"][:, :, blk], dz=ref["dz"][:, :, blk], h=ref["h"][d], c=ref["c"][d])
            if d == 1:
                got = {k: _reverse(v, sw.lens) for k, v in got.items()}
            for k in ("gates", "dz"):
                assert _same(np.ascontiguousarray(got[k]), u[k]), "direction %d %s differs from a uni launch" % (d, k)
            for k in ("h", "c"):
                assert _same(got[k], u[k][0]), "direction %d %s differs from a uni launch" % (d, k)
    print(json.dumps({"lstm_bits_H%d_%s_%s" % (H, "bi" if ndir == 2 else "uni", mode): runs}))


# ------------------------------------------------------------------------------------------------ refusals
def _refused_without_launch(torch, H, B, ndir, peep):
    """The sweep call at (H, B, ndir) returns CTCB_EINVAL and launches nothing; returns the message."""
    from _ctcb import lib
    T = 1
    sw = _problem(torch, H, ndir, B, T, peep, seed=1, lens="full")
    ws = int(lib.ctcb_lstm_sweep_workspace_bytes(H, B))
    scratch = torch.zeros(ws, dtype=torch.uint8, device="cuda")
    gates = torch.from_numpy(sw.pre).cuda()
    h = [torch.zeros(T, B, H, device="cuda") for _ in range(ndir)]
    c = [torch.zeros(T, B, H, device="cuda") for _ in range(ndir)]
    p = lambda t: None if t is None else t.data_ptr()      # noqa: E731
    Ub, hB, cB = (sw.d_U[1], h[1], c[1]) if ndir == 2 else (None, None, None)
    st = torch.cuda.current_stream().cuda_stream
    n0 = lib.ctcb_launch_count()
    if peep:
        Pb = sw.d_P[1] if ndir == 2 else None
        rc = lib.ctcb_lstm_sweep_peephole_f32(0, T, B, H, p(sw.d_len), p(gates), p(sw.d_U[0]), p(Ub), p(sw.d_P[0]),
                                              p(Pb), p(h[0]), p(hB), p(c[0]), p(cB), None, None, p(scratch), ws, st)
    else:
        rc = lib.ctcb_lstm_sweep_f32(0, T, B, H, p(sw.d_len), p(gates), p(sw.d_U[0]), p(Ub), p(h[0]), p(hB), p(c[0]),
                                     p(cB), None, None, p(scratch), ws, st)
    msg = lib.ctcb_last_error().decode()
    torch.cuda.synchronize()
    assert rc == -1 and lib.ctcb_launch_count() == n0, (rc, msg)
    return msg


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("ndir", [1, 2])
def test_the_widest_layer_the_device_holds_runs_and_the_next_is_refused(ndir, mode, knobs, cuda):
    """The widest H the device holds co-resident (re-read U, CTAs per SM x SMs CTAs of 8 units over ndir directions)
    runs and matches float64; one more unit needs one more slice and is refused by the sweep and by ctcb_brnn_create,
    without a launch."""
    import _ctcb
    from _ctcb import lib
    torch = cuda
    peep = mode == "peep"
    _set(knobs)
    _, small = _plan(70, 8, ndir, peep)
    Hmax = 8 * (small["per_sm"] * _sms(torch) // ndir)
    B, T = 3, 3
    rc, plan = _plan(Hmax, B, ndir, peep)
    assert rc == 0 and plan == dict(KI=0, parts=1, per_sm=small["per_sm"], tiles=1), plan
    sw = _problem(torch, Hmax, ndir, B, T, peep, seed=11)
    r = sw.run()
    _check_exact(r, sw)
    fwd, dz = _check_forward(r, sw), _check_bptt(r, sw)
    assert _plan(Hmax + 1, B, ndir, peep)[0] == -1
    msg = _refused_without_launch(torch, Hmax + 1, B, ndir, peep)
    assert "layerSize %d" % (Hmax + 1) in msg and "co-resident" in msg, msg
    cfg = _ctcb.BrnnConfig(41, 32, Hmax + 1, 3, 2, 50, B, 10, 0.0, 20.0, int(ndir == 1), 1, 1, peephole=int(peep))
    h = ctypes.c_void_p()
    assert lib.ctcb_brnn_create(ctypes.byref(cfg), ctypes.byref(h)) == -1
    assert "layerSize %d" % (Hmax + 1) in lib.ctcb_last_error().decode()
    print(json.dumps({"lstm_widest_%s_%s" % ("bi" if ndir == 2 else "uni", mode):
                      dict(plan, H=Hmax, refused=msg, dz=dz, **fwd)}))
    assert fwd["gates"] <= C_FWD and fwd["c"] <= C_FWD and fwd["h"] <= C_FWD and fwd["act_exact"] <= C_ACT, fwd
    assert dz <= C_BPTT, dz


@pytest.mark.parametrize("mode", MODES)
def test_a_partition_count_the_device_cannot_hold_is_refused(mode, knobs, cuda):
    """CTCB_LSTM_PARTS above the capacity of the plan's kernel is refused before any launch, never a cooperative launch
    that cannot be co-resident; at the capacity it runs."""
    torch = cuda
    peep = mode == "peep"
    for H, ndir in ((1024, 2), (512, 2), (256, 1)):
        _set(knobs)
        _, wide = _plan(H, 8 * 500, ndir, peep)
        cap = wide["parts"]
        knobs("CTCB_LSTM_PARTS", str(cap + 1))
        assert _plan(H, 8 * 500, ndir, peep)[0] == -1
        msg = _refused_without_launch(torch, H, 8 * (cap + 1), ndir, peep)
        assert "CTCB_LSTM_PARTS=%d" % (cap + 1) in msg, msg
        knobs("CTCB_LSTM_PARTS", str(cap))
        assert _plan(H, 8 * (cap + 1), ndir, peep)[1]["parts"] == cap


def test_every_instantiation_and_partition_edge_was_reached(cuda):
    """The cases above reached all twelve lstm_sweep_kernel<KI, PEEP>, and in each mode a partition without a tile and
    a partition of several tiles whose last tile is partial."""
    if SEEN["cases"] < 2 * len(CASES):
        pytest.skip("run with the whole module: %d of %d cases ran" % (SEEN["cases"], 2 * len(CASES)))
    want = {(ki, peep) for ki in (0, 2, 4, 8, 16, 32) for peep in (False, True)}
    print(json.dumps({"lstm_plans_reached": dict(inst=sorted(SEEN["inst"]), empty=sorted(SEEN["empty"]),
                                                 multi=sorted(SEEN["multi"]))}))
    assert SEEN["inst"] == want, want - SEEN["inst"]
    assert SEEN["empty"] == {False, True} and SEEN["multi"] == {False, True}, SEEN


# ------------------------------------------------------------------------------------------------ dP alone
@pytest.mark.parametrize("T,B,H,ndir", [(1, 3, 64, 2), (9, 13, 70, 1), (37, 5, 512, 2), (300, 8, 1024, 2),
                                        (9, 7, 70, 2), (32, 32, 70, 2), (41, 25, 33, 2), (2, 4, 70, 2),
                                        (8, 1, 64, 1)])
def test_peephole_grad_matches_float64(T, B, H, ndir, cuda):
    """dP against float64 of the same float32 dz and c.  Each output is a sum of n = T B products, each product exact
    to u in float32 and the sum of fixed chunks of 1024 rows (8 interleaved partial sums of 128 products each, combined
    in a tree of 8, then the chunks in order): a recursive sum of m terms errs by at most (m - 1) u sum |terms|, so the
    bound is (128 + 8 + ceil(n / 1024) + 1) u sum |dz c'|.  Bi-directional H = 70 has a 32-column block across the
    direction boundary q = 3H; n = 1024 and 1025 end a chunk exactly and one row after.  A rerun is bit-identical,
    accumulate adds to what dP held (rounded once), 2^-20 dz gives 2^-20 dP, and nothing outside dP is written."""
    torch = cuda
    from _ctcb import lib, check
    rng = np.random.RandomState(T + B + H + ndir)
    G = ndir * 4 * H
    lens = rng.randint(1, T + 1, size=B)
    lens[0] = T
    mask = (np.arange(T)[:, None] < lens[None, :]).astype(np.float32)        # [T][B]
    dz = (rng.randn(T, B, G) * mask[:, :, None]).astype(np.float32)
    cs = [(rng.randn(T, B, H) * mask[:, :, None]).astype(np.float32) for _ in range(ndir)]
    start = [rng.randn(3, H).astype(np.float32) for _ in range(ndir)]
    dev = torch.device("cuda")
    d_dz = torch.from_numpy(dz).to(dev)
    d_dzs = torch.from_numpy(dz * SCALE).to(dev)
    d_c = [torch.from_numpy(c).to(dev) for c in cs]
    d_dP = [_buf(torch, np.full((3, H), np.nan, np.float32)) for _ in range(ndir)]
    nbytes = lib.ctcb_lstm_peephole_grad_workspace_bytes(T, B, H, ndir)
    ws = torch.zeros(nbytes, dtype=torch.uint8, device=dev)
    st = torch.cuda.current_stream().cuda_stream
    cB, dPb = (None, None) if ndir == 1 else (d_c[1].data_ptr(), d_dP[1][1].data_ptr())

    def run(acc, z=d_dz):
        check(lib.ctcb_lstm_peephole_grad_f32(T, B, H, z.data_ptr(), d_c[0].data_ptr(), cB, d_dP[0][1].data_ptr(),
                                              dPb, acc, ws.data_ptr(), nbytes, st))
        torch.cuda.synchronize()
        return [x[1].cpu().numpy().copy() for x in d_dP]

    first = run(0)
    again = run(0)
    scaled = run(0, d_dzs)
    for (_, v), s in zip(d_dP, start):
        v.copy_(torch.from_numpy(s))
    added = run(1)
    assert all(_guards_intact(w) for w, _ in d_dP), "dP's guard bands changed"
    n = T * B
    K = 128 + 8 + (n + 1023) // 1024 + 1
    worst = 0.0
    for d in range(ndir):
        blk = dz[:, :, d * 4 * H:(d + 1) * 4 * H].astype(np.float64)
        c = cs[d].astype(np.float64)
        cprev = np.zeros_like(c)
        if d == 0:
            cprev[1:] = c[:-1]
        else:
            cprev[:-1] = c[1:]
        terms = [blk[:, :, :H] * cprev, blk[:, :, H:2 * H] * cprev, blk[:, :, 3 * H:] * c]
        want = np.stack([x.sum(axis=(0, 1)) for x in terms])
        S = np.stack([np.abs(x).sum(axis=(0, 1)) for x in terms]) + 1e-30
        worst = max(worst, float(np.max(np.abs(first[d] - want) / (K * U32 * S))))
        assert _same(first[d], again[d])
        assert _same(added[d], first[d] + start[d])
        assert _same(scaled[d], first[d] * SCALE)
    print(json.dumps({"peephole_grad_T%d_B%d_H%d_%s" % (T, B, H, "bi" if ndir == 2 else "uni"):
                      dict(ratio_to_bound=worst, bound_C=K)}))
    assert worst <= 1.0
