"""What frame subsampling buys: whole steps at k = 1 against k = 2, and the stack / unstack kernels alone.

Three nets: C2 (H=512, numLayers=2, temporalLayer=1, B=32, T=200), C3 (H=1024, numLayers=3, temporalLayer=2, B=128,
T=800) and C2 with LSTM temporal layers, each built at k = 1 and at k = 2 with subsampleLayer = 1 and = temporalLayer.
Each arm is timed over whole optimisation steps (sgd.SGD.step_device: CUDA graph replay, host packing and upload
included as SGD.run does it), the arms alternated over two rounds after a warm-up; then the per-phase split of one eager
step (CUDA events inside the library) and the training workspace of each arm.  Then ctcb_frame_stack_f32 and
ctcb_frame_unstack_f32 alone at C3's size (102400 rows of 1024 units, k = 2) over --launches launches between CUDA
events; their bytes are one read and one write of every element (4 B each) and bytes/s is those over the kernel time,
against the H100 SXM data sheet's 3.35 TB/s.  The card's name, power limit and clock are read in the same run.  Prints
one JSON object (and writes it to --out).

    python tools/subsample_time.py [--steps 5] [--warmup 3] [--launches 100] [--nets c2,c3,c2_lstm] [--out FILE]
"""
import argparse
import ctypes
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "stanford-ctc_b200"), os.path.join(ROOT, "tools")]

import numpy as np  # noqa: E402

from accum_time import card_info, make_batch, one_step, phase_profile, time_steps  # noqa: E402

NETS = {
    "c2": dict(D=41, K=62, H=512, N=2, tl=1, T=200, L=30, B=32),
    "c3": dict(D=41, K=32, H=1024, N=3, tl=2, T=800, L=100, B=128),
    "c2_lstm": dict(D=41, K=62, H=512, N=2, tl=1, T=200, L=30, B=32, cell="lstm"),
}
HBM_TBPS = 3.35


def make_opt(c, k, sl):
    import nnets.brnnet as rnnet
    import sgd
    np.random.seed(33)
    nn = rnnet.NNet(c["D"], c["K"], c["H"], c["N"], c["T"], temporalLayer=c["tl"], maxUtts=c["B"], maxLabels=c["L"],
                    cell=c.get("cell", "relu"), subsample=k, subsampleLayer=sl)
    nn.initParams()
    opt = sgd.SGD(nn, c["T"], alpha=1e-5, momentum=0.9, batchSize=c["B"], verbose=False)
    opt.it = 11                      # past the momentum warm-up: one step shape
    return nn, opt


def time_kernels(torch, T, B, n, k, launches):
    """Each kernel alone at [T][B][n] <-> [ceil(T/k)][B][k n], best of three windows of `launches` launches."""
    from _ctcb import lib, check
    Tp = -(-T // k)
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.randn(T * B * n, device="cuda", generator=g)
    s = torch.empty(Tp * B * k * n, device="cuda")
    d = torch.empty_like(x)
    lens = torch.full((B,), T, dtype=torch.int32, device="cuda")
    tp = torch.empty(B, dtype=torch.int32, device="cuda")
    st = torch.cuda.current_stream().cuda_stream

    def stack():
        check(lib.ctcb_frame_stack_f32(x.data_ptr(), lens.data_ptr(), T, B, n, k, s.data_ptr(), tp.data_ptr(), st))

    def unstack():
        check(lib.ctcb_frame_unstack_f32(s.data_ptr(), lens.data_ptr(), T, B, n, k, d.data_ptr(), st))

    out = {}
    for name, fn in (("stack", stack), ("unstack", unstack)):
        nbytes = 4 * (T * B * n + Tp * B * k * n)
        for _ in range(10):
            fn()
        best = None
        for _ in range(3):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(launches):
                fn()
            e1.record()
            e1.synchronize()
            ms = e0.elapsed_time(e1) / launches
            best = ms if best is None else min(best, ms)
        tbps = nbytes / (best * 1e-3) / 1e12
        out[name] = dict(us=round(best * 1e3, 2), bytes=nbytes, TBps=round(tbps, 3),
                         share_of_3_35=round(tbps / HBM_TBPS, 3))
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--launches", type=int, default=100)
    ap.add_argument("--nets", default="c2,c3,c2_lstm")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("subsample_time.py measures on the GPU; no CUDA device is visible")
    torch.cuda.set_device(0)
    from _ctcb import lib
    res = {"card": card_info(torch), "steps": args.steps, "warmup": args.warmup, "launches": args.launches,
           "nets": {}}
    stream = torch.cuda.Stream()          # a stream of our own, as SGD.run uses (graphs need one)
    for name in args.nets.split(","):
        c = NETS[name]
        datas, labels = make_batch(c, c["B"], seed=33)
        arms = {"k1": (1, 1), "k2_L1": (2, 1), "k2_Ltl": (2, c["tl"])}
        out = {}
        with torch.cuda.stream(stream):
            opts = {a: make_opt(c, *kl) for a, kl in arms.items()}
            for a, (nn, opt) in opts.items():
                for _ in range(args.warmup):
                    one_step(opt, datas, labels)
            rec = {a: [] for a in opts}
            for _ in range(2):                   # alternate the arms: two rounds each
                for a, (nn, opt) in opts.items():
                    rec[a].append(time_steps(torch, opt, datas, labels, args.steps))
            for a, (nn, opt) in opts.items():
                out[a] = dict(ms_per_step_device=[round(r[0], 3) for r in rec[a]],
                              ms_per_step_wall=[round(r[1], 3) for r in rec[a]],
                              workspace_bytes=int(lib.ctcb_brnn_workspace_bytes(ctypes.byref(nn._cfg))),
                              phases_ms=phase_profile(torch, opt, datas, labels),
                              params_finite=bool(torch.isfinite(nn.params).all()))
            base = min(r[0] for r in rec["k1"])
            for a in ("k2_L1", "k2_Ltl"):
                out[a]["over_k1_step"] = round(min(r[0] for r in rec[a]) / base, 4)
            del opts
            torch.cuda.empty_cache()
        res["nets"][name] = dict(shape=c, arms=out)
    with torch.cuda.stream(stream):
        c = NETS["c3"]
        res["kernels_c3"] = time_kernels(torch, c["T"], c["B"], c["H"], 2, args.launches)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
