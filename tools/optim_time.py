"""What the optimiser update costs: Nesterov against AdaGrad and Adam.

  1. The update kernels alone at the C2, C3 and C4 parameter counts, CUDA events over --launches launches after a
     warm-up: Nesterov's look-ahead axpy plus its fused update (32 B per parameter), AdaGrad (20 B) and Adam (28 B),
     the three alternated over two rounds.  Bytes over time is reported against the data sheet's 3.35 TB/s.
  2. Whole optimisation steps (sgd.SGD.step_device: CUDA graph replay, host packing and upload included as SGD.run does
     it) at C2 and C3 with each rule, alternated over two rounds after a warm-up.
The card's name, power limit and max SM clock are read in the same run.  Prints one JSON object (and writes it to --out).

    python tools/optim_time.py [--launches 200] [--steps 20] [--warmup 6] [--out FILE]
"""
import argparse
import ctypes
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "stanford-ctc_b200"), os.path.join(ROOT, "tools")]

import numpy as np  # noqa: E402

from accum_time import card_info, make_batch, one_step, time_steps  # noqa: E402

SHAPES = {"c2": dict(D=41, K=62, H=512, N=2, tl=1, T=200, L=30, B=32),
          "c3": dict(D=41, K=32, H=1024, N=3, tl=2, T=800, L=100, B=128),
          "c4": dict(D=41, K=35, H=2048, N=5, tl=3, T=1500, L=150, B=32)}
RULES = ("nesterov", "adagrad", "adam")
BYTES = {"nesterov": 32, "adagrad": 20, "adam": 28}     # per parameter: reads and writes of w, states and g
HBM_BYTES_PER_S = 3.35e12                                 # H100 SXM data sheet


def param_count(c):
    from _ctcb import lib, BrnnConfig
    cfg = BrnnConfig(c["D"], c["K"], c["H"], c["N"], c["tl"], c["T"], c["B"], c["L"], 0.0, 20.0, 0)
    return int(lib.ctcb_brnn_param_count(ctypes.byref(cfg)))


def kernel_arms(torch, n):
    """One closure per rule that enqueues that rule's update launches over n parameters on the current stream."""
    from _ctcb import lib, check, ptr, current_stream
    f = lambda: torch.randn(n, device="cuda") * 1e-3
    w, g = f(), f()
    s1, s2 = f(), f().abs()
    gn = torch.tensor([1.0], device="cuda")
    nv = torch.tensor([4.0], device="cuda")
    step = torch.tensor([5], dtype=torch.int64, device="cuda")
    st = current_stream()

    def nesterov():
        check(lib.ctcb_axpy_f32(ptr(w), ptr(s1), 0.9, n, st))
        check(lib.ctcb_sgd_nesterov_step_f32(ptr(w), ptr(s1), ptr(g), n, 0.9, 1e-5, 1500.0, ptr(gn), ptr(nv), st))

    def adagrad():
        check(lib.ctcb_adagrad_step_f32(ptr(w), ptr(s2), ptr(g), n, 1e-5, 1500.0, ptr(gn), ptr(nv), ptr(step), st))

    def adam():
        check(lib.ctcb_adam_step_f32(ptr(w), ptr(s1), ptr(s2), ptr(g), n, 1e-5, 0.9, 0.999, 1e-8, 1500.0, ptr(gn),
                                     ptr(nv), ptr(step), st))
    return {"nesterov": nesterov, "adagrad": adagrad, "adam": adam}, (w, g, s1, s2)


def time_kernel(torch, fn, launches):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(launches):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / launches


def make_opt(c, rule):
    import nnets.brnnet as rnnet
    import sgd
    np.random.seed(33)
    nn = rnnet.NNet(c["D"], c["K"], c["H"], c["N"], c["T"], temporalLayer=c["tl"], maxUtts=c["B"], maxLabels=c["L"])
    nn.initParams()
    opt = sgd.SGD(nn, c["T"], alpha=1e-5, optimizer=rule, momentum=0.9, batchSize=c["B"], verbose=False)
    opt.it = 11                      # past the momentum warm-up: one step shape
    return nn, opt


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=6)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("optim_time.py measures on the GPU; no CUDA device is visible")
    torch.cuda.set_device(0)
    res = {"card": card_info(torch), "launches": args.launches, "steps": args.steps, "warmup": args.warmup,
           "kernels": {}, "steps_ms": {}}
    stream = torch.cuda.Stream()          # a stream of our own, as SGD.run uses (graphs need one)
    with torch.cuda.stream(stream):
        for name in ("c2", "c3", "c4"):
            n = param_count(SHAPES[name])
            arms, bufs = kernel_arms(torch, n)
            for fn in arms.values():
                time_kernel(torch, fn, 10)
            rec = {r: [] for r in RULES}
            for _ in range(2):
                for r in RULES:
                    rec[r].append(time_kernel(torch, arms[r], args.launches))
            out = {"params": n}
            for r in RULES:
                best = min(rec[r])
                out[r] = dict(ms=[round(x, 5) for x in rec[r]], bytes_per_param=BYTES[r],
                              TB_per_s=round(BYTES[r] * n / (best * 1e-3) / 1e12, 3),
                              fraction_of_3_35_TB_per_s=round(BYTES[r] * n / (best * 1e-3) / HBM_BYTES_PER_S, 3))
            res["kernels"][name] = out
            del arms, bufs
            torch.cuda.synchronize()
            torch.cuda.empty_cache()
        for name in ("c2", "c3"):
            c = SHAPES[name]
            datas, labels = make_batch(c, c["B"], seed=33)
            arms = {r: make_opt(c, r) for r in RULES}
            for nn, opt in arms.values():
                for _ in range(args.warmup):
                    one_step(opt, datas, labels)
            rec = {r: [] for r in RULES}
            for _ in range(2):
                for r, (nn, opt) in arms.items():
                    rec[r].append(time_steps(torch, opt, datas, labels, args.steps))
            out = {"shape": c}
            for r, (nn, opt) in arms.items():
                out[r] = dict(ms_per_step_device=[round(x[0], 4) for x in rec[r]],
                              ms_per_step_wall=[round(x[1], 4) for x in rec[r]],
                              params_finite=bool(torch.isfinite(nn.params).all()))
            res["steps_ms"][name] = out
            del arms, nn, opt
            torch.cuda.synchronize()
            torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
