"""What the Gaussian weight noise costs per optimisation step, and the noise pass on its own.

Shapes: C2 and C3 of bench.py, sigma = 0.075.  Each arm, without and with noise, is timed over whole optimisation steps
(sgd.SGD.step_device: CUDA graph replay, host packing and upload included as SGD.run does it, the step counter advanced
inside the graph), the arms alternated over two rounds after a warm-up.  The pass alone (ctcb_brnn_weight_noise_f32 on
the flat vector) is timed at the C2, C3 and C4 parameter counts with CUDA events around replays of one CUDA graph of
back-to-back launches, and set against the bytes it must move, 2 P 4 (one read and one write of the vector); the
"weight_noise" phase of one eager noisy step (ctcb_profile_*) times it inside the step.  The card's name, power limit
and clock are read in the same run.  Prints one JSON object (and writes it to --out).

    python tools/weight_noise_time.py [--steps 20] [--warmup 6] [--out FILE]
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

SHAPES = {"c2": dict(D=41, K=62, H=512, N=2, tl=1, T=200, L=30, B=32),
          "c3": dict(D=41, K=32, H=1024, N=3, tl=2, T=800, L=100, B=128),
          "c4": dict(D=41, K=35, H=2048, N=5, tl=3, T=1500, L=150, B=256)}
SIGMA = 0.075
HBM_TBS = 3.35          # H100 SXM data-sheet HBM3 bandwidth


def make_opt(c, noise):
    import nnets.brnnet as rnnet
    import sgd
    np.random.seed(33)
    nn = rnnet.NNet(c["D"], c["K"], c["H"], c["N"], c["T"], temporalLayer=c["tl"], maxUtts=c["B"], maxLabels=c["L"],
                    weightNoise=SIGMA if noise else 0.0)
    nn.initParams()
    opt = sgd.SGD(nn, c["T"], alpha=1e-5, momentum=0.9, batchSize=c["B"], verbose=False)
    opt.it = 11                      # past the momentum warm-up: one step shape
    return nn, opt


def time_pass(torch, c, reps=50, replays=20):
    """Microseconds per launch of the pass alone on the shape's flat vector, and the HBM rate that implies.  The handle
    is laid out for one frame of one utterance: the pass depends on the parameter vector only."""
    import _ctcb
    from _ctcb import lib, check, ptr
    cfg = _ctcb.BrnnConfig(c["D"], c["K"], c["H"], c["N"], c["tl"], 1, 1, 1, 0.0, 20.0)
    cfg.weightNoise = 1
    h = ctypes.c_void_p()
    check(lib.ctcb_brnn_create(ctypes.byref(cfg), ctypes.byref(h)))
    P = int(lib.ctcb_brnn_param_count(ctypes.byref(cfg)))
    x = torch.randn(P, device="cuda")
    y = torch.empty_like(x)
    step = torch.zeros(1, dtype=torch.int64, device="cuda")
    check(lib.ctcb_brnn_set_weight_noise(h, SIGMA, 33, ptr(step)))
    st = _ctcb.current_stream()

    def launch():
        check(lib.ctcb_brnn_weight_noise_f32(h, ptr(x), ptr(y), st))
    try:
        for _ in range(5):
            launch()
        torch.cuda.synchronize()
        check(lib.ctcb_graph_capture_begin(st))
        try:
            for _ in range(reps):
                launch()
        finally:
            g = ctypes.c_void_p()
            rc = lib.ctcb_graph_capture_end(st, ctypes.byref(g))
        check(rc)
        check(lib.ctcb_graph_launch(g, st))
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(replays):
            check(lib.ctcb_graph_launch(g, st))
        e1.record()
        torch.cuda.synchronize()
        lib.ctcb_graph_destroy(g)
    finally:
        lib.ctcb_brnn_destroy(h)
    us = 1e3 * e0.elapsed_time(e1) / (reps * replays)
    nbytes = 2 * P * 4
    return dict(params=P, us=round(us, 2), bytes=nbytes, tb_per_s=round(nbytes / us * 1e-6, 3),
                datasheet_bound_us=round(nbytes / (HBM_TBS * 1e6), 2))


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=6)
    ap.add_argument("--shapes", default="c2,c3")
    ap.add_argument("--pass-shapes", default="c2,c3,c4")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("weight_noise_time.py measures on the GPU; no CUDA device is visible")
    torch.cuda.set_device(0)
    res = {"card": card_info(torch), "steps": args.steps, "warmup": args.warmup, "sigma": SIGMA}
    stream = torch.cuda.Stream()          # a stream of our own, as SGD.run uses (graphs need one)
    with torch.cuda.stream(stream):
        for name in [s for s in args.shapes.split(",") if s]:
            c = SHAPES[name]
            datas, labels = make_batch(c, c["B"], seed=33)
            arms = {m: make_opt(c, m) for m in (False, True)}
            for nn, opt in arms.values():
                for _ in range(args.warmup):
                    one_step(opt, datas, labels)
            rec = {m: [] for m in arms}
            for _ in range(2):                   # alternate the arms: two rounds each
                for m, (nn, opt) in arms.items():
                    rec[m].append(time_steps(torch, opt, datas, labels, args.steps))
            out = {"shape": c}
            for m, (nn, opt) in arms.items():
                out["noise" if m else "plain"] = dict(ms_per_step_device=[round(r[0], 4) for r in rec[m]],
                                                      ms_per_step_wall=[round(r[1], 4) for r in rec[m]],
                                                      phases_ms=phase_profile(torch, opt, datas, labels),
                                                      params_finite=bool(torch.isfinite(nn.params).all()))
            best0, best1 = (min(r[0] for r in rec[m]) for m in (False, True))
            out["extra_ms_per_step"] = round(best1 - best0, 4)
            out["extra_fraction"] = round(best1 / best0 - 1.0, 4)
            del arms, nn, opt
            torch.cuda.synchronize()
            torch.cuda.empty_cache()
            res[name] = out
        res["pass_alone"] = {name: time_pass(torch, SHAPES[name]) for name in args.pass_shapes.split(",") if name}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
