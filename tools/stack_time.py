"""What each stacked temporal layer costs.

A C3-shaped step (H=1024, numLayers=3, B=128, T=800, D=41, K=32, |l|=100) with one block of 1, 2 and 3 temporal layers
starting at layer 1 (3 = every hidden layer, so that block ends at the top: allowTopTemporal), all at the same
numLayers.  Each arm is timed over whole optimisation steps (sgd.SGD.step_device: CUDA graph replay, host packing and
upload included as SGD.run does it), the arms alternated over two rounds after a warm-up; then one eager pass per arm
with the per-phase events of ctcb_profile_* shows where the time goes.  The card's name, power limit and clock are read
in the same run.  Prints one JSON object (and writes it to --out).

    python tools/stack_time.py [--steps 5] [--warmup 4] [--out FILE]
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

C3 = dict(D=41, K=32, H=1024, N=3, T=800, L=100, B=128)
TL = 1


def make_opt(c, k):
    import nnets.brnnet as rnnet
    import sgd
    np.random.seed(33)
    nn = rnnet.NNet(c["D"], c["K"], c["H"], c["N"], c["T"], temporalLayer=TL, numTemporal=k, maxUtts=c["B"],
                    maxLabels=c["L"], allowTopTemporal=True)
    nn.initParams()
    opt = sgd.SGD(nn, c["T"], alpha=1e-5, momentum=0.9, batchSize=c["B"], verbose=False)
    opt.it = 11                      # past the momentum warm-up: one step shape
    return nn, opt


def workspace_bytes(nn):
    from _ctcb import lib
    return int(lib.ctcb_brnn_workspace_bytes(ctypes.byref(nn._cfg)))


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=4)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("stack_time.py measures on the GPU; no CUDA device is visible")
    torch.cuda.set_device(0)
    res = {"card": card_info(torch), "shape": dict(C3, temporalLayer=TL), "steps": args.steps, "warmup": args.warmup}
    datas, labels = make_batch(C3, C3["B"], seed=33)
    stream = torch.cuda.Stream()          # a stream of our own, as SGD.run uses (graphs need one)
    out = {}
    with torch.cuda.stream(stream):
        arms = {k: make_opt(C3, k) for k in (1, 2, 3)}
        for k, (nn, opt) in arms.items():
            for _ in range(args.warmup):
                one_step(opt, datas, labels)
        rec = {k: [] for k in arms}
        for _ in range(2):                   # alternate the arms: two rounds each
            for k, (nn, opt) in arms.items():
                rec[k].append(time_steps(torch, opt, datas, labels, args.steps))
        for k, (nn, opt) in arms.items():    # where the time goes: per-phase events, an untimed eager pass
            out[k] = dict(ms_per_step_device=[round(r[0], 3) for r in rec[k]],
                          ms_per_step_wall=[round(r[1], 3) for r in rec[k]],
                          phases_ms=phase_profile(torch, opt, datas, labels),
                          workspace_bytes=workspace_bytes(nn), params_finite=bool(torch.isfinite(nn.params).all()),
                          sweep_error_flag=float(nn.record[3]))
        best1 = min(r[0] for r in rec[1])
        for k in (2, 3):
            out[k]["extra_ms_per_layer_vs_k1"] = round((min(r[0] for r in rec[k]) - best1) / (k - 1), 3)
    res["arms"] = out
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
