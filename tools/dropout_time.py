"""What inverted dropout on the ReLU hidden layers costs per optimisation step.

C2 (H=512, numLayers=2, temporalLayer=1, B=32, T=200: one dropped layer) and C3 (H=1024, numLayers=3, temporalLayer=2,
B=128, T=800: two dropped layers), each with p = 0 and p = 0.1.  Each arm is timed over whole optimisation steps
(sgd.SGD.step_device: CUDA graph replay, host packing and upload included as SGD.run does it, the dropout counter
advanced inside the graph), the arms alternated over two rounds after a warm-up; then one eager pass per arm with the
per-phase events of ctcb_profile_* (the "dropout" phase is the mask kernel).  The card's name, power limit and clock
are read in the same run.  Prints one JSON object (and writes it to --out).

    python tools/dropout_time.py [--steps 20] [--warmup 6] [--out FILE]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "stanford-ctc_b200"), os.path.join(ROOT, "tools")]

import numpy as np  # noqa: E402

from accum_time import card_info, make_batch, one_step, phase_profile, time_steps  # noqa: E402

SHAPES = {"c2": dict(D=41, K=62, H=512, N=2, tl=1, T=200, L=30, B=32),
          "c3": dict(D=41, K=32, H=1024, N=3, tl=2, T=800, L=100, B=128)}


def make_opt(c, p):
    import nnets.brnnet as rnnet
    import sgd
    np.random.seed(33)
    nn = rnnet.NNet(c["D"], c["K"], c["H"], c["N"], c["T"], temporalLayer=c["tl"], maxUtts=c["B"], maxLabels=c["L"],
                    dropout=p)
    nn.initParams()
    opt = sgd.SGD(nn, c["T"], alpha=1e-5, momentum=0.9, batchSize=c["B"], verbose=False)
    opt.it = 11                      # past the momentum warm-up: one step shape
    return nn, opt


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=6)
    ap.add_argument("--shapes", default="c2,c3")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("dropout_time.py measures on the GPU; no CUDA device is visible")
    torch.cuda.set_device(0)
    res = {"card": card_info(torch), "steps": args.steps, "warmup": args.warmup}
    stream = torch.cuda.Stream()          # a stream of our own, as SGD.run uses (graphs need one)
    with torch.cuda.stream(stream):
        for name in args.shapes.split(","):
            c = SHAPES[name]
            datas, labels = make_batch(c, c["B"], seed=33)
            arms = {p: make_opt(c, p) for p in (0.0, 0.1)}
            for nn, opt in arms.values():
                for _ in range(args.warmup):
                    one_step(opt, datas, labels)
            rec = {p: [] for p in arms}
            for _ in range(2):                   # alternate the arms: two rounds each
                for p, (nn, opt) in arms.items():
                    rec[p].append(time_steps(torch, opt, datas, labels, args.steps))
            out = {"shape": c}
            for p, (nn, opt) in arms.items():
                out["p=%g" % p] = dict(ms_per_step_device=[round(r[0], 4) for r in rec[p]],
                                       ms_per_step_wall=[round(r[1], 4) for r in rec[p]],
                                       phases_ms=phase_profile(torch, opt, datas, labels),
                                       params_finite=bool(torch.isfinite(nn.params).all()))
            best0, best1 = (min(r[0] for r in rec[p]) for p in (0.0, 0.1))
            out["extra_ms_per_step"] = round(best1 - best0, 4)
            out["extra_fraction"] = round(best1 / best0 - 1.0, 4)
            res[name] = out
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
