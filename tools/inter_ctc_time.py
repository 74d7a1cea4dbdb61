"""What the intermediate CTC loss costs a training step.

Two shapes: C2 (H=512, numLayers=2, temporalLayer=1, B=32, T=200, D=41, K=62, |l|=30) with the loss at layer 1, its
temporal layer, and C3 (H=1024, numLayers=3, temporalLayer=2, B=128, T=800, D=41, K=32, |l|=100) with the loss at layer
1, a ReLU layer, and at layer 2, its temporal layer; each against the same net without the loss (interWeight 0.3 where
on).  Each arm is timed over whole optimisation steps (sgd.SGD.step_device: CUDA graph replay, host packing and upload
included as SGD.run does it), the arms alternated over two rounds after a warm-up; then one eager pass per arm with the
per-phase events of ctcb_profile_* splits the step (the head's phases are inter_ctc, inter_ctc_delta, inter_ctc_dw).
The card's name, power limit and clock are read in the same run.  Prints one JSON object (and writes it to --out).

    python tools/inter_ctc_time.py [--steps 5] [--warmup 4] [--shapes c2,c3] [--out FILE]
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

SHAPES = {
    "c2": dict(D=41, K=62, H=512, N=2, tl=1, T=200, L=30, B=32, layers=(1,)),
    "c3": dict(D=41, K=32, H=1024, N=3, tl=2, T=800, L=100, B=128, layers=(1, 2)),
}
WEIGHT = 0.3


def make_opt(c, m):
    import nnets.brnnet as rnnet
    import sgd
    np.random.seed(33)
    nn = rnnet.NNet(c["D"], c["K"], c["H"], c["N"], c["T"], temporalLayer=c["tl"], maxUtts=c["B"], maxLabels=c["L"],
                    interLayer=m, interWeight=WEIGHT if m else 0.0)
    nn.initParams()
    opt = sgd.SGD(nn, c["T"], alpha=1e-5, momentum=0.9, batchSize=c["B"], verbose=False)
    opt.it = 11                      # past the momentum warm-up: one step shape
    return nn, opt


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=4)
    ap.add_argument("--shapes", default="c2,c3")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from _ctcb import lib
    if not torch.cuda.is_available():
        raise SystemExit("inter_ctc_time.py measures on the GPU; no CUDA device is visible")
    torch.cuda.set_device(0)
    res = {"card": card_info(torch), "steps": args.steps, "warmup": args.warmup, "interWeight": WEIGHT, "shapes": {}}
    stream = torch.cuda.Stream()          # a stream of our own, as SGD.run uses (graphs need one)
    for name in args.shapes.split(","):
        c = SHAPES[name]
        datas, labels = make_batch(c, c["B"], seed=33)
        out = {}
        with torch.cuda.stream(stream):
            arms = {"off": make_opt(c, 0)}
            arms.update(("inter_m%d" % m, make_opt(c, m)) for m in c["layers"])
            for arm, (nn, opt) in arms.items():
                for _ in range(args.warmup):
                    one_step(opt, datas, labels)
            rec = {arm: [] for arm in arms}
            for _ in range(2):                   # alternate the arms: two rounds each
                for arm, (nn, opt) in arms.items():
                    rec[arm].append(time_steps(torch, opt, datas, labels, args.steps))
            for arm, (nn, opt) in arms.items():
                out[arm] = dict(ms_per_step_device=[round(r[0], 3) for r in rec[arm]],
                                ms_per_step_wall=[round(r[1], 3) for r in rec[arm]],
                                phases_ms=phase_profile(torch, opt, datas, labels),
                                workspace_bytes=int(lib.ctcb_brnn_workspace_bytes(ctypes.byref(nn._cfg))),
                                params_finite=bool(torch.isfinite(nn.params).all()),
                                sweep_error_flag=float(nn.record[3]))
            base = min(r[0] for r in rec["off"])
            for arm in arms:
                if arm != "off":
                    out["%s_over_off_step" % arm] = round(min(r[0] for r in rec[arm]) / base, 4)
        res["shapes"][name] = dict(shape={k: v for k, v in c.items() if k != "layers"}, arms=out)
        del arms
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
