"""What self-conditioned CTC costs a training step and a forward-only call, over the intermediate CTC loss alone.

The shapes of tools/inter_ctc_time.py: C2 (H=512, numLayers=2, temporalLayer=1, B=32, T=200, D=41, K=62, |l|=30) with
m = 1, its temporal layer, and C3 (H=1024, numLayers=3, temporalLayer=2, B=128, T=800, D=41, K=32, |l|=100) with m = 1, a
ReLU layer below the temporal one, and m = 2, the temporal layer; at each m the InterCTC net (interWeight 0.3) against
the same net with selfCondition (W_c, b_c drawn non-zero, so no path is skipped).  Each arm is timed over whole
optimisation steps (sgd.SGD.step_device: CUDA graph replay, host packing and upload included as SGD.run does it) and
over forwardBatch of the step's utterances (host packing, upload and the copy of the probabilities included), the arms
alternated over two rounds after a warm-up; then one eager pass per arm with the per-phase events of ctcb_profile_*
splits the step (the conditioning's phases are self_cond and self_cond_bwd).  The card's name, power limit and clock
are read in the same run.  Prints one JSON object (and writes it to --out).

    python tools/self_cond_time.py [--steps 5] [--warmup 4] [--shapes c2,c3] [--out FILE]
"""
import argparse
import ctypes
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "stanford-ctc_b200"), os.path.join(ROOT, "tools")]

import numpy as np  # noqa: E402

from accum_time import card_info, make_batch, one_step, phase_profile, time_steps  # noqa: E402
from inter_ctc_time import SHAPES, WEIGHT  # noqa: E402


def make_opt(c, m, cond):
    import nnets.brnnet as rnnet
    import sgd
    import torch
    np.random.seed(33)
    nn = rnnet.NNet(c["D"], c["K"], c["H"], c["N"], c["T"], temporalLayer=c["tl"], maxUtts=c["B"], maxLabels=c["L"],
                    interLayer=m, interWeight=WEIGHT, selfCondition=cond)
    nn.initParams()
    if cond:
        rng = np.random.RandomState(5)
        nn.stack[-1][0].copy_(torch.from_numpy(rng.uniform(-0.05, 0.05, tuple(nn.stack[-1][0].shape)).astype(np.float32)))
        nn.stack[-1][1].copy_(torch.from_numpy(rng.uniform(-0.05, 0.05, tuple(nn.stack[-1][1].shape)).astype(np.float32)))
    opt = sgd.SGD(nn, c["T"], alpha=1e-5, momentum=0.9, batchSize=c["B"], verbose=False)
    opt.it = 11                      # past the momentum warm-up: one step shape
    return nn, opt


def time_forward(torch, nn, datas, calls):
    """ms per forwardBatch call of the step's utterances (it ends in a synchronisation)."""
    t0 = time.perf_counter()
    for _ in range(calls):
        nn.forwardBatch(datas)
    return (time.perf_counter() - t0) * 1e3 / calls


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
        raise SystemExit("self_cond_time.py measures on the GPU; no CUDA device is visible")
    torch.cuda.set_device(0)
    res = {"card": card_info(torch), "steps": args.steps, "warmup": args.warmup, "interWeight": WEIGHT, "shapes": {}}
    stream = torch.cuda.Stream()          # a stream of our own, as SGD.run uses (graphs need one)
    for name in args.shapes.split(","):
        c = SHAPES[name]
        datas, labels = make_batch(c, c["B"], seed=33)
        out = {}
        with torch.cuda.stream(stream):
            arms = {}
            for m in c["layers"]:
                arms["inter_m%d" % m] = make_opt(c, m, False)
                arms["cond_m%d" % m] = make_opt(c, m, True)
            for arm, (nn, opt) in arms.items():
                for _ in range(args.warmup):
                    one_step(opt, datas, labels)
                nn.forwardBatch(datas)
            rec = {arm: [] for arm in arms}
            fwd = {arm: [] for arm in arms}
            for _ in range(2):                   # alternate the arms: two rounds each
                for arm, (nn, opt) in arms.items():
                    rec[arm].append(time_steps(torch, opt, datas, labels, args.steps))
                    fwd[arm].append(time_forward(torch, nn, datas, args.steps))
            for arm, (nn, opt) in arms.items():
                out[arm] = dict(ms_per_step_device=[round(r[0], 3) for r in rec[arm]],
                                ms_per_step_wall=[round(r[1], 3) for r in rec[arm]],
                                ms_per_forward_batch=[round(x, 3) for x in fwd[arm]],
                                phases_ms=phase_profile(torch, opt, datas, labels),
                                workspace_bytes=int(lib.ctcb_brnn_workspace_bytes(ctypes.byref(nn._cfg))),
                                forward_workspace_bytes=int(lib.ctcb_brnn_forward_workspace_bytes(
                                    ctypes.byref(nn._cfg), None)),
                                params_finite=bool(torch.isfinite(nn.params).all()),
                                sweep_error_flag=float(nn.record[3]))
            for m in c["layers"]:
                a, b = "cond_m%d" % m, "inter_m%d" % m
                out["%s_over_%s_step" % (a, b)] = round(min(r[0] for r in rec[a]) / min(r[0] for r in rec[b]), 4)
                out["%s_over_%s_forward" % (a, b)] = round(min(fwd[a]) / min(fwd[b]), 4)
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
