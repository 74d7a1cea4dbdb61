"""What an LSTM step costs, against the clipped-ReLU step of the same net.

Two shapes: C2 (H=512, numLayers=2, temporalLayer=1, B=32, T=200, D=41, K=62, |l|=30) and C3 (H=1024, numLayers=3,
temporalLayer=2, B=128, T=800, D=41, K=32, |l|=100), each built with cell='relu' and cell='lstm'.  Each arm is timed
over whole optimisation steps (sgd.SGD.step_device: CUDA graph replay, host packing and upload included as SGD.run
does it), the arms alternated over two rounds after a warm-up; then one eager pass per arm with the per-phase events
of ctcb_profile_* gives the two sweeps alone (sweep_fwd, sweep_bptt) and the rest of the step.  The card's name, power
limit and clock are read in the same run.  Prints one JSON object (and writes it to --out).  With --peephole the two
arms are the LSTM net without and with peephole connections (peephole=True), and the ratio is theirs.  With --zoneout
the two arms are the LSTM net without and with zoneout (zoneoutCell=0.15, zoneoutHidden=0.05).

    python tools/lstm_time.py [--steps 5] [--warmup 4] [--shapes c2,c3] [--peephole | --zoneout] [--out FILE]
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
    "c2": dict(D=41, K=62, H=512, N=2, tl=1, T=200, L=30, B=32),
    "c3": dict(D=41, K=32, H=1024, N=3, tl=2, T=800, L=100, B=128),
}


def make_opt(c, cell, peephole=False, zoneout=False):
    import nnets.brnnet as rnnet
    import sgd
    np.random.seed(33)
    z = dict(zoneoutCell=0.15, zoneoutHidden=0.05) if zoneout else {}
    nn = rnnet.NNet(c["D"], c["K"], c["H"], c["N"], c["T"], temporalLayer=c["tl"], maxUtts=c["B"], maxLabels=c["L"],
                    cell=cell, peephole=peephole, **z)
    nn.initParams()
    opt = sgd.SGD(nn, c["T"], alpha=1e-5, momentum=0.9, batchSize=c["B"], verbose=False)
    opt.it = 11                      # past the momentum warm-up: one step shape
    return nn, opt


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=4)
    ap.add_argument("--shapes", default="c2,c3")
    ap.add_argument("--peephole", action="store_true", help="time LSTM with peepholes against LSTM without")
    ap.add_argument("--zoneout", action="store_true", help="time LSTM with zoneout against LSTM without")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from _ctcb import lib
    if not torch.cuda.is_available():
        raise SystemExit("lstm_time.py measures on the GPU; no CUDA device is visible")
    torch.cuda.set_device(0)
    res = {"card": card_info(torch), "steps": args.steps, "warmup": args.warmup, "shapes": {}}
    stream = torch.cuda.Stream()          # a stream of our own, as SGD.run uses (graphs need one)
    for name in args.shapes.split(","):
        c = SHAPES[name]
        datas, labels = make_batch(c, c["B"], seed=33)
        out = {}
        with torch.cuda.stream(stream):
            if args.zoneout:
                kinds = {"lstm": ("lstm", False, False), "lstm_zoneout": ("lstm", False, True)}
            elif args.peephole:
                kinds = {"lstm": ("lstm", False), "lstm_peephole": ("lstm", True)}
            else:
                kinds = {"relu": ("relu", False), "lstm": ("lstm", False)}
            arms = {arm: make_opt(c, *kind) for arm, kind in kinds.items()}
            for cell, (nn, opt) in arms.items():
                for _ in range(args.warmup):
                    one_step(opt, datas, labels)
            rec = {cell: [] for cell in arms}
            for _ in range(2):                   # alternate the arms: two rounds each
                for cell, (nn, opt) in arms.items():
                    rec[cell].append(time_steps(torch, opt, datas, labels, args.steps))
            for cell, (nn, opt) in arms.items():
                plan = (ctypes.c_int32 * 4)()
                if cell == "lstm_zoneout":
                    lib.ctcb_debug_lstm_zoneout_plan(c["H"], c["B"], 2, 0, plan)
                elif cell != "relu":
                    lib.ctcb_debug_lstm_plan(c["H"], c["B"], 2, int(kinds[cell][1]), plan)
                out[cell] = dict(ms_per_step_device=[round(r[0], 3) for r in rec[cell]],
                                 ms_per_step_wall=[round(r[1], 3) for r in rec[cell]],
                                 phases_ms=phase_profile(torch, opt, datas, labels),
                                 params=nn.nparams,
                                 workspace_bytes=int(lib.ctcb_brnn_workspace_bytes(ctypes.byref(nn._cfg))),
                                 params_finite=bool(torch.isfinite(nn.params).all()),
                                 sweep_error_flag=float(nn.record[3]),
                                 lstm_plan=dict(KI=plan[0], parts=plan[1], per_sm=plan[2], tiles_per_part=plan[3])
                                 if cell != "relu" else None)
            a, b = list(arms)
            out["%s_over_%s_step" % (b, a)] = round(min(r[0] for r in rec[b]) / min(r[0] for r in rec[a]), 4)
        res["shapes"][name] = dict(shape=c, arms=out)
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
